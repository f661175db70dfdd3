"""Writes tests/golden/yolox_loss.npz: the reference YOLOXLoss (src/losses/det/yolox_loss.py) on the seeded inputs of
oracle/yolox_loss_oracle.fixture_case, in fp32 on the CPU.

  CVPYTORCH_REFERENCE=<reference checkout> python tools/make_golden_yolox_loss.py

Per case ('a': 3 x 128², 3 classes; 'b': 2 x 160², 80 classes) it stores the seed (the first from 1 whose assignment has no near-tie in
float64, oracle.near_ties) and the reference's outputs: the loss terms and num_fg, the foreground mask, matched GT and matched IoU of every
anchor (captured from get_assignments), and the gradients of loss['loss'] with respect to the three head outputs."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import ref_shim  # noqa: E402
from oracle import yolox_loss_oracle as LO  # noqa: E402


def reference_run(mod, preds, targets, nc):
    loss = mod.YOLOXLoss(nc)
    A = sum(p.shape[2] * p.shape[3] for p in preds)
    B = targets.shape[0]
    fg = np.zeros((B, A), bool)
    mg = np.full((B, A), -1, np.int64)
    mi = np.zeros((B, A), np.float32)
    orig = loss.get_assignments

    def capture(batch_idx, *a, **k):
        res = orig(batch_idx, *a, **k)
        _, fg_mask, ious, inds, _ = res
        idx = fg_mask.nonzero()[:, 0].numpy()
        fg[batch_idx, idx] = True
        mg[batch_idx, idx] = inds.numpy()
        mi[batch_idx, idx] = ious.detach().numpy()
        return res
    loss.get_assignments = capture
    ps = [p.clone().requires_grad_(True) for p in preds]
    out = loss(ps, targets)
    out['loss'].backward()
    return out, (fg, mg, mi), [p.grad for p in ps]


def main():
    ref_shim.install()
    import src.losses.det.yolox_loss as mod
    torch.set_num_threads(1)
    res = {}
    for case, (B, H, nc) in LO.CASES.items():
        seed = 1
        while True:
            preds, targets = LO.fixture_case(seed, case)
            if not bool(LO.near_ties(preds, targets, LO.STRIDES, nc).any()):
                break
            seed += 1
        out, (fg, mg, mi), grads = reference_run(mod, preds, targets, nc)
        res[f'{case}_seed'] = np.array(seed)
        for k in ('loss', 'iou_loss', 'conf_loss', 'cls_loss', 'num_fg'):
            res[f'{case}_{k}'] = np.array(float(out[k].detach()), np.float32)
        res[f'{case}_fg'], res[f'{case}_matched_gt'], res[f'{case}_matched_iou'] = fg, mg, mi
        for i, g in enumerate(grads):
            res[f'{case}_grad{i}'] = g.numpy().astype(np.float32)
        dk = [int(m) for m in np.bincount(mg[fg].ravel())] if fg.any() else []
        print(case, 'seed', seed, {k: float(out[k].detach()) for k in ('loss', 'iou_loss', 'conf_loss', 'cls_loss', 'num_fg')}, 'fg', int(fg.sum()),
              'matches per GT row', dk)
    path = os.path.join(ROOT, 'tests', 'golden', 'yolox_loss.npz')
    np.savez_compressed(path, **res)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
