"""Writes tests/golden/yolov5_loss.npz: the reference YOLOv5Loss (src/losses/yolov5_loss.py:135-278) on the seeded inputs of
oracle/yolov5_train_oracle.loss_fixture_case, in fp32 on the CPU.

  CVPYTORCH_REFERENCE=<reference checkout> python tools/make_golden_yolov5_loss.py

The reference's build_targets does not run on current torch: `gj.clamp_(0, gain[3] - 1)` clamps an int64 tensor in place with float
tensor bounds, which raises "result type Float can't be cast to the desired output type Long".  Older torch converted the bounds to the
tensor's type.  This script does that, and only while it calls the reference: an in-place clamp of an integer tensor gets its tensor
bounds as Python ints (clamp_bounds_as_int).  ref_shim.install() is not changed.

Per case ('a': 3 x 128², 80 classes; 'b': 2 x 96 x 64, 1 class; see LOSS_CASES) it stores the seed and the reference's outputs: loss,
items (lbox, lobj, lcls), the gradients of loss with respect to the three detect outputs, and per level the candidate lists of
build_targets (image, anchor, gj, gi, class; tbox; anchor).  The inputs cover GTs on integer grid coordinates, a border GT, a
ratio-filtered GT, duplicate cells, nc = 1 and an empty image."""
import contextlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import ref_shim  # noqa: E402
from oracle import yolov5_train_oracle as O  # noqa: E402

SEEDS = {'a': 11, 'b': 12}


@contextlib.contextmanager
def clamp_bounds_as_int():
    orig = torch.Tensor.clamp_

    def clamp_(self, min=None, max=None):
        if not self.is_floating_point():
            min, max = (int(v) if isinstance(v, torch.Tensor) else v for v in (min, max))
        return orig(self, min, max)
    torch.Tensor.clamp_ = clamp_
    try:
        yield
    finally:
        torch.Tensor.clamp_ = orig


def reference_run(mod, preds, targets, nc):
    loss = mod.YOLOv5Loss(nc, anchors=O.ANCHORS, device='cpu')
    ps = [p.clone().requires_grad_(True) for p in preds]
    views = [p.view(p.shape[0], 3, 5 + nc, p.shape[2], p.shape[3]).permute(0, 1, 3, 4, 2) for p in ps]
    with clamp_bounds_as_int():
        total, items = loss(views, targets)
        tcls, tbox, indices, anch = loss.build_targets([v.detach() for v in views], targets)
    total.backward()
    cands = [(torch.stack((b, a, gj, gi, c), 1).int(), torch.cat((tb, an), 1)) for (b, a, gj, gi), c, tb, an in zip(indices, tcls, tbox, anch)]
    return total.detach(), items, [p.grad for p in ps], cands


def main():
    ref_shim.install()
    import src.losses.yolov5_loss as mod
    torch.set_num_threads(1)
    res = {}
    for case, seed in SEEDS.items():
        preds, targets = O.loss_fixture_case(seed, case)
        nc = O.LOSS_CASES[case][3]
        total, items, grads, cands = reference_run(mod, preds, targets, nc)
        res[f'{case}_seed'] = np.array(seed)
        res[f'{case}_loss'] = total.numpy().astype(np.float32)
        res[f'{case}_items'] = items.numpy().astype(np.float32)
        for i, g in enumerate(grads):
            res[f'{case}_grad{i}'] = g.numpy().astype(np.float32)
        for i, (ci, cb) in enumerate(cands):
            res[f'{case}_cand_idx{i}'] = ci.numpy()
            res[f'{case}_cand_box{i}'] = cb.numpy().astype(np.float32)
        # the oracle restatement must reproduce the reference before the fixture is written
        ps = [p.clone().requires_grad_(True) for p in preds]
        l2, i2, tg = O.yolov5_loss(ps, targets, torch.tensor(O.ANCHORS), nc)
        l2.backward()
        for (oi, ob), (ci, cb) in zip(O.candidate_lists(tg, preds[0].shape[0]), cands):
            assert torch.equal(oi, ci) and torch.equal(ob, cb)
        worst = max([float((l2.detach() - total).abs() / total.abs()), float(((i2 - items).abs() / items.abs().clamp_min(1e-12)).max())] +
                    [float((p.grad - g).abs().max() / g.abs().max()) for p, g in zip(ps, grads)])
        assert worst <= 1e-6, worst
        print(case, 'seed', seed, 'loss', float(total), 'items', items.tolist(), 'candidates', [int(c[0].shape[0]) for c in cands], 'oracle worst', worst)
    path = os.path.join(ROOT, 'tests', 'golden', 'yolov5_loss.npz')
    np.savez_compressed(path, **res)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
