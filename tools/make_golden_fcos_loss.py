"""Writes tests/golden/fcos_loss.npz: the reference FCOSLoss (src/losses/fcos_loss.py) on the seeded inputs of
oracle/fcos_loss_oracle.fixture_case, in fp32 on the CPU.

  CVPYTORCH_REFERENCE=<reference checkout> python tools/make_golden_fcos_loss.py

Per case ('a': 3 x 128², 3 classes; 'b': 1 x 192², 80 classes) it stores the inputs (the 15 head tensors, boxes, labels), the targets
GenTargets returns, the four losses and the gradients of total_loss with respect to the 15 head tensors.  It asserts that the oracle
reproduces them (targets bitwise, losses and gradients within 1e-6 relative) before writing."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import ref_shim  # noqa: E402
from oracle import fcos_loss_oracle as LO  # noqa: E402

NAMES = ('cls', 'cnt', 'reg')
LOSSES = ('cls_loss', 'cnt_loss', 'reg_loss', 'total_loss')


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def reference_run(mod, preds, boxes, labels):
    loss = mod.FCOSLoss()
    captured = {}
    orig = loss.target_layer.forward

    def capture(inputs):
        res = orig(inputs)
        captured['t'] = [r.detach().clone() for r in res]
        return res
    loss.target_layer.forward = capture
    ps = [[t.clone().requires_grad_(True) for t in level] for level in preds]
    out = loss(ps, boxes, labels)
    out[3].backward()
    return out, captured['t'], [[t.grad for t in level] for level in ps]


def main():
    ref_shim.install()
    import src.losses.fcos_loss as mod
    torch.set_num_threads(1)
    res = {}
    for case in LO.CASES:
        seed = 1
        preds, boxes, labels = LO.fixture_case(seed, case)
        out, (cls_t, cnt_t, reg_t), grads = reference_run(mod, preds, boxes, labels)
        # the oracle must reproduce the reference before anything is written
        qs = [[t.clone().requires_grad_(True) for t in level] for level in preds]
        o_out, (o_cls, o_cnt, o_reg, o_mg) = LO.losses(qs, boxes, labels)
        o_out[3].backward()
        assert torch.equal(o_cls, cls_t[..., 0]) and torch.equal(o_cnt, cnt_t[..., 0]) and torch.equal(o_reg, reg_t), case
        for k in range(4):
            assert _rel(o_out[k].detach(), out[k].detach()) <= 1e-6, (case, LOSSES[k])
        for i, name in enumerate(NAMES):
            for l, (q, g) in enumerate(zip(qs[i], grads[i])):
                assert _rel(q.grad, g) <= 1e-6, (case, name, l, _rel(q.grad, g))
        res[f'{case}_seed'] = np.array(seed)
        res[f'{case}_boxes'], res[f'{case}_labels'] = boxes.numpy(), labels.numpy()
        for i, name in enumerate(NAMES):
            for l in range(len(LO.STRIDES)):
                res[f'{case}_{name}{l}'] = preds[i][l].numpy()
                res[f'{case}_grad_{name}{l}'] = grads[i][l].numpy().astype(np.float32)
        res[f'{case}_cls_t'], res[f'{case}_cnt_t'], res[f'{case}_reg_t'] = cls_t.numpy(), cnt_t.numpy(), reg_t.numpy()
        for k, name in enumerate(LOSSES):
            res[f'{case}_{name}'] = np.array(float(out[k].detach()), np.float32)
        npos = (cnt_t[..., 0] > -1).sum(1).tolist()
        print(case, {n: float(out[k].detach()) for k, n in enumerate(LOSSES)}, 'positives per image', npos)
    path = os.path.join(ROOT, 'tests', 'golden', 'fcos_loss.npz')
    np.savez_compressed(path, **res)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
