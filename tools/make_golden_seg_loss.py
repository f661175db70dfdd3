"""Writes tests/golden/seg_loss.npz: the reference EncoderDecoder.loss_forward (src/models/segmentors/encoder_decoder.py, called unbound: it
does not use self) with the reference CrossEntropyLoss2d (src/losses/seg/cross_entropy_loss.py), in fp32 on the CPU, on the seeded inputs
of oracle/seg_loss_oracle.fixture_case.

  CVPYTORCH_REFERENCE=<reference checkout> python tools/make_golden_seg_loss.py

Per case (x4, x8, frac, ident, down, ignored; see seg_loss_oracle.CASES) it stores the head output, the label map, ignore_index,
loss_weight, the loss and the gradient of the loss with respect to the head output.  It asserts that the oracle reproduces them (loss
within 1e-6 relative, gradient within 1e-6 of its largest element; NaN loss and zero gradient for the all-ignored case) before writing."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import ref_shim  # noqa: E402
from oracle import seg_loss_oracle as SO  # noqa: E402


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def main():
    ref_shim.install()
    from src.losses.seg.cross_entropy_loss import CrossEntropyLoss2d
    from src.models.segmentors.encoder_decoder import EncoderDecoder
    torch.set_num_threads(1)
    res = {}
    for case in SO.CASES:
        pred, target, ignore, lw = SO.fixture_case(case)
        p = pred.clone().requires_grad_(True)
        out = EncoderDecoder.loss_forward(None, p, target, CrossEntropyLoss2d(ignore_index=ignore, loss_weight=lw))['ce_loss']
        out.backward()
        q = pred.double().requires_grad_(True)
        o = SO.loss(q, target, ignore, lw)
        o.backward()
        if case == 'ignored':
            assert torch.isnan(out) and torch.isnan(o) and not bool(p.grad.any()) and not bool(q.grad.any()), case
        else:
            assert _rel(o.detach(), out.detach()) <= 1e-6, (case, float(o), float(out))
            assert _rel(q.grad, p.grad) <= 1e-6, (case, _rel(q.grad, p.grad))
        res[f'{case}_pred'], res[f'{case}_target'] = pred.numpy(), target.numpy()
        res[f'{case}_ignore_index'], res[f'{case}_loss_weight'] = np.array(ignore), np.array(lw, np.float32)
        res[f'{case}_loss'], res[f'{case}_grad'] = np.array(float(out.detach()), np.float32), p.grad.numpy()
        print(case, float(out), 'valid pixels', int((target.long() != ignore).sum()))
    path = os.path.join(ROOT, 'tests', 'golden', 'seg_loss.npz')
    np.savez_compressed(path, **res)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
