"""tests/golden/darknet_train.npz: the REFERENCE's CSPDarknet (src/models/backbones/det/csp_darknet.py:25-129: Focus stem, four stages,
SPPF with the parallel (5, 9, 13) pools, stage4's CSPLayer with shortcut=False) in TRAINING mode on CPU in fp32, forward AND backward through
torch.autograd.  The configuration is CSPDarknet('cspdark_n', out_channels=[64, 128, 128, 128, 128]): widths 16, 32, 32, 32, 32, i.e.
YOLOX-n's 16-channel stem and 32-channel stage1 (hidden width 16), with stage2..4 narrowed to 32 channels so the file stays small; every
structure of the backbone is kept (the SPPF pools run on 16 channels).  Input 2x3x104x72: the maps are 52x36, 26x18, 13x9, 7x5 and 4x3
(ragged stride-2 parity classes; the 13x13 pool covers a whole map).  loss = sum_i sum(out_i * G_i).
The parameters, the input and the G_i are not stored: they are regenerated from the stored seeds -- parameters by
oracle/darknet_train_oracle.py:synthetic_state over the stored (key, shape) list (the distribution of tools/make_golden_train.py:randomize),
x and then G_0..2 by torch.randn from one CPU generator.  Stored: keys, shapes, seeds, the three outputs, every parameter gradient and the
running statistics after the step.  Run with CVPYTORCH_REFERENCE pointing at a checkout of the reference."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import ref_shim  # noqa: E402
from oracle import darknet_train_oracle as DO  # noqa: E402

SUBTYPE = 'cspdark_n'
OUT_CHANNELS = [64, 128, 128, 128, 128]
PARAM_SEED, DATA_SEED = 91, 92
B, H, W = 2, 104, 72


def main():
    ref_shim.install()
    from src.models.backbones.det.csp_darknet import CSPDarknet
    m = CSPDarknet(SUBTYPE, out_channels=OUT_CHANNELS)
    shapes = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    m.load_state_dict(DO.synthetic_state(shapes, seed=PARAM_SEED))
    m.train()
    g = torch.Generator().manual_seed(DATA_SEED)
    x = torch.randn(B, 3, H, W, generator=g)
    outs = m(x)
    Gs = [torch.randn(o.shape, generator=g) for o in outs]
    sum((o * G).sum() for o, G in zip(outs, Gs)).backward()
    out = {'cfg': np.array([B, H, W]), 'out_channels': np.array(OUT_CHANNELS), 'seeds': np.array([PARAM_SEED, DATA_SEED]),
           'keys': np.array([k for k, _ in shapes]), 'shapes': np.array([str(s_) for _, s_ in shapes])}
    for i, o in enumerate(outs):
        out[f'y{i}'] = o.detach().numpy()
    for k, p in m.named_parameters():
        out[f'grad_{k}'] = p.grad.numpy()
    for k, v in m.state_dict().items():
        if 'running_' in k:
            out[f'after_{k}'] = v.numpy()
    # the oracle restatement must reproduce the reference before the fixture is written
    ref_keys = {k for k in out if k.startswith(('y', 'grad_', 'after_'))}
    o2, g2, s2 = DO.train_step(x, Gs, DO.synthetic_state(shapes, seed=PARAM_SEED), subtype=SUBTYPE, out_channels=OUT_CHANNELS)
    got = {f'y{i}': v for i, v in enumerate(o2)}
    got.update({f'grad_{k}': v for k, v in g2.items()})
    got.update({f'after_{k}': v for k, v in s2.items()})
    assert set(got) == ref_keys
    worst = max(float((got[k] - torch.from_numpy(out[k])).abs().max() / (abs(out[k]).max() + 1e-12)) for k in ref_keys)
    assert worst <= 1e-5, worst
    print(SUBTYPE, OUT_CHANNELS, 'outputs', [tuple(o.shape) for o in outs], 'params', sum(p.numel() for p in m.parameters()), 'keys', len(shapes), 'oracle worst', worst)
    np.savez_compressed(os.path.join(ROOT, 'tests/golden/darknet_train.npz'), **out)


if __name__ == '__main__':
    main()
