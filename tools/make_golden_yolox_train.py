"""tests/golden/yolox_train.npz: the REFERENCE's YOLOXNeck (src/models/necks/yolox_neck.py:13-74) and YOLOXHead
(src/models/heads/yolox_head.py:14-88) in TRAINING mode on CPU in fp32, forward AND backward through torch.autograd.
The configuration keeps every width on the training path and the file small: YOLOXNeck(channels=[128, 128, 128], depth_mul=0.33,
width_mul=0.25) (widths 32, CSP hidden width 16) and YOLOXHead(num_classes=3, in_channels=[256, 256, 256], width_mul=0.125) (width 32);
feature maps 2x32x{12x20, 6x10, 3x5} with requires_grad, so the fixture also holds the gradients a backbone would receive.  The head maps
are 14x22, 8x12 and 5x7 (odd); the prediction convs have 3 (cls) and 5 (reg + obj) outputs.  loss = sum_i sum(out_i * G_i).
The parameters, the feature maps and the G_i are not stored: they are regenerated from the stored seeds -- parameters by
oracle/yolox_train_oracle.py:synthetic_state over the stored (key, shape) list, the three maps and then G_0..2 by torch.randn from one CPU
generator.  Stored: keys, shapes, seeds, configuration, the three outputs, the feature-map gradients, every parameter gradient and the
running statistics after the step.  Run with CVPYTORCH_REFERENCE pointing at a checkout of the reference."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import ref_shim  # noqa: E402
from oracle import yolox_train_oracle as XO  # noqa: E402

NECK = dict(channels=[128, 128, 128], depth_mul=0.33, width_mul=0.25)
HEAD = dict(num_classes=3, in_channels=[256, 256, 256], width_mul=0.125)
FEATS = [(2, 32, 12, 20), (2, 32, 6, 10), (2, 32, 3, 5)]
PARAM_SEED, DATA_SEED = 93, 94


def main():
    ref_shim.install()
    from src.models.heads.yolox_head import YOLOXHead
    from src.models.necks.yolox_neck import YOLOXNeck
    nk, hd = YOLOXNeck(**NECK), YOLOXHead(**HEAD)
    shapes = [('neck.' + k, tuple(v.shape)) for k, v in nk.state_dict().items()] + [('head.' + k, tuple(v.shape)) for k, v in hd.state_dict().items()]
    sd = XO.synthetic_state(shapes, seed=PARAM_SEED)
    nk.load_state_dict({k[len('neck.'):]: v for k, v in sd.items() if k.startswith('neck.')})
    hd.load_state_dict({k[len('head.'):]: v for k, v in sd.items() if k.startswith('head.')})
    nk.train()
    hd.train()
    g = torch.Generator().manual_seed(DATA_SEED)
    feats = [torch.randn(s, generator=g).requires_grad_(True) for s in FEATS]
    outs = hd(nk(feats))
    Gs = [torch.randn(o.shape, generator=g) for o in outs]
    sum((o * G).sum() for o, G in zip(outs, Gs)).backward()
    out = {'seeds': np.array([PARAM_SEED, DATA_SEED]), 'feat_shapes': np.array(FEATS), 'num_classes': np.array(HEAD['num_classes']),
           'depth_mul': np.array(NECK['depth_mul']), 'keys': np.array([k for k, _ in shapes]), 'shapes': np.array([str(s_) for _, s_ in shapes])}
    for i, o in enumerate(outs):
        out[f'y{i}'] = o.detach().numpy()
    for i, f in enumerate(feats):
        out[f'dx{i}'] = f.grad.numpy()
    for pre, m in (('neck.', nk), ('head.', hd)):
        for k, p in m.named_parameters():
            out[f'grad_{pre}{k}'] = p.grad.numpy()
        for k, v in m.state_dict().items():
            if 'running_' in k:
                out[f'after_{pre}{k}'] = v.numpy()
    # the oracle restatement must reproduce the reference before the fixture is written
    keys, sd2, feats2, Gs2, dm = XO.fixture_inputs(out)
    assert keys == [k for k, _ in shapes] and all(torch.equal(a, b.detach()) for a, b in zip(feats2, feats)) and all(torch.equal(a, b) for a, b in zip(Gs2, Gs))
    o2, dx2, g2, s2 = XO.train_step(feats2, Gs2, sd2, dm)
    got = {f'y{i}': v for i, v in enumerate(o2)}
    got.update({f'dx{i}': v for i, v in enumerate(dx2)})
    got.update({f'grad_{k}': v for k, v in g2.items()})
    got.update({f'after_{k}': v for k, v in s2.items()})
    ref_keys = {k for k in out if k.startswith(('y', 'dx', 'grad_', 'after_'))}
    assert set(got) == ref_keys, set(got) ^ ref_keys
    worst = max(float((got[k] - torch.from_numpy(out[k])).abs().max() / (abs(out[k]).max() + 1e-12)) for k in ref_keys)
    assert worst <= 1e-5, worst
    print(NECK, HEAD, 'outputs', [tuple(o.shape) for o in outs], 'params', sum(p.numel() for m in (nk, hd) for p in m.parameters()), 'keys', len(shapes),
          'oracle worst', worst)
    np.savez_compressed(os.path.join(ROOT, 'tests/golden/yolox_train.npz'), **out)


if __name__ == '__main__':
    main()
