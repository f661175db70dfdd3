"""tests/golden/yolov6_train.npz: the REFERENCE's YOLOv6 network -- YOLOv6EfficientRep (src/models/backbones/det/yolov6_efficient_rep.py),
YOLOv6RepBiPAN (src/models/necks/det/yolov6_repbipan.py) and YOLOv6Effidehead (src/models/heads/det/yolov6_effidehead.py) -- in TRAINING
mode on the CPU in fp32, forward AND backward through torch.autograd.

  CVPYTORCH_REFERENCE=<reference checkout> python tools/make_golden_yolov6_train.py

The configuration (oracle/yolov6_train_oracle.NET) is a narrowed YOLOv6-n that keeps every layer type: widths 16 and 32, RepBlocks of two
blocks (stride-2 and identity RepVGG blocks), SimCSPSPPF, BiFusions with c = 32 (the 96-channel concat), stride-1 and stride-2 ReLU
ConvModules and the SiLU head; 3 classes, a 2x3x64x96 image.  The BatchNorms keep the eps / momentum the reference modules' own
init_weights set.  loss = sum(pred_scores * G_0) + sum(pred_distri * G_1).  The parameters, the image and the G are not stored: they are
regenerated from the stored seeds (oracle/yolov6_train_oracle.synthetic_state over the stored (key, shape) list, then the image (torch.rand)
and G_0, G_1 (torch.randn) from one CPU generator).  Stored: keys, shapes, seeds, both outputs, every parameter gradient and the running
statistics after the step.  The oracle must reproduce it (on oracle/yolov6_train_oracle.fixture_scale) (1e-5 outputs and gradients, 1e-6 running statistics) before it is written."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import ref_shim  # noqa: E402
from oracle import yolov6_train_oracle as O  # noqa: E402

PARAM_SEED, DATA_SEED = 61, 62


def main():
    ref_shim.install()
    from src.models.backbones import build_backbone
    from src.models.heads import build_head
    from src.models.necks import build_neck
    bb = build_backbone(dict(O.NET['backbone'], name='YOLOv6EfficientRep'))
    nk = build_neck(dict(O.NET['neck'], name='YOLOv6RepBiPAN'))
    hd = build_head(dict(O.NET['head'], name='YOLOv6Effidehead'))
    mods = {'backbone.': bb, 'neck.': nk, 'head.': hd}
    for m in mods.values():
        for mm in m.modules():
            if isinstance(mm, torch.nn.BatchNorm2d):
                assert (mm.eps, mm.momentum) == (1e-3, 0.03), (type(m).__name__, mm.eps, mm.momentum)
    shapes = [(pre + k, tuple(v.shape)) for pre, m in mods.items() for k, v in m.state_dict().items()]
    sd = O.synthetic_state(shapes, seed=PARAM_SEED)
    for pre, m in mods.items():
        m.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)})
        m.train()
    g = torch.Generator().manual_seed(DATA_SEED)
    x = torch.rand(O.NET['image'], generator=g)
    _, scores, distri = hd(nk(bb(x)))
    Gs = [torch.randn(scores.shape, generator=g), torch.randn(distri.shape, generator=g)]
    ((scores * Gs[0]).sum() + (distri * Gs[1]).sum()).backward()
    out = {'seeds': np.array([PARAM_SEED, DATA_SEED]), 'keys': np.array([k for k, _ in shapes]), 'shapes': np.array([str(s_) for _, s_ in shapes]),
           'scores': scores.detach().numpy(), 'distri': distri.detach().numpy()}
    for pre, m in mods.items():
        for k, p in m.named_parameters():
            if p.requires_grad:
                assert p.grad is not None, pre + k
                out[f'grad_{pre}{k}'] = p.grad.numpy()
        for k, v in m.state_dict().items():
            if 'running_' in k:
                out[f'after_{pre}{k}'] = v.numpy()
    # the oracle restatement must reproduce the reference before the fixture is written
    keys, sd2, x2, Gs2 = O.net_fixture_inputs(out)
    assert keys == [k for k, _ in shapes] and torch.equal(x2, x) and all(torch.equal(a, b) for a, b in zip(Gs2, Gs))
    got = O.net_train_step(x2, Gs2, sd2)
    ref_keys = {k for k in out if k in ('scores', 'distri') or k.startswith(('grad_', 'after_'))}
    assert set(got) == ref_keys, set(got) ^ ref_keys
    err = {k: float((got[k] - torch.from_numpy(out[k])).abs().max()) / O.fixture_scale(k, out) for k in ref_keys}
    worst = max(v for k, v in err.items() if not k.startswith('after_'))
    worst_stats = max(v for k, v in err.items() if k.startswith('after_'))
    assert worst <= 1e-5 and worst_stats <= 1e-6, (worst, worst_stats, sorted((v, k) for k, v in err.items())[-6:])
    print('outputs', tuple(scores.shape), tuple(distri.shape), 'params', sum(p.numel() for m in mods.values() for p in m.parameters()), 'keys', len(shapes),
          'oracle worst', worst, worst_stats)
    np.savez_compressed(os.path.join(ROOT, 'tests/golden/yolov6_train.npz'), **out)


if __name__ == '__main__':
    main()
