"""tests/golden/yolov5_train.npz: the REFERENCE's YOLOv5 network -- YOLOv5CSPDarknet (src/models/backbones/det/yolov5_csp_darknet.py),
the old-API YOLOv5Neck (src/models/necks/yolov5_neck.py) and YOLOv5Detect (src/models/detects/yolov5_detect.py) -- in TRAINING mode on the
CPU in fp32, forward AND backward through torch.autograd.

  CVPYTORCH_REFERENCE=<reference checkout> python tools/make_golden_yolov5_train.py

The configuration (oracle/yolov5_train_oracle.NET) keeps every width on the training path and the file small: a YOLOv5-n backbone with
out_channels [64, 128, 128, 128, 128] (widths 16 and 32, C3 hidden width 16), the neck and detect at width 32, 3 classes, a 2x3x64x96
image; the detect outputs are 2x24x{8x12, 4x6, 2x3}.  loss = sum_i sum(out_i * G_i).  The parameters, the image and the G_i are not
stored: they are regenerated from the stored seeds -- parameters by oracle/yolov5_train_oracle.synthetic_state over the stored (key, shape)
list, then the image (torch.rand) and G_0..2 (torch.randn) from one CPU generator.  Stored: keys, shapes, seeds, the three outputs, every
parameter gradient and the running statistics after the step."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import ref_shim  # noqa: E402
from oracle import yolov5_train_oracle as O  # noqa: E402

PARAM_SEED, DATA_SEED = 95, 96


def main():
    ref_shim.install()
    import importlib
    from src.models.backbones import build_backbone
    from src.models.detects import build_detect
    oldneck = importlib.import_module('src.models.necks.yolov5_neck')
    bb = build_backbone(dict(O.NET['backbone'], name='YOLOv5CSPDarknet', out_stages=[2, 3, 4]))
    nk = oldneck.YOLOv5Neck(**O.NET['neck'])
    dt = build_detect(dict(O.NET['detect'], name='YOLOv5Detect', anchors=O.ANCHORS, depth_mul=0.33))
    mods = {'backbone.': bb, 'neck.': nk, 'detect.': dt}
    for m in mods.values():  # src/models/yolov5.py:196-205 init_weights
        for mm in m.modules():
            if isinstance(mm, torch.nn.BatchNorm2d):
                mm.eps, mm.momentum = 1e-3, 0.03
    shapes = [(pre + k, tuple(v.shape)) for pre, m in mods.items() for k, v in m.state_dict().items()]
    sd = O.synthetic_state(shapes, seed=PARAM_SEED)
    for pre, m in mods.items():
        m.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)})
        m.train()
    g = torch.Generator().manual_seed(DATA_SEED)
    x = torch.rand(O.NET['image'], generator=g)
    _, outs = dt(nk(bb(x)))
    outs = [o.permute(0, 1, 4, 2, 3).reshape(o.shape[0], -1, o.shape[2], o.shape[3]) for o in outs]  # (the detect convs' NCHW outputs)
    Gs = [torch.randn(o.shape, generator=g) for o in outs]
    sum((o * G).sum() for o, G in zip(outs, Gs)).backward()
    out = {'seeds': np.array([PARAM_SEED, DATA_SEED]), 'keys': np.array([k for k, _ in shapes]), 'shapes': np.array([str(s_) for _, s_ in shapes])}
    for i, o in enumerate(outs):
        out[f'y{i}'] = o.detach().numpy()
    for pre, m in mods.items():
        for k, p in m.named_parameters():
            out[f'grad_{pre}{k}'] = p.grad.numpy()
        for k, v in m.state_dict().items():
            if 'running_' in k:
                out[f'after_{pre}{k}'] = v.numpy()
    # the oracle restatement must reproduce the reference before the fixture is written
    keys, sd2, x2, Gs2 = O.net_fixture_inputs(out)
    assert keys == [k for k, _ in shapes] and torch.equal(x2, x) and all(torch.equal(a, b) for a, b in zip(Gs2, Gs))
    got = O.net_train_step(x2, Gs2, sd2)
    ref_keys = {k for k in out if k.startswith(('y', 'grad_', 'after_'))}
    assert set(got) == ref_keys, set(got) ^ ref_keys
    worst = max(float((got[k] - torch.from_numpy(out[k])).abs().max() / (abs(out[k]).max() + 1e-12)) for k in ref_keys)
    assert worst <= 1e-5, worst
    print('outputs', [tuple(o.shape) for o in outs], 'params', sum(p.numel() for m in mods.values() for p in m.parameters()), 'keys', len(shapes),
          'oracle worst', worst)
    np.savez_compressed(os.path.join(ROOT, 'tests/golden/yolov5_train.npz'), **out)


if __name__ == '__main__':
    main()
