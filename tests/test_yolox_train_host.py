"""YOLOX neck and head training (cvpytorch_b200.train.YOLOXNeck, YOLOXHead, ConvModule) without a GPU: the oracle against the reference
fixture, the drop-ins' module trees, the configurations they refuse, and the host-side argument checks of the new C entry points."""
import ast
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')
NECK = dict(channels=[128, 128, 128], depth_mul=0.33, width_mul=0.25)  # (the configuration of tools/make_golden_yolox_train.py)
HEAD = dict(num_classes=3, in_channels=[256, 256, 256], width_mul=0.125)


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def test_yolox_train_oracle_reproduces_reference_fixture():
    """oracle/yolox_train_oracle.py (functional neck + head, torch.autograd) vs the reference's own YOLOXNeck + YOLOXHead in fp32: outputs,
    feature-map gradients, every parameter gradient and the running statistics after the step, <= 1e-5.  The key list is the reference's and
    must equal the training drop-ins'."""
    from cvpytorch_b200 import train as T
    from oracle import yolox_train_oracle as XO
    g = np.load(os.path.join(GOLD, 'yolox_train.npz'))
    keys, sd, feats, Gs, dm = XO.fixture_inputs(g)
    outs, dxs, grads, stats = XO.train_step(feats, Gs, sd, dm)
    errs = {f'y{i}': _rel(o, g[f'y{i}']) for i, o in enumerate(outs)}
    errs.update({f'dx{i}': _rel(d, g[f'dx{i}']) for i, d in enumerate(dxs)})
    for k, v in grads.items():
        errs['grad ' + k] = _rel(v, g[f'grad_{k}'])
    for k, v in stats.items():
        errs['after ' + k] = _rel(v, g[f'after_{k}'])
    mine = ['neck.' + k for k in T.YOLOXNeck(**NECK).state_dict()] + ['head.' + k for k in T.YOLOXHead(**HEAD).state_dict()]
    assert mine == keys
    assert len([k for k in errs if k.startswith('grad ')]) == sum(1 for k in keys if 'running_' not in k and 'num_batches' not in k)
    worst = max(errs, key=errs.get)
    assert errs[worst] <= 1e-5, (worst, errs[worst])


def test_training_neck_head_keys_match_reference_and_inference_modules():
    """YOLOX-s neck and head: the neck.* / head.* keys and shapes of tests/golden/yolox_keys.npz (dumped from the reference) and those of the
    inference drop-ins; every BatchNorm has eps 1e-3 and momentum 0.03; cls / obj biases start at the prior-probability value."""
    from cvpytorch_b200 import train as T, yolox_models as Y
    g = np.load(os.path.join(GOLD, 'yolox_keys.npz'))
    ref = {str(k): tuple(ast.literal_eval(str(s))) for k, s in zip(g['keys'], g['shapes'])}
    neck_kw = dict(subtype='yolox_s', channels=[256, 512, 1024], depth_mul=0.33, width_mul=0.5)
    head_kw = dict(num_classes=80, subtype='yolox_s', in_channels=[256, 512, 1024], width_mul=0.5)
    for pre, m, inf in (('neck.', T.YOLOXNeck(**neck_kw), Y.YOLOXNeck(**neck_kw)), ('head.', T.YOLOXHead(**head_kw), Y.YOLOXHead(**head_kw))):
        got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        want = {k[len(pre):]: s for k, s in ref.items() if k.startswith(pre)}
        assert got == want
        assert list(got) == [k[len(pre):] for k in (str(k) for k in g['keys']) if k.startswith(pre)]
        assert list(got) == list(inf.state_dict()) and got == {k: tuple(v.shape) for k, v in inf.state_dict().items()}
        bns = [mod for mod in m.modules() if isinstance(mod, torch.nn.BatchNorm2d)]
        assert bns and all(b.eps == 1e-3 and b.momentum == 0.03 for b in bns)
    h = T.YOLOXHead(**head_kw)
    prior = -np.log((1 - 1e-2) / 1e-2)
    for conv in list(h.cls_preds) + list(h.obj_preds):
        assert torch.allclose(conv.bias, torch.full_like(conv.bias, prior))


@pytest.mark.parametrize('width_mul', [0.375, 0.75, 1.25])
def test_training_neck_head_refuse_non_training_widths(width_mul):
    """YOLOX-t / -m / -x necks: CSP hidden widths 48 / 96 / 160.  The head follows the same width rule: YOLOX-t's 96 raises, while -m's 192
    and -x's 320 are multiples of 64 and build."""
    from cvpytorch_b200 import train as T
    with pytest.raises(NotImplementedError):
        T.YOLOXNeck(channels=[256, 512, 1024], depth_mul=0.33, width_mul=width_mul)
    if int(256 * width_mul) % 64:
        with pytest.raises(NotImplementedError):
            T.YOLOXHead(80, in_channels=[256, 512, 1024], width_mul=width_mul)
    else:
        T.YOLOXHead(80, in_channels=[256, 512, 1024], width_mul=width_mul)
    with pytest.raises(NotImplementedError):
        T.YOLOXHead(80, in_channels=[256, 512, 1024], width_mul=0.125 * 3)


@pytest.mark.parametrize('kw', [dict(kernel_size=5, padding=2), dict(kernel_size=3, padding=0), dict(kernel_size=3, padding=1, stride=2),
                                dict(kernel_size=1, padding=2), dict(kernel_size=1, padding=0, activation='ReLU')])
def test_training_conv_module_refuses_unsupported_configurations(kw):
    from cvpytorch_b200 import train as T
    with pytest.raises(NotImplementedError):
        T.ConvModule(32, 32, **kw)


def test_training_neck_head_eval_cpu_and_geometry_refusals():
    from cvpytorch_b200 import _lib, train as T
    for sub, w in (('yolox_n', 0.25), ('yolox_s', 0.5), ('yolox_l', 1.0)):
        T.YOLOXNeck(sub, [256, 512, 1024], 0.33, w)
        T.YOLOXHead(80, sub, [256, 512, 1024], width_mul=w)
    T.ConvModule(32, 64, 1, 1, padding=1)
    T.ConvModule(32, 64, 1, 1, padding=0)
    nk = T.YOLOXNeck(**NECK).train()
    hd = T.YOLOXHead(**HEAD).train()
    feats = [torch.zeros(2, 32, 8, 8), torch.zeros(2, 32, 4, 4), torch.zeros(2, 32, 2, 2)]
    with pytest.raises(_lib.CvbError):
        nk(feats)  # CPU tensors: no fallback
    with pytest.raises(_lib.CvbError):
        hd(feats)
    nhwc = [f.permute(0, 2, 3, 1).to(torch.bfloat16) for f in feats]
    for bad in ([nhwc[0], nhwc[1], nhwc[1]], [nhwc[0][:, :7, :8], nhwc[1], nhwc[2]], [nhwc[0][:1], nhwc[1], nhwc[2]], [nhwc[0], nhwc[1][:, :, :3], nhwc[2]]):
        with pytest.raises(ValueError):
            nk.forward_nhwc(bad)
    with pytest.raises(ValueError):
        T.upsample_cat(nhwc[1], nhwc[1])
    nk.eval()
    hd.eval()
    with pytest.raises(RuntimeError):
        nk.forward_nhwc(nhwc)
    with pytest.raises(RuntimeError):
        hd.forward_nhwc(nhwc)


def test_training_c_abi_padding_prediction_and_upsample_arguments():
    """Every new entry point rejects bad arguments on the host, before the device is touched: paddings other than k = 1 with -1 / 0 / 1 and
    k = 3 with 1, an empty output, non-training widths, cout_pad that is not cout's next training width, a channel range outside the output,
    misaligned pointers, and upsample-concat channels that are not multiples of 8."""
    from cvpytorch_b200 import _lib
    L = _lib.lib()
    one = ctypes.c_void_p(16)
    odd = ctypes.c_void_p(18)

    def err(rc, text):
        assert rc != 0
        assert text in L.cvb_last_error_string(), L.cvb_last_error_string()
    for k, pad in ((1, 2), (1, -2), (3, 0), (3, -1), (3, 2)):
        err(L.cvb_train_conv_pad(one, 1, 8, 8, 32, one, 32, k, pad, one, None, None, None), b'padding')
        err(L.cvb_train_conv_wgrad_pad(one, one, 1, 8, 8, 32, 32, k, pad, one, None), b'padding')
    err(L.cvb_train_conv_pad(one, 1, 2, 8, 32, one, 32, 1, -1, one, None, None, None), b'empty output')
    err(L.cvb_train_conv_wgrad_pad(one, one, 1, 8, 1, 32, 32, 1, -1, one, None), b'empty output')
    for c in (24, 48, 96):
        err(L.cvb_train_conv_pad(one, 1, 8, 8, c, one, 32, 1, 1, one, None, None, None), b'multiples of 64')
        err(L.cvb_train_conv_wgrad_pad(one, one, 1, 8, 8, 32, c, 1, 1, one, None), b'multiples of 64')
        err(L.cvb_train_pred_conv(one, 1, 8, 8, c, one, 5, 16, one, one, 8, 0, None), b'cin must be')
    err(L.cvb_train_conv_pad(odd, 1, 8, 8, 32, one, 32, 1, 1, one, None, None, None), b'16-byte aligned')
    err(L.cvb_train_conv_wgrad_pad(one, odd, 1, 8, 8, 32, 32, 1, 1, one, None), b'16-byte aligned')
    for cout, cout_pad in ((5, 8), (5, 32), (17, 16), (33, 32), (80, 96), (80, 64), (0, 16)):
        err(L.cvb_train_pred_conv(one, 1, 8, 8, 32, one, cout, cout_pad, one, one, 85, 0, None), b'cout_pad')
        err(L.cvb_train_pred_grad(one, 1, 85, 8, 8, 0, cout, cout_pad, one, one, None), b'cout_pad')
    for c_tot, c_off, cout in ((8, 5, 4), (85, 6, 80), (5, -1, 5)):
        err(L.cvb_train_pred_conv(one, 1, 8, 8, 32, one, cout, 16 if cout <= 16 else 128, one, one, c_tot, c_off, None), b'outside')
        err(L.cvb_train_pred_grad(one, 1, c_tot, 8, 8, c_off, cout, 16 if cout <= 16 else 128, one, one, None), b'outside')
    err(L.cvb_train_pred_conv(odd, 1, 8, 8, 32, one, 5, 16, one, one, 8, 0, None), b'aligned')
    err(L.cvb_train_pred_conv(one, 1, 8, 8, 32, one, 5, 16, one, ctypes.c_void_p(18), 8, 0, None), b'aligned')
    err(L.cvb_train_pred_grad(one, 1, 8, 8, 8, 0, 5, 16, odd, one, None), b'aligned')
    err(L.cvb_train_pred_grad(ctypes.c_void_p(18), 1, 8, 8, 8, 0, 5, 16, one, one, None), b'aligned')
    for Ca, Cb in ((12, 16), (16, 20), (4, 4)):
        err(L.cvb_train_upsample_cat_fwd(one, 1, 4, 4, Ca, one, Cb, one, None), b'multiples of 8')
        err(L.cvb_train_upsample_cat_bwd(one, 1, 4, 4, Ca, Cb, one, one, None), b'multiples of 8')
    err(L.cvb_train_upsample_cat_fwd(one, 1, 4, 4, 16, odd, 16, one, None), b'16-byte aligned')
    err(L.cvb_train_upsample_cat_bwd(one, 1, 4, 4, 16, 16, one, odd, None), b'16-byte aligned')
    err(L.cvb_train_upsample_cat_fwd(one, 1, 0, 4, 16, one, 16, one, None), b'bad argument')
