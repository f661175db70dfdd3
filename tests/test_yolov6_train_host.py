"""YOLOv6 training, host side (no GPU): the oracle network against the reference fixture (tests/golden/yolov6_train.npz), the training
modules' state_dict keys against the inference modules' and the fixture's, the stem remap and the
transposed-conv GEMM layout / scatter / gather restated in float64 against F.conv2d / F.conv_transpose2d autograd, the host refusals of the
new C entry points and the refusals of the model and modules."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_yolov6_host import DICT, use_model  # noqa: E402

from cvpytorch_b200 import _lib, yolov6_models as M, yolov6_train as Y  # noqa: E402
from cvpytorch_b200.modules import _build  # noqa: E402
from oracle import yolov6_train_oracle as O  # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'yolov6_train.npz')


def test_oracle_reproduces_reference_fixture():
    """tests/golden/yolov6_train.npz is the reference's YOLOv6EfficientRep, YOLOv6RepBiPAN and YOLOv6Effidehead in training mode (fp32, CPU,
    torch.autograd) on a narrowed YOLOv6-n: the oracle network reproduces its outputs and every parameter gradient within 1e-5 and the
    running statistics after the step within 1e-6 (each on oracle.fixture_scale).  The fixture holds every layer type of the network."""
    f = np.load(GOLD)
    keys, sd, x, Gs = O.net_fixture_inputs(f)
    got = O.net_train_step(x, Gs, sd)
    ref = {k: f[k] for k in f.files if k in ('scores', 'distri') or k.startswith(('grad_', 'after_'))}
    assert set(got) == set(ref)
    for k in ref:
        err = float((got[k] - torch.from_numpy(ref[k])).abs().max()) / O.fixture_scale(k, ref)
        assert err <= (1e-6 if k.startswith('after_') else 1e-5), (k, err)
    assert sum(k.endswith('rbr_identity.weight') for k in keys) >= 2  # identity RepVGG blocks
    assert 'neck.Rep_p3.block.0.rbr_dense.conv.weight' in keys  # a RepBlock of two blocks
    assert sd['neck.bifusion1.cv3.conv.weight'].shape[1] == 96  # the zero-padded BiFusion concat
    assert 'backbone.stage4.2.cv7.conv.weight' in keys and 'neck.downsample1.conv.weight' in keys  # SimCSPSPPF, stride-2 ConvModule


@pytest.mark.parametrize('stype', ['n', 's'])
def test_training_module_keys_equal_inference_keys(stype):
    m = M.YOLOv6(DICT, use_model(stype))
    bcfg, ncfg, hcfg, sub = m._cfgs
    mods = (_build(M._TRAIN_BACKBONES, dict(bcfg, **sub)), _build(M._TRAIN_NECKS, dict(ncfg, **sub)), _build(M._TRAIN_HEADS, dict(hcfg, **sub)))
    for tm, im in zip(mods, (m.backbone, m.neck, m.head)):
        assert list(tm.state_dict()) == list(im.state_dict())
        assert {k: tuple(v.shape) for k, v in tm.state_dict().items()} == {k: tuple(v.shape) for k, v in im.state_dict().items()}
    if stype == 'n':  # the one width that is not a training width: bifusion1.cv3 reads 3 x 32 channels, run as 128
        assert mods[1].bifusion1.cv3.in_pad == 32 and mods[1].bifusion0.cv3.in_pad == 0


def test_stem_remap_float64():
    """A 3x3 / stride-2 / pad-1 conv of the image (and its 1x1 / stride-2 branch, zero-padded to 3x3) == a 3x3 / stride-1 / pad-1 conv of the
    Focus space-to-depth map (channel 3 (2 dx + dy) + c) with stem_weight_to_s2d's weight; autograd maps the weight gradient back."""
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 3, 22, 30, generator=g, dtype=torch.float64)
    s2d = torch.cat([x[:, :, dy::2, dx::2] for dx in (0, 1) for dy in (0, 1)], 1)  # patch 2 dx + dy: tl, bl, tr, br
    s2d = F.pad(s2d, (0, 0, 0, 0, 0, 4))
    G = torch.randn(2, 16, 11, 15, generator=g, dtype=torch.float64)
    for w0 in (torch.randn(16, 3, 3, 3, generator=g, dtype=torch.float64), F.pad(torch.randn(16, 3, 1, 1, generator=g, dtype=torch.float64), (1, 1, 1, 1))):
        w = w0.clone().requires_grad_()
        w2 = w0.clone().requires_grad_()
        ref = F.conv2d(x, w, None, 2, 1)
        got = F.conv2d(s2d, Y.stem_weight_to_s2d(w2), None, 1, 1)
        assert torch.allclose(got, ref, rtol=0, atol=1e-12)
        (ref * G).sum().backward()
        (got * G).sum().backward()
        assert torch.allclose(w2.grad, w.grad, rtol=0, atol=1e-10)


@pytest.mark.parametrize('h,w', [(3, 5), (8, 8)])
def test_conv_transpose_gemm_scatter_gather_float64(h, w):
    """ConvTranspose2d(c, c, 2, stride 2) == the 1x1 GEMM with _convt_weight(W) (4c columns, [py][px][cout]) + the scatter (column
    (py * 2 + px) c + o -> pixel (2y + py, 2x + px), channel o) + bias; the gather of d(out) back to the GEMM layout and the 1x1 backward
    give F.conv_transpose2d's input / weight / bias gradients."""
    g = torch.Generator().manual_seed(h * w)
    c = 8
    x = torch.randn(2, c, h, w, generator=g, dtype=torch.float64, requires_grad=True)
    wt = torch.randn(c, c, 2, 2, generator=g, dtype=torch.float64, requires_grad=True)
    b = torch.randn(c, generator=g, dtype=torch.float64, requires_grad=True)
    G = torch.randn(2, c, 2 * h, 2 * w, generator=g, dtype=torch.float64)
    ref = F.conv_transpose2d(x, wt, b, stride=2)
    (ref * G).sum().backward()
    wg = Y._convt_weight(wt.detach())
    u = F.conv2d(x.detach(), wg).permute(0, 2, 3, 1)  # NHWC [B, h, w, 4c]
    scat = u.reshape(2, h, w, 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(2, 2 * h, 2 * w, c) + b.detach()
    assert torch.allclose(scat.permute(0, 3, 1, 2), ref, rtol=0, atol=1e-12)
    Gn = G.permute(0, 2, 3, 1)
    du = Gn.reshape(2, h, 2, w, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(2, h, w, 4 * c)  # the gather
    dwg = torch.einsum('bhwo,bhwi->oi', du, x.detach().permute(0, 2, 3, 1))
    dx = torch.einsum('bhwo,oi->bhwi', du, wg[:, :, 0, 0]).permute(0, 3, 1, 2)
    wg2 = wt.detach().clone().requires_grad_()
    (Y._convt_weight(wg2)[:, :, 0, 0] * dwg).sum().backward()
    assert torch.allclose(dx, x.grad, rtol=0, atol=1e-10)
    assert torch.allclose(wg2.grad, wt.grad, rtol=0, atol=1e-10)
    assert torch.allclose(Gn.sum((0, 1, 2)), b.grad, rtol=0, atol=1e-10)


def _err(L, rc, text):
    assert rc != 0
    assert text in L.cvb_last_error_string(), L.cvb_last_error_string()


def test_c_abi_refusals():
    """Every new entry point refuses bad arguments on the host, before any launch."""
    L = _lib.lib()
    one = 1 << 20  # an aligned, never-dereferenced address
    _err(L, L.cvb_train_bn_relu_fwd(None, 4, 16, one, one, None), b'null pointer')
    _err(L, L.cvb_train_bn_relu_fwd(one, 0, 16, one, one, None), b'npix must be > 0')
    _err(L, L.cvb_train_bn_relu_fwd(one, 4, 12, one, one, None), b'C a multiple of 8 up to 2048')
    _err(L, L.cvb_train_bn_relu_fwd(one, 4, 2056, one, one, None), b'C a multiple of 8 up to 2048')
    _err(L, L.cvb_train_bn_relu_fwd(one + 8, 4, 16, one, one, None), b'16-byte')
    for k in range(6):
        a = [one] * 6
        a[k] = None
        _err(L, L.cvb_train_bn_relu_bwd(a[0], a[1], 4, 16, a[2], a[3], a[4], a[5], None), b'null pointer')
    _err(L, L.cvb_train_bn_relu_bwd(one, one, 4, 16, one, one, one, one + 2, None), b'16-byte')
    _err(L, L.cvb_train_bn_relu_bwd(one, one, 4, 16, one + 2, one, one, one, None), b'4-byte')
    _err(L, L.cvb_train_repvgg_fwd(one, None, None, 4, 16, one, one, None, one, None), b'null pointer')
    _err(L, L.cvb_train_repvgg_fwd(one, one, None, 4, 20, one, one, None, one, None), b'C a multiple of 8')
    _err(L, L.cvb_train_repvgg_fwd(one, one, one, 4, 16, one, one, None, one, None), b'x and stat_id go together')
    _err(L, L.cvb_train_repvgg_fwd(one, one, None, 4, 16, one, one, one, one, None), b'x and stat_id go together')
    _err(L, L.cvb_train_repvgg_fwd(one, one, one + 8, 4, 16, one, one, one, one, None), b'16-byte aligned')
    bwd = lambda x=None, sid=None, gid=None, dxid=None, npix=4, C=16, a=one: L.cvb_train_repvgg_bwd(  # noqa: E731
        one, a, one, one, x, npix, C, one, one, sid, one, one, gid, one, one, one, dxid, None)
    _err(L, bwd(a=None), b'null pointer')
    _err(L, bwd(npix=0), b'npix must be > 0')
    _err(L, bwd(x=one, sid=one, gid=one), b'go together')
    _err(L, bwd(x=one, sid=one, dxid=one), b'go together')
    _err(L, bwd(x=one, gid=one, dxid=one), b'x and stat_id go together')
    _err(L, bwd(x=one, sid=one, gid=one, dxid=one + 8), b'16-byte aligned')
    _err(L, L.cvb_train_repvgg_fwd(one, one, None, 4, 16, one + 2, one, None, one, None), b'4-byte aligned')
    _err(L, L.cvb_train_repvgg_bwd(one, one, one, one, None, 4, 16, one, one, None, one, one, None, one + 2, one, one, None, None), b'4-byte aligned')
    _err(L, L.cvb_train_convt_scatter(one, 1, 2, 2, 16, None, one, None), b'null pointer')
    _err(L, L.cvb_train_convt_scatter(one, 0, 2, 2, 16, one, one, None), b'B, h, w must be > 0')
    _err(L, L.cvb_train_convt_scatter(one, 1, 2, 2, 12, one, one, None), b'C a multiple of 8')
    _err(L, L.cvb_train_convt_scatter(one + 8, 1, 2, 2, 16, one, one, None), b'16-byte')
    _err(L, L.cvb_train_convt_gather(one, 1, 2, 2, 16, None, one, one, None), b'null pointer')
    _err(L, L.cvb_train_convt_gather(one, 1, 0, 2, 16, one, one, one, None), b'B, h, w must be > 0')
    _err(L, L.cvb_train_convt_gather(one, 1, 2, 2, 4096, one, one, one, None), b'C a multiple of 8 up to 2048')
    _err(L, L.cvb_train_convt_gather(one, 1, 2, 2, 16, one, one + 8, one, None), b'16-byte')
    _err(L, L.cvb_train_convt_gather(one, 1, 2, 2, 16, one + 2, one, one, None), b'4-byte')


def test_model_and_module_refusals():
    m = M.YOLOv6(DICT, use_model('s'))
    with pytest.raises(NotImplementedError, match="mode='train' has no CPU fallback"):
        m(torch.zeros(1, 3, 64, 64), [], mode='train')
    with pytest.raises(NotImplementedError, match='computes the loss'):
        m.loss[0](None, None)
    assert isinstance(m._train_loss, Y.YOLOv6Loss) and 'loss.0.proj' in m.state_dict() and not any('_train_loss' in k for k in m.state_dict())
    with pytest.raises(NotImplementedError, match='norm_eval and frozen_stages'):
        Y.YOLOv6EfficientRep('yolov6_s', norm_eval=True)
    with pytest.raises(NotImplementedError, match='norm_eval and frozen_stages'):
        Y.YOLOv6EfficientRep('yolov6_s', frozen_stages=1)
    for st in ('yolov6_t', 'yolov6_m', 'yolov6_l', 'yolov6_x'):
        with pytest.raises(NotImplementedError):
            Y.YOLOv6EfficientRep(st)
    with pytest.raises(NotImplementedError, match='use_dfl'):
        Y.YOLOv6Effidehead('yolov6_s', use_dfl=True)
    with pytest.raises(NotImplementedError, match='use_dfl'):
        Y.YOLOv6Effidehead('yolov6_s', fuse_ab=True)
    with pytest.raises(NotImplementedError, match='deployed'):
        Y.RepVGGBlock(64, 64, deploy=True)
    with pytest.raises(NotImplementedError, match='channels must be'):
        Y.RepVGGBlock(48, 64)
    with pytest.raises(NotImplementedError, match='channels must be'):
        Y.ConvModule(96, 32, 1)
    with pytest.raises(NotImplementedError, match='ReLU only'):
        Y.ConvModule(64, 64, 1, act_cfg=dict(type='SiLU'))
    with pytest.raises(NotImplementedError, match='kernel_size 1 or 3'):
        Y.ConvModule(64, 64, 1, stride=2)
    bn = torch.nn.BatchNorm2d(8)
    assert Y._bn_args(bn)[3] == bn.momentum  # a single-rank BatchNorm passes (and counts the step)
    # the YOLOv5 / YOLOX ConvModule keeps refusing ReLU
    from cvpytorch_b200 import train
    with pytest.raises(NotImplementedError):
        train.ConvModule(64, 64, 3, 1, 1, activation='ReLU')
