"""YOLOv6 drop-ins on the host (no GPU): constructor surface and state_dict keys against the reference's (tests/golden/yolov6_keys.npz), the
refusals, and the two weight remaps of the H100 graph checked in float64 against F.conv2d / F.conv_transpose2d."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cvpytorch_b200 import yolov6_models as M
from oracle import yolov6_oracle as V6

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
DICT = [{f'c{i}': 1.0} for i in range(80)]


def use_model(stype):
    """USE_MODEL of conf/det/yolov6/coco_yolov6_{n,s}.yml."""
    cfg = dict(TYPE=f'yolov6_{stype}',
               BACKBONE={'name': 'YOLOv6EfficientRep', 'out_stages': [1, 2, 3, 4], 'output_stride': 32, 'pretrained': False},
               NECK={'name': 'YOLOv6RepBiPAN', 'in_channels': [128, 256, 512, 1024], 'mid_channels': [128, 128, 256],
                     'out_channels': [128, 256, 512], 'num_blocks': [12, 12, 12, 12]},
               HEAD={'name': 'YOLOv6Effidehead', 'num_classes': 80, 'in_channels': [128, 256, 512], 'use_dfl': False, 'fuse_ab': False})
    if stype == 'n':
        cfg.update(DETECT={'name': 'YOLOv6Detect', 'in_channels': [128, 256, 512]},
                   LOSS={'name': 'YOLOv6Loss', 'num_classes': 80, 'use_dfl': False, 'reg_max': 0, 'iou_type': 'siou'})
    else:
        cfg.update(DETECT={'name': 'YOLOv6Detect', 'num_classes': 80, 'in_channels': [128, 256, 512], 'use_dfl': False, 'fuse_ab': False},
                   LOSS={'name': 'YOLOv6Loss', 'num_classes': 80})
    return cfg


class Attr:
    def __init__(self, d):
        self.__dict__.update(d)


@pytest.mark.parametrize('stype', ['n', 's'])
@pytest.mark.parametrize('as_attr', [False, True])
def test_state_dict_keys_and_strict_load(stype, as_attr):
    k = np.load(os.path.join(GOLD, 'yolov6_keys.npz'))
    cfg = use_model(stype)
    m = M.YOLOv6(DICT, Attr(cfg) if as_attr else cfg)
    sd = m.state_dict()
    assert list(sd.keys()) == list(k[f'{stype}_keys'])
    assert [','.join(str(s) for s in v.shape) for v in sd.values()] == list(k[f'{stype}_shapes'])
    assert sum(p.numel() for p in m.parameters()) == int(k[f'{stype}_params'])
    ref = V6.seeded_state_dict([(a, v.shape) for a, v in sd.items()], 7)
    m.load_state_dict(ref, strict=True)
    assert all(torch.equal(m.state_dict()[a], ref[a]) for a in ref)


def test_module_surfaces():
    bb = M.YOLOv6EfficientRep(subtype='yolov6_s', out_stages=[1, 2, 3, 4], output_stride=32, pretrained=False)
    assert bb.out_channels == [32, 64, 128, 256, 512] and bb.num_blocks == [2, 4, 6, 2]
    nk = M.YOLOv6RepBiPAN(subtype='yolov6_n', in_channels=[128, 256, 512, 1024], mid_channels=[128, 128, 256], out_channels=[128, 256, 512],
                          num_blocks=[12, 12, 12, 12])
    assert nk.in_channels == [32, 64, 128, 256] and nk.mid_channels == [32, 32, 64] and nk.num_blocks == [4, 4, 4, 4]
    hd = M.YOLOv6Effidehead(subtype='yolov6_s', num_classes=80, in_channels=[128, 256, 512], use_dfl=False, fuse_ab=False)
    assert hd.in_channels == [64, 128, 256] and hd.reg_max == 0 and tuple(hd.proj.shape) == (1,)
    assert all(bn.eps == 1e-3 for bn in bb.modules() if isinstance(bn, torch.nn.BatchNorm2d))
    dt = M.YOLOv6Detect(num_classes=80, in_channels=[128, 256, 512], use_dfl=False, fuse_ab=False)
    assert len(dt.state_dict()) == 0
    bf = M.BiFusion([64, 32], 32)
    assert [n for n, _ in bf.named_children()] == ['cv1', 'cv2', 'cv3', 'upsample', 'downsample']


@pytest.mark.parametrize('stype,match', [('t', '24-channel stem'), ('m', 'reg_max = 16'), ('l', 'reg_max = 16'), ('x', 'reg_max = 16')])
def test_refused_widths(stype, match):
    cfg = use_model('s')
    cfg['TYPE'] = f'yolov6_{stype}'
    with pytest.raises(NotImplementedError, match=match):
        M.YOLOv6(DICT, cfg)
    with pytest.raises(NotImplementedError, match=match):
        M.YOLOv6EfficientRep(subtype=f'yolov6_{stype}')
    with pytest.raises(NotImplementedError, match=match):
        M.YOLOv6Effidehead(subtype=f'yolov6_{stype}')


@pytest.mark.parametrize('key', ['use_dfl', 'fuse_ab'])
def test_refused_head_options(key):
    for part in ('HEAD', 'DETECT'):
        cfg = use_model('s')
        cfg[part] = dict(cfg[part], **{key: True})
        with pytest.raises(NotImplementedError, match=key):
            M.YOLOv6(DICT, cfg)


def test_refused_train_mode():
    m = M.YOLOv6(DICT, use_model('n'))
    with pytest.raises(NotImplementedError, match='train'):
        m(torch.zeros(1, 3, 64, 64), [], mode='train')
    with pytest.raises(NotImplementedError):
        m.loss[0](None, None)
    assert m(torch.zeros(1, 3, 64, 64), None, mode='infer') is None


def test_stem_s2d_remap_float64():
    """3x3 / stride 2 / pad 1 conv of the image == 3x3 / stride 1 / pad 1 conv of its space-to-depth map with the remapped weights."""
    g = torch.Generator().manual_seed(3)
    w = torch.randn(16, 3, 3, 3, generator=g, dtype=torch.float64)
    x = torch.randn(2, 3, 22, 30, generator=g, dtype=torch.float64)
    ref = F.conv2d(x, w, None, 2, 1)
    s2d = torch.zeros(2, 16, 11, 15, dtype=torch.float64)
    for dy in range(2):
        for dx in range(2):
            s2d[:, (dy * 2 + dx) * 3:(dy * 2 + dx) * 3 + 3] = x[:, :, dy::2, dx::2]
    w2 = M.repvgg_stem_weights_to_s2d(w)
    assert torch.equal(w2[:, :, 2, :], torch.zeros_like(w2[:, :, 2, :])) and torch.equal(w2[:, :, :, 2], torch.zeros_like(w2[:, :, :, 2]))
    assert torch.equal(w2[:, 12:], torch.zeros_like(w2[:, 12:]))
    assert (F.conv2d(s2d, w2, None, 1, 1) - ref).abs().max() < 1e-12


@pytest.mark.parametrize('h,w', [(5, 7), (4, 4)])
def test_conv_transpose_gemm_depth_to_space_float64(h, w):
    """ConvTranspose2d(c, c, 2, stride=2) == the packed 1x1 GEMM ([py][px][cout] columns) followed by the 2x depth-to-space."""
    g = torch.Generator().manual_seed(h * 10 + w)
    c = 16
    ct = torch.nn.ConvTranspose2d(c, c, 2, stride=2, bias=True).double()
    with torch.no_grad():
        ct.weight.copy_(torch.randn(ct.weight.shape, generator=g, dtype=torch.float64))
        ct.bias.copy_(torch.randn(ct.bias.shape, generator=g, dtype=torch.float64))
    x = torch.randn(2, c, h, w, generator=g, dtype=torch.float64)
    w64, b64 = M.conv_transpose2_weights(ct.weight, ct.bias)
    gemm = F.conv2d(x, w64, b64)  # [B, 4c, h, w], channel (py*2+px)*c + o
    out = torch.zeros(2, c, 2 * h, 2 * w, dtype=torch.float64)
    for py in range(2):
        for px in range(2):
            out[:, :, py::2, px::2] = gemm[:, (py * 2 + px) * c:(py * 2 + px + 1) * c]
    assert (out - F.conv_transpose2d(x, ct.weight.detach(), ct.bias.detach(), stride=2)).abs().max() < 1e-12
