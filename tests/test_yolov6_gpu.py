"""YOLOv6-n / YOLOv6-s on the H100 kernels against the reference fixtures (tests/golden/yolov6_*.npz) and the oracle (oracle/yolov6_oracle.py):
backbone / neck / head within 1e-3 of max|ref| (the tolerance of test_yolox_gpu.py), BiFusion at odd sizes, the decode kernel, the fused
640² graph with bit-identical NMS on the device's own z, the 'val' contract, batch independence and CUDA-graph replay."""
import os
import sys

import numpy as np
import pytest
import torch

from cvpytorch_b200 import ops
from cvpytorch_b200 import yolov6_models as M
from oracle import yolov6_oracle as V6

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_yolov6_host import DICT, use_model  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
SEEDS = {'n': 606, 's': 616}
TOL = 1e-3
DEV = torch.device('cuda:0')


def model(stype, seed=None):
    m = M.YOLOv6(DICT, use_model(stype))
    sd = m.state_dict()
    m.load_state_dict(V6.seeded_state_dict([(k, v.shape) for k, v in sd.items()], SEEDS[stype] if seed is None else seed), strict=True)
    return m.to(DEV).eval()


def sample_err(t, f, key):
    """error of t at the fixture's sample positions against the reference's samples, relative to the reference tensor's max|t|"""
    return float((V6.subsample(t.cpu()).double() - torch.from_numpy(f[key + '_sample']).double()).abs().max() / float(f[key + '_max']))


@pytest.mark.parametrize('stype', ['n', 's'])
def test_modules_against_reference_128(stype):
    """Each module on the reference's samples and, in full, on the oracle (pinned to the reference by test_yolov6_oracle_golden.py); the
    neck and head get the oracle's inputs, so an error does not carry over from the module before."""
    f = np.load(os.path.join(GOLD, 'yolov6_fwd128.npz'))
    m = model(stype)
    x = V6.fixture_input(V6.FWD_SEED, V6.FWD_SHAPE)
    zo, d = V6.forward(x, {k: v.cpu() for k, v in m.state_dict().items()})
    b = m.backbone(x.to(DEV))
    for i in range(4):
        assert sample_err(b[i], f, f'{stype}_backbone_{i}') < TOL and V6.rel_err(b[i].cpu(), d['backbone'][i]) < TOL, ('backbone', i)
    n = m.neck([t.to(DEV) for t in d['backbone']])
    for i in range(3):
        assert sample_err(n[i], f, f'{stype}_neck_{i}') < TOL and V6.rel_err(n[i].cpu(), d['neck'][i]) < TOL, ('neck', i)
    feats, cls, reg = m.head([t.to(DEV) for t in d['neck']])
    for i in range(3):
        assert sample_err(feats[i], f, f'{stype}_stems_{i}') < TOL and V6.rel_err(feats[i].cpu(), d['stems'][i]) < TOL, ('stems', i)
    assert sample_err(cls, f, f'{stype}_cls') < TOL and V6.rel_err(cls.cpu(), d['cls']) < TOL
    assert V6.rel_err(reg.cpu(), f[f'{stype}_reg']) < TOL
    m.predict(x.to(DEV))
    z = m._graph_for(x.to(DEV))['z'].cpu()
    assert sample_err(z, f, f'{stype}_z') < TOL and V6.rel_err(z, zo) < TOL


@pytest.mark.parametrize('h,w', [(5, 7), (3, 3), (4, 6)])
def test_bifusion_odd_sizes(h, w):
    torch.manual_seed(h * 31 + w)
    bf = M.BiFusion([48, 32], 32)
    for mod in bf.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eps = 1e-3
    sd = V6.seeded_state_dict([(k, v.shape) for k, v in bf.state_dict().items()], h * 7 + w)
    bf.load_state_dict(sd)
    bf = bf.to(DEV).eval()
    xs = [torch.randn(2, 32, h, w), torch.randn(2, 48, 2 * h, 2 * w), torch.randn(2, 32, 4 * h, 4 * w)]
    sdp = {'b.' + k: v for k, v in sd.items()}
    with torch.no_grad():
        ref = V6.bifusion(xs[0], xs[1], xs[2], sdp, 'b')
    out = bf([x.to(DEV) for x in xs])
    assert V6.rel_err(out.cpu(), ref) < TOL


def run_decode(cls, reg, strides, conf):
    """cls / reg: lists of fp32 NHWC CUDA tensors per level -> (z, det, idx, cnt) through cvb_yolov6_decode + ops.yolo_nms(hist_ready)."""
    B, nc = cls[0].shape[0], cls[0].shape[3]
    A = sum(c.shape[1] * c.shape[2] for c in cls)
    z = torch.full((B, A, nc + 5), float('nan'), device=DEV)
    ws = ops.NmsWorkspace(B, A, nc, device=DEV)
    ops.nms_reset(ws)
    off = 0
    for c, r, s in zip(cls, reg, strides):
        cv, rv = ops.CvbView(), ops.CvbView()
        for v, t in ((cv, c), (rv, r)):
            v.base, v.B, v.H, v.W, v.C, v.c_pitch, v.plane_stride = t.data_ptr(), t.shape[0], t.shape[1], t.shape[2], t.shape[3], t.shape[3], 0
        ops.yolov6_decode(cv, rv, nc, s, z, A, off, ws, conf, True)
        off += c.shape[1] * c.shape[2]
    det, idx, cnt = ops.yolo_nms(z, ws, conf, 0.65, True, hist_ready=True)
    torch.cuda.synchronize()
    return z, det, idx, cnt, ws


@pytest.mark.parametrize('nc', [1, 80, 13])
@pytest.mark.parametrize('conf', [0.03, 0.25])
def test_decode_kernel_against_oracle(nc, conf):
    g = torch.Generator().manual_seed(nc * 100 + int(conf * 100))
    shapes = [(13, 11), (7, 6), (3, 3)]  # odd level sizes
    cls = [torch.randn(2, h, w, nc, generator=g) * 2 - 3 for h, w in shapes]
    reg = [torch.rand(2, h, w, 4, generator=g) * 4 for h, w in shapes]
    z, det, idx, cnt, ws = run_decode([c.to(DEV) for c in cls], [r.to(DEV) for r in reg], [8, 16, 32], conf)
    zo = V6.detect(torch.cat([torch.sigmoid(c).reshape(2, -1, nc) for c in cls], 1), torch.cat([r.reshape(2, -1, 4) for r in reg], 1), shapes)
    zc = z.cpu()
    assert torch.equal(zc[..., :5], zo[..., :5])  # box and objectness: the reference's fp32 operation order, bit for bit
    assert (zc[..., 5:] - zo[..., 5:]).abs().max() < 1e-6  # sigmoid_fast
    assert int(ws.status[0]) == 0
    ref = V6.non_max_suppression(zc.numpy(), conf, 0.65)
    for b in range(2):
        k = int(cnt[b])
        assert k == ref[b][0].shape[0]
        assert np.array_equal(det[b, :k].cpu().numpy(), ref[b][0]) and np.array_equal(idx[b, :k].cpu().numpy().astype(np.int64), ref[b][1])


def test_fused_640_s_against_oracle():
    m = model('s')
    torch.manual_seed(640)
    x = torch.randn(2, 3, 640, 640)
    det, idx, cnt = m.predict(x.to(DEV))
    torch.cuda.synchronize()
    z = m._graph_for(x.to(DEV))['z'].cpu()
    zo, _ = V6.forward(x, {k: v.cpu() for k, v in m.state_dict().items()})
    assert V6.rel_err(z, zo) < TOL
    assert int(m.nms_status(x.to(DEV))[0]) == 0
    ref = V6.non_max_suppression(z.numpy(), m.conf_thres, m.iou_thres)
    for b in range(2):
        k = int(cnt[b])
        assert k == ref[b][0].shape[0] and k > 0
        assert np.array_equal(idx[b, :k].cpu().numpy().astype(np.int64), ref[b][1])
        assert np.array_equal(det[b, :k].cpu().numpy(), ref[b][0])


def test_post320_against_reference_rows():
    """s at 320²: the device z against the reference's boxes and candidate scores, and the device NMS on the device's z against the oracle
    NMS on the same z."""
    p = np.load(os.path.join(GOLD, 'yolov6_post320.npz'))
    m = model('s')
    x = V6.fixture_input(V6.POST_SEED, V6.POST_SHAPE).to(DEV)
    det, idx, cnt = m.predict(x)
    torch.cuda.synchronize()
    z = m._graph_for(x)['z'].cpu()
    zmax = float(p['z_max'])
    assert float((z[..., :4] - torch.from_numpy(p['boxes'])).abs().max()) < TOL * zmax
    r, c = torch.from_numpy(p['rows'].astype(np.int64)), torch.from_numpy(p['classes'].astype(np.int64))
    assert float((z[r[:, 0], r[:, 1], c + 5] - torch.from_numpy(p['scores'])).abs().max()) < TOL * zmax
    d, i = V6.non_max_suppression(z.numpy(), 0.03, 0.65)[0]
    k = int(cnt[0])
    assert k == d.shape[0] and np.array_equal(det[0, :k].cpu().numpy(), d) and np.array_equal(idx[0, :k].cpu().numpy().astype(np.int64), i)
    # the reference's detections: the same count up to candidates whose score sits within the z tolerance of the threshold
    assert abs(k - p['det'].shape[0]) <= 3


def test_val_contract_and_batch_independence():
    m = model('n')
    torch.manual_seed(5)
    x = torch.randn(3, 3, 256, 320)
    targets = [dict(pads=torch.tensor([8.0, 16.0]), scales=torch.tensor([0.5, 0.5]), width=torch.tensor(600.0), height=torch.tensor(480.0))
               for _ in range(3)]
    losses, outs = m(x.to(DEV), targets, mode='val')
    assert set(losses) == {'loss'} and float(losses['loss']) == 0.0
    assert len(outs) == 3 and all(set(o) == {'boxes', 'labels', 'scores'} for o in outs)
    det, _, cnt = m.predict(x.to(DEV))
    for b in range(3):
        k = int(cnt[b])
        rows = det[b, :k].cpu().clone()
        rows[:, [0, 2]] = ((rows[:, [0, 2]] - 16.0) / 0.5).clamp(0, 600)
        rows[:, [1, 3]] = ((rows[:, [1, 3]] - 8.0) / 0.5).clamp(0, 480)
        assert torch.allclose(outs[b]['boxes'], rows[:, :4], atol=1e-3) and torch.equal(outs[b]['scores'], rows[:, 4])
        assert torch.equal(outs[b]['labels'], rows[:, 5])
    # each image alone gives its rows of the batch
    full = [det[b, :int(cnt[b])].cpu().clone() for b in range(3)]
    for b in range(3):
        d1, _, c1 = m.predict(x[b:b + 1].to(DEV))
        assert int(c1[0]) == full[b].shape[0] and torch.equal(d1[0, :int(c1[0])].cpu(), full[b])


def test_thresholds_are_part_of_the_graph_key():
    m = model('n')
    x = torch.randn(1, 3, 128, 128).to(DEV)
    c1 = int(m.predict(x)[2][0])
    m.conf_thres = 0.5
    c2 = int(m.predict(x)[2][0])
    assert c2 <= c1 and len(m._graphs) == 2


def test_cuda_graph_replay():
    m = model('n')
    x = torch.randn(2, 3, 192, 192).to(DEV)
    det, idx, cnt = m.predict(x)
    ref = (det.clone(), idx.clone(), cnt.clone())
    G = m._graph_for(x)
    G['g'].capture()
    det.zero_()
    G['g'].replay()
    torch.cuda.synchronize()
    assert torch.equal(det, ref[0]) and torch.equal(idx, ref[1]) and torch.equal(cnt, ref[2])
