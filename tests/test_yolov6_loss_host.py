"""The YOLOv6 loss without a GPU: the oracle against the reference fixture and the edges it covers, the host-side argument checks of the
loss entry points, and the module surface of yolov6_train.YOLOv6Loss."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tools')):
    if p not in sys.path:
        sys.path.insert(0, p)
GOLD = os.path.join(ROOT, 'tests', 'golden', 'yolov6_loss.npz')


def _cases():
    from make_golden_yolov6_loss import CASES
    return CASES


def _oracle_case(name, dev='cpu', grad=True):
    from make_golden_yolov6_loss import CASES, case_inputs
    from oracle import yolov6_loss_oracle as LO
    _, B, H, W, nc, _, assigner, iou_type = CASES[name]
    shapes, scores, distri, gt = case_inputs(name)
    d = distri.to(dev).requires_grad_(grad)
    out, a = LO.losses(shapes, scores.to(dev), d, gt.to(dev), assigner, iou_type, nc)
    return out, a, d


def test_oracle_reproduces_reference_fixture():
    """oracle/yolov6_loss_oracle.py vs the reference YOLOv6Loss (tests/golden/yolov6_loss.npz): foreground set, target_gt_idx, labels,
    target boxes and soft labels bitwise; the loss and the pred_distri gradient within 1e-6 relative; the stored GT rows are the seeds'."""
    from make_golden_yolov6_loss import case_inputs
    g = np.load(GOLD)
    for name in _cases():
        assert np.array_equal(case_inputs(name)[3].numpy(), g[f'{name}_gt'])
        out, a, d = _oracle_case(name)
        (out['iou'] + out['dfl'] + out['class']).backward()
        flat = torch.from_numpy(g[f'{name}_fg']).long()
        assert torch.equal(a['fg'].reshape(-1).nonzero()[:, 0], flat), name
        assert np.array_equal(a['gt_idx'].reshape(-1)[flat].numpy(), g[f'{name}_gt_idx'])
        assert np.array_equal(a['labels'].reshape(-1)[flat].numpy(), g[f'{name}_labels'])
        assert np.array_equal(a['boxes'].reshape(-1, 4)[flat].numpy(), g[f'{name}_boxes'])
        assert np.array_equal(a['scores'].reshape(-1)[flat].numpy(), g[f'{name}_scores'])
        L = float(g[f'{name}_loss'])
        for k, wgt in (('iou', 2.5), ('dfl', 0.5), ('class', 1.0)):
            assert out[k].dtype == torch.float64
            assert abs(float(out[k].detach()) - wgt * L) <= 1e-6 * abs(wgt * L), (name, k)
        ref = torch.zeros(d.numel() // 4, 4)
        ref[flat] = torch.from_numpy(g[f'{name}_grad'])
        err = float((d.grad.reshape(-1, 4) - ref).abs().max() / ref.abs().max())
        assert err <= 1e-6, (name, err)


def test_fixture_covers_edges():
    """The fixture has: an image without GTs, padding rows, a row with x1 + y1 + x2 + y2 <= 0 (not a GT), an anchor claimed by two GTs
    whose winner did not select it, a TAL GT with fewer than 13 positive-metric anchors, both assigners and both IoU types, 80 classes
    at 640²."""
    from make_golden_yolov6_loss import CASES, case_inputs
    from oracle import yolov6_loss_oracle as LO
    assert {(c[6], c[7]) for c in CASES.values()} == {('atss', 'giou'), ('atss', 'siou'), ('tal', 'giou'), ('tal', 'siou')}
    assert any(c[2] == 640 and c[4] == 80 for c in CASES.values())
    seen = dict(empty=False, padding=False, nonpositive=False, stolen=False, few=False)
    for name, (_, B, H, W, nc, per_image, assigner, _) in CASES.items():
        shapes, scores, distri, gt = case_inputs(name)
        labels, boxes, mask, counts = LO.pack(gt, B)
        seen['empty'] |= bool((counts == 0).any())
        seen['padding'] |= bool((counts < boxes.shape[1]).any())
        seen['nonpositive'] |= bool(((boxes.sum(-1) <= 0) & (counts[:, None] > torch.arange(boxes.shape[1]))).any())
        anc, points, per_level, stride = LO.anchors(shapes)
        pts_s = points / stride
        pd = torch.cat([pts_s - distri[..., :2], pts_s + distri[..., 2:]], -1) * stride
        if assigner == 'atss':
            mask_pos, ov = LO.atss(anc, per_level, boxes, mask)
        else:
            mask_pos, ov, align = LO.tal(scores, pd, points, labels, boxes, mask, nc)
            ins = LO.inside(points, boxes)
            npos_metric = ((align * ins) > 0).sum(-1)
            seen['few'] |= bool(((npos_metric < 13) & (npos_metric > 0) & mask).any())
        multi = mask_pos.sum(1) > 1
        win = ov.argmax(1)
        chose = mask_pos.gather(1, win[:, None, :])[:, 0]
        seen['stolen'] |= bool((multi & ~chose).any())
    assert all(seen.values()), seen


def _err(L, rc, text):
    assert rc != 0
    assert text in L.cvb_last_error_string(), L.cvb_last_error_string()


def test_loss_c_abi_rejects_bad_arguments():
    """Every loss entry point rejects bad arguments on the host, before any launch: levels outside [1, 8], B, nc, nt, assigner and
    iou_type out of range, bad grid parameters, strides that are not positive integers, empty maps, too few anchors for TAL, missing or
    misaligned pointers and a short or misaligned workspace."""
    from cvpytorch_b200 import _lib
    from cvpytorch_b200.yolov6_train import loss_params
    L = _lib.lib()
    one, odd = 256, 260
    base = dict(shapes=[(8, 8), (4, 4), (2, 2)], strides=[8, 16, 32], nc=3, B=2, assigner='atss', iou_type='giou')

    def prm(**kw):
        a = dict(base, **kw)
        return loss_params(a['shapes'], a['strides'], a['nc'], a['B'], a['assigner'], a['iou_type'])

    def fwd(p, nt=4, scores=one, distri=one, gt=one, outs=(one,) * 7, ws=one, nbytes=1 << 30):
        return L.cvb_train_yolov6_loss_fwd(ctypes.byref(p), ctypes.c_void_p(scores), ctypes.c_void_p(distri), ctypes.c_void_p(gt), nt,
                                           *[ctypes.c_void_p(o) for o in outs], ctypes.c_void_p(ws), nbytes, None)

    def bwd(p, distri=one, ptrs=(one,) * 5, g=one):
        return L.cvb_train_yolov6_loss_bwd(ctypes.byref(p), ctypes.c_void_p(distri), *[ctypes.c_void_p(o) for o in ptrs], ctypes.c_void_p(g), None)

    bad = []
    p = prm(); p.nlev = 0; bad.append((p, b'1 to 8 levels supported'))
    p = prm(); p.nlev = 9; bad.append((p, b'1 to 8 levels supported'))
    bad.append((prm(B=0), b'batch must be in'))
    bad.append((prm(B=65536), b'batch must be in'))
    bad.append((prm(nc=0), b'num_classes must be in'))
    p = prm(); p.assigner = 2; bad.append((p, b'assigner must be'))
    p = prm(); p.iou_type = -1; bad.append((p, b'iou_type must be'))
    p = prm(); p.grid_cell_size = 0.0; bad.append((p, b'grid_cell_size and ori_img_size'))
    p = prm(); p.ori_img_size = -1.0; bad.append((p, b'grid_cell_size and ori_img_size'))
    p = prm(); p.grid_cell_offset = float('nan'); bad.append((p, b'grid_cell_size and ori_img_size'))
    bad.append((prm(strides=[8, 16, 0]), b'stride must be a positive integer'))
    bad.append((prm(strides=[8, 16.5, 32]), b'stride must be a positive integer'))
    bad.append((prm(strides=[8, 16, float('nan')]), b'stride must be a positive integer'))
    bad.append((prm(shapes=[(8, 8), (0, 4), (2, 2)]), b'map must be h, w in'))
    bad.append((prm(shapes=[(2, 2)], strides=[32], assigner='tal'), b'needs at least 13 anchors'))
    for p, text in bad:
        _err(L, fwd(p), text)
        _err(L, bwd(p), text)
        assert L.cvb_train_yolov6_loss_workspace_bytes(ctypes.byref(p), 4) == 0
    p = prm()
    _err(L, fwd(p, nt=-1), b'nt must be in')
    _err(L, fwd(p, nt=(1 << 24) + 1), b'nt must be in')
    _err(L, fwd(p, scores=0), b'pred_scores (4-byte aligned) and pred_distri (16-byte aligned)')
    _err(L, fwd(p, distri=one + 4), b'pred_scores (4-byte aligned) and pred_distri (16-byte aligned)')
    _err(L, fwd(p, gt=0), b'gt (8-byte aligned) is required')
    _err(L, fwd(p, gt=one + 4), b'gt (8-byte aligned) is required')
    for k in range(7):
        outs = [one] * 7
        outs[k] = 0
        _err(L, fwd(p, outs=outs), b'are required')
    for k in (1, 2, 3, 4, 5, 6):
        outs = [one] * 7
        outs[k] = one + (4 if k == 3 else 2)
        _err(L, fwd(p, outs=outs), b'aligned')
    _err(L, fwd(p, ws=0), b'workspace required')
    _err(L, fwd(p, ws=one + 16), b'256-byte aligned')
    need = L.cvb_train_yolov6_loss_workspace_bytes(ctypes.byref(p), 4)
    assert need > 0 and L.cvb_train_yolov6_loss_workspace_bytes(ctypes.byref(p), 400) > need
    assert L.cvb_train_yolov6_loss_workspace_bytes(ctypes.byref(p), -1) == 0
    _err(L, fwd(p, nbytes=need - 1), b'too small')
    _err(L, bwd(p, distri=0), b'pred_distri and grad_distri are required')
    _err(L, bwd(p, distri=one + 8), b'pred_distri and grad_distri are required')
    for k in range(5):
        ptrs = [one] * 5
        ptrs[k] = 0
        _err(L, bwd(p, ptrs=ptrs), b'are required')
    _err(L, bwd(p, g=0), b'are required')
    _err(L, bwd(p, g=one + 4), b'are required')


def test_loss_module_surface():
    """yolov6_train.YOLOv6Loss: the reference's constructor and `proj` parameter ((1,) for reg_max 0, (17,) for 16); use_dfl, 'ciou' and
    'diou' raise NotImplementedError; CPU inputs raise CvbError; malformed outputs and targets raise ValueError."""
    from cvpytorch_b200 import _lib
    from cvpytorch_b200.yolov6_train import YOLOv6Loss
    m = YOLOv6Loss()
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {'proj': (17,)}
    assert not m.proj.requires_grad and torch.equal(m.proj, torch.linspace(0, 16, 17))
    n = YOLOv6Loss(num_classes=80, reg_max=0, iou_type='siou')
    assert {k: tuple(v.shape) for k, v in n.state_dict().items()} == {'proj': (1,)}
    assert m.warmup_epoch == 4 and m.fpn_strides == [8, 16, 32] and m.loss_weight == {'class': 1.0, 'iou': 2.5, 'dfl': 0.5}
    for kw in (dict(use_dfl=True), dict(iou_type='ciou'), dict(iou_type='diou')):
        with pytest.raises(NotImplementedError):
            YOLOv6Loss(**kw)
    feats = [torch.zeros(1, 1, 8, 8), torch.zeros(1, 1, 4, 4), torch.zeros(1, 1, 2, 2)]
    outs = (feats, torch.zeros(1, 84, 80), torch.zeros(1, 84, 4))
    with pytest.raises(_lib.CvbError):
        m(outs, torch.zeros(2, 6))
    from cvpytorch_b200 import yolov6_train as YT
    with pytest.raises(ValueError):
        YT._gt_rows(torch.zeros(2, 5), 'cpu')
    with pytest.raises(_lib.CvbError):
        YT._gt_rows(torch.zeros(2, 6), 'cpu')
    with pytest.raises(ValueError):
        YT.loss_params([(8, 8)], [8, 16], 3, 1, 'atss', 'giou')
