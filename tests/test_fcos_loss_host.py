"""The FCOS loss without a GPU: the oracle against the reference fixture, the host-side argument checks of the loss entry points, and the
module surface of fcos_train.FCOSLoss."""
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
NAMES = ('cls', 'cnt', 'reg')
LOSSES = ('cls_loss', 'cnt_loss', 'reg_loss', 'total_loss')


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _fixture(g, case):
    n = len([k for k in g.files if k.startswith(f'{case}_cls') and k[len(case) + 4:].isdigit()])
    preds = [[torch.from_numpy(g[f'{case}_{name}{l}']) for l in range(n)] for name in NAMES]
    return preds, torch.from_numpy(g[f'{case}_boxes']), torch.from_numpy(g[f'{case}_labels'])


def test_oracle_reproduces_reference_fixture():
    """oracle/fcos_loss_oracle.py vs the reference FCOSLoss (tests/golden/fcos_loss.npz): the targets bitwise, the four losses and the
    gradients of total_loss with respect to all 15 head tensors within 1e-6 relative; the stored inputs are fixture_case's."""
    from oracle import fcos_loss_oracle as LO
    g = np.load(os.path.join(GOLD, 'fcos_loss.npz'))
    for case in LO.CASES:
        preds, boxes, labels = _fixture(g, case)
        p2, b2, l2 = LO.fixture_case(int(g[f'{case}_seed']), case)
        assert torch.equal(b2, boxes) and torch.equal(l2, labels) and all(torch.equal(x, y) for a, b in zip(p2, preds) for x, y in zip(a, b))
        qs = [[t.clone().requires_grad_(True) for t in lv] for lv in preds]
        out, (cls_t, cnt_t, reg_t, mg) = LO.losses(qs, boxes, labels)
        out[3].backward()
        assert np.array_equal(cls_t.numpy(), g[f'{case}_cls_t'][..., 0])
        assert np.array_equal(cnt_t.numpy(), g[f'{case}_cnt_t'][..., 0])
        assert np.array_equal(reg_t.numpy(), g[f'{case}_reg_t'])
        assert torch.equal(mg >= 0, cnt_t > -1)
        for k, name in enumerate(LOSSES):
            assert _rel(out[k].detach(), g[f'{case}_{name}']) <= 1e-6, (case, name)
        for i, name in enumerate(NAMES):
            for l, q in enumerate(qs[i]):
                assert _rel(q.grad, g[f'{case}_grad_{name}{l}']) <= 1e-6, (case, name, l)


def _point(x, y, stride, H, W):
    """index of the point (x, y) of the given stride in the A axis of an H x W input with strides 8..128."""
    from oracle import fcos_loss_oracle as LO
    o = 0
    for (h, w), s in zip(LO.level_shapes(H, W), LO.STRIDES):
        if s == stride:
            return o + ((y - s // 2) // s) * w + (x - s // 2) // s
        o += h * w
    raise ValueError(stride)


def test_fixture_covers_the_edges():
    """The fixture's GTs hit what they are placed for: padded rows, an image without GTs, labels -1 and nc + 1 on positives, an equal-area
    tie won by the first row, max(l, t, r, b) = 64 and 128 exactly at the limit (in range above, out of range below), a point on a box
    edge and a centre offset equal to the radius (both not positive)."""
    g = np.load(os.path.join(GOLD, 'fcos_loss.npz'))
    from oracle import fcos_loss_oracle as LO
    res = {}
    for case in LO.CASES:
        preds, boxes, labels = _fixture(g, case)
        res[case] = (boxes, labels) + tuple(LO.targets([tuple(c.shape[2:]) for c in preds[0]], boxes, labels))
    boxes, labels, cls_t, _, reg_t, mg = res['a']
    assert bool((labels == -1).any(1).all()) and int((mg[1] >= 0).sum()) == 0 and bool((boxes[1] == -1).all())
    lab = labels[0][mg[0].clamp(min=0)]
    assert bool(((lab == -1) & (mg[0] >= 0)).any()) and bool(((lab == 4) & (mg[0] >= 0)).any())
    a = _point(68, 68, 8, 128, 128)
    assert int(mg[2, a]) == 0 and float(reg_t[2, a].max()) == 64.0  # max = 64 is in (-1, 64]
    a = _point(28, 36, 8, 128, 128)
    assert float(boxes[2, 1, 0]) == 28.0 and int(mg[2, a]) != 1  # l = 0: not inside GT 1
    a = _point(100, 100, 8, 128, 128)
    assert int(mg[2, a]) != 2  # x - cx = 12 = radius: not in the centre region of GT 2
    boxes, labels, cls_t, _, reg_t, mg = res['b']
    a = _point(164, 60, 8, 192, 192)
    assert int(mg[0, a]) == 0 and int(cls_t[0, a]) == 5  # equal areas with row 1: the first row wins
    a = _point(168, 168, 16, 192, 192)
    assert int(mg[0, a]) == 2 and float(reg_t[0, a].max()) == 128.0  # max = 128 is in (64, 128]
    a = _point(104, 104, 16, 192, 192)
    assert int(mg[0, a]) != 3  # max = 64 is not in (64, 128]


def test_oracle_empty_gt_list_is_all_background():
    """m = 0: every point is background (the reference raises in torch.min), num_pos clamps to 1, and only the focal term is non-zero."""
    from oracle import fcos_loss_oracle as LO
    preds = LO.head_outputs(2, 3, LO.level_shapes(64, 64), LO.STRIDES, torch.Generator().manual_seed(3))
    out, (cls_t, cnt_t, reg_t, mg) = LO.losses(preds, torch.zeros(2, 0, 4), torch.zeros(2, 0, dtype=torch.long))
    assert bool((mg == -1).all()) and bool((cls_t == 0).all()) and bool((cnt_t == -1).all()) and bool((reg_t == -1).all())
    assert float(out[1]) == 0.0 and float(out[2]) == 0.0 and float(out[0]) > 0.0


def _err(L, rc, text):
    assert rc != 0
    assert text in L.cvb_last_error_string(), L.cvb_last_error_string()


def test_loss_c_abi_rejects_bad_arguments():
    """Every loss entry point rejects bad arguments on the host, before the device is touched: nlev outside [1, 8], per-level shapes
    against B, nc, the 1 and 4 channels and equal h, w; nc < 1, B < 1, m outside [0, 1024]; a stride that is not a positive integer;
    lo >= hi; missing or misaligned pointers; a short or misaligned workspace."""
    from cvpytorch_b200 import _lib
    L = _lib.lib()
    one, odd = 256, 258
    base = (((2, 3, 8, 8), (2, 1, 8, 8), (2, 4, 8, 8)), ((2, 3, 4, 4), (2, 1, 4, 4), (2, 4, 4, 4)))

    def args(shapes=base, strides=(8.0, 16.0), limits=((-1.0, 64.0), (64.0, 128.0)), B=2, m=4, ptr=one, boxes=one, labels=one):
        n = len(shapes)
        P = (ctypes.c_void_p * n)(*[ptr] * n)
        return (P, (ctypes.c_void_p * n)(*[one] * n), (ctypes.c_void_p * n)(*[one] * n),
                (ctypes.c_int32 * (12 * n))(*[d for lv in shapes for s in lv for d in s]), (ctypes.c_float * len(strides))(*strides),
                (ctypes.c_float * (2 * len(limits)))(*[v for r in limits for v in r]), n, ctypes.c_void_p(boxes), ctypes.c_void_p(labels), B, m)

    def fwd(a, mg=one, npos=one, tgt=None, out=one, ws=one, nbytes=1 << 30):
        return L.cvb_train_fcos_loss_fwd(*a, ctypes.c_void_p(mg), ctypes.c_void_p(npos), ctypes.c_void_p(tgt), ctypes.c_void_p(out), ctypes.c_void_p(ws),
                                         nbytes, None)

    def bwd(a, grads=None, gout=one, npos=one):
        n = a[6]
        g = grads if grads is not None else [(ctypes.c_void_p * n)(*[one] * n)] * 3
        return L.cvb_train_fcos_loss_bwd(*a, ctypes.c_void_p(one), ctypes.c_void_p(npos), ctypes.c_void_p(gout), *g, None)

    def lv(c, n, r):
        return (c, n, r)
    for call in (fwd, bwd):
        _err(L, call(args(shapes=[base[0]] * 9, strides=[8.0] * 9, limits=[(-1.0, 64.0)] * 9)), b'1 to 8 levels supported')
        _err(L, call(args(shapes=(), strides=(), limits=())), b'1 to 8 levels supported')
        _err(L, call(args(shapes=(lv((3, 3, 8, 8), (2, 1, 8, 8), (2, 4, 8, 8)), base[1]))), b'cls_logits must be')
        _err(L, call(args(shapes=(base[0], lv((2, 4, 4, 4), (2, 1, 4, 4), (2, 4, 4, 4))))), b'cls_logits must be')
        _err(L, call(args(shapes=(lv((2, 3, 0, 8), (2, 1, 0, 8), (2, 4, 0, 8)), base[1]))), b'cls_logits must be')
        _err(L, call(args(shapes=(lv((2, 3, 8, 8), (2, 2, 8, 8), (2, 4, 8, 8)), base[1]))), b'cnt_logits must be')
        _err(L, call(args(shapes=(lv((2, 3, 8, 8), (2, 1, 8, 7), (2, 4, 8, 8)), base[1]))), b'cnt_logits must be')
        _err(L, call(args(shapes=(lv((2, 3, 8, 8), (1, 1, 8, 8), (2, 4, 8, 8)), base[1]))), b'cnt_logits must be')
        _err(L, call(args(shapes=(lv((2, 3, 8, 8), (2, 1, 8, 8), (2, 3, 8, 8)), base[1]))), b'reg_preds must be')
        _err(L, call(args(shapes=(lv((2, 3, 8, 8), (2, 1, 8, 8), (2, 4, 7, 8)), base[1]))), b'reg_preds must be')
        _err(L, call(args(shapes=tuple(lv((2, 0, h, h), (2, 1, h, h), (2, 4, h, h)) for h in (8, 4)))), b'num_classes must be in')
        _err(L, call(args(B=0)), b'batch must be >= 1')
        _err(L, call(args(m=1025)), b'm must be in [0, 1024]')
        _err(L, call(args(m=-1)), b'm must be in [0, 1024]')
        _err(L, call(args(strides=(8.0, 0.0))), b'stride must be a positive integer')
        _err(L, call(args(strides=(-8.0, 16.0))), b'stride must be a positive integer')
        _err(L, call(args(strides=(8.0, 16.5))), b'stride must be a positive integer')
        _err(L, call(args(strides=(8.0, float('nan')))), b'stride must be a positive integer')
        _err(L, call(args(limits=((-1.0, 64.0), (128.0, 128.0)))), b'lo < hi')
        _err(L, call(args(limits=((64.0, -1.0), (64.0, 128.0)))), b'lo < hi')
        _err(L, call(args(limits=((float('nan'), 64.0), (64.0, 128.0)))), b'lo < hi')
        _err(L, call(args(ptr=odd)), b'output missing or not 4-byte aligned')
        _err(L, call(args(ptr=0)), b'output missing or not 4-byte aligned')
        _err(L, call(args(boxes=one + 4)), b'boxes (16-byte aligned)')
        _err(L, call(args(labels=0)), b'boxes (16-byte aligned) and labels')
        _err(L, call(args(labels=odd)), b'labels (4-byte aligned)')
    # m = 0 needs no boxes or labels
    _err(L, fwd(args(m=0, boxes=0, labels=0), mg=0), b'matched_gt, num_pos and out are required')
    _err(L, fwd(args(), npos=odd), b'4-byte aligned')
    _err(L, fwd(args(), out=odd), b'4-byte aligned')
    _err(L, fwd(args(), tgt=odd), b'targets must be 4-byte aligned')
    _err(L, fwd(args(), ws=one + 16), b'256-byte aligned')
    _err(L, fwd(args(), ws=0), b'workspace required')
    need = L.cvb_train_fcos_loss_workspace_bytes(2, 80, 3)
    assert need > 0 and L.cvb_train_fcos_loss_workspace_bytes(0, 80, 3) == 0 and L.cvb_train_fcos_loss_workspace_bytes(2, 80, 0) == 0
    assert L.cvb_train_fcos_loss_workspace_bytes(2, 8000, 80) > L.cvb_train_fcos_loss_workspace_bytes(2, 8000, 3)
    _err(L, fwd(args(), nbytes=need - 1), b'too small')
    _err(L, bwd(args(), gout=odd), b'grad_out are required, 4-byte aligned')
    _err(L, bwd(args(), npos=0), b'grad_out are required, 4-byte aligned')
    _err(L, bwd(args(), grads=[(ctypes.c_void_p * 2)(one, one), (ctypes.c_void_p * 2)(one, odd), (ctypes.c_void_p * 2)(one, one)]),
         b'gradient missing or not 4-byte aligned')
    n = 2
    _err(L, L.cvb_train_fcos_loss_bwd(*args(), ctypes.c_void_p(one), ctypes.c_void_p(one), ctypes.c_void_p(one), None,
                                      (ctypes.c_void_p * n)(one, one), (ctypes.c_void_p * n)(one, one), None), b'gcls, gcnt and greg are required')


def test_loss_module_surface():
    """fcos_train.FCOSLoss: the reference's constructor defaults, no parameters or buffers; CPU inputs raise CvbError (no fallback);
    mismatched level counts and malformed targets raise ValueError."""
    from cvpytorch_b200 import _lib, fcos_train as FT
    m = FT.FCOSLoss()
    assert m.strides == [8, 16, 32, 64, 128] and m.limit_range == [[-1, 64], [64, 128], [128, 256], [256, 512], [512, 999999]]
    assert list(m.state_dict()) == [] and list(m.parameters()) == [] and list(m.buffers()) == []
    preds = [[torch.zeros(1, 3, 4, 4)] * 5, [torch.zeros(1, 1, 4, 4)] * 5, [torch.zeros(1, 4, 4, 4)] * 5]
    with pytest.raises(_lib.CvbError):
        m(preds, torch.zeros(1, 2, 4), torch.zeros(1, 2, dtype=torch.long))
    with pytest.raises(ValueError):
        m([p[:4] for p in preds], torch.zeros(1, 2, 4), torch.zeros(1, 2, dtype=torch.long))
    with pytest.raises(ValueError):
        FT.FCOSLoss(strides=[8, 16], limit_range=[[-1, 64]])
    with pytest.raises(ValueError):
        FT._loss_targets(torch.zeros(1, 2, 5), torch.zeros(1, 2), 1, 3, None)
    with pytest.raises(ValueError):
        FT._loss_targets(torch.zeros(1, 2, 4), torch.zeros(1, 3), 1, 3, None)
    with pytest.raises(ValueError):
        FT._loss_targets(torch.zeros(1, 1025, 4), torch.zeros(1, 1025), 1, 3, None)
    with pytest.raises(_lib.CvbError):
        FT._loss_targets(torch.zeros(1, 2, 4), torch.zeros(1, 2), 1, 3, None)
