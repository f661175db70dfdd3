"""The segmentation loss without a GPU: the oracle against the reference fixture and against F.interpolate, the host-side argument checks of
the loss entry points, and the module surface of seg_train."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def test_oracle_reproduces_reference_fixture():
    """oracle/seg_loss_oracle.py vs the reference loss_forward + CrossEntropyLoss2d (tests/golden/seg_loss.npz): the stored inputs are
    fixture_case's; the loss within 1e-6 relative and the gradient within 1e-6 of its largest element; all ignored: NaN and zeros."""
    from oracle import seg_loss_oracle as SO
    g = np.load(os.path.join(GOLD, 'seg_loss.npz'))
    for case in SO.CASES:
        pred, target, ignore, lw = SO.fixture_case(case)
        assert np.array_equal(pred.numpy(), g[f'{case}_pred']) and np.array_equal(target.numpy(), g[f'{case}_target']), case
        assert target.numpy().dtype == g[f'{case}_target'].dtype
        assert int(g[f'{case}_ignore_index']) == ignore and float(g[f'{case}_loss_weight']) == np.float32(lw)
        q = pred.double().requires_grad_(True)
        out = SO.loss(q, target, ignore, lw)
        out.backward()
        if case == 'ignored':
            assert np.isnan(g[f'{case}_loss']) and torch.isnan(out) and not g[f'{case}_grad'].any() and not bool(q.grad.any())
            continue
        assert _rel(out.detach(), g[f'{case}_loss']) <= 1e-6, case
        assert _rel(q.grad, g[f'{case}_grad']) <= 1e-6, case
    # what the cases are built to cover
    _, t, _, _ = SO.fixture_case('x4')
    assert t.dtype == torch.uint8 and bool((t[1] == 255).all()) and bool((t[:, :3] == 255).all()) and bool((t[0] != 255).any())
    assert SO.CASES['x8'][7] == 0.4 and SO.CASES['x8'][4] == 8 * SO.CASES['x8'][2]


def test_oracle_matrices_match_interpolate():
    """z = Rh x Rw^T equals fp64 F.interpolate(bilinear, align_corners=False, size=) over up, down, integer, non-integer and identity size
    pairs.  The matrices take torch's fp32 index arithmetic (that of fp32 inputs), fp64 F.interpolate a double one: the source positions,
    and so the weights, differ by about in_size * 2^-24, which bounds the difference."""
    from oracle import seg_loss_oracle as SO
    g = torch.Generator().manual_seed(5)
    pairs = [(1, 1), (1, 7), (7, 1), (2, 3), (3, 2), (5, 5), (16, 64), (8, 64), (13, 96), (29, 192), (40, 17), (56, 23), (128, 512),
             (256, 1024), (33, 100), (100, 33), (64, 64), (3, 9), (9, 3), (17, 31)]
    for h, H in pairs:
        for w, W in ((h, H), (5, 12), (12, 5)):
            x = torch.randn(2, 3, h, w, generator=g, dtype=torch.float64)
            ref = F.interpolate(x, size=(H, W), mode='bilinear', align_corners=False)
            got = SO.upsample(x, H, W)
            assert float((got - ref).abs().max()) <= max(h, w) * 2.0 ** -22 * float(x.abs().max()), (h, w, H, W)
            if (h, w) == (H, W):
                assert torch.equal(got, x)
            Rh = SO.interp_matrix(H, h)
            assert torch.allclose(Rh.sum(1), torch.ones(H, dtype=torch.float64), atol=1e-6) and int((Rh != 0).sum(1).max()) <= 2


def test_oracle_refuses_out_of_range_labels():
    from oracle import seg_loss_oracle as SO
    pred = torch.zeros(1, 3, 4, 4, dtype=torch.float64)
    for bad in (3, -1):
        t = torch.zeros(1, 8, 8, dtype=torch.long)
        t[0, 2, 2] = bad
        with pytest.raises(IndexError):
            SO.loss(pred, t)


def _err(L, rc, text):
    assert rc != 0
    assert text in L.cvb_last_error_string(), L.cvb_last_error_string()


def test_loss_c_abi_rejects_bad_arguments():
    """Both entry points reject bad arguments on the host, before any launch: C outside [1, nc_max], B / h / w / H / W outside [1, 65535],
    B H W >= 2^31, an unknown dtype code, negative strides, missing or misaligned pointers, a missing, misaligned or short workspace."""
    from cvpytorch_b200 import _lib
    L = _lib.lib()
    one = 1 << 12
    ncm = L.cvb_train_seg_ce_nc_max()
    assert ncm >= 256

    def args(B=2, C=19, h=8, w=8, H=32, W=32, labels=one, dtype=_lib.CVB_SEG_U8, strides=(1024, 32, 1), preds=one):
        return (ctypes.c_void_p(preds), B, C, h, w, ctypes.c_void_p(labels), dtype, H, W, *strides, 255, 1.0)

    def fwd(a, lse=one, record=one, loss=one, ws=one, nbytes=1 << 30):
        return L.cvb_train_seg_ce_fwd(*a, ctypes.c_void_p(lse), ctypes.c_void_p(record), ctypes.c_void_p(loss), ctypes.c_void_p(ws), nbytes, None)

    def bwd(a, lse=one, record=one, gout=one, grad=one):
        return L.cvb_train_seg_ce_bwd(*a, ctypes.c_void_p(lse), ctypes.c_void_p(record), ctypes.c_void_p(gout), ctypes.c_void_p(grad), None)

    for call in (fwd, bwd):
        _err(L, call(args(C=0)), b'C must be in [1, %d]' % ncm)
        _err(L, call(args(C=ncm + 1)), b'C must be in [1, %d]' % ncm)
        _err(L, call(args(B=0)), b'B must be in')
        _err(L, call(args(B=65536)), b'B must be in')
        _err(L, call(args(h=0)), b'preds h, w must be in')
        _err(L, call(args(w=65536)), b'preds h, w must be in')
        _err(L, call(args(H=0)), b'label H, W must be in')
        _err(L, call(args(W=70000)), b'label H, W must be in')
        _err(L, call(args(B=1024, H=2048, W=1024)), b'B x H x W must be below 2^31')
        _err(L, call(args(dtype=3)), b'unknown label dtype code')
        _err(L, call(args(dtype=-1)), b'unknown label dtype code')
        _err(L, call(args(strides=(1024, -32, 1))), b'label strides must be >= 0')
        _err(L, call(args(strides=(1 << 40, 32, 1))), b'label strides too large')
        _err(L, call(args(preds=0)), b'preds missing or not 4-byte aligned')
        _err(L, call(args(preds=one + 2)), b'preds missing or not 4-byte aligned')
        _err(L, call(args(labels=0)), b'labels missing or not aligned')
        _err(L, call(args(labels=one + 2, dtype=_lib.CVB_SEG_I32)), b'labels missing or not aligned')
        _err(L, call(args(labels=one + 4, dtype=_lib.CVB_SEG_I64)), b'labels missing or not aligned')
    _err(L, fwd(args(), lse=0), b'lse, loss (4-byte aligned) and record (8-byte aligned) are required')
    _err(L, fwd(args(), record=one + 4), b'record (8-byte aligned)')
    _err(L, fwd(args(), loss=one + 1), b'are required')
    _err(L, fwd(args(), ws=0), b'workspace required')
    _err(L, fwd(args(), ws=one + 16), b'256-byte aligned')
    need = L.cvb_train_seg_ce_workspace_bytes(2, 32, 32)
    assert need > 0 and L.cvb_train_seg_ce_workspace_bytes(0, 32, 32) == 0 and L.cvb_train_seg_ce_workspace_bytes(1024, 2048, 1024) == 0
    assert L.cvb_train_seg_ce_workspace_bytes(8, 512, 1024) > L.cvb_train_seg_ce_workspace_bytes(2, 32, 32)
    _err(L, fwd(args(), nbytes=need - 1), b'too small')
    _err(L, bwd(args(), lse=0), b'lse, grad_out, grad_preds (4-byte aligned) and record (8-byte aligned) are required')
    _err(L, bwd(args(), record=one + 4), b'are required')
    _err(L, bwd(args(), gout=0), b'are required')
    _err(L, bwd(args(), grad=one + 2), b'are required')


class _PlainCE(torch.nn.Module):
    """A loss of the reference's shape that is not the drop-in: it sees whatever loss_forward hands it."""

    def __init__(self, name, seen):
        super().__init__()
        self.loss_name, self.seen = name, seen

    def forward(self, pred, target):
        self.seen.append(tuple(pred.shape))
        return F.cross_entropy(pred, target.long(), ignore_index=255)


def test_loss_module_surface():
    """seg_train.CrossEntropyLoss2d: the reference's constructor and loss_name, no parameters, buffers or state_dict keys; class weights,
    label smoothing and other reductions raise NotImplementedError; CPU inputs raise CvbError and bad shapes / dtypes raise before any
    launch.  loss_forward keeps the reference's asserts and hands other losses the upsampled preds, computed once, summed by name."""
    from cvpytorch_b200 import _lib, seg_train as ST
    m = ST.CrossEntropyLoss2d()
    assert m.loss_name == 'ce_loss' and m.ignore_index == 255 and m.loss_weight == 1.0
    assert ST.CrossEntropyLoss2d(loss_weight=0.4, loss_name='aux', ignore_index=-1).loss_name == 'aux'
    assert list(m.state_dict()) == [] and list(m.parameters()) == [] and list(m.buffers()) == []
    seg = torch.nn.Module()
    seg.loss = torch.nn.ModuleList([ST.CrossEntropyLoss2d()])
    assert list(seg.state_dict()) == []
    with pytest.raises(NotImplementedError):
        ST.CrossEntropyLoss2d(weight=torch.ones(19))
    with pytest.raises(NotImplementedError):
        ST.CrossEntropyLoss2d(label_smoothing=0.1)
    with pytest.raises(NotImplementedError):
        ST.CrossEntropyLoss2d(reduction='none')
    pred, target = torch.zeros(2, 19, 8, 8), torch.zeros(2, 32, 32, dtype=torch.uint8)
    with pytest.raises(_lib.CvbError):
        m(pred, target)
    with pytest.raises(ValueError):
        m(pred[0], target)
    with pytest.raises(ValueError):
        m(pred, target[0])
    with pytest.raises(ValueError):
        m(pred, target[:1])

    seen = []
    pred = torch.randn(2, 5, 8, 12)
    target = torch.randint(0, 5, (2, 32, 48))
    target[:, :2] = 255
    plain = [_PlainCE('ce_loss', seen), _PlainCE('ohem', seen), _PlainCE('ce_loss', seen)]
    got = ST.loss_forward(None, pred, target, torch.nn.ModuleList(plain))
    up = F.interpolate(pred, size=(32, 48), mode='bilinear', align_corners=False)
    one = F.cross_entropy(up, target, ignore_index=255)
    assert seen == [(2, 5, 32, 48)] * 3 and sorted(got) == ['ce_loss', 'ohem']
    assert torch.allclose(got['ce_loss'], 2 * one) and torch.allclose(got['ohem'], one)
    single = ST.loss_forward(None, pred, target, _PlainCE('x', []))
    assert list(single) == ['x']
    with pytest.raises(AssertionError):
        ST.loss_forward(None, pred[0], target, plain)
    with pytest.raises(AssertionError):
        ST.loss_forward(None, pred, target[0], plain)
    # the drop-in gets the low-resolution preds, so a CPU batch reaches its CUDA check
    with pytest.raises(_lib.CvbError):
        ST.loss_forward(None, pred, target, [_PlainCE('ohem', []), ST.CrossEntropyLoss2d()])
