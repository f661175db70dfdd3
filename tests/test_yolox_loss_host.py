"""The YOLOX loss without a GPU: the oracle against the reference fixture, the host-side argument checks of the loss entry points, and the
model-level training surface of yolox_models.YOLOX."""
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
KEYS = ('loss', 'iou_loss', 'conf_loss', 'cls_loss', 'num_fg')


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def test_oracle_reproduces_reference_fixture():
    """oracle/yolox_loss_oracle.py vs the reference YOLOXLoss (tests/golden/yolox_loss.npz): identical assignment, loss terms and head-output
    gradients within 1e-5 relative.  The fixture covers an image without GT, overlapping GTs, an in-centre-only GT, a GT over the padded
    border column / row and zero rows after each image's GTs; it has no near-tie and its dynamic k exceeds 1."""
    from oracle import yolox_loss_oracle as LO
    g = np.load(os.path.join(GOLD, 'yolox_loss.npz'))
    for case, (B, H, nc) in LO.CASES.items():
        preds, targets = LO.fixture_case(int(g[f'{case}_seed']), case)
        assert not bool(LO.near_ties(preds, targets, LO.STRIDES, nc).any())
        ps = [p.clone().requires_grad_(True) for p in preds]
        out, (fg, mg, mi) = LO.losses(ps, targets, LO.STRIDES, nc)
        out['loss'].backward()
        assert np.array_equal(fg.numpy(), g[f'{case}_fg'])
        assert np.array_equal(mg.numpy(), g[f'{case}_matched_gt'])
        assert _rel(mi, g[f'{case}_matched_iou']) <= 1e-5
        for k in KEYS:
            assert _rel(out[k].detach(), g[f'{case}_{k}']) <= 1e-5, (case, k)
        for i, p in enumerate(ps):
            assert _rel(p.grad, g[f'{case}_grad{i}']) <= 1e-5, (case, i)
        nl = LO.num_labels(targets)
        assert (nl < targets.shape[1]).any() and (case != 'a' or int(nl.min()) == 0)  # zero rows after nlabel; case a: an image without GT
        assert int(np.bincount(g[f'{case}_matched_gt'][g[f'{case}_fg']]).max()) > 1  # dynamic k > 1 somewhere


def _err(L, rc, text):
    assert rc != 0
    assert text in L.cvb_last_error_string(), L.cvb_last_error_string()


def test_loss_c_abi_rejects_bad_arguments():
    """Every loss entry point rejects bad arguments on the host, before the device is touched: level shapes against B and 5 + nc, nc < 1,
    max_gt outside [1, 1024], strides <= 0, misaligned pointers, missing outputs and a short workspace."""
    from cvpytorch_b200 import _lib
    L = _lib.lib()
    one, odd = 256, 258

    def args(shapes=((2, 8, 10, 10), (2, 8, 5, 5)), strides=(8.0, 16.0), nc=3, B=2, max_gt=4, ptr=one, tgt=one):
        n = len(shapes)
        return ((ctypes.c_void_p * n)(*[ptr] * n), (ctypes.c_int32 * (4 * n))(*[d for s in shapes for d in s]), (ctypes.c_float * n)(*strides),
                n, nc, ctypes.c_void_p(tgt), B, max_gt)

    def fwd(a, mg=one, mi=one, out=one, ws=one, nbytes=1 << 30):
        return L.cvb_train_yolox_loss_fwd(*a, ctypes.c_void_p(mg), ctypes.c_void_p(mi), ctypes.c_void_p(out), ctypes.c_void_p(ws), nbytes, None)

    def bwd(a, grads=None, gout=one):
        n = a[3]
        g = grads if grads is not None else (ctypes.c_void_p * n)(*[one] * n)
        return L.cvb_train_yolox_loss_bwd(*a, ctypes.c_void_p(one), ctypes.c_void_p(one), ctypes.c_void_p(one), ctypes.c_void_p(gout), g, None)

    for call in (fwd, bwd):
        _err(L, call(args(shapes=((2, 9, 10, 10), (2, 8, 5, 5)))), b'5 + num_classes')
        _err(L, call(args(shapes=((3, 8, 10, 10), (2, 8, 5, 5)))), b'5 + num_classes')
        _err(L, call(args(shapes=((2, 8, 0, 10), (2, 8, 5, 5)))), b'5 + num_classes')
        _err(L, call(args(nc=0, shapes=((2, 5, 10, 10), (2, 5, 5, 5)))), b'num_classes must be >= 1')
        _err(L, call(args(max_gt=1025)), b'max_gt must be in [1, 1024]')
        _err(L, call(args(max_gt=0)), b'max_gt must be in [1, 1024]')
        _err(L, call(args(strides=(8.0, 0.0))), b'stride must be > 0')
        _err(L, call(args(strides=(-8.0, 16.0))), b'stride must be > 0')
        _err(L, call(args(ptr=odd)), b'4-byte aligned')
        _err(L, call(args(tgt=odd)), b'targets must be 4-byte aligned')
        _err(L, call(args(B=0)), b'batch must be >= 1')
        _err(L, call(args(shapes=[(2, 8, 4, 4)] * 5, strides=[8.0] * 5)), b'levels supported')
    _err(L, fwd(args(), mg=0), b'matched_gt, matched_iou and out are required')
    _err(L, fwd(args(), out=odd), b'4-byte aligned')
    _err(L, fwd(args(), ws=one + 16), b'256-byte aligned')
    need = L.cvb_train_yolox_loss_workspace_bytes(2, 125)
    assert need > 0 and L.cvb_train_yolox_loss_workspace_bytes(0, 125) == 0
    _err(L, fwd(args(), nbytes=need - 1), b'too small')
    _err(L, bwd(args(), gout=odd), b'4-byte aligned')
    _err(L, bwd(args(), grads=(ctypes.c_void_p * 2)(one, odd)), b'gradient missing or not 4-byte aligned')


def test_loss_module_surface():
    """train.YOLOXLoss: the reference's constructor, no parameters or buffers; re-ID and L1 raise NotImplementedError; CPU outputs raise
    CvbError (no fallback)."""
    from cvpytorch_b200 import _lib, train as T
    m = T.YOLOXLoss(80)
    assert list(m.state_dict()) == [] and list(m.parameters()) == [] and m.strides == [8, 16, 32] and not m.use_l1
    with pytest.raises(NotImplementedError):
        T.YOLOXLoss(80, reid_dim=128, id_nums=[10] * 80)
    m.use_l1 = True
    with pytest.raises(NotImplementedError):
        m([torch.zeros(1, 85, 4, 4)] * 3, torch.zeros(1, 1, 5))
    m.use_l1 = False
    with pytest.raises(_lib.CvbError):
        m([torch.zeros(1, 85, 4, 4)] * 3, torch.zeros(1, 1, 5))


def _yolox(cfg=None):
    from cvpytorch_b200 import synth, yolox_models as XM
    return XM.YOLOX(dictionary=[{f'c{i}': 1.0} for i in range(80)], model_cfg=dict(cfg or synth.YOLOX_CFG))


def test_yolox_training_surface():
    """YOLOX keeps its state_dict keys with the loss and the training modules in place; the training modules use the model's own parameters
    and BatchNorm buffers and are not submodules; training mode with CPU images raises CvbError, eval mode with 'train' RuntimeError;
    a LOSS entry with re-ID raises NotImplementedError, and so do the widths the training kernels refuse (YOLOX-t, -m, -x)."""
    from cvpytorch_b200 import _lib, synth
    m = _yolox()
    keys = list(synth.yolox_template_state_dict().keys())
    assert list(m.state_dict()) == keys
    m.train()
    with pytest.raises(_lib.CvbError):
        m(torch.zeros(2, 3, 64, 64), [{'labels': torch.zeros(1), 'boxes': torch.ones(1, 4)}] * 2, 'train')
    mods = m._training_modules()
    assert list(m.state_dict()) == keys and len(list(m.modules())) == len(list(_yolox().modules()))
    params = {id(p) for p in m.parameters()}
    assert sum(1 for t in mods for _ in t.parameters()) == len(params) and all(id(p) in params for t in mods for p in t.parameters())
    bufs = {id(b) for b in m.buffers()}
    assert all(id(b) in bufs for t in mods for b in t.buffers())
    m.eval()
    with pytest.raises(RuntimeError, match=r'\.train\(\)'):
        m(torch.zeros(1, 3, 64, 64), None, 'train')
    with pytest.raises(NotImplementedError):
        _yolox({**synth.YOLOX_CFG, 'LOSS': {'name': 'YOLOXLoss', 'reid_dim': 64, 'id_nums': [5] * 80}})
    m = _yolox({**synth.YOLOX_CFG, 'LOSS': {'name': 'YOLOXLoss'}})
    m.loss.use_l1 = True
    assert list(m.state_dict()) == keys
    for sub, t in (('m', 'yolox_m'), ('t', 'yolox_tiny'), ('x', 'yolox_x')):
        cfg = {**synth.YOLOX_CFG, 'TYPE': t, 'BACKBONE': {**synth.YOLOX_CFG['BACKBONE'], 'subtype': 'yolox_' + sub}}
        with pytest.raises(NotImplementedError):
            _yolox(cfg).train()._training_modules()
