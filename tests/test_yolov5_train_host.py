"""CPU checks of the YOLOv5 training surface: the training modules' keys and tensors are the model's own, the refusals, the 6x6 stem weight
permutation, the loss oracle on hand-checked candidate cases, and the host-side argument checks of the new C entry points."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from cvpytorch_b200 import _lib, models as M, synth, yolov5_train as V  # noqa: E402
from oracle import yolov5_train_oracle as O  # noqa: E402

CLS80 = [{f'c{i}': 1.0} for i in range(80)]
GOLD = os.path.join(ROOT, 'tests', 'golden')


def _model(type_='yolov5_s'):
    return M.YOLOv5(CLS80, dict(synth.YOLOV5S_CFG, TYPE=type_))


def test_training_modules_are_bound_to_the_model():
    m = _model().train()
    mods = m._training_modules()
    for tm, im in zip(mods, (m.backbone, m.neck, m.detect)):
        assert list(tm.state_dict()) == list(im.state_dict())
        own = {k: id(v) for k, v in im.state_dict(keep_vars=True).items()}
        assert all(own[k] == id(v) for k, v in tm.state_dict(keep_vars=True).items())
    assert list(m.state_dict()) == list(_model().state_dict())
    assert isinstance(m.loss, V.YOLOv5Loss) and not list(m.loss.parameters()) and not list(m.loss.buffers())
    m.neck.up_1.conv.bn = nn.SyncBatchNorm(256)  # what convert_sync_batchnorm does: the next call binds the new module
    assert m._training_modules()[1].up_1.conv.bn is m.neck.up_1.conv.bn


def test_refusals():
    m = _model()
    with pytest.raises(RuntimeError, match=r'\.train\(\)'):
        m.eval()(torch.zeros((1, 3, 64, 64)), torch.zeros((0, 6)), 'train')
    with pytest.raises(_lib.CvbError):
        m.train()(torch.zeros((1, 3, 64, 64)), torch.zeros((0, 6)), 'train')
    with pytest.raises(NotImplementedError):
        _model('yolov5_m').train()._training_modules()
    with pytest.raises(NotImplementedError):
        V.YOLOv5Loss(80, anchors=M.YOLOv5.anchors, autobalance=True)
    with pytest.raises(NotImplementedError):
        M.YOLOv5(CLS80, dict(synth.YOLOV5S_CFG, LOSS={'name': 'YOLOXLoss'}))


def test_pack_targets():
    imgs = torch.zeros((2, 3, 8, 8))
    t = [{'labels': torch.tensor([3, 5]), 'boxes': torch.rand((2, 4))}, {'labels': torch.tensor([7]), 'boxes': torch.rand((1, 4))}]
    g = M.YOLOv5.pack_targets(imgs, t)
    assert g[:, 0].tolist() == [0, 0, 1] and g[:, 1].tolist() == [3, 5, 7] and torch.equal(g[:, 2:], torch.cat([t[0]['boxes'], t[1]['boxes']]))
    assert M.YOLOv5.pack_targets(imgs, g) is g


def test_stem_weight_permutation_round_trips():
    w = torch.randn(32, 3, 6, 6, dtype=torch.float64)
    w2 = V.stem_weight_to_s2d(w)
    img = torch.randn(2, 3, 16, 20, dtype=torch.float64)
    s2d = torch.cat([img[..., ::2, ::2], img[..., 1::2, ::2], img[..., ::2, 1::2], img[..., 1::2, 1::2]], 1)  # Focus patch order
    assert torch.allclose(nn.functional.conv2d(s2d, w2, padding=1), nn.functional.conv2d(img, w, stride=2, padding=2), atol=1e-12)
    wr = w.clone().requires_grad_(True)
    V.stem_weight_to_s2d(wr).backward(w2)
    assert torch.equal(wr.grad, w)  # a pure permutation: every element maps exactly once


def test_oracle_candidates_on_hand_cases():
    anchors = torch.tensor([[[1.0, 1.0]]])
    # (a) GT on integer grid coordinates (4, 4) of an 8x8 map: all 5 offsets, the -x / -y ones landing back on the centre cell (duplicates);
    # (b) at the right border (x = 1): the centre and +x cells clamp to column 7 and tbox uses the clamped column
    t = torch.tensor([[0, 0, 0.5, 0.5, 0.125, 0.125], [0, 0, 1.0, 0.3125, 0.125, 0.125]])
    (b, a, gj, gi, c), tbox, _ = O.build_targets([(8, 8)], t, anchors)[0]
    assert list(zip(gi.tolist(), gj.tolist())) == [(4, 4), (7, 2), (3, 4), (7, 2), (4, 3), (4, 4), (4, 4)]
    assert tbox[1, :2].tolist() == [1.0, 0.5] and tbox[3, :2].tolist() == [1.0, 0.5] and tbox[2, :2].tolist() == [1.0, 0.0]
    # ratio filter: a 10 x 1 box against a 1 x 1 anchor has max(r, 1 / r) = 10 >= 4
    assert O.build_targets([(8, 8)], torch.tensor([[0, 0, 0.5, 0.5, 1.25, 0.125]]), anchors)[0][1].shape[0] == 0


@pytest.mark.parametrize('case', sorted(O.LOSS_CASES))
def test_oracle_loss_reproduces_reference_fixture(case):
    """tests/golden/yolov5_loss.npz (tools/make_golden_yolov5_loss.py, the reference YOLOv5Loss): the candidate lists exactly, the loss,
    items and detect-output gradients within 1e-6."""
    f = np.load(os.path.join(GOLD, 'yolov5_loss.npz'))
    preds, targets = O.loss_fixture_case(int(f[f'{case}_seed']), case)
    ps = [p.clone().requires_grad_(True) for p in preds]
    loss, items, tg = O.yolov5_loss(ps, targets, torch.tensor(O.ANCHORS), O.LOSS_CASES[case][3])
    loss.backward()
    for i, (ci, cb) in enumerate(O.candidate_lists(tg, preds[0].shape[0])):
        assert np.array_equal(ci.numpy(), f[f'{case}_cand_idx{i}']) and np.array_equal(cb.numpy(), f[f'{case}_cand_box{i}']), i
    assert abs(float(loss.detach()) - float(f[f'{case}_loss'][0])) <= 1e-6 * abs(float(f[f'{case}_loss'][0]))
    assert np.allclose(items.numpy(), f[f'{case}_items'], rtol=1e-6, atol=0)
    for i, p in enumerate(ps):
        ref = f[f'{case}_grad{i}']
        assert np.abs(p.grad.numpy() - ref).max() <= 1e-6 * np.abs(ref).max(), i


def test_oracle_network_reproduces_reference_fixture():
    """tests/golden/yolov5_train.npz (tools/make_golden_yolov5_train.py, the reference backbone, neck and detect in training mode): outputs,
    every parameter gradient and the running statistics within 1e-5, max-normalised."""
    f = np.load(os.path.join(GOLD, 'yolov5_train.npz'))
    keys, sd, x, Gs = O.net_fixture_inputs(f)
    got = O.net_train_step(x, Gs, sd)
    ref_keys = {k for k in f.files if k.startswith(('y', 'grad_', 'after_'))}
    assert set(got) == ref_keys
    for k in ref_keys:
        assert float((got[k] - torch.from_numpy(f[k])).abs().max()) <= 1e-5 * (np.abs(f[k]).max() + 1e-12), k


def test_fixture_network_keys_are_the_training_modules():
    f = np.load(os.path.join(GOLD, 'yolov5_train.npz'))
    mods = {'backbone.': V.YOLOv5CSPDarknet(**O.NET['backbone']), 'neck.': V.YOLOv5Neck(**O.NET['neck']),
            'detect.': V.YOLOv5Detect(anchors=O.ANCHORS, **O.NET['detect'])}
    assert [str(k) for k in f['keys']] == [pre + k for pre, m in mods.items() for k in m.state_dict()]


def _abi_args(nlev=3, na=3, nc=80, B=2, nt=4, shapes=None, anchors_val=1.0, hyp0=4.0):
    n = nlev
    ptrs = (ctypes.c_void_p * n)(*([256] * n))
    sh = shapes or [B, na * (5 + nc), 8, 8] * n
    shapes_c = (ctypes.c_int32 * len(sh))(*sh)
    anc = (ctypes.c_float * (n * na * 2))(*([anchors_val] * (n * na * 2)))
    bal = (ctypes.c_float * n)(*([1.0] * n))
    hyp = (ctypes.c_float * 5)(hyp0, 0.05, 1.0, 0.5, 1.0)
    return ptrs, shapes_c, anc, bal, n, na, nc, 256, nt, hyp


def _abi_calls(args, out=256, grad_out=256):
    """(fwd rc, fwd error text, bwd rc, bwd error text) with every other argument valid: aligned (never dereferenced) pointers and a
    workspace size larger than any case needs.  No kernel launches: every call here fails validation."""
    L = _lib.lib()
    big = 1 << 40
    rc_f = L.cvb_train_yolov5_loss_fwd(*args, 256, 256, 256, out, 256, big, None)
    err_f = L.cvb_last_error_string().decode()
    g = (ctypes.c_void_p * 5)(*([256] * 5))
    rc_b = L.cvb_train_yolov5_loss_bwd(*args, 256, 256, 256, 256, big, grad_out, g, None)
    err_b = L.cvb_last_error_string().decode()
    return rc_f, err_f, rc_b, err_b


@pytest.mark.parametrize('kw,what', [(dict(nlev=0), 'levels'), (dict(nlev=5), 'levels'), (dict(na=0), 'anchors per level'), (dict(na=9), 'anchors per level'),
                                     (dict(nc=0), 'num_classes'), (dict(nt=-1), 'nt must be'),
                                     (dict(shapes=[2, 255, 8, 8, 3, 255, 4, 4, 2, 255, 2, 2]), 'level 1 output must be'),
                                     (dict(shapes=[2, 254, 8, 8] * 3), 'level 0 output must be'), (dict(anchors_val=0.0), 'must be positive'),
                                     (dict(hyp0=1.0), 'anchor_t')])
def test_c_abi_rejects_bad_arguments(kw, what):
    rc_f, err_f, rc_b, err_b = _abi_calls(_abi_args(**kw))
    assert rc_f == -1 and what in err_f, err_f  # CVB_ERR_INVALID, for this argument
    assert rc_b == -1 and what in err_b, err_b


def test_c_abi_valid_arguments_pass_validation():
    """Positive control: with every argument valid except the last one each entry point checks (out / grad_out), the refusal names that
    argument, so the cases above are refused for their own argument."""
    rc_f, err_f, rc_b, err_b = _abi_calls(_abi_args(), out=None, grad_out=None)
    assert rc_f == -1 and 'out [4] required' in err_f, err_f
    assert rc_b == -1 and 'grad_out [1] required' in err_b, err_b


def test_c_abi_workspace_bytes():
    L = _lib.lib()
    assert L.cvb_train_yolov5_loss_workspace_bytes(0, 3, 1) == 0 and L.cvb_train_yolov5_loss_workspace_bytes(3, 3, -1) == 0
    assert L.cvb_train_yolov5_loss_workspace_bytes(3, 3, 100) > L.cvb_train_yolov5_loss_workspace_bytes(3, 3, 10) > 0
    for fn in ('cvb_train_sppf_chain_fwd', 'cvb_train_sppf_chain_bwd'):
        f = getattr(L, fn)
        assert (f(None, 1, 1, 1, 8, None, None, None) if fn.endswith('fwd') else f(None, None, 1, 1, 1, 8, None, None, None)) == -1
