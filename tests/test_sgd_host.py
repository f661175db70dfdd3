"""The one-launch SGD drop-in without a GPU: the oracle's parameter groups against tests/golden/sgd_groups.npz (the reference's
build_optimizer) on the drop-in YOLOX-s and YOLOv5-s, the host checks of the C ABI, and every refusal of SGD.step before any launch."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DICT80 = [{f'c{i}': 1.0} for i in range(80)]


def _model(name):
    from cvpytorch_b200 import models as M, synth, yolox_models as XM
    return XM.YOLOX(dictionary=DICT80, model_cfg=dict(synth.YOLOX_CFG)) if name == 'yolox_s' else M.YOLOv5(DICT80, dict(synth.YOLOV5S_CFG))


@pytest.mark.parametrize('name', ['yolox_s', 'yolov5_s'])
def test_oracle_groups_reproduce_the_reference_fixture(name):
    from oracle import optim_oracle as O
    f = np.load(os.path.join(ROOT, 'tests', 'golden', 'sgd_groups.npz'))
    model = _model(name)
    groups = O.param_groups(model, O.CONFIGS[name])
    assert O.group_names(model, groups) == list(f[f'{name}:names'])
    assert len(groups) == {'yolox_s': 240, 'yolov5_s': 177}[name]
    for k in ('lr', 'weight_decay', 'momentum'):
        assert [g[k] for g in groups] == list(f[f'{name}:{k}']), k
    assert [g['nesterov'] for g in groups] == list(f[f'{name}:nesterov'])
    # one tensor per group, every parameter exactly once, and torch.optim.SGD accepts the groups as they are
    assert all(len(g['params']) == 1 for g in groups)
    assert sorted(id(g['params'][0]) for g in groups) == sorted(id(p) for p in model.parameters())
    torch.optim.SGD(groups)


def test_warmup_lr_follows_the_linear_warmup():
    from oracle import optim_oracle as O
    cfg = O.CONFIGS['yolox_s']
    assert O.warmup_lr(0, cfg) == 0.01 * 0.05 and O.warmup_lr(10000, cfg) == 0.01
    assert O.warmup_lr(2500, cfg) == 0.01 * (0.05 * 0.75 + 0.25)


def test_c_abi_rejects_bad_arguments_before_touching_the_device():
    from cvpytorch_b200 import _lib
    L = _lib.lib()
    table, odd = ctypes.c_void_p(256), ctypes.c_void_p(264)

    def rejects(rc, what):
        assert rc != 0
        assert what in L.cvb_last_error_string()

    def entries(*rows):
        return (_lib.CvbSgdEntry * len(rows))(*[_lib.CvbSgdEntry(*r) for r in rows])

    good = entries((256, 512, 1024, 2048, 10, 0))
    rejects(L.cvb_sgd_table_upload(None, 1, 1, table, None), b'null pointer')
    rejects(L.cvb_sgd_table_upload(good, 1, 1, None, None), b'null pointer')
    for n in (0, -1):
        rejects(L.cvb_sgd_table_upload(good, n, 1, table, None), b'n_entries must be > 0')
    for ng in (0, -2, _lib.CVB_SGD_MAX_GROUPS + 1):
        rejects(L.cvb_sgd_table_upload(good, 1, ng, table, None), b'n_groups must be in [1, 1024]')
    rejects(L.cvb_sgd_table_upload(good, 1, 1, odd, None), b'16-byte aligned')
    rejects(L.cvb_sgd_table_upload(entries((256, 512, None, None, 10, 0), (256, 512, None, None, -1, 0)), 2, 1, table, None),
            b'entry 1 has numel -1 < 0')
    rejects(L.cvb_sgd_table_upload(entries((256, 512, None, None, 10, 1)), 1, 1, table, None), b'entry 0 has group 1 outside [0, 1)')
    rejects(L.cvb_sgd_table_upload(entries((256, 512, None, None, 10, -1)), 1, 2, table, None), b'entry 0 has group -1')
    rejects(L.cvb_sgd_table_upload(entries((None, 512, None, None, 10, 0)), 1, 1, table, None), b'entry 0 has a null pointer')
    rejects(L.cvb_sgd_table_upload(entries((None, None, None, None, 0, 0), (256, None, None, None, 3, 0)), 2, 1, table, None),
            b'entry 1 has a null pointer')
    rejects(L.cvb_sgd_table_upload(entries((256, 512, 1024, None, 10, 0)), 1, 1, table, None), b'momentum buffer without valid flags')
    rejects(L.cvb_sgd_table_upload(entries((256, 512, None, 2048, 10, 0)), 1, 1, table, None), b'valid flags without a momentum buffer')

    groups = (_lib.CvbSgdGroup * 2)(_lib.CvbSgdGroup(0.1, 0.0, 0.9, _lib.CVB_SGD_MOMENTUM), _lib.CvbSgdGroup(0.1, 0.0, 0.0, 0))
    rejects(L.cvb_sgd_step(None, 1, groups, 2, None, None, None), b'null pointer')
    rejects(L.cvb_sgd_step(table, 1, None, 2, None, None, None), b'null pointer')
    for n in (0, -3):
        rejects(L.cvb_sgd_step(table, n, groups, 2, None, None, None), b'n_entries must be > 0')
    for ng in (0, _lib.CVB_SGD_MAX_GROUPS + 1):
        rejects(L.cvb_sgd_step(table, 1, groups, ng, None, None, None), b'n_groups must be in [1, 1024]')
    rejects(L.cvb_sgd_step(odd, 1, groups, 2, None, None, None), b'16-byte aligned')


def _params(*shapes):
    g = torch.Generator().manual_seed(5)
    ps = [torch.nn.Parameter(torch.randn(s, generator=g)) for s in shapes]
    for p in ps:
        p.grad = torch.randn(p.shape, generator=g)
    return ps


def _refused(opt, exc, match):
    from cvpytorch_b200 import _lib
    params = [p for g in opt.param_groups for p in g['params']]
    before = [p.detach().clone() for p in params]
    n0 = _lib.launch_count()
    with pytest.raises(exc, match=match):
        opt.step()
    assert _lib.launch_count() == n0
    assert all(torch.equal(p, b) for p, b in zip(params, before))


def test_step_refusals_before_any_launch():
    """Every refusal of SGD.step raises before a launch; the params stay as they were."""
    from cvpytorch_b200 import _lib
    from cvpytorch_b200.optim import SGD
    _lib.lib()
    _refused(SGD(_params(4, 5), lr=0.1, momentum=0.9, dampening=0.1), NotImplementedError, 'dampening')
    _refused(SGD(_params(4, 5), lr=0.1, maximize=True), NotImplementedError, 'maximize')
    _refused(SGD(_params(4, 5), lr=0.1, fused=True), NotImplementedError, 'fused')
    _refused(SGD(_params(4, 5), lr=0.1, differentiable=True), NotImplementedError, 'differentiable')
    _refused(SGD(_params(4, 5), lr=torch.tensor(0.1)), NotImplementedError, 'tensor lr')
    _refused(SGD(_params(4, 5), lr=0.1, weight_decay=torch.tensor(0.1)), NotImplementedError, 'tensor weight_decay')
    # a later group, added or edited after construction, is checked too
    opt = SGD(_params(4), lr=0.1, momentum=0.9)
    opt.add_param_group({'params': _params(3), 'dampening': 0.5})
    _refused(opt, NotImplementedError, 'group 1 sets dampening')

    sparse = _params((6, 4))
    sparse[0].grad = torch.sparse_coo_tensor(torch.tensor([[1, 3]]), torch.ones(2, 4), (6, 4))
    _refused(SGD(sparse, lr=0.1), NotImplementedError, 'sparse')
    half = _params(4, 5)
    half[1].data = half[1].data.half()
    half[1].grad = half[1].grad.half()
    _refused(SGD(half, lr=0.1), NotImplementedError, 'only fp32')
    f64 = _params(4, 5)
    f64[0].grad_dtype = None  # let the param hold a gradient of another dtype
    f64[0].grad = f64[0].grad.double()
    _refused(SGD(f64, lr=0.1), NotImplementedError, 'only fp32')
    strided = _params((4, 6), 5)
    strided[0].grad = torch.randn(6, 4).t()
    _refused(SGD(strided, lr=0.1), NotImplementedError, 'not contiguous')
    noncontig = _params(5)
    noncontig[0].data = torch.randn(5, 2)[:, 0]
    _refused(SGD(noncontig, lr=0.1), NotImplementedError, 'not contiguous')
    shaped = _params((4, 6))
    shaped[0].data = torch.randn(24)  # torch checks the shape when .grad is assigned, not when .data is
    _refused(SGD(shaped, lr=0.1), NotImplementedError, 'a gradient of shape')
    base = torch.randn(20)
    a, b = torch.nn.Parameter(base[0:12]), torch.nn.Parameter(base[8:20])
    a.grad, b.grad = torch.randn(12), torch.randn(12)
    _refused(SGD([a, b], lr=0.1), NotImplementedError, 'share memory')
    many = _params(*([2] * (_lib.CVB_SGD_MAX_GROUPS + 1)))
    _refused(SGD([{'params': [p]} for p in many], lr=0.1), NotImplementedError, '1025 param groups')
    # what the kernel could run but not on the CPU
    _refused(SGD(_params(4, 5), lr=0.1, momentum=0.9, nesterov=True, weight_decay=1e-4), _lib.CvbError, 'no CPU fallback')


def test_no_gradient_is_no_launch():
    from cvpytorch_b200 import _lib
    from cvpytorch_b200.optim import SGD
    ps = _params(4, 5)
    for p in ps:
        p.grad = None
    opt = SGD(ps, lr=0.1, momentum=0.9)
    n0 = _lib.launch_count()
    assert opt.step() is None and opt.step(lambda: 3.0) == 3.0
    assert _lib.launch_count() == n0 and opt.table_builds == 0 and not opt.state
    assert opt._step_supports_amp_scaling and 'grad_scaler' not in __import__('inspect').signature(opt.step).parameters
