"""SyncBatchNorm on the training path without a GPU: the host-side argument checks of the cross-rank BatchNorm entry points, and when the
training layers decide to synchronise (as nn.SyncBatchNorm.forward decides)."""
import ctypes
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def test_sync_bn_c_abi_rejects_bad_arguments_before_touching_the_device():
    """Null pointers, C not a multiple of 8 or above 2048, an empty shard, a world below one, misaligned records or count: rejected on the
    host by cvb_train_bn_partial / _merge / _silu_bwd_reduce / _silu_bwd_apply."""
    from cvpytorch_b200 import _lib
    L = _lib.lib()
    one, odd = ctypes.c_void_p(256), ctypes.c_void_p(260)

    def rejects(rc, what):
        assert rc != 0
        assert what in L.cvb_last_error_string()

    rejects(L.cvb_train_bn_partial(None, 16, 64, one, one, None), b'null')
    rejects(L.cvb_train_bn_partial(one, 16, 64, one, None, None), b'null')
    for npix, C in ((0, 64), (16, 12), (16, 0), (16, 2056)):
        rejects(L.cvb_train_bn_partial(one, npix, C, one, one, None), b'multiple of 8')
    rejects(L.cvb_train_bn_partial(odd, 16, 64, one, one, None), b'aligned')
    rejects(L.cvb_train_bn_partial(one, 16, 64, one, odd, None), b'aligned')

    args = lambda recs=one, world=2, C=64, rm=one, rv=one, count=one: (recs, world, C, one, one, 1e-3, 0.03, rm, rv, one, count, None)  # noqa: E731
    rejects(L.cvb_train_bn_merge(*args(recs=None)), b'null')
    rejects(L.cvb_train_bn_merge(*args(count=None)), b'null')
    rejects(L.cvb_train_bn_merge(*args(rm=None)), b'together')
    for world, C in ((0, 64), (-1, 64), (2, 20), (2, 4096)):
        rejects(L.cvb_train_bn_merge(*args(world=world, C=C)), b'world must be')
    rejects(L.cvb_train_bn_merge(*args(recs=odd)), b'aligned')
    rejects(L.cvb_train_bn_merge(*args(count=odd)), b'aligned')

    rejects(L.cvb_train_bn_silu_bwd_reduce(None, 0, one, 16, 64, one, one, None), b'null')
    rejects(L.cvb_train_bn_silu_bwd_reduce(one, 0, one, 16, 64, one, None, None), b'null')
    for npix, C in ((0, 64), (16, 12), (16, 2056)):
        rejects(L.cvb_train_bn_silu_bwd_reduce(one, 0, one, npix, C, one, one, None), b'multiple of 8')
    rejects(L.cvb_train_bn_silu_bwd_apply(one, 0, one, 16, 64, one, one, one, None, one, None), b'null')
    rejects(L.cvb_train_bn_silu_bwd_apply(one, 0, one, 16, 64, one, one, None, one, one, None), b'null')
    for npix, C in ((0, 64), (16, 12), (16, 2056)):
        rejects(L.cvb_train_bn_silu_bwd_apply(one, 0, one, npix, C, one, one, one, one, one, None), b'multiple of 8')
    rejects(L.cvb_train_bn_silu_bwd_apply(one, 0, one, 16, 64, one, one, one, odd, one, None), b'aligned')


def test_sync_decision_follows_the_batchnorm_module():
    """Without an initialised process group every BatchNorm runs the local statistics; convert_sync_batchnorm keeps the drop-ins' keys,
    parameters and buffers and puts an nn.SyncBatchNorm where the layers read their BatchNorm."""
    import torch.distributed as dist
    from cvpytorch_b200 import train as T
    assert not dist.is_initialized()
    m = T.CSPLayer(64, 64, n=1)
    params, keys = [id(p) for p in m.parameters()], list(m.state_dict())
    s = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m)
    assert s is m and list(m.state_dict()) == keys and [id(p) for p in m.parameters()] == params
    layers = [mod for mod in m.modules() if isinstance(mod, T._ConvBnSiLULayer)]
    assert len(layers) == 5 and all(isinstance(layer.bn, torch.nn.SyncBatchNorm) for layer in layers)
    assert all(T._sync_group(layer.bn) is None for layer in layers)
    assert T._sync_group(torch.nn.BatchNorm2d(8)) is None
