"""SyncBatchNorm through the YOLOv6 training layers without a GPU: the host-side argument checks of cvb_train_bn_relu_bwd_reduce / _apply and
cvb_train_repvgg_bwd_reduce / _apply, and when the YOLOv6 layers decide to synchronise."""
import ctypes
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_yolov6_host import DICT, use_model  # noqa: E402


def test_split_backward_c_abi_rejects_bad_arguments_before_touching_the_device():
    """Null pointers, npix 0, C not a multiple of 8 or above 2048, misaligned bf16 operands, fp32 operands or count, and identity-branch
    operands that do not come together: rejected on the host."""
    from cvpytorch_b200 import _lib
    L = _lib.lib()
    one, odd, odd8 = ctypes.c_void_p(1 << 20), ctypes.c_void_p((1 << 20) + 2), ctypes.c_void_p((1 << 20) + 8)

    def rejects(rc, what):
        assert rc != 0
        assert what in L.cvb_last_error_string(), L.cvb_last_error_string()

    for k in range(4):
        a = [one] * 4
        a[k] = None
        rejects(L.cvb_train_bn_relu_bwd_reduce(a[0], a[1], 16, 64, a[2], a[3], None), b'null pointer')
    for npix, C in ((0, 64), (16, 12), (16, 0), (16, 2056)):
        rejects(L.cvb_train_bn_relu_bwd_reduce(one, one, npix, C, one, one, None), b'multiple of 8 up to 2048')
    rejects(L.cvb_train_bn_relu_bwd_reduce(odd8, one, 16, 64, one, one, None), b'16-byte')
    rejects(L.cvb_train_bn_relu_bwd_reduce(one, one, 16, 64, one, odd, None), b'4-byte')

    for k in range(7):
        a = [one] * 7
        a[k] = None
        rejects(L.cvb_train_bn_relu_bwd_apply(a[0], a[1], 16, 64, a[2], a[3], a[4], a[5], a[6], None), b'null pointer')
    for npix, C in ((0, 64), (16, 12), (16, 2056)):
        rejects(L.cvb_train_bn_relu_bwd_apply(one, one, npix, C, one, one, one, one, one, None), b'multiple of 8 up to 2048')
    rejects(L.cvb_train_bn_relu_bwd_apply(one, one, 16, 64, one, one, one, one, odd8, None), b'16-byte')
    rejects(L.cvb_train_bn_relu_bwd_apply(one, one, 16, 64, one, odd, one, one, one, None), b'8-byte aligned')
    rejects(L.cvb_train_bn_relu_bwd_apply(one, one, 16, 64, one, one, one, ctypes.c_void_p((1 << 20) + 4), one, None), b'8-byte aligned')

    red = lambda g=one, x=None, sid=None, npix=16, C=64, sums=one, y3=one: L.cvb_train_repvgg_bwd_reduce(  # noqa: E731
        g, one, y3, one, x, npix, C, one, one, sid, sums, None)
    rejects(red(g=None), b'null pointer')
    rejects(red(sums=None), b'null pointer')
    for npix, C in ((0, 64), (16, 20), (16, 4096)):
        rejects(red(npix=npix, C=C), b'multiple of 8 up to 2048')
    rejects(red(x=one), b'x and stat_id go together')
    rejects(red(sid=one), b'x and stat_id go together')
    rejects(red(y3=odd8), b'16-byte aligned')
    rejects(red(x=odd8, sid=one), b'16-byte aligned')
    rejects(red(sums=odd), b'4-byte aligned')

    app = lambda x=None, sid=None, gid=None, dxid=None, npix=16, C=64, count=one, dy3=one, sums=one: L.cvb_train_repvgg_bwd_apply(  # noqa: E731
        one, one, one, one, x, npix, C, one, one, sid, one, one, gid, sums, count, dy3, one, dxid, None)
    rejects(app(count=None), b'null pointer')
    rejects(app(dy3=None), b'null pointer')
    for npix, C in ((0, 64), (16, 20), (16, 4096)):
        rejects(app(npix=npix, C=C), b'multiple of 8 up to 2048')
    rejects(app(x=one, sid=one, gid=one), b'go together')
    rejects(app(x=one, sid=one, dxid=one), b'go together')
    rejects(app(x=one, gid=one, dxid=one), b'x and stat_id go together')
    rejects(app(dy3=odd8), b'16-byte aligned')
    rejects(app(sums=odd), b'4-byte aligned')
    rejects(app(count=ctypes.c_void_p((1 << 20) + 4)), b'8-byte aligned')
    assert L.cvb_train_repvgg_bwd_apply(one, one, one, one, one, 16, 64, one, one, one, one, one, one, one, ctypes.c_void_p((1 << 20) + 4), one, one,
                                        one, None) != 0


class _FakeGroupBN(torch.nn.SyncBatchNorm):
    """A SyncBatchNorm that train._sync_group sees as spanning several ranks (a process group needs a second process)."""


def _fake_sync_group(real):
    sentinel = object()
    return sentinel, lambda bn: sentinel if isinstance(bn, _FakeGroupBN) else real(bn)


def test_sync_batchnorm_outside_a_process_group_is_local():
    import torch.distributed as dist
    from cvpytorch_b200 import train as T, yolov6_train as Y
    assert not dist.is_initialized()
    blk = torch.nn.SyncBatchNorm.convert_sync_batchnorm(Y.RepVGGBlock(64, 64))
    bns = (blk.rbr_dense.bn, blk.rbr_1x1.bn, blk.rbr_identity)
    assert all(isinstance(b, torch.nn.SyncBatchNorm) for b in bns)
    assert all(Y._bn_args(b)[4] is None for b in bns)
    cm = torch.nn.SyncBatchNorm.convert_sync_batchnorm(Y.ConvModule(64, 64, 3))
    assert isinstance(cm.bn, torch.nn.SyncBatchNorm) and cm._bn_inputs()[-1] is None and T._sync_group(cm.bn) is None


def test_mixed_repvgg_block_raises(monkeypatch):
    """A block whose BatchNorms do not all share one process group raises NotImplementedError naming the block, before any device work
    (the CPU input would otherwise be refused by the CUDA check); one whose three BatchNorms share it gets past the decision."""
    from cvpytorch_b200 import _lib, yolov6_train as Y
    sentinel, fake = _fake_sync_group(Y._sync_group)
    monkeypatch.setattr(Y, '_sync_group', fake)
    x = torch.zeros(1, 4, 4, 64, dtype=torch.bfloat16)
    for which in ('rbr_dense', 'rbr_1x1', 'rbr_identity'):
        blk = Y.RepVGGBlock(64, 64).train()
        if which == 'rbr_identity':
            blk.rbr_identity = _FakeGroupBN(64)
        else:
            getattr(blk, which).bn = _FakeGroupBN(64)
        with pytest.raises(NotImplementedError, match=r'RepVGGBlock\(64, 64, stride 1\).*all be local or all span the same process group'):
            blk(x)
    blk = Y.RepVGGBlock(64, 128, stride=2).train()
    blk.rbr_dense.bn = _FakeGroupBN(128)
    with pytest.raises(NotImplementedError, match=r'RepVGGBlock\(64, 128, stride 2\)'):
        blk(x)
    blk = Y.RepVGGBlock(64, 64).train()
    blk.rbr_dense.bn, blk.rbr_1x1.bn, blk.rbr_identity = _FakeGroupBN(64), _FakeGroupBN(64), _FakeGroupBN(64)
    with pytest.raises(_lib.CvbError, match='CUDA tensor required'):
        blk(x)


def test_training_modules_bind_the_converted_modules():
    """convert_sync_batchnorm on the YOLOv6 model: its training modules read the converted BatchNorms (128 for n and s), with the same
    parameters and buffers, so the layers see an nn.SyncBatchNorm at every forward."""
    from cvpytorch_b200 import yolov6_models as M
    for st in ('n', 's'):
        m = M.YOLOv6(DICT, use_model(st))
        keys = list(m.state_dict())
        torch.nn.SyncBatchNorm.convert_sync_batchnorm(m)
        assert list(m.state_dict()) == keys
        mods = m._training_modules()
        bns = [b for tm in mods for b in tm.modules() if isinstance(b, torch.nn.modules.batchnorm._BatchNorm)]
        assert len(bns) == 128 and all(isinstance(b, torch.nn.SyncBatchNorm) for b in bns)
        inference = {id(b) for b in m.modules() if isinstance(b, torch.nn.SyncBatchNorm)}
        assert all(id(b) in inference for b in bns)
