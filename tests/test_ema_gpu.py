"""The model EMA on the H100 (csrc/ema.cu, cvpytorch_b200.ema.ModelEMA) against oracle/ema_oracle.py run by torch on the same GPU, bit for
bit: the YOLOX-s and YOLOv5-s state dicts over many updates, awkward entry sizes and misaligned views, tensors replaced between updates,
the trainer's flow (training steps, EMA updates, validation, deep copies) and a DDP-wrapped model.  Deep copies of every model-level
drop-in after a 'val' call."""
import copy
import os
import sys
import tempfile

import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

DICT80 = [{f'c{i}': 1.0} for i in range(80)]


def _yolox():
    from cvpytorch_b200 import synth, yolox_models as XM
    return XM.YOLOX(dictionary=DICT80, model_cfg=dict(synth.YOLOX_CFG))


def _yolov5():
    from cvpytorch_b200 import models as M, synth
    return M.YOLOv5(DICT80, dict(synth.YOLOV5S_CFG))


def _train_step(model, g, scale=1e-2):
    """A seeded stand-in for an optimiser step: every floating entry moves, num_batches_tracked counts."""
    with torch.no_grad():
        for v in model.state_dict().values():
            if v.dtype.is_floating_point:
                v.add_(torch.randn(v.shape, generator=g).to(v.device), alpha=scale)
            else:
                v += 1


def _assert_equal(mine, ref):
    a, b = mine.ema.state_dict(), ref.ema.state_dict()
    assert list(a) == list(b)
    bad = [k for k in a if not torch.equal(a[k], b[k])]
    assert not bad, bad[:5]


def _run(model, updates0, n, seed, edit=None):
    from cvpytorch_b200.ema import ModelEMA
    from oracle import ema_oracle as O
    g = torch.Generator().manual_seed(seed)
    mine, ref = ModelEMA(model, updates=updates0), O.ModelEMA(model, updates=updates0)
    for i in range(n):
        _train_step(model, g)
        if edit:
            model = edit(i, model, mine) or model
        mine.update(model)
        ref.update(model)
        assert mine.updates == ref.updates == updates0 + i + 1
        _assert_equal(mine, ref)
    return mine


@pytest.mark.parametrize('build', [_yolox, _yolov5], ids=['yolox_s', 'yolov5_s'])
def test_state_dict_updates_bitwise_equal_to_the_oracle(cuda, build):
    from cvpytorch_b200 import _lib
    model = build().cuda().train()
    g = torch.Generator().manual_seed(7)
    for v in model.state_dict().values():  # "trained" weights: away from the initialisation
        if v.dtype.is_floating_point:
            v.copy_(torch.randn(v.shape, generator=g))
    n0 = _lib.launch_count()
    _run(model, 0, 30, seed=11)
    assert _lib.launch_count() - n0 == 30  # one launch per update
    _run(model, 10 ** 6, 5, seed=12)
    _run(model, 2 ** 31 + 5, 3, seed=13)


class _Awkward(nn.Module):
    """Entries of 0, 1, 3, 4k + 1 elements and more than one chunk, and views into one buffer at every offset modulo 16 bytes."""

    def __init__(self, device):
        super().__init__()
        for n in (0, 1, 3, 5, 4097, 3 * 4096 + 1, 1 << 20, (1 << 20) + 3):
            self.register_buffer(f'b{n}', torch.randn(n, device=device))
        big = torch.randn(4 * 20000 + 64, device=device)  # (made on the device: .cuda() would copy each view to its own allocation)
        for off in range(4):
            self.register_buffer(f'view{off}', big[off * 20001: off * 20001 + 20000 - off])
        self.register_buffer('count', torch.zeros((), dtype=torch.long))
        self.w = nn.Parameter(torch.randn(7, 3, 3, 3, device=device))


def test_awkward_sizes_and_misaligned_views(cuda):
    model = _Awkward(cuda)
    assert {model.get_buffer(f'view{o}').data_ptr() % 16 for o in range(4)} == {0, 4, 8, 12}

    def shift(i, model, mine):  # the EMA's copy of view0 moved 4 bytes off the model's alignment, then back
        if i in (2, 5):
            e = mine.ema.view0
            store = torch.empty(e.numel() + 1, device=e.device)
            store[1 - (i == 5):][:e.numel()] = e
            mine.ema.view0 = store[1 - (i == 5):][:e.numel()]
    _run(model, 0, 8, seed=21, edit=shift)
    _run(model, 123456, 3, seed=22)


def test_replaced_tensors_between_updates(cuda):
    """.cpu().cuda() of the model and of the EMA, load_state_dict(assign=True) and convert_sync_batchnorm: the next update still matches."""
    model = _yolox().cuda().train()

    def edit(i, model, mine):
        if i == 1:
            return model.cpu().cuda()
        if i == 2:
            mine.ema.cpu().cuda()
        if i == 3:
            model.load_state_dict({k: v.clone() for k, v in model.state_dict().items()}, assign=True)
        if i == 4:
            mine.ema.load_state_dict({k: v.clone() for k, v in mine.ema.state_dict().items()}, assign=True)
        if i == 5:
            return nn.SyncBatchNorm.convert_sync_batchnorm(model)
        if i == 6:
            mine.ema = nn.SyncBatchNorm.convert_sync_batchnorm(mine.ema)
    _run(model, 0, 8, seed=31, edit=edit)


def test_update_refusals_on_the_device(cuda):
    from cvpytorch_b200 import _lib
    from cvpytorch_b200.ema import ModelEMA
    from oracle import ema_oracle as O
    model = O.fixture_model().cuda()
    ema = ModelEMA(model)
    ema.ema[3].bias.data = ema.ema[3].bias.data.cpu()
    with pytest.raises(_lib.CvbError, match='no CPU fallback'):
        ema.update(model)
    ema = ModelEMA(model)
    ema.ema[1].running_var = ema.ema[1].running_var.half()
    with pytest.raises(NotImplementedError, match='only fp32'):
        ema.update(model)


def _yolox_batch(B=2, H=128):
    g = torch.Generator().manual_seed(77)
    imgs = torch.randn(B, 3, H, H, generator=g).cuda()
    targets = []
    for b in range(B):
        n = 3 + b
        c = 20 + torch.rand(n, 2, generator=g) * (H - 40)
        wh = 16 + torch.rand(n, 2, generator=g) * 40
        targets.append({'labels': torch.randint(0, 80, (n,), generator=g).cuda(), 'boxes': torch.cat([c, wh], 1).cuda()})
    return imgs, targets


def _yolov5_batch(B=2, size=256):
    g = torch.Generator().manual_seed(21)
    imgs = torch.rand((B, 3, size, size), generator=g).cuda()
    targets = []
    for i in range(B):
        n = 3 + i
        boxes = torch.cat([torch.rand((n, 2), generator=g) * 0.8 + 0.1, torch.rand((n, 2), generator=g) * 0.3 + 0.05], 1)
        targets.append({'labels': torch.randint(0, 80, (n,), generator=g), 'boxes': boxes})
    return imgs, targets


def _same_val(a, b):
    (la, oa), (lb, ob) = a, b
    assert set(la) == set(lb) and len(oa) == len(ob)
    for x, y in zip(oa, ob):
        assert set(x) == set(y) and all(torch.equal(x[k], y[k]) for k in x)


@pytest.mark.parametrize('kind', ['yolox', 'yolov5'])
def test_trainer_flow_ema_validation_and_deep_copies(cuda, kind):
    """trainer_det_yolox.py / trainer_det_yolov5.py: training steps each followed by ema.update(model); validation of ema.ema; deepcopy of
    ema.ema and of the model for the checkpoint.  The copies validate bitwise like the originals, and a training step of a copy leaves the
    original's parameters alone."""
    from cvpytorch_b200.ema import ModelEMA
    from oracle import ema_oracle as O
    model = (_yolox() if kind == 'yolox' else _yolov5()).cuda().train()
    imgs, targets = _yolox_batch() if kind == 'yolox' else _yolov5_batch()
    ema, ref = ModelEMA(model), O.ModelEMA(model)
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9)
    for _ in range(3):
        model(imgs, targets, 'train')['loss'].backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        ema.update(model)
        ref.update(model)
        _assert_equal(ema, ref)
    ema.ema.eval()
    val_targets = targets if kind == 'yolox' else None
    with torch.no_grad():
        got = ema.ema(imgs, val_targets, 'val')
        ema_copy = copy.deepcopy(ema.ema)
        assert ema.ema._graphs and not ema_copy._graphs
        _same_val(ema_copy(imgs, val_targets, 'val'), got)
        model.eval()
        mval = model(imgs, val_targets, 'val')
        model_copy = copy.deepcopy(model)
        _same_val(model_copy(imgs, val_targets, 'val'), mval)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    model_copy.train()
    copt = torch.optim.SGD(model_copy.parameters(), lr=0.01, momentum=0.9)
    model_copy(imgs, targets, 'train')['loss'].backward()
    copt.step()
    assert all(p.grad is None for p in model.parameters())
    after = model.state_dict()
    assert all(torch.equal(after[k], before[k]) for k in before)
    assert any(not torch.equal(model_copy.state_dict()[k], before[k]) for k in before)
    # the original still trains and validates on its own tensors
    model.train()
    model(imgs, targets, 'train')['loss'].backward()
    model.eval()
    with torch.no_grad():
        model(imgs, val_targets, 'val')


def test_deep_copy_of_fcos_and_encoder_decoder_after_val(cuda):
    from cvpytorch_b200 import synth
    torch.manual_seed(1029)
    fcos = synth.build_fcos(True)
    x = torch.randn(2, 3, 128, 128).cuda()
    with torch.no_grad():
        want = fcos(x, None, 'val')
        c = copy.deepcopy(fcos)
        got = c(x, None, 'val')
    assert fcos._graphs and c._graphs
    assert _flat_equal(got, want)
    seg = synth.build_deeplab(True)
    x = torch.randn(2, 3, 128, 256).cuda()
    with torch.no_grad():
        want = seg(x, torch.zeros(2, 128, 256), 'val')
        c = copy.deepcopy(seg)
        got = c(x, torch.zeros(2, 128, 256), 'val')
    assert torch.equal(got, want)


def _flat_equal(a, b):
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and torch.equal(a, b)
    if isinstance(a, dict):
        return isinstance(b, dict) and set(a) == set(b) and all(_flat_equal(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return type(a) is type(b) and len(a) == len(b) and all(_flat_equal(x, y) for x, y in zip(a, b))
    return a == b


def test_ddp_wrapped_model_world_of_one(cuda):
    """ModelEMA(DistributedDataParallel(model)) copies model.module and updates from it (the reference's is_parallel branch)."""
    import torch.distributed as dist
    from cvpytorch_b200.ema import ModelEMA
    from oracle import ema_oracle as O
    assert not dist.is_initialized()
    with tempfile.TemporaryDirectory() as tmp:
        dist.init_process_group('gloo', init_method='file://' + os.path.join(tmp, 'store'), rank=0, world_size=1)
        try:
            inner = O.fixture_model().cuda()
            ddp = nn.parallel.DistributedDataParallel(inner, device_ids=[0])
            ema, ref = ModelEMA(ddp), O.ModelEMA(ddp)
            assert type(ema.ema) is nn.Sequential and list(ema.ema.state_dict()) == list(inner.state_dict())
            opt = torch.optim.SGD(ddp.parameters(), lr=0.1)
            x = torch.randn(2, 3, 16, 16, generator=torch.Generator().manual_seed(3)).cuda()
            for _ in range(4):
                ddp(x).square().mean().backward()
                opt.step()
                opt.zero_grad()
                ema.update(ddp)
                ref.update(ddp)
                _assert_equal(ema, ref)
            ema.update_attr(ddp)
            assert not hasattr(ema.ema, 'process_group') and not hasattr(ema.ema, 'reducer')
        finally:
            dist.destroy_process_group()
