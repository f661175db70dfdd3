"""The segmentation loss on the H100 (csrc/seg_loss.cu, seg_train.CrossEntropyLoss2d) against the reference fixture, the fp64 oracle
(oracle/seg_loss_oracle.py) and torch's own fp32 path on this GPU.

The loss must be within 1e-5 relative and the gradient within 1e-5 of the oracle's largest gradient element."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, 'tests', 'golden')


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _kernel(pred, target, ignore_index=255, loss_weight=1.0):
    from cvpytorch_b200 import seg_train as ST
    p = pred.detach().clone().requires_grad_(True)
    out = ST.CrossEntropyLoss2d(ignore_index=ignore_index, loss_weight=loss_weight)(p, target)
    out.backward()
    return out.detach(), p.grad


def _oracle(pred, target, ignore_index=255, loss_weight=1.0):
    from oracle import seg_loss_oracle as SO
    q = pred.detach().double().requires_grad_(True)
    out = SO.loss(q, target, ignore_index, loss_weight)
    out.backward()
    return out.detach(), q.grad


def _check(pred, target, what, ignore_index=255, loss_weight=1.0):
    got, grad = _kernel(pred, target, ignore_index, loss_weight)
    ref, rgrad = _oracle(pred.float(), target, ignore_index, loss_weight)
    assert got.dtype == torch.float32 and got.dim() == 0
    assert _rel(got, ref) <= 1e-5, (what, float(got), float(ref))
    assert grad.shape == pred.shape and grad.dtype == pred.dtype
    assert _rel(grad.float(), rgrad) <= (1e-5 if pred.dtype == torch.float32 else 1e-2), (what, _rel(grad.float(), rgrad))
    return got, grad


def _case(seed, B, C, h, w, H, W, dtype=torch.int64, ignore=0.1, dev='cuda'):
    g = torch.Generator().manual_seed(seed)
    pred = torch.randn(B, C, h, w, generator=g) * 3
    target = torch.randint(0, C, (B, H, W), generator=g)
    target[torch.rand(B, H, W, generator=g) < ignore] = 255
    return pred.to(dev), target.to(dtype).to(dev)


def test_kernel_reproduces_reference_fixture(cuda):
    """tests/golden/seg_loss.npz (the reference loss_forward + CrossEntropyLoss2d on the CPU): ×4 with uint8 labels, a 255 border and an
    image wholly ignored, ×8 at loss_weight 0.4, 13×29 -> 96×192, identity, a downsample; and every pixel ignored (NaN loss, zero
    gradient)."""
    from oracle import seg_loss_oracle as SO
    g = np.load(os.path.join(GOLD, 'seg_loss.npz'))
    for case in SO.CASES:
        pred = torch.from_numpy(g[f'{case}_pred']).to(cuda)
        target = torch.from_numpy(g[f'{case}_target']).to(cuda)
        ignore, lw = int(g[f'{case}_ignore_index']), float(g[f'{case}_loss_weight'])
        got, grad = _kernel(pred, target, ignore, lw)
        if case == 'ignored':
            assert torch.isnan(got) and not bool(grad.any()), case
            continue
        assert _rel(got, g[f'{case}_loss']) <= 1e-5, case
        assert _rel(grad, g[f'{case}_grad']) <= 1e-5, case
        _check(pred, target, case, ignore, lw)


RATIOS = {'x1': (24, 40, 24, 40), 'x4': (16, 24, 64, 96), 'x8': (8, 12, 64, 96), 'frac': (13, 29, 96, 192), 'down': (40, 56, 17, 23)}
LABEL_DTYPES = [torch.uint8, torch.int32, torch.int64]


@pytest.mark.parametrize('ratio', list(RATIOS))
@pytest.mark.parametrize('C', [1, 2, 19, 150, 'max'])
@pytest.mark.parametrize('B', [1, 3])
def test_kernel_vs_oracle_matrix(cuda, B, C, ratio):
    from cvpytorch_b200 import seg_train as ST
    C = ST.nc_max() if C == 'max' else C
    h, w, H, W = RATIOS[ratio]
    k = list(RATIOS).index(ratio)
    dtype = LABEL_DTYPES[(k + B) % 3]
    pred, target = _case(100 * B + k + C, B, C, h, w, H, W, torch.int64 if dtype == torch.uint8 and C > 255 else dtype)
    _check(pred, target, f'B={B} C={C} {ratio}', loss_weight=(1.0, 0.4, 2.5)[k % 3])


@pytest.mark.parametrize('sizes', [(1, 1, 200, 300), (2, 3, 200, 150), (3, 250, 90, 700), (64, 64, 5, 7), (33, 100, 1, 1), (7, 5, 7, 41)])
def test_extreme_ratios(cuda, sizes):
    """A footprint larger than one shared-memory block (1×1 -> 200×300), steep x30 and x100 upsamples, steep downsamples whose rows and
    columns do not all reach a full-res pixel, 1×1 outputs and mixed up / down axes."""
    h, w, H, W = sizes
    pred, target = _case(h * w + H, 2, 6, h, w, H, W, torch.int32)
    _check(pred, target, str(sizes))


def test_label_views_dtypes_and_ignore_index(cuda):
    """Non-contiguous label views of each dtype are read in place; any int64 ignore_index works, negative included."""
    pred, target = _case(7, 2, 19, 16, 24, 64, 96, torch.int64)
    for dtype in LABEL_DTYPES:
        wide = torch.full((2, 64, 200), 255, dtype=dtype, device=cuda)
        wide[:, :, 7:103] = target.to(dtype)
        view = wide[:, :, 7:103]
        assert not view.is_contiguous()
        _check(pred, view, f'view {dtype}')
        _check(pred, target.to(dtype).transpose(1, 2).contiguous().transpose(1, 2), f'transposed {dtype}')
    t = target.clone()
    t[t == 255] = -1
    _check(pred, t, 'ignore -1', ignore_index=-1)
    t[t == -1] = 1 << 40
    _check(pred, t, 'ignore 2^40', ignore_index=1 << 40)


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_half_precision_preds(cuda, dtype):
    """fp16 / bf16 head outputs are cast to fp32 inside the loss; the gradient flows back through the cast in their dtype."""
    pred, target = _case(9, 3, 19, 16, 24, 64, 96, torch.uint8)
    pred = pred.to(dtype)
    _check(pred, target, str(dtype))


def test_matches_torch_fp32_path(cuda):
    """The torch path on this GPU, F.interpolate + F.cross_entropy (valid labels and 255 only), agrees within the fp32 tolerance."""
    for (B, C, h, w, H, W) in ((2, 19, 32, 64, 128, 256), (2, 150, 16, 16, 128, 128), (1, 11, 45, 60, 360, 480)):
        pred, target = _case(11 + C, B, C, h, w, H, W, torch.uint8)
        assert int(target[target != 255].max()) < C
        p = pred.clone().requires_grad_(True)
        ref = F.cross_entropy(F.interpolate(p, size=(H, W), mode='bilinear', align_corners=False), target.long(), ignore_index=255)
        ref.backward()
        got, grad = _kernel(pred, target)
        assert _rel(got, ref) <= 1e-5 and _rel(grad, p.grad) <= 1e-5, (B, C, h, w, H, W)


def test_cityscapes_training_shape(cuda):
    """DeepLabv3+ on Cityscapes: 8 × 19 × 128×256 -> 512×1024 with uint8 labels and a 255 share."""
    pred, target = _case(13, 8, 19, 128, 256, 512, 1024, torch.uint8, ignore=0.15)
    _check(pred, target, 'cityscapes')


def test_ignored_and_out_of_range_labels(cuda):
    """Every pixel ignored: NaN loss, zero gradient.  One image ignored: the mean over the other image.  A label C or -1 (with the default
    ignore_index 255) makes the loss and every gradient element NaN; torch raises there, and its CUDA kernel asserts, so the check is
    against the specification, not torch."""
    from cvpytorch_b200 import seg_train as ST
    pred, target = _case(15, 2, 19, 16, 24, 64, 96, torch.uint8)
    got, grad = _kernel(pred, torch.full_like(target, 255))
    assert torch.isnan(got) and not bool(grad.any())
    t = target.clone()
    t[1] = 255
    _check(pred, t, 'one image ignored')
    _, g1 = _kernel(pred, t)
    assert not bool(g1[1].any())
    for bad, dtype in ((19, torch.uint8), (19, torch.int64), (-1, torch.int64), (-1, torch.int32)):
        t = target.to(dtype)
        t[0, 5, 7] = bad
        got, grad = _kernel(pred, t)
        assert torch.isnan(got) and bool(torch.isnan(grad).all()), (bad, dtype)
        _, _, record = ST.seg_ce_forward(pred, t)
        assert record.tolist()[1] == 1


def test_runs_and_graph_replay_are_bitwise_identical(cuda):
    """Two runs and a CUDA-graph replay of forward + backward give the same bits."""
    from cvpytorch_b200 import seg_train as ST
    pred, target = _case(17, 4, 19, 64, 128, 256, 512, torch.uint8)
    loss = ST.CrossEntropyLoss2d()
    p = pred.clone().requires_grad_(True)

    def run():
        p.grad = None
        out = loss(p, target)
        out.backward()
        return out.detach().clone(), p.grad.clone()
    a, b = run(), run()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    static = {}

    def body():
        out = loss(p, target)
        out.backward()
        static['out'] = out.detach()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        p.grad = None
        body()
    torch.cuda.current_stream().wait_stream(side)
    p.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        body()
    p.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static['out'], a[0]) and torch.equal(p.grad, a[1])


def test_no_host_sync(cuda):
    """Forward and backward make no host sync."""
    from cvpytorch_b200 import seg_train as ST
    pred, target = _case(19, 2, 19, 32, 64, 128, 256, torch.uint8)
    loss = ST.CrossEntropyLoss2d()
    p = pred.clone().requires_grad_(True)
    loss(p, target).backward()  # first call: library load and kernel attributes
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = loss(p, target)
        out.backward()
    finally:
        torch.cuda.set_sync_debug_mode('default')
    torch.cuda.synchronize()
    assert torch.isfinite(out)


class _Segmenter(torch.nn.Module):
    """A small torch segmenter whose head runs at 1/4 of the input resolution."""

    def __init__(self, C):
        super().__init__()
        self.body = torch.nn.Sequential(torch.nn.Conv2d(3, 16, 3, 2, 1), torch.nn.BatchNorm2d(16), torch.nn.ReLU(),
                                        torch.nn.Conv2d(16, 32, 3, 2, 1), torch.nn.BatchNorm2d(32), torch.nn.ReLU())
        self.head = torch.nn.Conv2d(32, C, 1)

    def forward(self, x):
        return self.head(self.body(x))


class _TorchCE(torch.nn.Module):
    """The reference CrossEntropyLoss2d: loss_weight * nn.CrossEntropyLoss(ignore_index=255) on already upsampled preds."""
    loss_name = 'ce_loss'

    def __init__(self, loss_weight=1.0):
        super().__init__()
        self.loss_weight = loss_weight
        self.criterion = torch.nn.CrossEntropyLoss(ignore_index=255)

    def forward(self, pred, target):
        return self.loss_weight * self.criterion(pred, target.long())


def test_grad_scaler_training_matches_torch_path(cuda):
    """Four GradScaler + SGD steps of a small fp32 segmenter: training through seg_train.loss_forward (the drop-in CrossEntropyLoss2d plus a
    plain torch loss under the same name in the list) tracks training through F.interpolate + nn.CrossEntropyLoss."""
    from cvpytorch_b200 import seg_train as ST
    C = 19
    torch.manual_seed(0)
    a = _Segmenter(C).to(cuda)
    b = _Segmenter(C).to(cuda)
    b.load_state_dict(a.state_dict())
    g = torch.Generator().manual_seed(21)
    batches = []
    for _ in range(4):
        x = torch.randn(4, 3, 128, 192, generator=g)
        t = torch.randint(0, C, (4, 128, 192), generator=g).to(torch.uint8)
        t[:, :4] = 255
        batches.append((x.to(cuda), t.to(cuda)))

    def train(model, loss_fn, losses):
        opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9)
        scaler = torch.amp.GradScaler('cuda')
        seen = []
        for x, t in batches:
            opt.zero_grad()
            pred = model(x)
            assert bool(torch.isfinite(pred).all())
            out = loss_fn(None, pred, t, losses)
            total = sum(out.values())
            scaler.scale(total).backward()
            scaler.step(opt)
            scaler.update()
            seen.append({k: float(v.detach()) for k, v in out.items()})
        return seen
    def reference_loss_forward(self, preds, targets, loss):
        up = F.interpolate(preds, size=targets.shape[-2:], mode='bilinear', align_corners=False)
        losses = {}
        for l in loss:
            v = l(up, targets)
            losses[l.loss_name] = losses[l.loss_name] + v if l.loss_name in losses else v
        return losses
    sa = train(a, ST.loss_forward, torch.nn.ModuleList([ST.CrossEntropyLoss2d(), _TorchCE(0.4)]))
    sb = train(b, reference_loss_forward, torch.nn.ModuleList([_TorchCE(), _TorchCE(0.4)]))
    for x, y in zip(sa, sb):
        assert abs(x['ce_loss'] - y['ce_loss']) <= 1e-4 * abs(y['ce_loss']), (sa, sb)
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert _rel(pa, pb) <= 1e-3
