"""The FCOS loss on the H100 (csrc/fcos_loss.cu, fcos_train.FCOSLoss) against the reference fixture and the oracle (oracle/fcos_loss_oracle.py,
fp32 on this GPU).

matched_gt and the per-point targets must equal the oracle's bitwise; the four losses must be within 1e-5 relative and every head-output
gradient of total_loss within 1e-5 max-normalised."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, 'tests', 'golden')
NAMES = ('cls', 'cnt', 'reg')
LOSSES = ('cls_loss', 'cnt_loss', 'reg_loss', 'total_loss')


def _LO():
    from oracle import fcos_loss_oracle as LO
    return LO


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _leaves(preds, dtype=None):
    return [[(t.detach().to(dtype) if dtype else t.detach().clone()).requires_grad_(True) for t in lv] for lv in preds]


def _kernel(preds, boxes, labels, weights=None):
    """-> (the four losses, matched_gt int64 [B, A], targets [B, A, 5], gradients) through FCOSLoss; the backward of
    sum_i weights[i] out[i] (default: total_loss alone)."""
    from cvpytorch_b200 import fcos_train as FT
    LO = _LO()
    ps = _leaves(preds)
    out = FT.FCOSLoss()(ps, boxes, labels)
    w = weights if weights is not None else (0.0, 0.0, 0.0, 1.0)
    torch.autograd.backward([o for o in out], [torch.tensor(x, device=out[0].device) for x in w])
    b, lab = FT._loss_targets(boxes, labels, boxes.shape[0], preds[0][0].shape[1], preds[0][0].device)
    _, mg, _, tgt = FT.fcos_loss_forward([[t.detach() for t in lv] for lv in ps], b, lab, LO.STRIDES, LO.LIMIT_RANGE, return_targets=True)
    return out, mg.long(), tgt, [[t.grad for t in lv] for lv in ps]


def _oracle(preds, boxes, labels, weights=None):
    LO = _LO()
    ps = _leaves(preds)
    out, asg = LO.losses(ps, boxes, labels)
    w = weights if weights is not None else (0.0, 0.0, 0.0, 1.0)
    torch.autograd.backward([o for o in out], [torch.tensor(x, device=out[0].device) for x in w])
    return out, asg, [[t.grad for t in lv] for lv in ps]


def _check(preds, boxes, labels, what, weights=None):
    got, mg, tgt, grads = _kernel(preds, boxes, labels, weights)
    ref, (cls_t, cnt_t, reg_t, rmg), rgrads = _oracle(preds, boxes, labels, weights)
    assert torch.equal(mg, rmg), what
    assert torch.equal(tgt[..., 0], cnt_t) and torch.equal(tgt[..., 1:], reg_t), what
    for k, name in enumerate(LOSSES):
        assert _rel(got[k], ref[k]) < 1e-5, (what, name, float(got[k]), float(ref[k]))
    for i, name in enumerate(NAMES):
        for l, (g, r) in enumerate(zip(grads[i], rgrads[i])):
            assert _rel(g, r) < 1e-5, (what, name, l, _rel(g, r))
    return int((mg >= 0).sum())


def _random_case(seed, B, H, W, nc, counts, dev):
    """Seeded head outputs and padded targets: counts[b] random GTs in image b (8 to 60 % of the side), a few labelled outside 1..nc, -1 rows
    after them; a share of the positives predict their target exactly (GIoU ties)."""
    LO = _LO()
    g = torch.Generator().manual_seed(seed)
    m = max(counts)
    boxes = torch.full((B, m, 4), -1.0)
    labels = torch.full((B, m), -1, dtype=torch.long)
    for b, n in enumerate(counts):
        if n:
            wh = 8 + torch.rand(n, 2, generator=g) * torch.tensor([0.6 * W, 0.6 * H])
            xy = torch.rand(n, 2, generator=g) * (torch.tensor([W, H]) - wh)
            boxes[b, :n] = torch.cat([xy, xy + wh], 1)
            labels[b, :n] = torch.randint(1, nc + 1, (n,), generator=g)
            odd = torch.rand(n, generator=g) < 0.05
            labels[b, :n][odd] = torch.where(torch.rand(int(odd.sum()), generator=g) < 0.5, -1, nc + 1)
    preds = LO.head_outputs(B, nc, LO.level_shapes(H, W), LO.STRIDES, g)
    LO.tie_predictions(preds, boxes, labels, g, share=0.05)
    preds = [[t.to(dev) for t in lv] for lv in preds]
    return preds, boxes.to(dev), labels.to(dev)


def test_kernel_reproduces_reference_fixture(cuda):
    """tests/golden/fcos_loss.npz (the reference FCOSLoss on the CPU): matched GT, class and regression targets bitwise, the centerness
    target within 1 ulp (torch's CPU sqrt), the four losses within 1e-5 relative, the gradients of total_loss within 1e-5 max-normalised;
    and everything against the oracle on this GPU, the targets bitwise."""
    g = np.load(os.path.join(GOLD, 'fcos_loss.npz'))
    for case in _LO().CASES:
        n = len(_LO().STRIDES)
        preds = [[torch.from_numpy(g[f'{case}_{name}{l}']).to(cuda) for l in range(n)] for name in NAMES]
        boxes, labels = torch.from_numpy(g[f'{case}_boxes']).to(cuda), torch.from_numpy(g[f'{case}_labels']).to(cuda)
        got, mg, tgt, grads = _kernel(preds, boxes, labels)
        cnt_t, reg_t = torch.from_numpy(g[f'{case}_cnt_t'])[..., 0], torch.from_numpy(g[f'{case}_reg_t'])
        assert torch.equal(tgt[..., 1:].cpu(), reg_t), case
        # the centerness is one correctly rounded sqrt here and in torch on the GPU; torch's CPU sqrt, which wrote the fixture, rounds
        # about 0.6 % of fp32 values the other way: 1 ulp at most (bitwise against the oracle on this GPU in _check below)
        ulp = (tgt[..., 0].cpu().view(torch.int32).long() - cnt_t.view(torch.int32).long()).abs()
        assert int(ulp.max()) <= 1, case
        assert torch.equal((mg >= 0).cpu(), cnt_t > -1), case
        cls_t = torch.where(mg >= 0, labels.gather(1, mg.clamp(min=0)), torch.zeros_like(mg)).cpu()
        assert torch.equal(cls_t, torch.from_numpy(g[f'{case}_cls_t'])[..., 0]), case
        for k, name in enumerate(LOSSES):
            assert _rel(got[k], g[f'{case}_{name}']) < 1e-5, (case, name)
        for i, name in enumerate(NAMES):
            for l, gr in enumerate(grads[i]):
                assert _rel(gr, g[f'{case}_grad_{name}{l}']) < 1e-5, (case, name, l)
        _check(preds, boxes, labels, case)


SIZES = {'128': (128, 128), '800': (800, 800), '608x800': (608, 800)}


@pytest.mark.parametrize('size', list(SIZES))
@pytest.mark.parametrize('nc', [1, 3, 80])
@pytest.mark.parametrize('B', [1, 4, 16])
def test_kernel_vs_oracle_matrix(cuda, B, nc, size):
    """0 to 100 GTs per image; 800² has 100² + 50² + 25² + 13² + 7² = 13 343 points per image."""
    H, W = SIZES[size]
    counts = [[3, 0, 100, 17, 42, 1, 8, 64, 25, 0, 77, 5, 12, 30, 2, 90][i % 16] for i in range(B)]
    if B == 1:
        counts = [[7], [40], [100]][[1, 3, 80].index(nc)]
    preds, boxes, labels = _random_case(1000 * B + 10 * nc + len(size), B, H, W, nc, counts, cuda)
    if size == '800':
        assert sum(p.shape[2] * p.shape[3] for p in preds[0]) == 13343
    npos = _check(preds, boxes, labels, f'B={B} nc={nc} {size}')
    assert npos > 0


def test_empty_gt_list_and_all_padded_image(cuda):
    """m = 0 is an all-background batch (cnt and reg losses 0, num_pos clamps to 1); an image whose rows are all padding has no positive
    while the other image of the batch does."""
    from cvpytorch_b200 import fcos_train as FT
    preds, _, _ = _random_case(7, 2, 128, 128, 3, [1, 1], cuda)
    boxes, labels = torch.zeros(2, 0, 4, device=cuda), torch.zeros(2, 0, dtype=torch.long, device=cuda)
    got, mg, tgt, _ = _kernel(preds, boxes, labels)
    assert bool((mg == -1).all()) and bool((tgt == -1).all()) and float(got[1]) == 0.0 and float(got[2]) == 0.0
    _check(preds, boxes, labels, 'm=0')
    _, _, npos = FT.fcos_loss_forward(preds, boxes.contiguous(), labels.int().contiguous(), _LO().STRIDES, _LO().LIMIT_RANGE)
    assert npos.tolist() == [0, 0]
    preds, boxes, labels = _random_case(8, 2, 256, 256, 3, [6, 0], cuda)
    assert bool((boxes[1] == -1).all())
    got, mg, _, _ = _kernel(preds, boxes, labels)
    assert int((mg[1] >= 0).sum()) == 0 and int((mg[0] >= 0).sum()) > 0
    _check(preds, boxes, labels, 'all-padded image')


def _saturate(preds, boxes, labels):
    """Class logits whose sigmoid rounds to 1 against a 0 target (+30 at background points) and to 0 against a 1 target (-200 at the
    matched class of positives): inf cls_loss, NaN gradients there."""
    LO = _LO()
    shapes = [tuple(c.shape[2:]) for c in preds[0]]
    cls_t, _, _, mg = LO.targets(shapes, boxes, labels)
    o = 0
    for c in preds[0]:
        B, nc, h, w = c.shape
        ct = cls_t[:, o:o + h * w].reshape(B, h, w)
        bg = (ct == 0).nonzero()[::97]
        c[bg[:, 0], 0, bg[:, 1], bg[:, 2]] = 30.0
        fg = ((ct >= 1) & (ct <= nc)).nonzero()[::5]
        c[fg[:, 0], ct[fg[:, 0], fg[:, 1], fg[:, 2]] - 1, fg[:, 1], fg[:, 2]] = -200.0
        o += h * w


def test_saturated_logits_and_grad_scaler_skip(cuda):
    """inf losses and NaN gradients at the same places as the oracle; a GradScaler + SGD step skips exactly as it does with the oracle
    (parameters unchanged, scale halved), and an unsaturated step is taken by both."""
    preds, boxes, labels = _random_case(11, 4, 256, 256, 3, [5, 9, 0, 3], cuda)
    _saturate(preds, boxes, labels)
    got, mg, _, grads = _kernel(preds, boxes, labels)
    ref, (_, _, _, rmg), rgrads = _oracle(preds, boxes, labels)
    assert torch.equal(mg, rmg)
    assert float(got[0]) == float('inf') and float(ref[0]) == float('inf') and float(got[3]) == float('inf')
    assert _rel(got[1], ref[1]) < 1e-5 and _rel(got[2], ref[2]) < 1e-5
    nan = 0
    for i in range(3):
        for g, r in zip(grads[i], rgrads[i]):
            assert torch.equal(torch.isnan(g), torch.isnan(r)) and torch.equal(torch.isinf(g), torch.isinf(r))
            ok = torch.isfinite(r)
            assert _rel(g[ok], r[ok]) < 1e-5
            nan += int(torch.isnan(g).sum())
    assert nan > 0

    from cvpytorch_b200 import fcos_train as FT
    LO = _LO()

    def step(loss_fn, inputs):
        params = [torch.nn.Parameter(t.detach().clone()) for lv in inputs for t in lv]
        n = len(inputs[0])
        ps = [params[k * n:(k + 1) * n] for k in range(3)]
        opt = torch.optim.SGD(params, lr=0.1, momentum=0.9)
        scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 16)
        out = loss_fn(ps)
        scaler.scale(out[3]).backward()
        scaler.step(opt)
        scaler.update()
        return [p.detach() for p in params], scaler.get_scale()

    clean, _, _ = _random_case(11, 4, 256, 256, 3, [5, 9, 0, 3], cuda)
    for inputs, skips in ((preds, True), (clean, False)):
        kp, ks = step(lambda ps: FT.FCOSLoss()(ps, boxes, labels), inputs)
        op, os_ = step(lambda ps: LO.losses(ps, boxes, labels)[0], inputs)
        flat_in = [t for lv in inputs for t in lv]
        assert ks == os_ == (2.0 ** 15 if skips else 2.0 ** 16)
        # a taken step moves every tensor with a non-zero gradient (a level without positives leaves its reg / cnt maps unchanged)
        assert [torch.equal(a, x) for a, x in zip(kp, flat_in)] == [torch.equal(b, x) for b, x in zip(op, flat_in)]
        assert all(torch.equal(a, x) for a, x in zip(kp, flat_in)) == skips
        if not skips:
            for a, b, x in zip(kp, op, flat_in):
                assert _rel(a - x, b - x) < 1e-4


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_half_precision_head_outputs(cuda, dtype):
    """fp16 / bf16 head outputs (autocast) are cast to fp32 inside the loss and the gradients flow back through the cast in their dtype."""
    from cvpytorch_b200 import fcos_train as FT
    LO = _LO()
    preds, boxes, labels = _random_case(21, 4, 256, 256, 80, [4, 30, 0, 12], cuda)
    preds = [[t.to(dtype) for t in lv] for lv in preds]
    ps, qs = _leaves(preds), _leaves(preds)
    out = FT.FCOSLoss()(ps, boxes, labels)
    out[3].backward()
    ref, _ = LO.losses([[t.float() for t in lv] for lv in qs], boxes, labels)
    ref[3].backward()
    for k in range(4):
        assert out[k].dtype == torch.float32 and _rel(out[k], ref[k]) < 1e-5
    for a, b in zip(ps, qs):
        for x, y in zip(a, b):
            assert x.grad.dtype == dtype and _rel(x.grad.float(), y.grad.float()) < 1e-2


def test_each_output_gradient_scaled_separately(cuda):
    """The backward scales the three terms by their own incoming gradient plus the total's: each of the four outputs alone, and a mix."""
    preds, boxes, labels = _random_case(31, 4, 256, 256, 3, [6, 0, 20, 2], cuda)
    for w in ((1.0, 0.0, 0.0, 0.0), (0.0, 2.5, 0.0, 0.0), (0.0, 0.0, -0.75, 0.0), (0.0, 0.0, 0.0, 3.0), (0.5, -1.0, 2.0, 0.25)):
        _check(preds, boxes, labels, f'weights {w}', weights=w)


def test_runs_and_graph_replay_are_bitwise_identical(cuda):
    """Two runs and a CUDA-graph replay of forward + backward give the same bits; the loss makes no host sync while captured."""
    from cvpytorch_b200 import fcos_train as FT
    preds, boxes, labels = _random_case(41, 16, 800, 800, 80, [3, 0, 100, 17, 42, 1, 8, 64, 25, 0, 77, 5, 12, 30, 2, 90], cuda)
    loss = FT.FCOSLoss()
    ps = _leaves(preds)

    def run():
        for lv in ps:
            for t in lv:
                t.grad = None
        out = loss(ps, boxes, labels)
        out[3].backward()
        return torch.stack(out).detach().clone(), [t.grad.clone() for lv in ps for t in lv]
    a, b = run(), run()
    assert torch.equal(a[0], b[0]) and all(torch.equal(x, y) for x, y in zip(a[1], b[1]))
    static = {}

    def body():
        out = loss(ps, boxes, labels)
        out[3].backward()
        static['out'] = torch.stack(out)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for lv in ps:
            for t in lv:
                t.grad = None
        body()
    torch.cuda.current_stream().wait_stream(side)
    for lv in ps:
        for t in lv:
            t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        body()
    for lv in ps:
        for t in lv:
            t.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static['out'], a[0])
    assert all(torch.equal(t.grad, y) for t, y in zip([t for lv in ps for t in lv], a[1]))
