"""The YOLOX loss on the H100 (csrc/yolox_loss.cu, train.YOLOXLoss) and the model-level training forward (yolox_models.YOLOX, mode='train').

Assignments (foreground mask, matched GT) must equal the oracle's (oracle/yolox_loss_oracle.py, fp32 on this GPU) in every image without a
near-tie (oracle.near_ties, float64); the loss terms must be within 1e-5 relative and the head-output gradients within 1e-5 max-normalised of
the oracle's under the kernel's own assignment."""
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
KEYS = ('loss', 'iou_loss', 'conf_loss', 'cls_loss', 'num_fg')
STRIDES = (8, 16, 32)


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def _kernel(preds, targets, nc):
    """-> (loss dict, (fg, matched_gt, matched_iou), head-output gradients of loss['loss'])."""
    from cvpytorch_b200 import train as T
    ps = [p.detach().clone().requires_grad_(True) for p in preds]
    out = T.YOLOXLoss(nc)(ps, targets)
    out['loss'].backward()
    _, mg, mi = T.yolox_loss_forward([p.detach() for p in ps], targets, STRIDES, nc)
    return out, (mg >= 0, mg.long(), mi), [p.grad for p in ps]


def _oracle(preds, targets, nc, assignment=None):
    from oracle import yolox_loss_oracle as LO
    ps = [p.detach().clone().requires_grad_(True) for p in preds]
    out, asg = LO.losses(ps, targets, STRIDES, nc, assignment)
    out['loss'].backward()
    return out, asg, [p.grad for p in ps]


def _check(preds, targets, nc, what):
    """Kernel vs oracle; returns the number of images whose assignment was compared."""
    from oracle import yolox_loss_oracle as LO
    got, (fg, mg, mi), grads = _kernel(preds, targets, nc)
    torch.cuda.synchronize()
    ref, (rfg, rmg, rmi), _ = _oracle(preds, targets, nc)
    ties = LO.near_ties([p.cpu() for p in preds], targets.cpu(), STRIDES, nc)
    compared = 0
    for b in range(targets.shape[0]):
        if ties[b]:
            continue
        compared += 1
        assert torch.equal(fg[b], rfg[b]) and torch.equal(mg[b], rmg[b]), (what, b)
        assert _rel(mi[b], rmi[b]) < 1e-5, (what, b)
    under, _, rgrads = _oracle(preds, targets, nc, (fg, mg, mi))
    for k in KEYS:
        assert _rel(got[k], under[k]) < 1e-5, (what, k, float(got[k]), float(under[k]))
    for i, (g, r) in enumerate(zip(grads, rgrads)):
        assert _rel(g, r) < 1e-5, (what, i, _rel(g, r))
    return compared


def _random_case(seed, B, H, W, nc, ngts, far=False):
    """Seeded head outputs and targets: ngts[b] random GTs in image b (zero rows after them); 70 % of the anchors near a GT predict a
    jittered copy of it.  far: every GT lies far outside the image (no candidate anchor)."""
    g = torch.Generator().manual_seed(seed)
    G = max(max(ngts), 1)
    t = torch.zeros(B, G, 5)
    for b, n in enumerate(ngts):
        if n:
            wh = 8 + torch.rand(n, 2, generator=g) * torch.tensor([W / 3, H / 3])
            c = torch.rand(n, 2, generator=g) * torch.tensor([W, H]) + (10 * max(H, W) if far else 0)
            t[b, :n] = torch.cat([torch.randint(0, nc, (n, 1), generator=g).float(), c, wh], 1)
    preds = []
    for s in STRIDES:
        h, w = H // s + 2, W // s + 2
        p = torch.randn(B, 5 + nc, h, w, generator=g)
        p[:, 4:] = p[:, 4:] * 1.5 - 2.0
        yv, xv = torch.meshgrid(torch.arange(h).float(), torch.arange(w).float(), indexing='ij')
        xc, yc = (xv + 0.5) * s, (yv + 0.5) * s
        for b, n in enumerate(ngts):
            if not n:
                continue
            pick = torch.randint(0, n, (h, w), generator=g)
            cls, cx, cy, bw, bh = (t[b, :n, i][pick] for i in range(5))
            take = ((xc - cx).abs() < 2.5 * s + bw / 2) & ((yc - cy).abs() < 2.5 * s + bh / 2) & (torch.rand(h, w, generator=g) < 0.7)
            jit = torch.randn(4, h, w, generator=g)
            p[b, 0] = torch.where(take, (cx + 0.15 * bw * jit[0]) / s - xv, p[b, 0])
            p[b, 1] = torch.where(take, (cy + 0.15 * bh * jit[1]) / s - yv, p[b, 1])
            p[b, 2] = torch.where(take, torch.log(bw * (1 + 0.2 * jit[2]).clamp(min=0.3) / s), p[b, 2])
            p[b, 3] = torch.where(take, torch.log(bh * (1 + 0.2 * jit[3]).clamp(min=0.3) / s), p[b, 3])
            p[b, 4] = torch.where(take, p[b, 4] + 2.0, p[b, 4])
        preds.append(p.cuda())
    return preds, t.cuda()


def test_kernel_reproduces_reference_fixture(cuda):
    """tests/golden/yolox_loss.npz (the reference YOLOXLoss): identical assignment, loss terms within 1e-5 relative, gradients within 1e-5
    max-normalised.  The fixture has no near-tie."""
    from oracle import yolox_loss_oracle as LO
    g = np.load(os.path.join(GOLD, 'yolox_loss.npz'))
    for case, (B, H, nc) in LO.CASES.items():
        preds, targets = LO.fixture_case(int(g[f'{case}_seed']), case)
        got, (fg, mg, mi), grads = _kernel([p.cuda() for p in preds], targets.cuda(), nc)
        assert np.array_equal(fg.cpu().numpy(), g[f'{case}_fg'])
        assert np.array_equal(mg.cpu().numpy(), g[f'{case}_matched_gt'])
        assert _rel(mi, g[f'{case}_matched_iou']) < 1e-5
        for k in KEYS:
            assert _rel(got[k], g[f'{case}_{k}']) < 1e-5, (case, k)
        for i, gr in enumerate(grads):
            assert _rel(gr, g[f'{case}_grad{i}']) < 1e-5, (case, i, _rel(gr, g[f'{case}_grad{i}']))


@pytest.mark.parametrize('B', [1, 4, 16])
@pytest.mark.parametrize('nc', [1, 3, 80])
def test_kernel_vs_oracle_matrix(cuda, B, nc):
    """0 to 256 GTs per image at 128 x 160 (the image with 256 GTs is in every batch of 4 or more)."""
    counts = [[0, 1, 7, 256, 30, 3, 64, 12, 0, 100, 5, 17, 2, 40, 9, 150][i % 16] for i in range(B)]
    if B == 1:
        counts = [[5], [40], [256]][[1, 3, 80].index(nc)]
    preds, targets = _random_case(100 * B + nc, B, 128, 160, nc, counts)
    compared = _check(preds, targets, nc, f'B={B} nc={nc}')
    print('images compared (no near-tie):', compared, 'of', B)


def test_all_empty_batch_and_gt_without_candidates(cuda):
    """No GT at all: num_fg clamps to 1, everything is background.  A GT far outside the image has no candidate anchor and matches nothing."""
    preds, targets = _random_case(5, 3, 128, 128, 3, [0, 0, 0])
    out, (fg, _, _), _ = _kernel(preds, targets, 3)
    assert not bool(fg.any()) and float(out['num_fg']) == 1.0 and float(out['iou_loss'].detach()) == 0.0 and float(out['cls_loss'].detach()) == 0.0
    _check(preds, targets, 3, 'empty')
    preds, targets = _random_case(6, 2, 128, 128, 3, [2, 0], far=True)
    out, (fg, _, _), _ = _kernel(preds, targets, 3)
    assert not bool(fg.any()) and abs(float(out['num_fg']) - 0.5) < 1e-7
    _check(preds, targets, 3, 'far')


def test_yolox_s_640_shapes(cuda):
    """YOLOX-s at 640 x 640: 82² + 42² + 22² = 8972 anchors per image, 80 classes, 8 to 100 GTs per image."""
    preds, targets = _random_case(640, 4, 640, 640, 80, [8, 100, 37, 61])
    assert sum(p.shape[2] * p.shape[3] for p in preds) == 8972
    compared = _check(preds, targets, 80, '640')
    print('images compared (no near-tie):', compared, 'of 4')


def test_bitwise_reproducible_and_graph_replay(cuda):
    from cvpytorch_b200 import train as T
    preds, targets = _random_case(11, 4, 128, 160, 80, [3, 0, 50, 256])
    loss = T.YOLOXLoss(80)

    def step():
        ps = [p.detach().clone().requires_grad_(True) for p in preds]
        out = loss(ps, targets)
        out['loss'].backward()
        return torch.stack([out[k].detach() for k in KEYS]), [p.grad for p in ps]
    a, ga = step()
    b, gb = step()
    assert torch.equal(a, b) and all(torch.equal(x, y) for x, y in zip(ga, gb))
    static = [p.detach().clone().requires_grad_(True) for p in preds]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        out = loss(static, targets)
        out['loss'].backward()
    torch.cuda.current_stream().wait_stream(side)
    for p in static:
        p.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = loss(static, targets)
        out['loss'].backward()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(torch.stack([out[k].detach() for k in KEYS]), a)
    assert all(torch.equal(p.grad, g) for p, g in zip(static, ga))


def test_grad_output_scaling(cuda):
    """A GradScaler-scaled loss gives scale x the gradient; back-propagating conf_loss alone matches the oracle's."""
    from cvpytorch_b200 import train as T
    preds, targets = _random_case(12, 2, 128, 128, 3, [6, 9])
    loss = T.YOLOXLoss(3)
    ps = [p.clone().requires_grad_(True) for p in preds]
    loss(ps, targets)['loss'].backward()
    base = [p.grad.clone() for p in ps]
    scaler = torch.amp.GradScaler('cuda', init_scale=1024.0)
    ps = [p.clone().requires_grad_(True) for p in preds]
    scaler.scale(loss(ps, targets)['loss']).backward()
    for p, g in zip(ps, base):
        assert torch.equal(p.grad, g * 1024.0)
    ps = [p.clone().requires_grad_(True) for p in preds]
    out = loss(ps, targets)
    out['conf_loss'].backward()
    _, mg, mi = T.yolox_loss_forward(preds, targets, STRIDES, 3)
    from oracle import yolox_loss_oracle as LO
    qs = [p.clone().requires_grad_(True) for p in preds]
    ref, _ = LO.losses(qs, targets, STRIDES, 3, (mg >= 0, mg.long(), mi))
    ref['conf_loss'].backward()
    for p, q in zip(ps, qs):
        assert _rel(p.grad, q.grad) < 1e-5


# ------------------------------------------------------------------------------------------------ model level: YOLOX(mode='train')
def _model(seed=3):
    from cvpytorch_b200 import synth, yolox_models as XM
    from oracle import yolox_train_oracle as XO
    m = XM.YOLOX(dictionary=[{f'c{i}': 1.0} for i in range(80)], model_cfg=dict(synth.YOLOX_CFG))
    sd = XO.synthetic_state([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=seed)
    m.load_state_dict(sd, strict=False)
    return m.cuda().train()


def _batch(B=2, H=128):
    g = torch.Generator().manual_seed(77)
    imgs = torch.randn(B, 3, H, H, generator=g).cuda()
    targets = []
    for b in range(B):
        n = 3 + b
        c = 20 + torch.rand(n, 2, generator=g) * (H - 40)
        wh = 16 + torch.rand(n, 2, generator=g) * 40
        targets.append({'labels': torch.randint(0, 80, (n,), generator=g).cuda(), 'boxes': torch.cat([c, wh], 1).cuda()})
    return imgs, targets


def test_model_training_forward_matches_loss_on_head_outputs(cuda):
    """YOLOX-s at 2 x 128²: the training forward's loss equals train.YOLOXLoss on the head outputs of the same forward bitwise, its
    head-output gradients are within 1e-5 of the oracle loss's (under the kernel's assignment), and its parameter gradients match those of
    the chained training modules fed that head-output gradient."""
    from cvpytorch_b200 import train as T
    from oracle import yolox_loss_oracle as LO
    m = _model()
    keys = list(m.state_dict())
    imgs, targets = _batch()
    seen = {}
    inner = m.loss.forward

    def record(preds, gt, imgs=None):
        seen['heads'], seen['gt'] = preds, gt
        return inner(preds, gt)
    m.loss.forward = record
    out = m(imgs, targets, 'train')
    heads, gt = seen['heads'], seen['gt']
    assert list(m.state_dict()) == keys
    again = T.YOLOXLoss(80)([h.detach() for h in heads], gt)
    for k in KEYS:
        assert torch.equal(again[k], out[k]), k
    _, mg, mi = T.yolox_loss_forward([h.detach() for h in heads], gt, STRIDES, 80)
    hs = [h.detach().clone().requires_grad_(True) for h in heads]
    ref, _ = LO.losses(hs, gt, STRIDES, 80, (mg >= 0, mg.long(), mi))
    ref['loss'].backward()
    kh = torch.autograd.grad(out['loss'], heads, retain_graph=True)
    for a, b in zip(kh, hs):
        assert _rel(a, b.grad) < 1e-5

    def param_grads(fn):
        m.zero_grad(set_to_none=True)
        fn()
        return {n: p.grad.clone() for n, p in m.named_parameters()}
    # The network takes the head-output gradient rounded to bf16, where a 1e-7 difference between two fp32 gradients can flip an element's
    # rounding, and its backward-weight and BatchNorm reductions add with atomics in no fixed order.  So the loss's backward is checked in
    # two steps: its head-output gradient against the oracle's at 1e-5 (above), then the parameter gradients of the loss path against the
    # network fed that same head-output gradient: within 1e-5, or within 10x the spread of repeated identical backward passes.
    want = param_grads(lambda: torch.autograd.backward(heads, kh, retain_graph=True))
    got = param_grads(lambda: out['loss'].backward(retain_graph=True))
    again = param_grads(lambda: out['loss'].backward())
    errs = {n: (_rel(got[n], want[n]), max(_rel(again[n], got[n]), _rel(again[n], want[n]))) for n in got}
    bad = {n: e for n, e in errs.items() if e[0] > max(1e-5, 10 * e[1])}
    print('parameter gradients within 1e-5:', sum(e[0] <= 1e-5 for e in errs.values()), 'of', len(errs),
          'worst', max(errs.items(), key=lambda kv: kv[1][0]))
    assert not bad, bad


def test_model_trainer_steps_hand_off_to_eval_and_graph_capture(cuda):
    """The reference trainer's step logic (autocast + GradScaler + clip + SGD) on a fixed batch: the loss falls, every parameter gets a
    finite gradient; afterwards eval() + 'val' equals a fresh eval YOLOX loaded with model.state_dict(), bitwise.  Then the whole training
    step is captured as one CUDA graph and replayed."""
    from cvpytorch_b200 import synth, yolox_models as XM
    m = _model()
    imgs, targets = _batch()
    params = list(m.parameters())
    opt = torch.optim.SGD(params, lr=0.01, momentum=0.9)
    scaler = torch.amp.GradScaler('cuda', enabled=True)
    hist = []
    for it in range(10):
        with torch.autocast('cuda', enabled=True):
            losses = m(imgs, targets, 'train')
        scaler.scale(losses['loss']).backward()
        scaler.unscale_(opt)
        torch.nn.utils.clip_grad_norm_(params, 10.0)
        if it == 0:
            for n, p in m.named_parameters():
                assert p.grad is not None and torch.isfinite(p.grad).all(), n
        scaler.step(opt)
        scaler.update()
        opt.zero_grad(set_to_none=True)
        hist.append(float(losses['loss'].detach()))
    del losses  # (drops the eager steps' autograd graph before the capture below)
    print('loss', [round(v, 4) for v in hist])
    assert all(np.isfinite(hist)) and np.mean(hist[-3:]) < hist[0], hist
    m.eval()
    with torch.no_grad():
        _, got = m(imgs, None, 'val')
    fresh = XM.YOLOX(dictionary=[{f'c{i}': 1.0} for i in range(80)], model_cfg=dict(synth.YOLOX_CFG))
    fresh.load_state_dict(m.state_dict(), strict=True)
    fresh.cuda().eval()
    with torch.no_grad():
        _, want = fresh(imgs, None, 'val')
    for a, b in zip(got, want):
        assert all(torch.equal(a[k], b[k]) for k in ('boxes', 'labels', 'scores'))

    m.train()
    gt = m.pack_targets(imgs, targets)
    opt = torch.optim.SGD(params, lr=0.01, momentum=0.9)

    def step():
        losses = m(imgs, gt, 'train')
        losses['loss'].backward()
        torch.nn.utils.clip_grad_norm_(params, 10.0)
        opt.step()
        opt.zero_grad(set_to_none=False)
        return losses['loss']
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_loss = step()
    vals = []
    for _ in range(10):
        graph.replay()
        vals.append(float(static_loss.detach()))
    print('graph loss', [round(v, 4) for v in vals])
    assert all(np.isfinite(vals)) and np.mean(vals[-3:]) < vals[0], vals
