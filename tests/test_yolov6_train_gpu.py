"""YOLOv6 training on the H100: the BatchNorm + ReLU, RepVGG and transposed-conv passes (csrc/train_kernels.cu), the training modules of
yolov6_train.py and the model-level training forward (yolov6_models.YOLOv6, mode='train').

The element-wise passes are checked against float64 autograd on the same bf16 inputs; the network and the model against
oracle/yolov6_train_oracle.py (fp32 torch.autograd) with the criterion of the YOLOv5 / YOLOX network tests: every output, gradient and
running statistic within 3x the error of the same oracle step under bf16 autocast on this GPU, plus 1e-2."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_yolov6_host import DICT, use_model  # noqa: E402

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def _bn64(y, gamma, beta):
    """Training BatchNorm of NHWC float64 y over every pixel (biased variance, eps 1e-3)."""
    m = y.mean((0, 1, 2))
    v = y.var((0, 1, 2), unbiased=False)
    return (y - m) / torch.sqrt(v + 1e-3) * gamma + beta


def _stats(y, gamma, beta):
    from cvpytorch_b200 import train as T
    rm, rv = torch.zeros_like(gamma), torch.ones_like(gamma)
    return T.bn_stats(y, gamma, beta, rm, rv, 1e-3, 0.03)


@pytest.mark.parametrize('C', [16, 96, 128])
def test_bn_relu_passes_vs_float64(cuda, C):
    """cvb_train_bn_relu_fwd / _bwd: out, dy, dgamma and dbeta against float64 autograd of relu(bn(y)) on the same bf16 y and g."""
    from cvpytorch_b200 import _lib
    from cvpytorch_b200._lib import _p, _stream
    g = torch.Generator(device='cuda').manual_seed(C)
    y = (torch.randn((3, 9, 13, C), generator=g, device='cuda') * 2 + 0.5).bfloat16()
    gam, bet = torch.rand(C, generator=g, device='cuda') + 0.5, torch.randn(C, generator=g, device='cuda') * 0.3
    gout = torch.randn((3, 9, 13, C), generator=g, device='cuda').bfloat16()
    stat, g32 = _stats(y, gam, bet)
    npix = y.numel() // C
    outs = []
    for _ in range(2):
        out = torch.empty_like(y)
        _lib.check(_lib.lib().cvb_train_bn_relu_fwd(_p(y), npix, C, _p(stat), _p(out), _stream()))
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    sums, dy = torch.empty((2, C), device='cuda'), torch.empty_like(y)
    _lib.check(_lib.lib().cvb_train_bn_relu_bwd(_p(gout), _p(y), npix, C, _p(stat), _p(g32), _p(sums), _p(dy), _stream()))
    y64, gm64, bt64 = (t.double().requires_grad_() for t in (y, gam, bet))
    z64 = _bn64(y64, gm64, bt64)
    z64.backward(gout.double() * (outs[0] > 0))  # (the ReLU mask of the kernel's own output: a z within rounding of 0 may go either way)
    assert _rel(outs[0], F.relu(z64)) < 1e-2
    assert _rel(dy, y64.grad) < 2e-2
    assert _rel(sums[1], gm64.grad) < 1e-3 and _rel(sums[0], bt64.grad) < 1e-3


@pytest.mark.parametrize('ident', [False, True])
@pytest.mark.parametrize('C', [32, 64, 192])
def test_repvgg_passes_vs_float64(cuda, C, ident):
    """cvb_train_repvgg_fwd / _bwd: relu(bn3(y3) + bn1(y1) [+ bnid(x)]) and every branch's dy, dgamma and dbeta against float64 autograd on
    the same bf16 operands, with and without the identity branch; the forward identical run to run."""
    from cvpytorch_b200 import _lib
    from cvpytorch_b200._lib import _p, _stream
    g = torch.Generator(device='cuda').manual_seed(C + ident)
    shp = (2, 11, 17, C)
    ys = [(torch.randn(shp, generator=g, device='cuda') * (1 + i) + i).bfloat16() for i in range(3)]
    gb = [(torch.rand(C, generator=g, device='cuda') + 0.5, torch.randn(C, generator=g, device='cuda') * 0.3) for _ in range(3)]
    gout = torch.randn(shp, generator=g, device='cuda').bfloat16()
    nb = 3 if ident else 2
    st = [_stats(ys[i], *gb[i]) for i in range(nb)]
    npix = ys[0].numel() // C
    opt = lambda i: _p(ys[2]) if i else None  # noqa: E731
    outs = []
    for _ in range(2):
        a = torch.empty_like(ys[0])
        _lib.check(_lib.lib().cvb_train_repvgg_fwd(_p(ys[0]), _p(ys[1]), opt(ident), npix, C, _p(st[0][0]), _p(st[1][0]), _p(st[2][0]) if ident else None,
                                                   _p(a), _stream()))
        outs.append(a)
    assert torch.equal(outs[0], outs[1])
    a = outs[0]
    sums = torch.empty((4, C), device='cuda')
    d = [torch.empty_like(ys[0]) for _ in range(3)]
    _lib.check(_lib.lib().cvb_train_repvgg_bwd(_p(gout), _p(a), _p(ys[0]), _p(ys[1]), opt(ident), npix, C, _p(st[0][0]), _p(st[1][0]),
                                               _p(st[2][0]) if ident else None, _p(st[0][1]), _p(st[1][1]), _p(st[2][1]) if ident else None, _p(sums),
                                               _p(d[0]), _p(d[1]), _p(d[2]) if ident else None, _stream()))
    y64 = [t.double().requires_grad_() for t in ys[:nb]]
    p64 = [(gm.double().requires_grad_(), bt.double().requires_grad_()) for gm, bt in gb[:nb]]
    z64 = sum(_bn64(y64[i], *p64[i]) for i in range(nb))
    z64.backward(gout.double() * (a > 0))  # (the mask of the kernel's output, which the backward reads)
    assert _rel(a, F.relu(z64)) < 1e-2
    for i in range(nb):
        assert _rel(d[i], y64[i].grad) < 2e-2, i
        assert _rel(sums[1 + i], p64[i][0].grad) < 1e-3, i
        assert _rel(sums[0], p64[i][1].grad) < 1e-3, i
    if not ident:
        assert torch.equal(sums[3], torch.zeros_like(sums[3]))


@pytest.mark.parametrize('c,h,w', [(32, 5, 7), (64, 20, 20), (128, 3, 2)])
def test_conv_transpose_vs_float64(cuda, c, h, w):
    """BiFusion's ConvTranspose2d on the kernels (1x1 GEMM + cvb_train_convt_scatter; cvb_train_convt_gather + the 1x1 backward convs):
    output, input, weight and bias gradients against float64 F.conv_transpose2d autograd on the same bf16 operands; dbias bitwise
    reproducible."""
    from cvpytorch_b200 import yolov6_train as Y
    g = torch.Generator(device='cuda').manual_seed(c + h)
    x = torch.randn((3, h, w, c), generator=g, device='cuda').bfloat16().requires_grad_()
    wt = (torch.randn((c, c, 2, 2), generator=g, device='cuda') / c ** 0.5).bfloat16().float().requires_grad_()
    b = torch.randn(c, generator=g, device='cuda').requires_grad_()
    gout = torch.randn((3, 2 * h, 2 * w, c), generator=g, device='cuda').bfloat16()
    out = Y._ConvT2.apply(x, Y._convt_weight(wt), b)
    out.backward(gout)
    x64, w64, b64 = (t.detach().double().requires_grad_() for t in (x, wt, b))
    o64 = F.conv_transpose2d(x64.permute(0, 3, 1, 2), w64, b64, stride=2).permute(0, 2, 3, 1)
    o64.backward(gout.double())
    assert _rel(out, o64) < 1e-2
    assert _rel(x.grad, x64.grad) < 1e-2 and _rel(wt.grad, w64.grad) < 1e-2 and _rel(b.grad, b64.grad) < 1e-5
    du, db = Y.convt_gather(gout)
    assert torch.equal(du.view(3, h, w, 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(gout.shape), gout)
    assert torch.equal(Y.convt_gather(gout)[1], db)


def _modules(stype, nc=3):
    from cvpytorch_b200 import yolov6_models as M
    m = M.YOLOv6([{f'c{i}': 1.0} for i in range(nc)], _cfg(stype, nc)).cuda().train()
    return m


def _cfg(stype, nc):
    cfg = use_model(stype)
    cfg['HEAD'] = dict(cfg['HEAD'], num_classes=nc)
    cfg['LOSS'] = dict(cfg['LOSS'], num_classes=nc)
    if 'num_classes' in cfg['DETECT']:
        cfg['DETECT'] = dict(cfg['DETECT'], num_classes=nc)
    return cfg


def _randomise(m, seed):
    """Non-trivial weights: the reference zero-initialises the prediction convs, which would zero every gradient below them."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if k.endswith('weight') and p.dim() == 4:
                p.copy_(torch.randn(p.shape, generator=g) * (2.0 / (p.shape[1] * p.shape[2] * p.shape[3])) ** 0.5)
            elif 'bn' in k or 'rbr_identity' in k:
                p.copy_((torch.rand(p.shape, generator=g) + 0.5) if k.endswith('weight') else torch.randn(p.shape, generator=g) * 0.1)
            elif k.endswith('bias'):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)


@pytest.mark.parametrize('stype', ['n', 's'])
def test_network_step_vs_oracle(cuda, stype):
    """The training modules' backbone -> neck -> head step at 2x3x64x96 with 3 classes and loss = sum(out * G) over pred_scores and
    pred_distri: outputs, every parameter gradient (the class branch included) and every running statistic within 3x the error of the
    fp32 oracle step under bf16 autocast, plus 1e-2.  YOLOv6-n covers the padded 96-channel bifusion1.cv3 and the 16 / 32-wide blocks."""
    from oracle import yolov6_train_oracle as O
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    m = _modules(stype)
    _randomise(m, 5)
    g = torch.Generator().manual_seed(6)
    x = torch.rand((2, 3, 64, 96), generator=g).cuda()
    A = 8 * 12 + 4 * 6 + 2 * 3
    G = [torch.randn((2, A, 3), generator=g).cuda(), torch.randn((2, A, 4), generator=g).cuda()]
    state = {k: v.detach().clone() for k, v in m.state_dict().items() if k.startswith(('backbone.', 'neck.', 'head.'))}

    def oracle(autocast):
        sd = {k: v.clone().requires_grad_(v.dtype.is_floating_point and 'running_' not in k and 'proj' not in k) for k, v in state.items()}
        with torch.autocast('cuda', dtype=torch.bfloat16, enabled=autocast):
            _, s, d = O.network(x, sd)
        ((s.float() * G[0]).sum() + (d.float() * G[1]).sum()).backward()
        r = {'scores': s.detach().float(), 'distri': d.detach().float()}
        r.update({f'grad_{k}': v.grad for k, v in sd.items() if v.grad is not None})
        r.update({f'after_{k}': v for k, v in sd.items() if 'running_' in k})
        return r
    ref, auto = oracle(False), oracle(True)
    bb, nk, hd = m._training_modules()
    _, s, d = hd.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(x)))
    ((s * G[0]).sum() + (d * G[1]).sum()).backward()
    got = {'scores': s.detach(), 'distri': d.detach()}
    got.update({f'grad_{k}': p.grad for k, p in m.named_parameters() if p.grad is not None})
    got.update({f'after_{k}': v for k, v in m.state_dict().items() if 'running_' in k and k.startswith(('backbone.', 'neck.', 'head.'))})
    assert set(got) == set(ref) == set(auto)
    errs = {k: _rel(got[k], ref[k]) for k in ref}
    au = {k: _rel(auto[k].float(), ref[k]) for k in ref}
    print('worst error / (3 x autocast error + 1e-2):', round(max(errs[k] / (3 * au[k] + 1e-2) for k in ref), 3))
    bad = {k: (errs[k], au[k]) for k in ref if errs[k] > 3 * au[k] + 1e-2}
    assert not bad, bad


def test_network_step_vs_reference_fixture(cuda):
    """tests/golden/yolov6_train.npz (the reference's backbone, neck and head in training mode, fp32, a narrowed YOLOv6-n with widths 16 /
    32, 3 classes, 2x3x64x96): the training modules' outputs, every parameter gradient and every running statistic within 3x the error of
    the same oracle step under bf16 autocast on this GPU, plus 1e-2 (each on oracle.fixture_scale)."""
    from cvpytorch_b200 import yolov6_train as Y
    from oracle import yolov6_train_oracle as O
    torch.backends.cudnn.allow_tf32 = False
    f = np.load(os.path.join(ROOT, 'tests', 'golden', 'yolov6_train.npz'))
    keys, sd, x, Gs = O.net_fixture_inputs(f)
    ref = {k: torch.from_numpy(f[k]) for k in f.files if k in ('scores', 'distri') or k.startswith(('grad_', 'after_'))}
    with torch.autocast('cuda', dtype=torch.bfloat16):
        auto = O.net_train_step(x.cuda(), [G.cuda() for G in Gs], {k: v.cuda() for k, v in sd.items()})
    mods = {'backbone.': Y.YOLOv6EfficientRep(**O.NET['backbone']), 'neck.': Y.YOLOv6RepBiPAN(**O.NET['neck']),
            'head.': Y.YOLOv6Effidehead(**O.NET['head'])}
    for pre, m in mods.items():
        m.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}, strict=True)
        m.cuda().train()
    bb, nk, hd = mods.values()
    _, s, d = hd.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(x.cuda())))
    ((s * Gs[0].cuda()).sum() + (d * Gs[1].cuda()).sum()).backward()
    got = {'scores': s.detach(), 'distri': d.detach()}
    for pre, m in mods.items():
        got.update({f'grad_{pre}{k}': p.grad for k, p in m.named_parameters() if p.requires_grad})
        got.update({f'after_{pre}{k}': v for k, v in m.state_dict().items() if 'running_' in k})
    assert set(got) == set(ref) == set(auto)
    err = lambda a, k: float((a.detach().double().cpu() - ref[k].double()).abs().max()) / O.fixture_scale(k, ref)  # noqa: E731
    errs = {k: err(got[k], k) for k in ref}
    au = {k: err(auto[k].float(), k) for k in ref}
    print('worst error / (3 x autocast error + 1e-2):', round(max(errs[k] / (3 * au[k] + 1e-2) for k in ref), 3))
    bad = {k: (errs[k], au[k]) for k in ref if errs[k] > 3 * au[k] + 1e-2}
    assert not bad, bad


def _batch(B=4, size=320, nc=80, seed=21):
    """Images and per-image targets with (cx, cy, w, h) normalised by the loss's ori_img_size 640 (every box inside a size x size image)."""
    g = torch.Generator().manual_seed(seed)
    imgs = torch.rand((B, 3, size, size), generator=g).cuda()
    targets = []
    for i in range(B):
        n = 3 + i
        f = size / 640
        boxes = torch.cat([torch.rand((n, 2), generator=g) * 0.6 + 0.2, torch.rand((n, 2), generator=g) * 0.3 + 0.05], 1) * f
        targets.append({'labels': torch.randint(0, nc, (n,), generator=g), 'boxes': boxes})
    return imgs, targets


def test_model_loss_and_class_branch(cuda):
    """mode='train' returns {'iou', 'dfl', 'class', 'loss'}: bitwise yolov6_train.YOLOv6Loss (ATSS) on the head outputs it produced, loss =
    their sum; cls_convs / cls_preds keep .grad None while their BatchNorm running statistics move."""
    from cvpytorch_b200 import yolov6_train as Y
    m = _modules('s', 80)
    _randomise(m, 7)
    imgs, targets = _batch()
    gt = m.pack_targets(imgs, targets)
    seen = {}
    loss_fn = m._train_loss
    fwd = loss_fn.forward
    loss_fn.forward = lambda o, t, *a: (seen.update(o=(o[0], o[1].detach().clone(), o[2].detach().clone())), fwd(o, t, *a))[1]
    before = {k: v.clone() for k, v in m.state_dict().items() if 'running_mean' in k and 'cls_convs' in k}
    losses = m(imgs, targets, 'train')
    loss_fn.forward = fwd
    assert list(losses) == ['iou', 'dfl', 'class', 'loss']
    want = Y.YOLOv6Loss(80)(seen['o'], gt)
    for k in ('iou', 'dfl', 'class'):
        assert losses[k].dtype == torch.float64 and torch.equal(losses[k].detach(), want[k])
    assert torch.equal(losses['loss'].detach(), want['iou'] + want['dfl'] + want['class'])
    assert float(losses['loss'].detach()) > 0
    losses['loss'].backward()
    for k, p in m.named_parameters():
        if k.startswith(('head.cls_convs.', 'head.cls_preds.')):
            assert p.grad is None, k
        elif p.requires_grad:
            assert p.grad is not None and torch.isfinite(p.grad).all(), k
    after = m.state_dict()
    assert all(not torch.equal(before[k], after[k]) for k in before)


def test_model_gradients_follow_the_oracle(cuda):
    """One training step of YOLOv6-s against oracle/yolov6_train_oracle.network in fp32, with the same H100 YOLOv6Loss on its outputs: the
    loss (relative) and every parameter gradient (relative norm, as test_yolov5_train_gpu's model test) within 3x the error of the same
    oracle step under bf16 autocast, plus 1e-2."""
    from cvpytorch_b200 import yolov6_train as Y
    from oracle import yolov6_train_oracle as O
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    m = _modules('s', 80)
    _randomise(m, 9)
    imgs, targets = _batch()
    gt = m.pack_targets(imgs, targets)
    state = {k: v.detach().clone() for k, v in m.state_dict().items() if k.startswith(('backbone.', 'neck.', 'head.'))}

    def oracle(autocast):
        sd = {k: v.clone().requires_grad_(v.dtype.is_floating_point and 'running_' not in k and 'proj' not in k) for k, v in state.items()}
        with torch.autocast('cuda', dtype=torch.bfloat16, enabled=autocast):
            feats, s, d = O.network(imgs, sd)
        losses = Y.YOLOv6Loss(80)((feats, s.float(), d.float()), gt)
        loss = losses['iou'] + losses['dfl'] + losses['class']
        loss.backward()
        return loss, {k: v.grad for k, v in sd.items() if v.grad is not None}
    oloss, og = oracle(False)
    aloss, ag = oracle(True)
    losses = m(imgs, gt, 'train')
    losses['loss'].backward()
    lo, la, lk = (float(v.detach()) for v in (oloss, aloss, losses['loss']))
    print('loss: oracle', round(lo, 4), 'autocast', round(la, 4), 'kernels', round(lk, 4))
    assert abs(lk - lo) <= 3 * abs(la - lo) + 1e-2 * abs(lo)
    got = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    assert set(got) == set(og)
    bad, worst = [], 0.0
    for k, g in got.items():
        ref = og[k].double()
        e = float((g.double() - ref).norm() / (ref.norm() + 1e-30))
        e_ac = float((ag[k].double() - ref).norm() / (ref.norm() + 1e-30))
        worst = max(worst, e / (3 * e_ac + 1e-2))
        if e > 3 * e_ac + 1e-2:
            bad.append((k, round(e, 4), round(e_ac, 4)))
    print('worst error / (3 x autocast error + 1e-2):', round(worst, 3))
    assert not bad, bad


def test_model_trainer_steps_hand_off_to_eval_and_graph_capture(cuda):
    """The reference trainer's step logic (autocast + GradScaler + clip + SGD) runs 10 steps with finite losses; eval() then serves the
    trained weights exactly as a fresh eval YOLOv6 loaded with model.state_dict(); then the whole step captures as one CUDA graph and
    replays with the loss moving."""
    from cvpytorch_b200 import yolov6_models as M
    m = M.YOLOv6(DICT, use_model('s')).cuda().train()
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
        scaler.step(opt)
        scaler.update()
        opt.zero_grad(set_to_none=True)
        hist.append(float(losses['loss'].detach()))
    del losses
    print('loss', [round(v, 4) for v in hist])
    assert all(np.isfinite(hist)), hist
    m.eval()
    with torch.no_grad():
        got, _, cnt = m.predict(imgs)
        got, cnt = got.clone(), cnt.clone()
    fresh = M.YOLOv6(DICT, use_model('s'))
    fresh.load_state_dict(m.state_dict(), strict=True)
    fresh.cuda().eval()
    with torch.no_grad():
        want, _, wcnt = fresh.predict(imgs)
    assert torch.equal(cnt, wcnt) and torch.equal(got, want)

    m.train()
    gt = m.pack_targets(imgs, targets)
    opt = torch.optim.SGD(params, lr=0.01, momentum=0.9)

    def step():
        losses = m(imgs, gt, 'train')
        losses['loss'].backward()
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
    for _ in range(5):
        graph.replay()
        vals.append(float(static_loss.detach()))
    print('graph loss', [round(v, 4) for v in vals])
    assert all(np.isfinite(vals)) and len(set(vals)) > 1, vals
