"""Whole YOLOX CSPDarknet backbone TRAINING on the H100 kernels (cvpytorch_b200/train.py: Focus, SPPF, CSPDarknet; csrc/train_kernels.cu):
16- and 32-channel convolutions, the Focus space-to-depth kernel and the SPPF pooling kernels, then the whole backbone against the
reference fixture tests/golden/darknet_train.npz and against the oracle (oracle/darknet_train_oracle.py).

Narrow convolutions use the element-wise float64 bounds of tests/test_train_gpu.py's docstring.  A 16- or 32-channel K chunk is a 64-wide
chunk whose upper channels are zero, so the MMA chain is taps * kpad(cin) / 16 long (kpad = channels rounded up to 64); backward-weight
with cout = 16 or 32 is one 64-wide block, split over (2 * SMs) / (taps * cin blocks) CTAs.

Whole backbone: every output, every parameter gradient and every running statistic must have a max-normalised error against fp32 of at
most FACTOR * (the error of the same oracle step under torch.autocast(bfloat16) on this GPU) + FLOOR.  Measured on one H100 SXM (400 W power
limit), the median ratio kernels / autocast over all tensors is 0.83 (fixture), 0.78-0.94 (YOLOX-n, two runs) and 0.99-1.13 (YOLOX-s, two
runs); the largest ratio is 1.87, 1.50-2.06 and 1.88-2.33.  Runs differ because the backward-weight atomics add in no fixed order; a
wider version of the fixture (stages 2-4 at 64 channels) reached 2.34.  Where the largest ratios were located, they were BatchNorm gamma /
beta gradients of bottleneck convs (errors 0.5-0.8 against autocast's 0.2-0.4).  Those gradients are sums of dz * xhat over every pixel
that cancel to a few percent of their terms, so any bf16 step gets them only roughly; the kernels keep the gradient between layers in
bf16, where autocast runs the BatchNorm backward in fp32, hence the larger factor there.  FACTOR = 3 covers the measured 2.34 with margin;
FLOOR = 1e-2 covers tensors that autocast happens to get nearly exact.  The running
statistics carry the forward error of up to 35 layers (outputs 2-4 % off in both steps, running statistics up to 3.8 % off), so they use
the same rule rather than the C3 block's fixed 1e-2."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fp64ref as R  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
FACTOR, FLOOR = 3.0, 1e-2


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def _bf(t):
    return t.to(torch.bfloat16).float()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _kpad(c):
    return -(-c // 64) * 64


# (B, H, W, cin, cout, k, stride): 16 / 32-channel K chunks and N tiles in every pass; odd maps, B = 5, a 1x1 map under stride 2, and the
# stem / stage1 shapes of YOLOX-n and -s at a small image
@pytest.mark.parametrize('B,H,W,cin,cout,k,stride', [(2, 13, 9, 16, 32, 3, 1), (5, 7, 11, 32, 64, 3, 2), (3, 26, 18, 16, 32, 3, 2), (2, 9, 7, 64, 32, 1, 1),
                                                     (5, 11, 13, 32, 32, 1, 1), (2, 13, 9, 32, 32, 3, 1), (3, 9, 9, 32, 16, 1, 1), (5, 7, 9, 16, 16, 3, 1),
                                                     (2, 11, 7, 64, 16, 1, 1), (1, 1, 1, 16, 32, 3, 2), (4, 48, 64, 16, 32, 3, 1), (2, 32, 48, 32, 64, 3, 2),
                                                     (2, 12, 12, 128, 32, 3, 1), (2, 10, 10, 32, 128, 1, 1)])
def test_narrow_conv_forward_backward_data_backward_weight(cuda, B, H, W, cin, cout, k, stride):
    from cvpytorch_b200 import train as T
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + W + cin + cout + k + stride)
    x = _bf(torch.randn(B, cin, H, W, generator=g)).cuda().requires_grad_(True)
    w = _bf(torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).cuda().requires_grad_(True)
    y_ref = F.conv2d(x, w, None, stride, k // 2)
    dy = _bf(torch.randn(y_ref.shape, generator=g)).cuda()
    y_ref.backward(dy)
    xh = x.detach().permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    dyh = dy.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    wf, wb = T.pack_weights(w.detach())
    assert tuple(wf.shape) == (cout, k * k, _kpad(cin)) and tuple(wb.shape) == (cin, k * k, _kpad(cout))
    assert not bool(wf[..., cin:].any()) and not bool(wb[..., cout:].any())  # zero K padding
    yh = T.conv(xh, wf, cout, k, stride=stride)
    yp = _bf(torch.randn(B, H, W, cin, generator=g) * 2).cuda().to(torch.bfloat16)
    stat = torch.stack([torch.zeros(cin), torch.ones(cin), torch.rand(cin, generator=g) + 0.5, torch.randn(cin, generator=g) * 0.5]).cuda().contiguous()
    if stride == 1:
        dxh = T.conv(dyh, wb, cin, k)
        fused = T.conv(dyh, wb, cin, k, y_prev=yp, stat_prev=stat)
    else:
        dxh = T.conv_dgrad_s2(dyh, wb, cin, H, W)
        fused = T.conv_dgrad_s2(dyh, wb, cin, H, W, y_prev=yp, stat_prev=stat)
    dw = T.conv_wgrad(xh, dyh, k, stride)
    torch.cuda.synchronize()
    e = dict(y=_rel(yh.float().permute(0, 3, 1, 2), y_ref), dx=_rel(dxh.float().permute(0, 3, 1, 2), x.grad), dw=_rel(dw, w.grad))

    # element-wise vs float64 (tests/test_train_gpu.py docstring), chains over the zero-padded K
    xd, wd = x.detach(), w.detach()
    Ho, Wo = y_ref.shape[2:]

    def nhwc(t):
        return t.permute(0, 2, 3, 1)
    yr, ya = (nhwc(t) for t in R.conv_fwd(xd, wd, stride, k // 2))
    dxr, dxa = (nhwc(t) for t in R.conv_dgrad(dy, wd, xd.shape, stride, k // 2))
    dwr, dwa = R.conv_wgrad(xd, dy, wd.shape, stride, k // 2)
    g_f = R.mma_gamma(k * k * _kpad(cin))
    g_d = R.mma_gamma((k * k if stride == 1 else 4) * _kpad(cout))
    g_w = R.wgrad_gamma(B, Ho, Wo, cin, cout, k, _sms())
    r = {'y': R.check(yh, yr, R.BF16_REL * yr.abs() + (1 + R.BF16_REL) * g_f * ya, 'forward'),
         'dx': R.check(dxh, dxr, R.BF16_REL * dxr.abs() + (1 + R.BF16_REL) * g_d * dxa, 'backward-data'),
         'dw': R.check(dw, dwr, g_w * dwa, 'backward-weight')}
    z = yp.double() * stat[2].double() + stat[3].double()
    ref = dxr * R.silu_grad64(z)
    acc_err = g_d * dxa
    bound = (R.BF16_REL + 2 * R.U24) * ref.abs() + (1 + R.BF16_REL) * (1.1 * acc_err + (dxr.abs() + acc_err) * R.silu_grad_err(z))
    r["dx*silu'"] = R.check(fused, ref, bound, "backward-data with the SiLU' epilogue")
    print('max-normalised', e, 'worst error / bound', {k_: round(v, 3) for k_, v in r.items()})
    assert e['y'] < 6e-3 and e['dx'] < 6e-3 and e['dw'] < 2e-3, e


@pytest.mark.parametrize('B,H,W', [(2, 20, 12), (3, 34, 50), (1, 2, 2), (16, 640, 640)])
def test_focus_s2d_bit_exact(cuda, B, H, W):
    """cvb_train_focus_s2d == torch.cat of the reference's four slices (tl, bl, tr, br), rounded to bf16, NHWC, four zero channels."""
    from cvpytorch_b200 import train as T
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(H + W)).cuda()
    out = T.focus_s2d(x)
    ref = torch.cat((x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]), 1)
    ref = F.pad(ref.permute(0, 2, 3, 1), (0, 4)).to(torch.bfloat16)
    torch.cuda.synchronize()
    assert out.shape == ref.shape and torch.equal(out, ref)


def _tied_map(B, C, H, W, g):
    """bf16 values with many ties: half the channels on a coarse grid (a window holds the same maximum several times), half continuous,
    plus whole rows / columns set equal and a constant channel."""
    a = torch.randn(B, C, H, W, generator=g)
    a[:, : C // 2] = torch.randint(-3, 4, (B, C // 2, H, W), generator=g).float() * 0.5
    a[:, 1, :, W // 2:] = a[:, 1, :, :1]
    a[:, 2, H // 2:, :] = a[:, 2, :1, :]
    a[:, 3] = 1.25
    return a.to(torch.bfloat16)


@pytest.mark.parametrize('B,C,H,W', [(2, 64, 20, 20), (3, 32, 7, 5), (2, 16, 1, 1), (16, 256, 20, 20)])
def test_spp_pool_forward_backward(cuda, B, C, H, W):
    """Forward bit-exact against F.max_pool2d (5, 9, 13 in parallel); backward against float64 autograd of the same concatenation on the same
    values (same tie routing: the first maximum in row-major window order) within one bf16 rounding of the fp32 sum; bitwise reproducible."""
    from cvpytorch_b200 import train as T
    g = torch.Generator().manual_seed(B * C + H * W)
    a = _tied_map(B, C, H, W, g)
    ah = a.permute(0, 2, 3, 1).contiguous().cuda()
    cat, idx = T.spp_pool(ah)
    a64 = a.double().requires_grad_(True)
    ref = torch.cat([a64] + [F.max_pool2d(a64, k, 1, k // 2) for k in (5, 9, 13)], 1)
    assert torch.equal(cat.permute(0, 3, 1, 2).double().cpu(), ref.detach())
    gr = _bf(torch.randn(ref.shape, generator=g))
    ref.backward(gr.double())
    a_abs = a.double().requires_grad_(True)
    torch.cat([a_abs] + [F.max_pool2d(a_abs, k, 1, k // 2) for k in (5, 9, 13)], 1).backward(gr.double().abs())
    gh = gr.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16).cuda()
    da1 = T.spp_pool_backward(gh, idx)
    da2 = T.spp_pool_backward(gh, idx)
    torch.cuda.synchronize()
    assert torch.equal(da1, da2)
    terms = 1 + 25 + 81 + 169
    bound = R.BF16_REL * a64.grad.abs() + (1 + R.BF16_REL) * terms * R.U24 * a_abs.grad
    worst = R.check(da1.permute(0, 3, 1, 2), a64.grad, bound, 'SPPF pool backward')
    print('worst error / bound', round(worst, 3))


def _to_dev_state(sd, dev):
    return {k: torch.as_tensor(v).clone().to(dev) for k, v in sd.items()}


def _autocast_step(x, Gs, sd, **kw):
    """The oracle's training step on the GPU under torch.autocast(bfloat16): outputs, parameter gradients, running statistics."""
    from oracle import darknet_train_oracle as DO
    sdt = {}
    for k, v in sd.items():
        t = torch.as_tensor(v).clone().cuda()
        if t.dtype.is_floating_point and 'running_' not in k:
            t.requires_grad_(True)
        sdt[k] = t
    with torch.autocast('cuda', dtype=torch.bfloat16):
        outs = DO.csp_darknet(x.cuda(), sdt, **kw)
    sum((o.float() * G.cuda()).sum() for o, G in zip(outs, Gs)).backward()
    return [o.float() for o in outs], {k: v.grad for k, v in sdt.items() if v.requires_grad}, {k: v for k, v in sdt.items() if 'running_' in k}


def _kernel_step(sub, out_channels, x, Gs, sd):
    from cvpytorch_b200 import train as T
    m = T.CSPDarknet(sub, out_channels=out_channels)
    m.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
    m.cuda().train()
    outs = m(x.cuda())
    sum((o * G.cuda()).sum() for o, G in zip(outs, Gs)).backward()
    torch.cuda.synchronize()
    return m, outs


def _compare(m, outs, ref_outs, ref_grads, ref_stats, auto_outs, auto_grads, auto_stats):
    errs, auto = {}, {}
    for i, (o, r, a) in enumerate(zip(outs, ref_outs, auto_outs)):
        errs[f'y{i}'], auto[f'y{i}'] = _rel(o, r), _rel(a, r)
    for k, p in m.named_parameters():
        assert p.grad is not None, k
        errs['grad ' + k], auto['grad ' + k] = _rel(p.grad, ref_grads[k]), _rel(auto_grads[k], ref_grads[k])
    for k, v in m.state_dict().items():
        if 'running_' in k:
            errs['after ' + k], auto['after ' + k] = _rel(v, ref_stats[k]), _rel(auto_stats[k], ref_stats[k])
    ratio = {k: errs[k] / (auto[k] + 1e-12) for k in errs}
    worst = sorted(errs, key=lambda k: errs[k] - FACTOR * auto[k])[-5:]
    print('kernels vs fp32 (max-normalised): max', round(max(errs.values()), 4), 'autocast bf16 vs fp32: max', round(max(auto.values()), 4),
          'median kernel / autocast', round(float(np.median(list(ratio.values()))), 3))
    print('closest to the limit', {k: (round(errs[k], 4), round(auto[k], 4)) for k in worst}, 'largest ratio', round(max(ratio.values()), 3))
    bad = {k: (errs[k], auto[k]) for k in errs if errs[k] > FACTOR * auto[k] + FLOOR}
    assert not bad, bad


def test_csp_darknet_training_step_vs_reference_fixture(cuda):
    """Narrowed cspdark_n (widths 16, 32, 32, 32, 32) on 2x3x104x72 against the reference's CSPDarknet + torch.autograd in fp32."""
    g = np.load(os.path.join(GOLD, 'darknet_train.npz'))
    from oracle import darknet_train_oracle as DO
    keys, sd, x, Gs, oc = DO.fixture_inputs(g)
    m, outs = _kernel_step('cspdark_n', oc, x, Gs, sd)
    assert list(m.state_dict().keys()) == keys
    auto_outs, auto_grads, auto_stats = _autocast_step(x, Gs, sd, subtype='cspdark_n', out_channels=oc)
    ref_grads = {k[len('grad_'):]: torch.from_numpy(g[k]) for k in g.files if k.startswith('grad_')}
    ref_stats = {k[len('after_'):]: torch.from_numpy(g[k]) for k in g.files if k.startswith('after_')}
    _compare(m, outs, [torch.from_numpy(g[f'y{i}']) for i in range(3)], ref_grads, ref_stats, auto_outs, auto_grads, auto_stats)


@pytest.mark.parametrize('sub', ['cspdark_n', 'cspdark_s'])
def test_csp_darknet_training_step_vs_oracle(cuda, sub):
    """Stock YOLOX-n / YOLOX-s backbones (16 / 32-channel stems) on 2x3x128x96 against the oracle's fp32 step on this GPU (TF32 off)."""
    from cvpytorch_b200 import train as T
    from oracle import darknet_train_oracle as DO
    shapes = [(k, tuple(v.shape)) for k, v in T.CSPDarknet(sub).state_dict().items()]
    sd = DO.synthetic_state(shapes, seed=len(sub) + (1 if sub.endswith('s') else 0))
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 3, 128, 96, generator=g)
    ch = DO.widths(sub)
    Gs = [torch.randn(2, ch[i], 128 // 2 ** (i + 1), 96 // 2 ** (i + 1), generator=g) for i in (2, 3, 4)]
    ref_outs, ref_grads, ref_stats = DO.train_step(x.cuda(), [G.cuda() for G in Gs], _to_dev_state(sd, 'cuda'), subtype=sub)
    m, outs = _kernel_step(sub, [64, 128, 256, 512, 1024], x, Gs, sd)
    auto_outs, auto_grads, auto_stats = _autocast_step(x, Gs, sd, subtype=sub)
    _compare(m, outs, ref_outs, ref_grads, ref_stats, auto_outs, auto_grads, auto_stats)


def test_csp_darknet_hand_off_to_inference_module(cuda):
    """Train one SGD step on the kernels, load the state_dict into the inference yolox_models.CSPDarknet (strict=True) and evaluate: it
    matches oracle/yolox_oracle.backbone on the updated parameters within that path's tolerance (1e-3 of max|ref|).  A first training-mode
    forward with momentum None (cumulative average: running statistics = that batch's statistics) calibrates the seeded state; with the
    initial (0, 1) running statistics the eval-mode activations of the seeded network grow without bound over 35 layers.  The step clips the
    gradient norm to 10 like the reference trainer; unclipped, the seeded network's gradient moves the weights by hundreds."""
    from cvpytorch_b200 import train as T, yolox_models as Y
    from oracle import darknet_train_oracle as DO, yolox_oracle as YO
    m = T.CSPDarknet('cspdark_s')
    sd = DO.synthetic_state([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed=5)
    m.load_state_dict(sd)
    m.cuda().train()
    g = torch.Generator().manual_seed(12)
    x = torch.randn(2, 3, 128, 128, generator=g).cuda()
    bns = [mod for mod in m.modules() if isinstance(mod, torch.nn.BatchNorm2d)]
    for bn in bns:
        bn.momentum = None
    with torch.no_grad():
        m(x)
    for bn in bns:
        bn.momentum = 0.03
    outs = m(x)
    sum((o * torch.randn(o.shape, generator=g).cuda()).sum() for o in outs).backward()
    torch.nn.utils.clip_grad_norm_(m.parameters(), 10.0)  # (as the reference trainer's cfg.GRAD_CLIP: the seeded step's gradient norm is ~4e4)
    opt = torch.optim.SGD(m.parameters(), lr=0.01, momentum=0.9)
    opt.step()
    trained = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    inf = Y.CSPDarknet('cspdark_s')
    inf.load_state_dict(trained, strict=True)
    inf.cuda().eval()
    with torch.no_grad():
        got = inf(x)
    ref = YO.backbone(x.cpu().double(), {'backbone.' + k: v.double() for k, v in trained.items()})
    errs = [_rel(a, b) for a, b in zip(got, ref)]
    print('inference vs oracle after one training step', errs)
    assert max(errs) < 1e-3, errs


def test_csp_darknet_through_the_reference_trainer_train_step(cuda):
    """The backbone drop-in with a small torch head inside a copy of the reference's training-step logic (trainer.py:177-207: autocast,
    GradScaler, clip_grad, step, zero_grad): the loss falls and every backbone parameter gets a finite, non-zero gradient."""
    from cvpytorch_b200 import train as T
    torch.manual_seed(4)
    backbone = T.CSPDarknet('cspdark_n').cuda().train()
    heads = torch.nn.ModuleList([torch.nn.Conv2d(c, 8, 1) for c in backbone.out_channels]).cuda()
    params = list(backbone.parameters()) + list(heads.parameters())
    optimizer = torch.optim.SGD(params, lr=0.02, momentum=0.9)
    scaler = torch.amp.GradScaler('cuda', enabled=True)
    imgs = torch.randn(4, 3, 128, 128, device='cuda')
    targets = [torch.randn(4, 8, 128 // s, 128 // s, device='cuda') * 0.1 for s in (8, 16, 32)]
    hist = []
    for it in range(10):
        with torch.autocast('cuda', enabled=True):
            outs = [h(f) for h, f in zip(heads, backbone(imgs))]
            losses = {'loss': sum((o.float() - t).pow(2).mean() for o, t in zip(outs, targets))}
        scaler.scale(losses['loss']).backward()
        scaler.unscale_(optimizer)
        torch.nn.utils.clip_grad_norm_(params, 10.0)
        if it == 0:
            for k, p in backbone.named_parameters():
                assert p.grad is not None and torch.isfinite(p.grad).all() and float(p.grad.abs().max()) > 0, k
        scaler.step(optimizer)
        scaler.update()
        optimizer.zero_grad(set_to_none=True)
        hist.append(float(losses['loss']))
    print('loss', [round(v, 4) for v in hist])
    assert all(np.isfinite(hist)) and hist[-1] < 0.8 * hist[0], hist
