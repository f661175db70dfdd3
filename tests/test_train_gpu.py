"""SURVEY.md 8(f) rank 3 -- the YOLOX C3 block's TRAINING step (forward + backward) on the H100 kernels (cvpytorch_b200/train.py,
csrc/train_kernels.cu) against (1) torch on the same GPU, kernel by kernel, on bf16-representable inputs, and (2) the committed reference
fixture tests/golden/c3_train.npz = the reference CSPLayer + torch.autograd in fp32 on CPU (tools/make_golden_train.py).

Tolerances (bf16 step: 8 significant bits, |rounding| <= 2^-8 relative per stored activation / gradient; fp32 accumulation everywhere):
  single kernels, bf16 outputs        max|a-b| / max|b| <= 6e-3        fp32 outputs (wgrad, BN statistics)  <= 2e-3
  whole block vs the fp32 reference   forward <= 3e-2, d/dx and every parameter gradient <= 6e-2  (5-9 bf16 layers deep each way)

Element-wise bounds against float64 (tests/fp64ref.py: |out - ref| <= rel |ref| + gamma * absref, absref = the same operation on |inputs|):
  forward          gamma = (taps * cin / 16 + 16) * 2^-23       rel = 2^-8
  backward-data    gamma = (taps * cout / 16 + 16) * 2^-23      rel = 2^-8   (stride 2: at most 4 taps per parity class)
    with SiLU'     + |dx| * silu_grad_err(z): __expf is within 2 + floor(1.173 |z|) ulps, so a few 1e-6 (1 + |z|) absolute
  backward-weight  gamma = (8 * per + 16 + splits) * 2^-23      rel = 0      (fp32 output; `per` 128-pixel tiles of 8 MMAs each per CTA,
                                                                             then `splits` fp32 atomics, fp64ref.wgrad_split)
The cases with a CTA owning more than one pixel tile (per > 1, on 132 SMs): 16x48x48 1x1 64->64 (288 tiles of 16x1x8 over 264 splits,
per = 2) and 16x40x40 3x3 64->64 (200 tiles of 8x1x16 over 2 * 132 / 9 = 29 splits, per = 7, the last split has 4); every other case has
per = 1.

BatchNorm: the statistics are fp32 sums of y - y[0] over a tree of additions (pixels of one thread, the CTA's pixel lanes, one atomic per CTA;
the longest chain, fp64ref.red_chain, is 362..724 additions for 102 401 pixels, 19..259 for 129), finalised in double.  A chain of L fp32
additions is off by at most L * 2^-24 * sum|terms|; that bound is propagated to mean, variance, rstd, scale, shift and the running statistics
in test_bn_statistics_silu_forward_backward_vs_float64.  At 102 401 pixels it allows 1e-5..2e-5 relative of rstd per
(1 + ((y[0] - mean) / std)^2), at 129 pixels 1e-6..8e-6; the one-pass E[y^2] - mean^2 instead loses (mean / std)^2 times the same error."""
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


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def _bf(t):
    return t.to(torch.bfloat16).float()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _stat_prev(C, g):
    """BN statistics [4][C] of a producing layer with random per-channel scale and shift (rows 2, 3: all the SiLU' epilogue reads), so that a
    scale / shift read from the wrong output-channel tile changes the result."""
    return torch.stack([torch.zeros(C), torch.ones(C), torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.5]).cuda().contiguous()


def _conv_vs_float64(x, w, dy, k, stride, y, dx, dw, fused, y_prev, stat_prev):
    """Element-wise bounds of the module docstring.  x, w, dy: NCHW bf16-representable inputs; y, dx, fused (= dx * silu'(y_prev * s + t)):
    NHWC bf16 kernel outputs; dw: fp32 [cout, cin, k, k].  -> worst |error| / bound per output."""
    B, cin = x.shape[:2]
    cout, Ho, Wo = dy.shape[1:]
    pad = k // 2

    def nhwc(t):
        return t.permute(0, 2, 3, 1)

    yr, ya = (nhwc(t) for t in R.conv_fwd(x, w, stride, pad))
    dxr, dxa = (nhwc(t) for t in R.conv_dgrad(dy, w, x.shape, stride, pad))
    dwr, dwa = R.conv_wgrad(x, dy, w.shape, stride, pad)
    g_f = R.mma_gamma(k * k * cin)
    g_d = R.mma_gamma((k * k if stride == 1 else 4) * cout)
    g_w = R.wgrad_gamma(B, Ho, Wo, cin, cout, k, _sms())
    r = {'y': R.check(y, yr, R.BF16_REL * yr.abs() + (1 + R.BF16_REL) * g_f * ya, 'forward'),
         'dx': R.check(dx, dxr, R.BF16_REL * dxr.abs() + (1 + R.BF16_REL) * g_d * dxa, 'backward-data'),
         'dw': R.check(dw, dwr, g_w * dwa, 'backward-weight')}
    z = y_prev.double() * stat_prev[2].double() + stat_prev[3].double()
    ref = dxr * R.silu_grad64(z)
    acc_err = g_d * dxa  # |silu'| <= 1.1
    bound = (R.BF16_REL + 2 * R.U24) * ref.abs() + (1 + R.BF16_REL) * (1.1 * acc_err + (dxr.abs() + acc_err) * R.silu_grad_err(z))
    r["dx*silu'"] = R.check(fused, ref, bound, "backward-data with the SiLU' epilogue")
    return r


# cin 192 / 320: the last backward-weight cin block has one 64-channel panel; cout 192 / 320 / 384: 64-wide forward tiles (3 and 5 of them)
# and the backward-weight blocks of 64 / 128 channels; the backward-data SiLU' epilogue runs on cin = 192 (three 64-wide tiles), 256 (two
# 128-wide tiles) and 320; 1024 channels (dark5 of YOLOX-l: four cout blocks, eight cin blocks); per > 1 (module docstring)
@pytest.mark.parametrize('B,H,W,cin,cout,k', [(2, 16, 16, 64, 64, 1), (3, 20, 20, 128, 64, 3), (2, 13, 9, 64, 128, 3), (1, 40, 40, 128, 128, 1), (5, 8, 8, 256, 64, 1), (2, 10, 10, 256, 512, 1), (1, 12, 12, 512, 256, 3),  # (incl. the 256 / 512-channel layers of dark4 / dark5)
                                              (2, 10, 10, 192, 64, 1), (2, 9, 11, 192, 128, 3), (1, 12, 12, 320, 64, 1), (2, 7, 9, 320, 192, 3),
                                              (2, 10, 10, 64, 192, 3), (3, 12, 9, 128, 320, 1), (1, 10, 10, 192, 384, 3), (2, 6, 7, 384, 192, 1), (2, 8, 8, 256, 256, 3),
                                              (2, 6, 6, 1024, 1024, 1), (1, 5, 7, 1024, 1024, 3),
                                              (16, 48, 48, 64, 64, 1), (16, 40, 40, 64, 64, 3)])
def test_conv_forward_backward_data_backward_weight(cuda, B, H, W, cin, cout, k):
    from cvpytorch_b200 import train as T
    g = torch.Generator().manual_seed(B * 100 + H + cin + k)
    x = _bf(torch.randn(B, cin, H, W, generator=g)).cuda().requires_grad_(True)
    w = _bf(torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).cuda().requires_grad_(True)
    dy = _bf(torch.randn(B, cout, H, W, generator=g)).cuda()
    y_ref = F.conv2d(x, w, None, 1, k // 2)
    y_ref.backward(dy)
    xh = x.detach().permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    dyh = dy.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    wf, wb = T.pack_weights(w.detach())
    yh = T.conv(xh, wf, cout, k)
    dxh = T.conv(dyh, wb, cin, k)
    dw = T.conv_wgrad(xh, dyh, k)
    yp = _bf(torch.randn(B, H, W, cin, generator=g) * 2).cuda().to(torch.bfloat16)
    stat = _stat_prev(cin, g)
    fused = T.conv(dyh, wb, cin, k, y_prev=yp, stat_prev=stat)
    torch.cuda.synchronize()
    y, dx = yh.float().permute(0, 3, 1, 2), dxh.float().permute(0, 3, 1, 2)
    e = dict(y=_rel(y, y_ref), dx=_rel(dx, x.grad), dw=_rel(dw, w.grad))
    r = _conv_vs_float64(x.detach(), w.detach(), dy, k, 1, yh, dxh, dw, fused, yp, stat)
    print('max-normalised', e, 'worst error / bound', {k_: round(v, 3) for k_, v in r.items()}, 'per', R.wgrad_split(B, H, W, cin, cout, k, _sms())[2])
    assert e['y'] < 6e-3 and e['dx'] < 6e-3 and e['dw'] < 2e-3, e


def test_bn_silu_forward_backward_and_fused_silu_grad_epilogue(cuda):
    from cvpytorch_b200 import _lib, train as T
    B, H, W, C = 3, 12, 20, 128
    g = torch.Generator().manual_seed(7)
    y = _bf(torch.randn(B, C, H, W, generator=g) * 1.5 + 0.3).cuda().requires_grad_(True)
    gamma = (torch.rand(C, generator=g) + 0.5).cuda().requires_grad_(True)
    beta = (torch.randn(C, generator=g) * 0.3).cuda().requires_grad_(True)
    da = _bf(torch.randn(B, C, H, W, generator=g)).cuda()
    rm, rv = torch.zeros(C).cuda(), torch.ones(C).cuda()
    a_ref = F.silu(F.batch_norm(y, rm.clone(), rv.clone(), gamma, beta, True, 0.03, 1e-3))
    a_ref.backward(da)
    rm_ref, rv_ref = torch.zeros(C).cuda(), torch.ones(C).cuda()
    F.batch_norm(y.detach(), rm_ref, rv_ref, gamma.detach(), beta.detach(), True, 0.03, 1e-3)
    L = _lib.lib()
    yh = y.detach().permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    dah = da.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    npix = B * H * W
    stat, scratch = torch.empty(4, C, device='cuda'), torch.empty(2, C, device='cuda')
    _lib.check(L.cvb_train_bn_stats(T._p(yh), npix, C, T._p(gamma.detach()), T._p(beta.detach()), 1e-3, 0.03, T._p(rm), T._p(rv), T._p(scratch), T._p(stat), T._stream()), 'stats')
    a = torch.empty_like(yh)
    _lib.check(L.cvb_train_bn_silu_fwd(T._p(yh), npix, C, T._p(stat), T._p(a), T._stream()), 'fwd')
    sums, dy = torch.empty(2, C, device='cuda'), torch.empty_like(yh)
    _lib.check(L.cvb_train_bn_silu_bwd(T._p(dah), 0, T._p(yh), npix, C, T._p(stat), T._p(gamma.detach()), T._p(sums), T._p(dy), T._stream()), 'bwd')
    torch.cuda.synchronize()
    e = dict(a=_rel(a.float().permute(0, 3, 1, 2), a_ref), dy=_rel(dy.float().permute(0, 3, 1, 2), y.grad), dgamma=_rel(sums[1], gamma.grad), dbeta=_rel(sums[0], beta.grad),
             rm=_rel(rm, rm_ref), rv=_rel(rv, rv_ref), mean=_rel(stat[0], y.detach().mean((0, 2, 3))))
    print(e)
    assert e['a'] < 6e-3 and e['dy'] < 6e-3 and max(e['dgamma'], e['dbeta'], e['rm'], e['rv'], e['mean']) < 2e-3, e
    # the backward-data convolution with the producer's SiLU' in its epilogue == backward-data, then * silu'(z) (the separate pass)
    cout2 = 64
    w2 = _bf(torch.randn(cout2, C, 3, 3, generator=g) / (C * 9) ** 0.5).cuda()
    dy2 = _bf(torch.randn(B, H, W, cout2, generator=g)).cuda().to(torch.bfloat16)
    _, wb2 = T.pack_weights(w2)
    fused = T.conv(dy2, wb2, C, 3, y_prev=yh, stat_prev=stat).float()
    plain = T.conv(dy2, wb2, C, 3).float()
    z = yh.float() * stat[2] + stat[3]
    sg = torch.sigmoid(z)
    ref = plain * (sg * (1 + z * (1 - sg)))
    torch.cuda.synchronize()
    assert _rel(fused, ref) < 8e-3, _rel(fused, ref)  # (`plain` was rounded to bf16 before the multiplication, `fused` after)


@pytest.mark.parametrize('shift', [0, 10, 100])
@pytest.mark.parametrize('npix', [2, 7, 129, 102401])
@pytest.mark.parametrize('C', [8, 24, 64, 192, 1024, 2048])
def test_bn_statistics_silu_forward_backward_vs_float64(cuda, C, npix, shift):
    """cvb_train_bn_stats / _bn_silu_fwd / _bn_silu_bwd (g = d(loss)/da, and g = dz as fed by the fused backward-data epilogue) vs float64 on
    the same bf16 inputs: channels with mean = shift * std, C = 8..2048 (C = 24: 256 threads are not a multiple of the 3 vectors per pixel),
    2 pixels (Bessel's correction doubles the variance) to 102 401 (a remainder against the grid cap and the two-load loop).
    Each kernel is compared with float64 of the operation it computes, from the statistics / sums the previous kernel produced; the bounds
    propagate the summation bound of the module docstring (gs) and one 2^-24 rounding per fp32 operation."""
    from cvpytorch_b200 import _lib, train as T
    L, u = _lib.lib(), R.U24
    g = torch.Generator(device='cuda').manual_seed(C * 1000 + npix + shift)
    kw = dict(generator=g, device='cuda')
    std = torch.rand(C, **kw) * 1.5 + 0.5
    y = ((torch.randn(npix, C, **kw) + shift) * std).to(torch.bfloat16)
    gamma, beta = torch.rand(C, **kw) + 0.5, torch.randn(C, **kw) * 0.5
    rm0, rv0 = torch.randn(C, **kw), torch.rand(C, **kw) + 0.5
    eps, mom = 1e-3, 0.1
    rm, rv = rm0.clone(), rv0.clone()
    stat, scratch = torch.empty(4, C, device='cuda'), torch.empty(2, C, device='cuda')
    _lib.check(L.cvb_train_bn_stats(T._p(y), npix, C, T._p(gamma), T._p(beta), eps, mom, T._p(rm), T._p(rv), T._p(scratch), T._p(stat), T._stream()), 'stats')
    a = torch.empty_like(y)
    _lib.check(L.cvb_train_bn_silu_fwd(T._p(y), npix, C, T._p(stat), T._p(a), T._stream()), 'fwd')
    da = torch.randn(npix, C, **kw).to(torch.bfloat16)
    sums, dy = [torch.empty(2, C, device='cuda') for _ in range(2)], [torch.empty_like(y) for _ in range(2)]
    for is_dz in (0, 1):
        _lib.check(L.cvb_train_bn_silu_bwd(T._p(da), is_dz, T._p(y), npix, C, T._p(stat), T._p(gamma), T._p(sums[is_dz]), T._p(dy[is_dz]), T._stream()), 'bwd')
    torch.cuda.synchronize()
    gs = (R.red_chain(npix, C, _sms()) + 2) * u  # + the subtraction of the pivot and the square
    # statistics: mean, variance of the bf16 values in float64 (the kernel sums d = y - y[0]); forward; backward for both kinds of g
    r = R.bn_stats_check(y, gamma, beta, rm0, rv0, eps, mom, stat, rm, rv, gs)
    r.update(R.bn_silu_fwd_check(y, stat, a))
    for is_dz in (0, 1):
        r.update(R.bn_silu_bwd_check(da, is_dz, y, gamma, stat, sums[is_dz], dy[is_dz], gs))
    print('worst error / bound', {k: round(v, 3) for k, v in r.items()})


@pytest.mark.parametrize('case', ['c3_n1', 'c3_n2'])
def test_c3_training_step_vs_reference_fixture(cuda, case):
    from cvpytorch_b200 import train as T
    g = np.load(os.path.join(GOLD, 'c3_train.npz'))
    cin, cout, n, B, H, W = [int(v) for v in g[f'{case}_cfg']]
    m = T.CSPLayer(cin, cout, n=n)
    keys = [str(k) for k in g[f'{case}_keys']]
    assert list(m.state_dict().keys()) == keys  # same module tree / parameter names as the reference block
    m.load_state_dict({k: torch.from_numpy(g[f'{case}_sd_{k}']) for k in keys})
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eps, mod.momentum = 1e-3, 0.03
    m.cuda().train()
    x = torch.from_numpy(g[f'{case}_x']).cuda().requires_grad_(True)
    G = torch.from_numpy(g[f'{case}_G']).cuda()
    y = m(x)
    (y * G).sum().backward()
    torch.cuda.synchronize()
    errs = {'y': _rel(y, torch.from_numpy(g[f'{case}_y'])), 'dx': _rel(x.grad, torch.from_numpy(g[f'{case}_dx']))}
    for k, p in m.named_parameters():
        assert p.grad is not None, k
        errs['grad ' + k] = _rel(p.grad, torch.from_numpy(g[f'{case}_grad_{k}']))
    for k, v in m.state_dict().items():
        if 'running_' in k:
            errs['after ' + k] = _rel(v, torch.from_numpy(g[f'{case}_after_{k}']))
    print({k: round(v, 4) for k, v in errs.items()})
    assert errs['y'] < 3e-2, errs
    assert errs['dx'] < 6e-2 and max(v for k, v in errs.items() if k.startswith('grad ')) < 6e-2, errs
    assert max(v for k, v in errs.items() if k.startswith('after ')) < 1e-2, errs
    # one SGD step through the unchanged torch optimiser keeps working on the drop-in's parameters
    opt = torch.optim.SGD(m.parameters(), lr=0.01, momentum=0.9)
    opt.step()
    opt.zero_grad(set_to_none=True)
    y2 = m(x.detach())
    assert torch.isfinite(y2).all()


def test_c3_dropin_through_the_reference_trainer_train_step(cuda):
    """The drop-in block inside a copy of the reference's training-step logic (trainer.py:177-207: amp.autocast(enabled=cfg.AMP) ->
    scaler.scale(losses['loss']).backward() -> clip_grad -> scaler.step(optimizer) -> scaler.update() -> optimizer.zero_grad(set_to_none=True)),
    with unchanged torch modules before and after it: the loss goes down and every parameter of the block receives finite gradients."""
    from cvpytorch_b200 import train as T
    torch.manual_seed(3)
    stem = torch.nn.Conv2d(3, 128, 3, 2, 1).cuda()          # reference-side layer in front of the block
    block = T.CSPLayer(128, 128, n=2).cuda().train()
    head = torch.nn.Conv2d(128, 8, 1).cuda()                # reference-side layer behind it
    params = list(stem.parameters()) + list(block.parameters()) + list(head.parameters())
    optimizer = torch.optim.SGD(params, lr=0.02, momentum=0.9)
    scaler = torch.amp.GradScaler('cuda', enabled=True)
    imgs = torch.randn(4, 3, 64, 64, device='cuda')
    target = torch.randn(4, 8, 32, 32, device='cuda') * 0.1
    hist = []
    for it in range(8):
        with torch.autocast('cuda', enabled=True):           # cfg.AMP
            out = head(block(stem(imgs)))
            losses = {'loss': (out.float() - target).pow(2).mean()}
        scaler.scale(losses['loss']).backward()
        scaler.unscale_(optimizer)
        torch.nn.utils.clip_grad_norm_(params, 10.0)          # cfg.GRAD_CLIP
        if it == 0:
            for k, p in block.named_parameters():
                assert p.grad is not None and torch.isfinite(p.grad).all() and float(p.grad.abs().max()) > 0, k
        scaler.step(optimizer)
        scaler.update()
        optimizer.zero_grad(set_to_none=True)
        hist.append(float(losses['loss']))
    assert all(np.isfinite(hist)) and hist[-1] < 0.7 * hist[0], hist


# H or W of 1 (a parity class of the input is empty: the forward's fallback tensor map, backward-data skips that class), 2 and 3; B = 5 with
# 128-pixel boxes that span several images and do not divide the batch; cin 192 / 320 (64-wide backward-data tiles under the SiLU' epilogue)
@pytest.mark.parametrize('B,H,W,cin,cout', [(2, 16, 16, 64, 64), (2, 13, 9, 64, 128), (3, 26, 18, 128, 64), (1, 7, 30, 64, 128),
                                            (2, 1, 9, 64, 64), (3, 7, 1, 64, 128), (1, 1, 1, 128, 64), (4, 2, 3, 64, 64), (2, 3, 2, 128, 192), (5, 3, 3, 64, 64),
                                            (5, 5, 7, 128, 64), (5, 11, 9, 64, 128), (2, 11, 13, 192, 64), (2, 9, 7, 320, 192), (1, 9, 9, 128, 384)])
def test_stride2_conv_forward_backward_data_backward_weight(cuda, B, H, W, cin, cout):
    """3x3 / stride 2 / pad 1 (the downsampling BaseConv of every dark stage): forward through four parity tensor maps, backward-data as four
    parity sub-convolutions (with and without the SiLU' epilogue), backward-weight -- vs torch on bf16-representable inputs, odd sizes included,
    max-normalised, and element by element vs float64 (module docstring)."""
    from cvpytorch_b200 import train as T
    g = torch.Generator().manual_seed(B * 31 + H + W + cin)
    x = _bf(torch.randn(B, cin, H, W, generator=g)).cuda().requires_grad_(True)
    w = _bf(torch.randn(cout, cin, 3, 3, generator=g) / (cin * 9) ** 0.5).cuda().requires_grad_(True)
    y_ref = F.conv2d(x, w, None, 2, 1)
    dy = _bf(torch.randn(y_ref.shape, generator=g)).cuda()
    y_ref.backward(dy)
    xh = x.detach().permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    dyh = dy.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    wf, wb = T.pack_weights(w.detach())
    y = T.conv(xh, wf, cout, 3, stride=2)
    assert tuple(y.shape) == (B, y_ref.shape[2], y_ref.shape[3], cout)
    dx = T.conv_dgrad_s2(dyh, wb, cin, H, W)
    dw = T.conv_wgrad(xh, dyh, 3, stride=2)
    torch.cuda.synchronize()
    e = dict(y=_rel(y.float().permute(0, 3, 1, 2), y_ref), dx=_rel(dx.float().permute(0, 3, 1, 2), x.grad), dw=_rel(dw, w.grad))
    print(e)
    assert e['y'] < 6e-3 and e['dx'] < 6e-3 and e['dw'] < 2e-3, e
    # SiLU' epilogue on the strided stores
    yp = _bf(torch.randn(B, H, W, cin, generator=g) * 2).cuda().to(torch.bfloat16)
    stat = _stat_prev(cin, g)
    fused = T.conv_dgrad_s2(dyh, wb, cin, H, W, y_prev=yp, stat_prev=stat)
    z = yp.float() * stat[2] + stat[3]
    sg = torch.sigmoid(z)
    torch.cuda.synchronize()
    assert _rel(fused.float(), dx.float() * (sg * (1 + z * (1 - sg)))) < 8e-3
    r = _conv_vs_float64(x.detach(), w.detach(), dy, 3, 2, y, dx, dw, fused, yp, stat)
    print('worst error / bound', {k_: round(v, 3) for k_, v in r.items()})


def test_dark_stage_training_step_vs_reference_fixture(cuda):
    """stride-2 BaseConv + CSPLayer (one `dark` stage) forward + backward vs the reference modules + torch.autograd (fixture case 'dark')."""
    from cvpytorch_b200 import train as T
    g = np.load(os.path.join(GOLD, 'c3_train.npz'))
    down, csp = T.BaseConv(64, 128, 3, 2), T.CSPLayer(128, 128, n=1)
    m = torch.nn.Sequential(down, csp)
    keys = [str(k) for k in g['dark_keys']]
    assert list(m.state_dict().keys()) == keys
    m.load_state_dict({k: torch.from_numpy(g[f'dark_sd_{k}']) for k in keys})
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eps, mod.momentum = 1e-3, 0.03
    m.cuda().train()
    x = torch.from_numpy(g['dark_x']).cuda().requires_grad_(True)
    G = torch.from_numpy(g['dark_G']).cuda()
    y = csp.forward_nhwc(down(x.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16))).permute(0, 3, 1, 2).float()
    (y * G).sum().backward()
    torch.cuda.synchronize()
    errs = {'y': _rel(y, torch.from_numpy(g['dark_y'])), 'dx': _rel(x.grad, torch.from_numpy(g['dark_dx']))}
    for k, p in m.named_parameters():
        errs['grad ' + k] = _rel(p.grad, torch.from_numpy(g[f'dark_grad_{k}']))
    for k, v in m.state_dict().items():
        if 'running_' in k:
            errs['after ' + k] = _rel(v, torch.from_numpy(g[f'dark_after_{k}']))
    print({k: round(v, 4) for k, v in errs.items()})
    assert errs['y'] < 3e-2 and errs['dx'] < 6e-2 and max(v for k, v in errs.items() if k.startswith('grad ')) < 6e-2, errs
    assert max(v for k, v in errs.items() if k.startswith('after ')) < 1e-2, errs


@pytest.mark.parametrize('c,n,shortcut', [(256, 1, True), (512, 1, False), (1024, 1, False), (384, 1, True)])
def test_wider_c3_blocks_vs_oracle(cuda, c, n, shortcut):
    """dark4 / dark5 widths (256 / 512 channels; dark5 has shortcut=False; 1024 = dark5 of YOLOX-l), and 384 channels (hidden width 192:
    64-wide tiles and backward-weight blocks throughout): the drop-in vs the oracle's training step (reference block restated, torch.autograd,
    fp32 on the host) on seeded parameters -- same tolerances as the fixture test."""
    from cvpytorch_b200 import train as T
    from oracle import c3_train_oracle as CO
    sd = CO.synthetic_state(c, c, n, seed=c)
    g = torch.Generator().manual_seed(c + 1)
    x = torch.randn(2, c, 10, 12, generator=g)
    G = torch.randn(2, c, 10, 12, generator=g)
    sdt = {k: torch.as_tensor(v).clone().requires_grad_(True) if (torch.as_tensor(v).dtype.is_floating_point and 'running_' not in k) else torch.as_tensor(v).clone()
           for k, v in sd.items()}
    xr = x.clone().requires_grad_(True)
    yr = CO.csp_layer(xr, sdt, n, shortcut=shortcut)
    (yr * G).sum().backward()
    m = T.CSPLayer(c, c, n=n, shortcut=shortcut)
    m.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eps, mod.momentum = CO.BN_EPS, CO.BN_MOMENTUM
    m.cuda().train()
    xg = x.cuda().requires_grad_(True)
    y = m(xg)
    (y * G.cuda()).sum().backward()
    torch.cuda.synchronize()
    errs = {'y': _rel(y, yr), 'dx': _rel(xg.grad, xr.grad)}
    for k, p in m.named_parameters():
        errs['grad ' + k] = _rel(p.grad, sdt[k].grad)
    print({k: round(v, 4) for k, v in errs.items()})
    assert errs['y'] < 3e-2 and errs['dx'] < 6e-2 and max(v for k, v in errs.items() if k.startswith('grad ')) < 6e-2, errs
