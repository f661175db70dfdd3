"""YOLOX neck and head TRAINING on the H100 kernels (cvpytorch_b200/train.py: YOLOXNeck, YOLOXHead, ConvModule; csrc/train_kernels.cu):
the upsample-concat kernels, the padded 1x1 convolution, the prediction convs and their gradient kernel, then the neck + head against the
reference fixture tests/golden/yolox_train.npz and the whole network (backbone + neck + head) against the oracle.

Kernels: element-wise float64 bounds of tests/test_train_gpu.py's docstring (fp64ref.py), as in test_darknet_train_gpu.py.

Whole networks: every output, feature-map gradient, parameter gradient and running statistic must have a max-normalised error against fp32
of at most FACTOR * (the error of the same oracle step under torch.autocast(bfloat16) on this GPU) + FLOOR, the backbone's rule
(test_darknet_train_gpu.py).  Measured on one H100 80GB HBM3 (SXM, 400 W power limit) in two runs: the median ratio kernels / autocast
over all tensors is 0.71 (fixture), 0.85 (YOLOX-n) and 0.83 (YOLOX-s); the largest ratio is 2.42 (fixture), 2.07-2.24 (YOLOX-n) and
1.63-1.76 (YOLOX-s).  Runs differ because the backward-weight atomics add in no fixed order.  FACTOR = 3 is the backbone's factor and
covers these with margin."""
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
NECK = dict(channels=[128, 128, 128], depth_mul=0.33, width_mul=0.25)  # (the configuration of tools/make_golden_yolox_train.py)
HEAD = dict(num_classes=3, in_channels=[256, 256, 256], width_mul=0.125)
WIDTH = {'cspdark_n': 0.25, 'cspdark_s': 0.5}


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def _bf(t):
    return t.to(torch.bfloat16).float()


def _kpad(c):
    return -(-c // 64) * 64


@pytest.mark.parametrize('B,h,w,Ca,Cb', [(2, 3, 5, 32, 32), (2, 6, 10, 16, 32), (1, 1, 1, 16, 16), (3, 7, 9, 64, 128), (16, 40, 40, 128, 128)])
def test_upsample_cat_forward_backward(cuda, B, h, w, Ca, Cb):
    """Forward bit-exact against F.interpolate(nearest) + torch.cat; backward: db bit-exact, da within one bf16 rounding of the float64 2x2
    sum (plus the fp32 additions), bitwise reproducible."""
    from cvpytorch_b200 import train as T
    g = torch.Generator().manual_seed(B * 100 + h * 10 + w + Ca + Cb)
    a = torch.randn(B, Ca, h, w, generator=g).to(torch.bfloat16).cuda()
    b = torch.randn(B, Cb, 2 * h, 2 * w, generator=g).to(torch.bfloat16).cuda()
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()  # noqa: E731
    cat = T.upsample_cat(nhwc(a), nhwc(b))
    ref = torch.cat([F.interpolate(a.float(), scale_factor=2, mode='nearest'), b.float()], 1).to(torch.bfloat16)
    assert torch.equal(cat, nhwc(ref))
    gr = torch.randn(B, Ca + Cb, 2 * h, 2 * w, generator=g).to(torch.bfloat16)
    gh = nhwc(gr).cuda()
    da1, db1 = T.upsample_cat_backward(gh, Ca)
    da2, db2 = T.upsample_cat_backward(gh, Ca)
    torch.cuda.synchronize()
    assert torch.equal(da1, da2) and torch.equal(db1, db2)
    assert torch.equal(db1, gh[..., Ca:])
    ga = gr[:, :Ca].double()
    ref_da = F.avg_pool2d(ga, 2) * 4
    abs_da = F.avg_pool2d(ga.abs(), 2) * 4
    worst = R.check(da1.permute(0, 3, 1, 2), ref_da, R.BF16_REL * ref_da.abs() + (1 + R.BF16_REL) * 4 * R.U24 * abs_da, 'upsample-cat backward')
    print('worst error / bound', round(worst, 3))


# (B, H, W, cin, cout, pad): the head stems (1x1, padding 1; their backward-data is the padding -1 conv), odd maps, 16 / 32 / 64 / 128 / 256
# channels, and padding 0
@pytest.mark.parametrize('B,H,W,cin,cout,pad', [(2, 3, 5, 32, 32, 1), (2, 12, 20, 32, 32, 1), (2, 9, 7, 64, 128, 1), (3, 20, 16, 128, 64, 1),
                                                 (2, 5, 5, 256, 16, 1), (2, 11, 13, 16, 32, 0)])
def test_padded_1x1_conv_forward_backward_data_backward_weight(cuda, B, H, W, cin, cout, pad):
    from cvpytorch_b200 import train as T
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + W + cin + cout + pad)
    x = _bf(torch.randn(B, cin, H, W, generator=g)).cuda()
    w = _bf(torch.randn(cout, cin, 1, 1, generator=g) / cin ** 0.5).cuda()
    Ho, Wo = H + 2 * pad, W + 2 * pad
    dy = _bf(torch.randn(B, cout, Ho, Wo, generator=g)).cuda()
    xh, dyh = x.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16), dy.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    wf, wb = T.pack_weights(w)
    yh = T.conv(xh, wf, cout, 1, pad=pad)
    dxh = T.conv(dyh, wb, cin, 1, pad=-pad)
    dw = T.conv_wgrad(xh, dyh, 1, pad=pad)
    torch.cuda.synchronize()
    assert tuple(yh.shape) == (B, Ho, Wo, cout) and tuple(dxh.shape) == (B, H, W, cin)

    def nhwc(t):
        return t.permute(0, 2, 3, 1)
    yr, ya = (nhwc(t) for t in R.conv_fwd(x, w, 1, pad))
    dxr, dxa = (nhwc(t) for t in R.conv_dgrad(dy, w, x.shape, 1, pad))
    dwr, dwa = R.conv_wgrad(x, dy, w.shape, 1, pad)
    g_f, g_d = R.mma_gamma(_kpad(cin)), R.mma_gamma(_kpad(cout))
    g_w = R.wgrad_gamma(B, Ho, Wo, cin, cout, 1, torch.cuda.get_device_properties(0).multi_processor_count)
    r = {'y': R.check(yh, yr, R.BF16_REL * yr.abs() + (1 + R.BF16_REL) * g_f * ya, 'forward'),
         'dx': R.check(dxh, dxr, R.BF16_REL * dxr.abs() + (1 + R.BF16_REL) * g_d * dxa, 'backward-data'),
         'dw': R.check(dw, dwr, g_w * dwa, 'backward-weight')}
    print('worst error / bound', {k: round(v, 3) for k, v in r.items()})


@pytest.mark.parametrize('cout', [1, 3, 5, 80])
def test_prediction_conv_forward_and_pred_grad(cuda, cout):
    """cvb_train_pred_conv writes channels [c_off, c_off + cout) of an fp32 NCHW tensor (= conv + bias, the rest untouched);
    cvb_train_pred_grad's dy is the bf16 rounding of that gradient slice with zero padding, dbias its fp32 sum."""
    from cvpytorch_b200 import train as T
    B, h, w, cin, c_off = 3, 14, 22, 64, 2
    c_tot = cout + 5
    g = torch.Generator().manual_seed(cout)
    x = _bf(torch.randn(B, cin, h, w, generator=g)).cuda()
    wt = _bf(torch.randn(cout, cin, 1, 1, generator=g) / cin ** 0.5).cuda()
    bias = torch.randn(cout, generator=g).cuda()
    cp = T.pred_cout_pad(cout)
    wf, wb = T.pack_weights(F.pad(wt, (0, 0, 0, 0, 0, 0, 0, cp - cout)))
    out = torch.full((B, c_tot, h, w), float('nan'), device='cuda')
    T.pred_conv(x.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16), wf, cout, bias, out, c_off)
    torch.cuda.synchronize()
    yr, ya = R.conv_fwd(x, wt, 1, 0)
    ref = yr + bias.double().view(1, -1, 1, 1)
    bound = R.mma_gamma(_kpad(cin)) * ya + 2 * R.U24 * (yr.abs() + bias.double().abs().view(1, -1, 1, 1))
    worst = R.check(out[:, c_off:c_off + cout], ref, bound, 'prediction conv forward')
    assert torch.isnan(out[:, :c_off]).all() and torch.isnan(out[:, c_off + cout:]).all()
    gr = torch.randn(B, c_tot, h, w, generator=g).cuda()
    dy, db = T.pred_grad(gr, c_off, cout)
    torch.cuda.synchronize()
    assert tuple(dy.shape) == (B, h, w, cp)
    assert torch.equal(dy[..., :cout], gr[:, c_off:c_off + cout].permute(0, 2, 3, 1).to(torch.bfloat16)) and not bool(dy[..., cout:].any())
    gs = gr[:, c_off:c_off + cout].double()
    terms = B * -(-(h * w) // 256) + 8
    worst_b = R.check(db, gs.sum((0, 2, 3)), terms * R.U24 * gs.abs().sum((0, 2, 3)), 'prediction bias gradient')
    print('worst error / bound', round(worst, 3), round(worst_b, 3))


def _leaves(sd, dev):
    out = {}
    for k, v in sd.items():
        t = torch.as_tensor(v).clone().to(dev)
        if t.dtype.is_floating_point and 'running_' not in k:
            t.requires_grad_(True)
        out[k] = t
    return out


def _compare(named, ref, auto):
    """named / ref / auto: {tensor name: value} of the kernels, the fp32 reference and the bf16-autocast step."""
    errs = {k: _rel(v, ref[k]) for k, v in named.items()}
    au = {k: _rel(auto[k], ref[k]) for k in named}
    ratio = {k: errs[k] / (au[k] + 1e-12) for k in errs}
    worst = sorted(errs, key=lambda k: errs[k] - FACTOR * au[k])[-5:]
    print('kernels vs fp32 (max-normalised): max', round(max(errs.values()), 4), 'autocast bf16 vs fp32: max', round(max(au.values()), 4),
          'median kernel / autocast', round(float(np.median(list(ratio.values()))), 3))
    print('closest to the limit', {k: (round(errs[k], 4), round(au[k], 4)) for k in worst}, 'largest ratio', round(max(ratio.values()), 3))
    bad = {k: (errs[k], au[k]) for k in errs if errs[k] > FACTOR * au[k] + FLOOR}
    assert not bad, bad


def _collect(outs, dxs, mods, prefixed_grads=None):
    """-> {name: tensor} of outputs, feature gradients, parameter gradients and running statistics of the kernel modules {prefix: module}."""
    d = {f'y{i}': o for i, o in enumerate(outs)}
    d.update({f'dx{i}': x for i, x in enumerate(dxs)})
    for pre, m in mods.items():
        for k, p in m.named_parameters():
            assert p.grad is not None, pre + k
            d['grad_' + pre + k] = p.grad
        for k, v in m.state_dict().items():
            if 'running_' in k:
                d['after_' + pre + k] = v
    return d


def _oracle_named(outs, dxs, grads, stats):
    d = {f'y{i}': o for i, o in enumerate(outs)}
    d.update({f'dx{i}': x for i, x in enumerate(dxs)})
    d.update({'grad_' + k: v for k, v in grads.items()})
    d.update({'after_' + k: v for k, v in stats.items()})
    return d


def _neck_head_kernel_step(neck_kw, head_kw, sd, feats, Gs):
    from cvpytorch_b200 import train as T
    nk, hd = T.YOLOXNeck(**neck_kw), T.YOLOXHead(**head_kw)
    nk.load_state_dict({k[5:]: torch.as_tensor(v) for k, v in sd.items() if k.startswith('neck.')})
    hd.load_state_dict({k[5:]: torch.as_tensor(v) for k, v in sd.items() if k.startswith('head.')})
    nk.cuda().train()
    hd.cuda().train()
    xs = [f.cuda().requires_grad_(True) for f in feats]
    outs = hd.forward_nhwc(nk.forward_nhwc([x.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16) for x in xs]))
    for o in outs:
        assert o.dtype == torch.float32 and o.is_contiguous()
    sum((o * G.cuda()).sum() for o, G in zip(outs, Gs)).backward()
    torch.cuda.synchronize()
    return _collect(outs, [x.grad for x in xs], {'neck.': nk, 'head.': hd})


def _neck_head_autocast_step(sd, feats, Gs, depth_mul):
    from oracle import yolox_train_oracle as XO
    sdt = _leaves(sd, 'cuda')
    xs = [f.cuda().requires_grad_(True) for f in feats]
    with torch.autocast('cuda', dtype=torch.bfloat16):
        outs = XO.head(XO.neck(xs, sdt, depth_mul), sdt)
    sum((o.float() * G.cuda()).sum() for o, G in zip(outs, Gs)).backward()
    return _oracle_named([o.float() for o in outs], [x.grad for x in xs], {k: v.grad for k, v in sdt.items() if v.requires_grad},
                         {k: v for k, v in sdt.items() if 'running_' in k})


def test_neck_head_training_step_vs_reference_fixture(cuda):
    """Neck widths 32 / 16 and head width 32, 3 classes, feature maps 2x32x{12x20, 6x10, 3x5}, against the reference's YOLOXNeck + YOLOXHead
    and torch.autograd in fp32 (outputs, feature-map gradients, every parameter gradient, running statistics)."""
    from oracle import yolox_train_oracle as XO
    g = np.load(os.path.join(GOLD, 'yolox_train.npz'))
    keys, sd, feats, Gs, dm = XO.fixture_inputs(g)
    got = _neck_head_kernel_step(NECK, HEAD, sd, feats, Gs)
    ref = {k: torch.from_numpy(g[k]) for k in g.files if k.startswith(('y', 'dx', 'grad_', 'after_'))}
    assert set(got) == set(ref)
    _compare(got, ref, _neck_head_autocast_step(sd, feats, Gs, dm))


def _network_models(sub):
    from cvpytorch_b200 import train as T
    w = WIDTH[sub]
    return (T.CSPDarknet(sub), T.YOLOXNeck('yolox_' + sub[-1], [256, 512, 1024], 0.33, w),
            T.YOLOXHead(80, 'yolox_' + sub[-1], [256, 512, 1024], width_mul=w))


def _network_state(sub, seed):
    from oracle import yolox_train_oracle as XO
    shapes = [(pre + k, tuple(v.shape)) for pre, m in zip(('backbone.', 'neck.', 'head.'), _network_models(sub)) for k, v in m.state_dict().items()]
    return XO.synthetic_state(shapes, seed=seed)


@pytest.mark.parametrize('sub', ['cspdark_n', 'cspdark_s'])
def test_backbone_neck_head_training_step_vs_oracle(cuda, sub):
    """Stock YOLOX-n / YOLOX-s, 80 classes, on 2x3x128x160: train.CSPDarknet -> YOLOXNeck -> YOLOXHead chained through forward_nhwc against
    the oracle's fp32 step on this GPU (TF32 off): the three head outputs, every parameter gradient and every running statistic."""
    from oracle import yolox_train_oracle as XO
    sd = _network_state(sub, seed=7 + len(sub))
    g = torch.Generator().manual_seed(13)
    x = torch.randn(2, 3, 128, 160, generator=g)
    Gs = [torch.randn(2, 85, 128 // s + 2, 160 // s + 2, generator=g) for s in (8, 16, 32)]

    def oracle_step(autocast):
        sdt = _leaves(sd, 'cuda')
        with torch.autocast('cuda', dtype=torch.bfloat16, enabled=autocast):
            outs = XO.network(x.cuda(), sdt, sub)
        sum((o.float() * G.cuda()).sum() for o, G in zip(outs, Gs)).backward()
        return _oracle_named([o.float().detach() for o in outs], [], {k: v.grad for k, v in sdt.items() if v.requires_grad},
                             {k: v for k, v in sdt.items() if 'running_' in k})
    ref, auto = oracle_step(False), oracle_step(True)
    bb, nk, hd = _network_models(sub)
    mods = {'backbone.': bb, 'neck.': nk, 'head.': hd}
    for pre, m in mods.items():
        m.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)})
        m.cuda().train()
    outs = hd.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(x.cuda())))
    assert [tuple(o.shape) for o in outs] == [tuple(G.shape) for G in Gs]
    sum((o * G.cuda()).sum() for o, G in zip(outs, Gs)).backward()
    torch.cuda.synchronize()
    _compare(_collect(outs, [], mods), ref, auto)


def test_neck_head_hand_off_to_inference_modules(cuda):
    """One SGD step of the YOLOX-s neck + head on the kernels, then load_state_dict(strict=True) into the inference yolox_models.YOLOXNeck /
    YOLOXHead and evaluate: within 1e-3 of max|ref| of oracle/yolox_oracle.neck / head (float64) on the updated parameters.  As in the
    backbone's hand-off test, a first momentum-None forward calibrates the running statistics of the seeded state and the step clips the
    gradient norm to 10."""
    from cvpytorch_b200 import train as T, yolox_models as Y
    from oracle import yolox_oracle as YO, yolox_train_oracle as XO
    nk = T.YOLOXNeck('yolox_s', [256, 512, 1024], 0.33, 0.5)
    hd = T.YOLOXHead(80, 'yolox_s', [256, 512, 1024], width_mul=0.5)
    shapes = [(pre + k, tuple(v.shape)) for pre, m in (('neck.', nk), ('head.', hd)) for k, v in m.state_dict().items()]
    sd = XO.synthetic_state(shapes, seed=21)
    nk.load_state_dict({k[5:]: v for k, v in sd.items() if k.startswith('neck.')})
    hd.load_state_dict({k[5:]: v for k, v in sd.items() if k.startswith('head.')})
    nk.cuda().train()
    hd.cuda().train()
    g = torch.Generator().manual_seed(22)
    feats = [torch.randn(2, c, 128 // s, 160 // s, generator=g).cuda() for c, s in ((128, 8), (256, 16), (512, 32))]
    bns = [m for mod in (nk, hd) for m in mod.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    for bn in bns:
        bn.momentum = None
    with torch.no_grad():
        hd(nk(feats))
    for bn in bns:
        bn.momentum = 0.03
    outs = hd(nk(feats))
    sum((o * torch.randn(o.shape, generator=g).cuda()).sum() for o in outs).backward()
    params = list(nk.parameters()) + list(hd.parameters())
    torch.nn.utils.clip_grad_norm_(params, 10.0)
    torch.optim.SGD(params, lr=0.01, momentum=0.9).step()
    trained = {'neck.' + k: v.detach().cpu() for k, v in nk.state_dict().items()}
    trained.update({'head.' + k: v.detach().cpu() for k, v in hd.state_dict().items()})
    inf_n, inf_h = Y.YOLOXNeck('yolox_s', [256, 512, 1024], 0.33, 0.5), Y.YOLOXHead(80, 'yolox_s', [256, 512, 1024], width_mul=0.5)
    inf_n.load_state_dict({k[5:]: v for k, v in trained.items() if k.startswith('neck.')}, strict=True)
    inf_h.load_state_dict({k[5:]: v for k, v in trained.items() if k.startswith('head.')}, strict=True)
    inf_n.cuda().eval()
    inf_h.cuda().eval()
    with torch.no_grad():
        got = inf_h(inf_n(feats))
    sd64 = {k: v.double() if v.dtype.is_floating_point else v for k, v in trained.items()}
    ref = YO.head(YO.neck([f.cpu().double() for f in feats], sd64), sd64)
    errs = [_rel(a, b) for a, b in zip(got, ref)]
    print('inference vs oracle after one training step', errs)
    assert max(errs) < 1e-3, errs


def test_network_training_loop_captured_as_cuda_graph(cuda):
    """A trainer-style loop over backbone + neck + head (YOLOX-n, 80 classes): a stand-in loss on the three head outputs, backward and SGD
    captured as one CUDA graph and replayed.  The loss falls and every parameter gets a finite, non-zero gradient."""
    torch.manual_seed(6)
    bb, nk, hd = (m.cuda().train() for m in _network_models('cspdark_n'))
    params = [p for m in (bb, nk, hd) for p in m.parameters()]
    opt = torch.optim.SGD(params, lr=0.05, momentum=0.9)
    x = torch.randn(4, 3, 128, 128, device='cuda')
    targets = [torch.randn(4, 85, 128 // s + 2, 128 // s + 2, device='cuda') * 0.1 for s in (8, 16, 32)]

    def step():
        outs = hd.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(x)))
        loss = sum((o - t).pow(2).mean() for o, t in zip(outs, targets))
        loss.backward()
        torch.nn.utils.clip_grad_norm_(params, 10.0)
        return loss

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for it in range(2):
            loss = step()
            if it == 0:
                for p in params:
                    assert p.grad is not None and torch.isfinite(p.grad).all() and float(p.grad.abs().max()) > 0
            opt.step()
            opt.zero_grad(set_to_none=False)
        del loss  # (drops the eager step's autograd graph before capture)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_loss = step()
        opt.step()
        opt.zero_grad(set_to_none=False)
    hist = []
    for _ in range(16):
        graph.replay()
        hist.append(float(static_loss.detach()))
    print('loss', [round(v, 4) for v in hist])
    assert all(np.isfinite(hist)) and hist[-1] < 0.8 * hist[0], hist
