"""float64 references and element-wise error bounds for the training kernels (tests/test_train_gpu.py), for the split-fp16 inference
conv (split_conv_reference below) and for the split16 format and the aux kernels (tests/test_aux_kernels_gpu.py, test_fcos_gpu.py).

Each reference is computed in float64 on exactly the bf16 values the kernel reads, together with the same operation on the absolute values
of its inputs (`absref`).  absref bounds every partial sum of a dot product, so the fp32 accumulation error of one output element is at most
gamma * absref: a small output element gets a small tolerance, unlike a check normalised by the tensor's maximum.

    |out - ref| <= rel * |ref| + gamma * absref          element by element

The constants (derived, not fitted; see test_train_gpu.py for each kernel):
  rel   = 2^-8   bf16 keeps 8 significant bits, so round-to-nearest of the stored output is off by at most 2^-8 relative
                 (a value just above 1 + 2^-8 comes within a hair of that; 2^-9 is the average, not the bound)
  gamma = (number of chained K = 16 MMAs + 16) * 2^-23   one fp32 ulp per accumulation into the tensor-core accumulator, plus the 16
                 additions inside one K = 16 MMA; the products of two bf16 values are exact in fp32
"""
import math

import torch
import torch.nn.functional as F

BF16_REL = 2.0 ** -8
U23 = 2.0 ** -23  # one fp32 ulp relative: tensor-core accumulation
U24 = 2.0 ** -24  # fp32 round-to-nearest


def conv_fwd(x, w, stride, pad):
    """x [B,cin,H,W], w [cout,cin,k,k] (any float dtype) -> float64 conv, and the same conv of |x|, |w|."""
    x, w = x.double(), w.double()
    return F.conv2d(x, w, None, stride, pad), F.conv2d(x.abs(), w.abs(), None, stride, pad)


def conv_dgrad(dy, w, x_shape, stride, pad):
    """d(loss)/dx of conv_fwd for the output gradient dy, and the same with |dy|, |w|."""
    dy, w = dy.double(), w.double()
    f = torch.nn.grad.conv2d_input
    return f(x_shape, w, dy, stride, pad), f(x_shape, w.abs(), dy.abs(), stride, pad)


def conv_wgrad(x, dy, w_shape, stride, pad):
    """d(loss)/dw of conv_fwd for the output gradient dy, and the same with |x|, |dy|."""
    x, dy = x.double(), dy.double()
    f = torch.nn.grad.conv2d_weight
    return f(x, w_shape, dy, stride, pad), f(x.abs(), w_shape, dy.abs(), stride, pad)


def mma_gamma(k):
    """Accumulation error factor of a K = k dot product on the K = 16 bf16 MMAs (k a multiple of 16)."""
    return (math.ceil(k / 16) + 16) * U23


def silu_grad64(z):
    s = torch.sigmoid(z)
    return s * (1 + z * (1 - s))


def sigmoid_rel_err(z):
    """Relative error of 1 / (1 + __expf(-z)) in fp32: __expf(x) is within 2 + floor(1.173 |x|) ulps (CUDA programming guide, intrinsic
    functions), the addition and the division round once each."""
    return (2 + 1.173 * z.abs()) * U23 + 2 * U24


def silu_grad_err(z):
    """Absolute error of the kernels' silu'(z) = g * (1 + z * (1 - g)), g = sigmoid(z) as above: d silu' / d g = 1 + z (1 - 2 g), so an error
    e * g of g moves silu' by at most e * (1 + |z|); three more roundings of terms no larger than 1 + |z|."""
    return (sigmoid_rel_err(z) + 3 * U24) * (1 + z.abs())


def choose_box128(B, H, W):
    """Restates the kernels' pixel box choice (csrc/train_kernels.cu choose_box128): TW x TH x NB = 128 powers of two, fewest wasted rows."""
    best, box = -1.0, None
    tw = 1
    while tw <= 128:
        th = 1
        while tw * th <= 128:
            nb = 128 // (tw * th)
            tiles = -(-W // tw) * -(-H // th) * -(-B // nb)
            util = B * H * W / (tiles * 128.0) + 1e-6 * tw
            if util > best:
                best, box = util, (tw, th, nb)
            th *= 2
        tw *= 2
    return box


def wgrad_split(B, Ho, Wo, cin, cout, k, sms):
    """Restates cvb_train_conv_wgrad's launch: -> (m_tiles, splits, per), `per` = 128-pixel tiles one CTA accumulates before its atomics.
    cout = 16 or 32 runs as one 64-wide block."""
    tw, th, nb = choose_box128(B, Ho, Wo)
    m_tiles = -(-Wo // tw) * -(-Ho // th) * -(-B // nb)
    npan = 4 if (cout // 64) % 4 == 0 else (2 if (cout // 64) % 2 == 0 else 1)
    nblocks = 1 if cout < 64 else cout // (64 * npan)
    splits = (2 * sms) // (k * k * -(-cin // 128) * nblocks)
    splits = min(max(splits, 1), m_tiles)
    return m_tiles, splits, -(-m_tiles // splits)


def red_chain(npix, C, sms):
    """Longest fp32 addition chain of one channel's sum in bn_stats_kernel / bn_silu_bwd_reduce_kernel (csrc/train_kernels.cu red_grid):
    the pixels of one thread (+1 for the paired loads), the CTA's pixel lanes, one atomic per CTA."""
    lanes = 256 // (C // 8)
    grid = min(max(-(-npix // (lanes * 4)), 1), sms * 4)
    return -(-(-(-npix // grid)) // lanes) + 1 + lanes + grid


def wgrad_gamma(B, Ho, Wo, cin, cout, k, sms):
    """One CTA chains 8 MMAs (K = 16 pixels each) per tile it owns; `splits` CTAs then add their partial sums with fp32 atomics (every
    width: cout = 16 / 32 runs as one 64-wide block)."""
    _, splits, per = wgrad_split(B, Ho, Wo, cin, cout, k, sms)
    return (8 * per + 16 + splits) * U23


# ---------------------------------------------------------------------------------------------------- BatchNorm + SiLU training passes
# Each kernel is compared with float64 of the operation it computes, from the statistics / sums the previous kernel produced; the bounds
# propagate the summation bound gs (relative to the sum of |terms|: (red_chain + 2) * 2^-24 for the pivoted fp32 sums, see
# tests/test_train_gpu.py) and one 2^-24 rounding per fp32 operation.  y, da: [npix, C] bf16; stat [4][C] = mean, rstd, scale, shift.
def bn_stats_check(y, gamma, beta, rm0, rv0, eps, mom, stat, rm, rv, gs):
    """cvb_train_bn_stats' statistics and running statistics (rm0 / rv0 before, rm / rv after) -> {name: worst |error| / bound}."""
    u = U24
    y64, n = y.double(), float(y.shape[0])
    mean, var = y64.mean(0), y64.var(0, unbiased=False)
    d = y64 - y64[0]
    d_abs, d_sq, d_mean = d.abs().mean(0), (d * d).mean(0), d.mean(0)
    del d
    e_mean = gs * d_abs + u * mean.abs()
    e_var = gs * d_sq + 2 * d_mean.abs() * gs * d_abs
    rstd = 1 / torch.sqrt(var + eps)
    e_rstd = rstd * (0.5 * e_var / (var + eps) + 2 * u)
    g64, b64 = gamma.double(), beta.double()
    scale = g64 * rstd
    e_scale = g64 * e_rstd + u * scale
    e_shift = mean.abs() * e_scale + scale * e_mean + 2 * u * ((mean * scale).abs() + b64.abs())
    r = {'mean': check(stat[0], mean, e_mean, 'mean'), 'rstd': check(stat[1], rstd, e_rstd, 'rstd'),
         'scale': check(stat[2], scale, e_scale, 'scale'), 'shift': check(stat[3], b64 - mean * scale, e_shift, 'shift')}
    m = float(torch.tensor(mom, dtype=torch.float32))
    var_unb = var * n / max(n - 1, 1)
    rm_ref, rv_ref = (1 - m) * rm0.double() + m * mean, (1 - m) * rv0.double() + m * var_unb
    r['running_mean'] = check(rm, rm_ref, m * e_mean + 4 * u * ((1 - m) * rm0.double().abs() + m * mean.abs()), 'running_mean')
    r['running_var'] = check(rv, rv_ref, m * (e_var * n / max(n - 1, 1) + u * var_unb) + 4 * u * rv_ref, 'running_var')
    return r


def bn_silu_fwd_check(y, stat, a):
    """a = silu(y * scale + shift) with the kernel's scale / shift: one fma, __expf, an addition and a division, bf16 store."""
    z = y.double() * stat[2].double() + stat[3].double()
    a_ref = z * torch.sigmoid(z)
    return {'a': check(a, a_ref, BF16_REL * a_ref.abs() + (1 + BF16_REL) * (a_ref.abs() * sigmoid_rel_err(z) + 1.1 * U24 * z.abs()), 'a')}


def bn_silu_bwd_check(da, is_dz, y, gamma, stat, sums, dy, gs, gs_sum=None):
    """cvb_train_bn_silu_bwd with the kernel's mean / rstd / scale / shift: dz = g * silu'(z) (or g when is_dz), xhat = (y - mean) * rstd;
    sums = (sum dz, sum dz * xhat), dy.  gs_sum: the summation bound of sum dz alone (default gs; 0 where that sum is exact)."""
    u = U24
    gs_sum = gs if gs_sum is None else gs_sum
    y64, n = y.double(), float(y.shape[0])
    xhat = (y64 - stat[0].double()) * stat[1].double()
    g64d = da.double()
    if is_dz:
        dz, e_dz = g64d, torch.zeros_like(g64d)
    else:
        z = y64 * stat[2].double() + stat[3].double()
        dz = g64d * silu_grad64(z)
        e_dz = g64d.abs() * silu_grad_err(z) + u * dz.abs()
        del z
    tag = ' (g = dz)' if is_dz else ''
    r = {'sum dz' + tag: check(sums[0], dz.sum(0), gs_sum * dz.abs().sum(0) + e_dz.sum(0), 'sum dz' + tag)}
    dzx = (dz * xhat).abs()
    r['sum dz*xhat' + tag] = check(sums[1], (dz * xhat).sum(0), (gs + 3 * u) * dzx.sum(0) + (e_dz * xhat.abs()).sum(0), 'sum dz*xhat' + tag)
    del dzx
    # dy = gamma * rstd * (dz - S0 / n - xhat * S1 / n) from the kernel's sums: about eight fp32 roundings of terms of that size
    S0, S1 = sums[0].double() / n, sums[1].double() / n
    g64 = gamma.double()
    gr = (g64 * stat[1].double()).abs()
    dy_ref = g64 * stat[1].double() * (dz - S0 - xhat * S1)
    bound = BF16_REL * dy_ref.abs() + (1 + BF16_REL) * gr * (e_dz + 8 * u * (dz.abs() + S0.abs() + (xhat * S1).abs()))
    r['dy' + tag] = check(dy, dy_ref, bound, 'dy' + tag)
    return r


# ---------------------------------------------------------------------------------------------------- split-fp16 inference conv
SPLIT_REL = 2.0 ** -19   # see split_conv_reference
LAYER_BUDGET = 2e-5      # max|out - ref| / max|ref| of one layer (DESIGN.md 2)


def split64(t):
    """fp16 hi / lo planes [2, B, H, W, C] (a SplitTensor or its data, possibly a channel slice) -> float64 NCHW hi + lo."""
    d = t if torch.is_tensor(t) else t.data
    return (d[0].double() + d[1].double()).permute(0, 3, 1, 2)


def conv_out64(d):
    """The conv's output buffer (fp16 hi / lo planes [2, B, H, W, C] or fp32 [B, H, W, C]) -> float64 NCHW."""
    return split64(d) if d.dtype == torch.float16 else d.double().permute(0, 3, 1, 2)


def split_conv_sums(pairs, k, s=1, p=0, dil=1, w_window=0, out_h=None):
    """The conv kernel's dot products in float64, without bias or epilogue: for each (x [B, C, H, W], w [cout, K] in the packed K order)
    of `pairs`, the NCHW conv with the kernel's geometry (see split_conv_reference).  -> ([conv of each pair], taps, K per tap)."""
    x0, w0 = pairs[0]
    cout = w0.shape[0]
    if w_window:
        C = x0.shape[1]
        Ho = x0.shape[2] if out_h is None else out_h

        def conv(x, w):
            x = F.pad(x, (0, 0, p, max(0, Ho + k - 1 - p - x.shape[2])))[:, :, :Ho + k - 1]
            return F.conv2d(x, w.view(cout, k, w_window, C).permute(0, 3, 1, 2))
        return [conv(x, w) for x, w in pairs], k, w_window * C
    cin = x0.shape[1]
    return [F.conv2d(x, w.view(cout, k, k, cin).permute(0, 3, 1, 2), None, s, p, dil) for x, w in pairs], k * k, cin


def split_conv_reference(tin, wp, bp, k, s=1, p=0, dil=1, act='silu', residual=None, resid_first=0, resid_scale=1.0, up=None,
                         w_window=0, block_n=128, cout=None, out_h=None):
    """float64 reference of the fused conv kernel (csrc/conv_tc.cu) and the element-wise bound of its error -> (ref, bound), NCHW.

    Computed on the GPU from exactly the values the kernel reads: hi + lo of the split input `tin` ([2, B, H, W, C] fp16, a channel slice
    is fine) and of the packed weights `wp` ([2, cout_pad, K] from ops.pack_conv_weights), the fp32 bias `bp`, the split `residual`
    ([2, B, Ho, Wo, cout]) times `resid_scale`, and the fp32 `up` partial ([B, ceil(Ho/2), ceil(Wo/2), cout], nearest x2).  absref is the
    same conv on |x|, |w| plus |bias|, |up| (and |residual| when it enters before the activation): it bounds every partial sum.

        |out - ref| <= 2^-19 (|ref| + |residual|) + slope * gamma * absref
        gamma = mma_gamma(16 chain) + chain * 2^-25 + 2^-21

    Each constant follows from the kernel's arithmetic:
      chain   the MMAs (K = 16 each) chained into the hi*hi accumulator of one output element: taps * K_tap / 16.  It is also the
              chain rz_gain = 1 + 1.9e-8 * chain is computed from; the gain's own correction is at most 2^-25 per MMA of the chain.
        classic / halo loader, stride 2, dilation: taps = kh * kw, K_tap = cin.  The K order differs between loaders, not the chain.
        row-window stems (w_window = win): taps = kh filter rows of K_tap = win * C, the all-zero weight columns included; the kernel
              skips their MMAs (kskip) but rz_gain counts them, and counting them in gamma only loosens it.
        block_n = 256: hi*hi and both cross terms share one register accumulator (no separate cross accumulator), so the chain is three
              times as long: chain = 3 * taps * K_tap / 16.
      mma_gamma  one fp32 ulp (2^-23: the tensor core's adder truncates) per chained MMA plus 16 for the additions inside one MMA.
      2^-21   the dropped lo * lo products (|lo| <= 2^-11 |hi| on both operands) and the cross terms' own rounding.
      slope   1.1 for SiLU (|silu'| <= 1.1), 1 for ReLU and for no activation: the accumulation error passes through the activation.
      2^-19   the epilogue after the accumulator: the fast SiLU (~2^-22 relative), the fp32 additions of bias / up / residual and the
              hi / lo split of the output (~22 bits), relative to the output and to the residual added after the activation.

    w_window: out_h = the output height (default: the input height); filter row ky reads input row h + ky - p, rows past the input
    read TMA zero fill, and the input already carries the left zero columns."""
    x = split64(tin)
    cout = wp.shape[1] if cout is None else cout
    w = (wp[0].double() + wp[1].double())[:cout]
    (ref, absref), taps, k_tap = split_conv_sums([(x, w), (x.abs(), w.abs())], k, s, p, dil, w_window, out_h)
    b = bp[:cout].double().view(1, -1, 1, 1)
    ref, absref = ref + b, absref + b.abs()
    Ho, Wo = ref.shape[2:]
    if up is not None:
        u = F.interpolate(up.double().permute(0, 3, 1, 2), scale_factor=2, mode='nearest')[:, :, :Ho, :Wo]
        ref, absref = ref + u, absref + u.abs()
    rsum = split64(residual) * resid_scale if residual is not None else torch.zeros_like(ref)
    if resid_first:
        ref, absref = ref + rsum, absref + rsum.abs()
    if act == 'silu':
        ref = F.silu(ref)
    elif act == 'relu':
        ref = F.relu(ref)
    if residual is not None and not resid_first:
        ref = ref + rsum
    chain = (3 if block_n > 128 else 1) * taps * k_tap // 16
    gamma = mma_gamma(16 * chain) + chain * 2.0 ** -25 + 2.0 ** -21
    bound = SPLIT_REL * (ref.abs() + rsum.abs()) + (1.1 if act == 'silu' else 1.0) * gamma * absref + 1e-30
    return ref, bound


# ---------------------------------------------------------------------------------------------------- split16 format, aux kernels
SPLIT_OUT_REL = 2.0 ** -22  # hi + lo of an fp32 value keeps ~22 bits: |lo| <= 2^-11 |x|, rounded to 11 bits
SPLIT_OUT_ABS = 2.0 ** -25  # ... and where lo is an fp16 subnormal (spacing 2^-24) it is off by up to half a spacing


def split16(x):
    """The split16 format of fp32 values x (any shape, on any device) -> (hi, lo) fp16: hi = fp16_rn(sat(x)), lo = fp16_rn(sat(x - hi)),
    sat = saturate to +-65504 (NaN stays NaN): csrc/internal.h split_pair, DESIGN.md 2."""
    x = x.float()
    hi = x.clamp(-65504.0, 65504.0).half()
    lo = (x - hi.float()).clamp(-65504.0, 65504.0).half()
    return hi, lo


def split_out_bound(ref):
    """Rounding of an fp32 result to the split16 output format, element-wise."""
    return SPLIT_OUT_REL * ref.abs() + SPLIT_OUT_ABS


def gamma_n(n):
    """gamma_n = n u / (1 - n u), u = 2^-24: bound on the relative error of n chained fp32 roundings (Higham, Accuracy and Stability of
    Numerical Algorithms, lemma 3.1)."""
    return n * U24 / (1 - n * U24)


def groupnorm_reference(x64, groups, gamma, beta, eps, relu):
    """float64 GroupNorm (8 channels per group) of x64 [B, C, H, W] and the element-wise bound of csrc/aux_kernels.cu gn_stats / gn_apply
    -> (ref, bound).  From the kernels' arithmetic (u = 2^-24):
      the statistics sum x - pivot (pivot: the group's first channel at pixel 0) in fp32 over <= 64 values (+ the pivot subtraction and
      the square), then in double:  e_sum = 68 u mean|x - pivot|,  e_mean = e_sum + u |mean|  (fp32 mean),
      e_var = 68 u mean (x - pivot)^2 + 2 |mean - pivot| e_sum
      apply: |gamma| (|x - mean| rstd (e_var / (2 (var + eps)) + 2 u) + rstd e_mean) + 4 u (|gamma| rstd |x - mean| + |beta|)
      hi / lo fp16 output: split_out_bound."""
    B = x64.shape[0]
    u = U24
    g64, b64 = gamma.double()[None, :, None, None], beta.double()[None, :, None, None]
    ref = F.group_norm(x64, groups, g64.flatten(), b64.flatten(), eps)
    if relu:
        ref = F.relu(ref)
    xg = x64.reshape(B, groups, -1)
    d = xg - x64[:, ::8, 0, 0][..., None]
    mean, var = xg.mean(-1), xg.var(-1, unbiased=False)
    e_sum = 68 * u * d.abs().mean(-1)
    e_mean = e_sum + u * mean.abs()
    e_var = 68 * u * (d * d).mean(-1) + 2 * d.mean(-1).abs() * e_sum
    rstd = 1 / torch.sqrt(var + eps)

    def per_channel(s):
        return s.repeat_interleave(8, dim=1)[:, :, None, None]
    xm = (x64 - per_channel(mean)).abs()
    bound = (g64.abs() * (xm * per_channel(rstd * (e_var / (2 * (var + eps)) + 2 * u)) + per_channel(rstd * e_mean))
             + 4 * u * (g64.abs() * per_channel(rstd) * xm + b64.abs()) + split_out_bound(ref))
    return ref, bound


def max_rel(out, ref):
    """max |out - ref| / max |ref| (NaN if out has a NaN)."""
    out = out.double().to(ref.device)
    return float((out - ref).abs().max() / ref.abs().max().clamp_min(1e-300))


def check_conv(out, ref, bound, what):
    """The two checks of a conv output against split_conv_reference: (a) element-wise bound, (b) max |out - ref| / max |ref| within the
    single-layer budget.  (b) is the tighter one on deep-K layers, (a) on small outputs.  Returns max |out - ref| / bound."""
    r = check(out, ref, bound, what)
    e = max_rel(out, ref)
    assert e < LAYER_BUDGET, f'{what}: max|out - ref| / max|ref| = {e:.3g} exceeds {LAYER_BUDGET}'
    return r


def check(out, ref, bound, what):
    """Asserts |out - ref| <= bound element-wise (tensors of one shape; out is cast to float64) and returns max |out - ref| / bound.
    On failure the message names the worst element: index, value, reference and bound."""
    out = out.detach().double().to(ref.device)
    assert out.shape == ref.shape, (what, tuple(out.shape), tuple(ref.shape))
    err = (out - ref).abs()
    ratio = err / bound.clamp_min(1e-300)
    worst = int(torch.argmax(ratio.flatten()))
    r = float(ratio.flatten()[worst])
    if not (r <= 1.0):
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(worst), ref.shape))
        raise AssertionError(f'{what}: |out - ref| exceeds the bound {r:.3g}x at {idx}: out={float(out[idx]):.9g} ref={float(ref[idx]):.9g} '
                             f'bound={float(bound[idx]):.3g} ({int((ratio > 1).sum())} of {ratio.numel()} elements over)')
    return r
