"""float64 references and an element-wise error bound for the training kernels (tests/test_train_gpu.py).

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
    """Restates cvb_train_conv_wgrad's launch: -> (m_tiles, splits, per), `per` = 128-pixel tiles one CTA accumulates before its atomics."""
    tw, th, nb = choose_box128(B, Ho, Wo)
    m_tiles = -(-Wo // tw) * -(-Ho // th) * -(-B // nb)
    npan = 4 if (cout // 64) % 4 == 0 else (2 if (cout // 64) % 2 == 0 else 1)
    splits = (2 * sms) // (k * k * -(-cin // 128) * (cout // (64 * npan)))
    splits = min(max(splits, 1), m_tiles)
    return m_tiles, splits, -(-m_tiles // splits)


def wgrad_gamma(B, Ho, Wo, cin, cout, k, sms):
    """One CTA chains 8 MMAs (K = 16 pixels each) per tile it owns; `splits` CTAs then add their partial sums with fp32 atomics."""
    _, splits, per = wgrad_split(B, Ho, Wo, cin, cout, k, sms)
    return (8 * per + 16 + splits) * U23


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
