"""The inference path's pooling, resize, normalisation, layout and decode kernels (csrc/aux_kernels.cu, the YOLOX / FCOS decodes of
csrc/nms.cu) against float64, element by element, at the shapes and views where such kernels go wrong: channel slices of wider buffers,
partial 32-channel slabs, widths that end a pixel group or a tile partway, dilations past the map, grids that loop, ties, and the ends of
the split16 range.

Every reference is computed in float64 on exactly the values the kernel reads (hi + lo for split16 inputs).  Exact operations
(permutations, maxima, format conversion) are checked bit for bit; the rest against |out - ref| <= bound element-wise, with the bound
derived beside each test from the kernel's own operation order (u = 2^-24, fp64ref.gamma_n(n) for n chained roundings, and
fp64ref.split_out_bound for the rounding to the split16 output).  Outputs are written into a channel slice of a wider buffer filled with
NaN, and everything outside the slice must still be NaN afterwards.
"""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import fp64ref  # noqa: E402
from fp64ref import U24, gamma_n, split_out_bound  # noqa: E402

NAN = float('nan')
SPECIALS = [0.0, -0.0, 1e-6, -1e-6, 1e-9, -1e-9, 65504.0, -65504.0, 65520.0, -65520.0, 1e5, -1e5, float('inf'), float('-inf'), NAN]


def _ops():
    from cvpytorch_b200 import ops
    return ops


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def _bits(t):
    return t.contiguous().view({torch.float16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}[t.dtype])


def _assert_same_bits(a, b, what):
    """a and b equal bit for bit, except that any NaN matches any NaN."""
    an, bn = torch.isnan(a), torch.isnan(b)
    assert torch.equal(an, bn), f'{what}: NaN positions differ ({int((an != bn).sum())} elements)'
    ok = (_bits(a) == _bits(b)) | an
    assert bool(ok.all()), f'{what}: {int((~ok).sum())} of {ok.numel()} elements differ in their bits'


def _split_buf(B, H, W, C, c0=8, extra=8):
    """SplitTensor [2, B, H, W, c0 + C + extra] filled with NaN, and its channel slice [c0, c0 + C)."""
    t = _ops().SplitTensor(B, H, W, c0 + C + extra)
    t.data.fill_(NAN)
    return t, t.view(c0, C)


def _put_split(t, c0, x_nhwc):
    """Stores fp32 NHWC values into channels [c0, c0 + C) of t in the split16 format; returns the float64 values the kernels read."""
    hi, lo = fp64ref.split16(x_nhwc)
    C = x_nhwc.shape[-1]
    t.data[0, ..., c0:c0 + C] = hi
    t.data[1, ..., c0:c0 + C] = lo
    return hi.double() + lo.double()


def _get64(t, c0, C):
    return t.data[0, ..., c0:c0 + C].double() + t.data[1, ..., c0:c0 + C].double()


def _assert_outside_nan(data, c0, C, what):
    """Every element of the last dimension outside [c0, c0 + C) is still the NaN sentinel."""
    assert bool(torch.isnan(data[..., :c0]).all()) and bool(torch.isnan(data[..., c0 + C:]).all()), f'{what}: wrote outside its channel slice'


def _check(out, ref, bound, what):
    r = fp64ref.check(out, ref, bound, what)
    print(f'{what}: worst error / bound {r:.3f}')
    return r


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


# ---------------------------------------------------------------------------------------------------- format and layout
def _special_input(B, C, H, W, seed):
    g = _gen(seed)
    x = torch.randn(B, C, H, W, device='cuda', generator=g) * 10
    sp = torch.tensor(SPECIALS, device='cuda')
    pick = torch.rand(B, C, H, W, device='cuda', generator=g) < 0.5
    idx = torch.randint(0, len(SPECIALS), (B, C, H, W), device='cuda', generator=g)
    return torch.where(pick, sp[idx], x)


@pytest.mark.parametrize('C', [3, 8, 40, 85])
@pytest.mark.parametrize('W', [1, 31, 33])
def test_split_format_and_layout_adapters(cuda, C, W):
    """nchw_to_split, split_to_nchw, split_to_f32 and f32nhwc_to_nchw, all bit-exact: hi = fp16_rn(sat(x)), lo = fp16_rn(sat(x - hi)),
    and the read-back is hi.float() + lo.float() (one fp32 addition, the same in torch), on ±0, fp16 subnormals, ±65504, ±65520, ±1e5,
    ±inf and NaN, through channel slices on both sides."""
    ops = _ops()
    B, H = 2, 3
    x = _special_input(B, C, H, W, seed=C * 100 + W)
    t, v = _split_buf(B, H, W, C)
    ops.nchw_to_split(x, v)
    hi, lo = fp64ref.split16(_nhwc(x))
    _assert_same_bits(t.data[0, ..., 8:8 + C], hi, f'nchw_to_split hi C={C} W={W}')
    _assert_same_bits(t.data[1, ..., 8:8 + C], lo, f'nchw_to_split lo C={C} W={W}')
    _assert_outside_nan(t.data, 8, C, 'nchw_to_split')
    # values the format must keep: |x| <= 65504 to 2^-22 relative, up to 131008 through lo, beyond that and inf saturate, NaN stays NaN
    val = hi.float() + lo.float()
    xs = _nhwc(x)
    assert bool(torch.isnan(val).eq(torch.isnan(xs)).all())
    fin = xs.abs() <= 65504
    assert bool(((val - xs).abs() <= split_out_bound(xs).float())[fin].all())
    assert bool((val[xs == 65520] == 65520).all()) and bool((val[xs == 1e5] == 1e5).all())
    assert bool((val[xs == float('inf')] == 131008).all()) and bool((val[xs == float('-inf')] == -131008).all())
    # split16 -> NCHW fp32 from the slice
    out = ops.split_to_nchw(v)
    _assert_same_bits(out, _nchw(val), f'split_to_nchw C={C} W={W}')
    # split16 -> fp32 NHWC slice (8-channel vectors only)
    if C % 8 == 0:
        f = ops.F32Tensor(B, H, W, C + 16)
        f.data.fill_(NAN)
        ops.split_to_f32(v, f.view(8, C))
        _assert_same_bits(f.data[..., 8:8 + C], val, f'split_to_f32 C={C} W={W}')
        _assert_outside_nan(f.data, 8, C, 'split_to_f32')
    # fp32 NHWC slice -> NCHW
    f = ops.F32Tensor(B, H, W, C + 8)
    f.data.copy_(torch.randn(B, H, W, C + 8, device='cuda', generator=_gen(W)))
    f.data[..., 4:4 + C] = xs
    _assert_same_bits(ops.f32nhwc_to_nchw(f.view(4, C)), x, f'f32nhwc_to_nchw C={C} W={W}')


def test_layout_adapters_beyond_65535_image_rows(cuda):
    """B * H = 70 000 image rows (more than the launch grid's z limit of 65535) with W = 1, C = 8."""
    ops = _ops()
    B, C, H, W = 2, 8, 35000, 1
    x = torch.randn(B, C, H, W, device='cuda', generator=_gen(7))
    t, v = _split_buf(B, H, W, C)
    ops.nchw_to_split(x, v)
    hi, lo = fp64ref.split16(_nhwc(x))
    _assert_same_bits(t.data[0, ..., 8:8 + C], hi, 'nchw_to_split hi, 70000 rows')
    _assert_same_bits(t.data[1, ..., 8:8 + C], lo, 'nchw_to_split lo, 70000 rows')
    _assert_outside_nan(t.data, 8, C, 'nchw_to_split, 70000 rows')
    val = hi.float() + lo.float()
    _assert_same_bits(ops.split_to_nchw(v), _nchw(val), 'split_to_nchw, 70000 rows')
    f = ops.F32Tensor(B, H, W, C + 8)
    f.data[..., 4:4 + C] = val
    _assert_same_bits(ops.f32nhwc_to_nchw(f.view(4, C)), _nchw(val), 'f32nhwc_to_nchw, 70000 rows')


# ---------------------------------------------------------------------------------------------------- stem space-to-depth
def _s2d_reference(x):
    """[B, 3, H, W] -> [B, H/2, W/2, 16]: channel (dy * 2 + dx) * 3 + c holds x[b, c, 2 h2 + dy, 2 w2 + dx]; channels 12..15 are zero."""
    B, _, H, W = x.shape
    v = x.view(B, 3, H // 2, 2, W // 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(B, H // 2, W // 2, 12)
    return torch.cat([v, torch.zeros(B, H // 2, W // 2, 4, device=x.device)], -1)


@pytest.mark.parametrize('B,H,W', [(2, 6, 10), (1, 2, 2), (2, 1536, 1536)])
@pytest.mark.parametrize('pad_left', [0, 1, 2])
def test_stem_s2d(cuda, B, H, W, pad_left):
    """fp32 stem: bit-exact against the restated 2x2 space-to-depth, in a row-window layout whose pad columns stay untouched.
    2 x 1536^2 has more output pixels than the capped grid (132 * 32 CTAs of 256 threads), so the grid-stride loop runs twice."""
    if W > 64 and pad_left == 1:
        pytest.skip('the large map runs at pad_left 0 and 2')
    ops = _ops()
    x = torch.randn(B, 3, H, W, device='cuda', generator=_gen(H + pad_left)) * 3
    x[0, 0, 0, 0] = 70000.0  # saturates into lo
    Wd = W // 2 + pad_left + 2
    t = ops.SplitTensor(B, H // 2, Wd, 16)
    t.data.fill_(NAN)
    ops.stem_s2d(x, t.view(), pad_left=pad_left)
    hi, lo = fp64ref.split16(_s2d_reference(x))
    cols = slice(pad_left, pad_left + W // 2)
    _assert_same_bits(t.data[0, :, :, cols], hi, f'stem_s2d hi {B}x{H}x{W} pad {pad_left}')
    _assert_same_bits(t.data[1, :, :, cols], lo, f'stem_s2d lo {B}x{H}x{W} pad {pad_left}')
    assert bool(torch.isnan(t.data[:, :, :, :pad_left]).all()) and bool(torch.isnan(t.data[:, :, :, pad_left + W // 2:]).all()), \
        'stem_s2d wrote into the pad columns'


def test_stem_s2d_u8_unaligned_frame_no_channel_reversal(cuda):
    """u8 stem with reverse_channels=False on a frame that starts 2 bytes into its allocation: a W % 4 == 0 frame then takes the
    one-pixel-per-thread path.  Bit-exact against the fp32 stem on the reference's ToTensor + Normalize of the same frame."""
    from oracle import yolov5_oracle as YO
    ops = _ops()
    B, H, W = 2, 10, 24
    n = B * H * W * 3
    g = torch.Generator().manual_seed(11)
    buf = torch.randint(0, 256, (n + 4,), dtype=torch.uint8, generator=g).cuda()
    frame = buf[2:2 + n].view(B, H, W, 3)
    assert frame.data_ptr() % 4 == 2 and frame.is_contiguous()
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    x = YO.input_transform(frame.cpu(), mean, std, reverse_channels=False).cuda()
    for pad_left in (0, 1):
        a, b = ops.SplitTensor(B, H // 2, W // 2 + 3 * pad_left, 16), ops.SplitTensor(B, H // 2, W // 2 + 3 * pad_left, 16)
        b.data.fill_(NAN)
        ops.stem_s2d(x, a.view(), pad_left=pad_left)
        ops.stem_s2d(frame, b.view(), pad_left=pad_left, norm=dict(mean=mean, std=std, reverse_channels=False))
        cols = slice(pad_left, pad_left + W // 2)
        _assert_same_bits(b.data[:, :, :, cols], a.data[:, :, :, cols], f'stem_s2d_u8 pad {pad_left}')
        assert bool(torch.isnan(b.data[:, :, :, :pad_left]).all()) and bool(torch.isnan(b.data[:, :, :, pad_left + W // 2:]).all())


# ---------------------------------------------------------------------------------------------------- max pools
@pytest.mark.parametrize('H', [1, 2, 3, 4, 5, 37])
@pytest.mark.parametrize('W', [1, 2, 3, 4, 5, 37])
def test_maxpool3x3s2(cuda, H, W):
    """Exact against F.max_pool2d(3, 2, 1) in float64; where the maximum is unique the output's hi and lo words are the source element's;
    a NaN in a window gives NaN.  C in {8, 24, 64}; input and output are channel slices."""
    ops = _ops()
    B = 2
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    for C in (8, 24, 64):
        tin, vin = _split_buf(B, H, W, C)
        x = _put_split(tin, 8, torch.randn(B, H, W, C, device='cuda', generator=_gen(H * 64 + W + C)) * 5)
        ref, idx = F.max_pool2d(_nchw(x), 3, 2, 1, return_indices=True)
        tout, vout = _split_buf(B, Ho, Wo, C, c0=16)
        ops.maxpool3x3s2(vin, vout)
        _assert_same_bits(_get64(tout, 16, C), _nhwc(ref), f'maxpool3x3s2 {H}x{W} C={C}')
        _assert_outside_nan(tout.data, 16, C, f'maxpool3x3s2 {H}x{W} C={C}')
        # hi / lo words of the selected element (random values: every maximum is unique)
        for plane in (0, 1):
            src = _nchw(tin.data[plane, ..., 8:8 + C]).reshape(B, C, H * W)
            sel = torch.gather(src, 2, idx.reshape(B, C, -1)).reshape(B, C, Ho, Wo)
            _assert_same_bits(_nchw(tout.data[plane, ..., 16:16 + C]), sel, f'maxpool3x3s2 {H}x{W} C={C} plane {plane}')
        # NaN propagation: a NaN (in hi) anywhere in a window wins over any finite value before or after it
        tin.data[0, 0, H // 2, W // 2, 8] = NAN
        tin.data[0, 1, H - 1, 0, 8 + C - 1] = NAN
        x = _get64(tin, 8, C)
        ops.maxpool3x3s2(vin, vout)
        _assert_same_bits(_get64(tout, 16, C), _nhwc(F.max_pool2d(_nchw(x), 3, 2, 1)), f'maxpool3x3s2 {H}x{W} C={C} with NaN')
    # an all -inf window gives -inf
    tin, vin = _split_buf(1, H, W, 8)
    tin.data[0, ..., 8:16] = float('-inf')
    tin.data[1, ..., 8:16] = 0
    tout, vout = _split_buf(1, Ho, Wo, 8)
    ops.maxpool3x3s2(vin, vout)
    assert bool((_get64(tout, 8, 8) == float('-inf')).all())


def _pool5(x):
    return F.max_pool2d(x, 5, 1, 2)


@pytest.mark.parametrize('H,W', [(1, 1), (1, 9), (9, 1), (20, 20), (40, 80)])
@pytest.mark.parametrize('C', [8, 24])
def test_sppf_pool(cuda, H, W, C):
    """Exact against three chained F.max_pool2d(5, 1, 2) in float64, with x, y1, y2, y3 slices of one concat buffer (plus 8 sentinel
    channels); a NaN propagates.  40 x 80 = 3200 pixels is the largest map the shared-memory kernel takes."""
    ops = _ops()
    B = 2
    t, _ = _split_buf(B, H, W, 4 * C, c0=0)
    vx, v1, v2, v3 = (t.view(i * C, C) for i in range(4))
    for with_nan in (False, True):
        x = torch.randn(B, H, W, C, device='cuda', generator=_gen(H * 100 + W + C)) * 4
        if with_nan:
            x[0, H // 2, W - 1, 3] = NAN
            x[1, 0, 0, C - 1] = NAN
        x64 = _put_split(t, 0, x)
        t.data[:, ..., C:] = NAN
        ops.sppf_pool(vx, v1, v2, v3)
        p = _nchw(x64)
        for i, name in ((1, 'y1'), (2, 'y2'), (3, 'y3')):
            p = _pool5(p)
            _assert_same_bits(_get64(t, i * C, C), _nhwc(p), f'sppf {name} {H}x{W} C={C} nan={with_nan}')
        _assert_outside_nan(t.data, 0, 4 * C, f'sppf {H}x{W}')


def test_sppf_pool_rejects_map_above_shared_memory(cuda):
    from cvpytorch_b200._lib import CvbError
    ops = _ops()
    t, _ = _split_buf(1, 40, 81, 32, c0=0)
    with pytest.raises(CvbError):
        ops.sppf_pool(t.view(0, 8), t.view(8, 8), t.view(16, 8), t.view(24, 8))


# ---------------------------------------------------------------------------------------------------- depthwise 3x3
def _dw_case(B, H, W, C, dil, relu, seed):
    """Input slice c0 = 8 of a C + 16 buffer, output slice c0 = 16 of a C + 24 buffer (DeepLab's cat2 -> d0)."""
    ops = _ops()
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(C, 1, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(C, generator=g, dtype=torch.float64)
    w9c, bias = ops.pack_dw_weights(w, b)
    tin, vin = _split_buf(B, H, W, C)
    x = _put_split(tin, 8, torch.randn(B, H, W, C, device='cuda', generator=_gen(seed)) * 2)
    tout, vout = _split_buf(B, H, W, C, c0=16)
    ops.dwconv3x3(vin, w9c, bias, dil, vout, relu)
    # float64 reference on the fp32 weights / bias the kernel reads.  The kernel chains the (at most) nine taps with fmaf from the bias:
    # nine roundings, so |acc - ref| <= gamma_9 (|b| + sum |x w|) < 10 u (|b| + sum |x w|); ReLU does not increase it; then the split16 store.
    wk = w9c.double().t().reshape(C, 1, 3, 3)
    bk = bias.double()
    xn = _nchw(x)
    ref = F.conv2d(xn, wk, bk, 1, dil, dil, groups=C)
    absref = F.conv2d(xn.abs(), wk.abs(), bk.abs(), 1, dil, dil, groups=C)
    if relu:
        ref = F.relu(ref)
    bound = 10 * U24 * absref + split_out_bound(ref)
    what = f'dwconv3x3 {B}x{H}x{W} C={C} dil={dil} relu={relu}'
    _check(_nchw(_get64(tout, 16, C)), ref, bound, what)
    _assert_outside_nan(tout.data, 16, C, what)


@pytest.mark.parametrize('W', [1, 2, 3, 4, 5, 31, 32, 33, 65])
@pytest.mark.parametrize('dil', [1, 2, 6, 12, 24, 'max'])
def test_dwconv3x3(cuda, W, dil):
    """Both kernels (dilation 1: four pixels per thread, 32-column tiles; otherwise one pixel per thread) at widths that end a pixel
    group or a tile partway, H in {1, 7, 8, 9}, C in {8, 24, 40} (partial 32-channel slabs), and dilation >= max(H, W), where every
    off-centre tap is padding."""
    for i, H in enumerate((1, 7, 8, 9)):
        C = (8, 24, 40)[(i + W) % 3]
        d = max(H, W) if dil == 'max' else dil
        _dw_case(2, H, W, C, d, relu=(i % 2 == 0), seed=W * 1000 + i * 10 + (0 if dil == 'max' else dil))


@pytest.mark.parametrize('dil', [1, 2, 12])
def test_dwconv3x3_576_channels(cuda, dil):
    _dw_case(2, 9, 33, 576, dil, relu=False, seed=576 + dil)
    _dw_case(1, 17, 65, 576, dil, relu=True, seed=577 + dil)


# ---------------------------------------------------------------------------------------------------- global average pool
@pytest.mark.parametrize('H,W', [(1, 1), (1, 7), (15, 17), (16, 16), (1, 257), (64, 128), (128, 256)])
@pytest.mark.parametrize('shift', [0.0, 100.0])
def test_global_avgpool(cuda, H, W, shift):
    """npix in {1, 7, 255, 256, 257, 64*128, 128*256}; shift 100 gives inputs whose mean is 100x their spread.  Output: a [B,1,1,C] slice.
    Bound from the kernel's order: each of the 256 threads sums k = ceil(npix / 256) terms in sequence from 0 (k - 1 roundings), an
    8-level tree adds the partials (8 more roundings on every term), then one division by npix:
        |out - mean| <= gamma_(k+7) mean|x| + u |mean| + split16 store."""
    ops = _ops()
    B, C = 2, 24
    npix = H * W
    tin, vin = _split_buf(B, H, W, C)
    x = _put_split(tin, 8, torch.randn(B, H, W, C, device='cuda', generator=_gen(npix)) + shift)
    tout, vout = _split_buf(B, 1, 1, C)
    ops.global_avgpool(vin, vout)
    ref = x.mean((1, 2), keepdim=True)
    k = -(-npix // 256)
    bound = gamma_n(k + 7) * x.abs().mean((1, 2), keepdim=True) + U24 * ref.abs() + split_out_bound(ref)
    what = f'global_avgpool {H}x{W} shift {shift:g}'
    _check(_get64(tout, 8, C), ref, bound, what)
    _assert_outside_nan(tout.data, 8, C, what)


# ---------------------------------------------------------------------------------------------------- bilinear resize / upsample + argmax
def _bilinear_src(n_out, n_in):
    """Restates csrc/aux_kernels.cu bilinear_src in fp32: scale = in / out (fp32 division), s = max(fma(d + 0.5, scale, -0.5), 0) (the
    fused multiply-add is exact in float64 and rounded once to fp32), i0 = min(trunc(s), in - 1), i1 = min(i0 + 1, in - 1),
    l1 = s - i0 (exact).  -> (i0, i1, l1 fp32), on the GPU."""
    scale = float(torch.tensor(float(n_in), dtype=torch.float32) / torch.tensor(float(n_out), dtype=torch.float32))
    d = torch.arange(n_out, dtype=torch.float64, device='cuda')
    s = ((d + 0.5) * scale - 0.5).clamp_min(0.0).float()
    i0 = s.long().clamp_max(n_in - 1)
    i1 = (i0 + 1).clamp_max(n_in - 1)
    return i0, i1, s - i0.float()


def _bilinear_terms(x, Ho, Wo):
    """x [B, Hi, Wi, C] (any dtype) -> the kernel's four fp32 corner weights and corner values, [4, B, Ho, Wo, C] each, in float64."""
    Hi, Wi = x.shape[1], x.shape[2]
    h0, h1, lh = _bilinear_src(Ho, Hi)
    w0, w1, lw = _bilinear_src(Wo, Wi)
    lh, lw = lh[:, None], lw[None, :]
    one = torch.ones((), dtype=torch.float32, device='cuda')
    wts = [(one - lh) * (one - lw), (one - lh) * lw, lh * (one - lw), lh * lw]  # fp32 products, as in the kernel
    corners = [(h0, w0), (h0, w1), (h1, w0), (h1, w1)]
    vals = [x[:, hh][:, :, ww] for hh, ww in corners]
    return torch.stack([w.double()[None, :, :, None].expand_as(vals[0]) for w in wts]), torch.stack([v.double() for v in vals])


@pytest.mark.parametrize('Hi,Wi,Ho,Wo', [(8, 8, 16, 16), (8, 8, 32, 32), (5, 7, 40, 56), (37, 51, 51, 37), (51, 37, 37, 51),
                                         (64, 64, 7, 7), (1, 1, 9, 13), (9, 13, 1, 1), (13, 17, 13, 17)])
@pytest.mark.parametrize('C', [8, 40])
def test_bilinear_resize(cuda, Hi, Wi, Ho, Wo, C):
    """x2 / x4 / x8 up, 37 <-> 51, 64 -> 7, the 1 -> N broadcast of the image-pool branch, N -> 1, identity.  Source: slice c0 = 8; destination:
    slice c0 = C of a 2C + 8 buffer, like DeepLab's cat.  Reference: the kernel's fp32 corner weights (restated) times the values, summed
    in float64; the kernel accumulates the four products with fmaf from 0: four roundings, gamma_4 sum |w x|, then the split16 store."""
    ops = _ops()
    B = 2
    tin, vin = _split_buf(B, Hi, Wi, C)
    x = _put_split(tin, 8, torch.randn(B, Hi, Wi, C, device='cuda', generator=_gen(Hi * Wo + C)) * 3)
    tout = ops.SplitTensor(B, Ho, Wo, 2 * C + 8)
    tout.data.fill_(NAN)
    ops.bilinear_resize(vin, tout.view(C, C))
    out = _get64(tout, C, C)
    wts, vals = _bilinear_terms(x, Ho, Wo)
    ref = (wts * vals).sum(0)
    bound = gamma_n(4) * (wts * vals).abs().sum(0) + split_out_bound(ref)
    what = f'bilinear_resize {Hi}x{Wi}->{Ho}x{Wo} C={C}'
    _check(out, ref, bound, what)
    _assert_outside_nan(tout.data, C, C, what)
    # second opinion: PyTorch's own float64 interpolation.  Its source coordinate s is exact; the kernel's is rounded twice in fp32 (the
    # scale in / out and the fused multiply-add), up to 2^-23 s each way, which moves a value by up to that times the change between two
    # neighbouring inputs (<= 2 max|x|) per axis: max|out - ip| / max|x| <= 4 * 2^-23 * max(Hi, Wi) * 2 axes, plus the 2e-6 of the
    # kernel's own arithmetic.  (For integer ratios the scale is exact and this is far from tight.)
    ip = F.interpolate(_nchw(x), size=(Ho, Wo), mode='bilinear', align_corners=False)
    assert fp64ref.max_rel(_nchw(out), ip) < 2e-6 + 8 * 2.0 ** -23 * max(Hi, Wi), what
    if (Hi, Wi) == (Ho, Wo):
        assert torch.equal(out, x), 'identity resize must reproduce its input exactly'


@pytest.mark.parametrize('nc', [1, 2, 3, 4, 5, 19, 33])
@pytest.mark.parametrize('wide', [False, True])
def test_upsample_argmax(cuda, nc, wide):
    """Label = float64 argmax of the upsampled logits wherever the top-2 gap exceeds both values' bounds (the kernel's fp32 corner weights,
    four products summed: gamma_4 sum |w q| each).  Exact ties pick the lower class: class 1 repeats class 0's logits (a pair 1 apart)
    and class 6 repeats class 2's (4 apart: across a float4 step of the kernel's class loop).  Pitch round4(nc), or wider; every pad lane
    holds NaN and must be ignored.  Wo in {1, 255, 256, 257, 600} and one downsampling case."""
    ops = _ops()
    B = 2
    pitch = (nc + 3) // 4 * 4 + (8 if wide else 0)
    ties = [(0, 1)] if nc >= 2 else []
    if nc >= 7:
        ties.append((2, 6))
    cases = [(6, 9, 13, Wo) for Wo in (1, 255, 256, 257, 600)] + [(20, 640, 7, 257)]
    tie_hits = 0
    for (Hi, Wi, Ho, Wo) in cases:
        lg = ops.F32Tensor(B, Hi, Wi, pitch)
        lg.data.fill_(NAN)
        q = torch.randn(B, Hi, Wi, nc, device='cuda', generator=_gen(nc * 1000 + Wo + Wi)) * 2
        for lo_c, hi_c in ties:
            q[..., lo_c] += 2.0
            q[..., hi_c] = q[..., lo_c]
        lg.data[..., :nc] = q
        labels = torch.full((B, Ho, Wo), -1, dtype=torch.int64, device='cuda')
        ops.upsample_argmax(lg.view(0, nc), nc, labels)
        wts, vals = _bilinear_terms(q, Ho, Wo)
        ref = (wts * vals).sum(0)                       # [B, Ho, Wo, nc]
        bnd = gamma_n(4) * (wts * vals).abs().sum(0)
        best = ref.max(-1, keepdim=True).values
        arg = ref.argmax(-1)                            # first maximum: the lower class of an exact tie
        second = torch.where(ref == best, torch.full_like(ref, float('-inf')), ref).max(-1).values
        decided = (best[..., 0] - second) > 2 * bnd.max(-1).values
        what = f'upsample_argmax nc={nc} pitch={pitch} {Hi}x{Wi}->{Ho}x{Wo}'
        assert bool((labels >= 0).all() & (labels < nc).all()), what
        bad = decided & (labels != arg)
        assert not bool(bad.any()), f'{what}: {int(bad.sum())} labels differ from the float64 argmax where the gap exceeds the bound'
        print(f'{what}: {float(decided.float().mean()):.4f} of the pixels decided')
        for lo_c, _ in ties:
            tie_hits += int((decided & (arg == lo_c)).sum())
    if ties:
        assert tie_hits > 0, 'no decided pixel had a tied pair as its maximum'


# ---------------------------------------------------------------------------------------------------- GroupNorm
@pytest.mark.parametrize('groups', [1, 3, 12, 64, 300])
@pytest.mark.parametrize('H,W', [(1, 1), (1, 2), (7, 1), (13, 17), (100, 136)])
def test_groupnorm(cuda, groups, H, W):
    """GroupNorm without ReLU against float64 (bound: fp64ref.groupnorm_reference).  300 groups is more than 256, which launches the
    statistics kernel with one thread per group.  Image 0's group 0 is constant (var = 0, rstd = 1 / sqrt(eps)).  Slices in and out."""
    ops = _ops()
    B = 1 if groups * H * W > 64 * 100 * 136 else 2
    C = groups * 8
    g = _gen(groups * 7 + H * W)
    x = (torch.randn(B, H, W, C, device='cuda', generator=g) + 10) * 3
    x[0, ..., :8] = 3.0
    tin, vin = _split_buf(B, H, W, C)
    x64 = _put_split(tin, 8, x)
    gamma, beta = torch.rand(C, device='cuda', generator=g) + 0.5, torch.randn(C, device='cuda', generator=g)
    tout, vout = _split_buf(B, H, W, C, c0=16)
    ops.groupnorm_relu(vin, groups, gamma, beta, 1e-5, vout, ops.GroupNormWorkspace(B, groups), relu=False)
    ref, bound = fp64ref.groupnorm_reference(_nchw(x64), groups, gamma, beta, 1e-5, relu=False)
    what = f'groupnorm {B}x{H}x{W} groups={groups}'
    _check(_nchw(_get64(tout, 16, C)), ref, bound, what)
    _assert_outside_nan(tout.data, 16, C, what)


# ---------------------------------------------------------------------------------------------------- YOLOX / FCOS decode
def sigmoid_fast_rel_err(x):
    """Relative error of csrc/internal.h sigmoid_fast(x) = rcp.approx(1 + ex2.approx(fl(x * fl(-log2 e)))) against the exact sigmoid
    (not measured: derived).  The two roundings in the exponent t = x log2(e) move t by up to 2 u |t|, which scales 2^t by
    ln 2 * 2 u |t| = 2 u |x|; ex2.approx.ftz.f32 is within 2 ulp (2^-22 relative), 1 + e rounds once (u), rcp.approx.ftz.f32 is
    within 1 ulp (2^-23).  An error eps of e moves 1 / (1 + e) by at most eps relative.  1.001: the second-order terms."""
    return (2.0 ** -22 + 2 * U24 * x.abs() + U24 + 2.0 ** -23) * 1.001


EXPF_REL = 2.0 ** -22  # expf (full precision: the library is built without fast-math) is within 2 ulp


def _class_logits(B, H, W, nc, pitch, g):
    """Class logits in a view of pitch > nc, out to +-30, with exact ties: rows 0 mod 5 tie classes 3 and 4 (neighbouring lanes) at the top,
    rows 1 mod 5 tie c and c + 32 (one lane's stride) at the top."""
    q = torch.randn(B, H, W, nc, device='cuda', generator=g) * 3
    wide = torch.rand(B, H, W, 1, device='cuda', generator=g) < 0.3
    q = torch.where(wide, (torch.rand(B, H, W, nc, device='cuda', generator=g) * 2 - 1) * 30, q)
    rows = q.view(-1, nc)
    top = rows.max(-1).values + 0.5
    r = torch.arange(rows.shape[0], device='cuda')
    if nc >= 5:
        m = r % 5 == 0
        rows[m, 3] = top[m]
        rows[m, 4] = top[m]
    if nc >= 33:
        c = nc - 33
        m = r % 5 == 1
        rows[m, c] = top[m]
        rows[m, c + 32] = top[m]
    full = torch.full((B, H, W, pitch), NAN, device='cuda')
    full[..., :nc] = q
    return q, full


def _class_check(cls_out, q, what):
    """Class = float64 argmax of the sigmoids (first maximum on exact ties) wherever the top-2 gap exceeds twice the sigmoid bound;
    returns (best sigmoid in float64, its bound)."""
    s = torch.sigmoid(q.double())
    e = sigmoid_fast_rel_err(q.double()) * s
    best = s.max(-1, keepdim=True).values
    arg = s.argmax(-1)
    second = torch.where(s == best, torch.full_like(s, -1.0), s).max(-1).values
    decided = (best[..., 0] - second) > 2 * e.max(-1).values
    bad = decided & (cls_out != arg)
    assert not bool(bad.any()), f'{what}: {int(bad.sum())} classes differ from the float64 argmax where the gap exceeds the bound'
    print(f'{what}: {float(decided.float().mean()):.3f} of the rows decided')
    return best[..., 0], e.max(-1).values


@pytest.mark.parametrize('nc', [1, 31, 32, 33, 80, 100])
@pytest.mark.parametrize('H,W', [(1, 7), (5, 1), (4, 6)])
def test_yolox_decode(cuda, nc, H, W):
    """Every field of the candidate record against its float64 formula, B = 3, class view pitch nc + 5, candidate rows [off, off + H W) of
    a longer table whose other rows stay untouched.  Bounds (u = 2^-24):
      cx = (p0 + px) * stride: two roundings, gamma_2 (|p0| + px) stride;  w = expf(p2) * stride: (2^-22 + u) w;
      x1 = cx - w / 2 (w / 2 exact): e_cx + e_w / 2 + u |x1|;  obj = sigmoid_fast: sigmoid_fast_rel_err;
      class_conf = the largest class sigmoid: the largest class bound;  score = obj * conf: e_obj conf + obj e_conf + u score."""
    _yolox_case(nc, 3, H, W, 16.0)


def _yolox_case(nc, B, H, W, stride):
    ops = _ops()
    off = 5
    A = off + H * W + 4
    g = _gen(nc * 10 + H * W)
    ro = ops.F32Tensor(B, H, W, 8)
    ro.data.copy_(torch.randn(B, H, W, 8, device='cuda', generator=g))
    ro.data[..., 4] = (torch.rand(B, H, W, device='cuda', generator=g) * 2 - 1) * 30
    ro.data[..., 5:] = NAN
    pitch = nc + 5
    q, full = _class_logits(B, H, W, nc, pitch, g)
    cls = ops.F32Tensor(B, H, W, pitch)
    cls.data.copy_(full)
    ws = ops.YoloxWorkspace(B, A)
    ws.cand.fill_(NAN)
    ops.yolox_decode(ro.view(0, 5), cls.view(0, nc), nc, stride, ws, off)
    what = f'yolox_decode nc={nc} {B}x{H}x{W}'
    assert bool(torch.isnan(ws.cand[:, :off]).all()) and bool(torch.isnan(ws.cand[:, off + H * W:]).all()), f'{what}: wrote outside its rows'
    rec = ws.cand[:, off:off + H * W].double().view(B, H, W, 8)
    p = ro.data.double()
    px = torch.arange(W, device='cuda', dtype=torch.float64)[None, None, :].expand(B, H, W)
    py = torch.arange(H, device='cuda', dtype=torch.float64)[None, :, None].expand(B, H, W)
    cx, cy = (p[..., 0] + px) * stride, (p[..., 1] + py) * stride
    e_cx, e_cy = gamma_n(2) * (p[..., 0].abs() + px) * stride, gamma_n(2) * (p[..., 1].abs() + py) * stride
    w, h = torch.exp(p[..., 2]) * stride, torch.exp(p[..., 3]) * stride
    e_w, e_h = (EXPF_REL + U24) * w, (EXPF_REL + U24) * h
    for k, (ref, err) in enumerate([(cx - w / 2, e_cx + e_w / 2), (cy - h / 2, e_cy + e_h / 2), (cx + w / 2, e_cx + e_w / 2),
                                    (cy + h / 2, e_cy + e_h / 2)]):
        _check(rec[..., k], ref, err + U24 * ref.abs() + 1e-30, f'{what} box {k}')
    obj = torch.sigmoid(p[..., 4])
    e_obj = sigmoid_fast_rel_err(p[..., 4]) * obj
    _check(rec[..., 4], obj, e_obj, f'{what} obj')
    cls_out = rec[..., 6].long()
    assert torch.equal(rec[..., 6], cls_out.double()), what
    conf, e_conf = _class_check(cls_out, q, what)
    _check(rec[..., 5], conf, e_conf, f'{what} class_conf')
    _check(rec[..., 7], obj * conf, e_obj * conf + obj * e_conf + U24 * obj * conf * 1.001, f'{what} score')


@pytest.mark.parametrize('nc', [1, 31, 32, 33, 80, 100])
@pytest.mark.parametrize('B,H,W,stride,scale', [(3, 1, 9, 8, 0.75), (3, 6, 1, 128, 1.5), (3, 5, 7, 8, 1.0)])
def test_fcos_decode(cuda, nc, B, H, W, stride, scale):
    _fcos_case(nc, B, H, W, stride, scale)


def test_fcos_decode_more_rows_than_the_grid(cuda):
    """2 x 100 x 100 = 20 000 rows: more than the capped grid (132 * 16 CTAs of 8 warps = 16 896 rows) covers in one pass."""
    _fcos_case(80, 2, 100, 100, 8, 1.25)


def _fcos_case(nc, B, H, W, stride, scale):
    """Every field against its float64 formula; rows [off, off + H W) of a longer table, the others untouched.  Bounds (u = 2^-24):
      centre = px * stride + stride // 2: exact (small integers);  l = expf(fl(p0 * scale)): the rounded argument moves exp by u |p0 scale|
      relative, expf 2^-22: (2^-22 + u |p0 scale|) l;  x1 = cx - l: e_l + u |x1|;  cnt = sigmoid_fast;
      score = sqrtf(fl(conf * cnt)): half the relative error of the product (e_conf / conf + e_cnt / cnt + u), plus u for the sqrt;
      class = argmax + 1 (as _class_check)."""
    ops = _ops()
    off = 3
    N = off + H * W + 5
    g = _gen(nc * 10 + H * W + int(stride))
    pitch = nc + 5
    q, full = _class_logits(B, H, W, nc, pitch, g)
    cls = ops.F32Tensor(B, H, W, pitch)
    cls.data.copy_(full)
    rc = ops.F32Tensor(B, H, W, 8)
    rc.data.copy_(torch.randn(B, H, W, 8, device='cuda', generator=g))
    rc.data[..., 4] = (torch.rand(B, H, W, device='cuda', generator=g) * 2 - 1) * 30
    rc.data[..., 5:] = NAN
    ws = ops.FcosWorkspace(B, N)
    ws.scores.fill_(NAN)
    ws.boxes.fill_(NAN)
    ws.classes.fill_(-7)
    ops.fcos_decode(cls.view(0, nc), rc.view(0, 5), nc, stride, scale, ws, off)
    what = f'fcos_decode nc={nc} {B}x{H}x{W} stride {stride} scale {scale}'
    rows = slice(off, off + H * W)
    for t in (ws.scores, ws.boxes):
        assert bool(torch.isnan(t[:, :off]).all()) and bool(torch.isnan(t[:, off + H * W:]).all()), f'{what}: wrote outside its rows'
    assert bool((ws.classes[:, :off] == -7).all()) and bool((ws.classes[:, off + H * W:] == -7).all()), f'{what}: wrote outside its rows'
    p = rc.data.double()
    px = torch.arange(W, device='cuda', dtype=torch.float64)[None, None, :].expand(B, H, W)
    py = torch.arange(H, device='cuda', dtype=torch.float64)[None, :, None].expand(B, H, W)
    half = float(int(stride) // 2)
    cx, cy = px * stride + half, py * stride + half
    a = p[..., :4] * scale
    d = torch.exp(a)
    e_d = (EXPF_REL + U24 * a.abs()) * d
    box = ws.boxes[:, rows].double().view(B, H, W, 4)
    for k, ref in enumerate([cx - d[..., 0], cy - d[..., 1], cx + d[..., 2], cy + d[..., 3]]):
        _check(box[..., k], ref, e_d[..., k] + U24 * ref.abs() + 1e-30, f'{what} box {k}')
    cls_out = ws.classes[:, rows].view(B, H, W).long() - 1
    conf, e_conf = _class_check(cls_out, q, what)
    cnt = torch.sigmoid(p[..., 4])
    rel = 0.5 * (e_conf / conf + sigmoid_fast_rel_err(p[..., 4]) + U24) + U24
    score = torch.sqrt(conf * cnt)
    _check(ws.scores[:, rows].double().view(B, H, W), score, rel * score * 1.001, f'{what} score')
