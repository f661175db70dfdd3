"""Parity of the fused wgmma conv kernel (through the C ABI) against a float64 conv of exactly the values it reads
(fp64ref.split_conv_reference): every element within the derived error bound, and max|a-b|/max|b| <= 2e-5
(north_star budget is 1e-3 on end-to-end logits; a single layer must sit ~50x inside it).  The stem tests compare against torch fp32
conv2d of the original 6x6 conv on the same GPU (TF32 disabled)."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fp64ref  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = fp64ref.LAYER_BUDGET


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-12))


def _run_conv(cin, cout, k, s, p, B, H, W, act='silu', residual=False, up=False, f32_out=False, block_n=0, seed=0, dil=1, no_resident=0, halo=0):
    """Runs one conv into a NaN-filled output and checks it against the float64 reference of fp64ref.split_conv_reference: element by
    element within its bound, and max|out - ref| / max|ref| (returned) within the single-layer budget."""
    from cvpytorch_b200 import ops
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cin, H, W, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g) * 0.5
    Ho = (H + 2 * p - dil * (k - 1) - 1) // s + 1
    Wo = (W + 2 * p - dil * (k - 1) - 1) // s + 1
    tin = ops.SplitTensor(B, H, W, cin)
    ops.nchw_to_split(x.cuda(), tin.view())
    wp, bp = ops.pack_conv_weights(w.double(), b.double())
    c_pitch = (cout + 7) // 8 * 8
    tout = ops.F32Tensor(B, Ho, Wo, c_pitch) if f32_out else ops.SplitTensor(B, Ho, Wo, c_pitch)
    tout.data.fill_(float('nan'))
    res_t = up_t = None
    if up:
        up_t = ops.F32Tensor(B, (Ho + 1) // 2, (Wo + 1) // 2, cout)
        up_t.data.copy_(torch.randn(B, cout, (Ho + 1) // 2, (Wo + 1) // 2, generator=g).permute(0, 2, 3, 1))
    if residual:
        res_t = ops.SplitTensor(B, Ho, Wo, cout)
        ops.nchw_to_split(torch.randn(B, cout, Ho, Wo, generator=g).cuda(), res_t.view())
    plan = ops.ConvPlan(tin.view(), tout.view(0, cout), wp, bp, k, s, p, dil, act,
                        residual=res_t.view() if res_t else None, up_partial=up_t.view() if up_t else None,
                        block_n=block_n, no_resident=no_resident, halo=halo)
    plan.run()
    torch.cuda.synchronize()
    out = fp64ref.conv_out64(tout.data[..., :cout])
    ref, bound = fp64ref.split_conv_reference(tin, wp, bp, k, s, p, dil, act, residual=res_t, up=up_t.data if up else None,
                                              block_n=block_n, cout=cout)
    what = f'conv {cin}->{cout} k{k} s{s} p{p} d{dil} B{B} {H}x{W} {act} bn{block_n} halo{halo}'
    fp64ref.check(out, ref, bound, what)
    return fp64ref.max_rel(out, ref)


def test_layout_roundtrip(cuda):
    from cvpytorch_b200 import ops
    x = torch.randn(3, 40, 17, 23, device='cuda')
    t = ops.SplitTensor(3, 17, 23, 40)
    ops.nchw_to_split(x, t.view())
    y = ops.split_to_nchw(t.view())
    assert _rel(y, x) < 1e-6
    # channel-slice view
    y2 = ops.split_to_nchw(t.view(8, 16))
    assert _rel(y2, x[:, 8:24]) < 1e-6


# (cin, cout, k, s, p, B, H, W)
BASIC = [
    (64, 64, 1, 1, 0, 2, 16, 16),      # smallest GEMM: one K chunk, one N tile
    (128, 64, 1, 1, 0, 2, 16, 16),     # two K chunks
    (64, 128, 1, 1, 0, 2, 16, 16),     # BLOCK_N 128
    (64, 256, 1, 1, 0, 1, 16, 16),     # two N tiles
    (32, 32, 1, 1, 0, 2, 16, 16),      # 64B swizzle (BLOCK_K 32), 64B-swizzled store
    (16, 32, 3, 1, 1, 2, 16, 16),      # 32B swizzle (BLOCK_K 16): the stem formulation
    (64, 64, 3, 1, 1, 2, 16, 16),      # 3x3: shifted TMA boxes, zero-fill padding
    (64, 128, 3, 2, 1, 2, 16, 16),     # stride 2: parity tensor maps
    (32, 64, 3, 2, 1, 2, 32, 32),      # stride 2, BLOCK_K 32
    (256, 256, 3, 1, 1, 2, 20, 20),    # 20x20 map: box {4,4,8}
    (512, 256, 1, 1, 0, 3, 20, 20),    # batch not a multiple of the box
    (128, 128, 3, 1, 1, 1, 40, 40),
    (64, 64, 1, 1, 0, 1, 13, 19),      # ragged map: partial tiles, TMA clipping
    (64, 64, 3, 1, 1, 1, 13, 19),
    (64, 64, 3, 2, 1, 1, 13, 19),      # odd size with stride 2
]


@pytest.mark.parametrize('cfg', BASIC, ids=lambda c: 'x'.join(map(str, c)))
def test_conv_basic(cuda, cfg):
    cin, cout, k, s, p, B, H, W = cfg
    err = _run_conv(cin, cout, k, s, p, B, H, W)
    assert err < TOL, f'rel err {err}'


def test_conv_residual(cuda):
    assert _run_conv(64, 64, 3, 1, 1, 2, 16, 16, residual=True) < TOL
    assert _run_conv(32, 32, 3, 1, 1, 2, 24, 24, residual=True) < TOL


def test_conv_upsampled_partial(cuda):
    assert _run_conv(128, 128, 1, 1, 0, 2, 16, 16, up=True) < TOL
    assert _run_conv(256, 256, 1, 1, 0, 2, 40, 40, up=True, block_n=128) < TOL


def test_conv_f32_out_and_head_shape(cuda):
    assert _run_conv(128, 255, 1, 1, 0, 2, 16, 16, act=None, f32_out=True) < TOL
    assert _run_conv(64, 128, 1, 1, 0, 2, 16, 16, act=None, f32_out=True) < TOL


def test_conv_relu_none(cuda):
    assert _run_conv(64, 64, 1, 1, 0, 2, 16, 16, act='relu') < TOL
    assert _run_conv(64, 64, 1, 1, 0, 2, 16, 16, act=None) < TOL


def test_conv_block_n_variants(cuda):
    for bn in (32, 64, 128, 256):
        assert _run_conv(64, 256, 1, 1, 0, 2, 16, 16, block_n=bn) < TOL, bn


def test_conv_many_tiles_persistent(cuda):
    # more tiles than SMs: exercises the ring buffer across tiles
    assert _run_conv(64, 64, 1, 1, 0, 8, 80, 80) < TOL
    assert _run_conv(64, 64, 3, 1, 1, 8, 80, 80) < TOL
    assert _run_conv(128, 256, 3, 2, 1, 8, 80, 80) < TOL


def test_conv_resident_weights_vs_streamed(cuda):
    """small weight slabs stay resident in smem (ring streams activations only); both modes must agree with the reference,
    including the pinned-n-tile case (tiles_n = 2 / 4) and many tiles per CTA."""
    for cfg in [(64, 64, 1, 1, 0, 8, 80, 80), (128, 128, 1, 1, 0, 4, 80, 80), (64, 256, 1, 1, 0, 4, 40, 40), (32, 32, 3, 1, 1, 2, 64, 64),
                (64, 255, 1, 1, 0, 2, 40, 40)]:
        for nr in (0, 1):
            f32 = cfg[1] == 255
            assert _run_conv(*cfg, no_resident=nr, f32_out=f32, act=None if f32 else 'silu') < TOL, (cfg, nr)
    assert _run_conv(64, 256, 1, 1, 0, 4, 40, 40, block_n=64) < TOL  # tiles_n = 4, weights pinned per CTA


def test_conv_dilated(cuda):
    assert _run_conv(64, 64, 3, 1, 2, 1, 24, 24, dil=2) < TOL


@pytest.mark.parametrize('window', [0, 4])
@pytest.mark.parametrize('shape', [(2, 64, 96), (1, 128, 136), (3, 32, 40)])
def test_stem_s2d_equals_6x6_conv(cuda, window, shape):
    """space-to-depth + 3x3 conv == the reference's 6x6/s2/p2 stem conv (yolov5_csp_darknet.py:36-45); window=4 is the
    zero-padded row-window layout (one 128-byte K chunk = 4 adjacent s2d pixels) the model graph uses."""
    from cvpytorch_b200 import ops
    g = torch.Generator().manual_seed(5)
    B, H, W = shape
    x = torch.randn(B, 3, H, W, generator=g)
    w = torch.randn(32, 3, 6, 6, generator=g) / 108 ** 0.5
    b = torch.randn(32, generator=g)
    ref = F.silu(F.conv2d(x.cuda(), w.cuda(), b.cuda(), 2, 2))
    t = ops.SplitTensor(B, H // 2, W // 2 + (3 if window else 0), 16)
    ops.stem_s2d(x.cuda().contiguous(), t.view())
    w3 = ops.stem_weights_to_s2d(w.double())
    wp, bp = ops.pack_conv_weights(ops.window_weights(w3, window) if window else w3, b.double())
    out = ops.SplitTensor(B, H // 2, W // 2, 32)
    plan = ops.ConvPlan(t.view(), out.view(), wp, bp, 3, 1, 1, 1, 'silu', w_window=window)
    plan.run()
    y = ops.split_to_nchw(out.view())
    torch.cuda.synchronize()
    assert _rel(y, ref) < TOL


def test_sppf_pool(cuda):
    from cvpytorch_b200 import ops
    x = torch.randn(3, 64, 20, 20, device='cuda')
    t = ops.SplitTensor(3, 20, 20, 256)
    ops.nchw_to_split(x, t.view(0, 64))
    ops.sppf_pool(t.view(0, 64), t.view(64, 64), t.view(128, 64), t.view(192, 64))
    y = ops.split_to_nchw(t.view())
    xr = ops.split_to_nchw(t.view(0, 64))
    y1 = F.max_pool2d(xr, 5, 1, 2)
    y2 = F.max_pool2d(y1, 5, 1, 2)
    y3 = F.max_pool2d(y2, 5, 1, 2)
    ref = torch.cat([xr, y1, y2, y3], 1)
    torch.cuda.synchronize()
    assert torch.equal(y, ref)  # max is exact on the hi+lo values


def test_conv_3x3_shapes(cuda):
    """more 3x3 / stride 1 shapes: borders, ragged maps, many K chunks (ring wrap-around), two N tiles, residual epilogue,
    more tiles than SMs"""
    assert _run_conv(32, 32, 3, 1, 1, 3, 16, 16) < TOL
    assert _run_conv(64, 64, 3, 1, 1, 2, 24, 40) < TOL
    assert _run_conv(256, 128, 3, 1, 1, 2, 32, 24, act='relu') < TOL
    assert _run_conv(128, 256, 3, 1, 1, 2, 32, 32) < TOL
    assert _run_conv(96, 64, 3, 1, 1, 1, 16, 24) < TOL
    assert _run_conv(64, 64, 3, 1, 1, 4, 160, 160, residual=True) < TOL
    assert _run_conv(32, 32, 3, 1, 1, 2, 160, 160, residual=True) < TOL
    assert _run_conv(512, 64, 3, 1, 1, 1, 16, 16) < TOL   # chain of 288 MMAs: two main accumulators (three-MMA form)


# (cin, cout, k, s, p, B, H, W) -- layers the halo (copy / tap) loader applies to: every tap is a row-shifted descriptor view of a box
# that was loaded once per K chunk including the filter halo (include/cvb200.h CvbConvDesc.halo)
HALO = [
    (32, 32, 3, 1, 1, 2, 32, 32),      # BLOCK_K 32 (64B swizzle), resident weights
    (64, 64, 3, 1, 1, 2, 32, 32),      # 128B swizzle
    (64, 64, 3, 1, 1, 3, 80, 80),      # many tiles per CTA: ring wrap-around of the A slots and the weight ring
    (128, 128, 3, 1, 1, 2, 40, 40),    # two K chunks, streamed weights, partial tiles in H (40 = 2.5 x 16)
    (256, 256, 3, 1, 1, 1, 20, 20),    # two N tiles, ragged W (20 = 2.5 x 8)
    (64, 64, 3, 1, 1, 1, 13, 19),      # ragged map
    (32, 64, 3, 2, 1, 2, 64, 64),      # stride 2: four parity maps with their own halo boxes
    (64, 128, 3, 2, 1, 2, 32, 32),
    (128, 128, 3, 2, 1, 1, 26, 38),    # stride 2, odd parity-map sizes
    (64, 64, 3, 2, 1, 1, 13, 19),
    (96, 64, 3, 1, 1, 1, 16, 24),      # cin not a multiple of 64
    (512, 64, 3, 1, 1, 1, 16, 16),     # chain of 288 MMAs: two main accumulators
]


@pytest.mark.parametrize('mode', [1, 2])
@pytest.mark.parametrize('cfg', HALO, ids=lambda c: 'x'.join(map(str, c)))
def test_conv_halo_modes(cuda, cfg, mode):
    cin, cout, k, s, p, B, H, W = cfg
    err = _run_conv(cin, cout, k, s, p, B, H, W, halo=mode)
    assert err < TOL, f'rel err {err}'
    assert _run_conv(cin, cout, k, s, p, B, H, W, halo=-1) < TOL  # classic loader on the same layer


@pytest.mark.parametrize('mode', [1, 2])
def test_conv_halo_epilogues(cuda, mode):
    assert _run_conv(64, 64, 3, 1, 1, 2, 48, 48, residual=True, halo=mode) < TOL
    assert _run_conv(32, 32, 3, 1, 1, 2, 160, 160, residual=True, halo=mode) < TOL
    assert _run_conv(64, 64, 3, 1, 1, 2, 32, 32, act='relu', halo=mode) < TOL
    assert _run_conv(64, 128, 3, 1, 1, 2, 32, 32, act=None, f32_out=True, halo=mode) < TOL
    assert _run_conv(64, 64, 3, 1, 1, 2, 32, 32, no_resident=1, halo=mode) < TOL
    assert _run_conv(128, 128, 3, 1, 1, 4, 80, 80, residual=True, halo=mode) < TOL  # more tiles than SMs


@pytest.mark.parametrize('mode', [-1, 1, 2])
def test_stem_window_halo(cuda, mode):
    """row-window stem through the halo loader: one box of 18 window rows per tile, the three filter rows are views of it, and the
    K step of the all-zero fourth window column is skipped"""
    from cvpytorch_b200 import ops
    g = torch.Generator().manual_seed(6)
    for (B, H, W) in [(2, 64, 96), (1, 128, 136), (2, 320, 320)]:
        x = torch.randn(B, 3, H, W, generator=g)
        w = torch.randn(32, 3, 6, 6, generator=g) / 108 ** 0.5
        b = torch.randn(32, generator=g)
        ref = F.silu(F.conv2d(x.cuda(), w.cuda(), b.cuda(), 2, 2))
        t = ops.SplitTensor(B, H // 2, W // 2 + 3, 16)
        ops.stem_s2d(x.cuda().contiguous(), t.view())
        wp, bp = ops.pack_conv_weights(ops.window_weights(ops.stem_weights_to_s2d(w.double()), 4), b.double())
        out = ops.SplitTensor(B, H // 2, W // 2, 32)
        plan = ops.ConvPlan(t.view(), out.view(), wp, bp, 3, 1, 1, 1, 'silu', w_window=4, halo=mode)
        plan.run()
        y = ops.split_to_nchw(out.view())
        torch.cuda.synchronize()
        assert _rel(y, ref) < TOL, (B, H, W, mode)
