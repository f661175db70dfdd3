"""The ping-pong schedule of the fused conv kernel at block_n = 32 and 64 (CvbConvDesc.schedule = 2) against the cooperative one.

The narrow plans that run one CTA per SM take the ping-pong schedule.  It issues the same MMAs in the same K order for every output
element and runs the same epilogue arithmetic as the cooperative schedule, so the outputs must be bitwise equal.  The 128 -> 128 1x1
layers with cin <= 128 used to run as two 64-wide cooperative n-tiles; every plan of them (block_n 64 or 128, either schedule, 32- or
64-wide K chunks) keeps each element's chain of 16-wide K steps and its rz_gain, so they must be bitwise equal as well.

The ping-pong output is also checked element by element against a float64 convolution of exactly the values the kernel reads, with
the bound of fp64ref.split_conv_reference, and against the single-layer budget max|out - ref| / max|ref| < 2e-5.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fp64ref  # noqa: E402

pytestmark = pytest.mark.gpu


def _inputs(cin, cout, k, s, B, H, W, residual, up, seed):
    from cvpytorch_b200 import ops
    p = k // 2
    g = torch.Generator().manual_seed(seed)
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    x = torch.randn(B, cin, H, W, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g) * 0.5
    tin = ops.SplitTensor(B, H, W, cin)
    ops.nchw_to_split(x.cuda(), tin.view())
    wp, bp = ops.pack_conv_weights(w.double(), b.double())
    res_t = up_t = None
    if residual:
        res_t = ops.SplitTensor(B, Ho, Wo, cout)
        ops.nchw_to_split(torch.randn(B, cout, Ho, Wo, generator=g).cuda(), res_t.view())
    if up:
        up_t = ops.F32Tensor(B, (Ho + 1) // 2, (Wo + 1) // 2, cout)
        up_t.data.copy_(torch.randn(B, (Ho + 1) // 2, (Wo + 1) // 2, cout, generator=g))
    return tin, wp, bp, res_t, up_t, Ho, Wo


def _run(cin, cout, k, s, B, H, W, act='silu', residual=False, resid_first=0, resid_scale=1.0, up=False, f32_out=False, block_n=64,
         no_resident=0, sm_limit=0, halo=0, seed=0, variants=((1,), (2,))):
    """Runs the conv once per variant (schedule,) or (schedule, block_n), requires bitwise-equal outputs and checks the last one
    against float64."""
    from cvpytorch_b200 import ops
    p = k // 2
    tin, wp, bp, res_t, up_t, Ho, Wo = _inputs(cin, cout, k, s, B, H, W, residual, up, seed)
    c_pitch = (cout + 7) // 8 * 8
    outs = []
    for v in variants:
        sched, bn = v[0], (v[1] if len(v) > 1 else block_n)
        tout = ops.F32Tensor(B, Ho, Wo, c_pitch) if f32_out else ops.SplitTensor(B, Ho, Wo, c_pitch)
        tout.data.fill_(float('nan'))
        plan = ops.ConvPlan(tin.view(), tout.view(0, cout), wp, bp, k, s, p, 1, act, residual=res_t.view() if res_t else None,
                            up_partial=up_t.view() if up_t else None, block_n=bn, sm_limit=sm_limit, no_resident=no_resident,
                            residual_before_act=resid_first, residual_scale=resid_scale, halo=halo, schedule=sched)
        plan.run()
        torch.cuda.synchronize()
        outs.append(tout.data[..., :cout].clone())
    bits = torch.int32 if f32_out else torch.int16
    for v, o in zip(variants[1:], outs[1:]):
        assert torch.equal(outs[0].contiguous().view(bits), o.contiguous().view(bits)), f'{v} and {variants[0]} outputs differ'

    # float64 reference from the values the kernel reads
    c = outs[-1]
    ref, bound = fp64ref.split_conv_reference(tin, wp, bp, k, s, p, act=act, residual=res_t, resid_first=resid_first,
                                              resid_scale=resid_scale, up=up_t.data if up else None, block_n=bn, cout=cout)
    fp64ref.check_conv(fp64ref.conv_out64(c), ref, bound, f'conv {cin}->{cout} k{k} s{s} B{B} {H}x{W}')


# (name, kwargs).  halo=-1 keeps the 3x3 layers on the classic loader (the halo plans run two CTAs per SM).  At block_n = 32 only
# 64-wide K chunks run one CTA per SM, and at block_n = 64 16-wide ones only with a residual tile: the other plans fit two.
CASES = [
    # block_n = 64
    ('bn64_bk16_cin48_3x3_ragged_boxes_tma_residual', dict(cin=48, cout=64, k=3, s=1, B=3, H=13, W=19, residual=True, halo=-1)),
    ('bn64_bk16_cin16_1x1_batch1_tma_residual', dict(cin=16, cout=64, k=1, s=1, B=1, H=40, W=40, residual=True)),
    ('bn64_bk32_cin96_3x3_stride2', dict(cin=96, cout=64, k=3, s=2, B=2, H=33, W=30, halo=-1)),
    ('bn64_odd_tiles_per_cta', dict(cin=64, cout=64, k=3, s=1, B=2, H=20, W=28, sm_limit=5, halo=-1)),
    ('bn64_fewer_tiles_than_ctas', dict(cin=128, cout=64, k=1, s=1, B=1, H=16, W=16)),
    ('bn64_tiles_n2_pinned', dict(cin=64, cout=128, k=1, s=1, B=2, H=40, W=40)),
    ('bn64_relu_residual_before_act', dict(cin=64, cout=128, k=1, s=1, B=2, H=20, W=20, act='relu', residual=True, resid_first=1)),
    ('bn64_tiles_n2_streamed', dict(cin=64, cout=128, k=1, s=1, B=2, H=40, W=40, no_resident=1)),
    ('bn64_cout48_3x3', dict(cin=64, cout=48, k=3, s=1, B=2, H=24, W=24, halo=-1)),
    ('bn64_silu_tma_residual_3x3', dict(cin=64, cout=64, k=3, s=1, B=2, H=24, W=24, residual=True, halo=-1)),
    ('bn64_relu_3x3', dict(cin=128, cout=64, k=3, s=1, B=2, H=20, W=20, act='relu', halo=-1)),
    ('bn64_generic_up_partial_scaled_residual', dict(cin=128, cout=64, k=1, s=1, B=2, H=18, W=22, residual=True, resid_scale=0.75, up=True)),
    ('bn64_f32_out_cout40', dict(cin=128, cout=40, k=1, s=1, B=2, H=16, W=16, act=None, f32_out=True)),
    # block_n = 32
    ('bn32_3x3', dict(cin=64, cout=32, k=3, s=1, B=2, H=24, W=24, block_n=32, halo=-1)),
    ('bn32_tiles_n4_pinned', dict(cin=256, cout=128, k=1, s=1, B=2, H=20, W=20, block_n=32)),
    ('bn32_3x3_stride2_tma_residual', dict(cin=128, cout=32, k=3, s=2, B=2, H=33, W=30, block_n=32, residual=True, halo=-1)),
    ('bn32_relu_residual_before_act_batch1', dict(cin=128, cout=32, k=1, s=1, B=1, H=40, W=40, block_n=32, act='relu', residual=True,
                                                  resid_first=1)),
    ('bn32_relu_3x3_odd_tiles_per_cta', dict(cin=128, cout=32, k=3, s=1, B=2, H=20, W=28, block_n=32, act='relu', sm_limit=5, halo=-1)),
    ('bn32_streamed_cout24', dict(cin=128, cout=24, k=1, s=1, B=2, H=24, W=24, block_n=32, no_resident=1)),
    ('bn32_generic_up_partial_scaled_residual', dict(cin=64, cout=32, k=3, s=1, B=2, H=18, W=22, block_n=32, residual=True,
                                                     resid_scale=0.75, up=True, halo=-1)),
    ('bn32_f32_out_cout24', dict(cin=128, cout=24, k=1, s=1, B=2, H=16, W=16, block_n=32, act=None, f32_out=True)),
]


@pytest.mark.parametrize('name,kw', CASES, ids=[c[0] for c in CASES])
def test_pingpong_narrow_matches_cooperative(cuda, name, kw):
    _run(**kw)


def test_split_layer_plans_bitwise_equal(cuda):
    """The headline's 128 -> 128 1x1 layer at 80x80: the former auto plan (two 64-wide cooperative n-tiles, 32-wide K chunks), the
    current auto plan and every other block_n / schedule pair give bitwise-equal outputs."""
    _run(cin=128, cout=128, k=1, s=1, B=4, H=80, W=80, block_n=0, variants=((1, 64), (0, 0), (2, 64), (1, 128), (2, 128)))


def test_pingpong_rejected_where_unsupported(cuda):
    """Ping-pong is an error, not a silent fallback, on plans that run two CTAs per SM, on the halo loader, at block_n = 256 and on
    narrow n-tiles of a layer wider than 128 channels."""
    from cvpytorch_b200 import _lib
    with pytest.raises(_lib.CvbError, match='narrow n-tiles on a layer of more than 128 channels'):
        _run(cin=128, cout=256, k=1, s=1, B=1, H=16, W=16, block_n=64)
    with pytest.raises(_lib.CvbError, match='two CTAs per SM'):
        _run(cin=32, cout=32, k=1, s=1, B=1, H=16, W=16, block_n=32)
    with pytest.raises(_lib.CvbError, match='halo loader'):
        _run(cin=64, cout=64, k=3, s=1, B=1, H=16, W=16, halo=2)
    with pytest.raises(_lib.CvbError, match='block_n = 256'):
        _run(cin=64, cout=256, k=1, s=1, B=1, H=16, W=16, block_n=256)
