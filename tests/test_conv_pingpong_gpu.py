"""The ping-pong schedule of the fused conv kernel (CvbConvDesc.schedule = 2) against the cooperative one (schedule = 1).

Both schedules issue the same MMAs in the same K order for every output element and run the same epilogue arithmetic, so their outputs
must be bitwise equal.  The ping-pong output is also checked element by element against a float64 convolution of exactly the values the
kernel reads (hi + lo of the split input and weights), with the bound of fp64ref.split_conv_reference, and against the single-layer
budget max|out - ref| / max|ref| < 2e-5.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fp64ref  # noqa: E402

pytestmark = pytest.mark.gpu


def _run(cin, cout, k, s, B, H, W, act='silu', residual=False, resid_first=0, resid_scale=1.0, up=False, f32_out=False, block_n=128,
         no_resident=0, sm_limit=0, seed=0):
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
    c_pitch = (cout + 7) // 8 * 8
    outs = {}
    for sched in (1, 2):
        tout = ops.F32Tensor(B, Ho, Wo, c_pitch) if f32_out else ops.SplitTensor(B, Ho, Wo, c_pitch)
        tout.data.fill_(float('nan'))
        plan = ops.ConvPlan(tin.view(), tout.view(0, cout), wp, bp, k, s, p, 1, act, residual=res_t.view() if res_t else None,
                            up_partial=up_t.view() if up_t else None, block_n=block_n, sm_limit=sm_limit, no_resident=no_resident,
                            residual_before_act=resid_first, residual_scale=resid_scale, schedule=sched)
        plan.run()
        torch.cuda.synchronize()
        outs[sched] = tout.data.clone()
    a, c = outs[1][..., :cout], outs[2][..., :cout]
    bits = torch.int32 if f32_out else torch.int16
    assert torch.equal(a.contiguous().view(bits), c.contiguous().view(bits)), 'ping-pong and cooperative outputs differ'

    # float64 reference from the values the kernel reads
    ref, bound = fp64ref.split_conv_reference(tin, wp, bp, k, s, p, act=act, residual=res_t, resid_first=resid_first,
                                              resid_scale=resid_scale, up=up_t.data if up else None, block_n=block_n, cout=cout)
    fp64ref.check_conv(fp64ref.conv_out64(c), ref, bound, f'conv {cin}->{cout} k{k} s{s} B{B} {H}x{W}')


# (name, kwargs)
CASES = [
    ('odd_tiles_per_cta', dict(cin=128, cout=128, k=3, s=1, B=2, H=20, W=28, sm_limit=5)),
    ('fewer_tiles_than_ctas', dict(cin=128, cout=128, k=1, s=1, B=1, H=16, W=16)),
    ('single_tile', dict(cin=64, cout=128, k=3, s=1, B=1, H=8, W=8)),
    ('ragged_boxes', dict(cin=64, cout=128, k=3, s=1, B=3, H=13, W=19)),
    ('stride2', dict(cin=64, cout=128, k=3, s=2, B=2, H=33, W=30)),
    ('cout_not_multiple', dict(cin=64, cout=200, k=1, s=1, B=2, H=24, W=24)),
    ('tiles_n2_pinned', dict(cin=64, cout=256, k=1, s=1, B=2, H=40, W=40)),
    ('tiles_n4_pinned', dict(cin=64, cout=512, k=1, s=1, B=2, H=20, W=20)),
    ('tiles_n2_streamed', dict(cin=64, cout=256, k=1, s=1, B=2, H=40, W=40, no_resident=1)),
    ('deep_k_streamed', dict(cin=256, cout=256, k=1, s=1, B=4, H=40, W=40)),
    ('silu_tma_residual', dict(cin=128, cout=128, k=3, s=1, B=2, H=24, W=24, residual=True)),
    ('relu_residual_before_act', dict(cin=128, cout=128, k=1, s=1, B=2, H=24, W=24, act='relu', residual=True, resid_first=1)),
    ('generic_up_partial_scaled_residual', dict(cin=128, cout=128, k=1, s=1, B=2, H=18, W=22, residual=True, resid_scale=0.75, up=True)),
    ('f32_out', dict(cin=128, cout=255, k=1, s=1, B=2, H=16, W=16, act=None, f32_out=True)),
    ('batch1', dict(cin=256, cout=128, k=3, s=1, B=1, H=40, W=40)),
]


@pytest.mark.parametrize('name,kw', CASES, ids=[c[0] for c in CASES])
def test_pingpong_matches_cooperative(cuda, name, kw):
    _run(**kw)


def test_pingpong_rejected_where_unsupported(cuda):
    """block_n 256 and 64 plans run the cooperative schedule only; asking for ping-pong is an error, not a silent fallback."""
    from cvpytorch_b200 import _lib
    for bn in (64, 256):
        with pytest.raises(_lib.CvbError, match='ping-pong'):
            _run(cin=64, cout=256, k=1, s=1, B=1, H=16, W=16, block_n=bn)
