"""Where do the three roles of the conv kernel spend their time?  Attaches the per-CTA cycle counters (cvb_conv_plan_set_profile)
to single layers and prints, per role, the share of cycles spent waiting on each pipeline barrier.
  python tools/conv_pipeline_profile.py            (default layer list, classic and halo loaders)
  python tools/conv_pipeline_profile.py fill       (streamed-weight 3x3, stride-2 and 3x3 + residual layers, both schedules: how long the
                                                    MMA warps wait for the ring's full barriers, on which activations and weights arrive)"""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ['CVB_DIAG_LIB'] = '1'  # the diagnostics build (csrc/build.sh diag)
import torch  # noqa: E402

from cvpytorch_b200 import _lib, ops  # noqa: E402

LAYERS = [(64, 64, 3, 1, 80, 80, 64), (64, 64, 1, 1, 80, 80, 64), (32, 32, 3, 1, 160, 160, 64), (128, 128, 3, 1, 40, 40, 64),
          (128, 128, 1, 1, 40, 40, 64), (64, 64, 1, 1, 160, 160, 64), (256, 256, 3, 1, 20, 20, 64), (512, 512, 1, 1, 20, 20, 64)]
flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')


def profile(cin, cout, k, s, H, W, B, env, label, act='silu', resid=False, schedule=0):
    for kk in ('CVB_HALO', 'CVB_HALO_BK', 'CVB_HALO_CTAS', 'CVB_HALO_RES', 'CVB_DBG'):
        os.environ.pop(kk, None)
    os.environ.update(env)
    g = torch.Generator().manual_seed(0)
    tin = ops.SplitTensor(B, H, W, cin)
    tin.data.normal_(0, 1)
    tin.data[1].mul_(2 ** -11)
    w = torch.randn(cout, cin, k, k, generator=g, dtype=torch.float64) / (cin * k * k) ** 0.5
    wp, bp = ops.pack_conv_weights(w, torch.zeros(cout, dtype=torch.float64))
    Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
    out = ops.SplitTensor(B, Ho, Wo, cout)
    res = ops.SplitTensor(B, Ho, Wo, cout) if resid else None
    if res is not None:
        res.data.normal_(0, 1)
    plan = ops.ConvPlan(tin.view(), out.view(), wp, bp, k, s, k // 2, 1, act, residual=res.view() if res is not None else None,
                        schedule=schedule)
    grid = ctypes.c_int32(0)
    buf = torch.zeros(1024 * 16, dtype=torch.int64, device='cuda')
    _lib.check(_lib.lib().cvb_conv_plan_set_profile(plan.handle, buf.data_ptr(), ctypes.byref(grid)), 'set_profile')
    ts = []
    for _ in range(3):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        plan.run()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    c = buf[:grid.value * 16].view(grid.value, 16).double().mean(0).tolist()
    tot = max(c[4], 1.0)
    e = max(c[8], 1.0)  # MMA / epilogue warpgroup: total cycles (counter rows: see the end of conv_tc_kernel)
    print(f'{label:28s} {min(ts):.4f} ms grid {grid.value:3d} | producer cycles/CTA {c[0]:9.0f} waitA {c[1] / max(c[0], 1):5.1%} '
          f'waitB {c[2] / max(c[0], 1):5.1%} | MMA warpgroup cycles {c[8]:9.0f}: main loop {c[9] / e:5.1%} (full-barrier wait {c[14] / e:5.1%}) | '
          f'epilogue wait stage-free {c[10] / e:5.1%} ld+convert {c[11] / e:5.1%} barrier {c[12] / e:5.1%} store-issue {c[13] / e:5.1%}', flush=True)


if len(sys.argv) > 1 and sys.argv[1] == 'epi':
    # the HBM-bound 1x1 layers: where does the epilogue spend its time?  (dbg 4 = no accumulator reads / math / staging, 1 = no TMA stores)
    for L in [(64, 64, 1, 1, 160, 160, 64)]:
        print(f'layer cin {L[0]} cout {L[1]} k{L[2]} s{L[3]} {L[4]}x{L[5]} B{L[6]}')
        for dbg in (0, 1, 4, 5):
            profile(*L, {'CVB_HALO': '0', 'CVB_DBG': str(dbg)}, f'  classic dbg={dbg}')
    L = (64, 64, 1, 1, 160, 160, 64)
    print('no TMA stores (dbg 1) and: 256 = accumulator reads only, 512 = ld + activation, no split / staging stores')
    for act in ('silu', None):
        for dbg in (1, 1 | 256, 1 | 512):
            profile(*L, {'CVB_HALO': '0', 'CVB_DBG': str(dbg)}, f'  act={act} dbg={dbg}', act=act)
    sys.exit(0)

if len(sys.argv) > 1 and sys.argv[1] == 'fill':
    # the YOLOv5-s bs64 layers whose weights stream from L2 for every tile (no resident slab), classic loader; (..., residual)
    FILL = [(128, 128, 3, 1, 40, 40, 64, False), (256, 256, 3, 1, 20, 20, 64, False), (64, 64, 3, 1, 80, 80, 64, False),
            (32, 64, 3, 2, 320, 320, 64, False), (64, 128, 3, 2, 160, 160, 64, False), (128, 128, 3, 2, 80, 80, 64, False),
            (128, 256, 3, 2, 80, 80, 64, False), (256, 256, 3, 2, 40, 40, 64, False), (256, 512, 3, 2, 40, 40, 64, False),
            (64, 64, 3, 1, 80, 80, 64, True), (128, 128, 3, 1, 40, 40, 64, True), (256, 256, 3, 1, 20, 20, 64, True),
            (256, 256, 1, 1, 40, 40, 64, False), (512, 512, 1, 1, 20, 20, 64, False)]
    for L in FILL:
        print(f'layer cin {L[0]} cout {L[1]} k{L[2]} s{L[3]} {L[4]}x{L[5]} B{L[6]}{" + residual" if L[7] else ""}')
        for sched, name in ((1, 'cooperative'), (2, 'ping-pong')):
            try:
                profile(*L[:7], {'CVB_HALO': '0'}, f'  {name}', resid=L[7], schedule=sched)
            except _lib.CvbError as err:
                print(f'  {name}: not eligible ({err})')
    if len(sys.argv) > 2 and sys.argv[2] == 'cut':
        # without the counters (they slow the MMA issue): layer time (median of 15) with all weight tiles, half of them and none after
        # the first ring pass (CVB_DBG bits 10 / 11; results are wrong) -- what halving the weight traffic from L2 could save at most
        print('auto schedule, no counters: all weights | half the weight fills | first ring pass only')
        for L in FILL:
            row = []
            for dbg in ('0', '1024', '2048'):
                os.environ.update({'CVB_HALO': '0', 'CVB_DBG': dbg})
                cin, cout, k, s, H, W, B, resid = L
                tin = ops.SplitTensor(B, H, W, cin)
                tin.data.normal_(0, 1)
                w = torch.randn(cout, cin, k, k, dtype=torch.float64) / (cin * k * k) ** 0.5
                wp, bp = ops.pack_conv_weights(w, torch.zeros(cout, dtype=torch.float64))
                Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
                out = ops.SplitTensor(B, Ho, Wo, cout)
                res = ops.SplitTensor(B, Ho, Wo, cout) if resid else None
                plan = ops.ConvPlan(tin.view(), out.view(), wp, bp, k, s, k // 2, 1, 'silu', residual=res.view() if res is not None else None)
                plan.run()
                ts = []
                for _ in range(15):
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    plan.run()
                    e1.record()
                    torch.cuda.synchronize()
                    ts.append(e0.elapsed_time(e1))
                row.append(sorted(ts)[7])
            print(f'  {L}: {row[0]:.4f} | {row[1]:.4f} ({row[1] / row[0] - 1:+.1%}) | {row[2]:.4f} ({row[2] / row[0] - 1:+.1%})', flush=True)
    sys.exit(0)

if len(sys.argv) > 1 and sys.argv[1] == 'dbg':
    # which concurrent activity slows the MMAs of the halo loader down?  (diagnostic switches, see ConvKArgs.dbg; results are wrong)
    for L in [(64, 64, 3, 1, 80, 80, 64), (128, 128, 3, 1, 40, 40, 64)]:
        print(f'layer cin {L[0]} cout {L[1]} k{L[2]} s{L[3]} {L[4]}x{L[5]} B{L[6]}')
        for halo, ctas in (('0', '0'), ('2', '1'), ('2', '2')):
            for dbg in (0, 7, 31):
                env = {'CVB_HALO': halo, 'CVB_DBG': str(dbg)}
                if ctas != '0':
                    env['CVB_HALO_CTAS'] = ctas
                profile(*L, env, f'  halo={halo} ctas={ctas} dbg={dbg}')
    sys.exit(0)

for L in LAYERS:
    print(f'layer cin {L[0]} cout {L[1]} k{L[2]} s{L[3]} {L[4]}x{L[5]} B{L[6]}')
    profile(*L, {'CVB_HALO': '0'}, '  classic')
    if L[2] > 1:
        for ctas in ((1, 2) if L[1] <= 64 else (1,)):
            profile(*L, {'CVB_HALO': '2', 'CVB_HALO_CTAS': str(ctas)}, f'  halo2 ctas={ctas}')
            profile(*L, {'CVB_HALO': '1', 'CVB_HALO_CTAS': str(ctas)}, f'  halo1 ctas={ctas}')
