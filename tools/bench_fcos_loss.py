"""Benchmark of the FCOS loss on the H100 kernels (csrc/fcos_loss.cu, fcos_train.FCOSLoss).  Writes nothing; one JSON line, CUDA-event
times after warm-up, the card's name and power limit read in the same call.  Single GPU.

  python tools/bench_fcos_loss.py [--steps 20] [--warmup 5] [--batch 16]

FCOS at 800² (100² + 50² + 25² + 13² + 7² = 13 343 points per image), 80 classes, seeded head outputs, two GT loads: COCO-like (1 to 30
GTs per image) and heavy (100 per image).  Per load:
1. the loss forward + backward (FCOSLoss, backward of total_loss) captured as one CUDA graph;
2. the oracle (oracle/fcos_loss_oracle.py, ATen, eager) forward + backward on the same GPU tensors;
3. the kernels' own times from torch.profiler, and the focal passes' bytes (class logits read once forward, read once and the gradient
   written once backward) over those kernels' time, against the H100 SXM data-sheet 3.35 TB/s."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

from bench_darknet_train import _card  # noqa: E402
from bench_yolox_loss import _capture, _time  # noqa: E402

NC = 80
H = W = 800
HBM_TBS = 3.35


def _inputs(B, counts, gen, dev):
    from oracle import fcos_loss_oracle as LO
    m = max(counts)
    boxes = torch.full((B, m, 4), -1.0)
    labels = torch.full((B, m), -1, dtype=torch.long)
    for b, n in enumerate(counts):
        wh = 8 + torch.rand(n, 2, generator=gen) * 500
        xy = torch.rand(n, 2, generator=gen) * (torch.tensor([W, H]) - wh)
        boxes[b, :n] = torch.cat([xy, xy + wh], 1)
        labels[b, :n] = torch.randint(1, NC + 1, (n,), generator=gen)
    preds = LO.head_outputs(B, NC, LO.level_shapes(H, W), LO.STRIDES, gen, dev)
    return preds, boxes.to(dev), labels.to(dev)


def _kernel_times(fn, names, iters=5):
    """Mean device time per call (µs) of each named kernel over `iters` eager calls, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    res = {n: 0.0 for n in names}
    for ev in prof.key_averages():
        for n in names:
            if n in ev.key:
                res[n] += ev.device_time_total / iters
    return res


def _load(name, counts, B, K, warmup, gen, dev):
    from cvpytorch_b200 import fcos_train as FT
    from oracle import fcos_loss_oracle as LO
    preds, boxes, labels = _inputs(B, counts, gen, dev)
    loss = FT.FCOSLoss()
    ps = [[t.clone().requires_grad_(True) for t in lv] for lv in preds]
    flat = [t for lv in ps for t in lv]

    def step():
        for t in flat:
            t.grad = None
        loss(ps, boxes, labels)[3].backward()
    graph = _capture(step)
    for _ in range(max(3, warmup)):
        graph.replay()
    ms = _time(graph.replay, K)
    out = [float(o) for o in loss(ps, boxes, labels)]
    qs = [[t.clone().requires_grad_(True) for t in lv] for lv in preds]

    def oracle_step():
        for lv in qs:
            for t in lv:
                t.grad = None
        LO.losses(qs, boxes, labels)[0][3].backward()
    for _ in range(2):
        oracle_step()
    oracle_ms = _time(oracle_step, 3)
    ref = [float(o) for o in LO.losses(qs, boxes, labels)[0]]
    kt = _kernel_times(step, ('fcos_assign_kernel', 'fcos_focal_kernel', 'fcos_final_kernel', 'fcos_bwd_kernel'))
    A = sum(c.shape[2] * c.shape[3] for c in preds[0])
    logits_bytes = B * NC * A * 4
    focal_us = kt['fcos_focal_kernel'] + kt['fcos_bwd_kernel']
    focal_bytes = 3 * logits_bytes
    del graph
    return {'load': name, 'gts_total': int(sum(counts)), 'ms_graph': round(ms, 4), 'oracle_ms': round(oracle_ms, 3),
            'speedup_vs_oracle': round(oracle_ms / ms, 1), 'losses': [round(v, 6) for v in out],
            'max_rel_diff_vs_oracle': max(abs(a - b) / max(abs(b), 1e-30) for a, b in zip(out, ref)),
            'kernel_us': {k: round(v, 2) for k, v in kt.items()},
            'focal_passes': {'bytes': focal_bytes, 'us': round(focal_us, 2), 'tb_per_s': round(focal_bytes / focal_us / 1e6, 3) if focal_us else None,
                             'share_of_3.35_tbs': round(focal_bytes / focal_us / 1e6 / HBM_TBS, 3) if focal_us else None,
                             'bound_us_at_3.35_tbs': round(focal_bytes / (HBM_TBS * 1e6), 2)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20, help='timed graph replays per load')
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--batch', type=int, default=16, help='images per step')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_fcos_loss.py: no CUDA device; the loss has no CPU fallback')
    dev = torch.device('cuda:0')
    B, K = args.batch, args.steps
    gen = torch.Generator().manual_seed(2025)
    coco = [int(torch.randint(1, 31, (1,), generator=gen)) for _ in range(B)]
    loads = [_load('coco_like_1_to_30', coco, B, K, args.warmup, gen, dev), _load('heavy_100', [100] * B, B, K, args.warmup, gen, dev)]
    line = {'metric': 'ms FCOS loss fwd+bwd (800x800, 80 classes, bs%d, COCO-like GTs), CUDA graph' % B, 'value': loads[0]['ms_graph'],
            'unit': 'ms', 'n_gpus': 1, 'steps': K, 'warmup': max(3, args.warmup), 'higher_is_better': False, 'data': 'synthetic',
            'config': {'batch': B, 'classes': NC, 'points_per_image': 13343, 'image': [H, W]},
            'card': _card(0), 'loads': loads,
            'library_baseline': {'what': 'oracle/fcos_loss_oracle.losses fwd + bwd (ATen, eager, per-image loop for the positives) on the same GPU tensors'}}
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
