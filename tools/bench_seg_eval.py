"""Benchmark of the segmentation evaluator drop-in (cvpytorch_b200.seg_eval.SegmentationEvaluator, csrc/seg_eval.cu) on the H100.
Writes nothing; prints one JSON line with the card's name, power limit and SM clocks, read in the same call.  Single GPU.

  python tools/bench_seg_eval.py [--iters 200] [--images 20]

Label maps are 1024×2048 (Cityscapes' val size): uint8 gt with about 10 % ignore pixels (255), int64 pred, class frequencies falling
geometrically (class 0 about 30 % of the pixels, as Cityscapes' road), pred equal to gt on 85 % of the pixels.
  update[bs, nc]   update_us: one update() call, CUDA events over --iters calls (the Python wrapper included, so at bs1 it can be
                   host-bound); kernel_us: the kernel's device time from torch.profiler in a separate pass; bytes read over the kernel
                   time against the H100 SXM's 3.35 TB/s data-sheet HBM bandwidth.
  host[bs, nc]     the reference-style path on the same tensors: both maps copied to the host, then the numpy oracle's update
                   (mask, flat index, np.bincount) added to a float64 matrix; host clock.
  val_loop         ms per image of a bs1 × 1024×2048 val loop: the drop-in EncoderDecoder val forward (DeepLabv3+ R50, 19 classes)
                   followed by the drop-in update, against the same forward followed by the host path; host clock over --images images
                   ending in a device synchronise, two alternating rounds per arm."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
H, W = 1024, 2048


def card():
    """The card's name, power limit and SM clocks (read-only query)."""
    out = {'name': torch.cuda.get_device_name(torch.cuda.current_device())}
    try:
        q = subprocess.run(['nvidia-smi', f'--id={torch.cuda.current_device()}', '--query-gpu=power.limit,clocks.sm,clocks.max.sm',
                            '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=20)
        p, sm, sm_max = (v.strip() for v in q.stdout.strip().splitlines()[0].split(','))
        out.update(power_limit_w=float(p), sm_clock_mhz=float(sm), sm_clock_max_mhz=float(sm_max))
    except Exception:  # noqa: BLE001
        out.update(power_limit_w=None, sm_clock_mhz=None, sm_clock_max_mhz=None)
    return out


class _Dataset:
    def __init__(self, nc):
        self.num_classes = nc
        self.dictionary = [{f'c{i}': 1.0} for i in range(nc)]


def skewed(shape, nc, g, r=0.7):
    """Classes with P(c) proportional to r^c, by the inverse CDF of a uniform draw."""
    u = torch.rand(shape, generator=g, device='cuda', dtype=torch.float64)
    c = torch.floor(torch.log1p(-u * (1 - r ** nc)) / np.log(r)).to(torch.int64)
    return c.clamp_(0, nc - 1)


def label_maps(bs, nc, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    gt = skewed((bs, H, W), nc, g)
    pred = torch.where(torch.rand((bs, H, W), generator=g, device='cuda') < .85, gt, skewed((bs, H, W), nc, g))
    gt = torch.where(torch.rand((bs, H, W), generator=g, device='cuda') < .1, torch.full_like(gt, 255), gt).to(torch.uint8)
    return gt, pred


def host_update(cm, gt, pred, nc):
    from oracle import seg_eval_oracle as SO
    counts, err = SO.confusion_update(gt.cpu().numpy(), pred.cpu().numpy(), nc)
    assert not err
    cm += counts


def bench_update(bs, nc, iters):
    from cvpytorch_b200.seg_eval import SegmentationEvaluator
    gt, pred = label_maps(bs, nc)
    ev = SegmentationEvaluator(_Dataset(nc))
    ev.reset()
    for _ in range(5):
        ev.update(gt, pred)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        ev.update(gt, pred)
    b.record()
    b.synchronize()
    update_us = a.elapsed_time(b) * 1e3 / iters
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            ev.update(gt, pred)
        torch.cuda.synchronize()
    ks = [e for e in prof.events() if 'seg_confusion_kernel' in e.name]
    kernel_us = statistics.median(e.device_time for e in ks) if ks else None
    nbytes = gt.numel() * (gt.element_size() + pred.element_size())
    # the host path on the same tensors, and the check that both paths count the same pixels
    cm = np.zeros((nc, nc))
    times = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host_update(cm, gt, pred, nc)
        times.append(time.perf_counter() - t0)
    ev.reset()
    ev.update(gt, pred)
    equal = bool(np.array_equal(ev.confusion_matrix * 3, cm))
    return {'bs': bs, 'nc': nc, 'bytes': nbytes, 'update_us': round(update_us, 2), 'kernel_us': None if kernel_us is None else round(kernel_us, 2),
            'hbm_share': None if not kernel_us else round(nbytes / HBM_BYTES_PER_S * 1e6 / kernel_us, 3),
            'bound_us': round(nbytes / HBM_BYTES_PER_S * 1e6, 2), 'host_ms': round(statistics.median(times) * 1e3, 2), 'matrix_equal': equal}


def bench_val_loop(images):
    from cvpytorch_b200 import synth
    from cvpytorch_b200.seg_eval import SegmentationEvaluator
    model = synth.build_deeplab(True)
    nc = 19
    gt, _ = label_maps(1, nc, seed=1)
    g = torch.Generator(device='cuda').manual_seed(2)
    imgs = [torch.randn((1, 3, H, W), generator=g, device='cuda') for _ in range(4)]

    def device_arm(n):
        ev = SegmentationEvaluator(_Dataset(nc))
        ev.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(n):
            ev.update(gt, model(imgs[i % 4], gt, mode='val'))
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / n

    def host_arm(n):
        cm = np.zeros((nc, nc))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(n):
            host_update(cm, gt, model(imgs[i % 4], gt, mode='val'), nc)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / n

    def forward_only(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(n):
            model(imgs[i % 4], gt, mode='val')
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / n

    device_arm(2), host_arm(2), forward_only(2)  # warm-up: graph capture, module load
    res = {'device': [], 'host': [], 'forward_only': []}
    for _ in range(2):
        res['device'].append(device_arm(images) * 1e3)
        res['host'].append(host_arm(images) * 1e3)
        res['forward_only'].append(forward_only(images) * 1e3)
    return {k + '_ms_per_image': [round(v, 2) for v in vs] for k, vs in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--images', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_seg_eval.py needs a CUDA device')
    res = {'bench': 'seg_eval', 'card': card(), 'hw': [H, W]}
    res['update'] = [bench_update(bs, nc, args.iters if bs == 1 else max(args.iters // 8, 10)) for bs in (1, 16) for nc in (19, 150)]
    res['val_loop'] = bench_val_loop(args.images)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
