"""Times the YOLOv6 loss forward + backward (csrc/yolov6_loss.cu) as one CUDA graph at 640², bs64, 80 classes (the s config), with a
COCO-like GT load (1 to 30 per image) and a heavy one (100 per image), under ATSS and under TAL; next to the oracle
(oracle/yolov6_loss_oracle.py) in eager ATen on the same GPU.  Kernel times come from torch.profiler.  Prints one JSON line with the
card's name and power limit.

  python tools/bench_yolov6_loss.py [--iters 50]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cvpytorch_b200 import yolov6_train as YT  # noqa: E402
from oracle import yolov6_loss_oracle as LO  # noqa: E402


def power_limit():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'], capture_output=True, text=True,
                           timeout=20)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def workload(load, B=64, size=640, nc=80):
    gen = torch.Generator().manual_seed(5)
    shapes = LO.level_shapes(size, size)
    A = sum(h * w for h, w in shapes)
    scores, distri = LO.make_preds(gen, B, A, nc)
    per = [100] * B if load == 'heavy' else [int(torch.randint(1, 31, (), generator=gen)) for _ in range(B)]
    gt = LO.make_targets(gen, B, size, size, per, nc=nc)
    return shapes, scores.cuda(), distri.cuda(), gt.cuda()


def time_ms(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    args = ap.parse_args()
    res = {'gpu': torch.cuda.get_device_name(0), 'power_limit_w': power_limit(), 'B': 64, 'size': 640, 'nc': 80, 'cases': {}}
    for load in ('coco', 'heavy'):
        shapes, scores, distri, gt = workload(load)
        for assigner in ('atss', 'tal'):
            p = YT.loss_params(shapes, (8, 16, 32), 80, 64, assigner, 'giou')
            t = gt.double().contiguous()
            gout = torch.ones(3, dtype=torch.float64, device='cuda')

            def step():
                out, a = YT.yolov6_loss_forward(p, scores, distri, t)
                return YT.yolov6_loss_backward(p, distri, a, gout)
            st = torch.cuda.Stream()
            st.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(st):
                step()
            torch.cuda.current_stream().wait_stream(st)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                step()
            graph_ms = time_ms(graph.replay, args.iters)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    graph.replay()
                torch.cuda.synchronize()
            kern = {}
            for ev in prof.key_averages():
                if 'v6_' in ev.key:
                    name = ev.key.split('v6_')[1].split('_kernel')[0]
                    kern[name] = round(ev.device_time_total / max(ev.count, 1), 2)

            def oracle():
                d = distri.detach().requires_grad_(True)
                out, _ = LO.losses(shapes, scores, d, gt, assigner, 'giou', 80)
                (out['iou'] + out['dfl'] + out['class']).backward()
            oracle_ms = time_ms(oracle, 3)
            res['cases'][f'{load}_{assigner}'] = {'gts': int(gt.shape[0]), 'graph_ms': round(graph_ms, 4), 'kernel_us': kern,
                                                  'oracle_ms': round(oracle_ms, 2), 'speedup': round(oracle_ms / graph_ms, 1)}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
