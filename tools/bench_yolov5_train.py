"""Benchmark of the YOLOv5-s training step on the H100 kernels: YOLOv5(mode='train') + SGD as one CUDA graph, and the YOLOv5 loss
(csrc/yolov5_loss.cu) alone on the step's detect-output shapes.  Writes nothing; one JSON line, CUDA-event times after warm-up, the card's
name, power limit and maximum SM clock read in the same call, and the SM clock sampled during each timed window.  Single GPU.

  python tools/bench_yolov5_train.py [--steps 20] [--warmup 5] [--batch 64]

The batch default is conf/det/yolov5/coco_yolov5_s.yml's 64, at 640².  Targets: 2 to 20 seeded boxes per image.  The loss's share of the
step is (step with the loss - step with stand-in detect-output gradients) / step.  Step baseline: the oracle network (the reference's
layers, written functionally) + the oracle loss + SGD in eager PyTorch under bf16 autocast, channels_last, cuDNN, on the same GPU.  Loss baseline: the oracle loss
(oracle/yolov5_train_oracle.py, ATen, eager) fwd + bwd on host copies of the same tensors (the oracle's objectness targets follow the CPU's
index_put_ order), timed with a host clock."""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

from bench_darknet_train import _card  # noqa: E402
from bench_yolox_loss import _capture, _time  # noqa: E402

NC = 80
H = W = 640


def _targets(B, gen):
    rows = []
    for b in range(B):
        n = int(torch.randint(2, 21, (1,), generator=gen))
        rows.append(torch.cat([torch.full((n, 1), float(b)), torch.randint(0, NC, (n, 1), generator=gen).float(), torch.rand((n, 2), generator=gen) * 0.8 + 0.1,
                               torch.rand((n, 2), generator=gen) * 0.4 + 0.02], 1))
    return torch.cat(rows, 0)


def _clock(query):
    """One read-only nvidia-smi query of GPU 0 (e.g. clocks.sm, clocks.max.sm) -> MHz, or None."""
    try:
        out = subprocess.run(['nvidia-smi', '--id=0', f'--query-gpu={query}', '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=20)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001
        return None


def _time_with_clock(fn, K):
    """_time(fn, K) while a host thread samples the SM clock -> (ms per call, median SM MHz seen during the timed window)."""
    samples, stop = [], threading.Event()

    def poll():
        while not stop.is_set():
            v = _clock('clocks.sm')
            if v is not None:
                samples.append(v)
    t = threading.Thread(target=poll, daemon=True)
    t.start()
    try:
        ms = _time(fn, K)
    finally:
        stop.set()
        t.join()
    return ms, (sorted(samples)[len(samples) // 2] if samples else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20, help='timed steps')
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--batch', type=int, default=64, help='images per step')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_yolov5_train.py: no CUDA device; the training path has no CPU fallback')
    from cvpytorch_b200 import models as M, synth
    from oracle import yolov5_train_oracle as O
    dev = torch.device('cuda:0')
    B, K, warm = args.batch, args.steps, max(3, args.warmup)
    gen = torch.Generator().manual_seed(2024)
    model = M.YOLOv5([{f'c{i}': 1.0} for i in range(NC)], dict(synth.YOLOV5S_CFG)).to(dev).train()
    params = list(model.parameters())
    opt = torch.optim.SGD(params, lr=1e-4, momentum=0.9)
    x = torch.rand(B, 3, H, W, generator=gen).to(dev)
    gts = _targets(B, gen).to(dev)
    bb, nk, dt = model._training_modules()
    with torch.no_grad():
        outs = [o.detach() for o in dt.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(x)))]
    Gs = [torch.randn(o.shape, generator=gen).to(dev) * 1e-3 for o in outs]

    def train_step():
        model(x, gts, 'train')['loss'].backward()
        opt.step()
        opt.zero_grad(set_to_none=True)

    def standin_step():
        torch.autograd.backward(dt.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(x))), Gs)
        opt.step()
        opt.zero_grad(set_to_none=True)
    ps = [o.clone().requires_grad_(True) for o in outs]

    def loss_step():
        for p in ps:
            p.grad = None
        model.loss(ps, gts)[0].backward()
    res, clocks = {}, {}
    for name, fn in (('with_loss', train_step), ('stand_in', standin_step), ('loss', loss_step)):
        graph = _capture(fn)
        for _ in range(warm):
            graph.replay()
        res[name], clocks[name] = _time_with_clock(graph.replay, K)
        del graph

    # baseline: the oracle network (the reference's layers, functional) + the oracle loss, eager, bf16 autocast, channels_last, cuDNN
    torch.backends.cudnn.benchmark = True
    sd = {k: (v.detach().clone(memory_format=torch.channels_last) if v.dim() == 4 else v.detach().clone())
          .requires_grad_(v.dtype.is_floating_point and 'running_' not in k and k != 'detect.anchors') for k, v in model.state_dict().items()}
    leaves = [v for v in sd.values() if v.requires_grad]
    base_opt = torch.optim.SGD(leaves, lr=1e-4, momentum=0.9)
    xc = x.to(memory_format=torch.channels_last)
    anchors_dev = torch.tensor(M.YOLOv5.anchors)

    def baseline_step():
        with torch.autocast('cuda', dtype=torch.bfloat16):
            outs_b = O.network(xc, sd)
        O.yolov5_loss([o.float() for o in outs_b], gts, anchors_dev, NC)[0].backward()
        base_opt.step()
        base_opt.zero_grad(set_to_none=True)
    for _ in range(warm):
        baseline_step()
    res['baseline'], clocks['baseline'] = _time_with_clock(baseline_step, K)
    del sd, leaves, base_opt
    anchors = torch.tensor(M.YOLOv5.anchors)
    qs = [o.cpu().requires_grad_(True) for o in outs]
    gts_cpu = gts.cpu()

    def oracle_step():
        for q in qs:
            q.grad = None
        O.yolov5_loss(qs, gts_cpu, anchors, NC)[0].backward()
    oracle_step()
    t0 = time.perf_counter()
    for _ in range(3):
        oracle_step()
    oracle_ms = (time.perf_counter() - t0) / 3 * 1000.0
    line = {'metric': "ms YOLOv5-s training step (YOLOv5(mode='train') + SGD, 640x640, 80 classes, bs%d), CUDA graph" % B,
            'value': round(res['with_loss'], 3), 'unit': 'ms', 'n_gpus': 1, 'steps': K, 'warmup': warm, 'higher_is_better': False, 'data': 'synthetic',
            'img_per_s': round(B * 1000.0 / res['with_loss'], 1),
            'config': {'batch': B, 'gts_total': int(gts.shape[0]), 'gts_per_image': '2 to 20 (seeded)'},
            'card': dict(_card(0), max_sm_clock_mhz=_clock('clocks.max.sm')),
            'sm_clock_mhz_in_timed_windows': clocks,
            'baseline': {'what': 'oracle/yolov5_train_oracle.network + yolov5_loss + SGD, eager PyTorch, bf16 autocast, channels_last, cuDNN, same GPU',
                         'ms': round(res['baseline'], 3), 'img_per_s': round(B * 1000.0 / res['baseline'], 1)},
            'ms_stand_in_gradients': round(res['stand_in'], 3),
            'loss_share': round((res['with_loss'] - res['stand_in']) / res['with_loss'], 4),
            'loss': {'what': 'YOLOv5Loss fwd + bwd alone on the step\'s detect outputs, one CUDA graph', 'ms': round(res['loss'], 4),
                     'oracle_ms': round(oracle_ms, 3), 'oracle': 'oracle/yolov5_train_oracle.yolov5_loss fwd + bwd (ATen, eager) on copies of the same tensors on the host CPU'}}
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
