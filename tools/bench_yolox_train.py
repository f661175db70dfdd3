"""Benchmark of the whole YOLOX-s network TRAINING step on the H100 kernels: cvpytorch_b200.train.CSPDarknet -> YOLOXNeck -> YOLOXHead
(80 classes) chained through forward_nhwc, 640x640 images, bs16 per GPU (BASELINE.json configs[3]), fp32 NCHW images in, stand-in
gradients on the three fp32 head outputs (the loss stays in PyTorch), SGD with momentum, the whole step captured as one CUDA graph.
Prints one JSON line: images/s and ms/step, algorithmic TFLOP/s (3x the forward convolution FLOPs), the library baseline (the oracle
network under bf16 autocast, channels_last, cuDNN, same GPU) and the card's name and power limit.  Writes nothing.  Single GPU.

  python tools/bench_yolox_train.py [--steps 20] [--warmup 5] [--batch 16]

Shares the card query, the backbone's layer list and the clock sampler of tools/bench_darknet_train.py / bench.py."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from bench_darknet_train import _card, _darknet_convs  # noqa: E402

SUBTYPE, WIDTH, NUM_CLASSES = 'cspdark_s', 0.5, 80
HW = (640, 640)


def _neck_head_convs(H, W, width=WIDTH, num_classes=NUM_CLASSES, n=1):
    """(cin, cout, k, Ho, Wo) of every convolution of YOLOXNeck + YOLOXHead (yolox_neck.py:25-41, yolox_head.py:33-49) for an H x W image."""
    c = [int(v * width) for v in (256, 512, 1024)]
    hw = [(H // s, W // s) for s in (8, 16, 32)]

    def csp(cin, cout, h, w):
        hid = cout // 2
        return [(cin, hid, 1, h, w), (cin, hid, 1, h, w), (2 * hid, cout, 1, h, w)] + [(hid, hid, 1, h, w), (hid, hid, 3, h, w)] * n
    (h2, w2), (h1, w1), (h0, w0) = hw
    convs = [(c[2], c[1], 1, h0, w0)] + csp(2 * c[1], c[1], h1, w1) + [(c[1], c[0], 1, h1, w1)] + csp(2 * c[0], c[0], h2, w2)
    convs += [(c[0], c[0], 3, h1, w1)] + csp(2 * c[0], c[1], h1, w1) + [(c[1], c[1], 3, h0, w0)] + csp(2 * c[1], c[2], h0, w0)
    p = int(256 * width)
    for ci, (h, w) in zip(c, hw):
        h, w = h + 2, w + 2
        convs += [(ci, p, 1, h, w)] + [(p, p, 3, h, w)] * 4 + [(p, num_classes, 1, h, w), (p, 5, 1, h, w)]
    return convs


def _flops(B, H, W):
    fwd = sum(2.0 * B * ho * wo * ci * co * k * k for ci, co, k, ho, wo in _darknet_convs(SUBTYPE, H, W) + _neck_head_convs(H, W))
    return 3.0 * fwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20, help='timed steps')
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--batch', type=int, default=16, help='images per step')
    args = ap.parse_args()
    if args.steps < 1:
        raise SystemExit('bench_yolox_train.py: --steps must be >= 1')
    if not torch.cuda.is_available():
        raise SystemExit('bench_yolox_train.py: no CUDA device; the training path has no CPU fallback')
    from cvpytorch_b200 import _lib, train as T
    from oracle import yolox_train_oracle as XO
    dev = torch.device('cuda:0')
    B, (H, W), K = args.batch, HW, args.steps
    mods = {'backbone.': T.CSPDarknet(SUBTYPE), 'neck.': T.YOLOXNeck('yolox_s', [256, 512, 1024], 0.33, WIDTH),
            'head.': T.YOLOXHead(NUM_CLASSES, 'yolox_s', [256, 512, 1024], width_mul=WIDTH)}
    sd = XO.synthetic_state([(pre + k, tuple(v.shape)) for pre, m in mods.items() for k, v in m.state_dict().items()])
    for pre, m in mods.items():
        m.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)})
        m.to(dev).train()
    bb, nk, hd = mods.values()
    params = [p for m in mods.values() for p in m.parameters()]
    opt = torch.optim.SGD(params, lr=1e-3, momentum=0.9)
    gen = torch.Generator().manual_seed(1031)
    NBUF = 2
    xs = [torch.randn(B, 3, H, W, generator=gen).to(dev) for _ in range(NBUF)]
    Gs = [[torch.randn(B, 5 + NUM_CLASSES, H // s + 2, W // s + 2, generator=gen).to(dev) for s in (8, 16, 32)] for _ in range(NBUF)]

    def fwd_bwd(x, G):
        torch.autograd.backward(hd.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(x))), G)

    def eager_step(i):
        fwd_bwd(xs[i % NBUF], Gs[i % NBUF])
        opt.step()
        opt.zero_grad(set_to_none=True)

    sx, sG = xs[0].clone(), [t.clone() for t in Gs[0]]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fwd_bwd(sx, sG)
            opt.step()
            opt.zero_grad(set_to_none=True)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fwd_bwd(sx, sG)
        opt.step()
        opt.zero_grad(set_to_none=True)

    def step(i):
        sx.copy_(xs[i % NBUF])
        for d, s_ in zip(sG, Gs[i % NBUF]):
            d.copy_(s_)
        graph.replay()
    for i in range(max(3, args.warmup)):
        step(i)
    sampler = ClockSampler(0)
    sampler.start()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(K):
        step(i)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / K
    clocks = sampler.stop()
    n0 = _lib.launch_count()
    eager_step(0)
    torch.cuda.synchronize()
    launches = _lib.launch_count() - n0

    # library baseline on the same GPU: the oracle network through cuDNN / ATen under bf16 autocast, channels_last
    sdg = {}
    for k, v in sd.items():
        v = v.to(dev).contiguous(memory_format=torch.channels_last) if v.dim() == 4 else v.clone().to(dev)
        sdg[k] = v.requires_grad_(True) if v.dtype.is_floating_point and 'running_' not in k else v
    xn = xs[0].contiguous(memory_format=torch.channels_last)

    def lib_step():
        with torch.autocast('cuda', dtype=torch.bfloat16):
            outs = XO.network(xn, sdg, SUBTYPE)
        torch.autograd.backward(outs, [g_.to(o.dtype) for o, g_ in zip(outs, Gs[0])])
        for v in sdg.values():
            v.grad = None
    for _ in range(3):
        lib_step()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(10):
        lib_step()
    e1.record()
    torch.cuda.synchronize()
    lib_ms = e0.elapsed_time(e1) / 10
    flops = _flops(B, H, W)
    line = {'metric': 'images/sec YOLOX-s backbone + neck + head training step (640x640) fwd+bwd+SGD, bf16, bs16', 'value': round(B / (ms / 1e3), 2),
            'unit': 'images/sec', 'n_gpus': 1, 'steps': K, 'warmup': max(3, args.warmup), 'ms_per_step': round(ms, 4), 'higher_is_better': True,
            'dtype': 'bf16 (fp32 accumulate, fp32 master weights, fp32 head outputs)', 'data': 'synthetic',
            'config': {'workload': 'YOLOX-s (CSPDarknet cspdark_s + YOLOXNeck + YOLOXHead, 80 classes) on 640x640 images: fp32 NCHW images in, forward, '
                                   'backward from stand-in gradients on the three fp32 head outputs, SGD(momentum) update; the loss is not included',
                       'per_gpu_batch': B, 'cuda_graph': True},
            'card': _card(0), 'gpu_launches': int(launches), 'clocks': clocks,
            'algorithmic': {'gflop_per_step': round(flops / 1e9, 1), 'tflops': round(flops / ms / 1e9, 1),
                            'note': '3 x the forward convolution FLOPs of the step (forward, backward-data, backward-weight), from the layer shapes'},
            'library_baseline': {'what': 'the same network step through cuDNN / ATen (oracle/yolox_train_oracle.network under torch autocast bf16, '
                                         'channels_last) on this GPU', 'ms_per_step': round(lib_ms, 4), 'images_per_sec': round(B / (lib_ms / 1e3), 2)}}
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
