"""Benchmark of the YOLOX-s CSPDarknet backbone TRAINING step on the H100 kernels (cvpytorch_b200.train.CSPDarknet): 640x640 images,
bs16 per GPU (BASELINE.json configs[3]: batch 128 over 8 GPUs), fp32 NCHW images in, stand-in gradients on the three outputs, SGD with
momentum, the whole step captured as one CUDA graph.  Prints one JSON line: images/s and ms/step, algorithmic TFLOP/s (3x the forward
convolution FLOPs from the layer shapes), the library baseline (the oracle backbone under bf16 autocast, channels_last, cuDNN, same GPU),
the CPU oracle leg, and the card's name and power limit.  Writes nothing.

  python tools/bench_darknet_train.py [--steps 20] [--warmup 5] [--batch 16] [--cpu-steps 2] [--graph 1]
  torchrun --nproc_per_node 8 tools/bench_darknet_train.py          (data-parallel: one fp32 gradient all-reduce per step)

Shares the clock sampler, the distributed set-up and the CPU-thread probe of bench.py."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import ClockSampler, _dist_setup, pick_cpu_threads  # noqa: E402

DARKNET_CFG = dict(subtype='cspdark_s', hw=(640, 640), batch=16,
                   metric='images/sec YOLOX-s CSPDarknet backbone training step (640x640) fwd+bwd+SGD, bf16, bs16 per GPU',
                   workload='the YOLOX-s backbone (CSPDarknet cspdark_s: Focus stem, four stages, SPPF; 35 convolutions, 4.2 M parameters) on 640x640 '
                            'images, training step: fp32 NCHW images in, forward, backward from stand-in gradients on the three outputs (dark3 / dark4 / '
                            'dark5, NHWC bf16), gradient all-reduce, SGD(momentum) update; bf16 activations / gradients, fp32 master weights; bs16 per GPU '
                            '= BASELINE.json configs[3] (batch 128 over 8 GPUs) without the neck, head and loss')


def _darknet_convs(subtype, H, W):
    """(cin, cout, k, Ho, Wo) of every convolution of CSPDarknet(subtype) on an H x W image (csp_darknet.py:53-89); the stem counts its 12 real
    input channels."""
    from oracle import darknet_train_oracle as DO
    ch, nl = DO.widths(subtype), DO.depths(subtype)
    h, w = H // 2, W // 2
    convs = [(12, ch[0], 3, h, w)]

    def csp(c, n):
        hid = c // 2
        return [(c, hid, 1, h, w), (c, hid, 1, h, w), (2 * hid, c, 1, h, w)] + [(hid, hid, 1, h, w), (hid, hid, 3, h, w)] * n
    for i in range(1, 5):
        h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        convs.append((ch[i - 1], ch[i], 3, h, w))
        if i == 4:
            convs += [(ch[4], ch[4] // 2, 1, h, w), (2 * ch[4], ch[4], 1, h, w)]
        convs += csp(ch[i], nl[i - 1])
    return convs


def _darknet_flops(B, H, W, subtype):
    fwd = sum(2.0 * B * ho * wo * ci * co * k * k for ci, co, k, ho, wo in _darknet_convs(subtype, H, W))
    return 3.0 * fwd  # forward + backward-data + backward-weight (the stem has no backward-data: counted anyway, as the algorithmic convention)


def _card(local):
    """The card's name and power limit (read-only query)."""
    name = torch.cuda.get_device_name(local)
    try:
        out = subprocess.run(['nvidia-smi', f'--id={local}', '--query-gpu=power.limit', '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=20)
        power = float(out.stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001
        power = None
    return {'name': name, 'power_limit_w': power}


def _darknet_cpu(steps, B=1):
    """The oracle's backbone training step (reference restated, torch.autograd) on the host cores: bounded sample."""
    from cvpytorch_b200 import train as T
    from oracle import darknet_train_oracle as DO
    c = DARKNET_CFG
    H, W = c['hw']
    sd = DO.synthetic_state([(k, tuple(v.shape)) for k, v in T.CSPDarknet(c['subtype']).state_dict().items()])
    ch = DO.widths(c['subtype'])
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, 3, H, W, generator=g)
    Gs = [torch.randn(B, ch[i], H >> (i + 1), W >> (i + 1), generator=g) for i in (2, 3, 4)]
    cores = pick_cpu_threads(lambda: DO.train_step(x[:, :, :128, :128], [G[:, :, :128 >> (i + 3), :128 >> (i + 3)] for i, G in enumerate(Gs)], sd, subtype=c['subtype']))
    torch.set_num_threads(cores)
    DO.train_step(x, Gs, sd, subtype=c['subtype'])
    t0 = time.perf_counter()
    for _ in range(steps):
        DO.train_step(x, Gs, sd, subtype=c['subtype'])
    dt = time.perf_counter() - t0
    return B * steps / dt, cores, dt / steps, f'{steps} steps x bs{B} {H}x{W} forward+backward of the backbone, torch {torch.__version__} fp32 autograd, {cores} threads'


def run_darknet_train_arm(args):
    """The training step of the YOLOX-s CSPDarknet backbone on the H100 kernels (cvpytorch_b200/train.py)."""
    from cvpytorch_b200 import _lib, train as T
    from oracle import darknet_train_oracle as DO
    c = DARKNET_CFG
    dist, world, rank, local, dev, numa, barrier, max_over_ranks = _dist_setup()
    B = args.batch or c['batch']
    H, Wd = c['hw']
    K, W = args.steps, max(3, args.warmup)
    m = T.CSPDarknet(c['subtype'])
    sd = DO.synthetic_state([(k, tuple(v.shape)) for k, v in m.state_dict().items()])
    m.load_state_dict(sd)
    m.to(dev).train()
    params = [p for p in m.parameters()]
    opt = torch.optim.SGD(params, lr=1e-3, momentum=0.9)
    NBUF = 2
    gen = torch.Generator().manual_seed(1029 + rank)
    ch = DO.widths(c['subtype'])
    out_hw = [(H >> (i + 1), Wd >> (i + 1)) for i in (2, 3, 4)]
    xs = [torch.randn(B, 3, H, Wd, generator=gen).to(dev) for _ in range(NBUF)]  # fp32 NCHW images, as the data loader delivers them
    Gs = [[torch.randn(B, h, w, ch[i], generator=gen).to(dev).to(torch.bfloat16) for i, (h, w) in zip((2, 3, 4), out_hw)] for _ in range(NBUF)]

    def allreduce_grads():
        if world == 1:
            return
        flat = torch.cat([p.grad.reshape(-1) for p in params])
        dist.all_reduce(flat)
        flat /= world
        off = 0
        for p in params:
            p.grad.copy_(flat[off:off + p.numel()].view_as(p.grad))
            off += p.numel()

    def fwd_bwd(x, G):
        torch.autograd.backward(m.forward_nhwc(x), G)

    def step(i):
        fwd_bwd(xs[i % NBUF], Gs[i % NBUF])
        allreduce_grads()
        opt.step()
        opt.zero_grad(set_to_none=True)

    graphed = None
    eager_step = step
    if args.graph and world == 1:
        try:
            sx = xs[0].clone()
            sG = [t.clone() for t in Gs[0]]
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    fwd_bwd(sx, sG)
                    opt.step()
                    opt.zero_grad(set_to_none=True)
            torch.cuda.current_stream().wait_stream(side)
            graphed = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graphed):
                fwd_bwd(sx, sG)
                opt.step()
                opt.zero_grad(set_to_none=True)

            def step(i):  # noqa: F811
                sx.copy_(xs[i % NBUF])
                for d, s_ in zip(sG, Gs[i % NBUF]):
                    d.copy_(s_)
                graphed.replay()
            for i in range(W):
                step(i)
        except Exception as ex:  # noqa: BLE001
            print(f'[bench] CUDA graph capture of the training step failed ({ex}); timing the eager step', file=sys.stderr)
            graphed = None
            step = eager_step
    if graphed is None:
        for i in range(W):
            step(i)
    barrier()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    t0.record()
    for i in range(K):
        step(i)
    t1.record()
    barrier()
    total_ms = max_over_ranks(t0.elapsed_time(t1))
    clocks = sampler.stop() if rank == 0 else None
    n0 = _lib.launch_count()
    eager_step(0)
    torch.cuda.synchronize()
    launches = _lib.launch_count() - n0
    value = world * B * K / (total_ms / 1e3)

    # library baseline on the same GPU: the oracle's backbone through cuDNN / ATen under bf16 autocast, channels_last
    lib_ms = None
    try:
        sdg = {}
        for k, v in sd.items():
            v = v.to(dev).contiguous(memory_format=torch.channels_last) if v.dim() == 4 else v.clone().to(dev)
            sdg[k] = v.requires_grad_(True) if v.dtype.is_floating_point and 'running_' not in k else v
        xn = xs[0].contiguous(memory_format=torch.channels_last)
        Gn = [t.permute(0, 3, 1, 2) for t in Gs[0]]  # (an NHWC tensor seen as NCHW: channels_last strides)

        def lib_step():
            with torch.autocast('cuda', dtype=torch.bfloat16):
                outs = DO.csp_darknet(xn, sdg, subtype=c['subtype'])
            torch.autograd.backward(outs, [g_.to(o.dtype) for o, g_ in zip(outs, Gn)])
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
        del sdg
    except Exception as ex:  # noqa: BLE001  (context number only)
        lib_ms = None
        print(f'[bench] library baseline skipped: {ex}', file=sys.stderr)
    if rank == 0:
        flops = _darknet_flops(B, H, Wd, c['subtype'])
        ms = total_ms / K
        cpu_v, cores, spt, sample = _darknet_cpu(args.cpu_steps) if (args.cpu_steps > 0 and world == 1) else (None, 0, 0, 'skipped (timed at N=1 only)' if world > 1 else 'skipped')
        line = {'metric': c['metric'], 'value': round(value, 2), 'unit': 'images/sec', 'n_gpus': world, 'steps': K, 'warmup': W, 'ms_per_step': round(ms, 4),
                'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None, 'dtype': 'bf16 (fp32 accumulate, fp32 master weights)', 'data': 'synthetic',
                'config': {'workload': c['workload'], 'global_batch': world * B, 'per_gpu_batch': B, 'parallelism': f'dp{world}', 'cuda_graph': graphed is not None,
                           'collective': 'one NCCL all-reduce of the flat fp32 gradient bucket per step' if world > 1 else 'none (N=1)', 'numa_node': numa},
                'card': _card(local), 'gpu_launches': int(launches), 'clocks': clocks,
                'algorithmic': {'gflop_per_step': round(flops / 1e9, 1), 'tflops': round(flops / ms / 1e9, 1),
                                'note': '3 x the forward convolution FLOPs of the step (forward, backward-data, backward-weight), from the layer shapes'},
                'library_baseline': {'what': 'the same backbone step through cuDNN / ATen (oracle/darknet_train_oracle.py under torch autocast bf16, channels_last) on this GPU',
                                     'ms_per_step': round(lib_ms, 4) if lib_ms else None, 'images_per_sec': round(B / (lib_ms / 1e3), 2) if lib_ms else None},
                'cpu_baseline': {'value': round(cpu_v, 4) if cpu_v else None, 'unit': 'images/sec', 'cores': cores, 'kind': 'port', 'sample': sample}}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()




def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20, help='timed steps')
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--batch', type=int, default=0, help='images per GPU per step (default 16)')
    ap.add_argument('--graph', type=int, default=1, help='1 (default): the timed steps replay one captured CUDA graph; 0: eager launches')
    ap.add_argument('--cpu-steps', type=int, default=2, help='CPU oracle steps timed on rank 0 (0 = skip)')
    args = ap.parse_args()
    if args.steps < 1:
        raise SystemExit('bench_darknet_train.py: --steps must be >= 1')
    if not torch.cuda.is_available():
        raise SystemExit('bench_darknet_train.py: no CUDA device; the training path has no CPU fallback')
    args.cpu_steps = min(args.cpu_steps, 2)
    run_darknet_train_arm(args)


if __name__ == '__main__':
    main()
