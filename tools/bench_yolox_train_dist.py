"""Benchmark of the data-parallel YOLOX-s TRAINING step with SyncBatchNorm on the H100 kernels: cvpytorch_b200.train.CSPDarknet -> YOLOXNeck
-> YOLOXHead (80 classes) converted with nn.SyncBatchNorm.convert_sync_batchnorm, as the reference trainer does under cfg.distributed,
640x640 images, bs16 per GPU (BASELINE.json configs[3]: batch 128 over 8 GPUs), stand-in gradients on the three fp32 head outputs, one flat
fp32 gradient all-reduce, SGD with momentum, the whole step captured as one CUDA graph.

The synced step adds two collectives per BatchNorm layer (74 layers: an all-gather of the statistics records in forward, an all-reduce of
two [C] sums in backward).  The same step with local BatchNorm statistics (per-GPU batch of 16) runs in the same call, alternating with the
synced one, so that the line reports what the cross-rank statistics cost.  Prints one JSON line on rank 0 with both arms' ms/step and
images/s, and the card's name and power limit.  Writes nothing.

  torchrun --nproc_per_node 8 tools/bench_yolox_train_dist.py [--steps 20] [--warmup 5] [--batch 16] [--rounds 3]
  python tools/bench_yolox_train_dist.py            (one GPU: no collective, both arms run the local statistics)

Shares the layer list and FLOP count of tools/bench_yolox_train.py and the distributed set-up, card query and clock sampler of bench.py /
tools/bench_darknet_train.py."""
import argparse
import copy
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

from bench import ClockSampler, _dist_setup  # noqa: E402
from bench_darknet_train import _card  # noqa: E402
from bench_yolox_train import HW, NUM_CLASSES, SUBTYPE, WIDTH, _flops  # noqa: E402


def _arm(mods, xs, Gs, world, dist, steps_warm):
    """One arm: its own optimiser, one CUDA graph of fwd + bwd + the flat gradient all-reduce + SGD.  -> (step(i), keep): `keep` holds what
    the graph reads and writes besides its own pool (the optimiser's momentum buffers, the static inputs); it must outlive the replays."""
    bb, nk, hd = mods
    params = [p for m in mods for p in m.parameters()]
    opt = torch.optim.SGD(params, lr=1e-3, momentum=0.9)

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

    sx, sG = xs[0].clone(), [t.clone() for t in Gs[0]]

    def body():
        torch.autograd.backward(hd.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(sx))), sG)
        allreduce_grads()
        opt.step()
        opt.zero_grad(set_to_none=True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            body()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        body()

    def step(i):
        sx.copy_(xs[i % len(xs)])
        for d, s_ in zip(sG, Gs[i % len(Gs)]):
            d.copy_(s_)
        graph.replay()
    for i in range(steps_warm):
        step(i)
    return step, (graph, opt, body, sx, sG, mods)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20, help='timed steps per arm and round')
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--batch', type=int, default=16, help='images per GPU per step')
    ap.add_argument('--rounds', type=int, default=3, help='alternations of the two arms')
    args = ap.parse_args()
    if args.steps < 1 or args.rounds < 1:
        raise SystemExit('bench_yolox_train_dist.py: --steps and --rounds must be >= 1')
    if not torch.cuda.is_available():
        raise SystemExit('bench_yolox_train_dist.py: no CUDA device; the training path has no CPU fallback')
    from cvpytorch_b200 import train as T
    from oracle import yolox_train_oracle as XO
    dist, world, rank, local, dev, numa, barrier, max_over_ranks = _dist_setup()
    B, (H, W), K = args.batch, HW, args.steps
    mods = {'backbone.': T.CSPDarknet(SUBTYPE), 'neck.': T.YOLOXNeck('yolox_s', [256, 512, 1024], 0.33, WIDTH),
            'head.': T.YOLOXHead(NUM_CLASSES, 'yolox_s', [256, 512, 1024], width_mul=WIDTH)}
    sd = XO.synthetic_state([(pre + k, tuple(v.shape)) for pre, m in mods.items() for k, v in m.state_dict().items()])
    for pre, m in mods.items():
        m.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)})
        m.to(dev).train()
    local_mods = list(mods.values())
    synced_mods = [torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(m)) for m in local_mods]
    n_sync = sum(isinstance(b, torch.nn.SyncBatchNorm) for m in synced_mods for b in m.modules())
    gen = torch.Generator().manual_seed(1031 + rank)
    xs = [torch.randn(B, 3, H, W, generator=gen).to(dev) for _ in range(2)]
    Gs = [[torch.randn(B, 5 + NUM_CLASSES, H // s + 2, W // s + 2, generator=gen).to(dev) for s in (8, 16, 32)] for _ in range(2)]
    warm = max(3, args.warmup)
    built = {'sync_bn': _arm(synced_mods, xs, Gs, world, dist, warm), 'local_bn': _arm(local_mods, xs, Gs, world, dist, warm)}
    arms = {name: step for name, (step, _) in built.items()}
    barrier()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for name, step in arms.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            barrier()
            t0.record()
            for i in range(K):
                step(i)
            t1.record()
            barrier()
            times[name].append(max_over_ranks(t0.elapsed_time(t1)) / K)
    clocks = sampler.stop() if rank == 0 else None
    if rank == 0:
        flops = _flops(B, H, W)
        res = {}
        for name, ms_list in times.items():
            ms = statistics.median(ms_list)
            res[name] = {'ms_per_step': round(ms, 4), 'images_per_sec': round(world * B / (ms / 1e3), 2), 'ms_per_round': [round(v, 4) for v in ms_list],
                         'tflops': round(flops / ms / 1e9, 1)}
        line = {'metric': f'images/sec YOLOX-s backbone + neck + head training step (640x640) with SyncBatchNorm over {world} GPU(s), bf16, bs{B} per GPU',
                'value': res['sync_bn']['images_per_sec'], 'unit': 'images/sec', 'n_gpus': world, 'steps': K, 'warmup': warm, 'rounds': args.rounds,
                'ms_per_step': res['sync_bn']['ms_per_step'], 'higher_is_better': True, 'scaling': 'weak',
                'dtype': 'bf16 (fp32 accumulate, fp32 master weights, fp32 head outputs)', 'data': 'synthetic',
                'config': {'workload': 'YOLOX-s (CSPDarknet cspdark_s + YOLOXNeck + YOLOXHead, 80 classes) on 640x640 images: forward, backward from '
                                       'stand-in gradients on the three fp32 head outputs, one flat fp32 gradient all-reduce, SGD(momentum); the loss is '
                                       'not included', 'global_batch': world * B, 'per_gpu_batch': B, 'parallelism': f'dp{world}', 'cuda_graph': True,
                           'sync_bn_layers': n_sync, 'collectives_per_step': 2 * n_sync + 1 if world > 1 else 0, 'numa_node': numa},
                'arms': res, 'sync_over_local': round(res['sync_bn']['ms_per_step'] / res['local_bn']['ms_per_step'], 4),
                'card': _card(local), 'clocks': clocks,
                'note': 'medians over the rounds; the two arms alternate in each round. At one GPU SyncBatchNorm runs the local statistics '
                        '(a world of one), so the two arms run the same kernels.'}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
