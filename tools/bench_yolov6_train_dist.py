"""Benchmark of the data-parallel YOLOv6-s TRAINING step with SyncBatchNorm on the H100 kernels: YOLOv6(mode='train') converted with
nn.SyncBatchNorm.convert_sync_batchnorm, as the reference trainer does under cfg.distributed, 640x640 images, bs64 per GPU
(conf/det/yolov6/coco_yolov6_s.yml's BATCH_SIZE), 80 classes, the seeded targets of tools/bench_yolov6_train.py, backward, one flat fp32
gradient all-reduce, SGD with momentum, the whole step captured as one CUDA graph.

The synced step issues one all-gather of the statistics records per BatchNorm in forward (128) and one all-reduce per layer in backward:
one [4][C] buffer per RepVGG block (35), one [2][C] buffer per ReLU ConvModule (19) and per SiLU head ConvModule (9), less the layers
whose backward does not run (the reference discards the class loss, so the three head.cls_convs get no gradient).  The script counts the
collectives one synced step actually issues and prints that count.  The same step with local BatchNorm statistics runs in the same call,
alternating with the synced one, so that the line reports what the cross-rank statistics cost.  Prints one JSON line on rank 0 with both
arms' ms/step and images/s, the card's name and power limit and the SM clock sampled during the timed windows.  Writes nothing.

  torchrun --nproc_per_node 8 tools/bench_yolov6_train_dist.py [--steps 10] [--warmup 3] [--batch 64] [--rounds 3]
  python tools/bench_yolov6_train_dist.py            (one GPU: no collective, both arms run the local statistics)

Shares the distributed set-up, card query and clock sampler of bench.py / tools/bench_darknet_train.py and the model config and targets of
tools/bench_yolov6_train.py."""
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
from bench_yolov5_train import _targets  # noqa: E402
from bench_yolov6_train import CFG, H, NC, W  # noqa: E402


class _CollectiveCounter:
    """Counts the torch.distributed collectives issued while `active` (the statistics' all-gathers and all-reduces of one synced step)."""

    def __init__(self, dist):
        self.active, self.counts = False, {'all_gather_into_tensor': 0, 'all_reduce': 0}
        for name in self.counts:
            fn = getattr(dist, name)
            setattr(dist, name, self._wrap(name, fn))

    def _wrap(self, name, fn):
        def call(*args, **kw):
            if self.active:
                self.counts[name] += 1
            return fn(*args, **kw)
        return call


def _arm(model, x, gts, world, dist, counter, steps_warm):
    """One arm: its own optimiser, one CUDA graph of mode='train' + backward + the flat gradient all-reduce + SGD.  -> (step, keep): `keep`
    holds what the graph reads and writes besides its own pool; it must outlive the replays.  The first eager step runs with the collective
    counter on, before the gradient all-reduce."""
    params = [p for p in model.parameters() if p.requires_grad]
    opt = torch.optim.SGD(params, lr=1e-4, momentum=0.9)

    def allreduce_grads():
        if world == 1:
            return
        live = [p for p in params if p.grad is not None]  # (head.cls_convs / cls_preds: no gradient)
        flat = torch.cat([p.grad.reshape(-1) for p in live])
        dist.all_reduce(flat)
        flat /= world
        off = 0
        for p in live:
            p.grad.copy_(flat[off:off + p.numel()].view_as(p.grad))
            off += p.numel()

    def body(count=False):
        counter.active = count
        model(x, gts, 'train')['loss'].backward()
        counter.active = False
        allreduce_grads()
        opt.step()
        opt.zero_grad(set_to_none=True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        body(count=True)
        body()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        body()
    for _ in range(steps_warm):
        graph.replay()
    return graph.replay, (graph, opt, body, model)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10, help='timed steps per arm and round')
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--batch', type=int, default=64, help='images per GPU per step')
    ap.add_argument('--rounds', type=int, default=3, help='alternations of the two arms')
    args = ap.parse_args()
    if args.steps < 1 or args.rounds < 1:
        raise SystemExit('bench_yolov6_train_dist.py: --steps and --rounds must be >= 1')
    if not torch.cuda.is_available():
        raise SystemExit('bench_yolov6_train_dist.py: no CUDA device; the training path has no CPU fallback')
    from cvpytorch_b200 import yolov6_models as M
    dist, world, rank, local, dev, numa, barrier, max_over_ranks = _dist_setup()
    counter = _CollectiveCounter(dist)
    B, K = args.batch, args.steps
    gen = torch.Generator().manual_seed(2024 + rank)
    local_model = M.YOLOv6([{f'c{i}': 1.0} for i in range(NC)], dict(CFG)).to(dev).train()
    synced_model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(local_model))
    n_sync = sum(isinstance(b, torch.nn.SyncBatchNorm) for tm in synced_model._training_modules() for b in tm.modules())
    x = torch.rand(B, 3, H, W, generator=gen).to(dev)
    gts = _targets(B, gen).to(dev)
    warm = max(3, args.warmup)
    counts = {}
    built = {}
    for name, m in (('sync_bn', synced_model), ('local_bn', local_model)):
        built[name] = _arm(m, x, gts, world, dist, counter, warm)
        counts[name] = dict(counter.counts)
        counter.counts = {k: 0 for k in counter.counts}
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
            for _ in range(K):
                step()
            t1.record()
            barrier()
            times[name].append(max_over_ranks(t0.elapsed_time(t1)) / K)
    clocks = sampler.stop() if rank == 0 else None
    if rank == 0:
        res = {}
        for name, ms_list in times.items():
            ms = statistics.median(ms_list)
            res[name] = {'ms_per_step': round(ms, 4), 'images_per_sec': round(world * B / (ms / 1e3), 2), 'ms_per_round': [round(v, 4) for v in ms_list]}
        sc = counts['sync_bn']
        line = {'metric': f"images/sec YOLOv6-s training step (YOLOv6(mode='train') + backward + SGD, 640x640, 80 classes) with SyncBatchNorm "
                          f'over {world} GPU(s), bs{B} per GPU',
                'value': res['sync_bn']['images_per_sec'], 'unit': 'images/sec', 'n_gpus': world, 'steps': K, 'warmup': warm, 'rounds': args.rounds,
                'ms_per_step': res['sync_bn']['ms_per_step'], 'higher_is_better': True, 'scaling': 'weak', 'data': 'synthetic',
                'config': {'workload': "YOLOv6-s (coco_yolov6_s.yml USE_MODEL, 80 classes) on 640x640 images: mode='train' (network + YOLOv6Loss), "
                                       'backward, one flat fp32 gradient all-reduce, SGD(momentum)', 'global_batch': world * B, 'per_gpu_batch': B,
                           'gts_total_rank0': int(gts.shape[0]), 'parallelism': f'dp{world}', 'cuda_graph': True, 'sync_bn_layers': n_sync,
                           'numa_node': numa},
                'collectives_per_synced_step': {'forward_all_gather': sc['all_gather_into_tensor'], 'backward_all_reduce': sc['all_reduce'],
                                                'gradient_all_reduce': 1 if world > 1 else 0},
                'arms': res, 'sync_over_local': round(res['sync_bn']['ms_per_step'] / res['local_bn']['ms_per_step'], 4),
                'card': _card(local), 'sm_clock_mhz_in_timed_windows': clocks,
                'note': 'medians over the rounds; the two arms alternate in each round. ' +
                        ('At one GPU SyncBatchNorm runs the local statistics (a world of one): both arms run the same kernels and issue no '
                         'collective, so the cross-rank cost is not measured.' if world == 1 else
                         'Collectives counted on one eager synced step, excluding the gradient all-reduce.')}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
