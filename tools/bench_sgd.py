"""Benchmark of the trainer's optimiser step: cvpytorch_b200.optim.SGD (one launch, csrc/sgd.cu) against torch.optim.SGD, both under
torch.amp.GradScaler, over the groups build_optimizer makes for YOLOX-s and YOLOv5-s (oracle/optim_oracle.param_groups: one group per
tensor), with seeded gradients.  The two arms alternate in one call.  Writes nothing; one JSON line with the card's name and power limit
read in the same call.  Single GPU.

  python tools/bench_sgd.py [--steps 100] [--launches 200]

Per model:
  step_ms          `scaler.step(opt); scaler.update()` wall time, host clock with a device synchronise before and after (median), per arm;
  kernel_us        CUDA-event time of cvb_sgd_step alone over `launches` back-to-back launches, and bound_us = 20 B per element (read param,
                   grad and momentum buffer, write param and buffer) over the data-sheet 3.35 TB/s of the H100 SXM;
  table_builds     how many of the drop-in's `steps` (warm-up included) rebuilt its device table (gradients are re-created every step, as
                   zero_grad(set_to_none=True) leaves them);
  bitwise_equal    params and momentum buffers of the two arms after the timed steps."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

from bench_darknet_train import _card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
DICT80 = [{f'c{i}': 1.0} for i in range(80)]


def _models():
    from cvpytorch_b200 import models as M, synth, yolox_models as XM
    return {'yolox_s': lambda: XM.YOLOX(dictionary=DICT80, model_cfg=dict(synth.YOLOX_CFG)),
            'yolov5_s': lambda: M.YOLOv5(DICT80, dict(synth.YOLOV5S_CFG))}


def _wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def bench(name, build, steps, launches):
    from cvpytorch_b200 import _lib
    from cvpytorch_b200.optim import SGD
    from oracle import optim_oracle as O
    cfg = O.CONFIGS[name]
    model = build().cuda().train()
    params = [g['params'][0] for g in O.param_groups(model, cfg)]
    shadow = {id(p): torch.nn.Parameter(p.detach().clone()) for p in params}
    arms = {'drop_in': (SGD(O.param_groups(model, cfg)), params),
            'torch': (torch.optim.SGD([dict(g, params=[shadow[id(g['params'][0])]]) for g in O.param_groups(model, cfg)]),
                      [shadow[id(p)] for p in params])}
    scalers = {k: torch.amp.GradScaler('cuda', init_scale=2.0 ** 16) for k in arms}
    numel = sum(p.numel() for p in params)
    g = torch.Generator(device='cuda').manual_seed(1)
    times = {k: [] for k in arms}
    for i in range(steps + 5):
        grads = [torch.randn(p.shape, device='cuda', generator=g) * 2.0 ** 10 for p in params]
        for k, (opt, ps) in arms.items():
            for p, gr in zip(ps, grads):
                p.grad = gr.clone()
            scalers[k].scale(torch.ones((), device='cuda'))  # the trainer's scaler.scale(loss): creates the scale on first use
            t = _wall(lambda: (scalers[k].step(opt), scalers[k].update()))
            if i >= 5:
                times[k].append(t)
            opt.zero_grad(set_to_none=True)
    mine, ref = arms['drop_in'][0], arms['torch'][0]
    equal = all(torch.equal(p, shadow[id(p)]) and torch.equal(mine.state[p]['momentum_buffer'], ref.state[shadow[id(p)]]['momentum_buffer'])
                for p in params)
    builds = mine.table_builds
    for p in params:
        p.grad = torch.randn(p.shape, device='cuda', generator=g)
    mine.step()
    table, n = mine._table
    groups = (_lib.CvbSgdGroup * len(mine.param_groups))(*[_lib.CvbSgdGroup(0.0, 0.0, 0.9, _lib.CVB_SGD_MOMENTUM | _lib.CVB_SGD_NESTEROV)
                                                          for _ in mine.param_groups])
    stream = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(launches):  # lr 0: the params stay, the buffers see the same traffic
        _lib.check(L.cvb_sgd_step(table.data_ptr(), n, groups, len(mine.param_groups), None, None, stream))
    e1.record()
    torch.cuda.synchronize()
    kernel_us = e0.elapsed_time(e1) / launches * 1e3
    bound_us = 20 * numel / HBM_BYTES_PER_S * 1e6
    return {'model': name, 'groups': len(params), 'elements': numel,
            'step_ms': {k: round(statistics.median(v), 3) for k, v in times.items()},
            'kernel_us': round(kernel_us, 2), 'bound_us': round(bound_us, 2), 'kernel_share_of_bound': round(bound_us / kernel_us, 3),
            'table_builds': builds, 'steps': steps + 5, 'bitwise_equal': equal}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=100)
    ap.add_argument('--launches', type=int, default=200)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_sgd.py times the H100 path: it needs cuda:0'
    torch.cuda.set_device(0)
    print(json.dumps({'card': _card(0), 'sgd': [bench(k, b, a.steps, a.launches) for k, b in _models().items()]}))


if __name__ == '__main__':
    main()
