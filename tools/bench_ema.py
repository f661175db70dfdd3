"""Benchmark of the model EMA update (csrc/ema.cu through cvpytorch_b200.ema.ModelEMA) against the reference's semantics in eager torch
(oracle/ema_oracle.ModelEMA: three ATen launches per floating entry), on the YOLOX-s and YOLOv5-s state dicts, alternating the two in one
call.  Writes nothing; one JSON line with the card's name and power limit read in the same call.  Single GPU.

  python tools/bench_ema.py [--updates 200] [--steps 20] [--batch 16]

Per model:
  update_ms      wall time of one update(model), host clock around the call with a device synchronise before and after (median);
  kernel_us      CUDA-event time of cvb_ema_update alone over `updates` back-to-back launches of the model's table, and bound_us = the bytes it
                 must move (read ema and src, write ema: 12 B per element) over the data-sheet 3.35 TB/s of the H100 SXM;
  check_ms       the drop-in's host cost per update: two state_dict(keep_vars=True) walks and the table signature (median);
  oracle_ms      wall time of the same update by the eager oracle (median).
Trainer step (YOLOX-s, 640², eager, as trainer_det_yolox.py runs it): YOLOX(imgs, targets, 'train') + backward + SGD + ema.update(model),
CUDA-event time per step with either EMA, alternated."""
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


def _seeded(model, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for v in model.state_dict().values():
            if v.dtype.is_floating_point:
                v.copy_(torch.randn(v.shape, generator=g))
    return model


def _wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def bench_update(name, build, updates):
    from cvpytorch_b200 import _lib
    from cvpytorch_b200.ema import ModelEMA
    from oracle import ema_oracle as O
    model = _seeded(build().cuda().train(), 1)
    mine, ref = ModelEMA(model), O.ModelEMA(model)
    sd = model.state_dict()
    numel = sum(v.numel() for v in sd.values() if v.dtype.is_floating_point)
    for _ in range(5):
        mine.update(model)
        ref.update(model)
    t_mine, t_ref, t_check = [], [], []
    for _ in range(updates):
        t_ref.append(_wall(lambda: ref.update(model)))
        t_mine.append(_wall(lambda: mine.update(model)))
        t0 = time.perf_counter()
        pairs = mine._pairs(model)
        _ = [(e.data_ptr(), s.data_ptr(), e.dtype, s.dtype, e.shape, s.shape, e.is_contiguous(), s.is_contiguous()) for _, e, s in pairs]
        t_check.append((time.perf_counter() - t0) * 1e3)
    assert all(torch.equal(a, b) for a, b in zip(mine.ema.state_dict().values(), ref.ema.state_dict().values()))
    table, n = mine._table
    stream = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(updates):
        _lib.check(L.cvb_ema_update(table.data_ptr(), n, 0.9999, 1 - 0.9999, stream))
    e1.record()
    torch.cuda.synchronize()
    kernel_us = e0.elapsed_time(e1) / updates * 1e3
    bound_us = 12 * numel / HBM_BYTES_PER_S * 1e6
    return {'model': name, 'entries': n, 'elements': numel, 'update_ms': round(statistics.median(t_mine), 3),
            'oracle_ms': round(statistics.median(t_ref), 3), 'check_ms': round(statistics.median(t_check), 3),
            'kernel_us': round(kernel_us, 2), 'bound_us': round(bound_us, 2), 'kernel_share_of_bound': round(bound_us / kernel_us, 3),
            'oracle_launches_per_update': 3 * n}


def bench_step(steps, B):
    from cvpytorch_b200.ema import ModelEMA
    from oracle import ema_oracle as O
    model = _seeded(_models()['yolox_s']().cuda().train(), 2)
    g = torch.Generator().manual_seed(3)
    imgs = torch.randn(B, 3, 640, 640, generator=g).cuda()
    targets = []
    for _ in range(B):
        n = int(torch.randint(2, 21, (1,), generator=g))
        c = 40 + torch.rand(n, 2, generator=g) * 560
        targets.append({'labels': torch.randint(0, 80, (n,), generator=g).cuda(), 'boxes': torch.cat([c, 16 + torch.rand(n, 2, generator=g) * 200], 1).cuda()})
    opt = torch.optim.SGD(model.parameters(), lr=1e-4, momentum=0.9)
    emas = {'oracle': O.ModelEMA(model), 'drop_in': ModelEMA(model)}

    def step(ema):
        model(imgs, targets, 'train')['loss'].backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        ema.update(model)
    for ema in emas.values():
        for _ in range(3):
            step(ema)
    times = {k: [] for k in emas}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(steps):
        for k, ema in emas.items():
            torch.cuda.synchronize()
            e0.record()
            step(ema)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
    return {'batch': B, 'step_ms_oracle_ema': round(statistics.median(times['oracle']), 3),
            'step_ms_drop_in_ema': round(statistics.median(times['drop_in']), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--updates', type=int, default=200)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--batch', type=int, default=16)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_ema.py times the H100 path: it needs cuda:0'
    torch.cuda.set_device(0)
    out = {'card': _card(0), 'update': [bench_update(k, b, a.updates) for k, b in _models().items()]}
    if a.steps > 0:
        out['trainer_step'] = bench_step(a.steps, a.batch)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
