"""Benchmark of the segmentation loss on the H100 kernels (csrc/seg_loss.cu, seg_train.CrossEntropyLoss2d) against the torch path
(F.interpolate + F.cross_entropy + backward) on the same tensors.  Writes nothing; one JSON line, CUDA-event times after warm-up, the
card's name and power limit read in the same call.  Single GPU.

  python tools/bench_seg_loss.py [--steps 50] [--warmup 5]

Shapes: DeepLabv3+ Cityscapes training (8 x 19 x 128x256 -> 512x1024) with uint8 and with int64 labels, and PSPNet's auxiliary head (x8:
8 x 19 x 64x128 -> 512x1024, loss_weight 0.4).  Per shape:
1. forward + backward, eager and captured as one CUDA graph, for both paths;
2. the kernels' own times from torch.profiler (a separate run), the bytes they need (preds read twice, the gradient written once, the
   labels read twice, the saved lse written and read) over that time against the H100 SXM data-sheet 3.35 TB/s, and the exponentials;
3. torch.cuda.max_memory_allocated above the inputs for one forward + backward of each path;
4. the loss and gradient difference between the paths."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench_darknet_train import _card  # noqa: E402
from bench_fcos_loss import _kernel_times  # noqa: E402
from bench_yolox_loss import _capture, _time  # noqa: E402

HBM_TBS = 3.35
KERNELS = ('seg_ce_fwd_kernel', 'seg_ce_final_kernel', 'seg_ce_bwd_kernel')


def _inputs(B, C, h, w, H, W, dtype, gen, dev):
    pred = (torch.randn(B, C, h, w, generator=gen) * 3).to(dev)
    target = torch.randint(0, C, (B, H, W), generator=gen)
    target[torch.rand(B, H, W, generator=gen) < 0.1] = 255
    return pred, target.to(dtype).to(dev)


def _peak(fn):
    """Bytes allocated above the current level at the peak of one call."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def _shape(name, B, C, h, w, H, W, dtype, lw, K, warmup, gen, dev):
    from cvpytorch_b200 import seg_train as ST
    pred, target = _inputs(B, C, h, w, H, W, dtype, gen, dev)
    loss = ST.CrossEntropyLoss2d(loss_weight=lw)
    p = pred.clone().requires_grad_(True)
    q = pred.clone().requires_grad_(True)

    def fused():
        p.grad = None
        loss(p, target).backward()

    def torch_path():
        q.grad = None
        up = F.interpolate(q, size=(H, W), mode='bilinear', align_corners=False)
        (lw * F.cross_entropy(up, target.long(), ignore_index=255)).backward()

    res = {'shape': name, 'B': B, 'C': C, 'in': [h, w], 'out': [H, W], 'labels': str(dtype).replace('torch.', ''), 'loss_weight': lw}
    for tag, fn in (('fused', fused), ('torch', torch_path)):
        for _ in range(warmup):
            fn()
        res[f'{tag}_eager_ms'] = round(_time(fn, K), 4)
        graph = _capture(fn)
        for _ in range(warmup):
            graph.replay()
        res[f'{tag}_graph_ms'] = round(_time(graph.replay, K), 4)
        del graph
        res[f'{tag}_peak_mb'] = round(_peak(fn) / 2 ** 20, 1)
    res['speedup_graph'] = round(res['torch_graph_ms'] / res['fused_graph_ms'], 1)
    res['speedup_eager'] = round(res['torch_eager_ms'] / res['fused_eager_ms'], 1)
    fused()
    torch_path()
    lf = float(loss(p.detach(), target))
    lt = float(lw * F.cross_entropy(F.interpolate(q.detach(), size=(H, W), mode='bilinear', align_corners=False), target.long(), ignore_index=255))
    res['loss'] = [lf, lt]
    res['loss_rel_diff'] = abs(lf - lt) / abs(lt)
    res['grad_rel_diff'] = float((p.grad - q.grad).abs().max() / q.grad.abs().max())
    kt = _kernel_times(fused, KERNELS)
    us = sum(kt.values())
    px = B * H * W
    need = 3 * B * C * h * w * 4 + 2 * px * target.element_size() + 2 * px * 4
    res['kernel_us'] = {k: round(v, 2) for k, v in kt.items()}
    res['kernels'] = {'us': round(us, 2), 'bytes': need, 'tb_per_s': round(need / us / 1e6, 3) if us else None,
                      'bound_us_at_3.35_tbs': round(need / (HBM_TBS * 1e6), 2), 'exps': 2 * px * C,
                      'torch_full_res_bytes_estimate': 9 * B * C * H * W * 4}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50, help='timed calls per arm')
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_seg_loss.py: no CUDA device; the loss has no CPU fallback')
    dev = torch.device('cuda:0')
    gen = torch.Generator().manual_seed(2026)
    K, wu = args.steps, max(3, args.warmup)
    shapes = [_shape('deeplabv3plus_cityscapes_u8', 8, 19, 128, 256, 512, 1024, torch.uint8, 1.0, K, wu, gen, dev),
              _shape('deeplabv3plus_cityscapes_i64', 8, 19, 128, 256, 512, 1024, torch.int64, 1.0, K, wu, gen, dev),
              _shape('pspnet_aux_x8', 8, 19, 64, 128, 512, 1024, torch.uint8, 0.4, K, wu, gen, dev)]
    line = {'metric': 'ms seg CE loss fwd+bwd (8x19x128x256 -> 512x1024, uint8 labels), CUDA graph', 'value': shapes[0]['fused_graph_ms'],
            'unit': 'ms', 'n_gpus': 1, 'steps': K, 'warmup': wu, 'higher_is_better': False, 'data': 'synthetic', 'card': _card(0),
            'shapes': shapes,
            'library_baseline': {'what': 'F.interpolate(bilinear, align_corners=False) + F.cross_entropy(ignore_index=255) + backward, fp32, '
                                         'same GPU tensors'}}
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
