"""Benchmark of the YOLOv6-s training step on the H100 kernels: YOLOv6(mode='train') + backward + SGD as one CUDA graph.  Writes nothing;
one JSON line, CUDA-event times after warm-up, the card's name, power limit and maximum SM clock read by one nvidia-smi query, and the SM
clock sampled during each timed window.  Single GPU.

  python tools/bench_yolov6_train.py [--steps 20] [--warmup 5] [--batch 64]

The batch default is conf/det/yolov6/coco_yolov6_s.yml's 64, at 640², 80 classes; targets: 2 to 20 seeded boxes per image.  The loss's
share of the step is (step with the loss - step with stand-in head-output gradients) / step.  centre_tap: the five stride-2 1x1 RepVGG
branches (the stem and the four downsamples) run as zero-padded 3x3 / stride-2 convs; their forward, backward-weight and backward-data
convs are timed alone, and 8/9 of that is the MMA work a k = 1 / stride-2 conv path would not do.  Baseline: the oracle network
(oracle/yolov6_train_oracle.py) + the oracle loss (oracle/yolov6_loss_oracle.py) + SGD in eager PyTorch under bf16 autocast,
channels_last, cuDNN, on the same GPU."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

from bench_yolov5_train import _targets, _time_with_clock  # noqa: E402
from bench_yolox_loss import _capture  # noqa: E402

NC = 80
H = W = 640
CFG = dict(TYPE='yolov6_s',
           BACKBONE={'name': 'YOLOv6EfficientRep', 'out_stages': [1, 2, 3, 4], 'output_stride': 32, 'pretrained': False},
           NECK={'name': 'YOLOv6RepBiPAN', 'in_channels': [128, 256, 512, 1024], 'mid_channels': [128, 128, 256], 'out_channels': [128, 256, 512],
                 'num_blocks': [12, 12, 12, 12]},
           HEAD={'name': 'YOLOv6Effidehead', 'num_classes': NC, 'in_channels': [128, 256, 512], 'use_dfl': False, 'fuse_ab': False},
           DETECT={'name': 'YOLOv6Detect', 'num_classes': NC, 'in_channels': [128, 256, 512], 'use_dfl': False, 'fuse_ab': False},
           LOSS={'name': 'YOLOv6Loss', 'num_classes': NC})  # conf/det/yolov6/coco_yolov6_s.yml USE_MODEL


def _card():
    """One read-only nvidia-smi query of GPU 0: the card's name, power limit (W) and maximum SM clock (MHz)."""
    import subprocess
    try:
        out = subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=20)
        name, power, clock = (v.strip() for v in out.stdout.strip().splitlines()[0].split(','))
        return {'name': name, 'power_limit_w': float(power), 'max_sm_clock_mhz': float(clock)}
    except Exception:  # noqa: BLE001
        return {'name': torch.cuda.get_device_name(0), 'power_limit_w': None, 'max_sm_clock_mhz': None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20, help='timed steps')
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--batch', type=int, default=64, help='images per step')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_yolov6_train.py: no CUDA device; the training path has no CPU fallback')
    from cvpytorch_b200 import train as T, yolov6_models as M
    from oracle import yolov6_loss_oracle as LO, yolov6_train_oracle as O
    dev = torch.device('cuda:0')
    B, K, warm = args.batch, args.steps, max(3, args.warmup)
    gen = torch.Generator().manual_seed(2024)
    model = M.YOLOv6([{f'c{i}': 1.0} for i in range(NC)], dict(CFG)).to(dev).train()
    params = list(model.parameters())
    opt = torch.optim.SGD(params, lr=1e-4, momentum=0.9)
    x = torch.rand(B, 3, H, W, generator=gen).to(dev)
    gts = _targets(B, gen).to(dev)
    bb, nk, hd = model._training_modules()
    with torch.no_grad():
        _, _, d0 = hd.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(x)))
    G = torch.randn(d0.shape, generator=gen).to(dev) * 1e-3

    def train_step():
        model(x, gts, 'train')['loss'].backward()
        opt.step()
        opt.zero_grad(set_to_none=True)

    def standin_step():
        (hd.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(x)))[2] * G).sum().backward()
        opt.step()
        opt.zero_grad(set_to_none=True)

    # the centre-tap branches: each stride-2 RepVGG block's 1x1 weight zero-padded to 3x3, at the block's input shape
    shapes, h = [], None
    with torch.no_grad():
        h = T.focus_s2d(x)
        shapes.append((h.shape, 16, bb.stem.out_channels, 1))  # the stem: a stride-1 3x3 over the space-to-depth map
        h = bb.stem(x)
        for i in range(1, 5):
            blk = getattr(bb, f'stage{i}')[0]
            shapes.append((h.shape, blk.in_channels, blk.out_channels, 2))
            h = getattr(bb, f'stage{i}')(h)
    branch = []
    for shp, cin, cout, s in shapes:
        xb = torch.randn(shp, generator=gen).to(dev).bfloat16()
        wf, wb = T.pack_weights(torch.randn(cout, cin, 3, 3, generator=gen).to(dev) * 1e-2)
        y = T.conv(xb, wf, cout, 3, stride=s)
        branch.append((xb, wf, wb, cout, s, torch.randn(y.shape, generator=gen).to(dev).bfloat16()))

    def branch_step():
        for xb, wf, wb, cout, s, dy in branch:
            T.conv(xb, wf, cout, 3, stride=s)
            T.conv_wgrad(xb, dy, 3, s)
            if s == 2:
                T.conv_dgrad_s2(dy, wb, xb.shape[3], xb.shape[1], xb.shape[2])
    res, clocks = {}, {}
    for name, fn in (('with_loss', train_step), ('stand_in', standin_step), ('centre_tap', branch_step)):
        graph = _capture(fn)
        for _ in range(warm):
            graph.replay()
        res[name], clocks[name] = _time_with_clock(graph.replay, K)
        del graph

    # baseline: the oracle network + the oracle loss + SGD, eager, bf16 autocast, channels_last, cuDNN
    torch.backends.cudnn.benchmark = True
    sd = {k: (v.detach().clone(memory_format=torch.channels_last) if v.dim() == 4 else v.detach().clone())
          .requires_grad_(v.dtype.is_floating_point and 'running_' not in k and 'proj' not in k)
          for k, v in model.state_dict().items() if k.startswith(('backbone.', 'neck.', 'head.'))}
    leaves = [v for v in sd.values() if v.requires_grad]
    base_opt = torch.optim.SGD(leaves, lr=1e-4, momentum=0.9)
    xc = x.to(memory_format=torch.channels_last)
    lshapes = LO.level_shapes(H, W)

    def baseline_step():
        with torch.autocast('cuda', dtype=torch.bfloat16):
            _, s, d = O.network(xc, sd)
        out, _ = LO.losses(lshapes, s.float().detach(), d.float(), gts, 'atss', 'giou', NC)
        (out['iou'] + out['dfl'] + out['class']).backward()
        base_opt.step()
        base_opt.zero_grad(set_to_none=True)
    for _ in range(warm):
        baseline_step()
    res['baseline'], clocks['baseline'] = _time_with_clock(baseline_step, K)
    line = {'metric': "ms YOLOv6-s training step (YOLOv6(mode='train') + backward + SGD, 640x640, 80 classes, bs%d), CUDA graph" % B,
            'value': round(res['with_loss'], 3), 'unit': 'ms', 'n_gpus': 1, 'steps': K, 'warmup': warm, 'higher_is_better': False, 'data': 'synthetic',
            'img_per_s': round(B * 1000.0 / res['with_loss'], 1),
            'config': {'batch': B, 'gts_total': int(gts.shape[0]), 'gts_per_image': '2 to 20 (seeded)', 'assigner': 'atss'},
            'card': _card(),
            'sm_clock_mhz_in_timed_windows': clocks,
            'baseline': {'what': 'oracle/yolov6_train_oracle.network + yolov6_loss_oracle.losses + SGD, eager PyTorch, bf16 autocast, channels_last, '
                                 'cuDNN, same GPU', 'ms': round(res['baseline'], 3), 'img_per_s': round(B * 1000.0 / res['baseline'], 1)},
            'ms_stand_in_gradients': round(res['stand_in'], 3),
            'loss_share': round((res['with_loss'] - res['stand_in']) / res['with_loss'], 4),
            'centre_tap': {'what': 'fwd + wgrad + dgrad of the five zero-padded stride-2 1x1 branches, one CUDA graph',
                           'ms': round(res['centre_tap'], 3), 'extra_ms_est': round(res['centre_tap'] * 8 / 9, 3),
                           'share_of_step': round(res['centre_tap'] * 8 / 9 / res['with_loss'], 4)}}
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
