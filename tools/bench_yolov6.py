"""YOLOv6-s inference throughput on the H100 kernels: 640², batch 64, through YOLOv6.predict (network + decode + NMS, one device
synchronise per timed window), against the oracle network (oracle/yolov6_oracle.py: the reference's ops in torch, cuDNN, fp32, TF32
off) + its decode on the same GPU.  Seeded weights (oracle.yolov6_oracle.seeded_state_dict).  Warm-up, then CUDA events around
`--iters` calls for each side, alternated `--rounds` times; reads the card name and power limit in the same run.
Prints one JSON line.  Usage: python tools/bench_yolov6.py [--batch 64] [--size 640] [--iters 20] [--rounds 3]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cvpytorch_b200 import yolov6_models as M  # noqa: E402
from oracle import yolov6_oracle as V6  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def timed(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--size', type=int, default=640)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_yolov6: needs a CUDA device')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    dev = torch.device('cuda:0')
    dictionary = [{f'c{i}': 1.0} for i in range(80)]
    cfg = dict(TYPE='yolov6_s', BACKBONE={'name': 'YOLOv6EfficientRep', 'out_stages': [1, 2, 3, 4], 'output_stride': 32, 'pretrained': False},
               NECK={'name': 'YOLOv6RepBiPAN', 'in_channels': [128, 256, 512, 1024], 'mid_channels': [128, 128, 256],
                     'out_channels': [128, 256, 512], 'num_blocks': [12, 12, 12, 12]},
               HEAD={'name': 'YOLOv6Effidehead', 'num_classes': 80, 'in_channels': [128, 256, 512], 'use_dfl': False, 'fuse_ab': False},
               DETECT={'name': 'YOLOv6Detect', 'num_classes': 80, 'in_channels': [128, 256, 512], 'use_dfl': False, 'fuse_ab': False},
               LOSS={'name': 'YOLOv6Loss', 'num_classes': 80})
    m = M.YOLOv6(dictionary, cfg)
    sd = V6.seeded_state_dict([(k, v.shape) for k, v in m.state_dict().items()], 616)
    m.load_state_dict(sd, strict=True)
    m = m.to(dev).eval()
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    x = torch.randn(a.batch, 3, a.size, a.size, generator=torch.Generator().manual_seed(1)).to(dev)

    def ours():
        m.predict(x)

    def torch_ref():
        V6.forward(x, sd_dev)

    for _ in range(3):  # warm-up: graph build, plans, cuDNN algorithm choice
        ours()
        torch_ref()
    torch.cuda.synchronize()
    t_ours, t_ref = [], []
    for _ in range(a.rounds):
        t_ours.append(timed(ours, a.iters))
        t_ref.append(timed(torch_ref, a.iters))
    z = m._graph_for(x)['z'][:2].float().cpu()
    zo = V6.forward(x[:2].cpu(), sd)[0]
    best_o, best_r = min(t_ours), min(t_ref)
    print(json.dumps(dict(model='yolov6_s', batch=a.batch, size=a.size, card=card(), ours_img_s=round(a.batch / best_o, 1),
                          torch_cudnn_img_s=round(a.batch / best_r, 1), ours_ms=[round(t * 1e3, 2) for t in t_ours],
                          torch_ms=[round(t * 1e3, 2) for t in t_ref], speedup=round(best_r / best_o, 3), z_rel_err=V6.rel_err(z, zo))))


if __name__ == '__main__':
    main()
