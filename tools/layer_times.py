"""Per-layer timing of the fused YOLOv5-s graph on the GPU (CUDA events, L2 flushed between repetitions).
Prints one row per step: name, shape, ms, algorithmic TFLOP/s, algorithmic GB/s (split16 = 4 B/elt in+out+weights),
and the two per-layer roofline bounds (tensor: 3x fp16 MMA work on the measured bf16 peak; HBM: measured copy peak)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from cvpytorch_b200 import synth  # noqa: E402


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
    which = sys.argv[2] if len(sys.argv) > 2 else 'yolov5s'
    reps = 5
    dev = torch.device('cuda:0')
    SH = SW = 640
    if which == 'fcos':
        model, SH, SW = synth.build_fcos(True), 800, 800
    elif which == 'deeplab':
        model, SH, SW = synth.build_deeplab(True), 1024, 2048
    elif which == 'yolox':
        model = synth.build_yolox(True)
    else:
        model = synth.build_yolov5s(True)
    G = model.build_graph(B, SH, SW, dev)
    g = G['g']
    torch.manual_seed(1029)
    G['holder']['x'] = torch.randn(B, 3, SH, SW, device=dev)
    g.run()
    torch.cuda.synchronize()
    peaks = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json'))) if os.path.exists(os.path.join(ROOT, 'MEASURED_PEAKS.json')) else {}
    # without measured peaks: the H100 SXM data-sheet rates (dense bf16, HBM3) that DESIGN.md and BASELINE.md use
    P = float(peaks.get('bf16_tflops', 989.0))
    BW = float(peaks.get('hbm_gbs', 3350.0))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    rows = []
    li = 0
    tot = tot_bound = 0.0
    for kind, obj in g.steps:
        ts = []
        for _ in range(reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            if kind == 'conv':
                obj.run()
            else:
                obj()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ms = sorted(ts)[len(ts) // 2]
        tot += ms
        if kind == 'conv':
            name, cin, cout, k, s, Ho, Wo = g.layer_log[li]
            li += 1
            flops = 2.0 * B * Ho * Wo * cout * cin * k * k
            in_elems = B * (Ho * s) * (Wo * s) * cin  # (stem rows report the s2d view)
            byts = 4.0 * (in_elems + B * Ho * Wo * cout) + 4.0 * cout * cin * k * k
            t_tensor = 3 * flops / (P * 1e12) * 1e3
            t_hbm = byts / (BW * 1e9) * 1e3
            bound = max(t_tensor, t_hbm)
            tot_bound += bound
            rows.append(f'{name:34s} {cin:4d}->{cout:4d} k{k} s{s} {Ho:3d}x{Wo:<3d} {ms:8.4f} ms  {flops / ms / 1e9:8.1f} TF/s  {byts / ms / 1e6:8.1f} GB/s  '
                        f'bound {bound:7.4f} ms ({"T" if t_tensor > t_hbm else "M"})  frac {bound / ms:5.2f}')
        else:
            rows.append(f'{"<aux step>":34s} {"":31s} {ms:8.4f} ms')
    print('\n'.join(rows))
    print(f'sum of per-step medians: {tot:.3f} ms  (B={B}, {which}) -> {B / tot * 1e3:.0f} img/s; sum of per-layer conv bounds {tot_bound:.3f} ms; peaks: {P} TF/s, {BW} GB/s')


if __name__ == '__main__':
    main()
