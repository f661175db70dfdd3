"""Benchmark of the YOLOX loss on the H100 kernels (csrc/yolox_loss.cu) and of the whole YOLOX-s training step with it.  Writes nothing; one
JSON line, CUDA-event times after warm-up, the card's name and power limit read in the same call.  Single GPU.

  python tools/bench_yolox_loss.py [--steps 20] [--warmup 5] [--batch 16]

1. The loss forward + backward alone (train.YOLOXLoss, YOLOX-s 640² head outputs, 80 classes, 8 to 100 seeded GTs per image) captured as one
   CUDA graph, next to the oracle loss (oracle/yolox_loss_oracle.py, ATen, eager) on the same GPU tensors.
2. The full YOLOX(mode='train') + SGD step as one CUDA graph, next to the stand-in-gradient step of tools/bench_yolox_train.py (the same
   network and optimiser, the head outputs' gradients given instead of computed by the loss)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

from bench_darknet_train import _card  # noqa: E402

STRIDES = (8, 16, 32)
NC = 80
H = W = 640


def _inputs(B, gen, dev):
    """Head outputs [B, 85, h + 2, w + 2] with 70 % of the anchors near a GT predicting a jittered copy of it, and targets [B, 100, 5]."""
    counts = [int(torch.randint(8, 101, (1,), generator=gen)) for _ in range(B)]
    t = torch.zeros(B, max(counts), 5)
    for b, n in enumerate(counts):
        wh = 12 + torch.rand(n, 2, generator=gen) * 200
        t[b, :n] = torch.cat([torch.randint(0, NC, (n, 1), generator=gen).float(), torch.rand(n, 2, generator=gen) * 640, wh], 1)
    preds = []
    for s in STRIDES:
        h, w = H // s + 2, W // s + 2
        p = torch.randn(B, 5 + NC, h, w, generator=gen)
        p[:, 4:] = p[:, 4:] * 1.5 - 3.0
        yv, xv = torch.meshgrid(torch.arange(h).float(), torch.arange(w).float(), indexing='ij')
        for b, n in enumerate(counts):
            pick = torch.randint(0, n, (h, w), generator=gen)
            _, cx, cy, bw, bh = (t[b, :n, i][pick] for i in range(5))
            take = ((xv + 0.5) * s - cx).abs().lt(2.5 * s + bw / 2) & ((yv + 0.5) * s - cy).abs().lt(2.5 * s + bh / 2)
            take &= torch.rand(h, w, generator=gen) < 0.7
            p[b, 0] = torch.where(take, cx / s - xv + 0.1 * torch.randn(h, w, generator=gen), p[b, 0])
            p[b, 1] = torch.where(take, cy / s - yv + 0.1 * torch.randn(h, w, generator=gen), p[b, 1])
            p[b, 2] = torch.where(take, torch.log(bw / s), p[b, 2])
            p[b, 3] = torch.where(take, torch.log(bh / s), p[b, 3])
        preds.append(p.to(dev))
    return preds, t.to(dev), sum(counts)


def _time(fn, K):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(K):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / K


def _capture(fn):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return graph


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20, help='timed steps')
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--batch', type=int, default=16, help='images per step')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_yolox_loss.py: no CUDA device; the loss has no CPU fallback')
    from cvpytorch_b200 import synth, train as T, yolox_models as XM
    from oracle import yolox_loss_oracle as LO, yolox_train_oracle as XO
    dev = torch.device('cuda:0')
    B, K = args.batch, args.steps
    gen = torch.Generator().manual_seed(2024)
    preds, targets, ngt = _inputs(B, gen, dev)

    # 1. the loss alone
    loss = T.YOLOXLoss(NC)
    ps = [p.clone().requires_grad_(True) for p in preds]

    def loss_step():
        for p in ps:
            p.grad = None
        loss(ps, targets)['loss'].backward()
    g_loss = _capture(loss_step)
    for _ in range(max(3, args.warmup)):
        g_loss.replay()
    loss_ms = _time(g_loss.replay, K)
    num_fg = float(loss(ps, targets)['num_fg'])
    qs = [p.clone().requires_grad_(True) for p in preds]

    def oracle_step():
        for q in qs:
            q.grad = None
        LO.losses(qs, targets, STRIDES, NC)[0]['loss'].backward()
    for _ in range(2):
        oracle_step()
    oracle_ms = _time(oracle_step, 3)

    # 2. the whole training step, with the loss and with stand-in head-output gradients
    model = XM.YOLOX(dictionary=[{f'c{i}': 1.0} for i in range(NC)], model_cfg=dict(synth.YOLOX_CFG))
    model.load_state_dict(XO.synthetic_state([(k, tuple(v.shape)) for k, v in model.state_dict().items()]), strict=False)
    model.to(dev).train()
    params = list(model.parameters())
    opt = torch.optim.SGD(params, lr=1e-4, momentum=0.9)
    x = torch.randn(B, 3, H, W, generator=gen).to(dev)
    Gs = [torch.randn(p.shape, generator=gen).to(dev) for p in preds]
    bb, nk, hd = model._training_modules()

    def train_step():
        model(x, targets, 'train')['loss'].backward()
        opt.step()
        opt.zero_grad(set_to_none=True)

    def standin_step():
        torch.autograd.backward(hd.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(x))), Gs)
        opt.step()
        opt.zero_grad(set_to_none=True)
    res = {}
    for name, fn in (('with_loss', train_step), ('stand_in', standin_step)):
        graph = _capture(fn)
        for _ in range(max(3, args.warmup)):
            graph.replay()
        res[name] = _time(graph.replay, K)
        del graph
    line = {'metric': 'ms YOLOX loss fwd+bwd (YOLOX-s 640x640 head outputs, 80 classes, bs%d), CUDA graph' % B, 'value': round(loss_ms, 4),
            'unit': 'ms', 'n_gpus': 1, 'steps': K, 'warmup': max(3, args.warmup), 'higher_is_better': False, 'data': 'synthetic',
            'config': {'batch': B, 'gts_total': ngt, 'gts_per_image': '8 to 100 (seeded)', 'num_fg_ratio': round(num_fg, 3), 'anchors_per_image': 8972},
            'card': _card(0),
            'library_baseline': {'what': 'oracle/yolox_loss_oracle.losses fwd + bwd (ATen, eager, per-image loop) on the same GPU tensors',
                                 'ms': round(oracle_ms, 3)},
            'train_step': {'what': "YOLOX(mode='train') + SGD(momentum) as one CUDA graph, YOLOX-s 640x640, bf16 kernels, fp32 head outputs",
                           'ms_with_loss': round(res['with_loss'], 3), 'ms_stand_in_gradients': round(res['stand_in'], 3),
                           'loss_share': round((res['with_loss'] - res['stand_in']) / res['with_loss'], 4)}}
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
