"""YOLOv5 training on the H100: the loss (csrc/yolov5_loss.cu, yolov5_train.YOLOv5Loss), the chained SPPF pools, the 6x6 stem and the
model-level training forward (models.YOLOv5, mode='train').

The loss is checked against oracle/yolov5_train_oracle.py (fp32 torch on the CPU, which restates the reference): the candidate lists
exactly, the loss terms within 1e-5 relative and the detect-output gradients within 1e-5 max-normalised."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
ANCHORS = [[[1.25, 1.625], [2.0, 3.75], [4.125, 2.875]],
           [[1.875, 3.8125], [3.875, 2.8125], [3.6875, 7.4375]],
           [[3.625, 2.8125], [4.875, 6.1875], [11.65625, 10.1875]]]


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def _preds(B, nc, size, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn((B, 3 * (5 + nc), size // s, size // s), generator=g) * 1.5).cuda() for s in (8, 16, 32)]


def _targets(B, nt, nc, seed, awkward=True):
    """nt random rows (image, class, cx, cy, w, h) plus, with `awkward`, the cases the candidate logic branches on: GTs on integer grid
    coordinates (all 5 offsets), border GTs (the clamp reaching tbox), a GT the ratio filter drops, two GTs on one cell, a class outside
    [0, nc); image B - 1 stays empty when B > 1."""
    g = torch.Generator().manual_seed(seed)
    imgs = max(B - 1, 1)
    rows = torch.cat([torch.randint(0, imgs, (nt, 1), generator=g).float(), torch.randint(0, nc, (nt, 1), generator=g).float(),
                      torch.rand((nt, 2), generator=g) * 0.9 + 0.05, torch.rand((nt, 2), generator=g) * 0.3 + 0.02], 1)
    if awkward:
        extra = torch.tensor([[0, 0, 0.25, 0.5, 0.1, 0.12],        # integer coordinates on every level of a 256 / 640 map: 5 offsets
                              [0, nc - 1, 1.0, 1.0, 0.05, 0.06],      # borders: the centre cell clamps, tbox uses the clamped cell
                              [0, 0, 0.5, 0.5, 0.9, 0.004],           # extreme ratio: dropped on most anchors
                              [0, 0, 0.3, 0.3, 0.1, 0.1], [0, nc - 1, 0.3001, 0.3001, 0.11, 0.09],  # the same cells
                              [0, nc + 3, 0.6, 0.7, 0.2, 0.2]])       # class outside [0, nc)
        rows = torch.cat([rows, extra], 0)
    return rows.cuda()


def _kernel(preds, targets, nc, scale=1.0):
    from cvpytorch_b200 import yolov5_train as V
    ps = [p.detach().clone().requires_grad_(True) for p in preds]
    loss, items = V.YOLOv5Loss(nc, anchors=ANCHORS)(ps, targets)
    (loss * scale).backward()
    return loss.detach(), items, [p.grad for p in ps]


def _oracle(preds, targets, nc):
    from oracle import yolov5_train_oracle as O
    ps = [p.detach().cpu().clone().requires_grad_(True) for p in preds]
    loss, items, tg = O.yolov5_loss(ps, targets.cpu(), torch.tensor(ANCHORS), nc)
    loss.backward()
    return loss.detach(), items, [p.grad for p in ps], O.candidate_lists(tg, preds[0].shape[0])


def _check(preds, targets, nc):
    from cvpytorch_b200 import yolov5_train as V
    loss, items, grads = _kernel(preds, targets, nc)
    oloss, oitems, ograds, ocand = _oracle(preds, targets, nc)
    _, (ci, cb, nca), _ = V.yolov5_loss_forward([p.float().contiguous() for p in preds], targets, torch.tensor(ANCHORS), (4.0, 1.0, 0.4),
                                                (4.0, 0.05, 1.0, 0.5, 1.0), nc)
    for l, (oi, ob) in enumerate(ocand):
        n = int(nca[l])
        assert n == oi.shape[0], (l, n, oi.shape[0])
        assert torch.equal(ci[l, :n].cpu(), oi), l
        assert torch.equal(cb[l, :n].cpu().view(torch.int32), ob.contiguous().view(torch.int32)), l  # (tbox and anchor bits)
    assert _rel(loss, oloss) < 1e-5, (loss, oloss)
    for a, b in zip(items, oitems):
        assert abs(float(a) - float(b)) <= 1e-5 * max(abs(float(b)), 1e-12) + 1e-12, (items, oitems)
    for g, og in zip(grads, ograds):
        assert _rel(g, og) < 1e-5


def test_loss_awkward_targets(cuda):
    _check(_preds(4, 80, 256, 0), _targets(4, 12, 80, 1), 80)


@pytest.mark.parametrize('B', [1, 2, 16])
@pytest.mark.parametrize('nc', [1, 3, 80])
def test_loss_matrix(cuda, B, nc):
    _check(_preds(B, nc, 128, B * 100 + nc), _targets(B, 3 * B + 1, nc, B + nc), nc)


def test_loss_no_targets(cuda):
    _check(_preds(2, 80, 128, 5), torch.zeros((0, 6), device='cuda'), 80)


def test_loss_640_shapes(cuda):
    _check(_preds(4, 80, 640, 7), _targets(4, 40, 80, 8), 80)


def test_loss_bitwise_reproducible_graph_replay_and_grad_scaling(cuda):
    from cvpytorch_b200 import yolov5_train as V
    preds, targets = _preds(8, 80, 256, 9), _targets(8, 30, 80, 10)
    a, b = _kernel(preds, targets, 80), _kernel(preds, targets, 80)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and all(torch.equal(x, y) for x, y in zip(a[2], b[2]))
    s = _kernel(preds, targets, 80, scale=1024.0)
    for x, y in zip(s[2], a[2]):
        assert _rel(x, y * 1024.0) < 1e-6

    ps = [p.detach().clone().requires_grad_(True) for p in preds]
    crit = V.YOLOv5Loss(80, anchors=ANCHORS)

    def run():
        for p in ps:
            p.grad = None
        loss, _ = crit(ps, targets)
        loss.backward()
        return loss
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = run()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static.detach(), a[0])
    assert all(torch.equal(p.grad, g) for p, g in zip(ps, a[2]))


def test_loss_accepts_reference_views(cuda):
    from cvpytorch_b200 import yolov5_train as V
    preds, targets = _preds(2, 80, 128, 11), _targets(2, 5, 80, 12)
    views = [p.view(2, 3, 85, p.shape[2], p.shape[3]).permute(0, 1, 3, 4, 2) for p in preds]
    crit = V.YOLOv5Loss(80, anchors=ANCHORS)
    assert torch.equal(crit(views, targets)[0], crit(preds, targets)[0])


def test_sppf_chain_matches_autograd_on_ties(cuda):
    """Forward bit-exact; backward equal to autograd through three nn.MaxPool2d(5, 1, 2) on tie-heavy bf16 inputs (fp32 autograd)."""
    from cvpytorch_b200 import train as T
    g = torch.Generator().manual_seed(3)
    for B, H, W, C in ((2, 20, 20, 64), (1, 7, 9, 16), (2, 13, 5, 32)):
        a = torch.randint(-3, 4, (B, H, W, C), generator=g).to(torch.bfloat16).cuda()  # seven values: ties everywhere
        gc = torch.randn((B, H, W, 4 * C), generator=g).to(torch.bfloat16).cuda()
        x = a.permute(0, 3, 1, 2).float().requires_grad_(True)
        mp = nn.MaxPool2d(5, 1, 2)
        y1 = mp(x)
        y2 = mp(y1)
        y3 = mp(y2)
        ref = torch.cat([x, y1, y2, y3], 1)
        ref.backward(gc.permute(0, 3, 1, 2).float())
        ai = a.clone().requires_grad_(True)
        cat = T._SppfChain.apply(ai)
        assert torch.equal(cat.permute(0, 3, 1, 2).float(), ref.detach())
        cat.backward(gc)
        want = x.grad.permute(0, 2, 3, 1)
        got = ai.grad.float()
        assert torch.equal(got != 0, want.to(torch.bfloat16).float() != 0)
        assert (got - want).abs().max() <= (want.abs() * 2 ** -8).max() + 1e-6


def test_stem_matches_torch_fp64(cuda):
    """The 6x6 / s2 / p2 stem (focus_s2d + permuted 3x3 conv): forward, weight gradient and BatchNorm path against fp64 torch on
    bf16-rounded inputs."""
    from cvpytorch_b200 import yolov5_train as V
    torch.manual_seed(0)
    st = V.StemConv(3, 32).cuda().train()
    st.bn.eps, st.bn.momentum = 1e-3, 0.03  # (what YOLOv5CSPDarknet sets)
    img = torch.rand((2, 3, 64, 96), device='cuda')
    out = st(img)
    g = torch.randn_like(out.float()).to(torch.bfloat16)
    out.backward(g)
    ref = nn.Sequential(nn.Conv2d(3, 32, 6, 2, 2, bias=False), nn.BatchNorm2d(32, eps=1e-3, momentum=0.03), nn.SiLU()).double().cuda().train()
    with torch.no_grad():
        ref[0].weight.copy_(st.conv.weight.to(torch.bfloat16).double())
    imgr = img.to(torch.bfloat16).double()
    y = ref(imgr)
    y.backward(g.permute(0, 3, 1, 2).double())
    assert _rel(out.permute(0, 3, 1, 2).double(), y) < 2e-2
    assert _rel(st.conv.weight.grad, ref[0].weight.grad) < 2e-2
    assert _rel(st.bn.weight.grad, ref[1].weight.grad) < 2e-2
    assert _rel(st.bn.running_var, ref[1].running_var) < 1e-2


def _model():
    from cvpytorch_b200 import models as M, synth
    return M.YOLOv5([{f'c{i}': 1.0} for i in range(80)], dict(synth.YOLOV5S_CFG)).cuda().train()


def _batch(B=4, size=256):
    g = torch.Generator().manual_seed(21)
    imgs = torch.rand((B, 3, size, size), generator=g).cuda()
    targets = []
    for i in range(B):
        n = 3 + i
        boxes = torch.cat([torch.rand((n, 2), generator=g) * 0.8 + 0.1, torch.rand((n, 2), generator=g) * 0.3 + 0.05], 1)
        targets.append({'labels': torch.randint(0, 80, (n,), generator=g), 'boxes': boxes})
    return imgs, targets


def test_model_training_forward_matches_loss_on_detect_outputs(cuda):
    from cvpytorch_b200 import yolov5_train as V
    m = _model()
    imgs, targets = _batch()
    gts = m.pack_targets(imgs, targets)
    assert gts.shape == (sum(t['labels'].shape[0] for t in targets), 6)
    seen = {}
    forward = m.loss.forward
    m.loss.forward = lambda p, t: (seen.update(p=[x.detach().clone() for x in p]), forward(p, t))[1]
    losses = m(imgs, gts, 'train')
    assert set(losses) == {'loss', 'box_loss', 'obj_loss', 'cls_loss'}
    assert [tuple(p.shape) for p in seen['p']] == [(4, 255, 32, 32), (4, 255, 16, 16), (4, 255, 8, 8)]
    loss, items = V.YOLOv5Loss(80, anchors=ANCHORS)(seen['p'], gts)
    assert torch.equal(losses['loss'].detach(), loss)
    assert torch.equal(torch.stack([losses['box_loss'], losses['obj_loss'], losses['cls_loss']]), items)
    assert torch.isfinite(loss).all() and float(loss) > 0


def test_network_step_vs_reference_fixture(cuda):
    """tests/golden/yolov5_train.npz (the reference's backbone, neck and detect in training mode, fp32, a narrowed YOLOv5-n at widths 16 /
    32, 3 classes, 2x3x64x96): the training modules' outputs, every parameter gradient and every running statistic, max-normalised, within
    3x the error of the same oracle step under bf16 autocast on this GPU, plus 1e-2 (the criterion of the YOLOX network tests)."""
    from cvpytorch_b200 import yolov5_train as V
    from oracle import yolov5_train_oracle as O
    torch.backends.cudnn.allow_tf32 = False
    f = np.load(os.path.join(ROOT, 'tests', 'golden', 'yolov5_train.npz'))
    keys, sd, x, Gs = O.net_fixture_inputs(f)
    ref = {k: torch.from_numpy(f[k]) for k in f.files if k.startswith(('y', 'grad_', 'after_'))}
    with torch.autocast('cuda', dtype=torch.bfloat16):
        auto = O.net_train_step(x.cuda(), [G.cuda() for G in Gs], {k: v.cuda() for k, v in sd.items()})
    mods = {'backbone.': V.YOLOv5CSPDarknet(**O.NET['backbone']), 'neck.': V.YOLOv5Neck(**O.NET['neck']),
            'detect.': V.YOLOv5Detect(anchors=O.ANCHORS, **O.NET['detect'])}
    for pre, m in mods.items():
        m.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}, strict=True)
        m.cuda().train()
    bb, nk, dt = mods.values()
    outs = dt.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(x.cuda())))
    sum((o * G.cuda()).sum() for o, G in zip(outs, Gs)).backward()
    got = {f'y{i}': o.detach() for i, o in enumerate(outs)}
    for pre, m in mods.items():
        got.update({f'grad_{pre}{k}': p.grad for k, p in m.named_parameters()})
        got.update({f'after_{pre}{k}': v for k, v in m.state_dict().items() if 'running_' in k})
    assert set(got) == set(ref) == set(auto)
    errs = {k: _rel(got[k], ref[k]) for k in ref}
    au = {k: _rel(auto[k].float(), ref[k]) for k in ref}
    print('worst error / (3 x autocast error + 1e-2):', round(max(errs[k] / (3 * au[k] + 1e-2) for k in ref), 3))
    bad = {k: (errs[k], au[k]) for k in ref if errs[k] > 3 * au[k] + 1e-2}
    assert not bad, bad


def test_model_step_gradients_follow_the_oracle_network(cuda):
    """One training step of the whole model against oracle/yolov5_train_oracle.network + yolov5_loss in fp32 (torch.autograd): the loss
    within 2 %, and every parameter gradient within 3x the error of the same oracle step under bf16 autocast, plus 1e-2 (the criterion of
    the YOLOX network tests)."""
    from oracle import yolov5_train_oracle as O
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    m = _model()
    imgs, targets = _batch()
    gts = m.pack_targets(imgs, targets)
    state = {k: v.detach().clone() for k, v in m.state_dict().items()}

    def oracle(autocast):
        sd = {k: v.clone().requires_grad_(v.dtype.is_floating_point and 'running_' not in k and k != 'detect.anchors') for k, v in state.items()}
        with torch.autocast('cuda', dtype=torch.bfloat16, enabled=autocast):
            outs = O.network(imgs, sd)
        loss = O.yolov5_loss([o.float().cpu() for o in outs], gts.cpu(), torch.tensor(ANCHORS), 80)[0]
        loss.backward()
        return loss, {k: v.grad for k, v in sd.items() if v.grad is not None}
    oloss, og = oracle(False)
    _, ag = oracle(True)
    losses = m(imgs, gts, 'train')
    losses['loss'].backward()
    assert abs(float(losses['loss'].detach()) - float(oloss.detach())) < 0.02 * abs(float(oloss.detach()))
    bad, worst = [], 0.0
    for k, p in m.named_parameters():
        ref = og[k].double()
        e = float((p.grad.double() - ref).norm() / (ref.norm() + 1e-30))
        e_ac = float((ag[k].double() - ref).norm() / (ref.norm() + 1e-30))
        worst = max(worst, e / (3 * e_ac + 1e-2))
        if e > 3 * e_ac + 1e-2:
            bad.append((k, round(e, 4), round(e_ac, 4)))
    print('worst error / (3 x autocast error + 1e-2):', round(worst, 3))
    assert not bad, bad


def test_model_trainer_steps_hand_off_to_eval_and_graph_capture(cuda):
    """The reference trainer's step logic (autocast + GradScaler + clip + SGD) runs with finite losses and gradients (the gradient itself
    is checked against the oracle above); then eval() serves the trained weights exactly as a fresh eval YOLOv5 loaded with
    model.state_dict(); then the whole step captures as one CUDA graph and replays."""
    from cvpytorch_b200 import models as M, synth
    m = _model()
    imgs, targets = _batch()
    params = list(m.parameters())
    opt = torch.optim.SGD(params, lr=0.01, momentum=0.9)
    scaler = torch.amp.GradScaler('cuda', enabled=True)
    hist = []
    for it in range(10):
        with torch.autocast('cuda', enabled=True):
            losses = m(imgs, targets, 'train')
        scaler.scale(losses['loss']).backward()
        scaler.unscale_(opt)
        torch.nn.utils.clip_grad_norm_(params, 10.0)
        if it == 0:
            for n, p in m.named_parameters():
                assert p.grad is not None and torch.isfinite(p.grad).all(), n
        scaler.step(opt)
        scaler.update()
        opt.zero_grad(set_to_none=True)
        hist.append(float(losses['loss'].detach()))
    del losses
    print('loss', [round(v, 4) for v in hist])
    assert all(np.isfinite(hist)), hist
    m.eval()
    with torch.no_grad():
        got, _, cnt = m.predict(imgs)
        got, cnt = got.clone(), cnt.clone()
    fresh = M.YOLOv5([{f'c{i}': 1.0} for i in range(80)], dict(synth.YOLOV5S_CFG))
    fresh.load_state_dict(m.state_dict(), strict=True)
    fresh.cuda().eval()
    with torch.no_grad():
        want, _, wcnt = fresh.predict(imgs)
    assert torch.equal(cnt, wcnt) and torch.equal(got, want)

    m.train()
    gt = m.pack_targets(imgs, targets)
    opt = torch.optim.SGD(params, lr=0.01, momentum=0.9)

    def step():
        losses = m(imgs, gt, 'train')
        losses['loss'].backward()
        torch.nn.utils.clip_grad_norm_(params, 10.0)
        opt.step()
        opt.zero_grad(set_to_none=False)
        return losses['loss']
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_loss = step()
    vals = []
    for _ in range(10):
        graph.replay()
        vals.append(float(static_loss.detach()))
    print('graph loss', [round(v, 4) for v in vals])
    assert all(np.isfinite(vals)) and len(set(vals)) > 1, vals  # (the replays train: the loss moves)
