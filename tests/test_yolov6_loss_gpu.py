"""The YOLOv6 loss kernels (csrc/yolov6_loss.cu) on the H100: against the reference fixture, against the oracle over batch / classes /
size / GT load / assigner / IoU type with ties, the no-positive cases, half-precision heads, per-output gradient scaling, and
reproducibility under a CUDA graph."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tools')):
    if p not in sys.path:
        sys.path.insert(0, p)
GOLD = os.path.join(ROOT, 'tests', 'golden', 'yolov6_loss.npz')
DEV = 'cuda'
pytestmark = pytest.mark.gpu


def _run(shapes, scores, distri, gt, assigner, iou_type, nc):
    from cvpytorch_b200 import yolov6_train as YT
    p = YT.loss_params(shapes, (8, 16, 32), nc, distri.shape[0], assigner, iou_type)
    d = distri.to(DEV).float().contiguous()
    out, a = YT.yolov6_loss_forward(p, scores.to(DEV).float().contiguous(), d, gt.to(DEV).double().contiguous())
    g = YT.yolov6_loss_backward(p, d, a, torch.ones(3, dtype=torch.float64, device=DEV))
    return out, a, g


def _gmax_err(g, ref):
    return float((g.double() - ref.double()).abs().max() / max(float(ref.double().abs().max()), 1e-30))


def test_fixture():
    """fg_mask, target_gt_idx and labels bitwise; target boxes and soft labels within 1e-12; losses within 1e-6; the gradient of the
    summed dict within 1e-5 max-normalised, zero at background anchors."""
    from make_golden_yolov6_loss import CASES, case_inputs
    g = np.load(GOLD)
    for name, (_, B, H, W, nc, _, assigner, iou_type) in CASES.items():
        shapes, scores, distri, gt = case_inputs(name)
        out, a, grad = _run(shapes, scores, distri, gt, assigner, iou_type, nc)
        flat = torch.from_numpy(g[f'{name}_fg']).long()
        assert torch.equal(a['fg'].reshape(-1).nonzero()[:, 0].cpu(), flat), name
        assert np.array_equal(a['gt_idx'].reshape(-1)[flat.to(DEV)].cpu().numpy(), g[f'{name}_gt_idx'])
        assert np.array_equal(a['labels'].reshape(-1)[flat.to(DEV)].cpu().numpy(), g[f'{name}_labels'])
        assert np.abs(a['boxes'].reshape(-1, 4)[flat.to(DEV)].cpu().numpy() - g[f'{name}_boxes']).max() <= 1e-12
        assert np.abs(a['scores'].reshape(-1)[flat.to(DEV)].cpu().numpy() - g[f'{name}_scores']).max() <= 1e-12
        L = float(g[f'{name}_loss'])
        for k, w in enumerate((2.5, 0.5, 1.0)):
            assert abs(float(out[k]) - w * L) <= 1e-6 * w * L, (name, k)
        ref = torch.zeros(B * distri.shape[1], 4)
        ref[flat] = torch.from_numpy(g[f'{name}_grad'])
        assert _gmax_err(grad.reshape(-1, 4).cpu(), ref) <= 1e-5, name


def _matrix_case(seed, B, size, nc, n_max, ties):
    from oracle import yolov6_loss_oracle as LO
    gen = torch.Generator().manual_seed(seed)
    shapes = LO.level_shapes(size, size)
    A = sum(h * w for h, w in shapes)
    scores, distri = LO.make_preds(gen, B, A, nc)
    per = [int(torch.randint(0, n_max + 1, (), generator=gen)) for _ in range(B)]
    gt = LO.make_targets(gen, B, size, size, per, nc=nc, min_wh=4.0)
    if ties and gt.shape[0]:
        # GT centres on cell corners (distance ties at the 9th place) and zero scores (zero-metric ties at the 13th)
        k = gt.shape[0] // 2
        gt[:k, 2:4] = (torch.round(gt[:k, 2:4] * 640 / 8) * 8 / 640).float()
        scores[:, ::3] = 0.0
    return shapes, scores, distri, gt


@pytest.mark.parametrize('B,size,nc,n_max', [(1, 64, 1, 3), (4, 320, 3, 30), (4, 640, 80, 100), (64, 320, 80, 30), (64, 640, 80, 100)])
@pytest.mark.parametrize('assigner', ['atss', 'tal'])
def test_matches_oracle(B, size, nc, n_max, assigner):
    """The kernels against the oracle run on the GPU (lowest index wins every tie), for GIoU and SIoU, with and without ties."""
    from oracle import yolov6_loss_oracle as LO
    for ties in (False, True):
        shapes, scores, distri, gt = _matrix_case(1000 + B + size + nc + ties, B, size, nc, n_max, ties)
        for iou_type in ('giou', 'siou'):
            out, a, grad = _run(shapes, scores, distri, gt, assigner, iou_type, nc)
            d = distri.to(DEV).requires_grad_(True)
            o_out, o = LO.losses(shapes, scores.to(DEV), d, gt.to(DEV), assigner, iou_type, nc)
            (o_out['iou'] + o_out['dfl'] + o_out['class']).backward()
            fg = o['fg']
            assert torch.equal(a['fg'].bool(), fg), (ties, iou_type)
            assert torch.equal(a['gt_idx'].long()[fg], o['gt_idx'][fg])
            assert torch.equal(a['labels'].long(), o['labels'])
            assert torch.equal(a['boxes'][fg], o['boxes'][fg])
            assert float((a['scores'] - o['scores']).abs().max()) <= 1e-12
            ref = float(o_out['iou'].detach())
            assert abs(float(out[0]) - ref) <= 1e-6 * max(abs(ref), 1e-30), (ties, iou_type, float(out[0]), ref)
            if o['num_pos']:
                assert _gmax_err(grad, d.grad) <= 1e-5


def test_no_positives():
    """An empty target list and a batch whose GTs claim no anchor give 0 * sum(pred_distri) (NaN with a non-finite distance) and a zero
    gradient; pred_scores gets no gradient."""
    from cvpytorch_b200.yolov6_train import YOLOv6Loss
    m = YOLOv6Loss(num_classes=3)
    feats = [torch.zeros(2, 1, s, s, device=DEV) for s in (8, 4, 2)]
    sc = torch.rand(2, 84, 3, device=DEV, requires_grad=True)
    far = torch.tensor([[0, 1, 5.0, 5.0, 0.01, 0.01]], device=DEV)  # centre far outside the 64² grid: no candidate inside it
    for gt in (torch.zeros(0, 6, device=DEV), far):
        d = torch.rand(2, 84, 4, device=DEV).requires_grad_(True)
        out = m((feats, sc, d), gt)
        assert all(v.dtype == torch.float64 and float(v) == 0.0 for v in out.values())
        sum(out.values()).backward()
        assert torch.equal(d.grad, torch.zeros_like(d)) and sc.grad is None
    d = torch.rand(2, 84, 4, device=DEV)
    d[1, 3, 2] = float('inf')
    assert all(torch.isnan(v) for v in m((feats, sc, d), far).values())


def test_half_heads_and_separate_gradients():
    """fp16 / bf16 heads give the fp32 head's loss within the cast's rounding and a gradient of their dtype; each dict entry's gradient
    is its weight times the others'."""
    from cvpytorch_b200.yolov6_train import YOLOv6Loss
    shapes, scores, distri, gt = _matrix_case(7, 4, 320, 80, 30, False)
    feats = [torch.zeros(4, 1, h, w, device=DEV) for h, w in shapes]
    m = YOLOv6Loss(num_classes=80)
    grads = {}
    for k in ('iou', 'dfl', 'class'):
        d = distri.to(DEV).requires_grad_(True)
        m((feats, scores.to(DEV), d), gt.to(DEV))[k].backward()
        grads[k] = d.grad
    assert torch.allclose(grads['iou'], grads['class'] * 2.5, rtol=1e-6, atol=0) and torch.allclose(grads['dfl'], grads['class'] * 0.5, rtol=1e-6, atol=0)
    for dt in (torch.float16, torch.bfloat16):
        d = distri.to(DEV, dt).requires_grad_(True)
        out = m((feats, scores.to(DEV, dt), d), gt.to(DEV), epoch_num=5)
        ref = m((feats, scores.to(DEV, dt).float(), d.detach().float()), gt.to(DEV), epoch_num=5)
        assert float(out['class']) == float(ref['class'])
        out['class'].backward()
        assert d.grad.dtype == dt and torch.isfinite(d.grad).all()


def test_deterministic_and_graph_replay():
    """Two runs and a CUDA-graph replay give the same bits (outputs, assignment and gradient)."""
    from cvpytorch_b200 import yolov6_train as YT
    for assigner in ('atss', 'tal'):
        shapes, scores, distri, gt = _matrix_case(99, 8, 640, 80, 100, True)
        p = YT.loss_params(shapes, (8, 16, 32), 80, 8, assigner, 'siou')
        s, d, t = scores.to(DEV), distri.to(DEV), gt.to(DEV).double()
        gout = torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64, device=DEV)

        def step():
            out, a = YT.yolov6_loss_forward(p, s, d, t)
            return out, a, YT.yolov6_loss_backward(p, d, a, gout)
        r1, r2 = step(), step()
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            step()
        torch.cuda.current_stream().wait_stream(st)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            r3 = step()
        graph.replay()
        torch.cuda.synchronize()
        for r in (r2, r3):
            assert torch.equal(r[0], r1[0]) and torch.equal(r[2], r1[2])
            assert all(torch.equal(r[1][k], r1[1][k]) for k in r1[1])
