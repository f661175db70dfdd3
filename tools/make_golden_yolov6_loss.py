"""Writes tests/golden/yolov6_loss.npz: the reference YOLOv6Loss (src/losses/det/yolov6_loss.py) with its ATSS and task-aligned assigners,
run on the CPU on the seeded inputs of CASES.

  CVPYTORCH_REFERENCE=<reference checkout> python tools/make_golden_yolov6_loss.py

The assigner outputs are captured by wrapping warmup_assigner / formal_assigner, and target_gt_idx by wrapping select_highest_overlaps.
Per case the file keeps the seed, the GT rows and, at the foreground anchors only (the rest is background: zero score, zero gradient),
the anchor index, target_gt_idx, label, target box, soft label and the gradient of the summed loss dict with respect to pred_distri; plus
the loss L, target_scores_sum and num_pos.  The oracle (oracle/yolov6_loss_oracle.py) must reproduce the assignment bitwise and the loss
and gradient within 1e-6 before anything is written, and every case must be free of ties at the top-k boundary (the reference's order
there is arbitrary).  A level with fewer than 9 anchors makes the reference ATSS raise (its candidate mask is sized for 9), so such grids
are checked against the oracle only."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import ref_shim  # noqa: E402
from oracle import yolov6_loss_oracle as LO  # noqa: E402

# name: (seed, B, H, W, nc, GTs per image, assigner, iou_type)
CASES = {
    'atss_giou': (11, 3, 128, 128, 3, (7, 12, 0), 'atss', 'giou'),
    'atss_siou': (11, 3, 128, 128, 3, (7, 12, 0), 'atss', 'siou'),
    'tal_giou': (11, 3, 128, 128, 3, (7, 12, 0), 'tal', 'giou'),
    'tal_siou': (11, 3, 128, 128, 3, (7, 12, 0), 'tal', 'siou'),
    'big_atss': (13, 1, 640, 640, 80, (30,), 'atss', 'giou'),
    'big_tal': (13, 1, 640, 640, 80, (30,), 'tal', 'siou'),
}


def case_inputs(name):
    """-> (shapes, pred_scores, pred_distri, gt) of a case, regenerated from its seed."""
    seed, B, H, W, nc, per_image, _, _ = CASES[name]
    gen = torch.Generator().manual_seed(seed)
    shapes = LO.level_shapes(H, W)
    A = sum(h * w for h, w in shapes)
    scores, distri = LO.make_preds(gen, B, A, nc)
    gt = LO.make_targets(gen, B, H, W, per_image, nc=nc)
    extra = [[0, 1, -10 / 640, -10 / 640, 30 / 640, 30 / 640],      # x1 + y1 + x2 + y2 <= 0: not a GT, but it overlaps anchors
             [1, 2, 20 / 640, 22 / 640, 10 / 640, 9 / 640]]         # a small GT: fewer than 13 anchors inside it
    gt = torch.cat([gt, torch.tensor([r for r in extra if r[0] < B], dtype=torch.float32)])
    return shapes, scores, distri, gt


def reference_run(mod, utils_mods, name):
    seed, B, H, W, nc, _, assigner, iou_type = CASES[name]
    shapes, scores, distri, gt = case_inputs(name)
    loss = mod.YOLOv6Loss(num_classes=nc, iou_type=iou_type, reg_max=0)
    cap = {}
    for am in utils_mods:
        orig = am.select_highest_overlaps

        def wrapped(mask_pos, overlaps, n, _orig=orig):
            r = _orig(mask_pos, overlaps, n)
            cap['gt_idx'] = r[0].clone()
            return r
        am.select_highest_overlaps = wrapped
    for attr in ('warmup_assigner', 'formal_assigner'):
        a = getattr(loss, attr)
        f = a.forward

        def wrapped_fwd(*args, _f=f, **kw):
            r = _f(*args, **kw)
            cap['assign'] = [t.clone() for t in r]
            return r
        a.forward = wrapped_fwd
    feats = [torch.zeros(B, 1, h, w) for h, w in shapes]
    d = distri.clone().requires_grad_(True)
    s = scores.clone().requires_grad_(True)
    out = loss((feats, s, d), gt.clone(), 0 if assigner == 'atss' else 4)
    (out['iou'] + out['dfl'] + out['class']).backward()
    assert s.grad is None
    return out, cap, d.grad


def check_ties(name, shapes, scores, distri, gt):
    """No equal values straddle the top-k boundary of a real GT (ATSS distances; TAL metrics of in-GT anchors)."""
    seed, B, H, W, nc, _, assigner, _ = CASES[name]
    anc, points, per_level, stride = LO.anchors(shapes)
    labels, boxes, mask, _ = LO.pack(gt, B)
    if assigner == 'atss':
        gc = (boxes[..., :2] + boxes[..., 2:]) / 2.0
        ac = (anc[:, :2] + anc[:, 2:]) / 2.0
        dist = (gc[..., None, :] - ac).pow(2).sum(-1).sqrt()
        o = 0
        for n in per_level:
            if n > 9:
                v = torch.sort(dist[..., o:o + n], -1).values
                assert not bool(((v[..., 8] == v[..., 9]) & mask).any()), (name, 'distance tie at the 9th place')
            o += n
    else:
        pts_s = points / stride
        pd = torch.cat([pts_s - distri[..., :2], pts_s + distri[..., 2:]], -1) * stride
        ov = LO.iou_pairs(boxes, pd)
        metric = LO.class_scores(scores, labels, nc) * ov.pow(6.0)
        ins = LO.inside(points, boxes)
        metric = metric * ins
        v = torch.sort(metric, -1, descending=True).values
        edge = v[..., 12:13]
        tied_in = ((metric == edge) & ins).sum(-1)
        ambiguous = (v[..., 12] == v[..., 13]) & (tied_in > 0) & mask
        assert not bool(ambiguous.any()), (name, 'metric tie at the 13th place')


def main():
    ref_shim.install()
    import src.losses.det.yolov6_loss as mod
    import src.models.assigners.atss_assigner as am1
    import src.models.assigners.tal_assigner as am2
    torch.set_num_threads(1)
    res = {}
    for name, (seed, B, H, W, nc, per_image, assigner, iou_type) in CASES.items():
        shapes, scores, distri, gt = case_inputs(name)
        check_ties(name, shapes, scores, distri, gt)
        out, cap, grad = reference_run(mod, (am1, am2), name)
        labels, tboxes, tscores, fg = cap['assign']
        gt_idx = cap['gt_idx']
        d = distri.clone().requires_grad_(True)
        o_out, o = LO.losses(shapes, scores, d, gt, assigner, iou_type, nc)
        (o_out['iou'] + o_out['dfl'] + o_out['class']).backward()
        assert torch.equal(o['fg'], fg.bool()), name
        assert torch.equal(o['gt_idx'][fg], gt_idx[fg]), name
        assert torch.equal(o['labels'][fg], labels.long()[fg]), name
        assert torch.equal(o['boxes'][fg], tboxes[fg]), name
        soft = tscores.sum(-1)
        assert torch.equal(o['scores'], soft.double()), (name, float((o['scores'] - soft.double()).abs().max()))
        for k in ('iou', 'dfl', 'class'):
            assert out[k].dtype == torch.float64 and o_out[k].dtype == torch.float64, (name, k, out[k].dtype)
            assert abs(float(o_out[k]) - float(out[k])) <= 1e-6 * abs(float(out[k])), (name, k)
        gerr = float((d.grad - grad).abs().max() / grad.abs().max())
        assert gerr <= 1e-6, (name, gerr)
        flat = fg.reshape(-1).nonzero()[:, 0]
        A = fg.shape[1]
        res[f'{name}_seed'] = np.array(seed)
        res[f'{name}_gt'] = gt.numpy()
        res[f'{name}_fg'] = flat.numpy().astype(np.int32)
        res[f'{name}_gt_idx'] = gt_idx.reshape(-1)[flat].numpy().astype(np.int32)
        res[f'{name}_labels'] = labels.reshape(-1)[flat].numpy().astype(np.int32)
        res[f'{name}_boxes'] = tboxes.reshape(-1, 4)[flat].numpy()
        res[f'{name}_scores'] = soft.reshape(-1)[flat].double().numpy()
        res[f'{name}_grad'] = grad.reshape(-1, 4)[flat].numpy()
        res[f'{name}_loss'] = np.array(float(out['class']))
        res[f'{name}_tss'] = np.array(float(tscores.sum()))
        print(name, 'L', float(out['class']), 'positives', int(fg.sum()), 'of', B * A, 'gerr', gerr)
    path = os.path.join(ROOT, 'tests', 'golden', 'yolov6_loss.npz')
    np.savez_compressed(path, **res)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
