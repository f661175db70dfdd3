"""Functional torch restatement of the YOLOX training loss (src/losses/det/yolox_loss.py:73-436): decode, SimOTA label assignment and the
IoU / objectness / class losses, written from the algorithm (DESIGN.md §4.3).  fp32 in the reference's operation order, one image at a time;
differentiable in the head outputs (the assignment is computed without gradient).

  losses(preds, targets, strides, num_classes, assignment=None) -> dict(loss, iou_loss, conf_loss, cls_loss, num_fg), (fg, matched_gt, matched_iou)
  near_ties(preds, targets, strides, num_classes) -> bool [B]: images whose assignment is decided by an fp64 gap below the tie tolerance
  fixture_case(seed, case) -> (preds, targets): the seeded inputs of tests/golden/yolox_loss.npz

Tie rule (the reference leaves it to torch.topk / torch.min): a GT takes its k lowest costs with the lower anchor index first on equal costs,
and an anchor taken by several GTs goes to the lowest GT index among its equal minimal costs.  A GT in an image without candidate anchors
(the reference's topk raises there) matches nothing.  `assignment` = (fg bool [B, A], matched_gt long [B, A] (-1: background), matched_iou
[B, A]) replaces the assignment, so that losses and gradients can be compared under another implementation's assignment."""
import torch
import torch.nn.functional as F

CENTER_RADIUS = 2.5
TOPK = 10


def decode(preds, strides):
    """[B, 5 + nc, h, w] per level -> (outputs [B, A, 5 + nc] with xy = (p + grid) s and wh = exp(p) s, grid x [A], grid y [A], stride [A])."""
    outs, gxs, gys, ss = [], [], [], []
    for p, s in zip(preds, strides):
        B, C, h, w = p.shape
        yv, xv = torch.meshgrid(torch.arange(h), torch.arange(w), indexing='ij')
        grid = torch.stack((xv, yv), 2).view(1, h * w, 2).to(p)
        x = p.permute(0, 2, 3, 1).reshape(B, h * w, C)
        outs.append(torch.cat([(x[..., :2] + grid) * s, torch.exp(x[..., 2:4]) * s, x[..., 4:]], -1))
        gxs.append(grid[0, :, 0])
        gys.append(grid[0, :, 1])
        ss.append(torch.full((h * w,), float(s), dtype=p.dtype, device=p.device))
    return torch.cat(outs, 1), torch.cat(gxs), torch.cat(gys), torch.cat(ss)


def num_labels(targets):
    """The number of rows with a positive sum; an image uses its FIRST nlabel rows."""
    return (targets.sum(2) > 0).sum(1)


def pair_iou(a, b):
    """IoU [Na, Nb] of (cx, cy, w, h) boxes a [Na, 4] and b [Nb, 4], no epsilon."""
    tl = torch.max(a[:, None, :2] - a[:, None, 2:] / 2, b[:, :2] - b[:, 2:] / 2)
    br = torch.min(a[:, None, :2] + a[:, None, 2:] / 2, b[:, :2] + b[:, 2:] / 2)
    area_a, area_b = torch.prod(a[:, 2:], 1), torch.prod(b[:, 2:], 1)
    en = (tl < br).type(tl.type()).prod(dim=2)
    area_i = torch.prod(br - tl, 2) * en
    return area_i / (area_a[:, None] + area_b - area_i)


def iou_loss(pred, target):
    """1 - iou^2 per row, iou with +1e-16 in the denominator."""
    tl = torch.max(pred[:, :2] - pred[:, 2:] / 2, target[:, :2] - target[:, 2:] / 2)
    br = torch.min(pred[:, :2] + pred[:, 2:] / 2, target[:, :2] + target[:, 2:] / 2)
    area_p, area_g = torch.prod(pred[:, 2:], 1), torch.prod(target[:, 2:], 1)
    en = (tl < br).type(tl.type()).prod(dim=1)
    area_i = torch.prod(br - tl, 1) * en
    iou = area_i / (area_p + area_g - area_i + 1e-16)
    return 1 - iou ** 2


def _candidates(gt_box, xc, yc, ss):
    """-> (in_box [G, A], in_center [G, A]): the anchor centre strictly inside the GT box / inside GT centre +- 2.5 stride."""
    def inside(l, t, r, b):
        return torch.stack([xc[None] - l, yc[None] - t, r - xc[None], b - yc[None]], 2).min(dim=-1).values > 0.0
    cx, cy, w, h = (gt_box[:, i:i + 1] for i in range(4))
    in_box = inside(cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h)
    rad = CENTER_RADIUS * ss[None]
    return in_box, inside(cx - rad, cy - rad, cx + rad, cy + rad)


def _assign_image(out, gt_cls, gt_box, gx, gy, ss, nc, ties=None):
    """SimOTA for one image: out [A, 5 + nc] decoded (no grad) -> (fg [A], matched_gt [A], matched_iou [A]).  `ties` (a list): records
    whether a decision had an fp64 gap below the tolerance (the inputs are then expected in float64)."""
    A, G = out.shape[0], gt_box.shape[0]
    fg = torch.zeros(A, dtype=torch.bool, device=out.device)
    mg = torch.full((A,), -1, dtype=torch.long, device=out.device)
    mi = torch.zeros(A, dtype=out.dtype, device=out.device)
    if G == 0:
        return fg, mg, mi
    xc, yc = gx * ss + 0.5 * ss, gy * ss + 0.5 * ss
    in_box, in_ctr = _candidates(gt_box, xc, yc, ss)
    ci = (in_box.any(0) | in_ctr.any(0)).nonzero()[:, 0]
    n = ci.numel()
    if n == 0:  # no candidate anchor: every GT of the image matches nothing
        return fg, mg, mi
    both = in_box[:, ci] & in_ctr[:, ci]
    ious = pair_iou(gt_box, out[ci, :4])
    onehot = F.one_hot(gt_cls.to(torch.int64), nc).to(out.dtype).unsqueeze(1).repeat(1, n, 1)
    q = out[ci, 5:5 + nc].unsqueeze(0).repeat(G, 1, 1).sigmoid() * out[ci, 4:5].unsqueeze(0).repeat(G, 1, 1).sigmoid()
    cls_cost = F.binary_cross_entropy(q.sqrt(), onehot, reduction='none').sum(-1)
    cost = cls_cost + 3.0 * (-torch.log(ious + 1e-8)) + 100000.0 * (~both)
    top = torch.topk(ious, min(TOPK, n), dim=1).values
    ksum = top.sum(1)
    dk = torch.clamp(ksum.int(), min=1)
    M = torch.zeros_like(cost)
    for g in range(G):
        order = torch.sort(cost[g], stable=True).indices
        k = int(dk[g])
        M[g, order[:k]] = 1.0
        if ties is not None:
            frac = float(ksum[g] - torch.floor(ksum[g]))
            cs = cost[g, order]
            gap = float(cs[k] - cs[k - 1]) if k < n else float('inf')
            if min(frac, 1 - frac) < 1e-5 or gap < 1e-5 * abs(float(cs[k - 1])):
                ties.append(True)
    multi = M.sum(0) > 1
    if multi.any():
        cm = cost[:, multi]
        am = cm.argmin(0)
        if ties is not None and G > 1:
            srt = torch.sort(cm, dim=0).values
            if bool(((srt[1] - srt[0]) < 1e-5 * srt[0].abs()).any()):
                ties.append(True)
        M[:, multi] = 0.0
        M[am, multi] = 1.0
    fgc = M.sum(0) > 0.0
    m = M[:, fgc].argmax(0)
    sel = ci[fgc]
    fg[sel] = True
    mg[sel] = m
    mi[sel] = ious[m, fgc.nonzero()[:, 0]]
    return fg, mg, mi


def assign(preds, targets, strides, num_classes):
    """(fg bool [B, A], matched_gt long [B, A], matched_iou [B, A]) of the SimOTA assignment."""
    with torch.no_grad():
        out, gx, gy, ss = decode(preds, strides)
        nl = num_labels(targets).tolist()
        res = [_assign_image(out[b], targets[b, :nl[b], 0], targets[b, :nl[b], 1:5], gx, gy, ss, num_classes) for b in range(out.shape[0])]
    return tuple(torch.stack(t) for t in zip(*res))


def near_ties(preds, targets, strides, num_classes):
    """bool [B]: the image's assignment in float64 has a k-th boundary cost gap or a conflict argmin gap below 1e-5 |cost|, or a top-10
    IoU sum within 1e-5 of an integer.  An implementation in fp32 may decide such an image either way."""
    with torch.no_grad():
        p64 = [p.detach().double() for p in preds]
        t64 = targets.double()
        out, gx, gy, ss = decode(p64, strides)
        nl = num_labels(t64).tolist()
        flags = []
        for b in range(out.shape[0]):
            ties = []
            _assign_image(out[b], t64[b, :nl[b], 0], t64[b, :nl[b], 1:5], gx, gy, ss, num_classes, ties=ties)
            flags.append(bool(ties))
    return torch.tensor(flags)


def losses(preds, targets, strides, num_classes, assignment=None):
    """-> (the reference's loss dict, the assignment used).  Differentiable in preds."""
    out, _, _, _ = decode(preds, strides)
    if assignment is None:
        assignment = assign(preds, targets, strides, num_classes)
    fg, mg, mi = assignment
    fg, mg, mi = fg.to(out.device), mg.to(out.device).long(), mi.to(out.device, out.dtype)
    B = out.shape[0]
    num_gts = int(num_labels(targets).sum())
    num_fg = max(int(fg.sum()), 1)
    rows = torch.cat([targets[b, mg[b][fg[b]]] for b in range(B)], 0)
    reg_t = rows[:, 1:5].to(out.dtype)
    cls_t = F.one_hot(rows[:, 0].to(torch.int64), num_classes).to(out.dtype) * mi[fg].unsqueeze(-1)
    l_iou = iou_loss(out[..., :4][fg], reg_t).sum() / num_fg
    l_obj = F.binary_cross_entropy_with_logits(out[..., 4].reshape(-1, 1), fg.reshape(-1, 1).to(out.dtype), reduction='none').sum() / num_fg
    l_cls = F.binary_cross_entropy_with_logits(out[..., 5:5 + num_classes][fg], cls_t, reduction='none').sum() / num_fg
    loss = 5.0 * l_iou + l_obj + l_cls
    fg_r = torch.tensor(num_fg / max(num_gts, 1), device=out.device, dtype=out.dtype)
    return {'loss': loss, 'conf_loss': l_obj, 'cls_loss': l_cls, 'iou_loss': 5.0 * l_iou, 'num_fg': fg_r}, (fg, mg, mi)


# ------------------------------------------------------------------------------------------------ seeded inputs of the golden fixture
# case -> (batch, image size, num_classes); the GT layout of every image is fixed by _case_gts
CASES = {'a': (3, 128, 3), 'b': (2, 160, 80)}
STRIDES = (8, 16, 32)


def _case_gts(case, H, gen):
    """Per image a list of (class, cx, cy, w, h): random boxes, an overlapping pair (conflicts), a 2x2 GT that is inside a centre region but
    contains no anchor centre (in-centre only), a GT at the right edge whose anchors include the head's padded column, and an image without GT."""
    def rnd(nc):
        u = torch.rand(5, generator=gen)
        w, h = 24 + 40 * float(u[3]), 24 + 40 * float(u[4])
        return [float(int(u[0] * nc)), 20 + (H - 40) * float(u[1]), 20 + (H - 40) * float(u[2]), w, h]
    nc = CASES[case][2]
    if case == 'a':
        a = rnd(nc)
        pair = [a, [float((a[0] + 1) % nc), a[1] + 5.0, a[2] + 4.0, a[3] * 0.9, a[4] * 0.95]]
        return [pair + [rnd(nc), [0.0, 17.0, 17.0, 2.0, 2.0]],
                [],
                [rnd(nc), [float(nc - 1), H - 6.0, 60.0, 40.0, 36.0], rnd(nc)]]
    a = rnd(nc)
    return [[rnd(nc), a, [float(int(a[0] + 7) % nc), a[1] - 4.0, a[2] + 6.0, a[3] * 1.1, a[4] * 0.9], rnd(nc), rnd(nc), rnd(nc)],
            [rnd(nc), [float(nc - 2), 60.0, H - 5.0, 36.0, 40.0], rnd(nc)]]


def fixture_case(seed, case):
    """-> (preds: fp32 [B, 5 + nc, H/s + 2, W/s + 2] per stride, targets fp32 [B, max_gt, 5]), zero rows after each image's GTs.  Anchors
    near a GT predict a jittered copy of it (so that dynamic k exceeds 1); the others predict random boxes."""
    B, H, nc = CASES[case]
    gen = torch.Generator().manual_seed(seed)
    gts = _case_gts(case, H, gen)
    G = max(len(g) for g in gts)
    targets = torch.zeros(B, G, 5)
    for b, rows in enumerate(gts):
        if rows:
            targets[b, :len(rows)] = torch.tensor(rows)
    preds = []
    for s in STRIDES:
        h = w = H // s + 2
        p = torch.randn(B, 5 + nc, h, w, generator=gen)
        p[:, 2:4] += float(torch.log(torch.tensor(2.0)))
        p[:, 4:] = p[:, 4:] * 1.5 - 2.0
        yv, xv = torch.meshgrid(torch.arange(h), torch.arange(w), indexing='ij')
        xc, yc = (xv.float() + 0.5) * s, (yv.float() + 0.5) * s
        for b, rows in enumerate(gts):
            for cls, cx, cy, bw, bh in rows:
                near = ((xc - cx).abs() < 2.5 * s + bw / 2) & ((yc - cy).abs() < 2.5 * s + bh / 2)
                take = near & (torch.rand(h, w, generator=gen) < 0.7)
                if bw < 4:  # the tiny GT: one anchor of the finest level predicts it (dynamic k 1, a clear winner)
                    take = ((xc - cx).abs() + (yc - cy).abs() == ((xc - cx).abs() + (yc - cy).abs()).min()) & (s == STRIDES[0])
                jit = torch.randn(4, h, w, generator=gen)
                p[b, 0][take] = ((cx + 0.15 * bw * jit[0]) / s - xv.float())[take]
                p[b, 1][take] = ((cy + 0.15 * bh * jit[1]) / s - yv.float())[take]
                p[b, 2][take] = torch.log((bw * (1 + 0.2 * jit[2]).clamp(min=0.3)) / s)[take]
                p[b, 3][take] = torch.log((bh * (1 + 0.2 * jit[3]).clamp(min=0.3)) / s)[take]
                p[b, 4][take] += 2.0
                p[b, 5 + int(cls)][take] += 2.5
        preds.append(p)
    return preds, targets
