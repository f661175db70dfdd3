"""Torch restatement of the YOLOv6 training loss (src/losses/det/yolov6_loss.py) with its ATSS and task-aligned assigners
(src/models/assigners/), written from the algorithm, for the CPU fixture and the GPU comparison of csrc/yolov6_loss.cu.

Dtypes follow the reference: the packed targets, IoUs, distances, thresholds and the box loss are float64; anchors, pred boxes and the
ATSS soft labels float32.  Ties at the top-k boundary take the lowest anchor index (a stable sort), the rule of the kernels; torch.topk
leaves that order undefined.  Rows whose image index truncates outside [0, B) are dropped.  Labels outside [0, nc) give a zero class
score.  Everything materialises [B, n_max_boxes, A]: this is an oracle, not a fast path.
"""
import math

import torch

STRIDES = (8, 16, 32)
LOSS_WEIGHT = {'class': 1.0, 'iou': 2.5, 'dfl': 0.5}


def anchors(shapes, strides=STRIDES, grid_cell_size=5.0, grid_cell_offset=0.5, device='cpu'):
    """shapes [(h, w)] per level -> (anchor boxes fp32 [A, 4], anchor points fp32 [A, 2], anchors per level, stride fp32 [A, 1])."""
    boxes, points, counts, stride = [], [], [], []
    for (h, w), s in zip(shapes, strides):
        xs = (torch.arange(w, device=device) + grid_cell_offset) * s
        ys = (torch.arange(h, device=device) + grid_cell_offset) * s
        gy, gx = torch.meshgrid(ys, xs, indexing='ij')
        half = grid_cell_size * s * 0.5
        boxes.append(torch.stack([gx - half, gy - half, gx + half, gy + half], -1).reshape(-1, 4).float())
        points.append(torch.stack([gx, gy], -1).reshape(-1, 2).float())
        counts.append(h * w)
        stride.append(torch.full((h * w, 1), float(s), device=device))
    return torch.cat(boxes), torch.cat(points), counts, torch.cat(stride)


def pack(gt, B, ori_img_size=640):
    """gt [n, 6] (image, label, cx, cy, w, h normalised) -> (labels fp64 [B, m], boxes fp64 [B, m, 4] xyxy pixels, mask_gt bool [B, m], count [B]);
    each image's rows in input order, padding rows (-1, 0, 0, 0, 0)."""
    dev = gt.device
    g = gt.detach().double()
    v = g[:, 0] if g.numel() else g.new_zeros(0)
    keep = (v > -1) & (v < B)
    img = torch.where(keep, v.trunc(), torch.full_like(v, B)).long()
    order = torch.sort(img, stable=True).indices
    counts = torch.bincount(img[keep], minlength=B)[:B] if g.numel() else torch.zeros(B, dtype=torch.long, device=dev)
    m = int(counts.max()) if B else 0
    rows = torch.zeros(B, m, 5, dtype=torch.float64, device=dev)
    rows[..., 0] = -1
    if m:
        sel = order[:int(keep.sum())]
        first = torch.cumsum(counts, 0) - counts
        ib = img[sel]
        rank = torch.arange(sel.numel(), device=dev) - first[ib]
        rows[ib, rank] = g[sel, 1:6]
    box = rows[..., 1:5] * torch.tensor(float(ori_img_size), dtype=torch.float32, device=dev)
    x1 = box[..., 0] - box[..., 2] * 0.5
    y1 = box[..., 1] - box[..., 3] * 0.5
    boxes = torch.stack([x1, y1, x1 + box[..., 2], y1 + box[..., 3]], -1)
    mask = boxes.sum(-1) > 0
    return rows[..., 0], boxes, mask, counts


def iou_pairs(g, p, eps=1e-9):
    """IoU of GT boxes g [B, m, 4] (fp64) with boxes p [B, A, 4] (fp32 areas stay fp32) -> [B, m, A]; areas clipped at 0."""
    gi, pj = g[:, :, None, :], p[:, None, :, :]
    lo = torch.maximum(gi[..., :2], pj[..., :2])
    hi = torch.minimum(gi[..., 2:], pj[..., 2:])
    ov = (hi - lo).clip(0).prod(-1)
    a1 = (g[..., 2:] - g[..., :2]).clip(0).prod(-1)[..., None]
    a2 = (p[..., 2:] - p[..., :2]).clip(0).prod(-1)[:, None, :]
    return ov / (a1 + a2 - ov + eps)


def iou_anchor_boxes(g, anc):
    """bbox_overlaps 'iou' of GT boxes g [B, m, 4] with the anchor boxes anc [A, 4] -> [B, m, A], union clamped to 1e-6."""
    a1 = ((g[..., 2] - g[..., 0]) * (g[..., 3] - g[..., 1]))[..., None]
    a2 = (anc[:, 2] - anc[:, 0]) * (anc[:, 3] - anc[:, 1])
    lo = torch.max(g[..., None, :2], anc[:, :2])
    hi = torch.min(g[..., None, 2:], anc[:, 2:])
    wh = (hi - lo).clamp(min=0)
    ov = wh[..., 0] * wh[..., 1]
    union = torch.max(a1 + a2 - ov, torch.tensor([1e-6], dtype=ov.dtype, device=ov.device))
    return ov / union


def inside(points, g, eps=1e-9):
    """anchor points [A, 2] strictly inside the GT boxes g [B, m, 4] -> bool [B, m, A]."""
    d = torch.cat([points - g[..., None, :2], g[..., None, 2:] - points], -1)
    return d.min(-1).values > eps


def resolve(mask_pos, overlaps):
    """An anchor claimed by several GTs goes to the first maximum of overlaps over all of its image's rows -> (gt_idx [B, A], fg [B, A], mask_pos)."""
    m = mask_pos.shape[1]
    multi = mask_pos.sum(1) > 1
    if m and bool(multi.any()):
        win = torch.nn.functional.one_hot(overlaps.argmax(1), m).permute(0, 2, 1).bool()
        mask_pos = torch.where(multi[:, None, :], win, mask_pos)
    return mask_pos.to(torch.uint8).argmax(1) if m else mask_pos.new_zeros(mask_pos.shape[0], mask_pos.shape[2], dtype=torch.long), \
        mask_pos.any(1), mask_pos


def atss(anc, counts_per_level, boxes, mask, topk=9):
    """ATSS positives -> (mask_pos bool [B, m, A], overlaps fp64 [B, m, A])."""
    B, m = boxes.shape[:2]
    ov = iou_anchor_boxes(boxes, anc)
    gc = (boxes[..., :2] + boxes[..., 2:]) / 2.0
    ac = (anc[:, :2] + anc[:, 2:]) / 2.0
    dist = (gc[..., None, :] - ac).pow(2).sum(-1).sqrt()
    cand = []
    o = 0
    for n in counts_per_level:
        k = min(topk, n)
        cand.append(torch.sort(dist[..., o:o + n], dim=-1, stable=True).indices[..., :k] + o)
        o += n
    cand = torch.cat(cand, -1)
    cov = ov.gather(-1, cand)
    n = cov.shape[-1]
    mean = cov.sum(-1, keepdim=True) / n
    thr = mean + ((cov - mean) ** 2).sum(-1, keepdim=True).div(n - 1).sqrt()
    pos = torch.zeros_like(ov, dtype=torch.bool).scatter(-1, cand, cov > thr)
    mask_pos = pos & inside(ac, boxes) & mask[..., None]
    return mask_pos, ov


def class_scores(pred_scores, labels, nc):
    """pred_scores [B, A, nc] at each GT's truncated label -> fp32 [B, m, A], 0 for labels outside [0, nc)."""
    lab = labels.trunc().long()
    valid = (lab >= 0) & (lab < nc)
    sc = pred_scores.detach().float().gather(2, lab.clamp(0, nc - 1)[:, None, :].expand(-1, pred_scores.shape[1], -1)).permute(0, 2, 1)
    return torch.where(valid[..., None], sc, torch.zeros_like(sc))


def tal(pred_scores, pd, points, labels, boxes, mask, nc, topk=13):
    """Task-aligned positives -> (mask_pos bool [B, m, A], overlaps fp64 [B, m, A], align fp64 [B, m, A])."""
    ov = iou_pairs(boxes, pd)
    align = class_scores(pred_scores, labels, nc).pow(1.0) * ov.pow(6.0)
    ins = inside(points, boxes)
    metric = align * ins
    top = torch.sort(metric, dim=-1, descending=True, stable=True).indices[..., :topk]
    sel = torch.zeros_like(ins).scatter(-1, top, True)
    return sel & ins & mask[..., None], ov, align


def box_loss(p, t, iou_type, eps=1e-10):
    """1 - GIoU or 1 - SIoU of pred boxes p (fp32 [N, 4] xyxy) against targets t (fp64 [N, 4]), element-wise -> fp64 [N, 1]."""
    px1, py1, px2, py2 = p.split(1, -1)
    tx1, ty1, tx2, ty2 = t.split(1, -1)
    inter = (torch.min(px2, tx2) - torch.max(px1, tx1)).clamp(0) * (torch.min(py2, ty2) - torch.max(py1, ty1)).clamp(0)
    pw, ph = px2 - px1, py2 - py1 + eps
    tw, th = tx2 - tx1, ty2 - ty1 + eps
    union = pw * ph + tw * th - inter + eps
    iou = inter / union
    cw = torch.max(px2, tx2) - torch.min(px1, tx1)
    ch = torch.max(py2, ty2) - torch.min(py1, ty1)
    if iou_type == 'giou':
        hull = cw * ch + eps
        return 1.0 - (iou - (hull - union) / hull)
    dx = (tx1 + tx2 - px1 - px2) * 0.5 + eps
    dy = (ty1 + ty2 - py1 - py2) * 0.5 + eps
    r = torch.pow(dx ** 2 + dy ** 2, 0.5)
    sx, sy = torch.abs(dx) / r, torch.abs(dy) / r
    sin_a = torch.where(sx > pow(2, 0.5) / 2, sy, sx)
    angle = torch.cos(torch.arcsin(sin_a) * 2 - math.pi / 2)
    g = angle - 2
    dist = 2 - torch.exp(g * (dx / cw) ** 2) - torch.exp(g * (dy / ch) ** 2)
    ow = torch.abs(pw - tw) / torch.max(pw, tw)
    oh = torch.abs(ph - th) / torch.max(ph, th)
    shape = torch.pow(1 - torch.exp(-1 * ow), 4) + torch.pow(1 - torch.exp(-1 * oh), 4)
    return 1.0 - (iou - 0.5 * (dist + shape))


def losses(shapes, pred_scores, pred_distri, gt, assigner='atss', iou_type='giou', nc=80, strides=STRIDES, grid_cell_size=5.0,
           grid_cell_offset=0.5, ori_img_size=640, loss_weight=LOSS_WEIGHT):
    """-> (dict iou / dfl / class of the box loss L, assignment dict).  pred_distri may require grad; pred_scores gets none.
    The assignment: fg [B, A] bool, gt_idx [B, A], labels [B, A] (nc for background), boxes fp64 [B, A, 4] pixels, scores fp64 [B, A]."""
    dev = pred_distri.device
    B = pred_distri.shape[0]
    anc, points, per_level, stride = anchors(shapes, strides, grid_cell_size, grid_cell_offset, dev)
    labels, boxes, mask, counts = pack(gt, B, ori_img_size)
    pts_s = points / stride
    lt, rb = pred_distri.split(2, -1)
    pred = torch.cat([pts_s - lt, pts_s + rb], -1)
    pd = pred.detach() * stride
    m, A = boxes.shape[1], anc.shape[0]
    if m == 0:
        fg = torch.zeros(B, A, dtype=torch.bool, device=dev)
        gt_idx = torch.zeros(B, A, dtype=torch.long, device=dev)
        tboxes = torch.zeros(B, A, 4, dtype=torch.float64, device=dev)
        score = torch.zeros(B, A, dtype=torch.float64, device=dev)
        lab = torch.full((B, A), nc, dtype=torch.long, device=dev)
    else:
        if assigner == 'atss':
            mask_pos, ov = atss(anc, per_level, boxes, mask)
            gt_idx, fg, mask_pos = resolve(mask_pos, ov)
        else:
            mask_pos, ov, align = tal(pred_scores, pd, points, labels, boxes, mask, nc)
            gt_idx, fg, mask_pos = resolve(mask_pos, ov)
        bi = torch.arange(B, device=dev)[:, None]
        glab = labels.trunc().long()[bi, gt_idx]
        valid = fg & (glab >= 0) & (glab < nc)
        lab = torch.where(fg, glab, torch.full_like(glab, nc))
        tboxes = boxes[bi, gt_idx]
        if assigner == 'atss':
            soft = iou_pairs(boxes, pd).mul(mask_pos).amax(1).float()
            score = torch.where(valid, soft, torch.zeros_like(soft)).double()
        else:
            am = align * mask_pos
            pos_align = am.amax(-1, keepdim=True)
            pos_ov = (ov * mask_pos).amax(-1, keepdim=True)
            norm = (am * pos_ov / (pos_align + 1e-9)).amax(1)
            score = torch.where(valid, norm, torch.zeros_like(norm))
    tb = tboxes / stride
    npos = int(fg.sum())
    if npos == 0:
        L = pred_distri.float().sum() * 0.0
        S = score.sum()
    else:
        w = score[fg]
        if assigner == 'atss':
            w = w.float()
            S = w.sum()
        else:
            S = w.sum()
        l = box_loss(pred[fg], tb[fg], iou_type) * w[:, None]
        L = l.sum() if float(S) == 0 else l.sum() / S
    out = {'iou': loss_weight['iou'] * L, 'dfl': loss_weight['dfl'] * L, 'class': loss_weight['class'] * L}
    return out, dict(fg=fg, gt_idx=gt_idx, labels=lab, boxes=tboxes, scores=score, num_pos=npos, target_scores_sum=S, counts=counts)


def level_shapes(H, W, strides=STRIDES):
    return [(H // s, W // s) for s in strides]


def make_targets(gen, B, H, W, n_per_image, ori_img_size=640, nc=80, min_wh=8.0, max_wh=None):
    """Random GT rows [n, 6] fp32 (image, label, cx, cy, w, h normalised by ori_img_size) inside an H x W image, images interleaved."""
    max_wh = max_wh or min(H, W) * 0.6
    rows = []
    for b, n in enumerate(n_per_image):
        for _ in range(n):
            w = min_wh + float(torch.rand((), generator=gen)) * (max_wh - min_wh)
            h = min_wh + float(torch.rand((), generator=gen)) * (max_wh - min_wh)
            cx = w / 2 + float(torch.rand((), generator=gen)) * (W - w)
            cy = h / 2 + float(torch.rand((), generator=gen)) * (H - h)
            lab = int(torch.randint(0, nc, (), generator=gen))
            rows.append([b, lab, cx / ori_img_size, cy / ori_img_size, w / ori_img_size, h / ori_img_size])
    t = torch.tensor(rows, dtype=torch.float32).reshape(-1, 6)
    if t.shape[0]:
        t = t[torch.randperm(t.shape[0], generator=gen)]
    return t


def make_preds(gen, B, A, nc, dmax=6.0):
    """pred_scores fp32 [B, A, nc] in (0, 1), pred_distri fp32 [B, A, 4] in (0.25, dmax) stride units."""
    scores = torch.sigmoid(torch.randn(B, A, nc, generator=gen) * 2.0)
    distri = 0.25 + torch.rand(B, A, 4, generator=gen) * (dmax - 0.25)
    return scores, distri
