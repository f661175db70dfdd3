"""Functional restatement of the FCOS training loss (src/losses/fcos_loss.py: GenTargets + FCOSLoss) for the tests of csrc/fcos_loss.cu.

fp32 in the reference's operation order and differentiable in the head outputs, on any device.  Every assignment quantity is one correctly
rounded fp32 operation, so the targets are bitwise the reference's:
  point (x, y) = (column stride + stride // 2, row stride + stride // 2) per level
  (l, t, r, b) = (x - x1, y - y1, x2 - x, y2 - y); a pair is positive when min(l, t, r, b) > 0, lo < max(l, t, r, b) <= hi (limits in fp32)
                 and max(x - cx, y - cy, cx - x, cy - y) < fp32(1.5 stride), cx = (x1 + x2) / 2
  the matched GT is the first minimum over the m rows of (l + r)(t + b), 99999999 where the pair is not positive; a point without a positive
  pair is background (class 0, centerness -1, regression -1)
  centerness = sqrt((min(l, r) min(t, b)) / (max(l, r) max(t, b) + 1e-10))
Losses: the sigmoid focal loss (alpha 0.25, gamma 2) over every point and class against the one-hot of the label (a label outside 1..nc has
an all-zero row), BCE-with-logits of the centerness and 1 - GIoU (G_area.clamp(1e-10)) over the positives; each a per-image sum over
max(num_pos_b, 1), averaged over the batch.  m = 0 (no GT rows) is an all-background batch here (the reference raises in torch.min)."""
import torch
import torch.nn.functional as F

STRIDES = (8, 16, 32, 64, 128)
LIMIT_RANGE = ((-1, 64), (64, 128), (128, 256), (256, 512), (512, 999999))
NOT_POS = 99999999.0
CASES = {'a': (3, 128, 3), 'b': (1, 192, 80)}  # batch, image side, classes


def points(shapes, strides, device=None):
    """-> (x, y, level) of every point, fp32 [A] / long [A], levels in order and row-major within a level."""
    xs, ys, lv = [], [], []
    for l, ((h, w), s) in enumerate(zip(shapes, strides)):
        col = torch.arange(w, dtype=torch.float32, device=device) * s + s // 2
        row = torch.arange(h, dtype=torch.float32, device=device) * s + s // 2
        xs.append(col[None, :].expand(h, w).reshape(-1))
        ys.append(row[:, None].expand(h, w).reshape(-1))
        lv.append(torch.full((h * w,), l, dtype=torch.long, device=device))
    return torch.cat(xs), torch.cat(ys), torch.cat(lv)


def targets(shapes, boxes, labels, strides=STRIDES, limit_range=LIMIT_RANGE):
    """boxes fp32 [B, m, 4] (x1, y1, x2, y2; -1 rows pad), labels [B, m] -> (cls long [B, A], cnt fp32 [B, A], reg fp32 [B, A, 4],
    matched_gt long [B, A], -1 = background)."""
    dev = boxes.device
    x, y, lv = points(shapes, strides, dev)
    B, m = boxes.shape[0], boxes.shape[1]
    A = x.shape[0]
    if m == 0:
        return (torch.zeros(B, A, dtype=torch.long, device=dev), torch.full((B, A), -1.0, device=dev), torch.full((B, A, 4), -1.0, device=dev),
                torch.full((B, A), -1, dtype=torch.long, device=dev))
    lo = torch.tensor([float(r[0]) for r in limit_range], dtype=torch.float32, device=dev)[lv][None, :, None]
    hi = torch.tensor([float(r[1]) for r in limit_range], dtype=torch.float32, device=dev)[lv][None, :, None]
    rad = torch.tensor([s * 1.5 for s in strides], dtype=torch.float32, device=dev)[lv][None, :, None]
    px, py = x[None, :, None], y[None, :, None]
    x1, y1, x2, y2 = (boxes[..., k][:, None, :] for k in range(4))
    off = torch.stack([px - x1, py - y1, x2 - px, y2 - py], -1)  # [B, A, m, 4]
    area = (off[..., 0] + off[..., 2]) * (off[..., 1] + off[..., 3])
    cx, cy = (x1 + x2) / 2, (y1 + y2) / 2
    cmax = torch.stack([px - cx, py - cy, cx - px, cy - py], -1).max(-1).values
    omax = off.max(-1).values
    pos = (off.min(-1).values > 0) & (omax > lo) & (omax <= hi) & (cmax < rad)
    idx = torch.where(pos, area, torch.full_like(area, NOT_POS)).min(-1).indices  # the first minimum
    fg = pos.any(-1)
    reg = off.gather(2, idx[:, :, None, None].expand(B, A, 1, 4)).squeeze(2)
    lr_min, lr_max = torch.min(reg[..., 0], reg[..., 2]), torch.max(reg[..., 0], reg[..., 2])
    tb_min, tb_max = torch.min(reg[..., 1], reg[..., 3]), torch.max(reg[..., 1], reg[..., 3])
    cnt = ((lr_min * tb_min) / (lr_max * tb_max + 1e-10)).sqrt()
    cls = labels.long().gather(1, idx)
    return (torch.where(fg, cls, torch.zeros_like(cls)), torch.where(fg, cnt, torch.full_like(cnt, -1.0)),
            torch.where(fg[..., None], reg, torch.full_like(reg, -1.0)), torch.where(fg, idx, torch.full_like(idx, -1)))


def flat(outs):
    """Per-level [B, c, h, w] -> [B, A, c] in point order."""
    B, c = outs[0].shape[:2]
    return torch.cat([o.permute(0, 2, 3, 1).reshape(B, -1, c) for o in outs], 1)


def focal_sum(logits, onehot, gamma=2.0, alpha=0.25):
    """Sigmoid focal loss summed over the last two dims: logits, onehot [B, A, nc] -> [B]."""
    p = logits.sigmoid()
    pt = p * onehot + (1.0 - p) * (1.0 - onehot)
    w = alpha * onehot + (1.0 - alpha) * (1.0 - onehot)
    return (-w * torch.pow(1.0 - pt, gamma) * pt.log()).sum((1, 2))


def giou_sum(p, t):
    """sum of 1 - GIoU over rows of ltrb predictions p and targets t [n, 4]."""
    inter_w = (torch.min(p[:, 2], t[:, 2]) + torch.min(p[:, 0], t[:, 0])).clamp(min=0)
    inter_h = (torch.min(p[:, 3], t[:, 3]) + torch.min(p[:, 1], t[:, 1])).clamp(min=0)
    overlap = inter_w * inter_h
    union = ((p[:, 2] + p[:, 0]) * (p[:, 3] + p[:, 1]) + (t[:, 2] + t[:, 0]) * (t[:, 3] + t[:, 1])) - overlap
    enc_w = (torch.max(p[:, 2], t[:, 2]) + torch.max(p[:, 0], t[:, 0])).clamp(min=0)
    enc_h = (torch.max(p[:, 3], t[:, 3]) + torch.max(p[:, 1], t[:, 1])).clamp(min=0)
    enclose = enc_w * enc_h
    giou = overlap / union - (enclose - union) / enclose.clamp(1e-10)
    return (1.0 - giou).sum()


def losses(preds, boxes, labels, strides=STRIDES, limit_range=LIMIT_RANGE):
    """preds = [cls_logits, cnt_logits, reg_preds] (lists of [B, c, h, w]) -> ((cls_loss, cnt_loss, reg_loss, total_loss),
    (cls_t, cnt_t, reg_t, matched_gt))."""
    cls_l, cnt_l, reg_l = preds
    if not len(cls_l) == len(cnt_l) == len(reg_l) == len(strides) == len(limit_range):
        raise ValueError('one stride and one limit range per level')
    shapes = [tuple(c.shape[2:]) for c in cls_l]
    cls_t, cnt_t, reg_t, matched = targets(shapes, boxes, labels, strides, limit_range)
    B, nc = cls_l[0].shape[:2]
    x_cls, x_cnt, x_reg = flat(cls_l), flat(cnt_l)[..., 0], flat(reg_l)
    mask = cnt_t > -1
    num_pos = mask.sum(1).clamp(min=1).float()
    onehot = (torch.arange(1, nc + 1, device=cls_t.device)[None, None, :] == cls_t[..., None]).float()
    cls_sum = focal_sum(x_cls, onehot)
    cnt_sum = torch.stack([F.binary_cross_entropy_with_logits(x_cnt[b][mask[b]], cnt_t[b][mask[b]], reduction='sum') for b in range(B)])
    reg_sum = torch.stack([giou_sum(x_reg[b][mask[b]], reg_t[b][mask[b]]) for b in range(B)])
    cls_loss, cnt_loss, reg_loss = (cls_sum / num_pos).mean(), (cnt_sum / num_pos).mean(), (reg_sum / num_pos).mean()
    return (cls_loss, cnt_loss, reg_loss, cls_loss + cnt_loss + reg_loss), (cls_t, cnt_t, reg_t, matched)


def level_shapes(H, W, strides=STRIDES):
    return [(-(-H // s), -(-W // s)) for s in strides]


def head_outputs(B, nc, shapes, strides, gen, device=None):
    """Seeded head outputs: class logits ~ 1.5 N - 2, centerness logits ~ N, ltrb predictions exp(0.6 N) 2 stride (positive, as the
    reference's ScaleExp gives)."""
    cls, cnt, reg = [], [], []
    for (h, w), s in zip(shapes, strides):
        cls.append(torch.randn(B, nc, h, w, generator=gen) * 1.5 - 2.0)
        cnt.append(torch.randn(B, 1, h, w, generator=gen))
        reg.append(torch.exp(torch.randn(B, 4, h, w, generator=gen) * 0.6) * (2.0 * s))
    if device is not None:
        cls, cnt, reg = [[t.to(device) for t in ts] for ts in (cls, cnt, reg)]
    return [cls, cnt, reg]


def tie_predictions(preds, boxes, labels, gen, share=0.2):
    """Sets a share of the positives' ltrb predictions to their targets exactly (every torch.min / torch.max of the GIoU ties) and as many
    again on channel 0 only."""
    reg = preds[2]
    shapes = [tuple(r.shape[2:]) for r in reg]
    _, _, reg_t, matched = targets(shapes, boxes, labels)
    u = torch.rand(matched.shape, generator=gen).to(matched.device)
    o = 0
    for r in reg:
        h, w = r.shape[2:]
        n = h * w
        fg, uu, t = matched[:, o:o + n] >= 0, u[:, o:o + n], reg_t[:, o:o + n].permute(0, 2, 1).reshape(r.shape)
        full = (fg & (uu < share)).reshape(r.shape[0], 1, h, w)
        one = (fg & (uu >= share) & (uu < 2 * share)).reshape(r.shape[0], 1, h, w)
        r.copy_(torch.where(full, t, r))
        r[:, :1].copy_(torch.where(one, t[:, :1], r[:, :1]))
        o += n


def _pad(rows, m):
    b = torch.full((m, 4), -1.0)
    lab = torch.full((m,), -1, dtype=torch.long)
    for i, (box, c) in enumerate(rows):
        b[i] = torch.tensor(box, dtype=torch.float32)
        lab[i] = c
    return b, lab


def _random_rows(n, H, nc, gen):
    rows = []
    for _ in range(n):
        u = torch.rand(4, generator=gen)
        w, h = 16 + float(u[0]) * (H * 0.6), 16 + float(u[1]) * (H * 0.6)
        x1, y1 = float(u[2]) * (H - w), float(u[3]) * (H - h)
        rows.append(([x1, y1, x1 + w, y1 + h], 1 + int(torch.randint(0, nc, (1,), generator=gen))))
    return rows


def fixture_case(seed, case):
    """-> (preds [cls, cnt, reg] lists, boxes fp32 [B, m, 4], labels long [B, m]).
    'a' (3 x 128², 3 classes): image 0 has random GTs, one labelled -1 and one nc + 1, and padded rows; image 1 has only padded rows; image 2
        has a GT with max(l, t, r, b) = 64 exactly at a stride-8 point, one with a stride-8 point on its left edge, and one whose centre
        offset equals the stride-8 radius exactly at a point.
    'b' (1 x 192², 80 classes): two overlapping GTs of equal area (the first row wins), one with max(l, t, r, b) = 128 exactly at a
        stride-16 point, one with 64 exactly at a stride-16 point, random GTs and padded rows.
    The class logits are multiples of 1/8, which keeps the stored fixture small: the inputs and the background gradients take few distinct
    values and compress."""
    B, H, nc = CASES[case]
    gen = torch.Generator().manual_seed(seed)
    if case == 'a':
        img0 = _random_rows(3, H, nc, gen) + [([20.0, 30.0, 90.0, 100.0], -1), ([50.0, 10.0, 120.0, 70.0], nc + 1)]
        img2 = [([4.0, 40.0, 124.0, 100.0], 1),    # point (68, 68): l = 64 (stride 8, range (-1, 64])
                ([28.0, 20.0, 60.0, 52.0], 2),     # point (28, y): l = 0, on the edge
                ([60.0, 80.0, 116.0, 120.0], 3)]   # point (100, 100): x - cx = 12 = 1.5 * 8
        rows = [img0, [], img2]
    else:
        img0 = [([120.0, 30.0, 200.0, 90.0], 5), ([124.0, 34.0, 204.0, 94.0], 7),  # equal areas at point (164, 60)
                ([40.0, 100.0, 260.0, 240.0], 11),   # point (168, 168): l = 128 (stride 16, range (64, 128])
                ([40.0, 70.0, 150.0, 140.0], 12)] + _random_rows(4, H, nc, gen)  # point (104, 104): l = 64, not in (64, 128]
        rows = [img0]
    m = max(len(r) for r in rows) + 2
    padded = [_pad(r, m) for r in rows]
    boxes = torch.stack([p[0] for p in padded])
    labels = torch.stack([p[1] for p in padded])
    preds = head_outputs(B, nc, level_shapes(H, H), STRIDES, gen)
    preds[0] = [torch.round(c * 8.0) / 8.0 for c in preds[0]]
    tie_predictions(preds, boxes, labels, gen)
    return preds, boxes, labels
