"""CPU functional restatement of the YOLOv5 training loss (src/losses/yolov5_loss.py:135-278): build_targets' candidate list and the CIoU box,
objectness and class BCE terms, in fp32 torch so that torch.autograd gives the reference gradient with respect to the detect outputs.

Differences from the reference, all where the reference cannot run or is undefined:
  - the in-place clamp of the grid cell uses integer bounds (the reference's float bounds raise on current torch; older torch did this);
  - a class outside [0, nc) gets no one-hot entry and an image index outside [0, B) matches nothing (the reference raises IndexError);
  - the objectness target of a cell hit by several candidates is the last one's, in candidate order.  The reference's index_put_ leaves
    the winner of duplicate indices unspecified: on the CPU it is the last write only while the copy runs serially, which stops at a
    few thousand candidates (a 64-image batch with 2 to 20 targets per image passes it).
"""
import torch
import torch.nn.functional as F


def build_targets(shapes, targets, anchors, anchor_t=4.0):
    """shapes: [(ny, nx)] per level; targets fp32 [nt, 6] (image, class, cx, cy, w, h) normalised; anchors fp32 [nlev, na, 2] in grid units.
    -> per level (b, a, gj, gi, cls) int64 [n] each and (tbox fp32 [n, 4], anchor fp32 [n, 2]), in the reference's order (offset-major:
    centre, +x, +y, -x, -y; then anchor; then target)."""
    na, nt, dev = anchors.shape[1], targets.shape[0], targets.device
    anchors = anchors.to(dev)
    gain = torch.ones(7, device=dev)
    ai = torch.arange(na, device=dev).float().view(na, 1).repeat(1, nt)
    tt = torch.cat((targets.repeat(na, 1, 1), ai[:, :, None]), 2)
    g = 0.5
    off = torch.tensor([[0, 0], [1, 0], [0, 1], [-1, 0], [0, -1]], device=dev).float() * g
    out = []
    for i, (ny, nx) in enumerate(shapes):
        anc = anchors[i]
        gain[2:6] = torch.tensor([nx, ny, nx, ny], device=dev).float()
        t = tt * gain
        if nt:
            r = t[:, :, 4:6] / anc[:, None]
            j = torch.max(r, 1. / r).max(2)[0] < anchor_t
            t = t[j]
            gxy = t[:, 2:4]
            gxi = gain[[2, 3]] - gxy
            j, k = ((gxy % 1. < g) & (gxy > 1.)).T
            l, m = ((gxi % 1. < g) & (gxi > 1.)).T
            j = torch.stack((torch.ones_like(j), j, k, l, m))
            t = t.repeat((5, 1, 1))[j]
            offsets = (torch.zeros_like(gxy)[None] + off[:, None])[j]
        else:
            t = tt[0]
            offsets = 0
        b, c = t[:, :2].long().T
        gxy, gwh = t[:, 2:4], t[:, 4:6]
        gij = (gxy - offsets).long()
        gi, gj = gij.T
        a = t[:, 6].long()
        gj.clamp_(0, ny - 1)  # (in place on views of gij: tbox below uses the clamped cell)
        gi.clamp_(0, nx - 1)
        tbox = torch.cat((gxy - gij, gwh), 1)
        out.append(((b, a, gj.clone(), gi.clone(), c), tbox, anc[a]))
    return out


def bbox_ciou(box1, box2, eps=1e-7):
    """bbox_iou(box1 [4, n], box2 [n, 4], x1y1x2y2=False, CIoU=True) (yolov5_loss.py:11-52), alpha detached."""
    box2 = box2.T
    b1_x1, b1_x2 = box1[0] - box1[2] / 2, box1[0] + box1[2] / 2
    b1_y1, b1_y2 = box1[1] - box1[3] / 2, box1[1] + box1[3] / 2
    b2_x1, b2_x2 = box2[0] - box2[2] / 2, box2[0] + box2[2] / 2
    b2_y1, b2_y2 = box2[1] - box2[3] / 2, box2[1] + box2[3] / 2
    inter = (torch.min(b1_x2, b2_x2) - torch.max(b1_x1, b2_x1)).clamp(0) * (torch.min(b1_y2, b2_y2) - torch.max(b1_y1, b2_y1)).clamp(0)
    w1, h1 = b1_x2 - b1_x1, b1_y2 - b1_y1 + eps
    w2, h2 = b2_x2 - b2_x1, b2_y2 - b2_y1 + eps
    union = w1 * h1 + w2 * h2 - inter + eps
    iou = inter / union
    cw = torch.max(b1_x2, b2_x2) - torch.min(b1_x1, b2_x1)
    ch = torch.max(b1_y2, b2_y2) - torch.min(b1_y1, b2_y1)
    c2 = cw ** 2 + ch ** 2 + eps
    rho2 = ((b2_x1 + b2_x2 - b1_x1 - b1_x2) ** 2 + (b2_y1 + b2_y2 - b1_y1 - b1_y2) ** 2) / 4
    v = (4 / torch.pi ** 2) * torch.pow(torch.atan(w2 / h2) - torch.atan(w1 / h1), 2)
    with torch.no_grad():
        alpha = v / (v - iou + (1 + eps))
    return iou - (rho2 / c2 + v * alpha)


def yolov5_loss(preds, targets, anchors, num_classes, hyp_box=0.05, hyp_obj=1.0, hyp_cls=0.5, balance=(4.0, 1.0, 0.4), gr=1.0, anchor_t=4.0):
    """preds: fp32 NCHW [B, na (5 + nc), ny, nx] (requires_grad for the gradient).  -> (loss [1], items [3], the build_targets lists)."""
    na, no = anchors.shape[1], num_classes + 5
    B, dev = preds[0].shape[0], preds[0].device
    p = [x.view(B, na, no, x.shape[2], x.shape[3]).permute(0, 1, 3, 4, 2) for x in preds]
    tg = build_targets([(x.shape[2], x.shape[3]) for x in preds], targets, anchors, anchor_t)
    lcls, lbox, lobj = torch.zeros(1, device=dev), torch.zeros(1, device=dev), torch.zeros(1, device=dev)
    pw = torch.tensor([1.0], device=dev)
    for i, pi in enumerate(p):
        (b, a, gj, gi, c), tbox, anch = tg[i]
        keep = (b >= 0) & (b < B)
        b, a, gj, gi, c, tbox, anch = b[keep], a[keep], gj[keep], gi[keep], c[keep], tbox[keep], anch[keep]
        tobj = torch.zeros_like(pi[..., 0])
        n = b.shape[0]
        if n:
            ps = pi[b, a, gj, gi]
            pxy = ps[:, :2].sigmoid() * 2. - 0.5
            pwh = (ps[:, 2:4].sigmoid() * 2) ** 2 * anch
            iou = bbox_ciou(torch.cat((pxy, pwh), 1).T, tbox)
            lbox += (1.0 - iou).mean()
            score_iou = iou.detach().clamp(0).type(tobj.dtype)
            cell = ((b * na + a) * pi.shape[2] + gj) * pi.shape[3] + gi  # (the last candidate of each cell sets its target)
            order = torch.arange(n, device=dev)
            last = torch.full((tobj.numel(),), -1, dtype=torch.long, device=dev).scatter_reduce(0, cell, order, 'amax')
            win = last[cell] == order
            tobj[b[win], a[win], gj[win], gi[win]] = ((1.0 - gr) + gr * score_iou)[win]
            if num_classes > 1:
                t = torch.zeros_like(ps[:, 5:])
                ok = (c >= 0) & (c < num_classes)
                t[torch.arange(n, device=dev)[ok], c[ok]] = 1.0
                lcls += F.binary_cross_entropy_with_logits(ps[:, 5:], t, pos_weight=pw)
        lobj += F.binary_cross_entropy_with_logits(pi[..., 4], tobj, pos_weight=pw) * balance[i]
    lbox *= hyp_box
    lobj *= hyp_obj
    lcls *= hyp_cls
    return (lbox + lobj + lcls) * B, torch.cat((lbox, lobj, lcls)).detach(), tg


def candidate_lists(tg, B):
    """build_targets' lists as the kernels report them: per level int [n, 5] (image, anchor, gj, gi, class) and fp32 [n, 6] (tbox, anchor)."""
    res = []
    for (b, a, gj, gi, c), tbox, anch in tg:
        keep = (b >= 0) & (b < B)
        res.append((torch.stack((b, a, gj, gi, c), 1)[keep].int(), torch.cat((tbox, anch), 1)[keep]))
    return res


# ------------------------------------------------------------------------------------------------ the YOLOv5 network in training mode
def conv_module(x, sd, prefix, ksize, stride=1, padding=None):
    """conv (no bias) -> BatchNorm (batch statistics) -> SiLU: c3_train_oracle.base_conv with an explicit padding (the 6x6 stem's 2)."""
    from oracle.c3_train_oracle import BN_EPS, BN_MOMENTUM
    y = F.conv2d(x, sd[prefix + '.conv.weight'], None, stride, (ksize - 1) // 2 if padding is None else padding)
    y = F.batch_norm(y, sd[prefix + '.bn.running_mean'], sd[prefix + '.bn.running_var'], sd[prefix + '.bn.weight'], sd[prefix + '.bn.bias'], True,
                     BN_MOMENTUM, BN_EPS)
    return F.silu(y)


def _c3(x, sd, prefix, n, shortcut):
    """C3 / CSPLayer with either key family (conv1 / conv2 / conv3 or cv1 / cv2 / cv3)."""
    a, b, c = ('cv1', 'cv2', 'cv3') if prefix + '.cv1.conv.weight' in sd else ('conv1', 'conv2', 'conv3')
    x1 = conv_module(x, sd, f'{prefix}.{a}', 1)
    x2 = conv_module(x, sd, f'{prefix}.{b}', 1)
    for i in range(n):
        y = conv_module(conv_module(x1, sd, f'{prefix}.m.{i}.{a}', 1), sd, f'{prefix}.m.{i}.{b}', 3)
        x1 = y + x1 if shortcut else y
    return conv_module(torch.cat((x1, x2), 1), sd, f'{prefix}.{c}', 1)


def network(x, sd, depth_mul=0.33):
    """YOLOv5 (yolov5_csp_darknet.py, yolov5_neck.py, yolov5_detect.py) in training mode over a state_dict with the model's keys: NCHW image
    -> the detect convs' outputs [B, na (5 + nc), ny, nx].  The stem is the 6x6 / stride-2 / pad-2 conv, SPPF the chained 5x5 pools."""
    nb = [max(round(n * depth_mul), 1) for n in (3, 6, 9, 3)]
    nn_ = max(round(3 * depth_mul), 1)
    h = conv_module(x, sd, 'backbone.stem', 6, 2, 2)
    feats = []
    for i in range(1, 5):
        s = f'backbone.stage{i}'
        h = _c3(conv_module(h, sd, s + '.0', 3, 2), sd, s + '.1', nb[i - 1], i < 4)
        if i == 4:
            t = conv_module(h, sd, s + '.2.conv1', 1)
            y1 = F.max_pool2d(t, 5, 1, 2)
            y2 = F.max_pool2d(y1, 5, 1, 2)
            h = conv_module(torch.cat((t, y1, y2, F.max_pool2d(y2, 5, 1, 2)), 1), sd, s + '.2.conv2', 1)
        if i >= 2:
            feats.append(h)
    x3, x4, x5 = feats
    up = lambda t: F.interpolate(t, scale_factor=2, mode='nearest')  # noqa: E731
    x4_t = conv_module(x5, sd, 'neck.up_1.conv', 1)
    x4_up = _c3(torch.cat((up(x4_t), x4), 1), sd, 'neck.up_1.fuse', nn_, False)
    x3_t = conv_module(x4_up, sd, 'neck.up_2.conv', 1)
    x3_up = _c3(torch.cat((up(x3_t), x3), 1), sd, 'neck.up_2.fuse', nn_, False)
    x4_down = _c3(torch.cat((conv_module(x3_up, sd, 'neck.down_1.down', 3, 2), x3_t), 1), sd, 'neck.down_1.fuse', nn_, False)
    x5_down = _c3(torch.cat((conv_module(x4_down, sd, 'neck.down_2.down', 3, 2), x4_t), 1), sd, 'neck.down_2.fuse', nn_, False)
    return [F.conv2d(f, sd[f'detect.m.{i}.weight'], sd[f'detect.m.{i}.bias']) for i, f in enumerate((x3_up, x4_down, x5_down))]


# ------------------------------------------------------------------------------------------------ fixture inputs (tests/golden/yolov5_*.npz)
ANCHORS = [[[1.25, 1.625], [2.0, 3.75], [4.125, 2.875]],
           [[1.875, 3.8125], [3.875, 2.8125], [3.6875, 7.4375]],
           [[3.625, 2.8125], [4.875, 6.1875], [11.65625, 10.1875]]]  # src/models/yolov5.py:157-159 (grid units)
# loss cases: (B, H, W, num_classes); the last image of each case has no target
LOSS_CASES = {'a': (3, 128, 128, 80), 'b': (2, 96, 64, 1)}


def loss_fixture_case(seed, case):
    """The detect outputs and targets of a loss fixture case, regenerated from its seed: outputs [B, 3 (5 + nc), H / s, W / s] ~ 1.5 N(0, 1),
    then 4 random targets per image (the last image empty), then the fixed rows the candidate logic branches on: a GT on integer grid
    coordinates (the 5 offsets, the -x / -y ones back on the centre cell), a GT at the (1, 1) border (the clamp reaches tbox), a GT the ratio
    filter drops on most anchors, and two GTs in the same cells."""
    B, H, W, nc = LOSS_CASES[case]
    g = torch.Generator().manual_seed(seed)
    preds = [torch.randn((B, 3 * (5 + nc), H // s, W // s), generator=g) * 1.5 for s in (8, 16, 32)]
    n = 4 * (B - 1)
    rows = torch.cat([torch.arange(B - 1).repeat_interleave(4).float()[:, None], torch.randint(0, nc, (n, 1), generator=g).float(),
                      torch.rand((n, 2), generator=g) * 0.9 + 0.05, torch.rand((n, 2), generator=g) * 0.3 + 0.02], 1)
    extra = torch.tensor([[0, 0, 0.25, 0.5, 0.1, 0.12], [0, nc - 1, 1.0, 1.0, 0.05, 0.06], [0, 0, 0.5, 0.5, 0.9, 0.004],
                          [0, 0, 0.3, 0.3, 0.1, 0.1], [0, nc - 1, 0.3001, 0.3001, 0.11, 0.09]])
    return preds, torch.cat([rows, extra], 0)


# network fixture: a narrowed YOLOv5-n whose every width is on the training path (16 and 32 channels), 3 classes, a 2 x 3 x 64 x 96 image
NET = dict(backbone=dict(subtype='yolov5_n', out_channels=[64, 128, 128, 128, 128]),
           neck=dict(in_channels=[128, 128, 128], out_channels=[128, 128, 128], depth_mul=0.33, width_mul=0.25),
           detect=dict(num_classes=3, in_channels=[128, 128, 128], width_mul=0.25), image=(2, 3, 64, 96))


def synthetic_state(keys_shapes, seed=0):
    """Seeded parameters for a YOLOv5 (key, shape) list: conv / BatchNorm entries as darknet_train_oracle.synthetic_state(seed); detect conv
    weights ~ N(0, 1 / fan_in) and biases ~ N(0, 0.5^2) drawn in list order from a second generator seeded with seed + 1; the anchors buffer
    is the model's."""
    from oracle import darknet_train_oracle as DO
    det = lambda k: k.startswith('detect.')  # noqa: E731
    base = DO.synthetic_state([(k, s) for k, s in keys_shapes if not det(k)], seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    sd = {}
    for k, shape in keys_shapes:
        if not det(k):
            sd[k] = base[k]
        elif k == 'detect.anchors':
            sd[k] = torch.tensor(ANCHORS)
        elif k.endswith('.weight'):
            sd[k] = torch.randn(shape, generator=g) / (shape[1] * shape[2] * shape[3]) ** 0.5
        elif k.endswith('.bias'):
            sd[k] = torch.randn(shape, generator=g) * 0.5
        else:
            raise KeyError(k)
    return sd


def net_fixture_inputs(f):
    """The parameters, image and output gradients of tests/golden/yolov5_train.npz regenerated from its seeds as
    tools/make_golden_yolov5_train.py drew them -> (keys, state_dict, image, [G_0, G_1, G_2])."""
    import ast
    keys = [str(k) for k in f['keys']]
    shapes = [(k, tuple(ast.literal_eval(str(s)))) for k, s in zip(keys, f['shapes'])]
    param_seed, data_seed = (int(v) for v in f['seeds'])
    g = torch.Generator().manual_seed(data_seed)
    x = torch.rand(NET['image'], generator=g)
    Gs = [torch.randn(tuple(int(d) for d in f[f'y{i}'].shape), generator=g) for i in range(3)]
    return keys, synthetic_state(shapes, seed=param_seed), x, Gs


def net_train_step(x, Gs, sd_np):
    """One forward + backward of `network` with loss = sum_i sum(out_i * G_i) -> ({y_i, grad_<param>, after_<running stat>}: tensors)."""
    sd = {k: torch.as_tensor(v).clone().requires_grad_(torch.as_tensor(v).dtype.is_floating_point and 'running_' not in k and k != 'detect.anchors')
          for k, v in sd_np.items()}
    outs = network(x, sd)
    sum((o * G).sum() for o, G in zip(outs, Gs)).backward()
    res = {f'y{i}': o.detach() for i, o in enumerate(outs)}
    res.update({f'grad_{k}': v.grad for k, v in sd.items() if v.requires_grad})
    res.update({f'after_{k}': v for k, v in sd.items() if 'running_' in k})
    return res
