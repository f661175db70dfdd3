"""ORACLE (test infrastructure only -- never imported by the product path).

CPU fp32 restatement of the reference's FCOS-R50 inference forward against a reference-format ``state_dict``:
ResNet-50 (third-party torchvision.models.resnet50, wrapped by src/models/backbones/seg/resnet.py:27-154; torchvision is
not vendored -- the Bottleneck algorithm is restated here from its published definition: 1x1 -> 3x3(stride) -> 1x1, BN after
each, ReLU after the first two and after the residual add, 1x1(stride)+BN downsample on the first block of a layer),
FCOSFPN (src/models/necks/fcos_fpn.py:12-55), FCOSHead (src/models/heads/fcos_head.py:22-84),
FCOSDetect (src/models/detects/fcos_detect.py:34-186).  Pinned against the reference modules run in the build
container by tools/make_golden.py -> tests/golden/fcos_*.npz.
"""
import numpy as np
import torch
import torch.nn.functional as F

RESNET50_BLOCKS = (3, 4, 6, 3)
BN_EPS = 1e-5  # torchvision BatchNorm2d default; the FCOS model does not override it (src/models/fcos.py:52-61)
STRIDES = (8, 16, 32, 64, 128)


def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + '.running_mean'], sd[p + '.running_var'], sd[p + '.weight'], sd[p + '.bias'], False, 0.0, BN_EPS)


def bottleneck(x, sd, p, stride):
    """torchvision.models.resnet.Bottleneck.forward (v1.5: stride on conv2)."""
    out = F.relu(_bn(F.conv2d(x, sd[p + '.conv1.weight']), sd, p + '.bn1'))
    out = F.relu(_bn(F.conv2d(out, sd[p + '.conv2.weight'], None, stride, 1), sd, p + '.bn2'))
    out = _bn(F.conv2d(out, sd[p + '.conv3.weight']), sd, p + '.bn3')
    if (p + '.downsample.0.weight') in sd:
        x = _bn(F.conv2d(x, sd[p + '.downsample.0.weight'], None, stride), sd, p + '.downsample.1')
    return F.relu(out + x)


def resnet50(x, sd, prefix='backbone.', out_stages=(2, 3, 4)):
    """ResNet.forward (src/models/backbones/seg/resnet.py:139-154), non-deep stem (:81-83): conv7x7 s2 p3 + BN + ReLU,
    maxpool 3x3 s2 p1, layer1..4."""
    x = F.relu(_bn(F.conv2d(x, sd[prefix + 'stem.0.weight'], None, 2, 3), sd, prefix + 'stem.1'))
    x = F.max_pool2d(x, 3, 2, 1)
    outs = []
    for li, nb in enumerate(RESNET50_BLOCKS, start=1):
        for bi in range(nb):
            x = bottleneck(x, sd, f'{prefix}layer{li}.{bi}', 2 if (bi == 0 and li > 1) else 1)
        if li in out_stages:
            outs.append(x)
    return outs


def fcos_fpn(feats, sd, prefix='neck.'):
    """FCOSFPN.forward (src/models/necks/fcos_fpn.py:40-55)."""
    C3, C4, C5 = feats
    conv = lambda x, n, s=1, p=0: F.conv2d(x, sd[f'{prefix}{n}.weight'], sd[f'{prefix}{n}.bias'], s, p)
    P3, P4, P5 = conv(C3, 'prj_3'), conv(C4, 'prj_4'), conv(C5, 'prj_5')
    P4 = P4 + F.interpolate(P5, size=P4.shape[2:], mode='nearest')
    P3 = P3 + F.interpolate(P4, size=P3.shape[2:], mode='nearest')
    P3, P4, P5 = conv(P3, 'conv_3', 1, 1), conv(P4, 'conv_4', 1, 1), conv(P5, 'conv_5', 1, 1)
    P6 = conv(P5, 'conv_out6', 2, 1)
    P7 = conv(F.relu(P6), 'conv_out7', 2, 1)
    return [P3, P4, P5, P6, P7]


def fcos_head(levels, sd, prefix='head.'):
    """FCOSHead.forward (src/models/heads/fcos_head.py:69-84): towers of 4 x (3x3 conv + GroupNorm(32) + ReLU) shared over the
    levels; cls 3x3, centerness 3x3 on the regression tower (cnt_on_reg), reg 3x3 then exp(scale_i * x) (ScaleExp :13-19)."""
    def tower(x, name):
        for i in range(4):
            x = F.conv2d(x, sd[f'{prefix}{name}.{3 * i}.weight'], sd[f'{prefix}{name}.{3 * i}.bias'], 1, 1)
            x = F.relu(F.group_norm(x, 32, sd[f'{prefix}{name}.{3 * i + 1}.weight'], sd[f'{prefix}{name}.{3 * i + 1}.bias'], 1e-5))
        return x

    cls, cnt, reg = [], [], []
    for i, P in enumerate(levels):
        c, r = tower(P, 'cls_conv'), tower(P, 'reg_conv')
        cls.append(F.conv2d(c, sd[prefix + 'cls_logits.weight'], sd[prefix + 'cls_logits.bias'], 1, 1))
        cnt.append(F.conv2d(r, sd[prefix + 'cnt_logits.weight'], sd[prefix + 'cnt_logits.bias'], 1, 1))
        reg.append(torch.exp(F.conv2d(r, sd[prefix + 'reg_pred.weight'], sd[prefix + 'reg_pred.bias'], 1, 1) * sd[f'{prefix}scale_exp.{i}.scale']))
    return cls, cnt, reg


def coords_fmap2orig(h, w, stride):
    """src/models/detects/fcos_detect.py:14-31."""
    sx = torch.arange(0, w * stride, stride, dtype=torch.float32)
    sy = torch.arange(0, h * stride, stride, dtype=torch.float32)
    yy, xx = torch.meshgrid(sy, sx, indexing='ij')
    return torch.stack([xx.reshape(-1), yy.reshape(-1)], -1) + stride // 2


def box_nms(boxes, scores, thr):
    """FCOSDetect.box_nms (:108-139): '+1' areas, intersection without +1, keeps iou <= thr evaluated in float32
    (tensor <= python float), descending score order (ties: lower index first here; the reference's sort is unstable)."""
    boxes = np.asarray(boxes, np.float32)
    n = boxes.shape[0]
    if n == 0:
        return np.zeros((0,), np.int64)
    x1, y1, x2, y2 = boxes[:, 0], boxes[:, 1], boxes[:, 2], boxes[:, 3]
    areas = (x2 - x1 + np.float32(1)) * (y2 - y1 + np.float32(1))
    order = np.argsort(-np.asarray(scores, np.float32), kind='stable')
    thr32 = np.float32(thr)
    keep = []
    while order.size > 0:
        i = order[0]
        keep.append(int(i))
        if order.size == 1:
            break
        rest = order[1:]
        xmin = np.maximum(x1[rest], x1[i])
        ymin = np.maximum(y1[rest], y1[i])
        xmax = np.minimum(x2[rest], x2[i])
        ymax = np.minimum(y2[rest], y2[i])
        inter = np.maximum(xmax - xmin, np.float32(0)) * np.maximum(ymax - ymin, np.float32(0))
        with np.errstate(divide='ignore', invalid='ignore'):
            iou = inter / (areas[i] + areas[rest] - inter)
        order = rest[iou <= thr32]
    return np.asarray(keep, np.int64)


def fcos_detect(cls, cnt, reg, score_threshold=0.05, nms_iou_threshold=0.6, max_num=1000, strides=STRIDES):
    """FCOSDetect.forward + _post_process (:42-105).  Returns per image (scores [n], classes [n] (1-based), boxes [n,4],
    loc [n] = index of the kept location in the concatenated level order) -- variable length instead of the reference's
    torch.stack (which fails when images keep different counts)."""
    B = cls[0].shape[0]
    cat = lambda xs: torch.cat([x.permute(0, 2, 3, 1).reshape(B, -1, x.shape[1]) for x in xs], 1)
    cls_l, cnt_l, reg_p = cat(cls), cat(cnt), cat(reg)
    coords = torch.cat([coords_fmap2orig(x.shape[2], x.shape[3], s) for x, s in zip(cls, strides)], 0)
    cls_p, cnt_p = cls_l.sigmoid(), cnt_l.sigmoid()
    sc, cl = torch.max(cls_p, dim=-1)
    sc = torch.sqrt(sc * cnt_p.squeeze(-1))
    cl = cl + 1
    boxes = torch.cat([coords[None] - reg_p[..., :2], coords[None] + reg_p[..., 2:]], -1)
    out = [post_process(sc[b].numpy(), cl[b].numpy(), boxes[b].numpy(), score_threshold, nms_iou_threshold, max_num) for b in range(B)]
    return out, (sc, cl, boxes)


def post_process(s, c, b, score_threshold=0.05, nms_iou_threshold=0.6, max_num=1000):
    """FCOSDetect._post_process (:60-105) on the decoded arrays of ONE image: scores [N], classes [N] (1-based), boxes [N,4]
    -> (scores [n], classes [n], boxes [n,4], loc [n])."""
    k = min(max_num, s.shape[-1])
    top = np.argsort(-s, kind='stable')[:k]  # torch.topk(sorted=True); ties: lower index first (defined here)
    s_t, c_t, b_t = s[top], c[top], b[top]
    m = s_t >= np.float32(score_threshold)
    s_m, c_m, b_m, loc = s_t[m], c_t[m], b_t[m], top[m]
    if s_m.size == 0:
        return s_m, c_m, b_m, loc
    off = c_m.astype(np.float32) * (b_m.max() + np.float32(1))  # batched_nms (:141-153)
    keep = box_nms(b_m + off[:, None], s_m, nms_iou_threshold)
    return s_m[keep], c_m[keep], b_m[keep], loc[keep]


def forward(x, sd):
    with torch.no_grad():
        feats = resnet50(x, sd)
        levels = fcos_fpn(feats, sd)
        cls, cnt, reg = fcos_head(levels, sd)
    return feats, levels, cls, cnt, reg
