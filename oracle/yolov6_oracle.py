"""ORACLE (test infrastructure only -- never imported by the product path).

CPU restatement in torch of the reference's YOLOv6-n / YOLOv6-s inference path (TYPE yolov6_n / yolov6_s, use_dfl False, fuse_ab False):
  backbone  YOLOv6EfficientRep.forward   src/models/backbones/det/yolov6_efficient_rep.py:58-66 (stem RepVGGBlock stride 2, stages of
            RepVGGBlock(stride 2) + RepBlock, SimCSPSPPF in stage 4: modules/yolo_modules.py:218-242, RepVGGBlock.forward :322-331 with the
            three training-form branches summed, RepBlock :465-471)
  neck      YOLOv6RepBiPAN.forward       src/models/necks/det/yolov6_repbipan.py:60-80 (BiFusion yolo_modules.py:245-265)
  head      YOLOv6Effidehead.forward     src/models/heads/det/yolov6_effidehead.py:129-148 (eval branch)
  detect    YOLOv6Detect.forward         src/models/detects/yolov6_detect.py:36-50 (generate_anchors mode 'af', dist2bbox 'xywh')
  nms       non_max_suppression          src/models/yolov6.py:32-107 (torchvision.ops.nms restated by oracle.nms_oracle.greedy_nms)

Pinned against the reference's own modules by tools/make_golden_yolov6.py (tests/golden/yolov6_*.npz).  Like oracle.nms_oracle, the
max_nms cut (:92-93) uses a stable sort where the reference's argsort is unstable; inputs without exactly tied scores behave identically."""
import numpy as np
import torch
import torch.nn.functional as F

from .nms_oracle import greedy_nms, xywh2xyxy

STRIDES = [8, 16, 32]
BN_EPS = 1e-3


def seeded_state_dict(keys_shapes, seed):
    """Deterministic weights and BN statistics for the (key, shape) list of a model, in key order: any module with the same keys in the same
    order gets the same tensors.  Conv weights ~ N(0, 1.2^2 / fan_in); BN gamma U(0.25, 0.75) (activations stay O(1) through the summed
    RepVGG branches), beta N(0, 0.2^2), mean N(0, 0.3^2), var U(0.5, 1.5); the head's class-logit bias near the reference's prior (-4.6)
    and its distance bias at 3 cells so that the detections are sparse and the boxes well formed, as in a trained model."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shape in keys_shapes:
        shape = tuple(int(s) for s in shape)
        if k.endswith('num_batches_tracked'):
            sd[k] = torch.zeros(shape, dtype=torch.int64)
        elif k.endswith('proj'):
            sd[k] = torch.linspace(0, shape[0] - 1, shape[0])
        elif k.endswith('running_mean'):
            sd[k] = torch.randn(shape, generator=g) * 0.3
        elif k.endswith('running_var'):
            sd[k] = torch.rand(shape, generator=g) + 0.5
        elif k.endswith('weight') and len(shape) == 1:
            sd[k] = torch.rand(shape, generator=g) * 0.5 + 0.25
        elif k.endswith('weight'):
            fan = int(np.prod(shape[1:]))
            scale = 0.4 if ('cls_preds' in k or 'reg_preds' in k) else 1.2
            sd[k] = torch.randn(shape, generator=g) * (scale / fan ** 0.5)
        elif 'cls_preds' in k:
            sd[k] = torch.randn(shape, generator=g) * 1.0 - 4.6
        elif 'reg_preds' in k:
            sd[k] = torch.randn(shape, generator=g) * 0.3 + 3.0
        else:
            sd[k] = torch.randn(shape, generator=g) * 0.2
    return sd


def bn(y, sd, p):
    return F.batch_norm(y, sd[p + '.running_mean'], sd[p + '.running_var'], sd[p + '.weight'], sd[p + '.bias'], False, 0.0, BN_EPS)


def conv_module(x, sd, p, stride=1, pad=0, act='relu'):
    """bricks ConvModule: act(BN(conv(x))) (no conv bias with a norm)."""
    y = bn(F.conv2d(x, sd[p + '.conv.weight'], None, stride, pad), sd, p + '.bn')
    return F.relu(y) if act == 'relu' else F.silu(y) if act == 'silu' else y


def repvgg(x, sd, p, stride=1):
    """RepVGGBlock.forward: relu(rbr_dense(x) + rbr_1x1(x) + rbr_identity(x))."""
    y = conv_module(x, sd, p + '.rbr_dense', stride, 1, None) + conv_module(x, sd, p + '.rbr_1x1', stride, 0, None)
    if p + '.rbr_identity.weight' in sd:
        y = y + bn(x, sd, p + '.rbr_identity')
    return F.relu(y)


def rep_block(x, sd, p):
    x = repvgg(x, sd, p + '.conv1')
    i = 0
    while f'{p}.block.{i}.rbr_dense.conv.weight' in sd:
        x = repvgg(x, sd, f'{p}.block.{i}')
        i += 1
    return x


def sim_csp_sppf(x, sd, p):
    x1 = conv_module(conv_module(conv_module(x, sd, p + '.cv1'), sd, p + '.cv3', 1, 1), sd, p + '.cv4')
    y0 = conv_module(x, sd, p + '.cv2')
    y1 = F.max_pool2d(x1, 5, 1, 2)
    y2 = F.max_pool2d(y1, 5, 1, 2)
    y3 = conv_module(conv_module(torch.cat([x1, y1, y2, F.max_pool2d(y2, 5, 1, 2)], 1), sd, p + '.cv5'), sd, p + '.cv6', 1, 1)
    return conv_module(torch.cat((y0, y3), 1), sd, p + '.cv7')


def backbone(x, sd, prefix='backbone.'):
    """-> the four stage outputs (out_stages [1, 2, 3, 4] of the YAML configs)."""
    x = repvgg(x, sd, prefix + 'stem', 2)
    outs = []
    for i in range(1, 5):
        p = f'{prefix}stage{i}'
        x = rep_block(repvgg(x, sd, p + '.0', 2), sd, p + '.1')
        if i == 4:
            x = sim_csp_sppf(x, sd, p + '.2')
        outs.append(x)
    return outs


def bifusion(x0, x1, x2, sd, p):
    u = F.conv_transpose2d(x0, sd[p + '.upsample.weight'], sd[p + '.upsample.bias'], stride=2)
    d = conv_module(conv_module(x2, sd, p + '.cv2'), sd, p + '.downsample', 2, 1)
    return conv_module(torch.cat((u, conv_module(x1, sd, p + '.cv1'), d), 1), sd, p + '.cv3')


def neck(feats, sd, prefix='neck.'):
    x3, x2, x1, x0 = feats
    p = prefix
    fpn_out0 = conv_module(x0, sd, p + 'reduce_layer0')
    f_out0 = rep_block(bifusion(fpn_out0, x1, x2, sd, p + 'bifusion0'), sd, p + 'Rep_p4')
    fpn_out1 = conv_module(f_out0, sd, p + 'reduce_layer1')
    pan_out2 = rep_block(bifusion(fpn_out1, x2, x3, sd, p + 'bifusion1'), sd, p + 'Rep_p3')
    pan_out1 = rep_block(torch.cat([conv_module(pan_out2, sd, p + 'downsample2', 2, 1), fpn_out1], 1), sd, p + 'Rep_n3')
    pan_out0 = rep_block(torch.cat([conv_module(pan_out1, sd, p + 'downsample1', 2, 1), fpn_out0], 1), sd, p + 'Rep_n4')
    return [pan_out2, pan_out1, pan_out0]


def head(feats, sd, prefix='head.'):
    """-> (stem outputs, cls scores [B, L, nc] after the sigmoid, reg distances [B, L, 4])."""
    stems, cls_l, reg_l = [], [], []
    for i, x in enumerate(feats):
        b = x.shape[0]
        s = conv_module(x, sd, f'{prefix}stems.{i}', act='silu')
        c = conv_module(s, sd, f'{prefix}cls_convs.{i}', 1, 1, 'silu')
        r = conv_module(s, sd, f'{prefix}reg_convs.{i}', 1, 1, 'silu')
        co = F.conv2d(c, sd[f'{prefix}cls_preds.{i}.weight'], sd[f'{prefix}cls_preds.{i}.bias'])
        ro = F.conv2d(r, sd[f'{prefix}reg_preds.{i}.weight'], sd[f'{prefix}reg_preds.{i}.bias'])
        stems.append(s)
        cls_l.append(torch.sigmoid(co).reshape(b, co.shape[1], -1))
        reg_l.append(ro.reshape(b, 4, -1))
    return stems, torch.cat(cls_l, -1).permute(0, 2, 1), torch.cat(reg_l, -1).permute(0, 2, 1)


def detect(cls_scores, reg, level_shapes, strides=STRIDES):
    """generate_anchors(is_eval=True, mode='af') + dist2bbox(..., 'xywh') * stride + cat(box, ones, cls) in fp32."""
    pts, st = [], []
    dev = reg.device
    for (h, w), s in zip(level_shapes, strides):
        sy, sx = torch.meshgrid(torch.arange(h, device=dev) + 0.5, torch.arange(w, device=dev) + 0.5, indexing='ij')
        pts.append(torch.stack([sx, sy], -1).float().reshape(-1, 2))
        st.append(torch.full((h * w, 1), float(s), device=dev))
    a, st = torch.cat(pts), torch.cat(st)
    lt, rb = reg[..., :2], reg[..., 2:]
    x1y1, x2y2 = a - lt, a + rb
    box = torch.cat([(x1y1 + x2y2) / 2, x2y2 - x1y1], -1) * st
    return torch.cat([box, torch.ones_like(box[..., :1]), cls_scores], -1)


def forward(x, sd):
    """-> (z [B, L, 5 + nc], dict of intermediates: backbone, neck, stems, cls, reg)."""
    with torch.no_grad():
        b = backbone(x, sd)
        n = neck(b, sd)
        stems, cls_scores, reg = head(n, sd)
        z = detect(cls_scores, reg, [f.shape[2:] for f in n])
    return z, dict(backbone=b, neck=n, stems=stems, cls=cls_scores, reg=reg)


def non_max_suppression(prediction, conf_thres=0.03, iou_thres=0.65, multi_label=True, max_det=300, max_nms=30000, max_wh=4096):
    """src/models/yolov6.py:32-107 (numpy, float32).  Returns per image (det [n,6] = xyxy, conf, cls ; idx [n] int64 = row*nc + cls)."""
    prediction = np.asarray(prediction, dtype=np.float32)
    nc = prediction.shape[2] - 5
    conf32 = np.float32(conf_thres)
    multi_label = multi_label and nc > 1
    out = []
    for x in prediction:
        sel = np.nonzero((x[:, 4] > conf32) & (x[:, 5:].max(1) > conf32))[0]  # :52
        x = x[sel].copy()
        empty = (np.zeros((0, 6), np.float32), np.zeros((0,), np.int64))
        if x.shape[0] == 0:
            out.append(empty)
            continue
        x[:, 5:] *= x[:, 4:5]  # :72
        box = xywh2xyxy(x[:, :4])
        if multi_label:
            i, j = np.nonzero(x[:, 5:] > conf32)
            det = np.concatenate([box[i], x[i, j + 5][:, None], j[:, None].astype(np.float32)], 1)
            ids = sel[i].astype(np.int64) * nc + j
        else:
            j = x[:, 5:].argmax(1)
            conf = x[np.arange(x.shape[0]), j + 5]
            m = conf > conf32
            det = np.concatenate([box, conf[:, None], j[:, None].astype(np.float32)], 1)[m]
            ids = (sel.astype(np.int64) * nc + j)[m]
        if det.shape[0] == 0:
            out.append(empty)
            continue
        if det.shape[0] > max_nms:  # :92-93 (stable here)
            top = np.argsort(-det[:, 4], kind='stable')[:max_nms]
            det, ids = det[top], ids[top]
        boxes = det[:, :4] + det[:, 5:6] * np.float32(max_wh)
        keep = greedy_nms(boxes, det[:, 4], iou_thres, max_keep=max_det)
        out.append((det[keep].astype(np.float32), ids[keep]))
    return out


FWD_SEED, FWD_SHAPE = 1029, (2, 3, 128, 128)    # tests/golden/yolov6_fwd128.npz
POST_SEED, POST_SHAPE = 2029, (1, 3, 320, 320)  # tests/golden/yolov6_post320.npz
SAMPLES = 2048


def fixture_input(seed, shape):
    """The seeded N(0, 1) input image batch of a fixture (regenerated, not stored)."""
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def subsample(t, n=SAMPLES):
    """The elements of t kept in a fixture: the flattened tensor at a stride of ceil(numel / n), about n values spread over every
    image, channel and position."""
    flat = torch.as_tensor(t).reshape(-1)
    return flat[::-(-flat.numel() // n)]


def sparse_candidates(z, conf):
    """(boxes [B, L, 4], rows, classes, scores) of z: every row's box and the class scores above conf, which is all the multi-label NMS
    reads (a row without such a score is dropped by the `max cls > conf` filter, a score not above conf is never selected)."""
    z = np.asarray(z, dtype=np.float32)
    b, r, c = np.nonzero(z[..., 5:] > np.float32(conf))
    return z[..., :4].copy(), np.stack([b, r], 1).astype(np.int32), c.astype(np.int16), z[b, r, c + 5]


def dense_from_candidates(boxes, rows, classes, scores, nc):
    """z with the candidates of sparse_candidates, objectness 1 and every other class score 0: the same NMS result as the full z."""
    z = np.zeros(boxes.shape[:2] + (5 + nc,), np.float32)
    z[..., :4], z[..., 4] = boxes, 1.0
    z[rows[:, 0], rows[:, 1], classes.astype(np.int64) + 5] = scores
    return z


def rel_err(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))
