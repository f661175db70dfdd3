"""ORACLE (test infrastructure only -- never imported by the product path).

CPU restatement of the reference's YOLOX neck and head IN TRAINING MODE, forward and backward, on top of the backbone oracle
(darknet_train_oracle.conv_module / csp_layer):
  YOLOXNeck    src/models/necks/yolox_neck.py:13-74      lateral 1x1, up2 + cat, C3_p4, reduce 1x1, up2 + cat, C3_p3, then bottom-up
                                                         (3x3 / 2 conv + cat, CSPLayer) twice; every CSPLayer with shortcut=False
  YOLOXHead    src/models/heads/yolox_head.py:14-88      per level: 1x1 stem with padding 1, two 3x3 ConvModules per branch, prediction
                                                         convs with bias; output cat(reg, obj, cls) [B, 5 + num_classes, h + 2, w + 2]
written functionally over a state_dict with the reference's key names (prefixes 'neck.' and 'head.').  The backward is torch.autograd's.
Pinned against the reference's own modules by tools/make_golden_yolox_train.py -> tests/golden/yolox_train.npz (<= 1e-5)."""
import torch
import torch.nn.functional as F

from oracle import darknet_train_oracle as DO
from oracle.c3_train_oracle import BN_EPS, BN_MOMENTUM


def head_conv(x, sd, prefix, ksize, padding):
    """ConvModule (convs.py) as the head builds it: conv without bias (any padding) -> BatchNorm (batch statistics) -> SiLU."""
    y = F.conv2d(x, sd[prefix + '.conv.weight'], None, 1, padding)
    y = F.batch_norm(y, sd[prefix + '.bn.running_mean'], sd[prefix + '.bn.running_var'], sd[prefix + '.bn.weight'], sd[prefix + '.bn.bias'], True,
                     BN_MOMENTUM, BN_EPS)
    return y * torch.sigmoid(y)


def neck_depths(depth_mul):
    return [max(round(n * depth_mul), 1) for n in (3, 3, 3, 3)]


def neck(feats, sd, depth_mul=1.0, prefix='neck'):
    """[x2, x1, x0] (NCHW, x2 the largest) -> [pan_out2, pan_out1, pan_out0]."""
    p = prefix + '.' if prefix else ''
    n = neck_depths(depth_mul)
    x2, x1, x0 = feats

    def up(t):
        return F.interpolate(t, scale_factor=2, mode='nearest')
    fpn_out0 = DO.conv_module(x0, sd, p + 'lateral_conv0', 1)
    f_out0 = DO.csp_layer(torch.cat([up(fpn_out0), x1], 1), sd, p + 'C3_p4', n[0], False)
    fpn_out1 = DO.conv_module(f_out0, sd, p + 'reduce_conv1', 1)
    pan_out2 = DO.csp_layer(torch.cat([up(fpn_out1), x2], 1), sd, p + 'C3_p3', n[1], False)
    p_out1 = torch.cat([DO.conv_module(pan_out2, sd, p + 'bu_conv2', 3, 2), fpn_out1], 1)
    pan_out1 = DO.csp_layer(p_out1, sd, p + 'C3_n3', n[2], False)
    p_out0 = torch.cat([DO.conv_module(pan_out1, sd, p + 'bu_conv1', 3, 2), fpn_out0], 1)
    pan_out0 = DO.csp_layer(p_out0, sd, p + 'C3_n4', n[3], False)
    return [pan_out2, pan_out1, pan_out0]


def head(feats, sd, prefix='head'):
    """-> per level cat(reg, obj, cls) [B, 5 + num_classes, h + 2, w + 2] (num_classes from cls_preds' weight)."""
    p = prefix + '.' if prefix else ''
    outs = []
    for k, x in enumerate(feats):
        x = head_conv(x, sd, f'{p}stems.{k}', 1, 1)
        c = head_conv(head_conv(x, sd, f'{p}cls_convs.{k}.0', 3, 1), sd, f'{p}cls_convs.{k}.1', 3, 1)
        r = head_conv(head_conv(x, sd, f'{p}reg_convs.{k}.0', 3, 1), sd, f'{p}reg_convs.{k}.1', 3, 1)
        cls = F.conv2d(c, sd[f'{p}cls_preds.{k}.weight'], sd[f'{p}cls_preds.{k}.bias'])
        reg = F.conv2d(r, sd[f'{p}reg_preds.{k}.weight'], sd[f'{p}reg_preds.{k}.bias'])
        obj = F.conv2d(r, sd[f'{p}obj_preds.{k}.weight'], sd[f'{p}obj_preds.{k}.bias'])
        outs.append(torch.cat([reg, obj, cls], 1))
    return outs


def network(x, sd, subtype='cspdark_s'):
    """Image -> CSPDarknet(subtype) -> YOLOXNeck -> YOLOXHead of the stock YOLOX model of that size (keys 'backbone.', 'neck.', 'head.')."""
    depth_mul = DO.CFG[subtype.split('_')[1]][0]
    return head(neck(DO.csp_darknet(x, sd, subtype, prefix='backbone'), sd, depth_mul), sd)


def _leaves(sd_np):
    sd = {}
    for k, v in sd_np.items():
        t = torch.as_tensor(v).clone()
        if t.dtype.is_floating_point and 'running_' not in k:
            t.requires_grad_(True)
        sd[k] = t
    return sd


def train_step(feats, Gs, sd_np, depth_mul=1.0):
    """Neck + head, one forward + backward with loss = sum_i sum(out_i * G_i).  feats: [x2, x1, x0] NCHW.  Returns (outs, [d loss / d feat_i],
    {param: grad}, {running stat: value after the step})."""
    sd = _leaves(sd_np)
    feats = [f.detach().clone().requires_grad_(True) for f in feats]
    outs = head(neck(feats, sd, depth_mul), sd)
    sum((o * G).sum() for o, G in zip(outs, Gs)).backward()
    grads = {k: v.grad for k, v in sd.items() if v.requires_grad}
    stats = {k: v for k, v in sd.items() if 'running_' in k}
    return [o.detach() for o in outs], [f.grad for f in feats], grads, stats


def _is_pred(k):
    return any(s in k for s in ('cls_preds.', 'reg_preds.', 'obj_preds.'))


def synthetic_state(keys_shapes, seed=0):
    """Seeded parameters for a (key, shape) list: conv / BatchNorm entries as darknet_train_oracle.synthetic_state(seed) over the list without
    the prediction convs; prediction-conv weights ~ N(0, 1 / fan_in) and biases ~ N(0, 0.5^2), drawn in list order from a second generator
    seeded with seed + 1."""
    base = DO.synthetic_state([(k, s) for k, s in keys_shapes if not _is_pred(k)], seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    sd = {}
    for k, shape in keys_shapes:
        if not _is_pred(k):
            sd[k] = base[k]
        elif k.endswith('.weight'):
            fan = 1
            for d in shape[1:]:
                fan *= d
            sd[k] = torch.randn(shape, generator=g) / fan ** 0.5
        elif k.endswith('.bias'):
            sd[k] = torch.randn(shape, generator=g) * 0.5
        else:
            raise KeyError(k)
    return sd


def fixture_inputs(g):
    """The parameters, feature maps and output gradients of tests/golden/yolox_train.npz, regenerated from its seeds exactly as
    tools/make_golden_yolox_train.py drew them -> (keys, state_dict, [x2, x1, x0], [G_0, G_1, G_2], depth_mul)."""
    import ast
    keys = [str(k) for k in g['keys']]
    shapes = [(k, tuple(ast.literal_eval(str(s)))) for k, s in zip(keys, g['shapes'])]
    param_seed, data_seed = (int(v) for v in g['seeds'])
    feat_shapes = [tuple(int(v) for v in s) for s in g['feat_shapes']]
    nc = int(g['num_classes'])
    gen = torch.Generator().manual_seed(data_seed)
    feats = [torch.randn(s, generator=gen) for s in feat_shapes]
    Gs = [torch.randn(B, 5 + nc, h + 2, w + 2, generator=gen) for B, _, h, w in feat_shapes]
    return keys, synthetic_state(shapes, seed=param_seed), feats, Gs, float(g['depth_mul'])
