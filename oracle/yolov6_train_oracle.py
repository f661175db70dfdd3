"""Functional restatement of the YOLOv6-n / -s training network (src/models/backbones/det/yolov6_efficient_rep.py, necks/det/yolov6_repbipan.py,
heads/det/yolov6_effidehead.py in training mode, with the blocks of src/models/modules/yolo_modules.py) in torch, over a state_dict with the
model's keys (backbone.*, neck.*, head.*): RepVGG blocks with three BatchNorms on batch statistics, conv -> BN -> ReLU / SiLU, BiFusion's
ConvTranspose2d and SimCSPSPPF's chained pools.  fp32 NCHW; torch.autograd gives the reference gradient.  The running statistics in the
state_dict are updated in place, as nn.BatchNorm2d does (momentum 0.03, eps 1e-3: the reference's init_weights).
"""
import torch
import torch.nn.functional as F

EPS, MOMENTUM = 1e-3, 0.03


def _bn(x, sd, pre):
    return F.batch_norm(x, sd[pre + 'running_mean'], sd[pre + 'running_var'], sd[pre + 'weight'], sd[pre + 'bias'], True, MOMENTUM, EPS)


def conv_bn(x, sd, pre, stride=1, act='relu'):
    """ConvModule: conv (no bias, padding k // 2) -> BatchNorm -> act ('relu', 'silu' or None)."""
    w = sd[pre + 'conv.weight']
    y = _bn(F.conv2d(x, w, None, stride, w.shape[2] // 2), sd, pre + 'bn.')
    return F.relu(y) if act == 'relu' else (F.silu(y) if act == 'silu' else y)


def repvgg(x, sd, pre, stride=1):
    """relu(bn(conv3x3(x)) + bn(conv1x1(x)) [+ bn(x)]) (yolo_modules.py:317-327)."""
    z = conv_bn(x, sd, pre + 'rbr_dense.', stride, None) + conv_bn(x, sd, pre + 'rbr_1x1.', stride, None)
    if pre + 'rbr_identity.weight' in sd:
        z = z + _bn(x, sd, pre + 'rbr_identity.')
    return F.relu(z)


def rep_block(x, sd, pre):
    x = repvgg(x, sd, pre + 'conv1.')
    i = 0
    while f'{pre}block.{i}.rbr_dense.conv.weight' in sd:
        x = repvgg(x, sd, f'{pre}block.{i}.')
        i += 1
    return x


def sim_csp_sppf(x, sd, pre):
    x1 = conv_bn(conv_bn(conv_bn(x, sd, pre + 'cv1.'), sd, pre + 'cv3.'), sd, pre + 'cv4.')
    y0 = conv_bn(x, sd, pre + 'cv2.')
    y1 = F.max_pool2d(x1, 5, 1, 2)
    y2 = F.max_pool2d(y1, 5, 1, 2)
    y3 = conv_bn(conv_bn(torch.cat([x1, y1, y2, F.max_pool2d(y2, 5, 1, 2)], 1), sd, pre + 'cv5.'), sd, pre + 'cv6.')
    return conv_bn(torch.cat((y0, y3), 1), sd, pre + 'cv7.')


def bifusion(x0, x1, x2, sd, pre):
    u = F.conv_transpose2d(x0, sd[pre + 'upsample.weight'], sd[pre + 'upsample.bias'], stride=2)
    d = conv_bn(conv_bn(x2, sd, pre + 'cv2.'), sd, pre + 'downsample.', 2)
    return conv_bn(torch.cat((u, conv_bn(x1, sd, pre + 'cv1.'), d), 1), sd, pre + 'cv3.')


def backbone(img, sd, out_stages=(1, 2, 3, 4)):
    h = repvgg(img, sd, 'backbone.stem.', 2)
    outs = []
    for i in range(1, 5):
        h = rep_block(repvgg(h, sd, f'backbone.stage{i}.0.', 2), sd, f'backbone.stage{i}.1.')
        if i == 4:
            h = sim_csp_sppf(h, sd, 'backbone.stage4.2.')
        if i in out_stages:
            outs.append(h)
    return outs


def neck(feats, sd):
    x3, x2, x1, x0 = feats
    fpn_out0 = conv_bn(x0, sd, 'neck.reduce_layer0.')
    f_out0 = rep_block(bifusion(fpn_out0, x1, x2, sd, 'neck.bifusion0.'), sd, 'neck.Rep_p4.')
    fpn_out1 = conv_bn(f_out0, sd, 'neck.reduce_layer1.')
    pan_out2 = rep_block(bifusion(fpn_out1, x2, x3, sd, 'neck.bifusion1.'), sd, 'neck.Rep_p3.')
    pan_out1 = rep_block(torch.cat([conv_bn(pan_out2, sd, 'neck.downsample2.', 2), fpn_out1], 1), sd, 'neck.Rep_n3.')
    pan_out0 = rep_block(torch.cat([conv_bn(pan_out1, sd, 'neck.downsample1.', 2), fpn_out0], 1), sd, 'neck.Rep_n4.')
    return [pan_out2, pan_out1, pan_out0]


def head(feats, sd):
    """-> (stem outputs, pred_scores = sigmoid(cls) [B, A, nc], pred_distri [B, A, 4]) (yolov6_effidehead.py:126-147)."""
    xs, scores, distri = [], [], []
    for i, f in enumerate(feats):
        t = conv_bn(f, sd, f'head.stems.{i}.', act='silu')
        xs.append(t)
        c = F.conv2d(conv_bn(t, sd, f'head.cls_convs.{i}.', act='silu'), sd[f'head.cls_preds.{i}.weight'], sd[f'head.cls_preds.{i}.bias'])
        r = F.conv2d(conv_bn(t, sd, f'head.reg_convs.{i}.', act='silu'), sd[f'head.reg_preds.{i}.weight'], sd[f'head.reg_preds.{i}.bias'])
        scores.append(torch.sigmoid(c).flatten(2).permute(0, 2, 1))
        distri.append(r.flatten(2).permute(0, 2, 1))
    return xs, torch.cat(scores, 1), torch.cat(distri, 1)


def network(img, sd):
    """img fp32 NCHW -> the head's training output (stem outputs, pred_scores, pred_distri)."""
    return head(neck(backbone(img, sd), sd), sd)


# ------------------------------------------------------------------------------------------------ the network fixture (tests/golden/yolov6_train.npz)
# A narrowed YOLOv6-n (widths 16 and 32) that keeps every layer type: the stem, stride-2 RepVGG blocks, identity RepVGG blocks, RepBlocks of
# one and of two blocks (backbone stage 1, neck Rep_p3), SimCSPSPPF, BiFusions with c = 32 (the zero-padded 96-channel concat), stride-1 and
# stride-2 ReLU ConvModules and the SiLU head (16 and 32 wide); 3 classes, a 2x3x64x96 image.
NET = dict(backbone=dict(subtype='yolov6_n', out_channels=[64, 128, 128, 128, 128], num_blocks=[6, 3, 3, 3], out_stages=[1, 2, 3, 4]),
           neck=dict(subtype='yolov6_n', in_channels=[128, 128, 128, 128], mid_channels=[128, 128, 128], out_channels=[64, 128, 64],
                     num_blocks=[3, 3, 6, 3]),
           head=dict(subtype='yolov6_n', num_classes=3, in_channels=[64, 128, 64], use_dfl=False, fuse_ab=False), image=(2, 3, 64, 96))


def synthetic_state(keys_shapes, seed=0):
    """Seeded parameters for a YOLOv6 (key, shape) list, drawn in list order from one generator: BatchNorm gamma in [0.5, 1.5), beta ~
    N(0, 0.3^2), running statistics (0, 1); conv / transposed-conv / prediction weights ~ N(0, 1.4^2 / fan_in); other biases ~ N(0, 0.5^2);
    head.proj (reg_max + 1 entries) its linspace."""
    g = torch.Generator().manual_seed(seed)
    bns = {k[:-len('running_mean')] for k, _ in keys_shapes if k.endswith('running_mean')}
    sd = {}
    for k, shape in keys_shapes:
        pre, _, leaf = k.rpartition('.')
        pre += '.'
        if pre in bns:
            sd[k] = {'weight': lambda: torch.rand(shape, generator=g) + 0.5, 'bias': lambda: torch.randn(shape, generator=g) * 0.3,
                     'running_mean': lambda: torch.zeros(shape), 'running_var': lambda: torch.ones(shape),
                     'num_batches_tracked': lambda: torch.zeros((), dtype=torch.long)}[leaf]()
        elif k == 'head.proj':
            sd[k] = torch.linspace(0, shape[0] - 1, shape[0])
        elif leaf == 'weight' and len(shape) == 4:
            fan = shape[1] * shape[2] * shape[3]
            sd[k] = torch.randn(shape, generator=g) * (1.4 / fan ** 0.5)
        elif leaf == 'bias':
            sd[k] = torch.randn(shape, generator=g) * 0.5
        else:
            raise KeyError(k)
    return sd


def net_fixture_inputs(f):
    """The parameters, image and output gradients of tests/golden/yolov6_train.npz regenerated from its seeds as
    tools/make_golden_yolov6_train.py drew them -> (keys, state_dict, image, [G_scores, G_distri])."""
    import ast
    keys = [str(k) for k in f['keys']]
    shapes = [(k, tuple(ast.literal_eval(str(s)))) for k, s in zip(keys, f['shapes'])]
    param_seed, data_seed = (int(v) for v in f['seeds'])
    g = torch.Generator().manual_seed(data_seed)
    x = torch.rand(NET['image'], generator=g)
    Gs = [torch.randn(tuple(int(d) for d in f[k].shape), generator=g) for k in ('scores', 'distri')]
    return keys, synthetic_state(shapes, seed=param_seed), x, Gs


def net_train_step(x, Gs, sd_np):
    """One forward + backward of `network` with loss = sum(pred_scores * G_0) + sum(pred_distri * G_1) -> ({scores, distri, grad_<param>,
    after_<running stat>}: tensors)."""
    sd = {k: torch.as_tensor(v).clone().requires_grad_(torch.as_tensor(v).dtype.is_floating_point and 'running_' not in k and 'proj' not in k)
          for k, v in sd_np.items()}
    _, s, d = network(x, sd)
    ((s.float() * Gs[0]).sum() + (d.float() * Gs[1]).sum()).backward()
    res = {'scores': s.detach().float(), 'distri': d.detach().float()}
    res.update({f'grad_{k}': v.grad for k, v in sd.items() if v.requires_grad})
    res.update({f'after_{k}': v for k, v in sd.items() if 'running_' in k})
    return res


def fixture_scale(key, ref):
    """The scale an entry of the network fixture is compared on: its own max magnitude, except for BiFusion's transposed-conv bias.  That
    bias reaches the loss only through cv3 (a 1x1 conv) and cv3's batch-statistics BatchNorm, which removes any per-channel constant, so its
    exact gradient is zero and the stored values are rounding noise: they are compared on the scale of the same layer's weight gradient.
    ref: the fixture's {key: array}."""
    if key.endswith('upsample.bias'):
        key = key[:-len('bias')] + 'weight'
    return float(abs(torch.as_tensor(ref[key])).max()) + 1e-12
