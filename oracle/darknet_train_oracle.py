"""ORACLE (test infrastructure only -- never imported by the product path).

CPU restatement of the reference's YOLOX backbone IN TRAINING MODE, forward and backward, on top of the C3 block of c3_train_oracle.py:
  Focus        src/models/modules/yolo_modules.py:19-37           cat(tl, bl, tr, br patches) -> ConvModule 3x3
  SPPF         src/models/modules/yolo_modules.py:165-194         conv1 -> cat[x, maxpool5(x), maxpool9(x), maxpool13(x)] (parallel) -> conv2
  CSPDarknet   src/models/backbones/det/csp_darknet.py:25-129     stem, stage1..3 = (3x3 / 2 conv, CSPLayer), stage4 = (3x3 / 2 conv, SPPF,
                                                                  CSPLayer shortcut=False)
written functionally over a state_dict with the reference's key names.  The activation is Swish, x * sigmoid(x), as the reference's
ConvModule computes it.  The backward is torch.autograd's.  Pinned against the reference's own modules by tools/make_golden_darknet_train.py
-> tests/golden/darknet_train.npz (forward outputs, every parameter gradient and the running statistics, <= 1e-5)."""
import torch
import torch.nn.functional as F

from oracle.c3_train_oracle import BN_EPS, BN_MOMENTUM

CFG = {"n": [0.33, 0.25], "t": [0.33, 0.375], "s": [0.33, 0.5], "m": [0.67, 0.75], "l": [1.0, 1.0], "x": [1.33, 1.25]}


def conv_module(x, sd, prefix, ksize, stride=1):
    y = F.conv2d(x, sd[prefix + '.conv.weight'], None, stride, (ksize - 1) // 2)
    y = F.batch_norm(y, sd[prefix + '.bn.running_mean'], sd[prefix + '.bn.running_var'], sd[prefix + '.bn.weight'], sd[prefix + '.bn.bias'], True,
                     BN_MOMENTUM, BN_EPS)
    return y * torch.sigmoid(y)


def csp_layer(x, sd, prefix, n, shortcut):
    x1 = conv_module(x, sd, prefix + '.conv1', 1)
    x2 = conv_module(x, sd, prefix + '.conv2', 1)
    for i in range(n):
        y = conv_module(conv_module(x1, sd, f'{prefix}.m.{i}.conv1', 1), sd, f'{prefix}.m.{i}.conv2', 3)
        x1 = y + x1 if shortcut else y
    return conv_module(torch.cat((x1, x2), 1), sd, prefix + '.conv3', 1)


def focus(x, sd, prefix):
    tl, tr, bl, br = x[..., ::2, ::2], x[..., ::2, 1::2], x[..., 1::2, ::2], x[..., 1::2, 1::2]
    return conv_module(torch.cat((tl, bl, tr, br), 1), sd, prefix + '.conv', 3)


def sppf(x, sd, prefix, ksizes=(5, 9, 13)):
    x = conv_module(x, sd, prefix + '.conv1', 1)
    x = torch.cat([x] + [F.max_pool2d(x, k, 1, k // 2) for k in ksizes], 1)
    return conv_module(x, sd, prefix + '.conv2', 1)


def depths(subtype, layers=(3, 9, 9, 3)):
    return [max(round(n * CFG[subtype.split('_')[1]][0]), 1) for n in layers]


def widths(subtype, out_channels=(64, 128, 256, 512, 1024)):
    return [int(c * CFG[subtype.split('_')[1]][1]) for c in out_channels]


def csp_darknet(x, sd, subtype='cspdark_s', out_channels=(64, 128, 256, 512, 1024), layers=(3, 9, 9, 3), out_stages=(2, 3, 4), prefix=''):
    """-> list of the `out_stages` outputs (NCHW)."""
    p = prefix + '.' if prefix else ''
    nl = depths(subtype, layers)
    h = focus(x, sd, p + 'stem')
    outs = []
    for i in range(1, 5):
        s = f'{p}stage{i}'
        h = conv_module(h, sd, s + '.0', 3, 2)
        if i < 4:
            h = csp_layer(h, sd, s + '.1', nl[i - 1], True)
        else:
            h = csp_layer(sppf(h, sd, s + '.1'), sd, s + '.2', nl[3], False)
        if i in out_stages:
            outs.append(h)
    return outs


def train_step(x, Gs, sd_np, **kw):
    """One forward + backward with loss = sum_i sum(out_i * G_i).  sd_np: name -> numpy array or tensor.  Returns (outs, {param: grad},
    {running stat: value after the step})."""
    sd = {}
    for k, v in sd_np.items():
        t = torch.as_tensor(v).clone()
        if t.dtype.is_floating_point and 'running_' not in k:
            t.requires_grad_(True)
        sd[k] = t
    outs = csp_darknet(x, sd, **kw)
    sum((o * G).sum() for o, G in zip(outs, Gs)).backward()
    grads = {k: v.grad for k, v in sd.items() if v.requires_grad}
    stats = {k: v for k, v in sd.items() if 'running_' in k}
    return [o.detach() for o in outs], grads, stats


def synthetic_state(keys_shapes, seed=0):
    """Seeded parameters for the given (key, shape) list (a backbone's state_dict): conv weights ~ N(0, 1.4^2 / fan_in), BN gamma in
    [0.5, 1.5), beta ~ N(0, 0.3^2), running statistics (0, 1) -- the distribution of tools/make_golden_train.py:randomize."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shape in keys_shapes:
        if k.endswith('conv.weight'):
            fan = 1
            for d in shape[1:]:
                fan *= d
            sd[k] = torch.randn(shape, generator=g) * (1.4 / fan ** 0.5)
        elif k.endswith('bn.weight'):
            sd[k] = torch.rand(shape, generator=g) + 0.5
        elif k.endswith('bn.bias'):
            sd[k] = torch.randn(shape, generator=g) * 0.3
        elif k.endswith('running_mean'):
            sd[k] = torch.zeros(shape)
        elif k.endswith('running_var'):
            sd[k] = torch.ones(shape)
        elif k.endswith('num_batches_tracked'):
            sd[k] = torch.zeros((), dtype=torch.long)
        else:
            raise KeyError(k)
    return sd


def output_shapes(B, H, W, subtype='cspdark_s', out_channels=(64, 128, 256, 512, 1024), out_stages=(2, 3, 4)):
    """[B, C, h, w] of the `out_stages` outputs on a B x 3 x H x W image (H, W even; each stage halves the map, rounding up)."""
    ch = widths(subtype, out_channels)
    h, w, shapes = H // 2, W // 2, []
    for i in range(1, 5):
        h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        if i in out_stages:
            shapes.append((B, ch[i], h, w))
    return shapes


def fixture_inputs(g, subtype='cspdark_n'):
    """The parameters, image and output gradients of tests/golden/darknet_train.npz, regenerated from its seeds exactly as
    tools/make_golden_darknet_train.py drew them -> (keys, state_dict, x, [G_0, G_1, G_2], out_channels)."""
    import ast
    keys = [str(k) for k in g['keys']]
    shapes = [(k, tuple(ast.literal_eval(str(s)))) for k, s in zip(keys, g['shapes'])]
    param_seed, data_seed = (int(v) for v in g['seeds'])
    B, H, W = (int(v) for v in g['cfg'])
    oc = [int(c) for c in g['out_channels']]
    gen = torch.Generator().manual_seed(data_seed)
    x = torch.randn(B, 3, H, W, generator=gen)
    Gs = [torch.randn(s, generator=gen) for s in output_shapes(B, H, W, subtype, oc)]
    return keys, synthetic_state(shapes, seed=param_seed), x, Gs, oc
