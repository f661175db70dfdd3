"""Training-step drop-ins for the YOLOX backbone (SURVEY.md 8(f) rank 3, BASELINE.json configs[3]): forward AND backward on the H100 kernels.

Mirrors (paths relative to the reference checkout), with the same constructor arguments and state_dict keys:
  BaseConv     src/models/modules/yolox_modules.py:35-55    nn.Conv2d(bias=False) -> nn.BatchNorm2d -> SiLU, training mode (batch statistics)
  Bottleneck   src/models/modules/yolox_modules.py:79-96    1x1 -> 3x3 (+ shortcut)
  CSPLayer     src/models/modules/yolox_modules.py:99-129   conv1 | conv2 -> bottlenecks -> cat -> conv3
  Focus        src/models/modules/yolo_modules.py:19-37     2x2 space-to-depth (patches tl, bl, tr, br) -> 3x3 conv 12 -> cout
  SPPF         src/models/modules/yolo_modules.py:165-194   conv1 -> cat[x, maxpool5, maxpool9, maxpool13] (parallel pools) -> conv2
  CSPDarknet   src/models/backbones/det/csp_darknet.py:25-129   stem, four stages, SPPF in stage4
  YOLOXNeck    src/models/necks/yolox_neck.py:13-74           top-down (upsample + concat) and bottom-up (stride-2 conv + concat) CSP path
  ConvModule   src/models/modules/convs.py                     conv -> BN -> SiLU as the YOLOX head builds it (1x1 stems with padding 1)
  YOLOXHead    src/models/heads/yolox_head.py:14-88            stems, cls / reg branches, prediction convs with bias -> fp32 NCHW outputs
  YOLOXLoss    src/losses/det/yolox_loss.py:73-436             SimOTA assignment, IoU / objectness / class losses and their gradient

Channel counts of every convolution: 16, 32 or multiples of 64 (YOLOX-n, -s and -l; the 24 / 48 / 80-wide -t, -m and -x raise).  The
prediction convs (num_classes, 4 and 1 outputs) run as GEMMs zero-padded to the next such width.

What runs where: every convolution (forward, backward-data, backward-weight) is a bf16 wgmma implicit GEMM and every BatchNorm / SiLU pass
(statistics, apply, backward reductions, backward apply) is a kernel of libcvb200.so (csrc/train_kernels.cu).  torch.autograd only chains the
per-layer Functions and adds the gradients of the shortcut / concat fan-outs (tensor plumbing); the YOLOX loss is csrc/yolox_loss.cu
(YOLOXLoss below); the optimiser stays in PyTorch, as in the reference trainer (trainer.py:177-207).  Precision: bf16 activations / gradients, fp32 accumulation, fp32 master weights and fp32
weight gradients (BASELINE.json configs[3] asks for a bf16 step).  No CPU fallback: CPU tensors raise.

Inside a block activations are NHWC bf16; `CSPLayer.forward` accepts / returns the reference's NCHW tensors (layout change at the boundary).
"""
import ctypes
import math

import torch
import torch.distributed as dist
import torch.nn as nn

from . import _lib
from ._lib import _p, _stream


def _ptrs(ts):
    """ctypes void* array of the tensors' data pointers."""
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _shapes4(ts):
    """ctypes int32 array of four dims per tensor: its 4-D shape, or zeros for a tensor that is not 4-D (which the C entry points refuse)."""
    return (ctypes.c_int32 * (4 * len(ts)))(*[int(d) for t in ts for d in (tuple(t.shape) if t.dim() == 4 else (0, 0, 0, 0))])


def _floats(vs):
    """ctypes float array of the values."""
    vs = [float(v) for v in vs]
    return (ctypes.c_float * len(vs))(*vs)


def _workspace(nbytes, dev):
    """A device workspace of the size a *_workspace_bytes entry point returned (at least one byte, so it has an address)."""
    return torch.empty((max(int(nbytes), 1),), dtype=torch.uint8, device=dev)


def _check_cuda(t, what):
    if not t.is_cuda:
        raise _lib.CvbError(f'{what}: CUDA tensor required (the H100 training path has no CPU fallback)')


def kpad(c):
    """K width of a packed weight row: 16 and 32 channels are one zero-padded 64-channel chunk."""
    return -(-c // 64) * 64


def channels_ok(c):
    return c in (16, 32) or (c > 0 and c % 64 == 0)


def pack_weights(w):
    """fp32 [cout,cin,k,k] -> (bf16 [cout,k*k,kpad(cin)] forward / wgrad layout, bf16 [cin,k*k,kpad(cout)] backward-data operand)."""
    cout, cin, k, _ = w.shape
    wf = torch.empty((cout, k * k, kpad(cin)), dtype=torch.bfloat16, device=w.device)
    wb = torch.empty((cin, k * k, kpad(cout)), dtype=torch.bfloat16, device=w.device)
    _lib.check(_lib.lib().cvb_train_pack_weights(_p(w.detach().float().contiguous()), cout, cin, k, _p(wf), _p(wb), _stream()), 'cvb_train_pack_weights')
    return wf, wb


def conv(x, w_packed, cout, k, y_prev=None, stat_prev=None, stride=1, pad=None):
    """x NHWC bf16 [B,H,W,cin] -> [B,Ho,Wo,cout] (pad k//2, or `pad` at stride 1: -1, 0 or 1 with k = 1).  (y_prev, stat_prev): SiLU' epilogue
    of the producing layer (backward-data only)."""
    B, H, W, cin = x.shape
    p = k // 2 if pad is None else pad
    Ho, Wo = (H + 2 * p - k) // stride + 1, (W + 2 * p - k) // stride + 1
    out = torch.empty((B, Ho, Wo, cout), dtype=torch.bfloat16, device=x.device)
    if pad is None:
        _lib.check(_lib.lib().cvb_train_conv(_p(x), B, H, W, cin, _p(w_packed), cout, k, stride, _p(out), _p(y_prev), _p(stat_prev), _stream()), 'cvb_train_conv')
    else:
        if stride != 1:
            raise ValueError('train.conv: an explicit padding is for stride-1 convolutions')
        _lib.check(_lib.lib().cvb_train_conv_pad(_p(x), B, H, W, cin, _p(w_packed), cout, k, pad, _p(out), _p(y_prev), _p(stat_prev), _stream()),
                   'cvb_train_conv_pad')
    return out


def conv_dgrad_s2(dy, w_bwd, cin, H, W, y_prev=None, stat_prev=None):
    """Backward-data of the 3x3 / stride 2 / pad 1 convolution: dy [B,Ho,Wo,cout] -> dx [B,H,W,cin] (four parity sub-convolutions)."""
    B, Ho, Wo, cout = dy.shape
    dx = torch.empty((B, H, W, cin), dtype=torch.bfloat16, device=dy.device)
    _lib.check(_lib.lib().cvb_train_conv_dgrad_s2(_p(dy), B, Ho, Wo, cout, _p(w_bwd), cin, H, W, _p(dx), _p(y_prev), _p(stat_prev), _stream()),
               'cvb_train_conv_dgrad_s2')
    return dx


def conv_wgrad(x, dy, k, stride=1, pad=None):
    """-> fp32 [cout, cin, k, k] (the nn.Conv2d layout).  `pad`: as in conv (stride 1)."""
    B, H, W, cin = x.shape
    cout = dy.shape[3]
    dw = torch.zeros((cout, k * k, cin), dtype=torch.float32, device=x.device)
    if pad is None:
        _lib.check(_lib.lib().cvb_train_conv_wgrad(_p(x), _p(dy), B, H, W, cin, cout, k, stride, _p(dw), _stream()), 'cvb_train_conv_wgrad')
    else:
        if stride != 1:
            raise ValueError('train.conv_wgrad: an explicit padding is for stride-1 convolutions')
        _lib.check(_lib.lib().cvb_train_conv_wgrad_pad(_p(x), _p(dy), B, H, W, cin, cout, k, pad, _p(dw), _stream()), 'cvb_train_conv_wgrad_pad')
    return dw.view(cout, k, k, cin).permute(0, 3, 1, 2)


def _to_nhwc(x, what):
    """A drop-in's NCHW input -> the NHWC bf16 layout of the training layers (CUDA only)."""
    _check_cuda(x, what)
    return x.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)


def _to_nchw(x, dtype):
    """An NHWC bf16 layer output -> the reference's NCHW layout in `dtype` (a permuted view, converted only when dtype is not bf16)."""
    return x.permute(0, 3, 1, 2).to(dtype)


def _require_training(m, message):
    """The drop-ins use batch statistics only: eval() goes through the inference modules."""
    if not m.training:
        raise RuntimeError(message)


def _require_widths(widths, message):
    """NotImplementedError(message(bad widths)) unless every channel count is 16, 32 or a multiple of 64."""
    bad = sorted({c for c in widths if not channels_ok(c)})
    if bad:
        raise NotImplementedError(message(bad))


def _bn_momentum(bn):
    """Counts the step and returns the running-statistics momentum nn.BatchNorm2d would use (momentum None: cumulative average)."""
    bn.num_batches_tracked += 1
    return bn.momentum if bn.momentum is not None else 1.0 / float(bn.num_batches_tracked)


def _set_bn(m):
    """Every BatchNorm of `m` gets the reference YOLOX's eps 1e-3 and momentum 0.03."""
    for mod in m.modules():
        if isinstance(mod, nn.BatchNorm2d):
            mod.eps, mod.momentum = 1e-3, 0.03


def _sync_group(bn):
    """The process group whose ranks' pixels `bn` normalises over, or None (this device's batch only).  Decided at every forward as
    nn.SyncBatchNorm.forward decides it: an nn.SyncBatchNorm in training mode, torch.distributed initialised, and more than one rank in the
    module's process_group (None: the default group)."""
    if not (isinstance(bn, nn.SyncBatchNorm) and bn.training and dist.is_available() and dist.is_initialized()):
        return None
    group = bn.process_group if bn.process_group else dist.group.WORLD
    return group if dist.get_world_size(group) > 1 else None


def bn_stats(y, gamma, beta, running_mean, running_var, eps, momentum):
    """Batch statistics of y NHWC bf16 [..., C] -> (stat fp32 [4, C] = mean, rstd, scale, shift; fp32 gamma).  Updates the running statistics."""
    C = y.shape[-1]
    stat = torch.empty((4, C), dtype=torch.float32, device=y.device)
    scratch = torch.empty((2, C), dtype=torch.float32, device=y.device)
    g32, b32 = gamma.detach().float().contiguous(), beta.detach().float().contiguous()
    _lib.check(_lib.lib().cvb_train_bn_stats(_p(y), y.numel() // C, C, _p(g32), _p(b32), float(eps), float(momentum), _p(running_mean), _p(running_var),
                                             _p(scratch), _p(stat), _stream()), 'cvb_train_bn_stats')
    return stat, g32


def batch_stats(y, gamma, beta, running_mean, running_var, eps, momentum, group=None):
    """bn_stats over this device's pixels (group None) or, with a process group (SyncBatchNorm), over every rank's -> (stat, fp32 gamma,
    count): count is the global pixel count, fp64 [1] on the device, with a process group (None otherwise).  Updates the running statistics."""
    if group is None:
        return (*bn_stats(y, gamma, beta, running_mean, running_var, eps, momentum), None)
    L = _lib.lib()
    C = y.shape[-1]
    npix = y.numel() // C
    stat = torch.empty((4, C), dtype=torch.float32, device=y.device)
    scratch = torch.empty((2, C), dtype=torch.float32, device=y.device)
    g32, b32 = gamma.detach().float().contiguous(), beta.detach().float().contiguous()
    # every rank's (mean, M2, count) record, gathered in rank order and merged on the device
    world = dist.get_world_size(group)
    rec = torch.empty((2 * C + 1,), dtype=torch.float64, device=y.device)
    _lib.check(L.cvb_train_bn_partial(_p(y), npix, C, _p(scratch), _p(rec), _stream()), 'cvb_train_bn_partial')
    recs = torch.empty((world * (2 * C + 1),), dtype=torch.float64, device=y.device)  # (flat: gloo's all-gather wants world x the input)
    dist.all_gather_into_tensor(recs, rec, group=group)
    count = torch.empty((1,), dtype=torch.float64, device=y.device)
    _lib.check(L.cvb_train_bn_merge(_p(recs), world, C, _p(g32), _p(b32), float(eps), float(momentum), _p(running_mean), _p(running_var),
                                    _p(stat), _p(count), _stream()), 'cvb_train_bn_merge')
    return stat, g32, count


def _conv_bn_silu(x, weight, gamma, beta, running_mean, running_var, eps, momentum, group, k, stride=1, pad=None, act='silu'):
    """a = act(bn_train(conv(x, weight))) (act 'silu' or 'relu') -> (a, (y, stat, g32, wb), count): what _bn_silu_backward /
    _bn_relu_backward and the backward convolutions need (the conv output, the BN statistics, fp32 gamma and the backward-data weights)
    and, with a process group (SyncBatchNorm), the global pixel count on the device (None otherwise).  Updates the running statistics."""
    cout = weight.shape[0]
    wf, wb = pack_weights(weight)
    y = conv(x, wf, cout, k, stride=stride, pad=pad)
    stat, g32, count = batch_stats(y, gamma, beta, running_mean, running_var, eps, momentum, group)
    a = torch.empty_like(y)
    fwd = 'cvb_train_bn_relu_fwd' if act == 'relu' else 'cvb_train_bn_silu_fwd'
    _lib.check(getattr(_lib.lib(), fwd)(_p(y), y.numel() // cout, cout, _p(stat), _p(a), _stream()), fwd)
    return a, (y, stat, g32, wb), count


def _bn_silu_backward(g, g_is_dz, y, stat, g32, group=None, count=None):
    """g = d(loss)/d(a), or d(loss)/d(z) with z the BN output when g_is_dz (a SiLU' epilogue already applied) -> (dy = d(loss)/d(y),
    dgamma, dbeta).  With a process group (SyncBatchNorm): dgamma and dbeta stay this rank's sums (DDP averages them like every other
    gradient); dy takes the sums over every rank and the global pixel count `count` of the forward."""
    g = g.contiguous()
    cout = y.shape[3]
    npix = y.shape[0] * y.shape[1] * y.shape[2]
    L = _lib.lib()
    sums = torch.empty((2, cout), dtype=torch.float32, device=y.device)
    dy = torch.empty_like(y)
    if group is None:
        _lib.check(L.cvb_train_bn_silu_bwd(_p(g), int(g_is_dz), _p(y), npix, cout, _p(stat), _p(g32), _p(sums), _p(dy), _stream()), 'cvb_train_bn_silu_bwd')
        return dy, sums[1].clone(), sums[0].clone()
    _lib.check(L.cvb_train_bn_silu_bwd_reduce(_p(g), int(g_is_dz), _p(y), npix, cout, _p(stat), _p(sums), _stream()), 'cvb_train_bn_silu_bwd_reduce')
    dgamma, dbeta = sums[1].clone(), sums[0].clone()
    dist.all_reduce(sums, group=group)
    _lib.check(L.cvb_train_bn_silu_bwd_apply(_p(g), int(g_is_dz), _p(y), npix, cout, _p(stat), _p(g32), _p(sums), _p(count), _p(dy), _stream()),
               'cvb_train_bn_silu_bwd_apply')
    return dy, dgamma, dbeta


def _bn_relu_backward(g, y, stat, g32, group=None, count=None):
    """g = d(loss)/d(a), a = relu(bn(y)) -> (dy, dgamma, dbeta).  With a process group (SyncBatchNorm): as _bn_silu_backward."""
    g = g.contiguous()
    cout = y.shape[3]
    npix = y.numel() // cout
    L = _lib.lib()
    sums = torch.empty((2, cout), dtype=torch.float32, device=y.device)
    dy = torch.empty_like(y)
    if group is None:
        _lib.check(L.cvb_train_bn_relu_bwd(_p(g), _p(y), npix, cout, _p(stat), _p(g32), _p(sums), _p(dy), _stream()), 'cvb_train_bn_relu_bwd')
        return dy, sums[1].clone(), sums[0].clone()
    _lib.check(L.cvb_train_bn_relu_bwd_reduce(_p(g), _p(y), npix, cout, _p(stat), _p(sums), _stream()), 'cvb_train_bn_relu_bwd_reduce')
    dgamma, dbeta = sums[1].clone(), sums[0].clone()
    dist.all_reduce(sums, group=group)
    _lib.check(L.cvb_train_bn_relu_bwd_apply(_p(g), _p(y), npix, cout, _p(stat), _p(g32), _p(sums), _p(count), _p(dy), _stream()),
               'cvb_train_bn_relu_bwd_apply')
    return dy, dgamma, dbeta


class _ConvBnSiLU(torch.autograd.Function):
    """a = silu(bn_train(conv(x, W))) (or relu: act='relu') with the backward the reference obtains from torch.autograd, on the H100 kernels."""

    @staticmethod
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, eps, momentum, group, k, stride=1, pad=None, act='silu'):
        _check_cuda(x, 'BaseConv (H100 training)')
        a, saved, count = _conv_bn_silu(x, weight, gamma, beta, running_mean, running_var, eps, momentum, group, k, stride, pad, act)
        ctx.save_for_backward(x, *saved)
        ctx.k, ctx.stride, ctx.pad, ctx.act = k, stride, pad, act
        ctx.group, ctx.count = group, count
        ctx.need_dx = x.requires_grad
        return a

    @staticmethod
    def backward(ctx, da):
        x, y, stat, g32, wb = ctx.saved_tensors
        k = ctx.k
        B, H, W, cin = x.shape
        if ctx.act == 'relu':
            dy, dgamma, dbeta = _bn_relu_backward(da, y, stat, g32, ctx.group, ctx.count)
        else:
            dy, dgamma, dbeta = _bn_silu_backward(da, False, y, stat, g32, ctx.group, ctx.count)
        dw = conv_wgrad(x, dy, k, ctx.stride, ctx.pad)
        dx = None
        if ctx.need_dx:
            if ctx.stride == 2:
                dx = conv_dgrad_s2(dy, wb, cin, H, W)
            else:  # backward-data of a padding-p conv: the same conv over dy with the rotated weights and padding k - 1 - p
                dx = conv(dy, wb, cin, k, pad=None if ctx.pad is None else k - 1 - ctx.pad)
        return dx, dw, dgamma, dbeta, None, None, None, None, None, None, None, None, None


class _BottleneckChain(torch.autograd.Function):
    """Bottleneck body  t = BaseConv1x1(x);  u = BaseConv3x3(t)  as ONE autograd node, so that the backward-data convolution of the 3x3 applies
    the 1x1 layer's SiLU' in its epilogue (dz_t leaves the tensor core already multiplied; d(loss)/dt is never written)."""

    @staticmethod
    def forward(ctx, x, w1, g1, b1, rm1, rv1, eps1, mom1, grp1, w2, g2, b2, rm2, rv2, eps2, mom2, grp2):
        _check_cuda(x, 'Bottleneck (H100 training)')
        t, saved1, n1 = _conv_bn_silu(x, w1, g1, b1, rm1, rv1, eps1, mom1, grp1, 1)
        u, saved2, n2 = _conv_bn_silu(t, w2, g2, b2, rm2, rv2, eps2, mom2, grp2, 3)
        ctx.save_for_backward(x, t, *saved1, *saved2)
        ctx.sync = ((grp1, n1), (grp2, n2))
        ctx.need_dx = x.requires_grad
        return u

    @staticmethod
    def backward(ctx, du):
        x, t, y1, st1, g1f, wb1, y2, st2, g2f, wb2 = ctx.saved_tensors
        sync1, sync2 = ctx.sync
        dy2, dg2, db2 = _bn_silu_backward(du, False, y2, st2, g2f, *sync2)
        dw2 = conv_wgrad(t, dy2, 3)
        dz1 = conv(dy2, wb2, y1.shape[3], 3, y_prev=y1, stat_prev=st1)  # backward-data of the 3x3 with the 1x1 layer's SiLU' in the epilogue
        dy1, dg1, db1 = _bn_silu_backward(dz1, True, y1, st1, g1f, *sync1)
        dw1 = conv_wgrad(x, dy1, 1)
        dx = conv(dy1, wb1, x.shape[3], 1) if ctx.need_dx else None
        return dx, dw1, dg1, db1, None, None, None, None, None, dw2, dg2, db2, None, None, None, None, None


class _ConvBnSiLULayer(nn.Module):
    """conv (no bias) -> BatchNorm (batch statistics) -> SiLU as one _ConvBnSiLU, with the reference's conv / bn / act children.
    forward: NHWC bf16 in -> NHWC bf16 out.  `padding` None: k // 2 through cvb_train_conv (stride 1 or 2); otherwise cvb_train_conv_pad."""
    drop_in = None  # the public module named in the eval() refusal
    act = 'silu'  # the activation after the BatchNorm: 'silu', or 'relu' (yolov6_train.ConvModule)

    def __init__(self, in_channels, out_channels, ksize, stride=1, padding=None):
        super().__init__()
        self.conv = nn.Conv2d(in_channels, out_channels, ksize, stride, ksize // 2 if padding is None else padding, bias=False)
        self.bn = nn.BatchNorm2d(out_channels)
        self.act = nn.SiLU(inplace=True)  # (parameter-free; kept for module-tree parity with the reference)
        self.ksize, self.stride, self.padding = ksize, stride, padding

    def _bn_inputs(self):
        """Counts the step -> the _ConvBnSiLU / _BottleneckChain arguments of this layer's BatchNorm (an nn.BatchNorm2d, or the
        nn.SyncBatchNorm convert_sync_batchnorm put in its place: then the statistics span the ranks of its process group)."""
        bn = self.bn
        return bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps, _bn_momentum(bn), _sync_group(bn)

    def forward(self, x):
        return self._layer(x, self.conv.weight)

    def _layer(self, x, weight):
        _require_training(self, f'{type(self).__module__}.{self.drop_in} is the TRAINING drop-in (batch statistics); use the inference modules for eval()')
        return _ConvBnSiLU.apply(x, weight, *self._bn_inputs(), self.ksize, self.stride, self.padding, self.act)


class BaseConv(_ConvBnSiLULayer):
    """src/models/modules/yolox_modules.py:35-55 (act='silu', groups=1; stride 1, or stride 2 with ksize 3 = the downsampling conv in front of
    every CSPLayer of the YOLOX backbone).  forward: NHWC bf16 in -> NHWC bf16 out."""
    drop_in = 'BaseConv'

    def __init__(self, in_channels, out_channels, ksize, stride, groups=1, bias=False, act='silu'):
        if not (stride == 1 or (stride == 2 and ksize == 3)) or groups != 1 or bias or act != 'silu' or ksize not in (1, 3):
            raise NotImplementedError('H100 training BaseConv: ksize in {1,3}, stride 1 (or 2 with ksize 3), groups 1, no bias, SiLU')
        _require_widths((in_channels, out_channels),
                        lambda bad: f'H100 training BaseConv: channel counts must be 16, 32 or multiples of 64 (got {in_channels} -> {out_channels})')
        super().__init__(in_channels, out_channels, ksize, stride)

    def forward_nchw(self, x):
        """Reference interface (NCHW in / out) for a stand-alone BaseConv, e.g. the stride-2 conv of a `dark` stage."""
        return _to_nchw(self.forward(_to_nhwc(x, 'BaseConv (H100 training)')), x.dtype)


class Bottleneck(nn.Module):
    """src/models/modules/yolox_modules.py:79-96 (depthwise=False)."""

    def __init__(self, in_channels, out_channels, shortcut=True, expansion=0.5, depthwise=False, act='silu'):
        super().__init__()
        if depthwise:
            raise NotImplementedError('depthwise bottlenecks are not on the H100 training path')
        hidden_channels = int(out_channels * expansion)
        self.conv1 = BaseConv(in_channels, hidden_channels, 1, stride=1, act=act)
        self.conv2 = BaseConv(hidden_channels, out_channels, 3, stride=1, act=act)
        self.use_add = shortcut and in_channels == out_channels

    def forward(self, x):
        return _bottleneck(self, x, self.conv1, self.conv2, self.use_add)


def _bottleneck(m, x, c1, c2, use_add):
    """The body of a YOLOX Bottleneck / YOLOv5 C3 bottleneck: c2(c1(x)) as one _BottleneckChain (+ x when use_add)."""
    _require_training(m, 'training drop-in: call .train()')
    y = _BottleneckChain.apply(x, c1.conv.weight, *c1._bn_inputs(), c2.conv.weight, *c2._bn_inputs())
    if use_add:
        y = y + x
    return y


class CSPLayer(nn.Module):
    """src/models/modules/yolox_modules.py:99-129.  forward(x NCHW) -> NCHW (reference interface); `forward_nhwc` keeps the internal layout."""

    def __init__(self, in_channels, out_channels, n=1, shortcut=True, expansion=0.5, depthwise=False, act='silu'):
        super().__init__()
        hidden_channels = int(out_channels * expansion)
        self.conv1 = BaseConv(in_channels, hidden_channels, 1, stride=1, act=act)
        self.conv2 = BaseConv(in_channels, hidden_channels, 1, stride=1, act=act)
        self.conv3 = BaseConv(2 * hidden_channels, out_channels, 1, stride=1, act=act)
        self.m = nn.Sequential(*[Bottleneck(hidden_channels, hidden_channels, shortcut, 1.0, depthwise, act=act) for _ in range(n)])

    def forward_nhwc(self, x):
        x_1 = self.conv1(x)
        x_2 = self.conv2(x)
        x_1 = self.m(x_1)
        return self.conv3(torch.cat((x_1, x_2), dim=3))

    def forward(self, x):
        return _to_nchw(self.forward_nhwc(_to_nhwc(x, 'CSPLayer (H100 training)')), x.dtype)


# ------------------------------------------------------------------------------------------------ whole backbone: Focus stem, SPPF, CSPDarknet
def focus_s2d(img):
    """fp32 NCHW [B,3,H,W] (H, W even) -> bf16 NHWC [B,H/2,W/2,16]: channel 3 * patch + c in the reference's patch order (tl, bl, tr, br),
    channels 12..15 zero."""
    _check_cuda(img, 'Focus (H100 training)')
    B, C, H, W = img.shape
    if C != 3:
        raise ValueError(f'Focus: a 3-channel image expected, got {C} channels')
    img = img.detach().float().contiguous()
    out = torch.empty((B, H // 2, W // 2, 16), dtype=torch.bfloat16, device=img.device)
    _lib.check(_lib.lib().cvb_train_focus_s2d(_p(img), B, H, W, _p(out), _stream()), 'cvb_train_focus_s2d')
    return out


def spp_pool(a):
    """a NHWC bf16 [B,H,W,C] -> (cat [B,H,W,4C] = [a | maxpool5 | maxpool9 | maxpool13], idx uint8 [3,B,H,W,C]: each window's winner)."""
    B, H, W, C = a.shape
    cat = torch.empty((B, H, W, 4 * C), dtype=torch.bfloat16, device=a.device)
    idx = torch.empty((3, B, H, W, C), dtype=torch.uint8, device=a.device)
    _lib.check(_lib.lib().cvb_train_spp_pool_fwd(_p(a), B, H, W, C, _p(cat), _p(idx), _stream()), 'cvb_train_spp_pool_fwd')
    return cat, idx


def spp_pool_backward(g, idx):
    """g = d(loss)/d(cat) [B,H,W,4C], idx of spp_pool -> d(loss)/d(a) [B,H,W,C] (deterministic gather, fp32 sums)."""
    B, H, W, C4 = g.shape
    da = torch.empty((B, H, W, C4 // 4), dtype=torch.bfloat16, device=g.device)
    _lib.check(_lib.lib().cvb_train_spp_pool_bwd(_p(g), _p(idx), B, H, W, C4 // 4, _p(da), _stream()), 'cvb_train_spp_pool_bwd')
    return da


class _SppPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a):
        _check_cuda(a, 'SPPF (H100 training)')
        cat, idx = spp_pool(a.contiguous())
        ctx.save_for_backward(idx)
        return cat

    @staticmethod
    def backward(ctx, g):
        idx, = ctx.saved_tensors
        return spp_pool_backward(g.contiguous(), idx)


class _StemConv(_ConvBnSiLULayer):
    """The Focus stem's ConvModule (keys conv.weight [cout,12,3,3], bn.*): on the kernels a 16 -> cout BaseConv over cvb_train_focus_s2d's
    output, with the weight zero-padded to 16 input channels (its gradient is the first 12).  Computes no input gradient."""
    drop_in = 'Focus'

    def __init__(self, in_channels, out_channels):
        super().__init__(in_channels, out_channels, 3)

    def forward(self, s2d):
        return self._layer(s2d, nn.functional.pad(self.conv.weight, (0, 0, 0, 0, 0, s2d.shape[3] - self.conv.weight.shape[1])))


class Focus(nn.Module):
    """src/models/modules/yolo_modules.py:19-37 (3-channel image, 3x3 stride-1 conv).  forward: NCHW fp32 image -> NCHW; forward_nhwc -> NHWC bf16.
    The image gets no gradient (an input with requires_grad raises)."""

    def __init__(self, in_channels, out_channels, kernel_sizes=1, stride=1, conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True), act_cfg=dict(type='Swish')):
        super().__init__()
        if in_channels != 3 or kernel_sizes != 3 or stride != 1:
            raise NotImplementedError('H100 training Focus: the 3-channel image, 3x3 conv, stride 1 (the YOLOX stem)')
        _require_widths((out_channels,), lambda bad: f'H100 training Focus: out_channels must be 16, 32 or a multiple of 64 (got {out_channels})')
        self.conv = _StemConv(in_channels * 4, out_channels)

    def forward_nhwc(self, x):
        if x.requires_grad:
            raise NotImplementedError('H100 training Focus computes no gradient for the input image: pass an image without requires_grad')
        return self.conv(focus_s2d(x))

    def forward(self, x):
        return _to_nchw(self.forward_nhwc(x), x.dtype)


def sppf_chain(a):
    """a NHWC bf16 [B,H,W,C] -> (cat [B,H,W,4C] = [a | y1 | y2 | y3], y_i = maxpool5(y_(i-1)), idx uint8 [3,B,H,W,C]: each stage's winner in
    the 5x5 window of its own input)."""
    B, H, W, C = a.shape
    cat = torch.empty((B, H, W, 4 * C), dtype=torch.bfloat16, device=a.device)
    idx = torch.empty((3, B, H, W, C), dtype=torch.uint8, device=a.device)
    _lib.check(_lib.lib().cvb_train_sppf_chain_fwd(_p(a), B, H, W, C, _p(cat), _p(idx), _stream()), 'cvb_train_sppf_chain_fwd')
    return cat, idx


def sppf_chain_backward(g, idx):
    """g = d(loss)/d(cat) [B,H,W,4C], idx of sppf_chain -> d(loss)/d(a) [B,H,W,C]: autograd through the chain (deterministic fp32 gathers)."""
    B, H, W, C4 = g.shape
    da = torch.empty((B, H, W, C4 // 4), dtype=torch.bfloat16, device=g.device)
    scratch = torch.empty((2, B, H, W, C4 // 4), dtype=torch.float32, device=g.device)
    _lib.check(_lib.lib().cvb_train_sppf_chain_bwd(_p(g), _p(idx), B, H, W, C4 // 4, _p(scratch), _p(da), _stream()), 'cvb_train_sppf_chain_bwd')
    return da


class _SppfChain(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a):
        _check_cuda(a, 'SPPF (H100 training)')
        cat, idx = sppf_chain(a.contiguous())
        ctx.save_for_backward(idx)
        return cat

    @staticmethod
    def backward(ctx, g):
        idx, = ctx.saved_tensors
        return sppf_chain_backward(g.contiguous(), idx)


class SPPF(nn.Module):
    """src/models/modules/yolo_modules.py:165-194: conv1 (C -> C/2) -> pools -> conv2 (2C -> C), with kernel_sizes (5, 9, 13) (YOLOX: the
    parallel pools [x | mp5 | mp9 | mp13]) or 5 (YOLOv5: the chained pools [x | y1 | y2 | y3], y_i = mp5(y_(i-1)): the same values, but the
    gradient of a tie goes where autograd through the chain sends it).  One kernel writes the concatenation conv2 reads.  forward: NCHW;
    forward_nhwc: NHWC bf16."""

    def __init__(self, in_channels, out_channels, kernel_sizes=(5, 9, 13), conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True),
                 act_cfg=dict(type='Swish'), init_cfg=None):
        super().__init__()
        chained = isinstance(kernel_sizes, int) and kernel_sizes == 5
        if not chained and (isinstance(kernel_sizes, int) or tuple(kernel_sizes) != (5, 9, 13)):
            raise NotImplementedError(f'H100 training SPPF: kernel_sizes (5, 9, 13) or 5 only (got {kernel_sizes})')
        self.kernel_sizes = kernel_sizes
        hidden_channels = in_channels // 2
        self.conv1 = BaseConv(in_channels, hidden_channels, 1, stride=1)
        # (parameter-free; module-tree parity)
        self.m = (nn.MaxPool2d(kernel_size=5, stride=1, padding=2) if chained else
                  nn.ModuleList([nn.MaxPool2d(kernel_size=ks, stride=1, padding=ks // 2) for ks in kernel_sizes]))
        self.conv2 = BaseConv(hidden_channels * 4, out_channels, 1, stride=1)
        self._pool = _SppfChain if chained else _SppPool

    def forward_nhwc(self, x):
        return self.conv2(self._pool.apply(self.conv1(x)))

    def forward(self, x):
        return _to_nchw(self.forward_nhwc(_to_nhwc(x, 'SPPF (H100 training)')), x.dtype)


def _nhwc(m, x):
    return m.forward_nhwc(x) if isinstance(m, (CSPLayer, SPPF)) else m(x)


def bound_training_modules(model, inference_modules, build):
    """The training modules of a model-level drop-in (build() -> a tuple, one per inference module), kept out of the model's module tree and
    whose parameters, buffers and BatchNorm modules ARE the inference modules' (re-bound by name on every call: .to() replaces buffer tensors,
    convert_sync_batchnorm replaces the BatchNorm modules, and the layers sync their statistics when they see an nn.SyncBatchNorm).  So
    state_dict(), the optimiser's parameters and the statistics eval() folds are the same tensors.  Built on the first call and cached in
    model.__dict__['_train_modules'], which a deepcopy or pickle of the model leaves None (modules._Standalone.__getstate__) so that the copy
    binds its own tensors; a training module whose keys differ from its inference module's raises NotImplementedError."""
    if model.__dict__.get('_train_modules') is None:
        mods = build()
        binds = []
        for tm, im in zip(mods, inference_modules):
            if list(tm.state_dict()) != list(im.state_dict()):
                raise NotImplementedError(f'{type(model).__name__} (H100) training: {type(im).__name__} keys differ from the training module\'s')
            for name, sub in tm.named_modules():  # (bound by name: the key lists are equal)
                if isinstance(sub, nn.modules.batchnorm._BatchNorm):  # the module itself, with its parameters and buffers
                    parent, _, leaf = name.rpartition('.')
                    binds.append((tm.get_submodule(parent)._modules, leaf, im.get_submodule(parent)._modules))
                elif sub._parameters or sub._buffers:
                    src = im.get_submodule(name)
                    binds += [(sub._parameters, k, src._parameters) for k in sub._parameters]
                    binds += [(sub._buffers, k, src._buffers) for k in sub._buffers]
        model.__dict__['_train_modules'] = (mods, binds)
    mods, binds = model._train_modules
    for dst, k, src in binds:
        dst[k] = src[k]
    return mods


class CSPDarknet(nn.Module):
    """src/models/backbones/det/csp_darknet.py:25-129, training mode, same constructor and state_dict keys.  Every BatchNorm gets eps 1e-3 and
    momentum 0.03 (the reference's init_weights).  forward(x): NCHW fp32 image -> list of NCHW outputs of `out_stages` (one tensor if a single
    stage); forward_nhwc(x): the same outputs as NHWC bf16, for chaining into later drop-ins.  Evaluation goes through the inference
    cvpytorch_b200.yolox_models.CSPDarknet, which loads this module's state_dict with strict=True."""
    cfg = {"n": [0.33, 0.25], "t": [0.33, 0.375], "s": [0.33, 0.5], "m": [0.67, 0.75], "l": [1.0, 1.0], "x": [1.33, 1.25]}

    def __init__(self, subtype='cspdark_s', out_channels=[64, 128, 256, 512, 1024], layers=[3, 9, 9, 3], spp_ksizes=(5, 9, 13), depthwise=False,
                 conv_cfg=None, norm_cfg=dict(type='BN', momentum=0.03, eps=0.001), act_cfg=dict(type='Swish'), out_stages=[2, 3, 4], output_stride=32,
                 backbone_path=None, pretrained=False, frozen_stages=-1, norm_eval=False):
        super().__init__()
        if depthwise:
            raise NotImplementedError('H100 training CSPDarknet: depthwise convolutions are not on the training path')
        if norm_eval:
            raise NotImplementedError('H100 training CSPDarknet: norm_eval=True (frozen BatchNorm statistics) is not on the training path')
        if frozen_stages >= 0:
            raise NotImplementedError('H100 training CSPDarknet: frozen_stages >= 0 is not on the training path')
        if isinstance(spp_ksizes, int) or tuple(spp_ksizes) != (5, 9, 13):
            raise NotImplementedError(f'H100 training CSPDarknet: spp_ksizes (5, 9, 13) only (got {spp_ksizes})')
        if (norm_cfg or {}).get('type', 'BN') != 'BN' or (act_cfg or {}).get('type') not in ('Swish', 'SiLU') or conv_cfg is not None:
            raise NotImplementedError('H100 training CSPDarknet: plain Conv2d, BatchNorm and Swish / SiLU only')
        self.subtype, self.out_stages, self.output_stride = subtype, out_stages, output_stride
        self.backbone_path, self.pretrained, self.frozen_stages, self.norm_eval = backbone_path, pretrained, frozen_stages, norm_eval
        depth_mul, width_mul = self.cfg[subtype.split('_')[1]]
        ch = list(map(lambda x: int(x * width_mul), out_channels))
        nl = list(map(lambda x: max(round(x * depth_mul), 1), layers))
        self.layers = nl
        _require_widths(ch + [c // 2 for c in ch[1:]],
                        lambda bad: f'H100 training CSPDarknet {subtype}: widths {bad} are not on the training path (channels must be 16, 32 or multiples of 64)')
        self.stem = Focus(3, ch[0], kernel_sizes=3)
        self.stage1 = nn.Sequential(BaseConv(ch[0], ch[1], 3, 2), CSPLayer(ch[1], ch[1], n=nl[0], shortcut=True))
        self.stage2 = nn.Sequential(BaseConv(ch[1], ch[2], 3, 2), CSPLayer(ch[2], ch[2], n=nl[1], shortcut=True))
        self.stage3 = nn.Sequential(BaseConv(ch[2], ch[3], 3, 2), CSPLayer(ch[3], ch[3], n=nl[2], shortcut=True))
        self.stage4 = nn.Sequential(BaseConv(ch[3], ch[4], 3, 2), SPPF(ch[4], ch[4], kernel_sizes=spp_ksizes), CSPLayer(ch[4], ch[4], n=nl[3], shortcut=False))
        self.out_channels = ch[out_stages[0]:out_stages[-1] + 1]
        _set_bn(self)

    def forward_nhwc(self, x):
        _require_training(self, 'cvpytorch_b200.train.CSPDarknet is the TRAINING drop-in (batch statistics); load its state_dict into '
                                'cvpytorch_b200.yolox_models.CSPDarknet for eval()')
        _check_cuda(x, 'CSPDarknet (H100 training)')
        h = self.stem.forward_nhwc(x)
        outs = []
        for i in range(1, 5):
            for m in getattr(self, f'stage{i}'):
                h = _nhwc(m, h)
            if i in self.out_stages:
                outs.append(h)
        return outs

    def forward(self, x):
        outs = [_to_nchw(o, x.dtype) for o in self.forward_nhwc(x)]
        return outs if len(self.out_stages) > 1 else outs[0]


# ------------------------------------------------------------------------------------------------ YOLOX neck and head
def upsample_cat(a, b):
    """a NHWC bf16 [B,h,w,Ca], b [B,2h,2w,Cb] -> [B,2h,2w,Ca+Cb] = [nearest_up2(a) | b] (the neck's nn.Upsample + torch.cat, upsampled map first)."""
    B, h, w, Ca = a.shape
    Cb = b.shape[3]
    if tuple(b.shape[:3]) != (B, 2 * h, 2 * w):
        raise ValueError(f'upsample_cat: b must be [B, 2h, 2w, Cb] for a [B, h, w, Ca] (got a {tuple(a.shape)}, b {tuple(b.shape)})')
    cat = torch.empty((B, 2 * h, 2 * w, Ca + Cb), dtype=torch.bfloat16, device=a.device)
    _lib.check(_lib.lib().cvb_train_upsample_cat_fwd(_p(a), B, h, w, Ca, _p(b), Cb, _p(cat), _stream()), 'cvb_train_upsample_cat_fwd')
    return cat


def upsample_cat_backward(g, Ca):
    """g = d(loss)/d(cat) [B,2h,2w,Ca+Cb] -> (da [B,h,w,Ca] = the 2x2 sums of g[..., :Ca], db = g[..., Ca:]); deterministic, fp32 sums."""
    B, H2, W2, C = g.shape
    da = torch.empty((B, H2 // 2, W2 // 2, Ca), dtype=torch.bfloat16, device=g.device)
    db = torch.empty((B, H2, W2, C - Ca), dtype=torch.bfloat16, device=g.device)
    _lib.check(_lib.lib().cvb_train_upsample_cat_bwd(_p(g), B, H2 // 2, W2 // 2, Ca, C - Ca, _p(da), _p(db), _stream()), 'cvb_train_upsample_cat_bwd')
    return da, db


class _UpsampleCat(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        _check_cuda(a, 'YOLOXNeck (H100 training)')
        ctx.ca = a.shape[3]
        return upsample_cat(a.contiguous(), b.contiguous())

    @staticmethod
    def backward(ctx, g):
        return upsample_cat_backward(g.contiguous(), ctx.ca)


def pred_cout_pad(c):
    """GEMM width of a prediction conv with c outputs: the next training width (16, 32 or a multiple of 64)."""
    return 16 if c <= 16 else (32 if c <= 32 else kpad(c))


def pred_conv(x, w_packed, cout, bias, out, c_off):
    """1x1 prediction conv with bias: x NHWC bf16 [B,h,w,cin], w_packed = pack_weights(weight zero-padded to pred_cout_pad(cout) rows)[0]
    -> out fp32 NCHW [B,Ctot,h,w] channels [c_off, c_off + cout) = conv + bias."""
    B, h, w, cin = x.shape
    _lib.check(_lib.lib().cvb_train_pred_conv(_p(x), B, h, w, cin, _p(w_packed), cout, pred_cout_pad(cout), _p(bias), _p(out), out.shape[1], c_off, _stream()),
               'cvb_train_pred_conv')


def pred_grad(g, c_off, cout):
    """g fp32 NCHW [B,Ctot,h,w] -> (dy bf16 NHWC [B,h,w,pred_cout_pad(cout)] = channels [c_off, c_off + cout) of g, zero-padded; dbias [cout])."""
    B, Ctot, h, w = g.shape
    cp = pred_cout_pad(cout)
    dy = torch.empty((B, h, w, cp), dtype=torch.bfloat16, device=g.device)
    db = torch.empty((cout,), dtype=torch.float32, device=g.device)
    _lib.check(_lib.lib().cvb_train_pred_grad(_p(g), B, Ctot, h, w, c_off, cout, cp, _p(dy), _p(db), _stream()), 'cvb_train_pred_grad')
    return dy, db


class _HeadPred(torch.autograd.Function):
    """One level's output [B, 5 + num_classes, h, w] fp32 NCHW = cat(reg_obj_preds(reg_feat), cls_preds(cls_feat)) (heads/yolox_head.py:75-85):
    reg (4) + obj (1) are one GEMM over reg_feat at channel 0, cls a second GEMM over cls_feat at channel 5, both writing the output in place."""

    @staticmethod
    def forward(ctx, reg_feat, cls_feat, w_ro, b_ro, w_cls, b_cls):
        _check_cuda(reg_feat, 'YOLOXHead (H100 training)')
        B, h, w, _ = reg_feat.shape
        out = torch.empty((B, w_ro.shape[0] + w_cls.shape[0], h, w), dtype=torch.float32, device=reg_feat.device)
        wbs = []
        for x, wt, b, c_off in ((reg_feat, w_ro, b_ro, 0), (cls_feat, w_cls, b_cls, w_ro.shape[0])):
            cout = wt.shape[0]
            wf, wb = pack_weights(nn.functional.pad(wt.detach().float(), (0, 0, 0, 0, 0, 0, 0, pred_cout_pad(cout) - cout)))
            pred_conv(x.contiguous(), wf, cout, b.detach().float().contiguous(), out, c_off)
            wbs.append(wb)
        ctx.save_for_backward(reg_feat, cls_feat, *wbs)
        ctx.couts = (w_ro.shape[0], w_cls.shape[0])
        return out

    @staticmethod
    def backward(ctx, g):
        reg_feat, cls_feat, wb_ro, wb_cls = ctx.saved_tensors
        g = g.contiguous()
        res = []
        for x, wb, c_off, cout, need in ((reg_feat, wb_ro, 0, ctx.couts[0], ctx.needs_input_grad[0]), (cls_feat, wb_cls, ctx.couts[0], ctx.couts[1], ctx.needs_input_grad[1])):
            dy, db = pred_grad(g, c_off, cout)
            dw = conv_wgrad(x, dy, 1)[:cout]
            dx = conv(dy, wb, x.shape[3], 1) if need else None
            res.append((dx, dw, db))
        (dx_ro, dw_ro, db_ro), (dx_cls, dw_cls, db_cls) = res
        return dx_ro, dx_cls, dw_ro, db_ro, dw_cls, db_cls


class ConvModule(_ConvBnSiLULayer):
    """src/models/modules/convs.py ConvModule as heads/yolox_head.py:33-49 builds it: conv (no bias) -> BatchNorm -> SiLU, training mode.
    kernel_size 1 or 3, stride 1, padding kernel_size // 2 or 1 (the head stems are 1x1 convs with padding 1).  forward: NHWC bf16 in / out."""
    drop_in = 'ConvModule'

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, activation='SiLU'):
        if kernel_size not in (1, 3) or stride != 1 or padding not in (kernel_size // 2, 1) or activation != 'SiLU':
            raise NotImplementedError('H100 training ConvModule: kernel_size 1 or 3, stride 1, padding kernel_size // 2 or 1, SiLU')
        _require_widths((in_channels, out_channels),
                        lambda bad: f'H100 training ConvModule: channel counts must be 16, 32 or multiples of 64 (got {in_channels} -> {out_channels})')
        super().__init__(in_channels, out_channels, kernel_size, stride, padding)


class YOLOXNeck(nn.Module):
    """src/models/necks/yolox_neck.py:13-74, training mode, same constructor and state_dict keys; BatchNorm eps 1e-3, momentum 0.03.
    forward_nhwc([x2, x1, x0] NHWC bf16) -> [pan_out2, pan_out1, pan_out0] NHWC bf16; forward takes and returns NCHW.  The top-down
    upsample + concat is one kernel each way (cvb_train_upsample_cat_*); the bottom-up concats are torch.cat, as in CSPLayer.  The maps must
    halve exactly (x2 = 2 x1 = 4 x0 in height and width).  Evaluation: load the state_dict into cvpytorch_b200.yolox_models.YOLOXNeck."""

    def __init__(self, subtype='yolox_s', channels=[256, 512, 1024], depth_mul=1.0, width_mul=1.0):
        super().__init__()
        assert isinstance(channels, list)
        self.subtype, self.channels, self.num_ins = subtype, channels, len(channels)
        c = list(map(lambda x: max(round(x * width_mul), 1), channels))
        n = list(map(lambda x: max(round(x * depth_mul), 1), [3, 3, 3, 3]))
        _require_widths(c + [int(v * 0.5) for v in c],
                        lambda bad: f'H100 training YOLOXNeck: widths {bad} are not on the training path (channels must be 16, 32 or multiples of 64)')
        self.upsample = nn.Upsample(scale_factor=2, mode='nearest')  # (parameter-free; module-tree parity)
        self.lateral_conv0 = BaseConv(c[2], c[1], 1, 1)
        self.C3_p4 = CSPLayer(2 * c[1], c[1], n[0], False)
        self.reduce_conv1 = BaseConv(c[1], c[0], 1, 1)
        self.C3_p3 = CSPLayer(2 * c[0], c[0], n[1], False)
        self.bu_conv2 = BaseConv(c[0], c[0], 3, 2)
        self.C3_n3 = CSPLayer(2 * c[0], c[1], n[2], False)
        self.bu_conv1 = BaseConv(c[1], c[1], 3, 2)
        self.C3_n4 = CSPLayer(2 * c[1], c[2], n[3], False)
        _set_bn(self)

    def forward_nhwc(self, x):
        _require_training(self, 'cvpytorch_b200.train.YOLOXNeck is the TRAINING drop-in (batch statistics); load its state_dict into '
                                'cvpytorch_b200.yolox_models.YOLOXNeck for eval()')
        if len(x) != self.num_ins:
            raise ValueError(f'YOLOXNeck: {self.num_ins} feature maps expected, got {len(x)}')
        x2, x1, x0 = x
        for big, small in ((x1, x0), (x2, x1)):
            if big.shape[0] != small.shape[0] or big.shape[1] != 2 * small.shape[1] or big.shape[2] != 2 * small.shape[2]:
                raise ValueError(f'YOLOXNeck: each feature map must be exactly twice the next one in height and width (got {[tuple(t.shape) for t in x]}, NHWC)')
        fpn_out0 = self.lateral_conv0(x0)
        f_out0 = self.C3_p4.forward_nhwc(_UpsampleCat.apply(fpn_out0, x1))
        fpn_out1 = self.reduce_conv1(f_out0)
        pan_out2 = self.C3_p3.forward_nhwc(_UpsampleCat.apply(fpn_out1, x2))
        pan_out1 = self.C3_n3.forward_nhwc(torch.cat((self.bu_conv2(pan_out2), fpn_out1), dim=3))
        pan_out0 = self.C3_n4.forward_nhwc(torch.cat((self.bu_conv1(pan_out1), fpn_out0), dim=3))
        return [pan_out2, pan_out1, pan_out0]

    def forward(self, x):
        return [_to_nchw(o, x[0].dtype) for o in self.forward_nhwc([_to_nhwc(t, 'YOLOX neck / head (H100 training)') for t in x])]


class YOLOXHead(nn.Module):
    """src/models/heads/yolox_head.py:14-88, training mode, same constructor and state_dict keys (stems, cls_convs, reg_convs, cls_preds,
    reg_preds, obj_preds), the prior-probability bias of cls_preds / obj_preds, BatchNorm eps 1e-3, momentum 0.03.  forward (NCHW maps) and
    forward_nhwc (NHWC bf16 maps, e.g. YOLOXNeck.forward_nhwc's) both return the reference's list of fp32 NCHW [B, 5 + num_classes, h + 2, w + 2]
    outputs (reg, obj, cls), contiguous, for the reference YOLOXLoss.  Widths: int(256 * width_mul) and the inputs must be 16, 32 or multiples of
    64.  Evaluation: load the state_dict into cvpytorch_b200.yolox_models.YOLOXHead."""

    def __init__(self, num_classes=80, subtype='yolox_s', in_channels=[256, 512, 1024], strides=[8, 16, 32], depth_mul=1.0, width_mul=1.0):
        super().__init__()
        self.num_classes, self.subtype, self.strides, self.n_anchors = num_classes, subtype, strides, 1
        ic = list(map(lambda x: max(round(x * width_mul), 1), in_channels))
        p = int(256 * width_mul)
        _require_widths(ic + [p],
                        lambda bad: f'H100 training YOLOXHead: widths {bad} are not on the training path (channels must be 16, 32 or multiples of 64)')
        self.stems, self.cls_convs, self.reg_convs = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        self.cls_preds, self.reg_preds, self.obj_preds = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        for c in ic:
            self.stems.append(ConvModule(c, p, 1, 1, padding=1))  # padding=1 on a 1x1 conv: every head map is 2 pixels larger
            self.cls_convs.append(nn.Sequential(ConvModule(p, p, 3, 1, 1), ConvModule(p, p, 3, 1, 1)))
            self.reg_convs.append(nn.Sequential(ConvModule(p, p, 3, 1, 1), ConvModule(p, p, 3, 1, 1)))
            self.cls_preds.append(nn.Conv2d(p, self.n_anchors * num_classes, 1, 1, 0))
            self.reg_preds.append(nn.Conv2d(p, 4, 1, 1, 0))
            self.obj_preds.append(nn.Conv2d(p, self.n_anchors * 1, 1, 1, 0))
        _set_bn(self)
        prior = -math.log((1 - 1e-2) / 1e-2)  # heads/yolox_head.py:54-72
        with torch.no_grad():
            for conv in list(self.cls_preds) + list(self.obj_preds):
                conv.bias.fill_(prior)

    def forward_nhwc(self, x):
        _require_training(self, 'cvpytorch_b200.train.YOLOXHead is the TRAINING drop-in (batch statistics); load its state_dict into '
                                'cvpytorch_b200.yolox_models.YOLOXHead for eval()')
        outputs = []
        for k, xx in enumerate(x):
            xx = self.stems[k](xx)  # (the stem's output fans out to both branches: autograd adds the two gradients)
            cls_feat = self.cls_convs[k](xx)
            reg_feat = self.reg_convs[k](xx)
            w_ro = torch.cat((self.reg_preds[k].weight, self.obj_preds[k].weight), 0)
            b_ro = torch.cat((self.reg_preds[k].bias, self.obj_preds[k].bias), 0)
            outputs.append(_HeadPred.apply(reg_feat, cls_feat, w_ro, b_ro, self.cls_preds[k].weight, self.cls_preds[k].bias))
        return outputs

    def forward(self, x):
        return self.forward_nhwc([_to_nhwc(t, 'YOLOX neck / head (H100 training)') for t in x])


# ------------------------------------------------------------------------------------------------ YOLOX loss (SimOTA assignment + the three terms)
def yolox_loss_forward(preds, targets, strides, num_classes):
    """preds: the head's fp32 NCHW outputs [B, 5 + num_classes, h, w] (CUDA, contiguous); targets fp32 [B, max_gt, 5] (class, cx, cy, w, h).
    -> (out fp32 [6] = loss, iou_loss, conf_loss, cls_loss, num_fg ratio, num_fg; matched_gt int32 [B, A], -1 = background; matched_iou [B, A])."""
    if len(preds) != len(strides):
        raise ValueError(f'YOLOXLoss: {len(strides)} strides for {len(preds)} outputs')
    B = preds[0].shape[0]
    A = sum(p.shape[2] * p.shape[3] for p in preds)
    dev = preds[0].device
    ws = _workspace(_lib.lib().cvb_train_yolox_loss_workspace_bytes(B, A), dev)
    out = torch.empty((6,), dtype=torch.float32, device=dev)
    matched_gt = torch.empty((B, A), dtype=torch.int32, device=dev)
    matched_iou = torch.empty((B, A), dtype=torch.float32, device=dev)
    _lib.check(_lib.lib().cvb_train_yolox_loss_fwd(_ptrs(preds), _shapes4(preds), _floats(strides), len(preds), num_classes, _p(targets), B, targets.shape[1], _p(matched_gt),
                                                   _p(matched_iou), _p(out), _p(ws), ws.numel(), _stream()), 'cvb_train_yolox_loss_fwd')
    return out, matched_gt, matched_iou


def yolox_loss_backward(preds, targets, strides, num_classes, matched_gt, matched_iou, out, grad_out):
    """d(sum_i grad_out[i] * out[i], i < 4) / d(preds) under the forward's assignment -> fp32 NCHW gradients shaped like preds."""
    grads = [torch.empty_like(p) for p in preds]
    _lib.check(_lib.lib().cvb_train_yolox_loss_bwd(_ptrs(preds), _shapes4(preds), _floats(strides), len(preds), num_classes, _p(targets), preds[0].shape[0],
                                                   targets.shape[1], _p(matched_gt), _p(matched_iou), _p(out), _p(grad_out), _ptrs(grads), _stream()),
               'cvb_train_yolox_loss_bwd')
    return grads


class _YOLOXLossFn(torch.autograd.Function):
    """out [6] = (loss, iou_loss, conf_loss, cls_loss, num_fg ratio, num_fg) of the head outputs; the assignment is kept for the backward
    (two [B, A] tensors), the gradient is recomputed from it and scaled by the incoming gradients of the four loss entries."""

    @staticmethod
    def forward(ctx, targets, strides, num_classes, *preds):
        out, matched_gt, matched_iou = yolox_loss_forward(preds, targets, strides, num_classes)
        ctx.save_for_backward(targets, matched_gt, matched_iou, out, *preds)
        ctx.strides, ctx.num_classes = strides, num_classes
        return out

    @staticmethod
    def backward(ctx, g):
        targets, matched_gt, matched_iou, out, *preds = ctx.saved_tensors
        grads = yolox_loss_backward(preds, targets, ctx.strides, ctx.num_classes, matched_gt, matched_iou, out, g.float().contiguous())
        return (None, None, None, *grads)


def _loss_targets(targets, B, device):
    """The reference's targets [B, max_gt, 5] as the contiguous fp32 CUDA tensor of the kernels (an empty GT list becomes one zero row)."""
    if not isinstance(targets, torch.Tensor) or targets.dim() != 3 or targets.shape[0] != B or targets.shape[2] != 5:
        raise ValueError(f'YOLOXLoss: targets must be a [B={B}, max_gt, 5] tensor of (class, cx, cy, w, h) rows')
    _check_cuda(targets, 'YOLOXLoss targets')
    t = targets.detach().to(device=device, dtype=torch.float32)
    if t.shape[1] == 0:
        t = torch.zeros((B, 1, 5), dtype=torch.float32, device=device)
    return t.contiguous()


class YOLOXLoss(nn.Module):
    """src/losses/det/yolox_loss.py:73-282 on the H100 kernels (csrc/yolox_loss.cu): same constructor, no parameters or buffers.
    forward(preds, targets) takes the head's list of fp32 NCHW outputs [B, 5 + num_classes, h, w] (CUDA) and targets [B, max_gt, 5] (class, cx,
    cy, w, h in pixels; at most 1024 rows) and returns the reference's dict {loss, conf_loss, cls_loss, iou_loss, num_fg} of device scalars,
    with no host sync: the whole loss can be captured in a CUDA graph.  The L1 (use_l1) and re-ID (reid_dim > 0) branches raise
    NotImplementedError."""

    def __init__(self, num_classes, reid_dim=0, id_nums=None, strides=[8, 16, 32], in_channels=[256, 512, 1024]):
        super().__init__()
        if reid_dim > 0:
            raise NotImplementedError('H100 YOLOXLoss: the re-ID branch (reid_dim > 0) is not implemented')
        self.n_anchors = 1
        self.num_classes = num_classes
        self.strides = strides
        self.reid_dim = reid_dim
        self.use_l1 = False
        self.in_channels = in_channels

    def forward(self, preds, targets, imgs=None):
        if self.use_l1:
            raise NotImplementedError('H100 YOLOXLoss: the L1 branch (use_l1 = True) is not implemented')
        if len(preds) != len(self.strides):
            raise ValueError(f'YOLOXLoss: {len(self.strides)} strides for {len(preds)} outputs')
        for p in preds:
            _check_cuda(p, 'YOLOXLoss')
        preds = [p.float().contiguous() for p in preds]
        out = _YOLOXLossFn.apply(_loss_targets(targets, preds[0].shape[0], preds[0].device), tuple(self.strides), self.num_classes, *preds)
        return {'loss': out[0], 'conf_loss': out[2], 'cls_loss': out[3], 'iou_loss': out[1], 'num_fg': out[4].detach()}
