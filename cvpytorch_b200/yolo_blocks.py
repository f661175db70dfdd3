"""Drop-in mirrors of the YOLOv6 / YOLOv7 building blocks that share the conv kernel family of the hot path (SURVEY.md 8 f-4).

Mirrors (paths relative to the reference checkout, same constructor arguments, same sub-module / parameter names => same ``state_dict`` keys):
  RepVGGBlock   src/models/modules/yolo_modules.py:268-386   3x3+BN, 1x1+BN and identity-BN branches summed, then ReLU
  BottleRep     :474-492                                      two RepVGG blocks + alpha * x shortcut
  RepBlock      :453-471                                      chain of RepVGG blocks / BottleReps
  Conv_C3       :412-424,  BepC3 :427-449                     CSP-style block around a RepBlock
  EELAN         :565-583                                      YOLOv7 E-ELAN: 1x1 || 1x1, two 2x(3x3) stages, concat(4) -> 1x1

H100 formulation: a RepVGG block is ALWAYS one wgmma 3x3 conv -- its three branches are folded on the host in float64 exactly like the
reference's ``switch_to_deploy`` / ``get_equivalent_kernel_bias`` (:333-385: BN-folded 3x3 + zero-padded BN-folded 1x1 + BN-folded
identity kernel), whether the module holds the training-form branches or the deployed ``rbr_reparam`` conv.  Every ``torch.cat`` is buffer
aliasing (producers write channel slices of the consumer's input); parallel 1x1 convs of the same input run as one GEMM.
Blocks are emitted into a parent graph (``emit``) or run stand-alone for tests (``forward``: NCHW fp32 in / out, inference only).
"""
import torch
import torch.nn as nn

from . import ops
from .modules import ConvModule, _Standalone, folded


class _Block(_Standalone):
    """stand-alone execution of a block as its own small graph (tests, brick-level use)"""

    def forward(self, x):
        return ops.split_to_nchw(self._run([x], lambda g, ins: self.emit(g, ins[0])).view())


def _fold_bn_identity(bn, channels):
    """the identity branch of RepVGG as a 3x3 kernel (yolo_modules.py:355-371): delta kernel scaled by gamma / std, bias beta - mean*gamma/std"""
    std = (bn.running_var.detach().double().cpu() + bn.eps).sqrt()
    t = bn.weight.detach().double().cpu() / std
    k = torch.zeros((channels, channels, 3, 3), dtype=torch.float64)
    k[torch.arange(channels), torch.arange(channels), 1, 1] = t
    return k, bn.bias.detach().double().cpu() - bn.running_mean.detach().double().cpu() * t


class RepVGGBlock(_Block):
    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, padding=1, dilation=1, groups=1, padding_mode='zeros', deploy=False,
                 use_se=False):
        super().__init__()
        if kernel_size != 3 or padding != 1 or dilation != 1 or groups != 1 or padding_mode != 'zeros' or use_se:
            raise NotImplementedError('RepVGGBlock variant not on the H100 hot path (3x3 / pad 1 / groups 1 only, like the reference asserts)')
        self.deploy, self.in_channels, self.out_channels, self.stride = deploy, in_channels, out_channels, stride
        norm_cfg = dict(type='BN', requires_grad=True)
        self.nonlinearity = nn.ReLU()
        self.se = nn.Identity()
        if deploy:
            self.rbr_reparam = nn.Conv2d(in_channels, out_channels, 3, stride, 1, bias=True)
        else:
            self.rbr_identity = nn.BatchNorm2d(in_channels) if out_channels == in_channels and stride == 1 else None
            self.rbr_dense = ConvModule(in_channels, out_channels, 3, stride, 1, norm_cfg=norm_cfg, act_cfg=None)
            self.rbr_1x1 = ConvModule(in_channels, out_channels, 1, stride, 0, norm_cfg=norm_cfg, act_cfg=None)

    def equivalent_kernel_bias(self):
        """float64 (kernel [O,I,3,3], bias [O]) of the block: get_equivalent_kernel_bias (:333-337) / the deployed conv as is"""
        if hasattr(self, 'rbr_reparam'):
            return self.rbr_reparam.weight.detach().double().cpu(), self.rbr_reparam.bias.detach().double().cpu()
        k3, b3 = folded(self.rbr_dense.conv, self.rbr_dense.bn)
        k1, b1 = folded(self.rbr_1x1.conv, self.rbr_1x1.bn)
        k = k3 + torch.nn.functional.pad(k1, [1, 1, 1, 1])
        b = b3 + b1
        if self.rbr_identity is not None:
            ki, bi = _fold_bn_identity(self.rbr_identity, self.in_channels)
            k, b = k + ki, b + bi
        return k, b

    def switch_to_deploy(self):
        """same state transition as the reference (:373-386): afterwards the module holds only ``rbr_reparam``"""
        if hasattr(self, 'rbr_reparam'):
            return
        k, b = self.equivalent_kernel_bias()
        dev = self.rbr_dense.conv.weight.device
        self.rbr_reparam = nn.Conv2d(self.in_channels, self.out_channels, 3, self.stride, 1, bias=True).to(dev)
        self.rbr_reparam.weight.data = k.float().to(dev)
        self.rbr_reparam.bias.data = b.float().to(dev)
        for name in ('rbr_dense', 'rbr_1x1', 'rbr_identity'):
            if hasattr(self, name):
                delattr(self, name)
        self.deploy = True
        self._drop_graphs()  # the next call runs the deployed conv's weights

    def emit(self, g, x, name='', **kw):
        k, b = self.equivalent_kernel_bias()
        return g.conv(x, k, b, 3, self.stride, 1, 'relu', name=name, **kw)


class BottleRep(_Block):
    def __init__(self, in_channels, out_channels, basic_block=RepVGGBlock, weight=False):
        super().__init__()
        self.conv1 = basic_block(in_channels, out_channels)
        self.conv2 = basic_block(out_channels, out_channels)
        self.shortcut = in_channels == out_channels
        self.alpha = nn.Parameter(torch.ones(1)) if weight else 1.0

    def emit(self, g, x, name='', out=None):
        t = self.conv1.emit(g, x, name + '.conv1')
        if not self.shortcut:
            return self.conv2.emit(g, t, name + '.conv2', out=out)
        alpha = float(self.alpha.detach()) if isinstance(self.alpha, torch.Tensor) else float(self.alpha)
        # outputs + alpha * x (:491): the shortcut rides in the second conv's epilogue (act(conv + bias) + alpha * residual)
        return self.conv2.emit(g, t, name + '.conv2', out=out, residual=x, residual_scale=alpha)


class RepBlock(_Block):
    def __init__(self, in_channels, out_channels, n=1, e=None, block=RepVGGBlock, basic_block=RepVGGBlock):
        super().__init__()
        self.conv1 = block(in_channels, out_channels)
        self.block = nn.Sequential(*(block(out_channels, out_channels) for _ in range(n - 1))) if n > 1 else None
        if block == BottleRep:
            self.conv1 = BottleRep(in_channels, out_channels, basic_block=basic_block, weight=True)
            n = n // 2
            self.block = nn.Sequential(*(BottleRep(out_channels, out_channels, basic_block=basic_block, weight=True) for _ in range(n - 1))) if n > 1 else None

    def emit(self, g, x, name='', out=None):
        blocks = [self.conv1] + (list(self.block) if self.block is not None else [])
        for i, b in enumerate(blocks):
            x = b.emit(g, x, f'{name}.{i}', **({'out': out} if (i == len(blocks) - 1 and out is not None) else {}))
        return x


class Conv_C3(_Block):
    """conv + BN + ReLU (or the given activation module) of the BepC3 block (:412-424)"""

    def __init__(self, c1, c2, k=1, s=1, p=None, g=1, act=True):
        super().__init__()
        if g != 1:
            raise NotImplementedError('grouped Conv_C3 is not on the H100 hot path')
        self.k, self.s = k, s
        self.conv = nn.Conv2d(c1, c2, k, s, k // 2, groups=g, bias=False)
        self.bn = nn.BatchNorm2d(c2)
        self.act = nn.ReLU() if act is True else (act if isinstance(act, nn.Module) else nn.Identity())
        if isinstance(self.act, nn.ReLU):
            self.act_name = 'relu'
        elif isinstance(self.act, nn.SiLU):
            self.act_name = 'silu'
        elif isinstance(self.act, nn.Identity):
            self.act_name = None
        else:
            raise NotImplementedError(f'activation {type(self.act).__name__} is not on the H100 hot path')

    def emit(self, g, x, name='', **kw):
        w, b = folded(self.conv, self.bn)
        return g.conv(x, w, b, self.k, self.s, self.k // 2, self.act_name, name=name, **kw)


class BepC3(_Block):
    def __init__(self, in_channels, out_channels, n=1, e=0.5, concat=True, block=RepVGGBlock):
        super().__init__()
        c_ = int(out_channels * e)
        self.cv1 = Conv_C3(in_channels, c_, 1, 1)
        self.cv2 = Conv_C3(in_channels, c_, 1, 1)
        self.cv3 = Conv_C3(2 * c_, out_channels, 1, 1)
        self.m = RepBlock(in_channels=c_, out_channels=c_, n=n, block=BottleRep, basic_block=block)
        self.concat = concat
        if not concat:
            self.cv3 = Conv_C3(c_, out_channels, 1, 1)

    def emit(self, g, x, name='', out=None):
        if not self.concat:
            return self.cv3.emit(g, self.m.emit(g, self.cv1.emit(g, x, name + '.cv1'), name + '.m'), name + '.cv3', out=out)
        # cv1 || cv2 as one GEMM writing [a | b]; the RepBlock chain ends in the first half again; cv3 reads the whole buffer (no torch.cat)
        w1, b1 = folded(self.cv1.conv, self.cv1.bn)
        w2, b2 = folded(self.cv2.conv, self.cv2.bn)
        assert self.cv1.act_name == self.cv2.act_name
        ch = w1.shape[0]
        y = g.new_act(x.H, x.W, 2 * ch)
        g.conv(x, torch.cat([w1, w2], 0), torch.cat([b1, b2], 0), 1, 1, 0, self.cv1.act_name, out=y, name=name + '.cv12')
        a = y.slice(0, ch)
        self.m.emit(g, a, name + '.m', out=a)
        return self.cv3.emit(g, y, name + '.cv3', out=out)


class EELAN(_Block):
    def __init__(self, c1, c2, c3, norm_cfg=dict(type='BN', requires_grad=True), act_cfg=dict(type='SiLU', inplace=True)):
        super().__init__()
        kw = dict(norm_cfg=norm_cfg, act_cfg=act_cfg)
        self.conv1 = ConvModule(c1, c2, 1, 1, 0, **kw)
        self.conv2 = ConvModule(c1, c2, 1, 1, 0, **kw)
        self.conv3 = nn.Sequential(ConvModule(c2, c2, 3, 1, 1, **kw), ConvModule(c2, c2, 3, 1, 1, **kw))
        self.conv4 = nn.Sequential(ConvModule(c2, c2, 3, 1, 1, **kw), ConvModule(c2, c2, 3, 1, 1, **kw))
        self.conv5 = ConvModule(c2 * 4, c3, 1, 1, 0, **kw)

    def emit(self, g, x, name='', out=None):
        c2 = self.conv1.out_channels
        cat = g.new_act(x.H, x.W, 4 * c2)  # [x1 | x2 | x3 | x4] (:578-582), every producer writes its slice
        w1, b1 = folded(self.conv1.conv, self.conv1.bn)
        w2, b2 = folded(self.conv2.conv, self.conv2.bn)
        g.conv(x, torch.cat([w1, w2], 0), torch.cat([b1, b2], 0), 1, 1, 0, self.conv1.act_name, out=cat.slice(0, 2 * c2), name=name + '.conv12')
        t = self.conv3[0].emit(g, cat.slice(c2, c2), name + '.conv3.0')
        self.conv3[1].emit(g, t, name + '.conv3.1', out=cat.slice(2 * c2, c2))
        t = self.conv4[0].emit(g, cat.slice(2 * c2, c2), name + '.conv4.0')
        self.conv4[1].emit(g, t, name + '.conv4.1', out=cat.slice(3 * c2, c2))
        return self.conv5.emit(g, cat, name + '.conv5', out=out)
