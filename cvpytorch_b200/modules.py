"""Drop-in ``nn.Module`` mirrors of the reference's hot-path building blocks.

Same constructor arguments, same sub-module / parameter names (=> identical ``state_dict`` keys, so reference
checkpoints load unchanged), same call signatures.  Instead of executing PyTorch ops, every module *emits* its
layers into a :class:`cvpytorch_b200.engine.GraphBuilder`; the model-level module then runs the fused graph
on the H100 through the C ABI.  Training is out of scope (inference path only): ``forward`` in training mode or
on a CPU tensor raises -- there is no fallback.

Mirrors (paths relative to the reference checkout):
  ConvModule            src/models/bricks/conv_module.py:20-214   (conv / bn / activate attribute names :131,:170,:178)
  Conv, Bottleneck, C3  src/models/modules/yolo11_modules.py:27-39, :173-183, :205-217
  DarknetBottleneck, CSPLayer, SPPF   src/models/modules/yolo_modules.py:40-104, :107-140, :165-194
  UpsamplingModule, DownsamplingModule  src/models/modules/yolo11_modules.py:388-408
"""

from copy import deepcopy

import torch
import torch.nn as nn

from . import _lib, ops
from .engine import GraphBuilder

BN_EPS = 1e-3


def _act_name(act_cfg):
    if act_cfg is None:
        return None
    t = act_cfg['type']
    if t in ('SiLU', 'Swish'):
        return 'silu'
    if t == 'ReLU':
        return 'relu'
    raise NotImplementedError(f'activation {t} is not on the H100 hot path')


def _bn_tuple(bn):
    return (bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)


def folded(conv, bn=None):
    """(w64 [O,I,k,k], b64 [O]) with eval-mode BN folded in (algebra of src/utils/fuse.py:33-54)."""
    return ops.fold_conv_bn(conv.weight, conv.bias, _bn_tuple(bn) if bn is not None else None)


class _EmitModule(nn.Module):
    """Base: modules on the fused path are not executed op by op."""

    def forward(self, *a, **k):  # pragma: no cover - guarded path
        raise RuntimeError(f'{type(self).__name__} is a H100 fused-path block: it is executed as part of its parent '
                           'backbone / neck / detect graph (call the parent module), not stand-alone')


class _Standalone(nn.Module):
    """Base of every drop-in that runs on its own (model, backbone, neck / head, brick, block): the module is built into a
    GraphBuilder graph once per input and the graph is replayed on later calls.

    ``_graph`` is the only way to that cache.  It rejects what the graph cannot run -- training mode (RuntimeError), and any input
    that is not a 4-D CUDA tensor on the current device (CvbError: plans, buffers and TMA descriptors belong to the device a graph
    was built on, INTEGRATION.md §4) -- before it looks anything up.  A graph is keyed by the input shapes, the device and the
    caller's extra key.  The weights are folded into the plans when a graph is built, so ``load_state_dict``, ``train()`` /
    ``eval()`` and ``RepVGGBlock.switch_to_deploy`` drop every graph of the module; weights changed any other way (in place, or
    by ``switch_to_deploy`` of a block inside a module that has run) take effect after the next ``eval()``.  Inference only: there
    is no CPU fallback."""

    def __init__(self):
        super().__init__()
        self._graphs = {}

    def _drop_graphs(self):
        self._graphs.clear()

    def __getstate__(self):
        """What copy.deepcopy and pickle take: the module without its device caches.  The graphs (plans that own C handles, buffers, TMA
        descriptors) are rebuilt on the copy's first eval-mode call, and the training modules (train.bound_training_modules, bound to THIS
        model's tensors) on its first training call, so the copy never runs on the original's parameters.  The original keeps both."""
        state = super().__getstate__()
        state['_graphs'] = {}
        if '_train_modules' in state:
            state['_train_modules'] = None
        return state

    def train(self, mode=True):
        self._drop_graphs()
        return super().train(mode)

    def _load_from_state_dict(self, *a, **k):
        self._drop_graphs()
        return super()._load_from_state_dict(*a, **k)

    def _graph(self, xs, build, *key):
        """The graph ``build()`` returned for inputs ``xs`` (a list of tensors), built on the first call with these shapes."""
        name = type(self).__name__
        if self.training:
            raise RuntimeError(f'{name}: the H100 path implements inference only; call .eval() first '
                               '(training stays on the reference implementation)')
        for x in xs:
            if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dim() == 4):
                raise _lib.CvbError(f'{name}: every input must be a 4-D CUDA tensor; there is no CPU fallback')
            if x.device.index != torch.cuda.current_device():
                raise _lib.CvbError(f'{name}: input lives on cuda:{x.device.index} but the current device is '
                                    f'cuda:{torch.cuda.current_device()}; call torch.cuda.set_device() first (one device per process)')
        key = tuple(tuple(x.shape) for x in xs) + (xs[0].device.index,) + key
        if key not in self._graphs:
            self._graphs[key] = build()
        return self._graphs[key]

    def _run(self, xs, emit=None, cin_align=1):
        """Runs ``emit(g, ins)`` (default ``self.emit``) on the NCHW fp32 maps ``xs`` and returns what it returned.  ``ins`` are
        split-NHWC input buffers with the channels of ``xs`` rounded up to a multiple of ``cin_align``; the extra channels stay zero."""
        def build():
            g = GraphBuilder(xs[0].shape[0], xs[0].device)
            ins = [g.new_act(x.shape[2], x.shape[3], (x.shape[1] + cin_align - 1) // cin_align * cin_align) for x in xs]
            return g, ins, (emit or self.emit)(g, ins)
        g, ins, outs = self._graph(xs, build)
        for x, v in zip(xs, ins):
            ops.nchw_to_split(x, v.slice(0, x.shape[1]).view())
        g.run()
        return outs

    def _run_image(self, x):
        """``forward`` of the image backbones: NCHW fp32 images -> the NCHW fp32 maps of ``out_stages`` (the map itself when there
        is one stage), from ``self.emit(g, image_getter, H, W)``."""
        def build():
            g, holder = GraphBuilder(x.shape[0], x.device), {}
            return g, holder, self.emit(g, lambda: holder['x'], x.shape[2], x.shape[3])
        g, holder, outs = self._graph([x], build)
        holder['x'] = x.contiguous().float()
        g.run()
        res = [ops.split_to_nchw(o.view()) for o in outs]
        return res if len(self.out_stages) > 1 else res[0]


class _Model(_Standalone):
    """Base of the model-level drop-ins (YOLOv5, YOLOX, YOLOv6, FCOS, EncoderDecoder): the reference's ``(dictionary=, model_cfg=)``
    constructor and ``forward(imgs, targets, mode)`` contract.  A subclass defines ``build_graph(B, H, W, device)`` (whose graph reads its
    input from holder['x']) and ``_val(imgs, targets)``; it overrides ``forward_train`` when it trains and ``_infer`` when its 'infer'
    result is not the detectors' None."""

    def __init__(self, dictionary, model_cfg):
        super().__init__()
        self.dictionary, self.model_cfg = dictionary, model_cfg
        self.num_classes = len(dictionary)

    def _cfg(self, key, *default):
        """``model_cfg[key]`` of a dict or an attribute config.  Without a default, a missing key raises KeyError naming it."""
        try:
            return self.model_cfg[key] if isinstance(self.model_cfg, dict) else getattr(self.model_cfg, key)
        except (KeyError, AttributeError):
            if default:
                return default[0]
            raise KeyError(f'{type(self).__name__}: model_cfg has no {key!r} entry') from None

    def forward(self, imgs, targets=None, mode='infer', **kwargs):
        if mode == 'infer':
            return self._infer(imgs)
        if mode not in ('train', 'val'):
            raise RuntimeError(f'{type(self).__name__} (H100): unknown mode {mode!r}')
        if isinstance(imgs, (list, tuple)):
            imgs = torch.stack(list(imgs))
        return self.forward_train(imgs, targets) if mode == 'train' else self._val(imgs, targets)

    def _infer(self, imgs):
        return None  # what the reference detectors return in 'infer' mode (yolov5.py:247-249, yolox.py:144-149, fcos.py:120-121)

    def forward_train(self, imgs, targets):
        raise RuntimeError(f"{type(self).__name__} (H100): only mode='val' (inference) is implemented; training stays on the reference")

    def _graph_for(self, imgs, *key):
        """The cached graph of ``build_graph`` for the NCHW images ``imgs``, keyed by their shape and ``key``."""
        return self._graph([imgs], lambda: self.build_graph(imgs.shape[0], imgs.shape[2], imgs.shape[3], imgs.device), *key)

    def _replay(self, x, *args):
        """Runs the graph ``_graph_for(x, *args)`` on the input ``x`` and returns its dict."""
        G = self._graph_for(x, *args)
        G['holder']['x'] = x
        G['g'].run()
        return G

    @staticmethod
    def _val_losses(device):
        # the reference returns its loss dict next to the val outputs; that loss is a training diagnostic and is not computed on the H100
        # path.  A zero 'loss' entry keeps the unchanged trainer alive (trainer.py:216-219 -> reduce_dict -> torch.stack needs a non-empty
        # dict under cfg.distributed)
        return {'loss': torch.zeros((), dtype=torch.float32, device=device)}


def _build(table, cfg):
    """Reference factory contract (src/models/{backbones,necks,heads,detects}/__init__.py): deepcopy the cfg, pop 'name',
    Class(**cfg); an unknown name raises NotImplementedError."""
    c = deepcopy(dict(cfg))
    name = c.pop('name')
    if name not in table:
        raise NotImplementedError(name)
    return table[name](**c)


def _pad_cin(w, n):
    """[O,I,k,k] weights with n zero input channels appended."""
    return nn.functional.pad(w, (0, 0, 0, 0, 0, n))


class _StandaloneBrick(_Standalone):
    """Brick-level drop-in (SURVEY.md 8b: ConvModule(conv_cfg=dict(type='B200Conv2d'), ...) inside an otherwise unchanged reference
    model): called on its own, the brick runs as a one-layer graph with the layout adapters at its boundary -- NCHW fp32 in, NCHW fp32
    out, like the reference's ConvModule.forward (conv_module.py:201-214).  Inside a H100 parent it is emitted into the parent's graph
    and this method is never used."""

    def forward(self, x):
        # the tensor-core path wants cin % 16 == 0: the input buffer gets zero channels up to it, read with zero weights.  The pad is
        # counted from the input's own channels, so an input whose channel count is not the brick's fails the conv's channel check.
        return ops.split_to_nchw(self._run([x], lambda g, ins: self._emit_padded(g, ins[0], x.shape[1]), cin_align=16).view())


class ConvModule(_StandaloneBrick):
    """conv -> BN -> activation bundle.  Keys: ``conv.weight``, ``bn.{weight,bias,running_mean,running_var,num_batches_tracked}``."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias='auto',
                 conv_cfg=None, norm_cfg=None, act_cfg=dict(type='ReLU'), inplace=True, with_spectral_norm=False,
                 padding_mode='zeros', order=('conv', 'norm', 'act')):
        super().__init__()
        if with_spectral_norm or padding_mode != 'zeros' or tuple(order) != ('conv', 'norm', 'act'):
            raise NotImplementedError('ConvModule variant not on the H100 hot path')
        if groups != 1 and not (groups == in_channels == out_channels and kernel_size == 3 and stride == 1 and padding == dilation):
            raise NotImplementedError('grouped conv: only depthwise 3x3 / stride 1 / padding == dilation is on the H100 hot path')
        self.groups = groups
        if conv_cfg is not None and conv_cfg.get('type') not in (None, 'Conv2d', 'Conv', 'B200Conv2d'):
            raise NotImplementedError(f'conv_cfg {conv_cfg}')
        if norm_cfg is not None and norm_cfg.get('type') not in ('BN', 'BN2d'):
            raise NotImplementedError(f'norm_cfg {norm_cfg} (only eval-mode BatchNorm folds into the conv)')
        self.with_norm = norm_cfg is not None
        self.with_act = act_cfg is not None
        if bias == 'auto':
            bias = not self.with_norm  # conv_module.py:108-110
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride, self.padding, self.dilation = kernel_size, stride, padding, dilation
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride, padding, dilation, groups=groups, bias=bias)
        if self.with_norm:
            self.bn = nn.BatchNorm2d(out_channels, eps=norm_cfg.get('eps', 1e-5), momentum=norm_cfg.get('momentum', 0.1))
        self.act_name = _act_name(act_cfg)
        nn.init.kaiming_normal_(self.conv.weight, a=0, mode='fan_out', nonlinearity='relu')  # conv_module.py:181-199

    def _emit_padded(self, g, x, cin):
        if self.groups != 1:
            return self.emit(g, x.slice(0, cin))
        w, b = folded(self.conv, self.bn if self.with_norm else None)
        return g.conv(x, _pad_cin(w, x.c - cin), b, self.kernel_size, self.stride, self.padding, self.act_name, dilation=self.dilation)

    def emit(self, g, x, name='', **kw):
        w, b = folded(self.conv, self.bn if self.with_norm else None)
        if self.groups != 1:  # depthwise: HBM-bound SIMT kernel (no tensor cores for 9 MACs per output)
            if self.act_name not in (None, 'relu'):
                raise NotImplementedError('depthwise conv: ReLU / no activation only')
            assert w.shape[0] == x.c, (name, w.shape[0], x.c)  # the kernel reads one weight column per input channel
            out = kw.get('out') or g.new_act(x.H, x.W, x.c)
            w9c, bias = ops.pack_dw_weights(w, b, device=g.device)
            g.buffers.append((w9c, bias))
            dil, relu = self.dilation, self.act_name == 'relu'
            g.fn(lambda: ops.dwconv3x3(x.view(), w9c, bias, dil, out.view(), relu))
            return out
        return g.conv(x, w, b, self.kernel_size, self.stride, self.padding, self.act_name, dilation=self.dilation, name=name, **kw)


class DepthwiseSeparableConvModule(_EmitModule):
    """src/models/bricks/depthwise_separable_conv_module.py:10-99: depthwise ConvModule + pointwise ConvModule."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, norm_cfg=None, act_cfg=dict(type='ReLU'),
                 dw_norm_cfg='default', dw_act_cfg='default', pw_norm_cfg='default', pw_act_cfg='default', **kwargs):
        super().__init__()
        dw_norm_cfg = dw_norm_cfg if dw_norm_cfg != 'default' else norm_cfg
        dw_act_cfg = dw_act_cfg if dw_act_cfg != 'default' else act_cfg
        pw_norm_cfg = pw_norm_cfg if pw_norm_cfg != 'default' else norm_cfg
        pw_act_cfg = pw_act_cfg if pw_act_cfg != 'default' else act_cfg
        self.depthwise_conv = ConvModule(in_channels, in_channels, kernel_size, stride=stride, padding=padding, dilation=dilation,
                                         groups=in_channels, norm_cfg=dw_norm_cfg, act_cfg=dw_act_cfg, **kwargs)
        self.pointwise_conv = ConvModule(in_channels, out_channels, 1, norm_cfg=pw_norm_cfg, act_cfg=pw_act_cfg, **kwargs)

    def emit(self, g, x, name='', out=None):
        d = self.depthwise_conv.emit(g, x, name + '.depthwise_conv')
        return self.pointwise_conv.emit(g, d, name + '.pointwise_conv', out=out)


class Conv(_StandaloneBrick):
    """Old-API conv block (yolo11_modules.py:27-39): keys ``conv.weight``, ``bn.*``; SiLU; autopad."""

    def __init__(self, c1, c2, k=1, s=1, p=None, g=1, act=True):
        super().__init__()
        if g != 1:
            raise NotImplementedError('grouped Conv is not on the H100 hot path')
        self.k, self.s = k, s
        self.p = k // 2 if p is None else p
        self.conv = nn.Conv2d(c1, c2, k, s, self.p, groups=g, bias=False)
        self.bn = nn.BatchNorm2d(c2)
        self.act_name = 'silu' if act is True else None
        if act is not True and act is not False and act is not None:
            raise NotImplementedError('custom activation module')

    def _emit_padded(self, g, x, cin):
        w, b = folded(self.conv, self.bn)
        return g.conv(x, _pad_cin(w, x.c - cin), b, self.k, self.s, self.p, self.act_name)

    def emit(self, g, x, name='', **kw):
        w, b = folded(self.conv, self.bn)
        return g.conv(x, w, b, self.k, self.s, self.p, self.act_name, name=name, **kw)


def _emit_csp(g, x, c1, c2, c3, blocks, shortcut, name, up_src=None, out=None):
    """Shared CSPLayer / C3 graph.  c1,c2,c3: conv blocks; blocks: [(b.conv1, b.conv2)].
    up_src: optional Val at half resolution whose nearest-upsampled version is the FIRST part of the (virtual)
    channel concat feeding c1/c2 -- handled as an fp32 partial GEMM (see engine docstring)."""
    w1, b1 = folded(c1.conv, c1.bn)
    w2, b2 = folded(c2.conv, c2.bn)
    wm = torch.cat([w1, w2], 0)
    bm = torch.cat([b1, b2], 0)
    ch = w1.shape[0]
    y = g.new_act(x.H, x.W, 2 * ch)
    if up_src is not None:
        cu = up_src.c
        assert wm.shape[1] == cu + x.c
        part = g.new_f32(up_src.H, up_src.W, 2 * ch)
        g.conv(up_src, wm[:, :cu].contiguous(), torch.zeros_like(bm), 1, 1, 0, None, f32_out=part, name=name + '.cv12.up_partial')
        g.conv(x, wm[:, cu:].contiguous(), bm, 1, 1, 0, 'silu', out=y, up_partial=part, name=name + '.cv12')
    else:
        g.conv(x, wm, bm, 1, 1, 0, 'silu', out=y, name=name + '.cv12')
    chain = y.slice(0, ch)
    if blocks:
        t = g.new_act(x.H, x.W, blocks[0][0].conv.weight.shape[0])
    for i, (ba, bb) in enumerate(blocks):
        wa, ba_ = folded(ba.conv, ba.bn)
        wb, bb_ = folded(bb.conv, bb.bn)
        g.conv(chain, wa, ba_, 1, 1, 0, 'silu', out=t, name=f'{name}.m.{i}.1x1')
        g.conv(t, wb, bb_, 3, 1, 1, 'silu', out=chain, residual=chain if shortcut else None, name=f'{name}.m.{i}.3x3')
    w3, b3 = folded(c3.conv, c3.bn)
    return g.conv(y, w3, b3, 1, 1, 0, 'silu', out=out, name=name + '.cv3')


class DarknetBottleneck(_EmitModule):
    def __init__(self, in_channels, out_channels, expansion=0.5, shortcut=True, depthwise=False, conv_cfg=None,
                 norm_cfg=dict(type='BN', requires_grad=True), act_cfg=dict(type='Swish'), init_cfg=None):
        super().__init__()
        if depthwise:
            raise NotImplementedError('depthwise bottleneck is not on the H100 hot path')
        hidden = int(out_channels * expansion)
        self.conv1 = ConvModule(in_channels, hidden, 1, conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg)
        self.conv2 = ConvModule(hidden, out_channels, 3, stride=1, padding=1, conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg)
        self.shortcut = shortcut and in_channels == out_channels


class CSPLayer(_EmitModule):
    """C3 in yolov5 (yolo_modules.py:107-140)."""

    def __init__(self, in_channels, out_channels, n=1, expansion=0.5, shortcut=True, depthwise=False, conv_cfg=None,
                 norm_cfg=dict(type='BN', requires_grad=True), act_cfg=dict(type='Swish')):
        super().__init__()
        hidden = int(out_channels * expansion)
        self.conv1 = ConvModule(in_channels, hidden, 1, stride=1, conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg)
        self.conv2 = ConvModule(in_channels, hidden, 1, stride=1, conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg)
        self.conv3 = ConvModule(2 * hidden, out_channels, 1, stride=1, conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg)
        self.m = nn.Sequential(*[DarknetBottleneck(hidden, hidden, 1.0, shortcut, depthwise, conv_cfg=conv_cfg, norm_cfg=norm_cfg,
                                                   act_cfg=act_cfg) for _ in range(n)])

    def emit(self, g, x, name='', out=None):
        blocks = [(b.conv1, b.conv2) for b in self.m]
        sc = all(b.shortcut for b in self.m) if len(self.m) else False
        return _emit_csp(g, x, self.conv1, self.conv2, self.conv3, blocks, sc, name, out=out)


class SPPF(_EmitModule):
    """yolo_modules.py:165-194 (int kernel_sizes path)."""

    def __init__(self, in_channels, out_channels, kernel_sizes=(5, 9, 13), conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True),
                 act_cfg=dict(type='Swish'), init_cfg=None):
        super().__init__()
        # int 5: three chained 5x5 pools; (5, 9, 13): three parallel pools of the same input -- identical values (a chain of two /
        # three 5x5 max pools IS the 9x9 / 13x13 max pool), so both run the same fused kernel
        if not ((isinstance(kernel_sizes, int) and kernel_sizes == 5) or tuple(kernel_sizes) == (5, 9, 13)):
            raise NotImplementedError('only SPPF with kernel_sizes=5 (chained) or (5, 9, 13) (parallel) is on the H100 hot path')
        self.kernel_sizes = kernel_sizes
        hidden = in_channels // 2
        self.conv1 = ConvModule(in_channels, hidden, 1, stride=1, conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg)
        if isinstance(kernel_sizes, int):
            self.m = nn.MaxPool2d(kernel_size=kernel_sizes, stride=1, padding=kernel_sizes // 2)  # parameter-free; kept for repr parity
        else:
            self.m = nn.ModuleList([nn.MaxPool2d(kernel_size=ks, stride=1, padding=ks // 2) for ks in kernel_sizes])
        self.conv2 = ConvModule(hidden * 4, out_channels, 1, stride=1, conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg)

    def emit(self, g, x, name='', out=None):
        hidden = self.conv1.out_channels
        s = g.new_act(x.H, x.W, 4 * hidden)
        self.conv1.emit(g, x, name + '.conv1', out=s.slice(0, hidden))
        v = [s.slice(i * hidden, hidden) for i in range(4)]
        g.fn(lambda: ops.sppf_pool(v[0].view(), v[1].view(), v[2].view(), v[3].view()))
        return self.conv2.emit(g, s, name + '.conv2', out=out)


class Bottleneck(_EmitModule):
    def __init__(self, c1, c2, shortcut=True, g=1, e=0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c_, c2, 3, 1, g=g)
        self.add = shortcut and c1 == c2


class C3(_EmitModule):
    def __init__(self, c1, c2, n=1, shortcut=True, g=1, e=0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c1, c_, 1, 1)
        self.cv3 = Conv(2 * c_, c2, 1)
        self.m = nn.Sequential(*[Bottleneck(c_, c_, shortcut, g, e=1.0) for _ in range(n)])

    def emit(self, g, x, name='', up_src=None, out=None):
        blocks = [(b.cv1, b.cv2) for b in self.m]
        sc = all(b.add for b in self.m) if len(self.m) else False
        return _emit_csp(g, x, self.cv1, self.cv2, self.cv3, blocks, sc, name, up_src=up_src, out=out)


class UpsamplingModule(_EmitModule):
    """yolo11_modules.py:388-397: x_conv = conv(x); fuse(cat([up(x_conv), y])) -> (fused, x_conv)."""

    def __init__(self, c1, c2, layer=3):
        super().__init__()
        self.conv = Conv(c1, c2, 1, 1)
        self.up = nn.UpsamplingNearest2d(scale_factor=2)
        self.fuse = C3(c2 * 2, c2, layer, False)

    def emit(self, g, x, y, name='', lateral_out=None):
        x_conv = self.conv.emit(g, x, name + '.conv', out=lateral_out)
        return self.fuse.emit(g, y, name + '.fuse', up_src=x_conv), x_conv


class DownsamplingModule(_EmitModule):
    """yolo11_modules.py:400-408: fuse(cat([down(x), y])).  `cat_buf` already holds y in its second half."""

    def __init__(self, c1, c2, layer=3):
        super().__init__()
        self.down = Conv(c1, c1, 3, 2)
        self.fuse = C3(c1 * 2, c2, layer, False)

    def emit(self, g, x, cat_buf, name=''):
        c1 = self.down.conv.out_channels
        self.down.emit(g, x, name + '.down', out=cat_buf.slice(0, c1))
        return self.fuse.emit(g, cat_buf, name + '.fuse')
