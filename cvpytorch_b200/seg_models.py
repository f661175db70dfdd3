"""Drop-in modules for the DeepLabv3+ (ResNet-50 v1c) segmentation path (inference only, H100 fused graph).

Mirrors (paths relative to the reference checkout):
  Deeplabv3PlusHead   src/models/heads/seg/deeplabv3plus_head.py:33-68  (+ Deeplabv3Head / ASPP deeplabv3_head.py:15-75,
                      DepthwiseSeparableASPPModule deeplabv3plus_head.py:14-29, BaseSegHead base_seg_head.py:13-37)
  EncoderDecoder      src/models/segmentors/encoder_decoder.py:21-150 ('val' branch :131-133)
  backbone            ResNet('resnet50v1c', out_stages=[1, 4]) -> cvpytorch_b200.fcos_models.ResNet

Graph notes: every ``torch.cat`` is a channel slice of one buffer (5x512 ASPP concat; 512+48 decoder concat padded to 576
so the following GEMM keeps 64-channel K chunks); the image-pool branch is avgpool -> 1x1 GEMM on a 1x1 map -> bilinear
"resize" (a broadcast); depthwise 3x3 (dilated) convs are an HBM-bound SIMT kernel, their 1x1 pointwise convs run on the
tensor-core kernel; the final bilinear upsample + argmax is one kernel (the [B,19,H,W] fp32 tensor never exists).
"""
import torch
import torch.nn as nn

from . import ops
from .engine import GraphBuilder
from .fcos_models import ResNet
from .modules import ConvModule, DepthwiseSeparableConvModule, _build, _Model, _Standalone, folded


class ASPPModules(nn.ModuleList):
    """DepthwiseSeparableASPPModule: index 0 = 1x1 ConvModule, others = depthwise-separable 3x3 with the given dilation."""

    def __init__(self, dilations, in_channels, channels, norm_cfg, act_cfg):
        super().__init__()
        self.dilations = dilations
        for d in dilations:
            if d == 1:
                self.append(ConvModule(in_channels, channels, 1, norm_cfg=norm_cfg, act_cfg=act_cfg))
            else:
                self.append(DepthwiseSeparableConvModule(in_channels, channels, 3, dilation=d, padding=d, norm_cfg=norm_cfg, act_cfg=act_cfg))


class Deeplabv3PlusHead(_Standalone):
    def __init__(self, low_in_channels, low_channels, dilations=(1, 6, 12, 18), num_classes=19, in_channels=None, channels=None,
                 dropout_ratio=0.1, conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True), act_cfg=dict(type='ReLU')):
        super().__init__()
        self.num_classes, self.in_channels, self.channels, self.dilations = num_classes, in_channels, channels, tuple(dilations)
        self.dropout = nn.Dropout2d(dropout_ratio) if dropout_ratio > 0 else None  # identity in eval mode
        self.cls_seg = nn.Conv2d(channels, num_classes, kernel_size=1)
        self.proj = nn.Sequential(nn.AdaptiveAvgPool2d(1), ConvModule(in_channels, channels, 1, norm_cfg=norm_cfg, act_cfg=act_cfg))
        self.aspp = ASPPModules(self.dilations, in_channels, channels, norm_cfg, act_cfg)
        self.reduce = ConvModule((len(self.dilations) + 1) * channels, channels, 3, padding=1, norm_cfg=norm_cfg, act_cfg=act_cfg)
        if low_in_channels <= 0:
            raise NotImplementedError('Deeplabv3PlusHead without the low-level branch is not on the H100 hot path')
        self.low_proj = ConvModule(low_in_channels, low_channels, 1, norm_cfg=norm_cfg, act_cfg=act_cfg)
        self.low_channels = low_channels
        self.fuse = nn.Sequential(
            DepthwiseSeparableConvModule(channels + low_channels, channels, 3, padding=1, norm_cfg=norm_cfg, act_cfg=act_cfg),
            DepthwiseSeparableConvModule(channels, channels, 3, padding=1, norm_cfg=norm_cfg, act_cfg=act_cfg))

    def emit(self, g, feats, name='head'):
        """feats = [low (H/4), high (H/32)] Vals.  Returns the fp32 logits tensor [B,H/4,W/4,32] (num_classes used)."""
        low, x = feats
        ch = self.channels
        nb = len(self.dilations) + 1
        cat = g.new_act(x.H, x.W, nb * ch)
        # image-pool branch (deeplabv3_head.py:59-62,70): avgpool -> 1x1 conv+BN+ReLU -> bilinear to the map size (a broadcast)
        pooled = g.new_act(1, 1, x.c)
        g.fn(lambda: ops.global_avgpool(x.view(), pooled.view()))
        pj = self.proj[1].emit(g, pooled, name + '.proj.1')
        s0 = cat.slice(0, ch)
        g.fn(lambda: ops.bilinear_resize(pj.view(), s0.view()))
        for i, m in enumerate(self.aspp):
            m.emit(g, x, f'{name}.aspp.{i}', out=cat.slice((i + 1) * ch, ch))
        r = self.reduce.emit(g, cat, name + '.reduce')
        # decoder: cat([bilinear(r -> low size), low_proj(low)]) in one buffer, channel-padded to a multiple of 64
        c_used = ch + self.low_channels
        c_pad = (c_used + 63) // 64 * 64
        cat2 = g.new_act(low.H, low.W, c_pad)   # zero-initialised: the pad channels stay 0
        up = cat2.slice(0, ch)
        g.fn(lambda: ops.bilinear_resize(r.view(), up.view()))
        self.low_proj.emit(g, low, name + '.low_proj', out=cat2.slice(ch, self.low_channels))
        # fuse[0]: depthwise over the padded buffer (zero weights on the pad channels), pointwise with zero-padded input channels
        f0 = self.fuse[0]
        wd, bd = folded(f0.depthwise_conv.conv, f0.depthwise_conv.bn)
        wd_p = torch.zeros((c_pad, 1, 3, 3), dtype=torch.float64)
        wd_p[:c_used] = wd
        bd_p = torch.zeros(c_pad, dtype=torch.float64)
        bd_p[:c_used] = bd
        w9c, bias = ops.pack_dw_weights(wd_p, bd_p, device=g.device)
        g.buffers.append((w9c, bias))
        d0 = g.new_act(low.H, low.W, c_pad)
        g.fn(lambda: ops.dwconv3x3(cat2.view(), w9c, bias, 1, d0.view(), True))
        wp, bp = folded(f0.pointwise_conv.conv, f0.pointwise_conv.bn)
        wp_p = torch.zeros((wp.shape[0], c_pad, 1, 1), dtype=torch.float64)
        wp_p[:, :c_used] = wp
        f = g.conv(d0, wp_p, bp, 1, 1, 0, 'relu', name=name + '.fuse.0.pointwise_conv')
        f = self.fuse[1].emit(g, f, name + '.fuse.1')
        logits = g.new_f32(low.H, low.W, (self.num_classes + 31) // 32 * 32)
        g.conv(f, *folded(self.cls_seg), 1, 1, 0, None, f32_out=logits, name=name + '.cls_seg')   # dropout is identity in eval
        return logits

    def forward(self, x):
        return ops.f32nhwc_to_nchw(self._run(x).view(0, self.num_classes))


_BACKBONES = {'ResNet': ResNet}
_HEADS = {'Deeplabv3PlusHead': Deeplabv3PlusHead}


def build_backbone(cfg):
    return _build(_BACKBONES, cfg)


def build_head(cfg):
    return _build(_HEADS, cfg)


class EncoderDecoder(_Model):
    """Model-level drop-in for src.models.segmentors.encoder_decoder.EncoderDecoder (inference: mode='val' -> int64 [B,H,W])."""

    def __init__(self, dictionary=None, model_cfg=None, *args, **kwargs):
        super().__init__(dictionary, model_cfg)
        self.input_size = [1024, 2048]
        self.dummy_input = torch.zeros(1, 3, self.input_size[0], self.input_size[1])
        if self._cfg('NECK', None) is not None or self._cfg('AUX_HEAD', None) is not None:
            raise NotImplementedError('NECK / AUX_HEAD are not on the H100 hot path')
        bcfg = dict(self._cfg('BACKBONE'))
        bcfg['pretrained'] = False
        self.backbone = build_backbone(bcfg)
        self.head = build_head(dict(self._cfg('HEAD')))

    def build_graph(self, B, H, W, device, out_hw=None):
        g = GraphBuilder(B, device)
        holder = {}
        feats = self.backbone.emit(g, lambda: holder['x'], H, W)
        logits = self.head.emit(g, feats)
        Ho, Wo = out_hw if out_hw is not None else (H, W)
        labels = torch.zeros((B, Ho, Wo), dtype=torch.int64, device=device)
        nc = self.head.num_classes
        g.fn(lambda: ops.upsample_argmax(logits.view(0, nc), nc, labels))
        g.buffers.append(labels)
        return dict(g=g, holder=holder, logits=logits, labels=labels, feats=feats)

    def _graph_for(self, imgs, out_hw=None):
        return self._graph([imgs], lambda: self.build_graph(imgs.shape[0], imgs.shape[2], imgs.shape[3], imgs.device, out_hw), out_hw)

    def predict(self, imgs, out_hw=None):
        """Device-only inference: int64 label map [B, Ho, Wo] (Ho, Wo default to the input size); no host sync.
        The returned tensor is the GRAPH-OWNED output buffer: the next call with the same shape overwrites it (zero-copy);
        ``forward()`` returns a fresh tensor like the reference does."""
        return self._replay(imgs.contiguous().float(), out_hw)['labels']

    def _infer(self, imgs):
        # the reference's 'infer' branch calls torch.argmax on a *list* and raises TypeError (SURVEY.md 3.3); the usable
        # inference path is 'val'.  Here 'infer' returns the label map at input resolution.
        return self.predict(imgs).clone()

    def _val(self, imgs, targets):
        out_hw = tuple(targets.shape[-2:]) if targets is not None else None
        # encoder_decoder.py:131-133: argmax(bilinear(preds -> targets size)); a fresh tensor per call like the reference (a caller may
        # keep predictions of several batches), the zero-copy graph buffer is only handed out by predict()
        return self.predict(imgs, out_hw).clone()
