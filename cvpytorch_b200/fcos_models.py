"""Drop-in modules for the FCOS-ResNet50 path (reference surface kept; inference only, H100 fused graph).

Mirrors (paths relative to the reference checkout):
  ResNet       src/models/backbones/seg/resnet.py:27-154  (wrapper around third-party torchvision.models.resnet50: keys
               stem.0/stem.1 (conv1/bn1), layerL.B.{conv1,bn1,conv2,bn2,conv3,bn3,downsample.0,downsample.1})
  FCOSFPN      src/models/necks/fcos_fpn.py:12-55
  FCOSHead     src/models/heads/fcos_head.py:22-84 (+ ScaleExp :13-19)
  FCOSDetect   src/models/detects/fcos_detect.py:34-186
  FCOS         src/models/fcos.py:24-169

Graph notes: BN folds into the convs; the ResNet bottleneck's ``out += identity; relu`` is the conv epilogue with
residual_before_act; the 7x7/s2 stem runs as 4 filter rows over the space-to-depth input (row-window mode); the FPN's
``P4 = prj_4(C4) + nearest_up(P5)`` is the up_partial epilogue; GroupNorm+ReLU is a two-pass kernel; decode, top-k and the
(class-offset, '+1'-area) NMS run on device with fixed-capacity outputs.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from . import _lib, ops
from .engine import GraphBuilder
from .modules import _build, _Model, _Standalone, folded


# =============================================================================================== ResNet-50
class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride, 1, bias=False)  # v1.5: stride on the 3x3
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride

    def emit(self, g, x, name):
        w, b = folded(self.conv1, self.bn1)
        t = g.conv(x, w, b, 1, 1, 0, 'relu', name=name + '.conv1')
        w, b = folded(self.conv2, self.bn2)
        t = g.conv(t, w, b, 3, self.stride, 1, 'relu', name=name + '.conv2')
        idn = x
        if self.downsample is not None:
            w, b = folded(self.downsample[0], self.downsample[1])
            idn = g.conv(x, w, b, 1, self.stride, 0, None, name=name + '.downsample')
        w, b = folded(self.conv3, self.bn3)
        return g.conv(t, w, b, 1, 1, 0, 'relu', residual=idn, residual_before_act=True, name=name + '.conv3')


def resnet_stem_weights_to_s2d(w64):
    """7x7/s2/p3 kernel [O,3,7,7] -> 4x4 kernel over the 16-channel space-to-depth input: filter row kh = 2*(a-2)+dy+3 with
    a in 0..3 (rows h-2..h+1), channel = (dy*2+dx)*3 + c; (a=0,dy=0) / (b=0,dx=0) have no source tap and stay zero."""
    O, I, kh, kw = w64.shape
    assert (I, kh, kw) == (3, 7, 7)
    out = torch.zeros((O, 16, 4, 4), dtype=torch.float64)
    for a in range(4):
        for dy in range(2):
            ky = 2 * (a - 2) + dy + 3
            if not 0 <= ky < 7:
                continue
            for b in range(4):
                for dx in range(2):
                    kx = 2 * (b - 2) + dx + 3
                    if not 0 <= kx < 7:
                        continue
                    for c in range(3):
                        out[:, (dy * 2 + dx) * 3 + c, a, b] = w64[:, c, ky, kx]
    return out


def deep_stem_weights_to_s2d(w64):
    """3x3/s2/p1 kernel [O,3,3,3] -> 2x2 kernel over the 16-channel space-to-depth input (rows h-1..h, cols w-1..w):
    filter row ky = 2*(a-1)+dy+1 with a in 0..1; (a=0,dy=0) has no source tap."""
    O, I, kh, kw = w64.shape
    assert (I, kh, kw) == (3, 3, 3)
    out = torch.zeros((O, 16, 2, 2), dtype=torch.float64)
    for a in range(2):
        for dy in range(2):
            ky = 2 * (a - 1) + dy + 1
            if not 0 <= ky < 3:
                continue
            for b in range(2):
                for dx in range(2):
                    kx = 2 * (b - 1) + dx + 1
                    if not 0 <= kx < 3:
                        continue
                    for c in range(3):
                        out[:, (dy * 2 + dx) * 3 + c, a, b] = w64[:, c, ky, kx]
    return out


class ResNet(_Standalone):
    def __init__(self, subtype='resnet50', out_stages=[2, 3, 4], output_stride=32, frozen_stages=-1, norm_eval=False, conv_cfg=None,
                 norm_cfg=dict(type='BN', requires_grad=True), classifier=False, num_classes=1000, backbone_path=None, pretrained=True):
        super().__init__()
        if subtype not in ('resnet50', 'resnet50v1c'):
            raise NotImplementedError(f'{subtype}: only resnet50 / resnet50v1c are on the H100 hot path in this round')
        if classifier:
            raise NotImplementedError('classifier head is not on the H100 hot path')
        # output_stride 8/16 is accepted and ignored exactly like the reference does for resnet50 (its dilation branch only
        # matches 'resnet18'/'resnet34' subtypes, src/models/backbones/seg/resnet.py:102-118; SURVEY.md 3.3).
        self.subtype, self.out_stages = subtype, out_stages
        self.deep_stem = subtype.endswith('c')
        if self.deep_stem:  # resnet.py:67-79
            self.stem = nn.Sequential(nn.Conv2d(3, 32, 3, 2, 1, bias=False), nn.BatchNorm2d(32), nn.ReLU(inplace=True),
                                      nn.Conv2d(32, 32, 3, 1, 1, bias=False), nn.BatchNorm2d(32), nn.ReLU(inplace=True),
                                      nn.Conv2d(32, 64, 3, 1, 1, bias=False), nn.BatchNorm2d(64), nn.ReLU(inplace=True))
        else:
            self.stem = nn.Sequential(nn.Conv2d(3, 64, 7, 2, 3, bias=False), nn.BatchNorm2d(64), nn.ReLU(inplace=True))
        self.maxpool = nn.MaxPool2d(3, 2, 1)
        inplanes = 64
        for li, (planes, blocks, stride) in enumerate(((64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)), start=1):
            layers = []
            for bi in range(blocks):
                s = stride if bi == 0 else 1
                ds = None
                if bi == 0 and (s != 1 or inplanes != planes * 4):
                    ds = nn.Sequential(nn.Conv2d(inplanes, planes * 4, 1, s, bias=False), nn.BatchNorm2d(planes * 4))
                layers.append(Bottleneck(inplanes, planes, s, ds))
                inplanes = planes * 4
            setattr(self, f'layer{li}', nn.Sequential(*layers))
        all_ch = [64, 256, 512, 1024, 2048]
        self.out_channels = [all_ch[o] for o in out_stages]

    def freeze_stages(self, n):  # called by the reference FCOS.train (fcos.py:77); a no-op for inference
        pass

    def emit(self, g, img_getter, H, W, name='backbone'):
        x0 = g.new_act(H // 2, W // 2 + 3, 16)
        if self.deep_stem:
            g.fn(lambda: ops.stem_s2d(img_getter(), x0.view(), pad_left=1))
            w, b = folded(self.stem[0], self.stem[1])
            t = g.new_act(H // 2, W // 2, 32)
            g.conv(x0, deep_stem_weights_to_s2d(w), b, 2, 1, 1, 'relu', out=t, w_window=4, name=name + '.stem.0')
            t = g.conv(t, *folded(self.stem[3], self.stem[4]), 3, 1, 1, 'relu', name=name + '.stem.3')
            c1 = g.conv(t, *folded(self.stem[6], self.stem[7]), 3, 1, 1, 'relu', name=name + '.stem.6')
        else:
            g.fn(lambda: ops.stem_s2d(img_getter(), x0.view(), pad_left=2))
            w, b = folded(self.stem[0], self.stem[1])
            c1 = g.new_act(H // 2, W // 2, 64)
            g.conv(x0, resnet_stem_weights_to_s2d(w), b, 4, 1, 2, 'relu', out=c1, w_window=4, name=name + '.stem')
        Hp, Wp = (H // 2 + 2 - 3) // 2 + 1, (W // 2 + 2 - 3) // 2 + 1
        x = g.new_act(Hp, Wp, 64)
        g.fn(lambda c1=c1, x=x: ops.maxpool3x3s2(c1.view(), x.view()))  # bind now: `x` is re-assigned below
        outs = []
        for li in range(1, 5):
            for bi, blk in enumerate(getattr(self, f'layer{li}')):
                x = blk.emit(g, x, f'{name}.layer{li}.{bi}')
            if li in self.out_stages:
                outs.append(x)
        return outs

    def forward(self, x):
        return self._run_image(x)


# =============================================================================================== FPN
class FCOSFPN(_Standalone):
    def __init__(self, in_channels=[512, 1024, 2048], out_channels=256):
        super().__init__()
        self.prj_3 = nn.Conv2d(in_channels[0], out_channels, 1)
        self.prj_4 = nn.Conv2d(in_channels[1], out_channels, 1)
        self.prj_5 = nn.Conv2d(in_channels[2], out_channels, 1)
        self.conv_5 = nn.Conv2d(out_channels, out_channels, 3, 1, 1)
        self.conv_4 = nn.Conv2d(out_channels, out_channels, 3, 1, 1)
        self.conv_3 = nn.Conv2d(out_channels, out_channels, 3, 1, 1)
        self.conv_out6 = nn.Conv2d(out_channels, out_channels, 3, 2, 1)
        self.conv_out7 = nn.Conv2d(out_channels, out_channels, 3, 2, 1)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_uniform_(m.weight, a=1)
                nn.init.constant_(m.bias, 0)

    def emit(self, g, feats, name='neck'):
        C3, C4, C5 = feats
        for hi, lo in ((C4, C5), (C3, C4)):
            if hi.H != 2 * lo.H or hi.W != 2 * lo.W:
                raise NotImplementedError('FCOSFPN on the H100 path needs exact 2x pyramid levels (input H, W multiples of 32)')
        oc = self.prj_5.out_channels
        f = lambda m: folded(m)
        p5 = g.conv(C5, *f(self.prj_5), 1, 1, 0, None, name=name + '.prj_5')
        p5f = g.new_f32(p5.H, p5.W, oc)
        g.fn(lambda: ops.split_to_f32(p5.view(), p5f.view()))
        p4 = g.conv(C4, *f(self.prj_4), 1, 1, 0, None, up_partial=p5f, name=name + '.prj_4')   # P4 = prj_4(C4) + up(P5)
        p4f = g.new_f32(p4.H, p4.W, oc)
        g.fn(lambda: ops.split_to_f32(p4.view(), p4f.view()))
        p3 = g.conv(C3, *f(self.prj_3), 1, 1, 0, None, up_partial=p4f, name=name + '.prj_3')   # P3 = prj_3(C3) + up(P4)
        P3 = g.conv(p3, *f(self.conv_3), 3, 1, 1, None, name=name + '.conv_3')
        P4 = g.conv(p4, *f(self.conv_4), 3, 1, 1, None, name=name + '.conv_4')
        P5 = g.conv(p5, *f(self.conv_5), 3, 1, 1, None, name=name + '.conv_5')
        P6 = g.conv(P5, *f(self.conv_out6), 3, 2, 1, None, name=name + '.conv_out6')
        P6r = g.conv(P5, *f(self.conv_out6), 3, 2, 1, 'relu', name=name + '.conv_out6.relu')   # input of conv_out7 is relu(P6)
        P7 = g.conv(P6r, *f(self.conv_out7), 3, 2, 1, None, name=name + '.conv_out7')
        return [P3, P4, P5, P6, P7]

    def forward(self, x):
        return [ops.split_to_nchw(o.view()) for o in self._run(x)]


# =============================================================================================== head
class ScaleExp(nn.Module):
    def __init__(self, init_value=1.0):
        super().__init__()
        self.scale = nn.Parameter(torch.tensor([init_value], dtype=torch.float32))


class FCOSHead(_Standalone):
    def __init__(self, num_classes, in_channel, GN=True, cnt_on_reg=True, prior=0.01):
        super().__init__()
        if not GN or not cnt_on_reg or in_channel % 8 != 0 or in_channel // 32 != 8:
            raise NotImplementedError('H100 FCOS head: GN=True, cnt_on_reg=True, 8 channels per group (in_channel=256)')
        self.num_classes, self.prior, self.cnt_on_reg = num_classes, prior, cnt_on_reg
        cls_branch, reg_branch = [], []
        for _ in range(4):
            cls_branch += [nn.Conv2d(in_channel, in_channel, 3, padding=1, bias=True), nn.GroupNorm(32, in_channel), nn.ReLU(True)]
            reg_branch += [nn.Conv2d(in_channel, in_channel, 3, padding=1, bias=True), nn.GroupNorm(32, in_channel), nn.ReLU(True)]
        self.cls_conv = nn.Sequential(*cls_branch)
        self.reg_conv = nn.Sequential(*reg_branch)
        self.cls_logits = nn.Conv2d(in_channel, num_classes, 3, padding=1)
        self.cnt_logits = nn.Conv2d(in_channel, 1, 3, padding=1)
        self.reg_pred = nn.Conv2d(in_channel, 4, 3, padding=1)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.normal_(m.weight, std=0.01)
                nn.init.constant_(m.bias, 0)
        nn.init.constant_(self.cls_logits.bias, -math.log((1 - prior) / prior))
        self.scale_exp = nn.ModuleList([ScaleExp(1.0) for _ in range(5)])

    def emit(self, g, levels, name='head'):
        """Returns per level (cls logits F32Tensor [B,h,w,>=nc], regcnt F32Tensor [B,h,w,8] = (l,t,r,b raw, cnt logit))."""
        gnws = ops.GroupNormWorkspace(g.B, 32, g.device)
        g.buffers.append(gnws)
        dev = g.device
        gn_params = {}
        for bname, seq in (('cls_conv', self.cls_conv), ('reg_conv', self.reg_conv)):
            for i in range(4):
                gn = seq[3 * i + 1]
                gn_params[(bname, i)] = (gn.weight.detach().float().to(dev).contiguous(), gn.bias.detach().float().to(dev).contiguous(), gn.eps)
        w_rc = torch.cat([self.reg_pred.weight.detach().double().cpu(), self.cnt_logits.weight.detach().double().cpu()], 0)
        b_rc = torch.cat([self.reg_pred.bias.detach().double().cpu(), self.cnt_logits.bias.detach().double().cpu()], 0)
        outs = []
        for li, P in enumerate(levels):
            feats = {}
            for bname, seq in (('cls_conv', self.cls_conv), ('reg_conv', self.reg_conv)):
                x = P
                for i in range(4):
                    y = g.conv(x, *folded(seq[3 * i]), 3, 1, 1, None, name=f'{name}.{bname}.{3 * i}.L{li}')
                    z = g.new_act(y.H, y.W, y.c)
                    gamma, beta, eps = gn_params[(bname, i)]
                    g.fn(lambda y=y, z=z, gamma=gamma, beta=beta, eps=eps: ops.groupnorm_relu(y.view(), 32, gamma, beta, eps, z.view(), gnws))
                    x = z
                feats[bname] = x
            cls = g.new_f32(P.H, P.W, (self.num_classes + 31) // 32 * 32)
            g.conv(feats['cls_conv'], *folded(self.cls_logits), 3, 1, 1, None, f32_out=cls, name=f'{name}.cls_logits.L{li}')
            rc = g.new_f32(P.H, P.W, 32)
            g.conv(feats['reg_conv'], w_rc, b_rc, 3, 1, 1, None, f32_out=rc, name=f'{name}.reg_cnt.L{li}')
            outs.append((cls, rc))
        return outs

    def forward(self, inputs):
        cls_l, cnt_l, reg_l = [], [], []
        for i, (cls, rc) in enumerate(self._run(inputs)):
            cls_l.append(ops.f32nhwc_to_nchw(cls.view(0, self.num_classes)))
            r = ops.f32nhwc_to_nchw(rc.view(0, 8))
            cnt_l.append(r[:, 4:5].contiguous())
            reg_l.append(torch.exp(r[:, 0:4] * self.scale_exp[i].scale.detach().to(r.device)))  # ScaleExp (boundary adapter only)
        return cls_l, cnt_l, reg_l


# =============================================================================================== detect
class FCOSDetect(nn.Module):
    def __init__(self, score_threshold, nms_iou_threshold, max_detection_boxes_num, strides):
        super().__init__()
        self.score_threshold = score_threshold
        self.nms_iou_threshold = nms_iou_threshold
        self.max_detection_boxes_num = max_detection_boxes_num
        self.strides = strides

    def emit(self, g, head_outs, num_classes, scales):
        N = sum(c.H * c.W for c, _ in head_outs)
        ws = ops.FcosWorkspace(g.B, N, min(self.max_detection_boxes_num, N), g.device)
        off = 0
        for (cls, rc), stride, sc in zip(head_outs, self.strides, scales):
            g.fn(lambda cls=cls, rc=rc, stride=stride, sc=sc, off=off: ops.fcos_decode(cls.view(0, num_classes), rc.view(0, 8), num_classes,
                                                                                        stride, sc, ws, off))
            off += cls.H * cls.W
        st, it = self.score_threshold, self.nms_iou_threshold
        g.fn(lambda: ops.fcos_nms(ws, st, it))
        return ws

    def forward(self, inputs):
        raise RuntimeError('FCOSDetect (H100): runs as part of the fused FCOS graph (call FCOS.forward / FCOS.predict)')


# =============================================================================================== factories + model
_BACKBONES = {'ResNet': ResNet}
_NECKS = {'FCOSFPN': FCOSFPN}
_HEADS = {'FCOSHead': FCOSHead}
_DETECTS = {'FCOSDetect': FCOSDetect}


def build_backbone(cfg):
    return _build(_BACKBONES, cfg)


def build_neck(cfg):
    return _build(_NECKS, cfg)


def build_head(cfg):
    return _build(_HEADS, cfg)


def build_detect(cfg):
    return _build(_DETECTS, cfg)


class FCOS(_Model):
    """Model-level drop-in for src.models.fcos.FCOS (inference path)."""

    def __init__(self, dictionary=None, model_cfg=None):
        super().__init__(dictionary, model_cfg)
        self.dummy_input = torch.zeros(1, 3, 800, 800)
        hcfg = dict(self._cfg('HEAD'))
        hcfg['num_classes'] = self.num_classes  # setup_extra_params (fcos.py:48-49)
        bcfg = dict(self._cfg('BACKBONE'))
        bcfg['pretrained'] = False  # no network on the box; weights come from load_state_dict
        self.backbone = build_backbone(bcfg)
        self.neck = build_neck(dict(self._cfg('NECK')))
        self.head = build_head(hcfg)
        self.detect = build_detect(dict(self._cfg('DETECT')))
        self.loss = None
        self.conf_thres = 0.05
        self.iou_thres = 0.6

    def build_graph(self, B, H, W, device):
        g = GraphBuilder(B, device)
        holder = {}
        feats = self.backbone.emit(g, lambda: holder['x'], H, W)
        levels = self.neck.emit(g, feats)
        head_outs = self.head.emit(g, levels)
        scales = [float(s.scale.detach()) for s in self.head.scale_exp]
        ws = self.detect.emit(g, head_outs, self.num_classes, scales)
        return dict(g=g, holder=holder, ws=ws, feats=feats, levels=levels, head=head_outs)

    def predict(self, imgs):
        """Device-only inference: (scores [B,K], classes [B,K] (1-based), boxes [B,K,4], loc [B,K], count [B]); no host sync.
        Graph-owned buffers (overwritten by the next call).  ``self._graph_for(imgs)['ws'].status[0] != 0`` flags a top-k
        capacity overflow of the last run; ``forward()`` checks it and raises."""
        ws = self._replay(imgs.contiguous().float())['ws']
        return ws.out_scores, ws.out_classes, ws.out_boxes, ws.out_loc, ws.out_count

    def _val(self, imgs, targets):
        """fcos.py:124-166: (losses, per-image {'boxes', 'labels', 'scores'})."""
        sc, cl, bx, _, cnt = self.predict(imgs)
        sc, cl, bx, cnt = sc.cpu(), cl.cpu(), bx.cpu(), cnt.cpu().tolist()
        if int(self._graph_for(imgs)['ws'].status[0]) != 0:
            raise _lib.CvbError('FCOS NMS: more than 4096 scores share the top-k threshold bin; the candidate set of this batch would be '
                                'truncated non-deterministically')
        img_h, img_w = imgs.shape[2:]
        outputs = []
        for i in range(imgs.shape[0]):
            k = cnt[i]
            t = targets[i] if targets is not None else {}
            b = bx[i, :k].clone()
            b[:, [0, 2]] = b[:, [0, 2]].clamp(min=0, max=img_h - 1)   # reference quirk: x clamped with img_h (fcos.py:141-142)
            b[:, [1, 3]] = b[:, [1, 3]].clamp(min=0, max=img_w - 1)
            scale = np.asarray(t['scales'].cpu() if 'scales' in t else [1.0, 1.0], dtype=np.float32)
            pad = np.asarray(t['pads'].cpu() if 'pads' in t else [0.0, 0.0], dtype=np.float32)
            width = float(t['width']) if 'width' in t else float(img_w)
            height = float(t['height']) if 'height' in t else float(img_h)
            bn = b.numpy()
            bn[:, [0, 2]] -= pad[1]
            bn[:, [1, 3]] -= pad[0]
            bn[:, [0, 2]] /= scale[1]
            bn[:, [1, 3]] /= scale[0]
            bn[:, [0, 2]] = bn[:, [0, 2]].clip(0, width)
            bn[:, [1, 3]] = bn[:, [1, 3]].clip(0, height)
            keep = sc[i, :k] > 0.05
            outputs.append({"boxes": torch.tensor(bn)[keep], "labels": cl[i, :k][keep].long(), "scores": sc[i, :k][keep]})
        return self._val_losses(imgs.device), outputs
