"""Drop-in modules for the YOLOX-s inference path (SURVEY.md 8 row a16; H100 fused graph, inference only).

Mirrors (paths relative to the reference checkout; the YAML route `conf/coco_yolox_s.yml` does not build in the reference --
SURVEY.md 3.5 row 3 -- so the drop-in follows the composite that does run):
  CSPDarknet   src/models/backbones/det/csp_darknet.py:25-129  (Focus stem `modules/yolo_modules.py:19-37`, CSPLayer :107-140,
               SPPF :165-194 with the parallel (5, 9, 13) pools == the chained 5x5 pools of the fused kernel)
  YOLOXNeck    src/models/necks/yolox_neck.py:13-74            (BaseConv / CSPLayer of `modules/yolox_modules.py:35-131`)
  YOLOXHead    src/models/heads/yolox_head.py:14-88            (ConvModule of `modules/convs.py`; the 1x1 stems carry padding=1,
               :35, so every head map is 2 pixels larger than its feature map: 82/42/22 at 640)
  YOLOX        src/models/yolox.py:71-187 ('val' branch :153-185) and yolox_post_process :18-68

`state_dict` keys and shapes equal the reference composite's (tests/golden/yolox_keys.npz).

Graph notes: Focus = the space-to-depth loader + a 3x3 conv in the row-window formulation of the YOLOv5 stem (weights
re-ordered from the reference's [tl, bl, tr, br] patch order); CSP blocks, zero-copy concats and the algebraic upsample+concat
fold are the YOLOv5 ones; per head level the first cls and reg 3x3 convs share one GEMM (N = 2 x 128), reg (4) and obj (1)
predictors share one fp32-output 1x1 GEMM, cls (80) is another; `cvb_yolox_decode` turns both into 8-float candidate records
and `cvb_yolox_nms` applies the score filter + torchvision.ops.batched_nms semantics per image."""
import numpy as np
import torch
import torch.nn as nn

from . import ops, train
from .engine import GraphBuilder
from .models import _YoloModel
from .modules import ConvModule, CSPLayer, SPPF, _build, _EmitModule, _emit_csp, _Standalone, folded


class Focus(_EmitModule):
    """yolo_modules.py:19-37: 2x2 space-to-depth ([tl, bl, tr, br] patches) followed by a ConvModule."""

    def __init__(self, in_channels, out_channels, kernel_sizes=1, stride=1, conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True),
                 act_cfg=dict(type='Swish')):
        super().__init__()
        if in_channels != 3 or kernel_sizes != 3 or stride != 1:
            raise NotImplementedError('Focus: only the 3-channel / 3x3 / stride-1 YOLOX stem is on the H100 hot path')
        self.conv = ConvModule(in_channels * 4, out_channels, kernel_sizes, stride, padding=(kernel_sizes - 1) // 2, conv_cfg=conv_cfg,
                               norm_cfg=norm_cfg, act_cfg=act_cfg)


def focus_weights_to_s2d(w64):
    """[O,12,3,3] Focus conv weights (reference patch order tl, bl, tr, br) -> [O,16,3,3] over the loader's space-to-depth
    channels (dy*2+dx)*3+c (tl, tr, bl, br; 4 zero pad channels)."""
    O, I, kh, kw = w64.shape
    assert (I, kh, kw) == (12, 3, 3)
    out = torch.zeros((O, 16, 3, 3), dtype=torch.float64)
    ref_to_mine = {0: 0, 1: 2, 2: 1, 3: 3}
    for gr, gm in ref_to_mine.items():
        out[:, gm * 3:gm * 3 + 3] = w64[:, gr * 3:gr * 3 + 3]
    return out


class CSPDarknet(_Standalone):
    cfg = {"n": [0.33, 0.25], "t": [0.33, 0.375], "s": [0.33, 0.5], "m": [0.67, 0.75], "l": [1.0, 1.0], "x": [1.33, 1.25]}

    def __init__(self, subtype='cspdark_s', out_channels=[64, 128, 256, 512, 1024], layers=[3, 9, 9, 3], spp_ksizes=(5, 9, 13),
                 depthwise=False, conv_cfg=None, norm_cfg=dict(type='BN', momentum=0.03, eps=0.001), act_cfg=dict(type='Swish'),
                 out_stages=[2, 3, 4], output_stride=32, backbone_path=None, pretrained=False, frozen_stages=-1, norm_eval=False):
        super().__init__()
        if depthwise:
            raise NotImplementedError('depthwise CSPDarknet is not on the H100 hot path')
        self.subtype, self.out_stages, self.output_stride = subtype, out_stages, output_stride
        depth_mul, width_mul = self.cfg[subtype.split('_')[1]]
        ch = list(map(lambda x: int(x * width_mul), out_channels))
        nl = list(map(lambda x: max(round(x * depth_mul), 1), layers))
        kw = dict(conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg)
        self.stem = Focus(3, ch[0], kernel_sizes=3, **kw)
        self.stage1 = nn.Sequential(ConvModule(ch[0], ch[1], 3, 2, padding=1, **kw), CSPLayer(ch[1], ch[1], n=nl[0], shortcut=True, **kw))
        self.stage2 = nn.Sequential(ConvModule(ch[1], ch[2], 3, 2, padding=1, **kw), CSPLayer(ch[2], ch[2], n=nl[1], shortcut=True, **kw))
        self.stage3 = nn.Sequential(ConvModule(ch[2], ch[3], 3, 2, padding=1, **kw), CSPLayer(ch[3], ch[3], n=nl[2], shortcut=True, **kw))
        self.stage4 = nn.Sequential(ConvModule(ch[3], ch[4], 3, 2, padding=1, **kw), SPPF(ch[4], ch[4], kernel_sizes=spp_ksizes, **kw),
                                    CSPLayer(ch[4], ch[4], n=nl[3], shortcut=False, **kw))
        self.out_channels = ch[out_stages[0]:out_stages[-1] + 1]
        for m in self.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.eps, m.momentum = 1e-3, 0.03

    def emit(self, g, img_getter, H, W, name='backbone', u8_norm=None):
        x0 = g.new_act(H // 2, W // 2 + 3, 16)  # zero-padded row-window layout, see YOLOv5CSPDarknet.emit
        g.fn(lambda: ops.stem_s2d(img_getter(), x0.view(), norm=u8_norm))
        w, b = folded(self.stem.conv.conv, self.stem.conv.bn)
        x = g.conv(x0, focus_weights_to_s2d(w), b, 3, 1, 1, 'silu', name=name + '.stem', w_window=4)
        outs = []
        for i in range(1, 5):
            stage = getattr(self, f'stage{i}')
            for j, m in enumerate(stage):
                x = m.emit(g, x, f'{name}.stage{i}.{j}')
            if i in self.out_stages:
                outs.append(x)
        return outs

    def forward(self, x):
        return self._run_image(x)


class BaseConv(ConvModule):
    """yolox_modules.py:35-58: conv (pad = (k-1)//2, no bias) + BN + SiLU; same keys as ConvModule."""

    def __init__(self, in_channels, out_channels, ksize, stride, groups=1, bias=False, act='silu'):
        if act != 'silu' or groups != 1 or bias:
            raise NotImplementedError('BaseConv variant not on the H100 hot path')
        super().__init__(in_channels, out_channels, ksize, stride, padding=(ksize - 1) // 2, norm_cfg=dict(type='BN', eps=1e-3, momentum=0.03),
                         act_cfg=dict(type='SiLU'))


class XBottleneck(_EmitModule):
    """yolox_modules.py:79-96."""

    def __init__(self, in_channels, out_channels, shortcut=True, expansion=0.5, act='silu'):
        super().__init__()
        hidden = int(out_channels * expansion)
        self.conv1 = BaseConv(in_channels, hidden, 1, stride=1, act=act)
        self.conv2 = BaseConv(hidden, out_channels, 3, stride=1, act=act)
        self.use_add = shortcut and in_channels == out_channels


class XCSPLayer(_EmitModule):
    """yolox_modules.py:99-131 (keys conv1/conv2/conv3/m.N.conv1/conv2, as yolo_modules.CSPLayer)."""

    def __init__(self, in_channels, out_channels, n=1, shortcut=True, expansion=0.5, depthwise=False, act='silu'):
        super().__init__()
        if depthwise:
            raise NotImplementedError('depthwise CSPLayer is not on the H100 hot path')
        hidden = int(out_channels * expansion)
        self.conv1 = BaseConv(in_channels, hidden, 1, stride=1, act=act)
        self.conv2 = BaseConv(in_channels, hidden, 1, stride=1, act=act)
        self.conv3 = BaseConv(2 * hidden, out_channels, 1, stride=1, act=act)
        self.m = nn.Sequential(*[XBottleneck(hidden, hidden, shortcut, 1.0, act=act) for _ in range(n)])

    def emit(self, g, x, name='', up_src=None, out=None):
        blocks = [(b.conv1, b.conv2) for b in self.m]
        sc = all(b.use_add for b in self.m) if len(self.m) else False
        return _emit_csp(g, x, self.conv1, self.conv2, self.conv3, blocks, sc, name, up_src=up_src, out=out)


class YOLOXNeck(_Standalone):
    def __init__(self, subtype='yolox_s', channels=[256, 512, 1024], depth_mul=1.0, width_mul=1.0):
        super().__init__()
        assert isinstance(channels, list)
        self.subtype, self.channels = subtype, channels
        c = list(map(lambda x: max(round(x * width_mul), 1), channels))
        n = list(map(lambda x: max(round(x * depth_mul), 1), [3, 3, 3, 3]))
        self.upsample = nn.Upsample(scale_factor=2, mode='nearest')
        self.lateral_conv0 = BaseConv(c[2], c[1], 1, 1)
        self.C3_p4 = XCSPLayer(2 * c[1], c[1], n[0], False)
        self.reduce_conv1 = BaseConv(c[1], c[0], 1, 1)
        self.C3_p3 = XCSPLayer(2 * c[0], c[0], n[1], False)
        self.bu_conv2 = BaseConv(c[0], c[0], 3, 2)
        self.C3_n3 = XCSPLayer(2 * c[0], c[1], n[2], False)
        self.bu_conv1 = BaseConv(c[1], c[1], 3, 2)
        self.C3_n4 = XCSPLayer(2 * c[1], c[2], n[3], False)

    def emit(self, g, feats, name='neck'):
        x2, x1, x0 = feats
        c1, c0 = self.lateral_conv0.out_channels, self.reduce_conv1.out_channels
        cat1 = g.new_act(x1.H, x1.W, 2 * c0)   # [bu_conv2(pan_out2) | fpn_out1]   (yolox_neck.py:63-64)
        cat0 = g.new_act(x0.H, x0.W, 2 * c1)   # [bu_conv1(pan_out1) | fpn_out0]   (:67-68)
        fpn_out0 = self.lateral_conv0.emit(g, x0, name + '.lateral_conv0', out=cat0.slice(c1, c1))
        f_out0 = self.C3_p4.emit(g, x1, name + '.C3_p4', up_src=fpn_out0)          # cat([up(fpn_out0), x1]) folded (:53-55)
        fpn_out1 = self.reduce_conv1.emit(g, f_out0, name + '.reduce_conv1', out=cat1.slice(c0, c0))
        pan_out2 = self.C3_p3.emit(g, x2, name + '.C3_p3', up_src=fpn_out1)
        self.bu_conv2.emit(g, pan_out2, name + '.bu_conv2', out=cat1.slice(0, c0))
        pan_out1 = self.C3_n3.emit(g, cat1, name + '.C3_n3')
        self.bu_conv1.emit(g, pan_out1, name + '.bu_conv1', out=cat0.slice(0, c1))
        pan_out0 = self.C3_n4.emit(g, cat0, name + '.C3_n4')
        return [pan_out2, pan_out1, pan_out0]

    def forward(self, x):
        assert len(x) == len(self.channels)
        return [ops.split_to_nchw(o.view()) for o in self._run(x)]


class HeadConv(ConvModule):
    """modules/convs.py ConvModule as used by heads/yolox_head.py:34-49 (conv without bias + BN + SiLU)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, activation='SiLU'):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding=padding, norm_cfg=dict(type='BN', eps=1e-3, momentum=0.03),
                         act_cfg=dict(type=activation))


class YOLOXHead(_Standalone):
    def __init__(self, num_classes=80, subtype='yolox_s', in_channels=[256, 512, 1024], strides=[8, 16, 32], depth_mul=1.0, width_mul=1.0):
        super().__init__()
        self.num_classes, self.subtype, self.strides, self.n_anchors = num_classes, subtype, strides, 1
        ic = list(map(lambda x: max(round(x * width_mul), 1), in_channels))
        p = int(256 * width_mul)
        self.stems, self.cls_convs, self.reg_convs = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        self.cls_preds, self.reg_preds, self.obj_preds = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        for c in ic:
            self.stems.append(HeadConv(c, p, 1, 1, padding=1))  # padding=1 on a 1x1 conv: heads/yolox_head.py:35
            self.cls_convs.append(nn.Sequential(HeadConv(p, p, 3, 1, 1), HeadConv(p, p, 3, 1, 1)))
            self.reg_convs.append(nn.Sequential(HeadConv(p, p, 3, 1, 1), HeadConv(p, p, 3, 1, 1)))
            self.cls_preds.append(nn.Conv2d(p, self.n_anchors * num_classes, 1, 1, 0))
            self.reg_preds.append(nn.Conv2d(p, 4, 1, 1, 0))
            self.obj_preds.append(nn.Conv2d(p, self.n_anchors * 1, 1, 1, 0))
        prior = -float(np.log((1 - 1e-2) / 1e-2))  # heads/yolox_head.py:54-72
        for conv in list(self.cls_preds) + list(self.obj_preds):
            nn.init.constant_(conv.bias, prior)

    def level_shapes(self, feats):
        return [(f.H + 2, f.W + 2) for f in feats]

    def num_candidates(self, feats):
        return sum(h * w for h, w in self.level_shapes(feats))

    def emit(self, g, feats, name='head'):
        """Returns per level (reg_obj fp32 [B,h,w,8] (5 used: reg 4, obj 1), cls fp32 [B,h,w,96] (num_classes used))."""
        outs = []
        for k, f in enumerate(feats):
            xx = self.stems[k].emit(g, f, f'{name}.stems.{k}')  # map grows by 2 (padding=1, 1x1)
            c0, r0 = self.cls_convs[k][0], self.reg_convs[k][0]
            wc, bc = folded(c0.conv, c0.bn)
            wr, br = folded(r0.conv, r0.bn)
            p = wc.shape[0]
            both = g.conv(xx, torch.cat([wc, wr], 0), torch.cat([bc, br], 0), 3, 1, 1, 'silu', name=f'{name}.cls_reg_convs.{k}.0')
            cls_feat = self.cls_convs[k][1].emit(g, both.slice(0, p), f'{name}.cls_convs.{k}.1')
            reg_feat = self.reg_convs[k][1].emit(g, both.slice(p, p), f'{name}.reg_convs.{k}.1')
            cls_out = g.new_f32(xx.H, xx.W, (self.num_classes + 31) // 32 * 32)
            g.conv(cls_feat, *folded(self.cls_preds[k]), 1, 1, 0, None, f32_out=cls_out, name=f'{name}.cls_preds.{k}')
            wro = torch.cat([self.reg_preds[k].weight.detach().double(), self.obj_preds[k].weight.detach().double()], 0)
            bro = torch.cat([self.reg_preds[k].bias.detach().double(), self.obj_preds[k].bias.detach().double()], 0)
            ro_out = g.new_f32(xx.H, xx.W, 32)
            g.conv(reg_feat, wro, bro, 1, 1, 0, None, f32_out=ro_out, name=f'{name}.reg_obj_preds.{k}')
            outs.append((ro_out, cls_out))
        return outs

    def forward(self, x):
        """list of NCHW CUDA feature maps -> list of [B, 5 + num_classes, h+2, w+2] raw outputs (reg, obj, cls), as the reference."""
        return [torch.cat([ops.f32nhwc_to_nchw(ro.view(0, 5)), ops.f32nhwc_to_nchw(cl.view(0, self.num_classes))], 1)
                for ro, cl in self._run(x)]


_BACKBONES = {'CSPDarknet': CSPDarknet, 'CspDarkNet': CSPDarknet}
_NECKS = {'YOLOXNeck': YOLOXNeck}
_HEADS = {'YOLOXHead': YOLOXHead}


def build_backbone(cfg):
    return _build(_BACKBONES, cfg)


def build_neck(cfg):
    return _build(_NECKS, cfg)


def build_head(cfg):
    return _build(_HEADS, cfg)


class YOLOX(_YoloModel):
    """Model-level drop-in for src.models.yolox.YOLOX: mode='val' runs the cached inference graph (eval()), mode='train' the training
    kernels and the YOLOXLoss (train()) over the same parameters."""
    cfg = {"nano": [0.33, 0.25], "tiny": [0.33, 0.375], "s": [0.33, 0.5], "m": [0.67, 0.75], "l": [1.0, 1.0], "x": [1.33, 1.25]}
    input_norm = dict(mean=(0.406, 0.456, 0.485), std=(0.225, 0.224, 0.229), reverse_channels=True)
    _parts = ('backbone', 'neck', 'head')

    def __init__(self, dictionary=None, model_cfg=None):
        super().__init__(dictionary, model_cfg)
        self.dummy_input = torch.zeros(1, 3, 640, 640)
        self.depth_mul, self.width_mul = self.cfg[self._cfg('TYPE').split('_')[1]]
        bcfg = dict(self._cfg('BACKBONE'))
        bcfg.pop('depth_mul', None)
        bcfg.pop('width_mul', None)
        bcfg['pretrained'] = False
        if bcfg.get('name') == 'CspDarkNet' and 'subtype' not in bcfg:
            bcfg['subtype'] = self._cfg('TYPE')  # the composite of SURVEY.md 3.5: CSPDarknet(subtype='yolox_s')
        ncfg = dict(self._cfg('NECK'), depth_mul=self.depth_mul, width_mul=self.width_mul)
        hcfg = dict(self._cfg('HEAD'), depth_mul=self.depth_mul, width_mul=self.width_mul, num_classes=self.num_classes)
        self.backbone = build_backbone(bcfg)
        self.neck = build_neck(ncfg)
        self.head = build_head(hcfg)
        self.stride = [8, 16, 32]
        self.conf_thr, self.nms_thr = 0.01, 0.65   # src/models/yolox.py:94-95
        lcfg = dict(self._loss_cfg('YOLOXLoss'), num_classes=self.num_classes)
        self.loss = train.YOLOXLoss(**lcfg)  # (no parameters or buffers: the state_dict keys stay the inference model's)
        # the training modules (train.CSPDarknet / YOLOXNeck / YOLOXHead), built on the first training forward over this model's own
        # parameters and buffers; kept out of the module tree so that state_dict(), parameters() and .to() see each tensor once
        self.__dict__['_train_modules'] = None
        self._cfgs = (bcfg, ncfg, hcfg)

    def build_graph(self, B, H, W, device, u8_input=False):
        g = GraphBuilder(B, device)
        holder = {}
        feats = self.backbone.emit(g, lambda: holder['x'], H, W, u8_norm=dict(self.input_norm) if u8_input else None)
        feats = self.neck.emit(g, feats)
        outs = self.head.emit(g, feats)
        A = sum(ro.H * ro.W for ro, _ in outs)
        ws = ops.YoloxWorkspace(B, A, device=device)
        off = 0
        for (ro, cl), s in zip(outs, self.stride):
            g.fn(lambda ro=ro, cl=cl, s=s, off=off: ops.yolox_decode(ro.view(0, 5), cl.view(0, self.num_classes), self.num_classes, float(s), ws, off))
            off += ro.H * ro.W
        g.fn(lambda: ops.yolox_nms(ws, self.conf_thr, self.nms_thr))
        return dict(g=g, holder=holder, outs=outs, ws=ws)

    def predict(self, imgs):
        """Device-only inference: (det [B,A,7] rows (x1,y1,x2,y2,obj,class_conf,class_pred) in kept order, count [B]); no host sync."""
        ws = self._replay(imgs.contiguous().float())['ws']
        return ws.det, ws.count

    def _build_training_parts(self):
        """(train.CSPDarknet, train.YOLOXNeck, train.YOLOXHead); the training kernels refuse YOLOX-t, -m and -x."""
        strip = lambda c: {k: v for k, v in c.items() if k != 'name'}  # noqa: E731
        bcfg, ncfg, hcfg = self._cfgs
        return train.CSPDarknet(**strip(bcfg)), train.YOLOXNeck(**strip(ncfg)), train.YOLOXHead(**strip(hcfg))

    def pack_targets(self, imgs, targets):
        """trans_specific_format (yolox.py:112-139): the per-image target dicts -> gt [B, max_labels, 5] rows (label, box) on the images'
        device, zero rows after each image's boxes.  A [B, max_labels, 5] tensor is taken as already packed."""
        if isinstance(targets, torch.Tensor):
            return targets
        max_labels = max(t['labels'].shape[0] for t in targets)
        gt = torch.zeros((len(targets), max_labels, 5), device=imgs.device)
        for i, t in enumerate(targets):
            n = t['labels'].shape[0]
            gt[i, :n, 0] = t['labels'].to(imgs.device, torch.float32)
            gt[i, :n, 1:] = t['boxes'].to(imgs.device, torch.float32)
        return gt

    def _loss_step(self, outputs, gt):
        """yolox.py:150-157, 186-187: the loss dict {loss, conf_loss, cls_loss, iou_loss, num_fg}."""
        return self.loss(outputs, gt)

    def _val(self, imgs, targets):
        det, cnt = self.predict(imgs)
        # yolox.py:165-178 on the device, then ONE device->host copy of the kept prefix
        kmax = max(int(cnt.max()), 1)
        det_h, cnt_h = ops.val_rows_to_host(det[:, :kmax].contiguous(), cnt, targets, imgs.shape[2:])
        outputs = []
        for i in range(det_h.shape[0]):
            pred = det_h[i, :cnt_h[i]]
            if pred.shape[0] == 0:  # yolox.py:182-184
                outputs.append({"boxes": torch.empty((0, 4)), "labels": torch.empty((0, 1)), "scores": torch.empty((0, 1))})
                continue
            outputs.append({"boxes": pred[:, :4].clone(), "labels": pred[:, 6], "scores": pred[:, 4] * pred[:, 5]})
        return self._val_losses(imgs.device), outputs
