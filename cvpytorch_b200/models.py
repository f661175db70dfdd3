"""Drop-in backbone / neck / detect / model modules for the YOLOv5 path (reference surface kept).

Mirrors (paths relative to the reference checkout):
  YOLOv5CSPDarknet   src/models/backbones/det/yolov5_csp_darknet.py:17-120 (+ det/base_yolo_backbone.py:16-113)
  YOLOv5Neck         src/models/necks/yolov5_neck.py:12-51   (the runnable old-API neck, SURVEY.md §3.5)
  YOLOv5Detect       src/models/detects/yolov5_detect.py:12-65
  YOLOv5             src/models/yolov5.py:156-287  (+ non_max_suppression :62-153)
  build_*            src/models/{backbones,necks,detects}/__init__.py factories

Component modules accept/return the reference's NCHW fp32 tensors (adapter kernels at the boundary); the
model-level module runs ONE fused graph end to end (split-NHWC internally, decode + batched NMS on device).
"""
import math
import os
from copy import deepcopy

import torch
import torch.nn as nn

from . import _lib, ops, train, yolov5_train
from .engine import GraphBuilder
from .modules import ConvModule, CSPLayer, DownsamplingModule, SPPF, UpsamplingModule, _build, _Model, _Standalone, folded


# =============================================================================================== backbone
class YOLOv5CSPDarknet(_Standalone):
    cfg = {"n": [0.33, 0.25], "t": [0.33, 0.375], "s": [0.33, 0.5], "m": [0.67, 0.75], "l": [1.0, 1.0], "x": [1.33, 1.25]}

    def __init__(self, subtype='cspdark_s', in_channels=3, out_channels=[64, 128, 256, 512, 1024], num_blocks=[3, 6, 9, 3],
                 spp_ksizes=5, depthwise=False, conv_cfg=None, norm_cfg=dict(type='BN', momentum=0.03, eps=0.001),
                 act_cfg=dict(type='SiLU', inplace=True), out_stages=[2, 3, 4], output_stride=32, backbone_path=None,
                 pretrained=False, frozen_stages=-1, norm_eval=False, **unused):
        super().__init__()
        if depthwise:
            raise NotImplementedError('depthwise YOLOv5 backbone is not on the H100 hot path')
        self.subtype = subtype
        self.out_stages = out_stages
        depth_mul, width_mul = self.cfg[subtype.split("_")[1]]
        self.out_channels = list(map(lambda x: int(x * width_mul), out_channels))
        self.num_blocks = list(map(lambda x: max(round(x * depth_mul), 1), num_blocks))
        self.in_channels = in_channels
        if in_channels != 3:
            raise NotImplementedError('stem expects 3 input channels')
        kw = dict(norm_cfg=norm_cfg, act_cfg=act_cfg)
        self.stem = ConvModule(in_channels, self.out_channels[0], kernel_size=6, stride=2, padding=2, **kw)
        for idx, (cin, cout, n) in enumerate(zip(self.out_channels[:-1], self.out_channels[1:], self.num_blocks)):
            stage = [ConvModule(cin, cout, kernel_size=3, stride=2, padding=1, **kw),
                     CSPLayer(cout, cout, n=n, shortcut=False if idx == 3 else True, **kw)]
            if idx == 3:
                stage.append(SPPF(cout, cout, kernel_sizes=spp_ksizes, **kw))
            self.add_module(f'stage{idx + 1}', nn.Sequential(*stage))
        self.init_weights()

    def init_weights(self):
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_uniform_(m.weight, a=math.sqrt(5))
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, nn.BatchNorm2d):
                m.eps = 1e-3
                m.momentum = 0.03

    def emit(self, g, img_nchw_getter, H, W, name='backbone', u8_norm=None):
        """img_nchw_getter() -> contiguous fp32 CUDA tensor [B,3,H,W] at run time (or uint8 [B,H,W,3] frames when the graph was
        built with ``u8_norm`` = ToTensor/Normalize constants, see ops.stem_s2d).  Returns list of Val."""
        # space-to-depth input in the zero-padded "row window" layout: one 128-byte K chunk = 4 adjacent s2d pixels
        x0 = g.new_act(H // 2, W // 2 + 3, 16)
        g.fn(lambda: ops.stem_s2d(img_nchw_getter(), x0.view(), norm=u8_norm))
        w, b = folded(self.stem.conv, self.stem.bn)
        x = g.conv(x0, ops.stem_weights_to_s2d(w), b, 3, 1, 1, 'silu', name=name + '.stem', w_window=4)
        outs = []
        for i in range(1, 5):
            stage = getattr(self, f'stage{i}')
            x = stage[0].emit(g, x, f'{name}.stage{i}.0')
            x = stage[1].emit(g, x, f'{name}.stage{i}.1')
            if len(stage) > 2:
                x = stage[2].emit(g, x, f'{name}.stage{i}.2')
            if i in self.out_stages:
                outs.append(x)
        return outs

    def forward(self, x):
        return self._run_image(x)


# =============================================================================================== neck
class YOLOv5Neck(_Standalone):
    def __init__(self, in_channels, out_channels, depth_mul=1.0, width_mul=1.0, **unused):
        super().__init__()
        assert isinstance(in_channels, list)
        self.in_channels = list(map(lambda x: max(round(x * width_mul), 1), in_channels))
        self.out_channels = list(map(lambda x: max(round(x * width_mul), 1), out_channels))
        layers = [3, 3, 3, 3]
        self.layers = list(map(lambda x: max(round(x * depth_mul), 1), layers))
        self.up_1 = UpsamplingModule(self.in_channels[2], self.in_channels[1], self.layers[0])
        self.up_2 = UpsamplingModule(self.in_channels[1], self.out_channels[0], self.layers[1])
        self.down_1 = DownsamplingModule(self.in_channels[0], self.in_channels[1], self.layers[2])
        self.down_2 = DownsamplingModule(self.in_channels[1], self.in_channels[2], self.layers[3])
        for m in self.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.eps = 1e-3
                m.momentum = 0.03

    def emit(self, g, feats, name='neck'):
        x3, x4, x5 = feats
        c1 = self.down_1.down.conv.out_channels  # lateral channels of level 4 -> concat at 1/16
        c2 = self.down_2.down.conv.out_channels
        cat1 = g.new_act(x4.H, x4.W, 2 * c1)   # [down_1(x3_up) | x3_t]
        cat2 = g.new_act(x5.H, x5.W, 2 * c2)   # [down_2(x4_down) | x4_t]
        x4_up, _ = self.up_1.emit(g, x5, x4, name + '.up_1', lateral_out=cat2.slice(c2, c2))
        x3_up, _ = self.up_2.emit(g, x4_up, x3, name + '.up_2', lateral_out=cat1.slice(c1, c1))
        x4_down = self.down_1.emit(g, x3_up, cat1, name + '.down_1')
        x5_down = self.down_2.emit(g, x4_down, cat2, name + '.down_2')
        return [x3_up, x4_down, x5_down]

    def forward(self, x):
        assert len(x) == len(self.in_channels)
        return [ops.split_to_nchw(o.view()) for o in self._run(x)]


# =============================================================================================== detect
class YOLOv5Detect(_Standalone):
    def __init__(self, num_classes=80, in_channels=[256, 512, 1024], stride=[8., 16., 32.], anchors=(), depth_mul=1.0, width_mul=1.0):
        super().__init__()
        in_channels = list(map(lambda x: int(x * width_mul), in_channels))
        self.num_classes = num_classes
        self.num_outputs = num_classes + 5
        self.num_layers = len(anchors)
        self.num_anchors = len(anchors[0])
        self.stride = stride
        self.register_buffer('anchors', torch.tensor(anchors).float())
        self.m = nn.ModuleList(nn.Conv2d(x, self.num_outputs * self.num_anchors, 1) for x in in_channels)
        self.init_weight()

    def init_weight(self, cf=None):
        for mi, s in zip(self.m, self.stride):
            b = mi.bias.view(self.num_anchors, -1)
            b.data[:, 4] += math.log(8 / (640 / s) ** 2)
            b.data[:, 5:] += math.log(0.6 / (self.num_classes - 0.999999)) if cf is None else torch.log(cf / cf.sum())
            mi.bias = torch.nn.Parameter(b.view(-1), requires_grad=True)

    def num_candidates(self, feats):
        return sum(self.num_anchors * f.H * f.W for f in feats)

    def emit(self, g, feats, name='detect', want_raw=True, nms_ws=None, conf_thres=0.001, multi_label=True):
        """Returns (z tensor [B, A, no] fp32 on device, [raw_i [B,na,ny,nx,no]] or None).
        nms_ws: the decode kernels also accumulate the NMS score histogram into this workspace (fused count pass)."""
        na, no = self.num_anchors, self.num_outputs
        A = self.num_candidates(feats)
        dev = g.device
        z = torch.zeros((g.B, A, no), dtype=torch.float32, device=dev)
        raws = []
        off = 0
        if nms_ws is not None:
            g.fn(lambda: ops.nms_reset(nms_ws))
        fused = (not want_raw) and no <= 85 and na <= 4 and all(f.c % 32 == 0 for f in feats) and os.environ.get('CVB_FUSED_DECODE', '1') != '0'
        for i, f in enumerate(feats):
            if fused:
                # the decode IS the conv's epilogue: z rows + NMS histogram / rowmax straight from the accumulator (no raw tensor, one launch)
                w, b = folded(self.m[i])
                anchors_px = self.anchors[i].detach().float().cpu() * float(self.stride[i])
                g.conv_yolo_head(f, w, b, na, no, anchors_px, float(self.stride[i]), z, A, off, nms_ws, conf_thres, multi_label,
                                 name=f'{name}.m.{i}')
                off += na * f.H * f.W
                continue
            cpitch = (na * no + 31) // 32 * 32
            raw = g.new_f32(f.H, f.W, cpitch)
            w, b = folded(self.m[i])
            g.conv(f, w, b, 1, 1, 0, None, f32_out=raw, name=f'{name}.m.{i}')
            anchors_px = (self.anchors[i].detach().float().cpu() * float(self.stride[i])).to(dev).contiguous()
            xp = torch.zeros((g.B, na, f.H, f.W, no), dtype=torch.float32, device=dev) if want_raw else None
            raws.append(xp)
            g.fn(lambda raw=raw, anchors_px=anchors_px, s=float(self.stride[i]), off=off, xp=xp:
                 ops.yolo_decode(raw.view(0, na * no), na, no, anchors_px, s, z, A, off, xp, nms_ws, conf_thres, multi_label))
            off += na * f.H * f.W
        g.buffers.append(z)
        return z, (raws if want_raw else None)

    def forward(self, x):
        z, raws = self._run(x)
        for i in range(len(x)):  # the reference replaces the list entries in place (yolov5_detect.py:42-44)
            x[i] = raws[i]
        return z, x


# =============================================================================================== factories
_BACKBONES = {'YOLOv5CSPDarknet': YOLOv5CSPDarknet, 'YOLOv5Backbone': YOLOv5CSPDarknet}
_NECKS = {'YOLOv5Neck': YOLOv5Neck}
_DETECTS = {'YOLOv5Detect': YOLOv5Detect}


def build_backbone(cfg):
    """src/models/backbones/__init__.py:61-134 contract: deepcopy, pop 'name', Class(**cfg); unknown -> NotImplementedError.
    'YOLOv5Backbone' (the name conf/coco_yolov5_s.yml:68 uses but the reference factory lacks) maps to YOLOv5CSPDarknet."""
    c = deepcopy(dict(cfg))
    if c.get('name') == 'YOLOv5Backbone':
        c.setdefault('subtype', 'yolov5_s')
        c.pop('depth_mul', None)
        c.pop('width_mul', None)
    elif c.get('name') == 'YOLOv5CSPDarknet':
        c.pop('depth_mul', None)   # injected by YOLOv5.setup_extra_params (yolov5.py:207-208), not a ctor arg
        c.pop('width_mul', None)
    return _build(_BACKBONES, c)


def build_neck(cfg):
    return _build(_NECKS, cfg)


def build_detect(cfg):
    return _build(_DETECTS, cfg)


# =============================================================================================== model
def non_max_suppression(prediction, conf_thres=0.25, iou_thres=0.45, classes=None, agnostic=False, multi_label=False,
                        labels=(), max_det=300, workspace=None, return_indices=False):
    """Device-side replacement of src/models/yolov5.py:62-153 with the same signature / return type
    (list of [n,6] tensors xyxy, conf, cls).  `classes`/`labels` (unused by the reference's callers) are not supported."""
    if classes is not None or labels:
        raise NotImplementedError('classes= / labels= filters are not on the H100 hot path')
    B, A, no = prediction.shape
    ws = workspace if workspace is not None else ops.NmsWorkspace(B, A, no - 5, max_det=max_det, device=prediction.device)
    det, idx, cnt = ops.yolo_nms(prediction.contiguous(), ws, conf_thres, iou_thres, multi_label, max_wh=0.0 if agnostic else 4096.0)
    cnt_h = cnt.cpu().tolist()  # the only host sync: the API returns variable-length tensors
    if int(ws.status[0]) != 0:
        raise _lib.CvbError('NMS candidate capacity overflow')
    out = [det[b, :cnt_h[b]] for b in range(B)]
    if return_indices:
        return out, [idx[b, :cnt_h[b]] for b in range(B)]
    return out


class _YoloModel(_Model):
    """What the YOLO drop-ins share: the training forward (YOLOv5, YOLOX, YOLOv6) and, for the ones whose cached graph ends in ops.yolo_nms
    (YOLOv5, YOLOv6), ``predict``, ``nms_status`` and the post-processing of forward(mode='val').  A trainer defines ``_parts`` (the names of
    its inference modules), ``_build_training_parts()`` (their training modules) and ``_loss_step(outputs, targets)``.  YOLOX replaces
    ``pack_targets``, ``predict`` and ``_val``; its graph ends in ops.yolox_nms, which has no status word, so ``nms_status`` does not apply."""

    def _loss_cfg(self, name):
        """The LOSS section's constructor arguments (the model's own loss when the section is missing); another loss raises NotImplementedError."""
        lcfg = dict(self._cfg('LOSS', None) or {'name': name})
        if lcfg.pop('name', name) != name:
            raise NotImplementedError(f'{type(self).__name__} (H100): only the {name} is on the training path')
        return lcfg

    @staticmethod
    def pack_targets(imgs, targets):
        """trans_specific_format (yolov5.py:221-245, detectors/yolo_detector.py:23-50): the per-image target dicts -> gts [nt, 6] rows (image, label, cx, cy, w, h) on the
        images' device.  A tensor is taken as already packed."""
        if isinstance(targets, torch.Tensor):
            return targets
        rows = [torch.cat([torch.full((t['labels'].shape[0], 1), float(i), device=imgs.device), t['labels'].to(imgs.device, torch.float32).view(-1, 1),
                           t['boxes'].to(imgs.device, torch.float32).view(-1, 4)], 1) for i, t in enumerate(targets)]
        return torch.cat(rows, 0) if rows else torch.zeros((0, 6), device=imgs.device)

    def _training_modules(self):
        """The training modules of ``_parts`` over this model's own parameters, buffers and BatchNorm modules (train.bound_training_modules).
        Widths the training kernels refuse raise NotImplementedError."""
        return train.bound_training_modules(self, tuple(getattr(self, p) for p in self._parts), self._build_training_parts)

    def forward_train(self, imgs, targets):
        """The reference's training forward on the H100 training kernels: backbone -> neck -> head over this model's parameters, then
        ``_loss_step`` (device tensors, no host sync)."""
        name = type(self).__name__
        if not self.training:
            raise RuntimeError(f"{name} (H100): mode='train' runs the training kernels (batch statistics); call .train() first")
        if not imgs.is_cuda:
            raise _lib.CvbError(f'{name} (H100) training: CUDA images required (the training path has no CPU fallback)')
        gts = self.pack_targets(imgs, targets)
        bb, nk, hd = self._training_modules()
        return self._loss_step(hd.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(imgs))), gts)

    def predict(self, imgs):
        """Device-only inference: returns (det [B,max_det,6] (x1,y1,x2,y2,conf,cls), det_idx [B,max_det] (row*nc + cls), det_count [B])
        device tensors, no host sync.  The tensors are the GRAPH-OWNED output buffers (overwritten by the next call with the same shape).
        ``nms_status(imgs)`` returns the device status word of the last run ([0] != 0: the NMS candidate capacity overflowed and the
        result is invalid); ``forward()`` checks it and raises."""
        ws = self._replay(imgs.contiguous().float())['ws']
        return ws.det, ws.det_idx, ws.det_count

    def nms_status(self, imgs):
        """Device int32[4] status of the NMS stage of the graph that serves `imgs` ([0] = candidate-capacity overflow flag)."""
        return self._graph_for(imgs)['ws'].status

    def _val(self, imgs, targets):
        """forward(imgs, targets, 'val'): (losses, per-image {'boxes', 'labels', 'scores'}) with the boxes rescaled and clipped to each
        image's original geometry, as the reference (yolov5.py:258-282, yolov6.py:209-227)."""
        det, _, cnt = self.predict(imgs)
        det_h, cnt_h = ops.val_rows_to_host(det.clone(), cnt, targets, imgs.shape[2:])
        if int(self.nms_status(imgs)[0]) != 0:  # (the copy above already synchronised)
            raise _lib.CvbError(f'{type(self).__name__} NMS: candidate capacity overflow (more keys in the threshold bin than the workspace '
                                'holds); the detections of this batch would be truncated non-deterministically')
        outputs = []
        for b in range(det_h.shape[0]):
            pred = det_h[b, :cnt_h[b]]
            outputs.append({"boxes": pred[:, :4].clone(), "labels": pred[:, 5], "scores": pred[:, 4]})
        return self._val_losses(imgs.device), outputs


class YOLOv5(_YoloModel):
    """Model-level drop-in for src.models.yolov5.YOLOv5.  forward(imgs, targets, mode) keeps the reference contract: mode 'val' (eval()) ->
    (losses_dict, outputs list of {'boxes','labels','scores'}) from the cached inference graph; mode 'train' (train()) -> the loss dict
    {'loss', 'box_loss', 'obj_loss', 'cls_loss'} from the training kernels and the YOLOv5Loss over the same parameters."""
    anchors = [[[1.25000, 1.62500], [2.00000, 3.75000], [4.12500, 2.87500]],
               [[1.87500, 3.81250], [3.87500, 2.81250], [3.68750, 7.43750]],
               [[3.62500, 2.81250], [4.87500, 6.18750], [11.65625, 10.18750]]]
    cfg = {"nano": [0.33, 0.25], "tiny": [0.33, 0.375], "s": [0.33, 0.5], "m": [0.67, 0.75], "l": [1.0, 1.0], "x": [1.33, 1.25]}
    _parts = ('backbone', 'neck', 'detect')

    def __init__(self, dictionary=None, model_cfg=None):
        super().__init__(dictionary, model_cfg)
        self.dummy_input = torch.zeros(1, 3, 640, 640)
        self.category = [v for d in self.dictionary for v in d.keys()]
        self.weight = [d[v] for d in self.dictionary for v in d.keys() if v in self.category]
        self.depth_mul, self.width_mul = self.cfg[self._cfg('TYPE').split("_")[1]]
        bcfg, ncfg, dcfg = dict(self._cfg('BACKBONE')), dict(self._cfg('NECK')), dict(self._cfg('DETECT'))
        bcfg.setdefault('subtype', self._cfg('TYPE'))
        ncfg.update(depth_mul=self.depth_mul, width_mul=self.width_mul)
        dcfg.update(depth_mul=self.depth_mul, width_mul=self.width_mul, anchors=self.anchors, num_classes=self.num_classes)
        self.backbone = build_backbone(bcfg)
        self.neck = build_neck(ncfg)
        self.detect = build_detect(dcfg)
        self.conf_thres = 0.001   # yolov5.py:189
        self.iou_thres = 0.6      # yolov5.py:190
        self.max_det = 300
        lcfg = self._loss_cfg('YOLOv5Loss')
        lcfg.update(anchors=self.anchors, num_classes=self.num_classes)  # yolov5.py:210-219 (setup_extra_params)
        self.loss = yolov5_train.YOLOv5Loss(**lcfg)  # (no parameters or buffers: the state_dict keys stay the inference model's)
        for m in self.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.eps = 1e-3
                m.momentum = 0.03
        # the training modules (yolov5_train.YOLOv5CSPDarknet / YOLOv5Neck / YOLOv5Detect), built on the first training forward over this
        # model's own parameters and buffers (train.bound_training_modules)
        self.__dict__['_train_modules'] = None
        self._cfgs = (bcfg, ncfg, dcfg)

    # ------------------------------------------------------------------ fused graph
    # ToTensor + Normalize of conf/coco_yolov5_s.yml:58-59 (det_transforms.py:85-109), used only by the uint8-frame entry points
    input_norm = dict(mean=(0.406, 0.456, 0.485), std=(0.225, 0.224, 0.229), reverse_channels=True)

    def build_graph(self, B, H, W, device, want_raw=False, u8_input=False):
        g = GraphBuilder(B, device)
        holder = {}
        feats = self.backbone.emit(g, lambda: holder['x'], H, W, u8_norm=dict(self.input_norm) if u8_input else None)
        feats = self.neck.emit(g, feats)
        conf, iou = self.conf_thres, self.iou_thres
        ws = ops.NmsWorkspace(B, self.detect.num_candidates(feats), self.num_classes, max_det=self.max_det, device=device)
        z, raws = self.detect.emit(g, feats, want_raw=want_raw, nms_ws=ws, conf_thres=conf, multi_label=True)
        g.fn(lambda: ops.yolo_nms(z, ws, conf, iou, True, hist_ready=True))
        return dict(g=g, holder=holder, z=z, raws=raws, ws=ws)

    def _graph_for(self, imgs, want_raw=False):
        u8 = imgs.dtype == torch.uint8
        B, H, W = (imgs.shape[0], imgs.shape[1], imgs.shape[2]) if u8 else (imgs.shape[0], imgs.shape[2], imgs.shape[3])
        # the thresholds are baked into the decode histogram / NMS steps of a graph: they are part of the key so that changing
        # model.conf_thres / iou_thres / max_det after the first forward takes effect (the reference reads them on every call, yolov5.py:262)
        return self._graph([imgs], lambda: self.build_graph(B, H, W, imgs.device, want_raw, u8_input=u8),
                           want_raw, u8, float(self.conf_thres), float(self.iou_thres), int(self.max_det))

    def predict_frames(self, frames_u8):
        """Device-only inference on camera frames: uint8 CUDA tensor [B,H,W,3] (BGR, already letterboxed to the network size).
        The reference's ToTensor + Normalize run inside the stem loader (``input_norm``); results equal ``predict`` on the
        tensor those transforms would have produced."""
        if self.training:
            raise RuntimeError('inference only: call .eval() first')
        if frames_u8.dtype != torch.uint8 or frames_u8.dim() != 4 or frames_u8.shape[3] != 3 or not frames_u8.is_cuda:
            raise ValueError('predict_frames expects a uint8 CUDA tensor [B,H,W,3]')
        ws = self._replay(frames_u8.contiguous())['ws']
        return ws.det, ws.det_idx, ws.det_count

    def _build_training_parts(self):
        """(yolov5_train.YOLOv5CSPDarknet, YOLOv5Neck, YOLOv5Detect); the training kernels refuse YOLOv5-m and -x."""
        strip = lambda c: {k: v for k, v in c.items() if k not in ('name', 'depth_mul', 'width_mul')}  # noqa: E731
        bcfg, ncfg, dcfg = self._cfgs
        return (yolov5_train.YOLOv5CSPDarknet(**strip(bcfg)), yolov5_train.YOLOv5Neck(**{k: v for k, v in ncfg.items() if k != 'name'}),
                yolov5_train.YOLOv5Detect(**{k: v for k, v in dcfg.items() if k != 'name'}))

    def _loss_step(self, outputs, gts):
        """yolov5.py:247-262: {loss [1], box_loss, obj_loss, cls_loss}."""
        loss, items = self.loss(outputs, gts)
        return {'loss': loss, 'box_loss': items[0], 'obj_loss': items[1], 'cls_loss': items[2]}
