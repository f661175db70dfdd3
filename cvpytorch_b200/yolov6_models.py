"""Drop-in modules for the YOLOv6-n / YOLOv6-s inference path (H100 fused graph, inference only).

Mirrors (paths relative to the reference checkout; same constructor arguments and sub-module names => same ``state_dict`` keys):
  YOLOv6EfficientRep  src/models/backbones/det/yolov6_efficient_rep.py:20-70 (+ det/base_yolo_backbone.py:16-53)
  SimCSPSPPF          src/models/modules/yolo_modules.py:218-242
  BiFusion            :245-265
  YOLOv6RepBiPAN      src/models/necks/det/yolov6_repbipan.py:16-82 (+ det/base_det_neck.py)
  YOLOv6Effidehead    src/models/heads/det/yolov6_effidehead.py:17-148 (+ det/base_yolo_head.py)
  YOLOv6Detect        src/models/detects/yolov6_detect.py:17-50 (anchors: anchors/yolov6_anchor_generator.py, mode='af')
  YOLOv6              conf/det/yolov6/coco_yolov6_{n,s}.yml USE_MODEL through detectors/yolo_detector.py (the keys), with the 'val'
                      contract of src/models/yolov6.py:193-235 (conf 0.03, iou 0.65, multi-label NMS :32-107, max_det 300)

Only the n and s widths run: every width of these two is a multiple of 16 (the conv kernel's cin % 16 == 0).  yolov6_t (24-channel
stem), yolov6_m / l / x (the reference head sets reg_max = 16 whatever use_dfl is, so its own eval forward fails at
reg_output.reshape([b, 4, l])), use_dfl=True and fuse_ab=True raise NotImplementedError.  forward(mode='train') runs the training mirrors
of yolov6_train.py on the training kernels and the H100 YOLOv6Loss.

Graph notes: the stem RepVGGBlock(3, c, stride 2) is one 3x3/s1 conv over the space-to-depth map (row-window loader of the YOLOv5
stem; only taps -1 and 0 are non-zero, ``repvgg_stem_weights_to_s2d``).  RepVGG blocks are folded to one 3x3 conv (yolo_blocks.py).
BiFusion's ConvTranspose2d(c, c, 2, stride=2) is a 1x1 GEMM with 4c output columns packed [py][px][cout] followed by
``cvb_depth_to_space2`` into channels [0, c) of the cv3 input buffer; the other two branches write the other slices of that buffer, so
no torch.cat exists.  In the head a level's cls_conv and reg_conv (3x3 of the same input) run as one GEMM with 2c columns; the class
logits and ltrb distances come out of fp32 1x1 GEMMs and ``cvb_yolov6_decode`` writes the z rows (objectness exactly 1.0) together with
the NMS pre-pass, after which the YOLOv5 NMS (ops.yolo_nms, hist_ready) selects the rows and scores the YOLOv6 NMS selects."""
import torch
import torch.nn as nn

from . import ops, yolov6_train
from .engine import GraphBuilder
from .models import _YoloModel
from .modules import ConvModule, _build, _EmitModule, _Standalone, folded
from .yolo_blocks import RepBlock, RepVGGBlock

STRIDES = [8, 16, 32]
BN_EPS, BN_MOMENTUM = 1e-3, 0.03  # every BatchNorm of the reference's YOLOv6 modules after its init_weights


def check_subtype(subtype):
    """'yolov6_n' / 'yolov6_s' (or any '<family>_n' / '_s') pass; the other widths raise NotImplementedError saying why."""
    stype = subtype.split('_')[1]
    if stype == 't':
        raise NotImplementedError(f'{subtype}: its 24-channel stem output is not a multiple of 16, which the H100 conv kernel needs '
                                  '(cin % 16 == 0); only YOLOv6-n and YOLOv6-s run')
    if stype in ('m', 'l', 'x'):
        raise NotImplementedError(f'{subtype}: the reference head sets reg_max = 16 for m / l / x whatever use_dfl is, so its own eval '
                                  'forward fails (reg_output.reshape([b, 4, l])); there is no working model to mirror. Only YOLOv6-n and '
                                  'YOLOv6-s run')
    if stype not in ('n', 's'):
        raise NotImplementedError(f'{subtype}: unknown YOLOv6 width')
    return stype


def _set_bn(module):
    for m in module.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.eps, m.momentum = BN_EPS, BN_MOMENTUM


def repvgg_stem_weights_to_s2d(w64):
    """Folded 3x3/s2/p1 kernel [O,3,3,3] -> the equivalent 3x3/s1/p1 kernel [O,16,3,3] over the 16-channel space-to-depth map.

    in(2h'+dy, 2w'+dx, c) sits at s2d channel (dy*2+dx)*3+c of pixel (h', w').  Output row oy reads input rows 2oy-1 (ky = 0: s2d row
    oy-1, dy = 1), 2oy (ky = 1: row oy, dy = 0) and 2oy+1 (ky = 2: row oy, dy = 1); likewise for columns.  s2d tap 2 (row oy+1) is zero."""
    O, I, kh, kw = w64.shape
    assert (I, kh, kw) == (3, 3, 3)
    tap = {0: (0, 1), 1: (1, 0), 2: (1, 1)}  # kernel index -> (s2d tap, sub-pixel offset)
    out = torch.zeros((O, 16, 3, 3), dtype=torch.float64)
    for ky, (a, dy) in tap.items():
        for kx, (b, dx) in tap.items():
            for c in range(3):
                out[:, (dy * 2 + dx) * 3 + c, a, b] = w64[:, c, ky, kx]
    return out


def conv_transpose2_weights(weight, bias):
    """nn.ConvTranspose2d(c, c, 2, stride=2) weight [Cin, Cout, 2, 2] and bias [Cout] -> the float64 1x1 GEMM [4*Cout, Cin, 1, 1] / [4*Cout]
    whose output column (py*2+px)*Cout + o is output pixel (2y+py, 2x+px), channel o (the layout cvb_depth_to_space2 reads)."""
    w = weight.detach().double().cpu()
    ci, co, kh, kw = w.shape
    assert (kh, kw) == (2, 2)
    w64 = w.permute(2, 3, 1, 0).reshape(4 * co, ci, 1, 1).contiguous()
    b64 = bias.detach().double().cpu().repeat(4)
    return w64, b64


# =============================================================================================== backbone
class SimCSPSPPF(_EmitModule):
    def __init__(self, in_channels, out_channels, kernel_size=5, e=0.5, conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True),
                 act_cfg=dict(type='Swish'), init_cfg=None):
        super().__init__()
        if kernel_size != 5:
            raise NotImplementedError('SimCSPSPPF: only the chained 5x5 pools are on the H100 hot path')
        c_ = int(out_channels * e)
        kw = dict(conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg)
        self.cv1 = ConvModule(in_channels, c_, 1, stride=1, **kw)
        self.cv2 = ConvModule(in_channels, c_, 1, stride=1, **kw)
        self.cv3 = ConvModule(c_, c_, 3, stride=1, padding=1, **kw)
        self.cv4 = ConvModule(c_, c_, 1, stride=1, **kw)
        self.m = nn.MaxPool2d(kernel_size=kernel_size, stride=1, padding=kernel_size // 2)  # parameter-free; kept for repr parity
        self.cv5 = ConvModule(4 * c_, c_, 1, stride=1, **kw)
        self.cv6 = ConvModule(c_, c_, 3, stride=1, padding=1, **kw)
        self.cv7 = ConvModule(2 * c_, out_channels, 1, stride=1, **kw)

    def emit(self, g, x, name='', out=None):
        c_ = self.cv1.out_channels
        assert self.cv1.act_name == self.cv2.act_name
        # [cv1(x) | y0 = cv2(x) | y3]: cv1 || cv2 as one GEMM, cv7 reads the [y0 | y3] half (= torch.cat((y0, y3)), :242)
        big = g.new_act(x.H, x.W, 3 * c_)
        w1, b1 = folded(self.cv1.conv, self.cv1.bn)
        w2, b2 = folded(self.cv2.conv, self.cv2.bn)
        g.conv(x, torch.cat([w1, w2], 0), torch.cat([b1, b2], 0), 1, 1, 0, self.cv1.act_name, out=big.slice(0, 2 * c_), name=name + '.cv12')
        t = self.cv3.emit(g, big.slice(0, c_), name + '.cv3')
        s = g.new_act(x.H, x.W, 4 * c_)  # [x1 | y1 | y2 | m(y2)] (:240)
        self.cv4.emit(g, t, name + '.cv4', out=s.slice(0, c_))
        v = [s.slice(i * c_, c_) for i in range(4)]
        g.fn(lambda: ops.sppf_pool(v[0].view(), v[1].view(), v[2].view(), v[3].view()))
        t = self.cv5.emit(g, s, name + '.cv5')
        self.cv6.emit(g, t, name + '.cv6', out=big.slice(2 * c_, c_))
        return self.cv7.emit(g, big.slice(c_, 2 * c_), name + '.cv7', out=out)


class YOLOv6EfficientRep(_Standalone):
    cfg = {"n": [0.33, 0.25], "t": [0.33, 0.375], "s": [0.33, 0.5], "m": [0.6, 0.75], "l": [1.0, 1.0], "x": [1.33, 1.25]}

    def __init__(self, subtype='cspdark_s', in_channels=3, out_channels=[64, 128, 256, 512, 1024], num_blocks=[6, 12, 18, 6], depthwise=False,
                 conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True), act_cfg=dict(type='SiLU', inplace=True), out_stages=[2, 3, 4],
                 output_stride=32, backbone_path=None, pretrained=False, frozen_stages=-1, norm_eval=False, **kwargs):
        super().__init__()
        check_subtype(subtype)
        if depthwise:
            raise NotImplementedError('depthwise YOLOv6 backbone is not on the H100 hot path')
        if in_channels != 3:
            raise NotImplementedError('YOLOv6EfficientRep: the stem expects 3 input channels')
        self.subtype, self.in_channels, self.out_stages, self.output_stride = subtype, in_channels, out_stages, output_stride
        depth_mul, width_mul = self.cfg[subtype.split('_')[1]]
        self.out_channels = list(map(lambda x: int(x * width_mul), out_channels))
        self.num_blocks = list(map(lambda x: max(round(x * depth_mul), 1), num_blocks))
        self.stem = RepVGGBlock(in_channels, self.out_channels[0], kernel_size=3, stride=2)
        for idx, (cin, cout, n) in enumerate(zip(self.out_channels[:-1], self.out_channels[1:], self.num_blocks)):
            stage = [RepVGGBlock(cin, cout, kernel_size=3, stride=2), RepBlock(cout, cout, n=n, block=RepVGGBlock)]
            if idx == 3:
                stage.append(SimCSPSPPF(cout, cout, act_cfg=dict(type='ReLU')))
            self.add_module(f'stage{idx + 1}', nn.Sequential(*stage))
        _set_bn(self)

    def emit(self, g, img_getter, H, W, name='backbone'):
        x0 = g.new_act(H // 2, W // 2 + 3, 16)  # zero-padded row-window layout, see YOLOv5CSPDarknet.emit
        g.fn(lambda: ops.stem_s2d(img_getter(), x0.view()))
        k, b = self.stem.equivalent_kernel_bias()
        x = g.conv(x0, repvgg_stem_weights_to_s2d(k), b, 3, 1, 1, 'relu', name=name + '.stem', w_window=4)
        outs = []
        for i in range(1, 5):
            for j, m in enumerate(getattr(self, f'stage{i}')):
                x = m.emit(g, x, f'{name}.stage{i}.{j}')
            if i in self.out_stages:
                outs.append(x)
        return outs

    def forward(self, x):
        return self._run_image(x)


# =============================================================================================== neck
class BiFusion(_Standalone):
    def __init__(self, in_channels, out_channels, conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True), act_cfg=dict(type='ReLU'),
                 init_cfg=None):
        super().__init__()
        kw = dict(conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg)
        self.cv1 = ConvModule(in_channels[0], out_channels, 1, 1, **kw)
        self.cv2 = ConvModule(in_channels[1], out_channels, 1, 1, **kw)
        self.cv3 = ConvModule(out_channels * 3, out_channels, 1, 1, **kw)
        self.upsample = nn.ConvTranspose2d(in_channels=out_channels, out_channels=out_channels, kernel_size=2, stride=2, bias=True)
        self.downsample = ConvModule(out_channels, out_channels, 3, 2, padding=1, **kw)

    def emit(self, g, x0, x1, x2, name='', out=None):
        """cv3(cat(upsample(x0), cv1(x1), downsample(cv2(x2)))): the three producers write the three channel slices of cv3's input."""
        c = self.cv3.out_channels
        cat = g.new_act(x1.H, x1.W, 3 * c)
        u = g.conv(x0, *conv_transpose2_weights(self.upsample.weight, self.upsample.bias), 1, 1, 0, None, name=name + '.upsample')
        dst = cat.slice(0, c)
        g.fn(lambda: ops.depth_to_space2(u.view(), dst.view()))
        self.cv1.emit(g, x1, name + '.cv1', out=cat.slice(c, c))
        t = self.cv2.emit(g, x2, name + '.cv2')
        self.downsample.emit(g, t, name + '.downsample', out=cat.slice(2 * c, c))
        return self.cv3.emit(g, cat, name + '.cv3', out=out)

    def forward(self, x):
        """x = [x0 (h, w), x1 (2h, 2w), x2 (4h, 4w)] NCHW CUDA maps -> the NCHW fp32 output, as the reference (:262-265)."""
        return ops.split_to_nchw(self._run(list(x), lambda g, ins: self.emit(g, *ins)).view())


class YOLOv6RepBiPAN(_Standalone):
    cfg = {"n": [0.33, 0.25], "t": [0.33, 0.375], "s": [0.33, 0.5], "m": [0.6, 0.75], "l": [1.0, 1.0], "x": [1.33, 1.25]}

    def __init__(self, subtype='yolov6_s', in_channels=[128, 256, 512, 1024], mid_channels=[128, 128, 256], out_channels=[128, 256, 512],
                 num_blocks=[12, 12, 12, 12], depthwise=False, conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True),
                 act_cfg=dict(type='ReLU', inplace=True), **kwargs):
        super().__init__()
        check_subtype(subtype)
        if depthwise:
            raise NotImplementedError('depthwise YOLOv6 neck is not on the H100 hot path')
        self.subtype = subtype
        depth_mul, width_mul = self.cfg[subtype.split('_')[1]]
        w = lambda cs: list(map(lambda x: max(round(x * width_mul), 1), cs))  # noqa: E731
        self.in_channels, self.mid_channels, self.out_channels = w(in_channels), w(mid_channels), w(out_channels)
        self.num_blocks = list(map(lambda x: max(round(x * depth_mul), 1), num_blocks))
        self.num_ins = len(self.in_channels)
        ic, mc, oc, nb = self.in_channels, self.mid_channels, self.out_channels, self.num_blocks
        kw = dict(norm_cfg=norm_cfg, act_cfg=act_cfg)
        self.reduce_layer0 = ConvModule(ic[3], mc[2], kernel_size=1, stride=1, padding=0, **kw)
        self.bifusion0 = BiFusion(in_channels=[ic[2], mc[2]], out_channels=mc[2])
        self.Rep_p4 = RepBlock(mc[2], mc[2], n=nb[3], block=RepVGGBlock)
        self.reduce_layer1 = ConvModule(mc[2], mc[1], kernel_size=1, stride=1, padding=0, **kw)
        self.bifusion1 = BiFusion(in_channels=[mc[2], mc[1]], out_channels=mc[1])
        self.Rep_p3 = RepBlock(mc[1], oc[0], n=nb[2], block=RepVGGBlock)
        self.downsample2 = ConvModule(oc[0], mc[0], kernel_size=3, stride=2, padding=1, **kw)
        self.Rep_n3 = RepBlock(mc[1] + mc[0], oc[1], n=nb[1], block=RepVGGBlock)
        self.downsample1 = ConvModule(oc[1], oc[1], kernel_size=3, stride=2, padding=1, **kw)
        self.Rep_n4 = RepBlock(mc[2] + oc[1], oc[2], n=nb[0], block=RepVGGBlock)
        _set_bn(self)

    def emit(self, g, feats, name='neck'):
        x3, x2, x1, x0 = feats
        mc, oc = self.mid_channels, self.out_channels
        cat_n4 = g.new_act(x0.H, x0.W, oc[1] + mc[2])  # [down_feat0 | fpn_out0]   (yolov6_repbipan.py:76-77)
        cat_n3 = g.new_act(x1.H, x1.W, mc[0] + mc[1])  # [down_feat1 | fpn_out1]   (:72-73)
        fpn_out0 = self.reduce_layer0.emit(g, x0, name + '.reduce_layer0', out=cat_n4.slice(oc[1], mc[2]))
        f_out0 = self.Rep_p4.emit(g, self.bifusion0.emit(g, fpn_out0, x1, x2, name + '.bifusion0'), name + '.Rep_p4')
        fpn_out1 = self.reduce_layer1.emit(g, f_out0, name + '.reduce_layer1', out=cat_n3.slice(mc[0], mc[1]))
        pan_out2 = self.Rep_p3.emit(g, self.bifusion1.emit(g, fpn_out1, x2, x3, name + '.bifusion1'), name + '.Rep_p3')
        self.downsample2.emit(g, pan_out2, name + '.downsample2', out=cat_n3.slice(0, mc[0]))
        pan_out1 = self.Rep_n3.emit(g, cat_n3, name + '.Rep_n3')
        self.downsample1.emit(g, pan_out1, name + '.downsample1', out=cat_n4.slice(0, oc[1]))
        pan_out0 = self.Rep_n4.emit(g, cat_n4, name + '.Rep_n4')
        return [pan_out2, pan_out1, pan_out0]

    def forward(self, x):
        assert len(x) == self.num_ins
        return [ops.split_to_nchw(o.view()) for o in self._run(list(x))]


# =============================================================================================== head / detect
class YOLOv6Effidehead(_Standalone):
    cfg = {"n": [0.33, 0.25], "t": [0.33, 0.375], "s": [0.33, 0.5], "m": [0.6, 0.75], "l": [1.0, 1.0], "x": [1.33, 1.25]}

    def __init__(self, subtype='yolov6_s', num_classes=80, in_channels=[128, 256, 512], num_anchors=1, reg_max=16, num_layers=3, stacked_convs=2,
                 depthwise=False, use_dfl=False, fuse_ab=False, conv_cfg=None, norm_cfg=dict(type='BN'), act_cfg=dict(type='SiLU'), **kwargs):
        super().__init__()
        check_subtype(subtype)
        if use_dfl:
            raise NotImplementedError('YOLOv6Effidehead: use_dfl=True (the distribution-focal regression of m / l / x) is not on the H100 hot path')
        if fuse_ab:
            raise NotImplementedError('YOLOv6Effidehead: fuse_ab=True (anchor-aided training branch) is not on the H100 hot path')
        if depthwise or num_layers != 3:
            raise NotImplementedError('YOLOv6Effidehead: only the 3-level, non-depthwise head is on the H100 hot path')
        if not 1 <= num_classes <= 91:
            raise NotImplementedError(f'YOLOv6Effidehead: 1..91 classes are supported by the decode kernel (got {num_classes})')
        self.subtype, self.fuse_ab, self.use_dfl = subtype, fuse_ab, use_dfl
        width_mul = self.cfg[subtype.split('_')[1]][1]
        self.in_channels = list(map(lambda x: max(round(x * width_mul), 1), in_channels))
        self.num_anchors, self.reg_max, self.stacked_convs = 1, 0, stacked_convs
        self.num_classes, self.num_outputs, self.num_layers = num_classes, num_classes + 5, num_layers
        self.stems, self.cls_convs, self.reg_convs = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        self.cls_preds, self.reg_preds = nn.ModuleList(), nn.ModuleList()
        self.proj_conv = nn.Conv2d(self.reg_max + 1, 1, 1, bias=False)
        kw = dict(conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg)
        for c in self.in_channels:
            self.stems.append(ConvModule(c, c, 1, 1, **kw))
            self.cls_convs.append(ConvModule(c, c, 3, 1, padding=1, **kw))
            self.reg_convs.append(ConvModule(c, c, 3, 1, padding=1, **kw))
            self.cls_preds.append(nn.Conv2d(c, num_classes * self.num_anchors, 1))
            self.reg_preds.append(nn.Conv2d(c, 4 * (self.num_anchors + self.reg_max), 1))
        self.proj = nn.Parameter(torch.linspace(0, self.reg_max, self.reg_max + 1), requires_grad=False)
        self.proj_conv.weight = nn.Parameter(self.proj.view([1, self.reg_max + 1, 1, 1]).clone().detach(), requires_grad=False)
        _set_bn(self)

    def emit(self, g, feats, name='head'):
        """Returns per level (cls fp32 [B,h,w,>=nc] class logits, reg fp32 [B,h,w,>=4] ltrb distances, stem output Val)."""
        outs = []
        for k, f in enumerate(feats):
            xx = self.stems[k].emit(g, f, f'{name}.stems.{k}')
            cc, rc = self.cls_convs[k], self.reg_convs[k]
            wc, bc = folded(cc.conv, cc.bn)
            wr, br = folded(rc.conv, rc.bn)
            assert cc.act_name == rc.act_name
            c = wc.shape[0]
            both = g.conv(xx, torch.cat([wc, wr], 0), torch.cat([bc, br], 0), 3, 1, 1, cc.act_name, name=f'{name}.cls_reg_convs.{k}')
            cls_out = g.new_f32(xx.H, xx.W, (self.num_classes + 31) // 32 * 32)
            g.conv(both.slice(0, c), *folded(self.cls_preds[k]), 1, 1, 0, None, f32_out=cls_out, name=f'{name}.cls_preds.{k}')
            reg_out = g.new_f32(xx.H, xx.W, 32)
            g.conv(both.slice(c, c), *folded(self.reg_preds[k]), 1, 1, 0, None, f32_out=reg_out, name=f'{name}.reg_preds.{k}')
            outs.append((cls_out, reg_out, xx))
        return outs

    def forward(self, x):
        """Eval forward of the reference (:129-148): list of NCHW CUDA maps -> (stem outputs (x, replaced in place as the reference does),
        cls scores [B, L, nc] (sigmoid), reg distances [B, L, 4]), L = sum of h*w over the levels in level / y / x order."""
        def emit(g, ins):
            outs = self.emit(g, ins)
            z = torch.zeros((g.B, sum(c.H * c.W for c, _, _ in outs), self.num_outputs), dtype=torch.float32, device=g.device)
            g.buffers.append(z)
            YOLOv6Detect.emit_decode(g, outs, self.num_classes, z)
            return outs, z
        outs, z = self._run(list(x), emit)
        for i, (_, _, xx) in enumerate(outs):
            x[i] = ops.split_to_nchw(xx.view())
        reg = torch.cat([ops.f32nhwc_to_nchw(r.view(0, 4)).flatten(2) for _, r, _ in outs], 2).permute(0, 2, 1)
        return x, z[..., 5:].clone(), reg


class YOLOv6Detect(_EmitModule):
    """No parameters.  Accepts the keys the configs pass (num_classes / use_dfl / fuse_ab, which the reference's BaseYOLODetect rejects) and
    refuses the values that are not on the H100 path.  Emitted into the model graph: the decode kernel writes z and the NMS pre-pass."""

    def __init__(self, subtype='yolov6_s', in_channels=[128, 256, 512], num_layers=3, strides=[8, 16, 32], conv_cfg=None, norm_cfg=dict(type='BN'),
                 act_cfg=dict(type='SiLU'), num_classes=80, use_dfl=False, fuse_ab=False, **kwargs):
        super().__init__()
        if use_dfl:
            raise NotImplementedError('YOLOv6Detect: use_dfl=True is not on the H100 hot path')
        if fuse_ab:
            raise NotImplementedError('YOLOv6Detect: fuse_ab=True is not on the H100 hot path')
        if num_layers != 3:
            raise NotImplementedError('YOLOv6Detect: only the 3-level (strides 8 / 16 / 32) detect is on the H100 hot path')
        self.subtype, self.in_channels, self.num_classes = subtype, in_channels, num_classes
        self.stride = torch.tensor(STRIDES)
        self.grid_cell_offset, self.grid_cell_size = 0.5, 5.0

    @staticmethod
    def emit_decode(g, head_outs, nc, z, nms_ws=None, conf_thres=0.001, multi_label=True):
        """z [B, A, 5 + nc] rows of every level (levels 8 / 16 / 32, then y, then x); nms_ws: the NMS pre-pass of yolo_nms(hist_ready)."""
        A = z.shape[1]
        if nms_ws is not None:
            g.fn(lambda: ops.nms_reset(nms_ws))
        off = 0
        for (cls, reg, _), s in zip(head_outs, STRIDES):
            g.fn(lambda cls=cls, reg=reg, s=s, off=off: ops.yolov6_decode(cls.view(0, nc), reg.view(0, 4), nc, float(s), z, A, off, nms_ws,
                                                                         conf_thres, multi_label))
            off += cls.H * cls.W
        assert off == A


_TRAIN_BACKBONES = {'YOLOv6EfficientRep': yolov6_train.YOLOv6EfficientRep}
_TRAIN_NECKS = {'YOLOv6RepBiPAN': yolov6_train.YOLOv6RepBiPAN}
_TRAIN_HEADS = {'YOLOv6Effidehead': yolov6_train.YOLOv6Effidehead}
_BACKBONES = {'YOLOv6EfficientRep': YOLOv6EfficientRep}
_NECKS = {'YOLOv6RepBiPAN': YOLOv6RepBiPAN}
_HEADS = {'YOLOv6Effidehead': YOLOv6Effidehead}
_DETECTS = {'YOLOv6Detect': YOLOv6Detect}


class YOLOv6Loss(nn.Module):
    """Holds the reference YOLOv6Loss's one parameter (``proj``, src/losses/det/yolov6_loss.py:45) so that the model's state_dict keys are
    the reference's (``loss.0.proj``).  It is not called: YOLOv6.forward(mode='train') computes the loss with a yolov6_train.YOLOv6Loss
    built from the same config."""

    def __init__(self, num_classes=80, fpn_strides=[8, 16, 32], grid_cell_size=5.0, grid_cell_offset=0.5, ori_img_size=640, warmup_epoch=4,
                 use_dfl=False, reg_max=16, iou_type='giou', loss_weight={'class': 1.0, 'iou': 2.5, 'dfl': 0.5}):
        super().__init__()
        self.num_classes, self.use_dfl, self.reg_max = num_classes, use_dfl, reg_max
        self.proj = nn.Parameter(torch.linspace(0, reg_max, reg_max + 1), requires_grad=False)

    def forward(self, *a, **k):
        raise NotImplementedError("YOLOv6 (H100): this holder only keeps the loss's state_dict key; YOLOv6.forward(mode='train') computes the "
                                  'loss (cvpytorch_b200.yolov6_train.YOLOv6Loss)')


class YOLOv6(_YoloModel):
    """Model-level drop-in for the reference's YOLOv6 (YAML route conf/det/yolov6/coco_yolov6_{n,s}.yml, USE_MODEL): same state_dict keys
    as its YOLODetector; forward(imgs, targets, 'val') runs the cached inference graph with the val contract of src/models/yolov6.py, and
    forward(imgs, targets, 'train') the training step of detectors/yolo_detector.py + single_stage.py: backbone -> neck -> head on the
    training kernels (yolov6_train), then the loss -> {'iou', 'dfl', 'class', 'loss'} fp64 device scalars.

    As the reference's YAML route: the loss is called without epoch_num, so ATSS assigns at every epoch (while warmup_epoch > 0); the class
    loss is discarded, so head.cls_convs.* and head.cls_preds.* get no gradient (.grad stays None; their BatchNorm running statistics still
    update, their forward runs)."""

    _parts = ('backbone', 'neck', 'head')

    def __init__(self, dictionary=None, model_cfg=None):
        super().__init__(dictionary, model_cfg)
        self.dummy_input = torch.zeros(1, 3, 640, 640)
        self.category = [v for d in self.dictionary for v in d.keys()]
        self.weight = [d[v] for d in self.dictionary for v in d.keys() if v in self.category]
        self.subtype = self._cfg('TYPE')
        check_subtype(self.subtype)
        sub = dict(subtype=self.subtype)  # yolo_detector.py:19-21
        self.backbone = _build(_BACKBONES, dict(dict(self._cfg('BACKBONE')), **sub))
        self.neck = _build(_NECKS, dict(dict(self._cfg('NECK')), **sub))
        self.head = _build(_HEADS, dict(dict(self._cfg('HEAD')), **sub))
        self.detect = _build(_DETECTS, dict(self._cfg('DETECT')))
        lcfg = self._loss_cfg('YOLOv6Loss')
        self.loss = nn.ModuleList([YOLOv6Loss(**lcfg)])
        self._cfgs = (dict(self._cfg('BACKBONE')), dict(self._cfg('NECK')), dict(self._cfg('HEAD')), sub)
        # the training loss (parameter-only: kept out of the module tree, so the state_dict keeps the reference's keys) and the training
        # modules, built on the first training forward over this model's own parameters and buffers (train.bound_training_modules)
        self.__dict__['_train_loss'] = yolov6_train.YOLOv6Loss(**lcfg)
        self.__dict__['_train_modules'] = None
        self.conf_thres, self.iou_thres, self.max_det = 0.03, 0.65, 300  # src/models/yolov6.py:150-151, :32

    def build_graph(self, B, H, W, device):
        g = GraphBuilder(B, device)
        holder = {}
        feats = self.neck.emit(g, self.backbone.emit(g, lambda: holder['x'], H, W))
        outs = self.head.emit(g, feats)
        nc, conf, iou = self.head.num_classes, float(self.conf_thres), float(self.iou_thres)
        A = sum(c.H * c.W for c, _, _ in outs)
        ws = ops.NmsWorkspace(B, A, nc, max_det=self.max_det, device=device)
        z = torch.zeros((B, A, nc + 5), dtype=torch.float32, device=device)
        g.buffers.append(z)
        YOLOv6Detect.emit_decode(g, outs, nc, z, ws, conf, True)
        g.fn(lambda: ops.yolo_nms(z, ws, conf, iou, True, hist_ready=True))
        return dict(g=g, holder=holder, z=z, ws=ws, outs=outs)

    def _graph_for(self, imgs):
        # the thresholds are baked into the decode histogram / NMS steps of a graph: part of the key, so that changing them takes effect
        return super()._graph_for(imgs, float(self.conf_thres), float(self.iou_thres), int(self.max_det))

    def _build_training_parts(self):
        """(yolov6_train.YOLOv6EfficientRep, YOLOv6RepBiPAN, YOLOv6Effidehead)."""
        bcfg, ncfg, hcfg, sub = self._cfgs
        return (_build(_TRAIN_BACKBONES, dict(bcfg, **sub)), _build(_TRAIN_NECKS, dict(ncfg, **sub)), _build(_TRAIN_HEADS, dict(hcfg, **sub)))

    def forward_train(self, imgs, targets):
        """The reference's training forward on the H100 training kernels -> {'iou', 'dfl', 'class', 'loss'} (fp64 device scalars, no host sync)."""
        if not imgs.is_cuda:
            raise NotImplementedError("YOLOv6 (H100): mode='train' has no CPU fallback: pass CUDA images")
        return super().forward_train(imgs, targets)

    def _loss_step(self, outputs, gt):
        losses = self._train_loss(outputs, gt)  # (no epoch_num: loss_forward, single_stage.py:97-103)
        losses['loss'] = losses['iou'] + losses['dfl'] + losses['class']
        return losses
