"""Training-step drop-ins for YOLOv5 (forward AND backward on the H100 kernels), next to the YOLOX ones of train.py.

Mirrors (paths relative to the reference checkout), with the same constructor arguments and state_dict keys:
  YOLOv5CSPDarknet  src/models/backbones/det/yolov5_csp_darknet.py:17-120  6x6 / s2 / p2 stem, four stages (stride-2 conv + C3), chained SPPF
  C3, Conv          src/models/modules/yolo11_modules.py:27-39, :173-217  (cv1 / cv2 / cv3 / m.i.cv1 / cv2 keys)
  UpsamplingModule, DownsamplingModule  src/models/modules/yolo11_modules.py:388-408
  YOLOv5Neck        src/models/necks/yolov5_neck.py:12-51
  YOLOv5Detect      src/models/detects/yolov5_detect.py:12-65  biased 1x1 convs -> fp32 NCHW [B, na (5 + nc), ny, nx]
  YOLOv5Loss        src/losses/yolov5_loss.py:135-278  build_targets, CIoU box, objectness and class BCE losses (csrc/yolov5_loss.cu)

The layers are train.py's (bf16 NHWC activations, fp32 master weights, every conv / BatchNorm / SiLU / pool on libcvb200.so); the
channel counts must be 16, 32 or multiples of 64, which YOLOv5-s meets (YOLOv5-m / -x raise NotImplementedError).  BatchNorm eps 1e-3,
momentum 0.03.  CPU tensors raise; evaluation goes through the inference modules of models.py, which load these modules' state_dict
with strict=True.
"""
import math

import torch
import torch.nn as nn

from . import _lib
from .train import (BaseConv, CSPLayer, SPPF, _bottleneck, _check_cuda, _ConvBnSiLULayer, _floats, _nhwc, _p, _ptrs, _require_training, _require_widths,
                    _set_bn, _shapes4, _stream, _to_nchw, _to_nhwc, _UpsampleCat, _workspace, conv, conv_wgrad, focus_s2d, pack_weights, pred_conv,
                    pred_cout_pad, pred_grad)


# ------------------------------------------------------------------------------------------------ backbone
def stem_weight_to_s2d(w):
    """fp32 [cout, 3, 6, 6] 6x6 / stride-2 / pad-2 stem weight -> [cout, 12, 3, 3] over focus_s2d's channels: W'[co, 3 (2 dx + dy) + ci, ty, tx]
    = W[co, ci, 2 ty + dy, 2 tx + dx] (the Focus patch order tl, bl, tr, br is patch = 2 dx + dy).  A torch permutation, so autograd maps the
    3x3 conv's weight gradient back onto the 6x6 weight."""
    co = w.shape[0]
    return w.view(co, 3, 3, 2, 3, 2).permute(0, 5, 3, 1, 2, 4).reshape(co, 12, 3, 3)


class StemConv(_ConvBnSiLULayer):
    """The YOLOv5 stem ConvModule (conv 3 -> cout, 6x6, stride 2, padding 2; keys conv.weight [cout, 3, 6, 6], bn.*): on the kernels,
    cvb_train_focus_s2d followed by a 3x3 / stride-1 / pad-1 conv over its 16 channels with stem_weight_to_s2d's weight (zero-padded from 12
    to 16 input channels).  forward: fp32 NCHW image (no gradient) -> NHWC bf16."""
    drop_in = 'YOLOv5CSPDarknet'

    def __init__(self, in_channels, out_channels):
        super().__init__(in_channels, out_channels, 6, 2, 2)
        self.ksize, self.stride, self.padding = 3, 1, None  # (what the kernels run)

    def forward(self, img):
        if img.requires_grad:
            raise NotImplementedError('H100 training YOLOv5 stem computes no gradient for the input image: pass an image without requires_grad')
        s2d = focus_s2d(img)
        return self._layer(s2d, nn.functional.pad(stem_weight_to_s2d(self.conv.weight), (0, 0, 0, 0, 0, s2d.shape[3] - 12)))


class YOLOv5CSPDarknet(nn.Module):
    """src/models/backbones/det/yolov5_csp_darknet.py:17-120, training mode, same constructor and state_dict keys.  forward(x): NCHW fp32 image
    -> list of NCHW outputs of out_stages; forward_nhwc(x): the same as NHWC bf16."""
    cfg = {"n": [0.33, 0.25], "t": [0.33, 0.375], "s": [0.33, 0.5], "m": [0.67, 0.75], "l": [1.0, 1.0], "x": [1.33, 1.25]}

    def __init__(self, subtype='cspdark_s', in_channels=3, out_channels=[64, 128, 256, 512, 1024], num_blocks=[3, 6, 9, 3], spp_ksizes=5,
                 depthwise=False, conv_cfg=None, norm_cfg=dict(type='BN', momentum=0.03, eps=0.001), act_cfg=dict(type='SiLU', inplace=True),
                 out_stages=[2, 3, 4], output_stride=32, backbone_path=None, pretrained=False, frozen_stages=-1, norm_eval=False, **unused):
        super().__init__()
        if depthwise or in_channels != 3 or spp_ksizes != 5:
            raise NotImplementedError('H100 training YOLOv5CSPDarknet: 3-channel images, no depthwise convs, the chained SPPF (spp_ksizes=5)')
        if norm_eval or frozen_stages >= 0:
            raise NotImplementedError('H100 training YOLOv5CSPDarknet: norm_eval and frozen_stages are not on the training path')
        self.subtype, self.out_stages = subtype, out_stages
        depth_mul, width_mul = self.cfg[subtype.split('_')[1]]
        ch = list(map(lambda x: int(x * width_mul), out_channels))
        nb = list(map(lambda x: max(round(x * depth_mul), 1), num_blocks))
        self.out_channels, self.num_blocks, self.in_channels = ch, nb, in_channels
        _require_widths(ch + [c // 2 for c in ch[1:]],
                        lambda bad: f'H100 training YOLOv5CSPDarknet {subtype}: widths {bad} are not on the training path (channels must be 16, 32 or multiples of 64)')
        self.stem = StemConv(in_channels, ch[0])
        for idx, (cin, cout, n) in enumerate(zip(ch[:-1], ch[1:], nb)):
            stage = [BaseConv(cin, cout, 3, 2), CSPLayer(cout, cout, n=n, shortcut=idx != 3)]
            if idx == 3:
                stage.append(SPPF(cout, cout, kernel_sizes=spp_ksizes))
            self.add_module(f'stage{idx + 1}', nn.Sequential(*stage))
        _set_bn(self)

    def forward_nhwc(self, x):
        _require_training(self, 'cvpytorch_b200.yolov5_train.YOLOv5CSPDarknet is the TRAINING drop-in (batch statistics); load its state_dict into '
                                'cvpytorch_b200.models.YOLOv5CSPDarknet for eval()')
        _check_cuda(x, 'YOLOv5CSPDarknet (H100 training)')
        h = self.stem(x)
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


# ------------------------------------------------------------------------------------------------ neck
class Conv(BaseConv):
    """yolo11_modules.py:27-39 (autopad, SiLU, groups 1): keys conv.weight, bn.*."""

    def __init__(self, c1, c2, k=1, s=1, p=None, g=1, act=True):
        if g != 1 or act is not True or (p is not None and p != k // 2):
            raise NotImplementedError('H100 training Conv: groups 1, SiLU, padding k // 2')
        super().__init__(c1, c2, k, s)


class C3Bottleneck(nn.Module):
    """yolo11_modules.py Bottleneck (keys cv1 / cv2): 1x1 -> 3x3 (+ shortcut)."""

    def __init__(self, c1, c2, shortcut=True, g=1, e=0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c_, c2, 3, 1, g=g)
        self.add = shortcut and c1 == c2

    def forward(self, x):
        return _bottleneck(self, x, self.cv1, self.cv2, self.add)


class C3(nn.Module):
    """yolo11_modules.py C3: cv1 | cv2 -> bottlenecks -> cat -> cv3 (the CSPLayer with the cv* key names)."""

    def __init__(self, c1, c2, n=1, shortcut=True, g=1, e=0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c1, c_, 1, 1)
        self.cv3 = Conv(2 * c_, c2, 1)
        self.m = nn.Sequential(*[C3Bottleneck(c_, c_, shortcut, g, e=1.0) for _ in range(n)])

    def forward_nhwc(self, x):
        return self.cv3(torch.cat((self.m(self.cv1(x)), self.cv2(x)), dim=3))


class UpsamplingModule(nn.Module):
    """yolo11_modules.py:388-397: x_conv = conv(x); fuse(cat([up(x_conv), y])) -> (fused, x_conv).  NHWC bf16."""

    def __init__(self, c1, c2, layer=3):
        super().__init__()
        self.conv = Conv(c1, c2, 1, 1)
        self.up = nn.UpsamplingNearest2d(scale_factor=2)  # (parameter-free; module-tree parity)
        self.fuse = C3(c2 * 2, c2, layer, False)

    def forward_nhwc(self, x, y):
        x_conv = self.conv(x)  # (fans out to the upsample and to the bottom-up concat: autograd adds the two gradients)
        return self.fuse.forward_nhwc(_UpsampleCat.apply(x_conv, y)), x_conv


class DownsamplingModule(nn.Module):
    """yolo11_modules.py:400-408: fuse(cat([down(x), y])).  NHWC bf16."""

    def __init__(self, c1, c2, layer=3):
        super().__init__()
        self.down = Conv(c1, c1, 3, 2)
        self.fuse = C3(c1 * 2, c2, layer, False)

    def forward_nhwc(self, x, y):
        return self.fuse.forward_nhwc(torch.cat((self.down(x), y), dim=3))


class YOLOv5Neck(nn.Module):
    """src/models/necks/yolov5_neck.py:12-51, training mode, same constructor and state_dict keys.  forward_nhwc([x3, x4, x5] NHWC bf16) ->
    [x3_up, x4_down, x5_down] NHWC bf16; forward takes and returns NCHW."""

    def __init__(self, in_channels, out_channels, depth_mul=1.0, width_mul=1.0, **unused):
        super().__init__()
        assert isinstance(in_channels, list)
        self.in_channels = list(map(lambda x: max(round(x * width_mul), 1), in_channels))
        self.out_channels = list(map(lambda x: max(round(x * width_mul), 1), out_channels))
        self.layers = list(map(lambda x: max(round(x * depth_mul), 1), [3, 3, 3, 3]))
        ic, oc = self.in_channels, self.out_channels
        _require_widths(ic + oc[:1] + [c // 2 for c in ic + oc[:1]],
                        lambda bad: f'H100 training YOLOv5Neck: widths {bad} are not on the training path (channels must be 16, 32 or multiples of 64)')
        self.up_1 = UpsamplingModule(ic[2], ic[1], self.layers[0])
        self.up_2 = UpsamplingModule(ic[1], oc[0], self.layers[1])
        self.down_1 = DownsamplingModule(ic[0], ic[1], self.layers[2])
        self.down_2 = DownsamplingModule(ic[1], ic[2], self.layers[3])
        _set_bn(self)

    def forward_nhwc(self, x):
        _require_training(self, 'cvpytorch_b200.yolov5_train.YOLOv5Neck is the TRAINING drop-in (batch statistics); load its state_dict into '
                                'cvpytorch_b200.models.YOLOv5Neck for eval()')
        if len(x) != len(self.in_channels):
            raise ValueError(f'YOLOv5Neck: {len(self.in_channels)} feature maps expected, got {len(x)}')
        x3, x4, x5 = x
        for big, small in ((x4, x5), (x3, x4)):
            if big.shape[0] != small.shape[0] or big.shape[1] != 2 * small.shape[1] or big.shape[2] != 2 * small.shape[2]:
                raise ValueError(f'YOLOv5Neck: each feature map must be exactly twice the next one in height and width (got {[tuple(t.shape) for t in x]}, NHWC)')
        x4_up, x4_t = self.up_1.forward_nhwc(x5, x4)
        x3_up, x3_t = self.up_2.forward_nhwc(x4_up, x3)
        x4_down = self.down_1.forward_nhwc(x3_up, x3_t)
        x5_down = self.down_2.forward_nhwc(x4_down, x4_t)
        return [x3_up, x4_down, x5_down]

    def forward(self, x):
        return [_to_nchw(o, x[0].dtype) for o in self.forward_nhwc([_to_nhwc(t, 'YOLOv5Neck (H100 training)') for t in x])]


# ------------------------------------------------------------------------------------------------ detect
class _PredConv(torch.autograd.Function):
    """One biased 1x1 conv x NHWC bf16 -> fp32 NCHW [B, cout, h, w] through the PRED epilogue (cout zero-padded to pred_cout_pad(cout))."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        _check_cuda(x, 'YOLOv5Detect (H100 training)')
        x = x.contiguous()
        B, h, w, _ = x.shape
        cout = weight.shape[0]
        out = torch.empty((B, cout, h, w), dtype=torch.float32, device=x.device)
        wf, wb = pack_weights(nn.functional.pad(weight.detach().float(), (0, 0, 0, 0, 0, 0, 0, pred_cout_pad(cout) - cout)))
        pred_conv(x, wf, cout, bias.detach().float().contiguous(), out, 0)
        ctx.save_for_backward(x, wb)
        return out

    @staticmethod
    def backward(ctx, g):
        x, wb = ctx.saved_tensors
        cout = g.shape[1]
        dy, db = pred_grad(g.contiguous(), 0, cout)
        dw = conv_wgrad(x, dy, 1)[:cout]
        dx = conv(dy, wb, x.shape[3], 1) if ctx.needs_input_grad[0] else None
        return dx, dw, db


class YOLOv5Detect(nn.Module):
    """src/models/detects/yolov5_detect.py:12-65, training mode, same constructor, state_dict keys (anchors buffer, m.i) and bias prior.
    forward_nhwc(feats NHWC bf16) -> the detect convs' fp32 NCHW outputs [B, na (5 + nc), ny, nx] (what YOLOv5Loss reads in place);
    forward(feats NCHW) -> (None, the reference's [B, na, ny, nx, 5 + nc] views of them)."""

    def __init__(self, num_classes=80, in_channels=[256, 512, 1024], stride=[8., 16., 32.], anchors=(), depth_mul=1.0, width_mul=1.0):
        super().__init__()
        in_channels = list(map(lambda x: int(x * width_mul), in_channels))
        _require_widths(in_channels, lambda bad: f'H100 training YOLOv5Detect: widths {bad} are not on the training path (channels must be 16, 32 or multiples of 64)')
        self.num_classes, self.num_outputs = num_classes, num_classes + 5
        self.num_layers, self.num_anchors = len(anchors), len(anchors[0])
        self.stride = stride
        self.register_buffer('anchors', torch.tensor(anchors).float())
        self.m = nn.ModuleList(nn.Conv2d(x, self.num_outputs * self.num_anchors, 1) for x in in_channels)
        for mi, s in zip(self.m, self.stride):  # yolov5_detect.py:28-35
            b = mi.bias.view(self.num_anchors, -1)
            b.data[:, 4] += math.log(8 / (640 / s) ** 2)
            b.data[:, 5:] += math.log(0.6 / (self.num_classes - 0.999999))
            mi.bias = torch.nn.Parameter(b.view(-1), requires_grad=True)

    def forward_nhwc(self, x):
        if not self.training:
            raise RuntimeError('cvpytorch_b200.yolov5_train.YOLOv5Detect is the TRAINING drop-in; load its state_dict into cvpytorch_b200.models.YOLOv5Detect for eval()')
        return [_PredConv.apply(f, mi.weight, mi.bias) for f, mi in zip(x, self.m)]

    def forward(self, x):
        outs = self.forward_nhwc([_to_nhwc(t, 'YOLOv5Detect (H100 training)') for t in x])
        na, no = self.num_anchors, self.num_outputs
        return None, [o.view(o.shape[0], na, no, o.shape[2], o.shape[3]).permute(0, 1, 3, 4, 2) for o in outs]


# ------------------------------------------------------------------------------------------------ loss
def _loss_args(preds, anchors, balance, hyp):
    return _ptrs(preds), _shapes4(preds), _floats(anchors.flatten().tolist()), _floats(balance[:len(preds)]), _floats(hyp)


def yolov5_loss_forward(preds, targets, anchors, balance, hyp, num_classes):
    """preds: fp32 NCHW [B, na (5 + nc), ny, nx] (CUDA, contiguous); targets fp32 [nt, 6] (image, class, cx, cy, w, h normalised); anchors
    [nlev, na, 2] in grid units (host); hyp = (anchor_t, box, obj, cls, gr).  -> (out [4] = loss, lbox, lobj, lcls; (cand_idx [nlev, cap, 5],
    cand_box [nlev, cap, 6], ncand [nlev]) the candidate lists; workspace)."""
    nlev, na = anchors.shape[0], anchors.shape[1]
    nt = targets.shape[0]
    dev = preds[0].device
    cap = max(5 * na * nt, 1)
    L = _lib.lib()
    ws = _workspace(L.cvb_train_yolov5_loss_workspace_bytes(nlev, na, nt), dev)
    out = torch.empty((4,), dtype=torch.float32, device=dev)
    cand_idx = torch.empty((nlev, cap, 5), dtype=torch.int32, device=dev)
    cand_box = torch.empty((nlev, cap, 6), dtype=torch.float32, device=dev)
    ncand = torch.empty((nlev,), dtype=torch.int32, device=dev)
    ptrs, shapes, anc, bal, hy = _loss_args(preds, anchors, balance, hyp)
    _lib.check(L.cvb_train_yolov5_loss_fwd(ptrs, shapes, anc, bal, len(preds), na, num_classes, _p(targets) if nt else None, nt, hy, _p(cand_idx),
                                           _p(cand_box), _p(ncand), _p(out), _p(ws), ws.numel(), _stream()), 'cvb_train_yolov5_loss_fwd')
    return out, (cand_idx, cand_box, ncand), ws


def yolov5_loss_backward(preds, targets, anchors, balance, hyp, num_classes, cands, ws, grad_out):
    """grad_out [1] (device) x d(loss)/d(preds) under the forward's candidates -> fp32 NCHW gradients shaped like preds."""
    grads = [torch.empty_like(p) for p in preds]
    ptrs, shapes, anc, bal, hy = _loss_args(preds, anchors, balance, hyp)
    cand_idx, cand_box, ncand = cands
    nt = targets.shape[0]
    _lib.check(_lib.lib().cvb_train_yolov5_loss_bwd(ptrs, shapes, anc, bal, len(preds), anchors.shape[1], num_classes, _p(targets) if nt else None, nt, hy,
                                                    _p(cand_idx), _p(cand_box), _p(ncand), _p(ws), ws.numel(), _p(grad_out), _ptrs(grads), _stream()),
               'cvb_train_yolov5_loss_bwd')
    return grads


class _YOLOv5LossFn(torch.autograd.Function):
    """out [4] = (loss, lbox, lobj, lcls); the backward scales the gradient by the incoming gradient of `loss` only (the items are detached
    in the reference)."""

    @staticmethod
    def forward(ctx, targets, meta, *preds):
        anchors, balance, hyp, nc = meta
        out, cands, ws = yolov5_loss_forward(preds, targets, anchors, balance, hyp, nc)
        ctx.save_for_backward(targets, ws, *cands, *preds)
        ctx.meta = meta
        return out

    @staticmethod
    def backward(ctx, g):
        targets, ws, ci, cb, nc_, *preds = ctx.saved_tensors
        anchors, balance, hyp, nc = ctx.meta
        grads = yolov5_loss_backward(preds, targets, anchors, balance, hyp, nc, (ci, cb, nc_), ws, g[:1].float().contiguous())
        return (None, None, *grads)


class YOLOv5Loss(nn.Module):
    """src/losses/yolov5_loss.py:135-278 on the H100 kernels (csrc/yolov5_loss.cu): same constructor, no parameters or buffers.
    forward(p, targets) takes the detect outputs -- fp32 NCHW [B, na (5 + nc), ny, nx] (CUDA) or the reference's [B, na, ny, nx, 5 + nc]
    views of them -- and targets [nt, 6] (image, class, cx, cy, w, h, normalised), and returns the reference's (loss [1], items [3] = lbox,
    lobj, lcls, detached) as device tensors with no host sync: the whole loss can be captured in a CUDA graph.  Defaults of the reference:
    anchor_t 4, balance [4, 1, 0.4], gr 1, no label smoothing, no focal loss.  autobalance=True raises NotImplementedError (it reads the
    objectness loss on the host every step)."""

    def __init__(self, num_classes, stride=[8., 16., 32.], anchors=(), hyp_box=0.05, hyp_obj=1.0, hyp_cls=0.5, device='cuda:0', autobalance=False):
        super().__init__()
        if autobalance:
            raise NotImplementedError('H100 YOLOv5Loss: autobalance (a host .item() every step) is not implemented')
        self.num_classes = num_classes
        self.num_layers, self.num_anchors = len(anchors), len(anchors[0])
        self.stride = list(stride)
        self.anchors_grid = torch.tensor(anchors, dtype=torch.float32)  # (a plain tensor, not a buffer: no state_dict entry)
        self.hyp_anchor_t, self.hyp_box, self.hyp_obj, self.hyp_cls, self.gr = 4.0, hyp_box, hyp_obj, hyp_cls, 1.0
        self.balance = {3: [4.0, 1.0, 0.4]}.get(self.num_layers, [4.0, 1.0, 0.25, 0.06, .02])
        self.autobalance = autobalance

    def _nchw(self, p):
        _check_cuda(p, 'YOLOv5Loss')
        if p.dim() == 5:  # the reference's [B, na, ny, nx, no] view -> [B, na * no, ny, nx] (a view when it permutes the NCHW output)
            B, na, ny, nx, no = p.shape
            p = p.permute(0, 1, 4, 2, 3).reshape(B, na * no, ny, nx)
        return p.float().contiguous()

    def forward(self, p, targets):
        if len(p) != self.num_layers:
            raise ValueError(f'YOLOv5Loss: {self.num_layers} levels for {len(p)} outputs')
        preds = [self._nchw(x) for x in p]
        if not isinstance(targets, torch.Tensor) or targets.dim() != 2 or targets.shape[1] != 6:
            raise ValueError('YOLOv5Loss: targets must be a [nt, 6] tensor of (image, class, cx, cy, w, h) rows')
        _check_cuda(targets, 'YOLOv5Loss targets')
        t = targets.detach().to(device=preds[0].device, dtype=torch.float32).contiguous()
        meta = (self.anchors_grid, tuple(self.balance), (self.hyp_anchor_t, self.hyp_box, self.hyp_obj, self.hyp_cls, self.gr), self.num_classes)
        out = _YOLOv5LossFn.apply(t, meta, *preds)
        return out[:1], out[1:].detach()
