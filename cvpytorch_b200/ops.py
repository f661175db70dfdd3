"""Python wrappers over the C ABI: device tensor containers + one function per cvb_* entry point.

PyTorch is used only as plumbing (device memory, streams); all arithmetic on the hot path happens in
libcvb200.so.  Host-side weight preparation (BN folding, hi/lo split, K-major packing) also lives here.
"""
import ctypes
from ctypes import byref, c_void_p

import torch

from . import _lib
from ._lib import (CVB_ACT_NONE, CVB_ACT_RELU, CVB_ACT_SILU, CVB_OUT_F32, CVB_OUT_SPLIT16, CVB_OUT_YOLO, CvbConvDesc, CvbNmsParams, CvbView,
                   CvbYoloDecode, _stream)

ACTS = {None: CVB_ACT_NONE, 'none': CVB_ACT_NONE, 'silu': CVB_ACT_SILU, 'swish': CVB_ACT_SILU, 'relu': CVB_ACT_RELU}


def _require_cuda(t, what):
    if not t.is_cuda:
        raise _lib.CvbError(f'{what}: tensor must live on a CUDA device (the H100 path has no CPU fallback)')


class SplitTensor:
    """NHWC activation stored as two fp16 planes [2, B, H, W, C] (hi, lo); x = hi + lo."""

    def __init__(self, B, H, W, C, device='cuda', data=None):
        self.B, self.H, self.W, self.C = B, H, W, C
        self.data = data if data is not None else torch.zeros((2, B, H, W, C), dtype=torch.float16, device=device)
        assert self.data.is_contiguous() and self.data.dtype == torch.float16

    def view(self, c0=0, c=None):
        c = self.C - c0 if c is None else c
        assert 0 <= c0 and c0 + c <= self.C and c0 % 8 == 0
        v = CvbView()
        v.base = self.data.data_ptr() + 2 * c0
        v.B, v.H, v.W, v.C = self.B, self.H, self.W, c
        v.c_pitch = self.C
        v.plane_stride = 2 * self.B * self.H * self.W * self.C
        return v

    def to_float_nhwc(self):
        """Debug helper: fp32 [B,H,W,C] = hi + lo (torch ops; not used on the hot path)."""
        return self.data[0].float() + self.data[1].float()


class F32Tensor:
    """Plain fp32 NHWC tensor [B, H, W, C] (partials, head logits)."""

    def __init__(self, B, H, W, C, device='cuda'):
        self.B, self.H, self.W, self.C = B, H, W, C
        self.data = torch.zeros((B, H, W, C), dtype=torch.float32, device=device)

    def view(self, c0=0, c=None):
        c = self.C - c0 if c is None else c
        assert c0 % 4 == 0 and c0 + c <= self.C
        v = CvbView()
        v.base = self.data.data_ptr() + 4 * c0
        v.B, v.H, v.W, v.C = self.B, self.H, self.W, c
        v.c_pitch = self.C
        v.plane_stride = 0
        return v


def null_view():
    v = CvbView()
    v.base = None
    return v


# --------------------------------------------------------------------------------------- host-side weight prep
def fold_conv_bn(weight, bias=None, bn=None):
    """Folds eval-mode BatchNorm into the conv (float64 on the host, rounded once to fp32).

    Algebra of the reference's src/utils/fuse.py:33-54:  W' = W * g/sqrt(var+eps),  b' = (b - mean) * g/sqrt(var+eps) + beta
    bn = (gamma, beta, running_mean, running_var, eps) or None.
    """
    w = weight.detach().double().cpu()
    b = torch.zeros(w.shape[0], dtype=torch.float64) if bias is None else bias.detach().double().cpu()
    if bn is not None:
        gamma, beta, mean, var, eps = bn
        scale = gamma.detach().double().cpu() / torch.sqrt(var.detach().double().cpu() + eps)
        w = w * scale.view(-1, 1, 1, 1)
        b = (b - mean.detach().double().cpu()) * scale + beta.detach().double().cpu()
    return w, b


def pack_conv_weights(w64, b64, cin_pad=None, device='cuda'):
    """[O,I,kh,kw] float64 -> (fp16 [2, O_pad, kh*kw*I_pad] K-major hi/lo planes, fp32 bias [O_pad])."""
    O, I, kh, kw = w64.shape
    cin_pad = I if cin_pad is None else cin_pad
    o_pad = (O + 7) // 8 * 8
    w = torch.zeros((o_pad, kh, kw, cin_pad), dtype=torch.float64)
    w[:O, :, :, :I] = w64.permute(0, 2, 3, 1)
    w = w.reshape(o_pad, kh * kw * cin_pad)
    if float(w.abs().max()) > 65504.0:  # fp16 hi would be inf and lo -inf -> NaN results; BN-folded weights are O(1)
        raise _lib.CvbError(f'pack_conv_weights: |weight| up to {float(w.abs().max()):.3g} exceeds the fp16 range of the hi/lo operand '
                            'format (65504); rescale the layer')
    hi = w.to(torch.float16)
    lo = (w - hi.double()).to(torch.float16)
    packed = torch.stack([hi, lo], 0).contiguous()
    bias = torch.zeros(o_pad, dtype=torch.float32)
    bias[:O] = b64.float()
    return packed.to(device), bias.to(device)


def pack_yolo_head_weights(w64, b64, na, no, device='cuda'):
    """Detect-head 1x1 conv [na*no, I, 1, 1] -> the CVB_OUT_YOLO layout: ONE ANCHOR PER 128-WIDE N-TILE (row a*128 + o = output channel
    a*no + o, the other rows zero), so that the fused-decode epilogue finds all `no` outputs of an (anchor, pixel) row in one accumulator tile."""
    O, I, kh, kw = w64.shape
    assert O == na * no and kh == 1 and kw == 1 and no <= 128
    w = torch.zeros((na * 128, I, 1, 1), dtype=torch.float64)
    b = torch.zeros((na * 128,), dtype=torch.float64)
    for a in range(na):
        w[a * 128:a * 128 + no] = w64[a * no:(a + 1) * no]
        b[a * 128:a * 128 + no] = b64[a * no:(a + 1) * no]
    return pack_conv_weights(w, b, device=device)


def yolo_decode_desc(na, no, anchors_px, stride, z, z_rows, z_off, nms_ws=None, conf_thres=0.001, multi_label=True):
    y = CvbYoloDecode()
    y.na, y.no = na, no
    ap = [float(v) for v in anchors_px.detach().float().cpu().reshape(-1).tolist()]
    assert len(ap) == 2 * na and na <= 4
    for i in range(8):
        y.anchors_px[i] = ap[i] if i < len(ap) else 0.0
    y.stride = float(stride)
    y.z = z.data_ptr()
    y.z_rows, y.z_off = int(z_rows), int(z_off)
    y.nms_workspace = nms_ws.ws_ptr if nms_ws is not None else None
    y.conf_thres = float(conf_thres)
    y.multi_label = 1 if multi_label else 0
    return y


def window_weights(w64, window):
    """[O,C,kh,kw] -> [O, window*C, kh, 1]: the kw taps of a filter row laid side by side (zeros for kx >= kw), matching
    CvbConvDesc.w_window (k = ky*window*C + kx*C + c)."""
    O, C, kh, kw = w64.shape
    out = torch.zeros((O, window * C, kh, 1), dtype=torch.float64)
    for kx in range(kw):
        out[:, kx * C:(kx + 1) * C, :, 0] = w64[:, :, :, kx]
    return out


def stem_weights_to_s2d(w64):
    """6x6/s2/p2 stem kernel [O,3,6,6] -> equivalent 3x3/s1/p1 kernel over the 16-channel space-to-depth input.

    in(2h'+dy, 2w'+dx, c) sits at s2d channel (dy*2+dx)*3+c of pixel (h', w'); kernel row kh = 2a+dy.
    """
    O, I, kh, kw = w64.shape
    assert (I, kh, kw) == (3, 6, 6)
    out = torch.zeros((O, 16, 3, 3), dtype=torch.float64)
    for a in range(3):
        for b in range(3):
            for dy in range(2):
                for dx in range(2):
                    for c in range(3):
                        out[:, (dy * 2 + dx) * 3 + c, a, b] = w64[:, c, 2 * a + dy, 2 * b + dx]
    return out


# --------------------------------------------------------------------------------------- op wrappers
class ConvPlan:
    """Owns a CvbConvPlan handle (host-side TMA descriptors + launch shape) and keeps its tensors alive."""

    def __init__(self, inp, out, weights, bias, k, stride=1, pad=0, dilation=1, act=None, residual=None,
                 up_partial=None, block_n=0, sm_limit=0, keepalive=(), w_window=0, no_resident=0, residual_before_act=0, halo=0, residual_scale=1.0,
                 yolo=None, schedule=0):
        """yolo: a CvbYoloDecode -> the conv's epilogue is the YOLOv5 decode (out_kind CVB_OUT_YOLO, see include/cvb200.h); `out` then only
        carries B/H/W with C = na * 128 and `weights` / `bias` must come from pack_yolo_head_weights.
        schedule: 0 = auto, 1 = cooperative, 2 = ping-pong (CvbConvDesc.schedule)."""
        d = CvbConvDesc()
        d.inp, d.out = inp, out
        d.weights = weights.data_ptr()
        d.cout_pad = weights.shape[1]
        d.bias = bias.data_ptr()
        d.kh = d.kw = k
        d.stride, d.pad, d.dilation = stride, pad, dilation
        d.act = ACTS[act]
        d.out_kind = CVB_OUT_F32 if out.plane_stride == 0 else CVB_OUT_SPLIT16
        if yolo is not None:
            d.out_kind = CVB_OUT_YOLO
            d.yolo = ctypes.pointer(yolo)
            self._yolo = yolo  # (the plan copies what it needs at creation; kept for introspection)
        d.residual = residual if residual is not None else null_view()
        d.up_partial = up_partial if up_partial is not None else null_view()
        d.block_n, d.sm_limit = block_n, sm_limit
        d.w_window = w_window
        d.no_resident = no_resident
        d.residual_before_act = residual_before_act
        d.halo = halo
        d.residual_scale = float(residual_scale)
        d.schedule = schedule
        self._keep = (weights, bias) + tuple(keepalive)
        self.handle = c_void_p()
        _lib.check(_lib.lib().cvb_conv_plan_create(byref(d), byref(self.handle)), 'cvb_conv_plan_create')

    def run(self):
        _lib.check(_lib.lib().cvb_conv_plan_run(self.handle, _stream()), 'cvb_conv_plan_run')

    def __del__(self):
        try:
            if getattr(self, 'handle', None) is not None and self.handle.value:
                _lib.lib().cvb_conv_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


def run_plans(plans):
    arr = (c_void_p * len(plans))(*[p.handle for p in plans])
    _lib.check(_lib.lib().cvb_conv_plan_run_many(arr, len(plans), _stream()), 'cvb_conv_plan_run_many')


def nchw_to_split(x, dst_view):
    _require_cuda(x, 'nchw_to_split')
    x = x.contiguous().float()
    B, C, H, W = x.shape
    _lib.check(_lib.lib().cvb_nchw_to_split(x.data_ptr(), B, C, H, W, byref(dst_view), _stream()), 'cvb_nchw_to_split')


def split_to_nchw(src_view, out=None, device=None):
    """device: where to allocate `out` (default: the current CUDA device -- the library runs one device per process and
    the stand-alone drop-ins, modules._Standalone, reject tensors that live elsewhere)."""
    if out is None:
        out = torch.empty((src_view.B, src_view.C, src_view.H, src_view.W), dtype=torch.float32,
                          device=device if device is not None else torch.device('cuda', torch.cuda.current_device()))
    _lib.check(_lib.lib().cvb_split_to_nchw(byref(src_view), out.data_ptr(), _stream()), 'cvb_split_to_nchw')
    return out


def f32nhwc_to_nchw(src_view, out=None, device=None):
    if out is None:
        out = torch.empty((src_view.B, src_view.C, src_view.H, src_view.W), dtype=torch.float32,
                          device=device if device is not None else torch.device('cuda', torch.cuda.current_device()))
    _lib.check(_lib.lib().cvb_f32nhwc_to_nchw(byref(src_view), out.data_ptr(), _stream()), 'cvb_f32nhwc_to_nchw')
    return out


def stem_s2d(x, dst_view, pad_left=None, norm=None):
    """x: fp32 NCHW [B,3,H,W] (the reference's model input), or uint8 NHWC [B,H,W,3] camera frames with
    ``norm = dict(mean=(..3), std=(..3), reverse_channels=bool)`` = the reference's ToTensor + Normalize fused into the loader.
    pad_left=None: 0 for a plain [B,H/2,W/2,16] target, 1 for the padded row-window layout (W/2+3 columns)."""
    _require_cuda(x, 'stem_s2d')
    assert x.is_contiguous()
    if x.dtype == torch.uint8:
        B, H, W, C = x.shape
        assert C == 3 and norm is not None, 'uint8 frames need [B,H,W,3] and normalisation constants'
        if pad_left is None:
            pad_left = 0 if dst_view.W == W // 2 else 1
        mean = (ctypes.c_float * 3)(*[float(v) for v in norm['mean']])
        std = (ctypes.c_float * 3)(*[float(v) for v in norm['std']])
        _lib.check(_lib.lib().cvb_stem_s2d_u8(x.data_ptr(), B, H, W, mean, std, 1 if norm.get('reverse_channels', True) else 0,
                                              byref(dst_view), pad_left, _stream()), 'cvb_stem_s2d_u8')
        return
    assert x.dtype == torch.float32
    B, C, H, W = x.shape
    assert C == 3
    if pad_left is None:
        pad_left = 0 if dst_view.W == W // 2 else 1
    _lib.check(_lib.lib().cvb_stem_s2d(x.data_ptr(), B, H, W, byref(dst_view), pad_left, _stream()), 'cvb_stem_s2d')


def maxpool3x3s2(x_view, y_view):
    _lib.check(_lib.lib().cvb_maxpool3x3s2(byref(x_view), byref(y_view), _stream()), 'cvb_maxpool3x3s2')


def split_to_f32(x_view, y_view):
    _lib.check(_lib.lib().cvb_split_to_f32nhwc(byref(x_view), byref(y_view), _stream()), 'cvb_split_to_f32nhwc')


class GroupNormWorkspace:
    def __init__(self, B, groups, device='cuda'):
        self.nbytes = int(_lib.lib().cvb_groupnorm_workspace_bytes(B, groups))
        self.buf = torch.zeros(self.nbytes // 8, dtype=torch.float64, device=device)


def groupnorm_relu(x_view, groups, gamma, beta, eps, y_view, ws, relu=True):
    _lib.check(_lib.lib().cvb_groupnorm_relu(byref(x_view), groups, gamma.data_ptr(), beta.data_ptr(), float(eps), 1 if relu else 0,
                                             byref(y_view), ws.buf.data_ptr(), ws.nbytes, _stream()), 'cvb_groupnorm_relu')


def sppf_pool(x, y1, y2, y3):
    _lib.check(_lib.lib().cvb_sppf_pool(byref(x), byref(y1), byref(y2), byref(y3), _stream()), 'cvb_sppf_pool')


def yolo_decode(raw_view, na, no, anchors_px, stride, z, z_rows, z_off, xperm=None, nms_ws=None, conf_thres=0.001, multi_label=True):
    """nms_ws: NmsWorkspace previously reset with nms_reset(); the decode then also fills the NMS score histogram."""
    _lib.check(_lib.lib().cvb_yolo_decode(byref(raw_view), na, no, anchors_px.data_ptr(), float(stride),
                                          z.data_ptr() if z is not None else None, z_rows, z_off,
                                          xperm.data_ptr() if xperm is not None else None,
                                          nms_ws.ws_ptr if nms_ws is not None else None, float(conf_thres),
                                          1 if multi_label else 0, _stream()), 'cvb_yolo_decode')


def yolov6_decode(cls_view, reg_view, nc, stride, z, z_rows, z_off, nms_ws=None, conf_thres=0.001, multi_label=True):
    """One YOLOv6 head level (fp32 NHWC class logits and ltrb distances) -> rows z_off .. z_off + h*w of z [B, z_rows, 5 + nc].
    nms_ws: NmsWorkspace previously reset with nms_reset(); the decode then also fills the NMS score histogram (yolo_nms hist_ready)."""
    _require_cuda(z, 'yolov6_decode')
    assert z.dtype == torch.float32 and z.is_contiguous() and tuple(z.shape[1:]) == (z_rows, nc + 5)
    _lib.check(_lib.lib().cvb_yolov6_decode(byref(cls_view), byref(reg_view), nc, float(stride), z.data_ptr(), z_rows, z_off,
                                            nms_ws.ws_ptr if nms_ws is not None else None, float(conf_thres), 1 if multi_label else 0,
                                            _stream()), 'cvb_yolov6_decode')


def depth_to_space2(src_view, dst_view):
    """split16 [B,h,w,4c] (channel (py*2+px)*c + o) -> split16 [B,2h,2w,c] (pixel (2y+py, 2x+px)), values copied exactly."""
    _lib.check(_lib.lib().cvb_depth_to_space2(byref(src_view), byref(dst_view), _stream()), 'cvb_depth_to_space2')


def nms_reset(ws):
    _lib.check(_lib.lib().cvb_nms_workspace_reset(ws.ws_ptr, ws.ws_bytes, ws.B, _stream()), 'cvb_nms_workspace_reset')


class NmsWorkspace:
    def __init__(self, B, A, nc, max_det=300, device='cuda'):
        self.B, self.A, self.nc, self.max_det = B, A, nc, max_det
        nbytes = int(_lib.lib().cvb_nms_workspace_bytes(B, A, nc))
        self.ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=device)
        off = (-self.ws.data_ptr()) % 256
        self.ws_ptr = self.ws.data_ptr() + off
        self.ws_bytes = nbytes
        # ONE flat result buffer [det B*M*6 f32 | det_idx B*M i32 | det_count B i32]: the three outputs are views of it, so the NMS
        # kernels write the wire format of the multi-GPU all-gather directly (dist.all_gather_packed; no packing kernels per step)
        M = max_det
        self.packed = torch.zeros((B * M * 7 + B,), dtype=torch.float32, device=device)
        self.det = self.packed[:B * M * 6].view(B, M, 6)
        self.det_idx = self.packed[B * M * 6:B * M * 7].view(torch.int32).view(B, M)
        self.det_count = self.packed[B * M * 7:].view(torch.int32)
        self.status = torch.zeros((4,), dtype=torch.int32, device=device)


def yolo_nms(prediction, ws, conf_thres=0.001, iou_thres=0.6, multi_label=True, max_nms=30000, max_wh=4096.0, hist_ready=False):
    """Batched NMS on device.  Returns (det [B,max_det,6], det_idx [B,max_det], det_count [B]) -- device tensors
    owned by `ws`; no host synchronisation happens here."""
    _require_cuda(prediction, 'yolo_nms')
    assert prediction.dtype == torch.float32 and prediction.is_contiguous()
    B, A, no = prediction.shape
    assert (B, A, no - 5) == (ws.B, ws.A, ws.nc)
    p = CvbNmsParams()
    p.B, p.A, p.nc = B, A, no - 5
    p.conf_thres, p.iou_thres = conf_thres, iou_thres
    p.multi_label = 1 if multi_label else 0
    p.max_nms, p.max_det, p.max_wh = max_nms, ws.max_det, max_wh
    p.hist_ready = 1 if hist_ready else 0
    _lib.check(_lib.lib().cvb_yolo_nms(prediction.data_ptr(), byref(p), ws.det.data_ptr(), ws.det_idx.data_ptr(),
                                       ws.det_count.data_ptr(), ws.ws_ptr, ws.ws_bytes, ws.status.data_ptr(), _stream()),
               'cvb_yolo_nms')
    return ws.det, ws.det_idx, ws.det_count


# --------------------------------------------------------------------------------------- FCOS post-processing
class FcosWorkspace:
    """Caller-owned buffers of the FCOS decode + top-k + NMS stage (fixed capacity, no host sync)."""

    def __init__(self, B, N, topk=1000, device='cuda'):
        self.B, self.N, self.topk = B, N, topk
        self.scores = torch.zeros((B, N), dtype=torch.float32, device=device)
        self.classes = torch.zeros((B, N), dtype=torch.int32, device=device)
        self.boxes = torch.zeros((B, N, 4), dtype=torch.float32, device=device)
        self.out_scores = torch.zeros((B, topk), dtype=torch.float32, device=device)
        self.out_classes = torch.zeros((B, topk), dtype=torch.int32, device=device)
        self.out_boxes = torch.zeros((B, topk, 4), dtype=torch.float32, device=device)
        self.out_loc = torch.zeros((B, topk), dtype=torch.int32, device=device)
        self.out_count = torch.zeros((B,), dtype=torch.int32, device=device)
        self.status = torch.zeros((4,), dtype=torch.int32, device=device)


def fcos_decode(cls_view, regcnt_view, nc, stride, scale, ws, loc_off):
    _lib.check(_lib.lib().cvb_fcos_decode(byref(cls_view), byref(regcnt_view), nc, float(stride), float(scale), ws.scores.data_ptr(),
                                          ws.classes.data_ptr(), ws.boxes.data_ptr(), ws.N, loc_off, _stream()), 'cvb_fcos_decode')


def fcos_nms(ws, score_thres=0.05, iou_thres=0.6, scores=None, classes=None, boxes=None):
    s = ws.scores if scores is None else scores
    c = ws.classes if classes is None else classes
    b = ws.boxes if boxes is None else boxes
    _lib.check(_lib.lib().cvb_fcos_nms(s.data_ptr(), c.data_ptr(), b.data_ptr(), ws.B, ws.N, float(score_thres), float(iou_thres), ws.topk,
                                       ws.out_scores.data_ptr(), ws.out_classes.data_ptr(), ws.out_boxes.data_ptr(), ws.out_loc.data_ptr(),
                                       ws.out_count.data_ptr(), ws.status.data_ptr(), _stream()), 'cvb_fcos_nms')
    return ws.out_scores, ws.out_classes, ws.out_boxes, ws.out_loc, ws.out_count


# --------------------------------------------------------------------------------------- DeepLab helpers
def pack_dw_weights(w64, b64, device='cuda'):
    """depthwise [C,1,3,3] float64 (BN folded) -> fp32 [9, C] tap-major + fp32 bias [C]."""
    C = w64.shape[0]
    return w64.reshape(C, 9).t().contiguous().float().to(device), b64.float().to(device)


def dwconv3x3(x_view, w9c, bias, dilation, y_view, relu=True):
    _lib.check(_lib.lib().cvb_dwconv3x3(byref(x_view), w9c.data_ptr(), bias.data_ptr(), dilation, 1 if relu else 0, byref(y_view), _stream()),
               'cvb_dwconv3x3')


def global_avgpool(x_view, y_view):
    _lib.check(_lib.lib().cvb_global_avgpool(byref(x_view), byref(y_view), _stream()), 'cvb_global_avgpool')


def bilinear_resize(x_view, y_view):
    _lib.check(_lib.lib().cvb_bilinear_resize(byref(x_view), byref(y_view), _stream()), 'cvb_bilinear_resize')


def upsample_argmax(logits_view, nc, labels):
    B, Ho, Wo = labels.shape
    assert labels.dtype == torch.int64 and labels.is_contiguous()
    _lib.check(_lib.lib().cvb_upsample_argmax(byref(logits_view), nc, labels.data_ptr(), Ho, Wo, _stream()), 'cvb_upsample_argmax')


# --------------------------------------------------------------------------------------- YOLOX post-processing
class YoloxWorkspace:
    """Caller-owned buffers of the YOLOX post-process: candidate records [B,A,8], kept rows det [B,A,7], count [B], NMS scratch."""

    def __init__(self, B, A, device='cuda'):
        self.B, self.A = B, A
        self.cand = torch.zeros((B, A, 8), dtype=torch.float32, device=device)
        self.det = torch.zeros((B, A, 7), dtype=torch.float32, device=device)
        self.count = torch.zeros((B,), dtype=torch.int32, device=device)
        nbytes = int(_lib.lib().cvb_yolox_workspace_bytes(B, A))
        self.scratch = torch.empty((nbytes + 15) // 16 * 4, dtype=torch.float32, device=device)
        self.scratch_bytes = nbytes


def yolox_decode(reg_obj_view, cls_view, num_classes, stride, ws, off):
    _lib.check(_lib.lib().cvb_yolox_decode(byref(reg_obj_view), byref(cls_view), num_classes, float(stride), ws.cand.data_ptr(), ws.A, off,
                                           _stream()), 'cvb_yolox_decode')


def yolox_nms(ws, conf_thres, iou_thres, vanilla_above=1000, cand=None):
    """cand: optional foreign candidate tensor [B,A,8] (tests); default = the records written by yolox_decode."""
    c = ws.cand if cand is None else cand
    assert c.is_cuda and c.dtype == torch.float32 and c.is_contiguous() and tuple(c.shape) == (ws.B, ws.A, 8)
    _lib.check(_lib.lib().cvb_yolox_nms(c.data_ptr(), ws.B, ws.A, float(conf_thres), float(iou_thres), int(vanilla_above), ws.det.data_ptr(),
                                        ws.count.data_ptr(), ws.scratch.data_ptr(), ws.scratch_bytes, _stream()), 'cvb_yolox_nms')
    return ws.det, ws.count


# --------------------------------------------------------------------------------------- output side (SURVEY.md 8 f-2)
def rescale_clip_boxes(rows, count, pads, scales, wh):
    """In place: rows [B,M,>=4] fp32 CUDA (x1,y1,x2,y2 first), count [B] int32, pads / scales / wh [B,2] fp32 CUDA (wh = width, height)."""
    _require_cuda(rows, 'rescale_clip_boxes')
    assert rows.dtype == torch.float32 and rows.is_contiguous() and rows.dim() == 3 and count.dtype == torch.int32
    for t in (pads, scales, wh):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == (rows.shape[0], 2)
    B, M, S = rows.shape
    _lib.check(_lib.lib().cvb_rescale_clip_boxes(rows.data_ptr(), B, M, S, count.data_ptr(), pads.data_ptr(), scales.data_ptr(), wh.data_ptr(),
                                                 _stream()), 'cvb_rescale_clip_boxes')
    return rows


def targets_to_device_geometry(targets, B, default_hw, device):
    """(pads, scales, wh) [B,2] fp32 device tensors from the reference's target dicts (identity when a key is missing)."""
    pads = torch.zeros((B, 2), dtype=torch.float32)
    scales = torch.ones((B, 2), dtype=torch.float32)
    wh = torch.tensor([[float(default_hw[1]), float(default_hw[0])]] * B, dtype=torch.float32)
    for i in range(B):
        t = targets[i] if targets is not None and i < len(targets) else {}
        if 'pads' in t:
            pads[i] = torch.as_tensor(t['pads']).float().cpu()
        if 'scales' in t:
            scales[i] = torch.as_tensor(t['scales']).float().cpu()
        if 'width' in t:
            wh[i, 0] = float(t['width'])
        if 'height' in t:
            wh[i, 1] = float(t['height'])
    return pads.to(device), scales.to(device), wh.to(device)


def val_rows_to_host(rows, count, targets, default_hw):
    """The val post-processing of the YOLO drop-ins: the boxes of rows [B,M,>=4] (a device tensor the caller owns) are rescaled and
    clipped in place to each image's original geometry (targets' pads / scales / width / height), then ONE device->host copy instead
    of one per image.  Returns (rows on the host, count as a list)."""
    pads, scales, wh = targets_to_device_geometry(targets, rows.shape[0], default_hw, rows.device)
    rescale_clip_boxes(rows, count, pads, scales, wh)
    return rows.cpu(), count.cpu().tolist()


def confusion_matrix(gt, pred, num_classes, out=None):
    """out [nc,nc] int64 CUDA (accumulated) += confusion matrix of the int64 CUDA label maps gt / pred (eval_segmentation.py:52-57)."""
    _require_cuda(gt, 'confusion_matrix')
    assert gt.dtype == torch.int64 and pred.dtype == torch.int64 and gt.shape == pred.shape and pred.is_cuda
    gt, pred = gt.contiguous(), pred.contiguous()
    if out is None:
        out = torch.zeros((num_classes, num_classes), dtype=torch.int64, device=gt.device)
    _lib.check(_lib.lib().cvb_confusion_matrix(gt.data_ptr(), pred.data_ptr(), gt.numel(), num_classes, out.data_ptr(), _stream()),
               'cvb_confusion_matrix')
    return out


# --------------------------------------------------------------------------------------- input side (SURVEY.md 8 f-1): letterbox
def letterbox_geometry(h, w, size=(640, 640), scaleup=True):
    """(scale, oh, ow, top, left) of the reference's Resize(keep_ratio=True) (det_transforms.py:177-189; python round() = half to even)."""
    scale = min(size[0] / h, size[1] / w)
    if not scaleup:
        scale = min(scale, 1.0)
    oh, ow = int(round(h * scale)), int(round(w * scale))
    padh, padw = (size[0] - oh) / 2, (size[1] - ow) / 2
    return scale, oh, ow, int(round(padh - 0.1)), int(round(padw - 0.1))


def letterbox_frames(frames, size=(640, 640), fill=(114, 114, 114), scaleup=True, out=None):
    """frames: list of uint8 CUDA tensors [h_i, w_i, 3] (camera frames of different sizes).  Returns (uint8 [B,size0,size1,3] letterboxed
    batch, pads [B,2] (top, left), scales [B,2]) -- the image and the `target["pads"]` / `target["scales"]` entries of the reference's
    Resize transform; the batch feeds YOLOv5.predict_frames (ToTensor + Normalize are fused into the stem loader)."""
    B = len(frames)
    dev = frames[0].device
    geom, pads, scales = [], [], []
    for f in frames:
        _require_cuda(f, 'letterbox_frames')
        assert f.dtype == torch.uint8 and f.dim() == 3 and f.shape[2] == 3 and f.is_contiguous()
        h, w = int(f.shape[0]), int(f.shape[1])
        scale, oh, ow, top, left = letterbox_geometry(h, w, size, scaleup)
        geom.append([h, w, oh, ow, top, left])
        pads.append([top, left])
        scales.append([scale, scale])
    ptrs = torch.tensor([f.data_ptr() for f in frames], dtype=torch.int64).to(dev)
    g = torch.tensor(geom, dtype=torch.int32).to(dev)
    if out is None:
        out = torch.empty((B, size[0], size[1], 3), dtype=torch.uint8, device=dev)
    fl = (ctypes.c_int32 * 3)(*[int(v) for v in fill])
    _lib.check(_lib.lib().cvb_letterbox_u8(ptrs.data_ptr(), g.data_ptr(), B, size[0], size[1], fl, out.data_ptr(), _stream()), 'cvb_letterbox_u8')
    return out, torch.tensor(pads, dtype=torch.float32), torch.tensor(scales, dtype=torch.float32)


# --------------------------------------------------------------------------------------- output side (SURVEY.md 8 f-2): COCO records
def coco_pack(rows, count, image_ids, id2category=None):
    """rows [B,M,>=6] fp32 CUDA (x1,y1,x2,y2,score,class; already rescaled / clipped), count [B] int32, image_ids [B] int64 (CUDA or list),
    id2category: optional list / tensor (dataset.id2category).  Returns (rec_ids [B*M,2] int64, rec_box [B*M,5] f32, total [1] int32) on
    the device: the first `total` records are valid -- eval_coco.py:87-111 without the per-image .tolist() loop."""
    _require_cuda(rows, 'coco_pack')
    assert rows.dtype == torch.float32 and rows.is_contiguous() and rows.dim() == 3 and count.dtype == torch.int32
    B, M, S = rows.shape
    dev = rows.device
    ids = torch.as_tensor(image_ids, dtype=torch.int64).to(dev).contiguous()
    cat = torch.as_tensor(id2category, dtype=torch.int32).to(dev).contiguous() if id2category is not None else None
    rec_ids = torch.zeros((B * M, 2), dtype=torch.int64, device=dev)
    rec_box = torch.zeros((B * M, 5), dtype=torch.float32, device=dev)
    total = torch.zeros((1,), dtype=torch.int32, device=dev)
    _lib.check(_lib.lib().cvb_coco_pack(rows.data_ptr(), B, M, S, count.data_ptr(), ids.data_ptr(), cat.data_ptr() if cat is not None else None,
                                        int(cat.numel()) if cat is not None else 0, rec_ids.data_ptr(), rec_box.data_ptr(), total.data_ptr(), _stream()),
               'cvb_coco_pack')
    return rec_ids, rec_box, total


# --------------------------------------------------------------------------------------- output side: COCO box mAP (csrc/coco_eval.cu)
def coco_eval_bbox(gt_key, gt_box, gt_area, gt_crowd, img_evaluated, det_img, det_cat, det_score, det_box, n_cats, iou_thrs, rec_thrs):
    """pycocotools COCOeval (bbox, default parameters) evaluate + accumulate + summarize on the device.  Ground truths: gt_key [G] int32
    (category index * n_images + image index, ascending, annotation order within a key), gt_box [G,4] xywh float64, gt_area [G] float64,
    gt_crowd [G] uint8.  img_evaluated [n_images] uint8 (images by ascending id).  Detections: det_img / det_cat [N] int32 (category -1:
    not evaluated), det_score [N] fp32, det_box [N,4] xywh float64.  All CUDA, contiguous.  Returns device tensors precision
    [10,101,K,4,3], recall [10,K,4,3], stats [12] (float64) and det_masks [N,4] int32 (bits 0..9 matched, 16..25 ignored per threshold)."""
    n_images, n_gt, n_det = img_evaluated.numel(), gt_key.numel(), det_img.numel()
    for name, lim, v in (('images', _lib.CVB_COCO_MAX_IMAGES, n_images), ('categories', _lib.CVB_COCO_MAX_CATS, n_cats),
                         ('ground truths', _lib.CVB_COCO_MAX_GT, n_gt), ('detections', _lib.CVB_COCO_MAX_DETS, n_det)):
        if v > lim:
            raise _lib.CvbError(f'coco_eval_bbox: {v} {name} exceed the limit of {lim}')
    specs = ((gt_key, torch.int32, (n_gt,)), (gt_box, torch.float64, (n_gt, 4)), (gt_area, torch.float64, (n_gt,)), (gt_crowd, torch.uint8, (n_gt,)),
             (img_evaluated, torch.uint8, (n_images,)), (det_img, torch.int32, (n_det,)), (det_cat, torch.int32, (n_det,)),
             (det_score, torch.float32, (n_det,)), (det_box, torch.float64, (n_det, 4)))
    for t, dtype, shape in specs:
        _require_cuda(t, 'coco_eval_bbox')
        if t.dtype != dtype or tuple(t.shape) != shape or not t.is_contiguous() or t.device != img_evaluated.device:
            raise _lib.CvbError(f'coco_eval_bbox: expected a contiguous {dtype} {shape} tensor on {img_evaluated.device}, got {t.dtype} '
                                f'{tuple(t.shape)} on {t.device}')
    dev = img_evaluated.device
    p = _lib.CvbCocoEvalParams(n_images, n_cats, n_gt, n_det)
    p.iou_thrs[:] = [float(x) for x in iou_thrs]
    p.rec_thrs[:] = [float(x) for x in rec_thrs]
    ws_bytes = _lib.lib().cvb_coco_eval_workspace_bytes(n_det, n_gt, n_cats)
    if ws_bytes == 0:
        raise _lib.CvbError(f'coco_eval_bbox: sizes outside the limits (n_det={n_det}, n_gt={n_gt}, n_cats={n_cats})')
    ws = torch.empty(ws_bytes + 256, dtype=torch.uint8, device=dev)
    ws_ptr = (ws.data_ptr() + 255) & ~255
    precision = torch.empty((10, 101, n_cats, 4, 3), dtype=torch.float64, device=dev)
    recall = torch.empty((10, n_cats, 4, 3), dtype=torch.float64, device=dev)
    stats = torch.empty((12,), dtype=torch.float64, device=dev)
    masks = torch.empty((n_det, 4), dtype=torch.int32, device=dev)
    ptr = lambda t: t.data_ptr() if t.numel() else None  # noqa: E731
    _lib.check(_lib.lib().cvb_coco_eval_bbox(ctypes.byref(p), ptr(gt_key), ptr(gt_box), ptr(gt_area), ptr(gt_crowd), img_evaluated.data_ptr(),
                                             ptr(det_img), ptr(det_cat), ptr(det_score), ptr(det_box), ptr(masks), precision.data_ptr(),
                                             recall.data_ptr(), stats.data_ptr(), ws_ptr, ws_bytes, _stream()), 'cvb_coco_eval_bbox')
    return precision, recall, stats, masks


# --------------------------------------------------------------------------------------- output side: segmentation confusion matrix (csrc/seg_eval.cu)
SEG_DTYPES = {torch.uint8: _lib.CVB_SEG_U8, torch.int32: _lib.CVB_SEG_I32, torch.int64: _lib.CVB_SEG_I64}


def seg_nc_max():
    """The largest class count cvb_seg_confusion_update accepts (nc² uint32 bins in one CTA's shared memory)."""
    return int(_lib.lib().cvb_seg_confusion_nc_max())


def seg_confusion_update(gt, pred, nc, matrix, err):
    """matrix [nc,nc] uint64 CUDA += the confusion matrix of the label maps gt / pred (uint8, int32 or int64, any shape, equal numel) by
    eval_segmentation.py's rule: pixels with 0 <= gt < nc count at flat index nc * gt + pred; flat indices outside [0, nc²) OR bit 0
    (negative) or bit 1 (too large) into err (int32 CUDA, first element).  Non-contiguous maps are made contiguous on the device; no host
    sync.  Batches above 2^31 - 1 pixels are counted in several launches."""
    for t in (gt, pred, matrix, err):
        _require_cuda(t, 'seg_confusion_update')
    dev = matrix.device
    if gt.device != dev or pred.device != dev or err.device != dev:
        raise _lib.CvbError(f'seg_confusion_update: gt on {gt.device}, pred on {pred.device}, err on {err.device}, the matrix on {dev}')
    if gt.dtype not in SEG_DTYPES or pred.dtype not in SEG_DTYPES:
        raise TypeError(f'seg_confusion_update: label maps must be uint8, int32 or int64 (got gt {gt.dtype}, pred {pred.dtype})')
    if gt.numel() != pred.numel():
        raise ValueError(f'seg_confusion_update: gt has {gt.numel()} elements and pred {pred.numel()}')
    if matrix.dtype != torch.uint64 or tuple(matrix.shape) != (nc, nc) or not matrix.is_contiguous():
        raise _lib.CvbError(f'seg_confusion_update: matrix must be a contiguous uint64 [{nc}, {nc}] tensor (got {matrix.dtype} {tuple(matrix.shape)})')
    if err.dtype != torch.int32 or err.numel() < 1:
        raise _lib.CvbError(f'seg_confusion_update: err must be an int32 tensor (got {err.dtype} with {err.numel()} elements)')
    gt, pred = gt.contiguous().view(-1), pred.contiguous().view(-1)
    n = gt.numel()
    for off in range(0, n, _lib.CVB_SEG_MAX_N):
        k = min(_lib.CVB_SEG_MAX_N, n - off)
        _lib.check(_lib.lib().cvb_seg_confusion_update(gt[off:].data_ptr(), SEG_DTYPES[gt.dtype], pred[off:].data_ptr(), SEG_DTYPES[pred.dtype], k, nc,
                                                       matrix.data_ptr(), err.data_ptr(), _stream()), 'cvb_seg_confusion_update')
