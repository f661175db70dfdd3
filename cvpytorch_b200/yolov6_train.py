"""YOLOv6 training on the H100 kernels: the loss (csrc/yolov6_loss.cu) and the YOLOv6-n / -s network (csrc/train_kernels.cu).

  YOLOv6Loss          src/losses/det/yolov6_loss.py: target packing, the ATSS (warm-up) or task-aligned assignment and the GIoU / SIoU box
                      loss with its gradient with respect to pred_distri, with no host sync (forward and backward can be captured in a CUDA graph)
  RepVGGBlock         src/models/modules/yolo_modules.py:268-327   relu(bn(conv3x3) + bn(conv1x1) [+ bn(x)]), batch statistics per branch
  RepBlock            :453-471
  ConvModule          conv -> BatchNorm -> ReLU (stride 1 or 2) of the backbone and neck
  SimCSPSPPF          :218-242
  BiFusion            :245-265   ConvTranspose2d(c, c, 2, stride 2) | cv1 | downsample(cv2) -> cv3
  YOLOv6EfficientRep  src/models/backbones/det/yolov6_efficient_rep.py:20-70
  YOLOv6RepBiPAN      src/models/necks/det/yolov6_repbipan.py:16-82
  YOLOv6Effidehead    src/models/heads/det/yolov6_effidehead.py:17-148, training forward (:126-147)

The network modules keep the inference modules' constructors and state_dict keys (yolov6_models.py, yolo_blocks.py); activations are NHWC
bf16 (forward_nhwc), as in yolov5_train.py.  A RepVGG block's two convolutions run on the conv kernel, each branch's statistics come from
cvb_train_bn_stats and one pass sums the branches and applies ReLU (cvb_train_repvgg_fwd); its backward is one reduce and one apply pass
(cvb_train_repvgg_bwd) before the convolutions' backward.  A stride-2 1x1 branch (the stem and the four downsamples) runs as the centre tap
of a 3x3 / stride-2 / pad-1 conv: its weight is zero-padded in torch, so autograd returns the 1x1 gradient.  The stem RepVGGBlock(3, c,
stride 2) runs over train.focus_s2d's map with both branch weights remapped in torch (stem_weight_to_s2d).  BiFusion's transposed conv is a
1x1 GEMM of 4c columns followed by cvb_train_convt_scatter; its backward gathers d(out) back (cvb_train_convt_gather).  YOLOv6-n's
96-channel bifusion1.cv3 input is zero-padded to 128 channels, and so is its weight (autograd slices the gradient).

nn.SyncBatchNorm (convert_sync_batchnorm, as the reference trainer does under cfg.distributed) normalises over every rank of its process
group, decided at every forward by train._sync_group.  A ReLU ConvModule takes train._conv_bn_silu's record -> all-gather -> merge path and
cvb_train_bn_relu_bwd_reduce -> all-reduce -> _apply.  A RepVGG block gathers and merges one record per branch (the identity branch's on the
block input) and all-reduces one [4][C] buffer in backward (cvb_train_repvgg_bwd_reduce / _apply); its three BatchNorms must all be local
or all share one process group, otherwise it raises NotImplementedError.  Without a process group (or in a world of one) the step issues
the same launches as with nn.BatchNorm2d.

The loss: head outputs are cast with .float().contiguous(), so fp16 / bf16 outputs under autocast work and their
gradients flow back through the cast.  The reference returns {'iou': 2.5 L, 'dfl': 0.5 L, 'class': 1.0 L} of its box loss L (its class
loss is computed and discarded), so pred_scores gets no gradient.  No CPU fallback: CPU tensors raise CvbError.  Divergences, each
documented in include/cvb200.h: the dict entries are fp64 also without positives (the reference returns fp32 there); rows whose image
index truncates outside [0, B) are dropped (the reference wraps -1); labels outside [0, nc) give a zero class score (the reference
raises); a level with fewer than 9 anchors takes all of them as ATSS candidates (the reference raises); on equal values at the top-k
boundary the lowest anchor index wins (torch.topk's order is undefined).
"""
import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, train
from .train import (_bn_momentum, _check_cuda, _ConvBnSiLULayer, _p, _require_training, _require_widths, _set_bn, _SppfChain, _stream, _sync_group,
                    _workspace, batch_stats, conv, conv_dgrad_s2, conv_wgrad, focus_s2d, pack_weights)
from .yolov5_train import _PredConv

LOSS_WEIGHT = {'class': 1.0, 'iou': 2.5, 'dfl': 0.5}


def loss_params(shapes, strides, nc, B, assigner, iou_type, grid_cell_size=5.0, grid_cell_offset=0.5, ori_img_size=640,
                loss_weight=LOSS_WEIGHT):
    """The CvbYolov6LossParams of level shapes [(h, w)], strides, nc, batch, assigner ('atss' / 'tal') and iou_type ('giou' / 'siou')."""
    if len(shapes) != len(strides) or not 1 <= len(shapes) <= _lib.CVB_YOLOV6_MAX_LEVELS:
        raise ValueError(f'YOLOv6Loss: {len(strides)} strides for {len(shapes)} feature maps (1 to {_lib.CVB_YOLOV6_MAX_LEVELS} levels)')
    p = _lib.CvbYolov6LossParams()
    p.B, p.nc, p.nlev = int(B), int(nc), len(shapes)
    for l, ((h, w), s) in enumerate(zip(shapes, strides)):
        p.h[l], p.w[l], p.strides[l] = int(h), int(w), float(s)
    p.grid_cell_size, p.grid_cell_offset, p.ori_img_size = float(grid_cell_size), float(grid_cell_offset), float(ori_img_size)
    p.assigner = {'atss': _lib.CVB_YOLOV6_ATSS, 'tal': _lib.CVB_YOLOV6_TAL}[assigner]
    p.iou_type = {'giou': _lib.CVB_YOLOV6_GIOU, 'siou': _lib.CVB_YOLOV6_SIOU}[iou_type]
    p.loss_weight[0], p.loss_weight[1], p.loss_weight[2] = (float(loss_weight[k]) for k in ('iou', 'dfl', 'class'))
    return p


def yolov6_loss_forward(params, pred_scores, pred_distri, gt):
    """pred_scores fp32 [B, A, nc], pred_distri fp32 [B, A, 4], gt fp64 [nt, 6] (CUDA, contiguous) -> (out fp64 [3] = iou, dfl, class,
    assignment dict: fg uint8 [B, A], gt_idx / labels int32 [B, A], boxes fp64 [B, A, 4], scores fp64 [B, A], stats fp64 [4] =
    (sum soft label (1 - IoU), target_scores_sum, num_pos, sum pred_distri))."""
    B, A = pred_distri.shape[:2]
    dev = pred_distri.device
    nt = gt.shape[0]
    ws = _workspace(_lib.lib().cvb_train_yolov6_loss_workspace_bytes(params, nt), dev)
    r = dict(fg=torch.empty((B, A), dtype=torch.uint8, device=dev), gt_idx=torch.empty((B, A), dtype=torch.int32, device=dev),
             labels=torch.empty((B, A), dtype=torch.int32, device=dev), boxes=torch.empty((B, A, 4), dtype=torch.float64, device=dev),
             scores=torch.empty((B, A), dtype=torch.float64, device=dev), stats=torch.empty((4,), dtype=torch.float64, device=dev))
    out = torch.empty((3,), dtype=torch.float64, device=dev)
    _lib.check(_lib.lib().cvb_train_yolov6_loss_fwd(params, _p(pred_scores), _p(pred_distri), _p(gt) if nt else None, nt, _p(r['fg']),
                                                    _p(r['gt_idx']), _p(r['labels']), _p(r['boxes']), _p(r['scores']), _p(r['stats']), _p(out),
                                                    _p(ws), ws.numel(), _stream()), 'cvb_train_yolov6_loss_fwd')
    return out, r


def yolov6_loss_backward(params, pred_distri, assignment, grad_out):
    """d(sum_k grad_out[k] out[k]) / d(pred_distri) under the forward's assignment -> fp32 [B, A, 4]."""
    g = torch.empty_like(pred_distri)
    a = assignment
    _lib.check(_lib.lib().cvb_train_yolov6_loss_bwd(params, _p(pred_distri), _p(a['fg']), _p(a['boxes']), _p(a['scores']), _p(a['stats']),
                                                    _p(grad_out), _p(g), _stream()), 'cvb_train_yolov6_loss_bwd')
    return g


class _YOLOv6LossFn(torch.autograd.Function):
    """out fp64 [3] of pred_distri; the assignment is kept for the backward.  pred_scores only feeds the TAL metric: no gradient."""

    @staticmethod
    def forward(ctx, params, gt, pred_scores, pred_distri):
        out, a = yolov6_loss_forward(params, pred_scores, pred_distri, gt)
        ctx.params = params
        ctx.save_for_backward(pred_distri, a['fg'], a['boxes'], a['scores'], a['stats'])
        return out

    @staticmethod
    def backward(ctx, g):
        pred_distri, fg, boxes, scores, stats = ctx.saved_tensors
        gd = yolov6_loss_backward(ctx.params, pred_distri, dict(fg=fg, boxes=boxes, scores=scores, stats=stats), g.double().contiguous())
        return None, None, None, gd


def _gt_rows(targets, device):
    t = targets['gt'] if isinstance(targets, dict) else targets
    if not isinstance(t, torch.Tensor) or t.dim() != 2 or t.shape[1] != 6:
        raise ValueError('YOLOv6Loss: targets must be a [n, 6] tensor of (image, label, cx, cy, w, h) rows')
    if t.shape[0]:
        _check_cuda(t, 'YOLOv6Loss targets')
    return t.detach().to(device=device, dtype=torch.float64).contiguous()


class YOLOv6Loss(nn.Module):
    """src/losses/det/yolov6_loss.py YOLOv6Loss on the H100 kernels: same constructor and the same `proj` parameter (shape (reg_max + 1,)).
    forward(outputs, targets, epoch_num=0, step_num=0) with outputs = (feats, pred_scores [B, A, nc], pred_distri [B, A, 4]) and targets
    the [n, 6] rows (image, label, cx, cy, w, h normalised by ori_img_size) returns {'iou', 'dfl', 'class'} fp64 device scalars.  feats
    only give the level shapes; step_num is unused.  ATSS runs while epoch_num < warmup_epoch, the task-aligned assigner after."""

    def __init__(self, num_classes=80, fpn_strides=[8, 16, 32], grid_cell_size=5.0, grid_cell_offset=0.5, ori_img_size=640, warmup_epoch=4,
                 use_dfl=False, reg_max=16, iou_type='giou', loss_weight={'class': 1.0, 'iou': 2.5, 'dfl': 0.5}):
        super().__init__()
        self.num_classes, self.fpn_strides = num_classes, list(fpn_strides)
        self.grid_cell_size, self.grid_cell_offset, self.ori_img_size = grid_cell_size, grid_cell_offset, ori_img_size
        self.warmup_epoch, self.use_dfl, self.reg_max = warmup_epoch, use_dfl, reg_max
        self.iou_type, self.loss_weight = iou_type.lower(), dict(loss_weight)
        self.proj = nn.Parameter(torch.linspace(0, reg_max, reg_max + 1), requires_grad=False)
        if use_dfl:
            raise NotImplementedError('YOLOv6Loss (H100): use_dfl=True (the distribution focal loss) is not supported')
        if self.iou_type not in ('giou', 'siou'):
            raise NotImplementedError(f"YOLOv6Loss (H100): iou_type '{iou_type}' is not supported ('giou' and 'siou' are)")

    def forward(self, outputs, targets, epoch_num=0, step_num=0):
        feats, pred_scores, pred_distri = outputs
        _check_cuda(pred_scores, 'YOLOv6Loss pred_scores')
        _check_cuda(pred_distri, 'YOLOv6Loss pred_distri')
        shapes = [tuple(f.shape[-2:]) for f in feats]
        B, A = pred_distri.shape[:2]
        if pred_distri.dim() != 3 or pred_distri.shape[2] != 4 or tuple(pred_scores.shape) != (B, A, self.num_classes):
            raise ValueError(f'YOLOv6Loss: pred_scores must be [B, A, {self.num_classes}] and pred_distri [B, A, 4] '
                             f'(got {tuple(pred_scores.shape)}, {tuple(pred_distri.shape)})')
        if sum(h * w for h, w in shapes) != A:
            raise ValueError(f'YOLOv6Loss: the feature maps {shapes} give {sum(h * w for h, w in shapes)} anchors, the predictions {A}')
        params = loss_params(shapes, self.fpn_strides, self.num_classes, B, 'atss' if epoch_num < self.warmup_epoch else 'tal', self.iou_type,
                             self.grid_cell_size, self.grid_cell_offset, self.ori_img_size, self.loss_weight)
        gt = _gt_rows(targets, pred_distri.device)
        out = _YOLOv6LossFn.apply(params, gt, pred_scores.detach().float().contiguous(), pred_distri.float().contiguous())
        return {'iou': out[0], 'dfl': out[1], 'class': out[2]}



# ================================================================================================ network
_WIDTHS = 'channels must be 16, 32 or multiples of 64'


def _bn_args(bn):
    """Counts the step -> (running_mean, running_var, eps, momentum, process group) of a BatchNorm with batch statistics: the group whose
    ranks' pixels it normalises over (train._sync_group), or None (this device's pixels)."""
    return bn.running_mean, bn.running_var, bn.eps, _bn_momentum(bn), _sync_group(bn)


def stem_weight_to_s2d(w):
    """fp32 [cout, 3, 3, 3] weight of a 3x3 / stride-2 / pad-1 conv -> [cout, 16, 3, 3] of the 3x3 / stride-1 / pad-1 conv over train.focus_s2d's
    map (channel 3 (2 dx + dy) + c: Focus's patch order tl, bl, tr, br; channels 12..15 zero).  Output row oy reads input rows 2 oy - 1
    (ky = 0: s2d row oy - 1, dy = 1), 2 oy (ky = 1: row oy, dy = 0) and 2 oy + 1 (ky = 2: row oy, dy = 1), likewise for columns; s2d tap 2 is
    zero.  yolov6_models.repvgg_stem_weights_to_s2d for this patch order, as torch indexing, so autograd maps the gradient back onto w."""
    if w.device not in _S2D_INDEX:  # (built once per device, so that a CUDA-graph capture copies nothing from the host)
        tap = {0: (0, 1), 1: (1, 0), 2: (1, 1)}  # kernel index -> (s2d tap, sub-pixel offset)
        rows = [((2 * dx + dy) * 3 + c, ta, tb, c, ky, kx) for ky, (ta, dy) in tap.items() for kx, (tb, dx) in tap.items() for c in range(3)]
        _S2D_INDEX[w.device] = torch.tensor(rows, dtype=torch.long).T.contiguous().to(w.device)
    dst_c, dst_a, dst_b, src_c, src_y, src_x = _S2D_INDEX[w.device]
    out = w.new_zeros((w.shape[0], 16, 3, 3))
    out[:, dst_c, dst_a, dst_b] = w[:, src_c, src_y, src_x]
    return out


_S2D_INDEX = {}


def repvgg_forward(x, w3, w1, bn3, bn1, bnid, stride, group=None):
    """a = relu(bn3(conv3x3(x, w3)) + bn1(conv(x, w1)) [+ bnid(x)]) with batch statistics -> (a, saved tensors of repvgg_backward, count).
    w1 is [cout, cin, 1, 1], or 3x3 (the zero-padded stride-2 1x1 branch).  bn*: (gamma, beta, running_mean, running_var, eps, momentum);
    bnid None: no identity branch.  group: the process group of all three BatchNorms (SyncBatchNorm: each branch's statistics span its
    ranks, and count is the global pixel count on the device, which the branches share), or None (this device's pixels; count None).
    Updates the running statistics."""
    B, H, W, cin = x.shape
    cout = w3.shape[0]
    wf3, wb3 = pack_weights(w3)
    wf1, wb1 = pack_weights(w1)
    y3 = conv(x, wf3, cout, 3, stride=stride)
    y1 = conv(x, wf1, cout, w1.shape[2], stride=stride)
    st3, g3, count = batch_stats(y3, *bn3, group)
    st1, g1, _ = batch_stats(y1, *bn1, group)
    stid, gid, _ = batch_stats(x, *bnid, group) if bnid is not None else (None, None, None)
    a = torch.empty_like(y3)
    _lib.check(_lib.lib().cvb_train_repvgg_fwd(_p(y3), _p(y1), _p(x) if bnid is not None else None, a.numel() // cout, cout, _p(st3), _p(st1), _p(stid),
                                               _p(a), _stream()), 'cvb_train_repvgg_fwd')
    return a, (y3, y1, st3, st1, stid, g3, g1, gid, wb3, wb1), count


def repvgg_backward(g, x, a, saved, need_dx, stride, group=None, count=None):
    """g = d(loss)/d(a) -> (dx or None, dw3, dw1, dgamma3, dgamma1, dgamma_id or None, dbeta): dbeta is every branch's beta gradient.  With
    a process group (SyncBatchNorm): dgamma and dbeta stay this rank's sums (DDP averages them like every other gradient); the dy of every
    branch takes the sums over every rank (one all-reduce of the [4][C] sums) and the forward's global pixel count `count`."""
    y3, y1, st3, st1, stid, g3, g1, gid, wb3, wb1 = saved
    B, H, W, cin = x.shape
    cout = y3.shape[3]
    npix = a.numel() // cout
    ident = stid is not None
    L = _lib.lib()
    g = g.contiguous()
    sums = torch.empty((4, cout), dtype=torch.float32, device=x.device)
    dy3, dy1 = torch.empty_like(y3), torch.empty_like(y1)
    dxid = torch.empty_like(x) if ident else None
    xid = _p(x) if ident else None
    if group is None:
        _lib.check(L.cvb_train_repvgg_bwd(_p(g), _p(a), _p(y3), _p(y1), xid, npix, cout, _p(st3), _p(st1), _p(stid), _p(g3), _p(g1), _p(gid), _p(sums),
                                          _p(dy3), _p(dy1), _p(dxid), _stream()), 'cvb_train_repvgg_bwd')
        local = sums
    else:
        _lib.check(L.cvb_train_repvgg_bwd_reduce(_p(g), _p(a), _p(y3), _p(y1), xid, npix, cout, _p(st3), _p(st1), _p(stid), _p(sums), _stream()),
                   'cvb_train_repvgg_bwd_reduce')
        local = sums.clone()
        dist.all_reduce(sums, group=group)
        _lib.check(L.cvb_train_repvgg_bwd_apply(_p(g), _p(a), _p(y3), _p(y1), xid, npix, cout, _p(st3), _p(st1), _p(stid), _p(g3), _p(g1), _p(gid),
                                                _p(sums), _p(count), _p(dy3), _p(dy1), _p(dxid), _stream()), 'cvb_train_repvgg_bwd_apply')
    k1 = 3 if wb1.shape[1] == 9 else 1  # (the stride-2 1x1 branch runs as a zero-padded 3x3)
    dw3 = conv_wgrad(x, dy3, 3, stride)
    dw1 = conv_wgrad(x, dy1, k1, stride)
    dx = None
    if need_dx:
        if stride == 2:
            dx = conv_dgrad_s2(dy3, wb3, cin, H, W) + conv_dgrad_s2(dy1, wb1, cin, H, W)
        else:
            dx = conv(dy3, wb3, cin, 3) + conv(dy1, wb1, cin, k1)
            if ident:
                dx = dx + dxid
    return dx, dw3, dw1, local[1].clone(), local[2].clone(), local[3].clone() if ident else None, local[0]


class _RepVGG(torch.autograd.Function):
    """One RepVGG block in training form (forward: repvgg_forward, backward: repvgg_backward).  meta = (running statistics, eps and momentum
    of the three BatchNorms (None: no identity branch), stride, process group of the block's BatchNorms or None)."""

    @staticmethod
    def forward(ctx, x, w3, w1, g3, b3, g1, b1, gid, bid, meta):
        _check_cuda(x, 'RepVGGBlock (H100 training)')
        m3, m1, mid, stride, group = meta
        a, saved, count = repvgg_forward(x, w3, w1, (g3, b3, *m3), (g1, b1, *m1), (gid, bid, *mid) if mid is not None else None, stride, group)
        ctx.save_for_backward(x, a, *saved)
        ctx.stride, ctx.need_dx = stride, x.requires_grad
        ctx.group, ctx.count = group, count
        return a

    @staticmethod
    def backward(ctx, g):
        x, a, *saved = ctx.saved_tensors
        dx, dw3, dw1, dg3, dg1, dgid, dbeta = repvgg_backward(g, x, a, saved, ctx.need_dx, ctx.stride, ctx.group, ctx.count)
        return dx, dw3, dw1, dg3, dbeta.clone(), dg1, dbeta.clone(), dgid, dbeta.clone() if dgid is not None else None, None


class _ConvBn(nn.Module):
    """A RepVGG branch's conv (no bias) + BatchNorm, with the inference ConvModule's keys (conv.weight, bn.*)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride, padding):
        super().__init__()
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride, padding, bias=False)
        self.bn = nn.BatchNorm2d(out_channels)


class RepVGGBlock(nn.Module):
    """yolo_modules.py:268-327 in training form (deploy=False), the keys of yolo_blocks.RepVGGBlock.  forward: NHWC bf16 in / out; stride 1
    or 2 (the 1x1 branch of a stride-2 block is the centre tap of a zero-padded 3x3)."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, padding=1, dilation=1, groups=1, padding_mode='zeros', deploy=False,
                 use_se=False):
        super().__init__()
        if kernel_size != 3 or padding != 1 or dilation != 1 or groups != 1 or padding_mode != 'zeros' or use_se or stride not in (1, 2):
            raise NotImplementedError('H100 training RepVGGBlock: 3x3 / pad 1 / groups 1, stride 1 or 2, no SE')
        if deploy:
            raise NotImplementedError('H100 training RepVGGBlock: a deployed (re-parameterised) block has no training form')
        _require_widths((in_channels, out_channels), lambda bad: f'H100 training RepVGGBlock: {_WIDTHS} (got {in_channels} -> {out_channels})')
        self.deploy, self.in_channels, self.out_channels, self.stride = deploy, in_channels, out_channels, stride
        self.nonlinearity = nn.ReLU()  # (parameter-free; module-tree parity)
        self.se = nn.Identity()
        self.rbr_identity = nn.BatchNorm2d(in_channels) if out_channels == in_channels and stride == 1 else None
        self.rbr_dense = _ConvBn(in_channels, out_channels, 3, stride, 1)
        self.rbr_1x1 = _ConvBn(in_channels, out_channels, 1, stride, 0)

    def _weights(self):
        w1 = self.rbr_1x1.conv.weight
        return self.rbr_dense.conv.weight, (F.pad(w1, (1, 1, 1, 1)) if self.stride == 2 else w1)

    def _block(self, x, w3, w1, stride):
        _require_training(self, 'cvpytorch_b200.yolov6_train.RepVGGBlock is the TRAINING drop-in (batch statistics); use the inference modules for eval()')
        bn3, bn1, bnid = self.rbr_dense.bn, self.rbr_1x1.bn, self.rbr_identity
        groups = {'rbr_dense.bn': _sync_group(bn3), 'rbr_1x1.bn': _sync_group(bn1)}
        if bnid is not None:
            groups['rbr_identity'] = _sync_group(bnid)
        group = groups['rbr_dense.bn']
        if any(g is not group for g in groups.values()):
            raise NotImplementedError(f'H100 training RepVGGBlock({self.in_channels}, {self.out_channels}, stride {self.stride}): its BatchNorms must all '
                                      'be local or all span the same process group (convert_sync_batchnorm converts all three); got ' +
                                      ', '.join(f'{k}: {"local" if g is None else "synced"}' for k, g in groups.items()))
        meta = tuple(_bn_args(bn)[:4] if bn is not None else None for bn in (bn3, bn1, bnid)) + (stride, group)
        return _RepVGG.apply(x, w3, w1, bn3.weight, bn3.bias, bn1.weight, bn1.bias, bnid.weight if bnid is not None else None,
                             bnid.bias if bnid is not None else None, meta)

    def forward(self, x):
        return self._block(x, *self._weights(), self.stride)


class StemRepVGGBlock(RepVGGBlock):
    """The backbone stem RepVGGBlock(3, c, stride 2): both branches as 3x3 / stride-1 convs over train.focus_s2d's 16-channel map, with
    stem_weight_to_s2d's weights.  forward: fp32 NCHW image (no gradient) -> NHWC bf16."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=2, **kw):
        if in_channels != 3 or stride != 2:
            raise NotImplementedError('H100 training YOLOv6 stem: RepVGGBlock(3, c, stride 2)')
        super().__init__(16, out_channels, kernel_size, stride, **kw)
        self.in_channels = in_channels
        self.rbr_dense = _ConvBn(in_channels, out_channels, 3, stride, 1)
        self.rbr_1x1 = _ConvBn(in_channels, out_channels, 1, stride, 0)

    def forward(self, img):
        if img.requires_grad:
            raise NotImplementedError('H100 training YOLOv6 stem computes no gradient for the input image: pass an image without requires_grad')
        w3, w1 = self._weights()
        return self._block(focus_s2d(img), stem_weight_to_s2d(w3), stem_weight_to_s2d(w1), 1)


class RepBlock(nn.Module):
    """yolo_modules.py:453-471 with RepVGG blocks."""

    def __init__(self, in_channels, out_channels, n=1, e=None, block=RepVGGBlock, basic_block=RepVGGBlock):
        super().__init__()
        if block not in (RepVGGBlock,) and getattr(block, '__name__', '') != 'RepVGGBlock':
            raise NotImplementedError('H100 training RepBlock: RepVGG blocks only (no BottleRep)')
        self.conv1 = RepVGGBlock(in_channels, out_channels)
        self.block = nn.Sequential(*(RepVGGBlock(out_channels, out_channels) for _ in range(n - 1))) if n > 1 else None

    def forward(self, x):
        x = self.conv1(x)
        return self.block(x) if self.block is not None else x


class ConvModule(_ConvBnSiLULayer):
    """conv (no bias) -> BatchNorm -> ReLU of the backbone and neck (the act_cfg ReLU ConvModule), training mode: kernel_size 1 or 3, stride 1
    or 2 (3x3), padding kernel_size // 2.  in_pad: zero channels appended to the input (and to the weight's input channels) so that a
    96-channel input runs as 128.  forward: NHWC bf16 in / out (the input already padded)."""
    drop_in = 'ConvModule (ReLU)'
    act = 'relu'

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=None, conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True),
                 act_cfg=dict(type='ReLU'), in_pad=0, **unused):
        padding = kernel_size // 2 if padding is None else padding
        if kernel_size not in (1, 3) or padding != kernel_size // 2 or stride not in (1, 2) or (stride == 2 and kernel_size != 3):
            raise NotImplementedError('H100 training ConvModule (ReLU): kernel_size 1 or 3, padding kernel_size // 2, stride 1 (or 2 with kernel_size 3)')
        if (act_cfg or {}).get('type') != 'ReLU' or (norm_cfg or {}).get('type', 'BN') != 'BN' or conv_cfg is not None:
            raise NotImplementedError('H100 training ConvModule (ReLU): plain Conv2d, BatchNorm and ReLU only')
        _require_widths((in_channels + in_pad, out_channels), lambda bad: f'H100 training ConvModule: {_WIDTHS} (got {in_channels} -> {out_channels})')
        super().__init__(in_channels, out_channels, kernel_size, stride)
        self.in_pad = in_pad

    def forward(self, x):
        w = self.conv.weight
        return self._layer(x, F.pad(w, (0, 0, 0, 0, 0, self.in_pad)) if self.in_pad else w)


class SimCSPSPPF(nn.Module):
    """yolo_modules.py:218-242 (ReLU, chained 5x5 pools: train.sppf_chain writes [x1 | y1 | y2 | m(y2)]).  forward: NHWC bf16."""

    def __init__(self, in_channels, out_channels, kernel_size=5, e=0.5, conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True),
                 act_cfg=dict(type='ReLU'), init_cfg=None):
        super().__init__()
        if kernel_size != 5:
            raise NotImplementedError('H100 training SimCSPSPPF: the chained 5x5 pools only')
        c_ = int(out_channels * e)
        kw = dict(conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg)
        self.cv1 = ConvModule(in_channels, c_, 1, stride=1, **kw)
        self.cv2 = ConvModule(in_channels, c_, 1, stride=1, **kw)
        self.cv3 = ConvModule(c_, c_, 3, stride=1, padding=1, **kw)
        self.cv4 = ConvModule(c_, c_, 1, stride=1, **kw)
        self.m = nn.MaxPool2d(kernel_size=kernel_size, stride=1, padding=kernel_size // 2)  # (parameter-free; module-tree parity)
        self.cv5 = ConvModule(4 * c_, c_, 1, stride=1, **kw)
        self.cv6 = ConvModule(c_, c_, 3, stride=1, padding=1, **kw)
        self.cv7 = ConvModule(2 * c_, out_channels, 1, stride=1, **kw)

    def forward(self, x):
        x1 = self.cv4(self.cv3(self.cv1(x)))
        y0 = self.cv2(x)
        y3 = self.cv6(self.cv5(_SppfChain.apply(x1)))
        return self.cv7(torch.cat((y0, y3), dim=3))


def _convt_weight(weight):
    """nn.ConvTranspose2d weight [cin, cout, 2, 2] -> the 1x1 GEMM weight [4 cout, cin, 1, 1], row (py * 2 + px) * cout + o (as
    yolov6_models.conv_transpose2_weights, in torch so that autograd maps the gradient back)."""
    ci, co = weight.shape[:2]
    return weight.permute(2, 3, 1, 0).reshape(4 * co, ci, 1, 1)


def convt_scatter(u, bias):
    """u NHWC bf16 [B,h,w,4c] (the GEMM output), bias fp32 [c] -> out [B,2h,2w,c]."""
    B, h, w, c4 = u.shape
    out = torch.empty((B, 2 * h, 2 * w, c4 // 4), dtype=torch.bfloat16, device=u.device)
    _lib.check(_lib.lib().cvb_train_convt_scatter(_p(u), B, h, w, c4 // 4, _p(bias), _p(out), _stream()), 'cvb_train_convt_scatter')
    return out


def convt_gather(g):
    """g = d(loss)/d(out) [B,2h,2w,c] -> (du [B,h,w,4c] in the GEMM layout, dbias fp32 [c])."""
    B, H2, W2, c = g.shape
    du = torch.empty((B, H2 // 2, W2 // 2, 4 * c), dtype=torch.bfloat16, device=g.device)
    scratch = torch.empty((256, c), dtype=torch.float32, device=g.device)
    dbias = torch.empty((c,), dtype=torch.float32, device=g.device)
    _lib.check(_lib.lib().cvb_train_convt_gather(_p(g), B, H2 // 2, W2 // 2, c, _p(scratch), _p(du), _p(dbias), _stream()), 'cvb_train_convt_gather')
    return du, dbias


class _ConvT2(torch.autograd.Function):
    """nn.ConvTranspose2d(c, c, 2, stride=2, bias) on NHWC bf16: the 1x1 GEMM (weight _convt_weight(W)) + cvb_train_convt_scatter."""

    @staticmethod
    def forward(ctx, x, wg, bias):
        _check_cuda(x, 'BiFusion (H100 training)')
        x = x.contiguous()
        wf, wb = pack_weights(wg)
        out = convt_scatter(conv(x, wf, wg.shape[0], 1), bias.detach().float().contiguous())
        ctx.save_for_backward(x, wb)
        return out

    @staticmethod
    def backward(ctx, g):
        x, wb = ctx.saved_tensors
        du, dbias = convt_gather(g.contiguous())
        dw = conv_wgrad(x, du, 1)
        dx = conv(du, wb, x.shape[3], 1) if ctx.needs_input_grad[0] else None
        return dx, dw, dbias


class BiFusion(nn.Module):
    """yolo_modules.py:245-265: cv3(cat(upsample(x0), cv1(x1), downsample(cv2(x2)))).  forward([x0, x1, x2] NHWC bf16) -> NHWC bf16.  A
    3c-channel concat that is not a training width (c = 32) is zero-padded to the next one, and so is cv3's weight."""

    def __init__(self, in_channels, out_channels, conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True), act_cfg=dict(type='ReLU'), init_cfg=None):
        super().__init__()
        kw = dict(conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg)
        c3 = out_channels * 3
        self.cv1 = ConvModule(in_channels[0], out_channels, 1, 1, **kw)
        self.cv2 = ConvModule(in_channels[1], out_channels, 1, 1, **kw)
        self.cv3 = ConvModule(c3, out_channels, 1, 1, in_pad=0 if train.channels_ok(c3) else train.pred_cout_pad(c3) - c3, **kw)
        self.upsample = nn.ConvTranspose2d(in_channels=out_channels, out_channels=out_channels, kernel_size=2, stride=2, bias=True)
        self.downsample = ConvModule(out_channels, out_channels, 3, 2, padding=1, **kw)

    def forward(self, x):
        parts = [_ConvT2.apply(x[0], _convt_weight(self.upsample.weight), self.upsample.bias), self.cv1(x[1]), self.downsample(self.cv2(x[2]))]
        if self.cv3.in_pad:
            t = parts[1]
            parts.append(t.new_zeros(t.shape[:3] + (self.cv3.in_pad,)))
        return self.cv3(torch.cat(parts, dim=3))


def _check_v6_subtype(subtype):
    from .yolov6_models import check_subtype
    check_subtype(subtype)


class YOLOv6EfficientRep(nn.Module):
    """yolov6_efficient_rep.py:20-70, training mode, the constructor and state_dict keys of yolov6_models.YOLOv6EfficientRep.
    forward_nhwc(img fp32 NCHW) -> the out_stages outputs, NHWC bf16."""
    cfg = {"n": [0.33, 0.25], "t": [0.33, 0.375], "s": [0.33, 0.5], "m": [0.6, 0.75], "l": [1.0, 1.0], "x": [1.33, 1.25]}

    def __init__(self, subtype='cspdark_s', in_channels=3, out_channels=[64, 128, 256, 512, 1024], num_blocks=[6, 12, 18, 6], depthwise=False,
                 conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True), act_cfg=dict(type='SiLU', inplace=True), out_stages=[2, 3, 4],
                 output_stride=32, backbone_path=None, pretrained=False, frozen_stages=-1, norm_eval=False, **kwargs):
        super().__init__()
        _check_v6_subtype(subtype)
        if depthwise or in_channels != 3:
            raise NotImplementedError('H100 training YOLOv6EfficientRep: 3-channel images, no depthwise convs')
        if norm_eval or frozen_stages >= 0:
            raise NotImplementedError('H100 training YOLOv6EfficientRep: norm_eval and frozen_stages are not on the training path')
        self.subtype, self.in_channels, self.out_stages, self.output_stride = subtype, in_channels, out_stages, output_stride
        depth_mul, width_mul = self.cfg[subtype.split('_')[1]]
        self.out_channels = list(map(lambda x: int(x * width_mul), out_channels))
        self.num_blocks = list(map(lambda x: max(round(x * depth_mul), 1), num_blocks))
        self.stem = StemRepVGGBlock(in_channels, self.out_channels[0], kernel_size=3, stride=2)
        for idx, (cin, cout, n) in enumerate(zip(self.out_channels[:-1], self.out_channels[1:], self.num_blocks)):
            stage = [RepVGGBlock(cin, cout, kernel_size=3, stride=2), RepBlock(cout, cout, n=n, block=RepVGGBlock)]
            if idx == 3:
                stage.append(SimCSPSPPF(cout, cout, act_cfg=dict(type='ReLU')))
            self.add_module(f'stage{idx + 1}', nn.Sequential(*stage))
        _set_bn(self)

    def forward_nhwc(self, x):
        _require_training(self, 'cvpytorch_b200.yolov6_train.YOLOv6EfficientRep is the TRAINING drop-in (batch statistics); load its state_dict '
                                'into cvpytorch_b200.yolov6_models.YOLOv6EfficientRep for eval()')
        _check_cuda(x, 'YOLOv6EfficientRep (H100 training)')
        h = self.stem(x)
        outs = []
        for i in range(1, 5):
            h = getattr(self, f'stage{i}')(h)
            if i in self.out_stages:
                outs.append(h)
        return outs


class YOLOv6RepBiPAN(nn.Module):
    """yolov6_repbipan.py:16-82, training mode, the constructor and state_dict keys of yolov6_models.YOLOv6RepBiPAN.  forward_nhwc([x3, x2, x1,
    x0] NHWC bf16, the backbone's four outputs) -> [pan_out2, pan_out1, pan_out0] NHWC bf16."""
    cfg = {"n": [0.33, 0.25], "t": [0.33, 0.375], "s": [0.33, 0.5], "m": [0.6, 0.75], "l": [1.0, 1.0], "x": [1.33, 1.25]}

    def __init__(self, subtype='yolov6_s', in_channels=[128, 256, 512, 1024], mid_channels=[128, 128, 256], out_channels=[128, 256, 512],
                 num_blocks=[12, 12, 12, 12], depthwise=False, conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True),
                 act_cfg=dict(type='ReLU', inplace=True), **kwargs):
        super().__init__()
        _check_v6_subtype(subtype)
        if depthwise:
            raise NotImplementedError('H100 training YOLOv6RepBiPAN: no depthwise convs')
        self.subtype = subtype
        depth_mul, width_mul = self.cfg[subtype.split('_')[1]]
        w = lambda cs: list(map(lambda x: max(round(x * width_mul), 1), cs))  # noqa: E731
        self.in_channels, self.mid_channels, self.out_channels = w(in_channels), w(mid_channels), w(out_channels)
        self.num_blocks = list(map(lambda x: max(round(x * depth_mul), 1), num_blocks))
        self.num_ins = len(self.in_channels)
        ic, mc, oc, nb = self.in_channels, self.mid_channels, self.out_channels, self.num_blocks
        kw = dict(norm_cfg=norm_cfg, act_cfg=dict(type='ReLU'))
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

    def forward_nhwc(self, x):
        _require_training(self, 'cvpytorch_b200.yolov6_train.YOLOv6RepBiPAN is the TRAINING drop-in (batch statistics); load its state_dict into '
                                'cvpytorch_b200.yolov6_models.YOLOv6RepBiPAN for eval()')
        if len(x) != self.num_ins:
            raise ValueError(f'YOLOv6RepBiPAN: {self.num_ins} feature maps expected, got {len(x)}')
        x3, x2, x1, x0 = x
        fpn_out0 = self.reduce_layer0(x0)
        f_out0 = self.Rep_p4(self.bifusion0([fpn_out0, x1, x2]))
        fpn_out1 = self.reduce_layer1(f_out0)
        pan_out2 = self.Rep_p3(self.bifusion1([fpn_out1, x2, x3]))
        pan_out1 = self.Rep_n3(torch.cat((self.downsample2(pan_out2), fpn_out1), dim=3))
        pan_out0 = self.Rep_n4(torch.cat((self.downsample1(pan_out1), fpn_out0), dim=3))
        return [pan_out2, pan_out1, pan_out0]


class YOLOv6Effidehead(nn.Module):
    """yolov6_effidehead.py:17-148, training mode, the constructor and state_dict keys of yolov6_models.YOLOv6Effidehead (SiLU stems and
    cls / reg convs: train.ConvModule).  forward_nhwc(feats NHWC bf16) -> the reference's training output (stem outputs as NCHW views,
    pred_scores = sigmoid(cls) fp32 [B, A, nc], pred_distri fp32 [B, A, 4]), levels concatenated in order, pixels in y / x order."""
    cfg = {"n": [0.33, 0.25], "t": [0.33, 0.375], "s": [0.33, 0.5], "m": [0.6, 0.75], "l": [1.0, 1.0], "x": [1.33, 1.25]}

    def __init__(self, subtype='yolov6_s', num_classes=80, in_channels=[128, 256, 512], num_anchors=1, reg_max=16, num_layers=3, stacked_convs=2,
                 depthwise=False, use_dfl=False, fuse_ab=False, conv_cfg=None, norm_cfg=dict(type='BN'), act_cfg=dict(type='SiLU'), **kwargs):
        super().__init__()
        _check_v6_subtype(subtype)
        if use_dfl or fuse_ab or depthwise or num_layers != 3:
            raise NotImplementedError('H100 training YOLOv6Effidehead: the 3-level, non-depthwise head without use_dfl / fuse_ab')
        if (act_cfg or {}).get('type') not in ('SiLU', 'Swish'):
            raise NotImplementedError('H100 training YOLOv6Effidehead: SiLU head convs only')
        self.subtype, self.fuse_ab, self.use_dfl = subtype, fuse_ab, use_dfl
        width_mul = self.cfg[subtype.split('_')[1]][1]
        self.in_channels = list(map(lambda x: max(round(x * width_mul), 1), in_channels))
        self.num_anchors, self.reg_max, self.stacked_convs = 1, 0, stacked_convs
        self.num_classes, self.num_outputs, self.num_layers = num_classes, num_classes + 5, num_layers
        self.stems, self.cls_convs, self.reg_convs = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        self.cls_preds, self.reg_preds = nn.ModuleList(), nn.ModuleList()
        self.proj_conv = nn.Conv2d(self.reg_max + 1, 1, 1, bias=False)
        for c in self.in_channels:
            self.stems.append(train.ConvModule(c, c, 1, 1, 0))
            self.cls_convs.append(train.ConvModule(c, c, 3, 1, 1))
            self.reg_convs.append(train.ConvModule(c, c, 3, 1, 1))
            self.cls_preds.append(nn.Conv2d(c, num_classes * self.num_anchors, 1))
            self.reg_preds.append(nn.Conv2d(c, 4 * (self.num_anchors + self.reg_max), 1))
        self.proj = nn.Parameter(torch.linspace(0, self.reg_max, self.reg_max + 1), requires_grad=False)
        self.proj_conv.weight = nn.Parameter(self.proj.view([1, self.reg_max + 1, 1, 1]).clone().detach(), requires_grad=False)
        _set_bn(self)

    def forward_nhwc(self, x):
        _require_training(self, 'cvpytorch_b200.yolov6_train.YOLOv6Effidehead is the TRAINING drop-in (batch statistics); load its state_dict '
                                'into cvpytorch_b200.yolov6_models.YOLOv6Effidehead for eval()')
        feats, scores, distri = [], [], []
        for i, f in enumerate(x):
            t = self.stems[i](f)  # (fans out to both branches: autograd adds the gradients that reach it)
            feats.append(t.permute(0, 3, 1, 2))
            cls = _PredConv.apply(self.cls_convs[i](t), self.cls_preds[i].weight, self.cls_preds[i].bias)
            reg = _PredConv.apply(self.reg_convs[i](t), self.reg_preds[i].weight, self.reg_preds[i].bias)
            scores.append(torch.sigmoid(cls).flatten(2).permute(0, 2, 1))
            distri.append(reg.flatten(2).permute(0, 2, 1))
        return feats, torch.cat(scores, 1), torch.cat(distri, 1)
