"""The YOLOv6 training loss on the H100 kernels (csrc/yolov6_loss.cu): a drop-in for src/losses/det/yolov6_loss.py YOLOv6Loss.

  YOLOv6Loss   target packing, the ATSS (warm-up) or task-aligned assignment and the GIoU / SIoU box loss with its gradient with respect
               to pred_distri, with no host sync (forward and backward can be captured in a CUDA graph)

The network stays in torch.  Head outputs are cast with .float().contiguous(), so fp16 / bf16 outputs under autocast work and their
gradients flow back through the cast.  The reference returns {'iou': 2.5 L, 'dfl': 0.5 L, 'class': 1.0 L} of its box loss L (its class
loss is computed and discarded), so pred_scores gets no gradient.  No CPU fallback: CPU tensors raise CvbError.  Divergences, each
documented in include/cvb200.h: the dict entries are fp64 also without positives (the reference returns fp32 there); rows whose image
index truncates outside [0, B) are dropped (the reference wraps -1); labels outside [0, nc) give a zero class score (the reference
raises); a level with fewer than 9 anchors takes all of them as ATSS candidates (the reference raises); on equal values at the top-k
boundary the lowest anchor index wins (torch.topk's order is undefined).
"""
import torch
import torch.nn as nn

from . import _lib
from .train import _check_cuda, _p, _stream, _workspace

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
