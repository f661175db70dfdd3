"""The FCOS training loss on the H100 kernels (csrc/fcos_loss.cu): a drop-in for src/losses/fcos_loss.py FCOSLoss.

  FCOSLoss   GenTargets' point assignment, the sigmoid focal, centerness BCE and GIoU losses and their gradient with respect to the head
             outputs, with no host sync (the loss forward and backward can be captured in a CUDA graph)

The network (ResNet-50, FPN, the GN heads, ScaleExp) stays in torch.  The head outputs are cast with .float().contiguous(), so fp16 / bf16
outputs under autocast work and their gradients flow back through the cast; the fp32 computation is the contract.  No CPU fallback: CPU
tensors raise CvbError.  Divergence: an empty GT list (m = 0) is an all-background batch here; the reference raises in torch.min.
"""
import torch
import torch.nn as nn

from . import _lib
from .train import _check_cuda, _floats, _p, _ptrs, _shapes4, _stream, _workspace

MAX_GT = 1024


def _levels(preds, strides, limit_range):
    """-> ctypes (cls, cnt, reg pointer arrays, shapes of each level's cls, cnt, reg, strides, limit ranges), validated by the C entry points."""
    cls, cnt, reg = preds
    return _ptrs(cls), _ptrs(cnt), _ptrs(reg), _shapes4([t for lv in zip(cls, cnt, reg) for t in lv]), _floats(strides), _floats(v for r in limit_range for v in r)


def fcos_loss_forward(preds, boxes, labels, strides, limit_range, return_targets=False):
    """preds = [cls_logits, cnt_logits, reg_preds]: per level fp32 NCHW [B, nc, h, w], [B, 1, h, w], [B, 4, h, w] (CUDA, contiguous);
    boxes fp32 [B, m, 4], labels int32 [B, m] (CUDA, contiguous, -1 rows pad).
    -> (out fp32 [4] = cls_loss, cnt_loss, reg_loss, total; matched_gt int32 [B, A], -1 = background; num_pos int32 [B]), and with
    return_targets the kernel's per-point targets fp32 [B, A, 5] = (centerness, l, t, r, b), -1 for background."""
    cls = preds[0]
    if not len(preds[0]) == len(preds[1]) == len(preds[2]) == len(strides) == len(limit_range):
        raise ValueError(f'FCOSLoss: {len(strides)} strides and {len(limit_range)} limit ranges for {[len(p) for p in preds]} outputs per kind')
    B, nc = cls[0].shape[0], cls[0].shape[1]
    A = sum(c.shape[2] * c.shape[3] for c in cls)
    dev = cls[0].device
    ws = _workspace(_lib.lib().cvb_train_fcos_loss_workspace_bytes(B, A, nc), dev)
    out = torch.empty((4,), dtype=torch.float32, device=dev)
    matched_gt = torch.empty((B, A), dtype=torch.int32, device=dev)
    num_pos = torch.empty((B,), dtype=torch.int32, device=dev)
    tgt = torch.empty((B, A, 5), dtype=torch.float32, device=dev) if return_targets else None
    pc, pn, pr, shapes, strd, lim = _levels(preds, strides, limit_range)
    _lib.check(_lib.lib().cvb_train_fcos_loss_fwd(pc, pn, pr, shapes, strd, lim, len(cls), _p(boxes), _p(labels), B, boxes.shape[1],
                                                  _p(matched_gt), _p(num_pos), _p(tgt), _p(out), _p(ws), ws.numel(), _stream()), 'cvb_train_fcos_loss_fwd')
    return (out, matched_gt, num_pos, tgt) if return_targets else (out, matched_gt, num_pos)


def fcos_loss_backward(preds, boxes, labels, strides, limit_range, matched_gt, num_pos, grad_out):
    """d(sum_i grad_out[i] * out[i]) / d(preds) under the forward's matched_gt and num_pos -> ([cls], [cnt], [reg]) fp32 NCHW gradients
    shaped like preds."""
    grads = [[torch.empty_like(t) for t in ts] for ts in preds]
    pc, pn, pr, shapes, strd, lim = _levels(preds, strides, limit_range)
    n = len(preds[0])
    gc, gn, gr = (_ptrs(ts) for ts in grads)
    _lib.check(_lib.lib().cvb_train_fcos_loss_bwd(pc, pn, pr, shapes, strd, lim, n, _p(boxes), _p(labels), preds[0][0].shape[0], boxes.shape[1],
                                                  _p(matched_gt), _p(num_pos), _p(grad_out), gc, gn, gr, _stream()), 'cvb_train_fcos_loss_bwd')
    return grads


class _FCOSLossFn(torch.autograd.Function):
    """out [4] = (cls_loss, cnt_loss, reg_loss, total) of the head outputs; the assignment (matched_gt [B, A], num_pos [B]) is kept for the
    backward, which recomputes the gradient from it scaled by the four incoming gradients."""

    @staticmethod
    def forward(ctx, boxes, labels, strides, limit_range, nlev, *tensors):
        preds = [list(tensors[k * nlev:(k + 1) * nlev]) for k in range(3)]
        out, matched_gt, num_pos = fcos_loss_forward(preds, boxes, labels, strides, limit_range)
        ctx.save_for_backward(boxes, labels, matched_gt, num_pos, *tensors)
        ctx.strides, ctx.limit_range, ctx.nlev = strides, limit_range, nlev
        return out

    @staticmethod
    def backward(ctx, g):
        boxes, labels, matched_gt, num_pos, *tensors = ctx.saved_tensors
        n = ctx.nlev
        preds = [list(tensors[k * n:(k + 1) * n]) for k in range(3)]
        grads = fcos_loss_backward(preds, boxes, labels, ctx.strides, ctx.limit_range, matched_gt, num_pos, g.float().contiguous())
        return (None, None, None, None, None, *grads[0], *grads[1], *grads[2])


def _loss_targets(boxes, labels, B, nc, device):
    """The reference's padded boxes [B, m, 4] and labels [B, m] as the contiguous fp32 / int32 CUDA tensors of the kernels."""
    if not isinstance(boxes, torch.Tensor) or boxes.dim() != 3 or boxes.shape[0] != B or boxes.shape[2] != 4:
        raise ValueError(f'FCOSLoss: target_boxes must be a [B={B}, m, 4] tensor of (x1, y1, x2, y2) rows')
    if not isinstance(labels, torch.Tensor) or labels.dim() != 2 or tuple(labels.shape) != tuple(boxes.shape[:2]):
        raise ValueError(f'FCOSLoss: target_labels must be a [B={B}, m={boxes.shape[1]}] tensor')
    if boxes.shape[1] > MAX_GT:
        raise ValueError(f'FCOSLoss: at most {MAX_GT} GT rows per image (got {boxes.shape[1]})')
    _check_cuda(boxes, 'FCOSLoss target_boxes')
    _check_cuda(labels, 'FCOSLoss target_labels')
    b = boxes.detach().to(device=device, dtype=torch.float32).contiguous()
    # labels outside 1..nc have no one-hot entry: clamping to [-1, nc + 1] keeps them outside while fitting int32
    lab = labels.detach().to(device=device).clamp(-1, nc + 1).to(torch.int32).contiguous()
    return b, lab


class FCOSLoss(nn.Module):
    """src/losses/fcos_loss.py FCOSLoss on the H100 kernels (csrc/fcos_loss.cu): same constructor, no parameters or buffers.
    forward(preds, target_boxes, target_labels) takes the head's [cls_logits, cnt_logits, reg_preds] lists of NCHW outputs (CUDA) and the
    padded targets of FCOS.trans_specific_format (boxes [B, m, 4] x1 y1 x2 y2 in pixels, labels [B, m], -1 rows pad, m <= 1024) and returns
    the reference's tuple (cls_loss, cnt_loss, reg_loss, total_loss) of 0-dim device tensors, with no host sync."""

    def __init__(self, strides=[8, 16, 32, 64, 128], limit_range=[[-1, 64], [64, 128], [128, 256], [256, 512], [512, 999999]]):
        super().__init__()
        if len(strides) != len(limit_range):
            raise ValueError(f'FCOSLoss: {len(strides)} strides for {len(limit_range)} limit ranges')
        self.strides = strides
        self.limit_range = limit_range

    def forward(self, preds, target_boxes, target_labels):
        cls, cnt, reg = preds
        if not len(cls) == len(cnt) == len(reg) == len(self.strides):
            raise ValueError(f'FCOSLoss: {len(self.strides)} strides for {len(cls)} / {len(cnt)} / {len(reg)} outputs')
        for t in (*cls, *cnt, *reg):
            _check_cuda(t, 'FCOSLoss')
        tensors = [t.float().contiguous() for t in (*cls, *cnt, *reg)]
        boxes, labels = _loss_targets(target_boxes, target_labels, cls[0].shape[0], cls[0].shape[1], cls[0].device)
        out = _FCOSLossFn.apply(boxes, labels, tuple(self.strides), tuple(tuple(r) for r in self.limit_range), len(cls), *tensors)
        return out[0], out[1], out[2], out[3]
