"""The segmentation cross-entropy loss on the H100 kernels (csrc/seg_loss.cu): a drop-in for src/losses/seg/cross_entropy_loss.py
CrossEntropyLoss2d that takes the head output at its own resolution and fuses EncoderDecoder.loss_forward's bilinear upsample to the
label size into the loss and its gradient.

  CrossEntropyLoss2d  loss_weight * CE(bilinear(pred -> H x W), target), mean over the pixels whose label is not ignore_index; the
                      upsampled [B, C, H, W] logits never exist, no host sync (forward and backward can be captured in a CUDA graph)
  loss_forward        EncoderDecoder.loss_forward that hands the low-resolution preds to the drop-in losses and the interpolated preds,
                      computed once, to any other loss in the list

The network stays in torch.  pred is cast with .float().contiguous(), so fp16 / bf16 heads under autocast work and their gradient flows
back through the cast; the fp32 computation is the contract.  Labels (uint8, int32 or int64, any strides) are read as they are.  No CPU
fallback: CPU tensors raise CvbError.  Divergence: a label outside [0, C) that is not ignore_index makes torch raise (CPU) or assert
(CUDA); here the loss and every gradient element are NaN, so GradScaler skips the step.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch import Tensor

from . import _lib
from .ops import SEG_DTYPES
from .train import _check_cuda, _p, _stream, _workspace


def nc_max():
    """The largest class count the loss kernels accept."""
    return int(_lib.lib().cvb_train_seg_ce_nc_max())


def _args(pred, target, ignore_index, loss_weight):
    B, C, h, w = pred.shape
    H, W = target.shape[-2:]
    return (_p(pred), B, C, h, w, _p(target), SEG_DTYPES[target.dtype], H, W, *target.stride(), int(ignore_index), float(loss_weight))


def seg_ce_forward(pred, target, ignore_index=255, loss_weight=1.0):
    """pred fp32 [B, C, h, w] contiguous CUDA, target [B, H, W] uint8 / int32 / int64 CUDA (any strides) -> (loss fp32 0-dim, lse fp32
    [B, H, W], record int64 [2] = (n_valid, n_bad)); lse and record are what the backward needs."""
    B, H, W = target.shape
    dev = pred.device
    ws = _workspace(_lib.lib().cvb_train_seg_ce_workspace_bytes(B, H, W), dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    lse = torch.empty((B, H, W), dtype=torch.float32, device=dev)
    record = torch.empty((2,), dtype=torch.int64, device=dev)
    _lib.check(_lib.lib().cvb_train_seg_ce_fwd(*_args(pred, target, ignore_index, loss_weight), _p(lse), _p(record), _p(loss), _p(ws), ws.numel(),
                                               _stream()), 'cvb_train_seg_ce_fwd')
    return loss, lse, record


def seg_ce_backward(pred, target, ignore_index, loss_weight, lse, record, grad_out):
    """grad_out fp32 [1] CUDA -> d(grad_out * loss) / d(pred), fp32 shaped like pred."""
    grad = torch.empty_like(pred)
    _lib.check(_lib.lib().cvb_train_seg_ce_bwd(*_args(pred, target, ignore_index, loss_weight), _p(lse), _p(record), _p(grad_out), _p(grad),
                                               _stream()), 'cvb_train_seg_ce_bwd')
    return grad


class _SegCEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target, ignore_index, loss_weight):
        loss, lse, record = seg_ce_forward(pred, target, ignore_index, loss_weight)
        ctx.save_for_backward(pred, target, lse, record)
        ctx.ignore_index, ctx.loss_weight = ignore_index, loss_weight
        return loss

    @staticmethod
    def backward(ctx, g):
        pred, target, lse, record = ctx.saved_tensors
        grad = seg_ce_backward(pred, target, ctx.ignore_index, ctx.loss_weight, lse, record, g.float().reshape(1).contiguous())
        return grad, None, None, None


class CrossEntropyLoss2d(nn.Module):
    """src/losses/seg/cross_entropy_loss.py CrossEntropyLoss2d on the H100 kernels: same constructor and loss_name, no parameters or buffers.
    forward(pred [B, C, h, w], target [B, H, W]) -> loss_weight * the mean cross-entropy of pred bilinearly upsampled to H x W
    (align_corners=False) over the pixels whose label is not ignore_index, a 0-dim fp32 device tensor.  With (h, w) == (H, W) that is the
    reference's result for an already upsampled pred.  Class weights, label smoothing and reductions other than 'mean' are not supported."""

    def __init__(self, weight=None, ignore_index=255, reduction='mean', label_smoothing=0.0, loss_weight=1.0, loss_name='ce_loss'):
        super().__init__()
        if weight is not None:
            raise NotImplementedError('CrossEntropyLoss2d (H100): class weights are not supported')
        if label_smoothing != 0.0:
            raise NotImplementedError('CrossEntropyLoss2d (H100): label_smoothing must be 0')
        if reduction != 'mean':
            raise NotImplementedError(f"CrossEntropyLoss2d (H100): only reduction='mean' is supported (got {reduction!r})")
        self.ignore_index = int(ignore_index)
        self.loss_weight = float(loss_weight)
        self._loss_name = loss_name

    @property
    def loss_name(self):
        return self._loss_name

    def forward(self, pred, target):
        if not isinstance(pred, Tensor) or pred.dim() != 4:
            raise ValueError('CrossEntropyLoss2d: pred must be a [B, C, h, w] tensor')
        if not isinstance(target, Tensor) or target.dim() != 3 or target.shape[0] != pred.shape[0]:
            raise ValueError(f'CrossEntropyLoss2d: target must be a [B={pred.shape[0]}, H, W] tensor')
        _check_cuda(pred, 'CrossEntropyLoss2d pred')
        _check_cuda(target, 'CrossEntropyLoss2d target')
        if target.device != pred.device:
            raise _lib.CvbError(f'CrossEntropyLoss2d: pred on {pred.device}, target on {target.device}')
        if target.dtype not in SEG_DTYPES:
            raise TypeError(f'CrossEntropyLoss2d: target is {target.dtype}; label maps must be uint8, int32 or int64')
        if not 1 <= pred.shape[1] <= nc_max():
            raise ValueError(f'CrossEntropyLoss2d: {pred.shape[1]} classes; 1 to {nc_max()} are supported')
        return _SegCEFn.apply(pred.float().contiguous(), target.detach(), self.ignore_index, self.loss_weight)


def loss_forward(self, preds, targets, loss):
    """src/models/segmentors/encoder_decoder.py EncoderDecoder.loss_forward with the upsample moved into the drop-in loss: each
    CrossEntropyLoss2d of this module gets the low-resolution preds; any other loss gets F.interpolate(preds, size=targets.shape[-2:],
    mode='bilinear', align_corners=False), computed once, as in the reference.  Losses sharing a loss_name are summed.
    Set EncoderDecoder.loss_forward = loss_forward to install it (self is not used)."""
    assert isinstance(preds, Tensor) and preds.ndim == 4, \
        f'preds must be Tensor type, and ndim == 4, but got {type(preds)} and {preds.ndim}'
    assert isinstance(targets, Tensor) and targets.ndim == 3, \
        f'targets must be Tensor type, and ndim == 3, but got {type(targets)} and {targets.ndim}'
    losses = dict()
    if not isinstance(loss, (list, nn.ModuleList)):
        loss = [loss]
    upsampled = None
    for l in loss:
        if isinstance(l, CrossEntropyLoss2d):
            v = l(preds, targets)
        else:
            if upsampled is None:
                upsampled = F.interpolate(preds, size=targets.shape[-2:], mode='bilinear', align_corners=False)
            v = l(upsampled, targets)
        if l.loss_name not in losses:
            losses[l.loss_name] = v
        else:
            losses[l.loss_name] += v
    return losses

