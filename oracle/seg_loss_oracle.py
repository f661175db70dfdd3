"""fp64 torch restatement of the segmentation training loss: EncoderDecoder.loss_forward's
F.interpolate(preds, size=targets.shape[-2:], mode='bilinear', align_corners=False) followed by CrossEntropyLoss2d
(src/losses/seg/cross_entropy_loss.py: loss_weight * nn.CrossEntropyLoss(ignore_index=..., reduction='mean')).

The upsample is written as two explicit matrices, Rh [H x h] and Rw [W x w], built from torch's index formula (scale = (float)in / out,
src = max((dst + 0.5) * scale - 0.5, 0), i0 = (int)src, i1 = i0 + (i0 < in - 1), weights 1 - l and l with l = src - i0, all in fp32 as
torch computes them for fp32 inputs), so that z = Rh x Rw^T for each plane.  Equal sizes give the identity.  The cross-entropy uses
logsumexp and the gradient comes from fp64 autograd; the matrix form states the backward gather directly: d x = Rh^T (d z) Rw.

fixture_case(name) builds the seeded inputs of tests/golden/seg_loss.npz (logits in multiples of 1/8, so the fixture compresses).
"""
import numpy as np
import torch


def interp_matrix(out_size, in_size):
    """[out_size, in_size] fp64: row o holds the two bilinear weights of output index o."""
    if out_size == in_size:
        return torch.eye(out_size, dtype=torch.float64)
    scale = np.float32(in_size) / np.float32(out_size)
    dst = np.arange(out_size, dtype=np.float32)
    src = np.maximum((dst + np.float32(0.5)) * scale - np.float32(0.5), np.float32(0.0)).astype(np.float32)
    i0 = np.minimum(src.astype(np.int64), in_size - 1)
    i1 = i0 + (i0 < in_size - 1)
    l1 = (src - i0.astype(np.float32)).astype(np.float32)
    l0 = (np.float32(1.0) - l1).astype(np.float32)
    R = np.zeros((out_size, in_size), dtype=np.float64)
    np.add.at(R, (np.arange(out_size), i0), l0.astype(np.float64))
    np.add.at(R, (np.arange(out_size), i1), l1.astype(np.float64))
    return torch.from_numpy(R)


def upsample(x, H, W):
    """x [B, C, h, w] -> [B, C, H, W] in fp64 through the two matrices."""
    Rh = interp_matrix(H, x.shape[2]).to(x.device)
    Rw = interp_matrix(W, x.shape[3]).to(x.device)
    return torch.einsum('Yi,bcij,Xj->bcYX', Rh, x.double(), Rw)


def loss(pred, target, ignore_index=255, loss_weight=1.0):
    """loss_weight * mean over the pixels whose label is not ignore_index of lse(z) - z_label, z = upsample(pred) in fp64 (NaN when every
    pixel is ignored, as torch's 'mean').  A label outside [0, C) that is not ignore_index raises IndexError, as torch does on the CPU.
    Differentiable with respect to pred."""
    B, C = pred.shape[:2]
    H, W = target.shape[-2:]
    z = upsample(pred, H, W)
    t = target.long()
    valid = t != ignore_index
    bad = valid & ((t < 0) | (t >= C))
    if bool(bad.any()):
        raise IndexError(f'seg_loss_oracle: {int(bad.sum())} labels outside [0, {C}) that are not ignore_index {ignore_index}')
    zf = z.permute(0, 2, 3, 1)[valid]                      # [n_valid, C]
    terms = torch.logsumexp(zf, dim=1) - zf.gather(1, t[valid][:, None])[:, 0]
    return loss_weight * (terms.sum() / valid.sum())


CASES = {
    # name: (B, C, h, w, H, W, label dtype, loss_weight)
    'x4': (3, 19, 16, 24, 64, 96, torch.uint8, 1.0),       # DeepLabv3+: a 255 border, image 1 wholly ignored
    'x8': (2, 5, 8, 12, 64, 96, torch.int64, 0.4),         # PSPNet's auxiliary FCN head
    'frac': (2, 7, 13, 29, 96, 192, torch.int32, 1.0),     # a non-integer ratio
    'ident': (2, 3, 24, 40, 24, 40, torch.int64, 1.0),     # already at label size
    'down': (2, 4, 40, 56, 17, 23, torch.uint8, 1.0),      # downsampling
    'ignored': (2, 3, 8, 8, 32, 32, torch.uint8, 1.0),     # every pixel ignored: NaN loss, zero gradient
}


def fixture_case(name, seed=0):
    """-> (pred fp32 [B, C, h, w], target [B, H, W], ignore_index, loss_weight) of one fixture case."""
    B, C, h, w, H, W, dtype, lw = CASES[name]
    g = torch.Generator().manual_seed(seed * 1000 + sorted(CASES).index(name))
    pred = torch.randint(-40, 41, (B, C, h, w), generator=g).float() / 8
    target = torch.randint(0, C, (B, H, W), generator=g)
    target[torch.rand(B, H, W, generator=g) < 0.1] = 255
    if name == 'x4':
        target[:, :3], target[:, :, -5:] = 255, 255
        target[1] = 255
    if name == 'ignored':
        target[:] = 255
    return pred, target.to(dtype), 255, lw
