"""Every training-kernel launch of the two real training steps, at its real shape: one YOLOv5-s step at 64 x 3 x 640² (the batch of
coco_yolov5_s.yml, tools/bench_yolov5_train.py) and one YOLOX-s step at 16 x 3 x 640² (tools/bench_yolox_train.py), both with 80 classes
and 2 to 20 targets per image.

LAUNCHES is the set of distinct signatures of the cvb_train_* calls of those two steps: the entry point, its integer and float arguments
(level shapes, strides, anchors and hyper-parameters of the losses included) and which pointer arguments are NULL ('*' = a tensor, None =
NULL; y_prev / stat_prev select the SiLU' epilogue).  test_launch_table_matches_the_steps records both steps through a proxy of
_lib.lib() and requires the recorded set to equal LAUNCHES, so a model change that adds a launch fails until its shape is listed here,
and so checked.  Each entry is then run stand-alone through the C ABI, outputs pre-filled with NaN (backward-weight accumulates into the
zeroed dw its contract asks for), in two ways:

(a) exact, integer operands.  bf16 operands in {-1, 0, 1} (integer biases and gradients) make every partial sum a kernel forms an integer
    below 2^24, so fp32 accumulation is exact in any order -- the tensor core's chained MMAs and the backward-weight's split atomics
    included -- and the kernel must equal float64: bf16 outputs bitwise equal to bf16_rn(float64), fp32 outputs equal.  The backward-weight
    sums one product per output pixel: at most 64 x 320² = 6.55 M < 2^24.  Unlike a bound of gamma * absref, which grows with the pixel
    count (about 7000 for the 6.55 M-pixel stem backward-weight with Gaussian operands), this sees one lost or doubled 128-pixel tile, a
    lost split or a parity class written to the wrong place (test_exact_check_sees_a_lost_tile_and_swapped_parity_classes).
      SiLU' epilogue     the accumulator is exact; the bound is the epilogue's own error (fp64ref.silu_grad_err) and the bf16 store.
      BatchNorm          y = per-channel pivot + {-1, 0, 1}: the pivoted sums (and sum dz for g = dz) are exact, so the bounds of the
                         statistics lose their summation term and keep a few fp32 roundings (EXACT_GS: the double finalisation).
                         sum dz * xhat (xhat is not an integer) keeps the summation bound.
      pooling, upsample-concat, Focus, weight packing   bitwise (integer gradient sums are exact, then one bf16 rounding).
(b) rounding, Gaussian operands: the element-wise float64 bounds of tests/test_train_gpu.py's docstring (fp64ref) at the same shape, for
    the convolutions, the prediction conv / bias gradient and BatchNorm: the accumulation precision that (a) cannot see.
The losses run their oracle checks (test_yolov5_train_gpu._check, test_yolox_loss_gpu._check) at the recorded level shapes and target
counts; each loss signature pair (forward, backward) shares one check.

The float64 references run on the GPU, so every signature runs at its full batch: on one H100 80GB HBM3 (SXM, 700 W power limit) the
whole file took 45 s (pytest's count; peak device memory under 20 GB)."""
import ctypes
import os
import sys
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fp64ref as R  # noqa: E402

pytestmark = pytest.mark.gpu
NC = 80
V5_B, X_B, SIZE = 64, 16, 640
EXACT_GS = 8 * 2.0 ** -53  # the double roundings of bn_finalize_kernel on exact sums
NAN = float('nan')

# (entry point, arguments without the stream): recorded from the two steps (test_launch_table_matches_the_steps prints the table)
LAUNCHES = [
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 102400, 128, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 102400, 256, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 102400, 64, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 107584, 128, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 1638400, 32, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 1638400, 64, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 25600, 128, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 25600, 256, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 25600, 512, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 28224, 128, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 409600, 128, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 409600, 32, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 409600, 64, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 6400, 256, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 6400, 512, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 6553600, 32, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 7744, 128, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 1, '*', 102400, 128, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 1, '*', 102400, 64, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 1, '*', 1638400, 32, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 1, '*', 25600, 128, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 1, '*', 25600, 256, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 1, '*', 409600, 32, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 1, '*', 409600, 64, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 1, '*', 6400, 256, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 102400, 128, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 102400, 256, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 102400, 64, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 107584, 128, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 1638400, 32, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 1638400, 64, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 25600, 128, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 25600, 256, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 25600, 512, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 28224, 128, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 409600, 128, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 409600, 32, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 409600, 64, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 6400, 256, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 6400, 512, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 6553600, 32, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 7744, 128, '*', '*')),
    ('cvb_train_bn_stats', ('*', 102400, 128, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 102400, 256, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 102400, 64, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 107584, 128, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 1638400, 32, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 1638400, 64, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 25600, 128, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 25600, 256, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 25600, 512, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 28224, 128, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 409600, 128, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 409600, 32, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 409600, 64, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 6400, 256, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 6400, 512, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 6553600, 32, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 7744, 128, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_conv', ('*', 16, 160, 160, 32, '*', 32, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 160, 160, 32, '*', 32, 3, 1, '*', '*', '*')),
    ('cvb_train_conv', ('*', 16, 160, 160, 32, '*', 32, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 160, 160, 32, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 160, 160, 64, '*', 128, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 160, 160, 64, '*', 32, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 160, 160, 64, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 1024, '*', 512, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 256, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 256, '*', 256, 3, 1, '*', '*', '*')),
    ('cvb_train_conv', ('*', 16, 20, 20, 256, '*', 256, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 256, '*', 512, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 512, '*', 1024, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 512, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 512, '*', 512, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 22, 22, 128, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 22, 22, 16, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 320, 320, 16, '*', 32, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 320, 320, 32, '*', 64, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 128, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 128, '*', 128, 3, 1, '*', '*', '*')),
    ('cvb_train_conv', ('*', 16, 40, 40, 128, '*', 128, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 128, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 128, '*', 512, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 256, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 256, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 256, '*', 256, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 256, '*', 512, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 512, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 42, 42, 128, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 42, 42, 16, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 128, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 128, '*', 128, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 128, '*', 256, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 128, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 256, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 64, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 64, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 64, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 64, '*', 64, 3, 1, '*', '*', '*')),
    ('cvb_train_conv', ('*', 16, 80, 80, 64, '*', 64, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 82, 82, 128, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 82, 82, 16, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 160, 160, 32, '*', 32, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 160, 160, 32, '*', 32, 3, 1, '*', '*', '*')),
    ('cvb_train_conv', ('*', 64, 160, 160, 32, '*', 32, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 160, 160, 32, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 160, 160, 64, '*', 128, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 160, 160, 64, '*', 32, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 160, 160, 64, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 1024, '*', 512, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 256, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 256, '*', 256, 3, 1, '*', '*', '*')),
    ('cvb_train_conv', ('*', 64, 20, 20, 256, '*', 256, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 256, '*', 512, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 512, '*', 1024, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 512, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 512, '*', 512, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 320, 320, 16, '*', 32, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 320, 320, 32, '*', 64, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 128, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 128, '*', 128, 3, 1, '*', '*', '*')),
    ('cvb_train_conv', ('*', 64, 40, 40, 128, '*', 128, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 128, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 128, '*', 512, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 256, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 256, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 256, '*', 256, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 256, '*', 512, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 512, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 128, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 128, '*', 128, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 128, '*', 256, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 128, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 256, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 256, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 64, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 64, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 64, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 64, '*', 64, 3, 1, '*', '*', '*')),
    ('cvb_train_conv', ('*', 64, 80, 80, 64, '*', 64, 3, 1, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 16, 160, 160, 64, '*', 32, 320, 320, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 16, 20, 20, 256, '*', 256, 40, 40, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 16, 20, 20, 512, '*', 256, 40, 40, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 16, 40, 40, 128, '*', 128, 80, 80, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 16, 40, 40, 256, '*', 128, 80, 80, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 16, 80, 80, 128, '*', 64, 160, 160, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 64, 160, 160, 64, '*', 32, 320, 320, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 64, 20, 20, 256, '*', 256, 40, 40, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 64, 20, 20, 512, '*', 256, 40, 40, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 64, 40, 40, 128, '*', 128, 80, 80, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 64, 40, 40, 256, '*', 128, 80, 80, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 64, 80, 80, 128, '*', 64, 160, 160, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 20, 20, 512, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 22, 22, 128, '*', 128, 3, 1, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 22, 22, 128, '*', 512, 1, -1, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 40, 40, 256, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 42, 42, 128, '*', 128, 3, 1, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 42, 42, 128, '*', 256, 1, -1, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 80, 80, 128, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 82, 82, 128, '*', 128, 1, -1, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 82, 82, 128, '*', 128, 3, 1, '*', None, None)),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 160, 160, 32, 32, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 160, 160, 32, 32, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 160, 160, 64, 128, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 160, 160, 64, 32, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 160, 160, 64, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 20, 20, 1024, 512, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 20, 20, 256, 256, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 20, 20, 256, 256, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 20, 20, 512, 256, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 20, 20, 512, 512, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 22, 22, 128, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 22, 22, 128, 16, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 320, 320, 16, 32, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 320, 320, 32, 64, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 128, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 128, 128, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 256, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 256, 256, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 256, 256, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 256, 512, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 512, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 42, 42, 128, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 42, 42, 128, 16, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 128, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 128, 128, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 128, 256, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 128, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 256, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 64, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 64, 64, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 82, 82, 128, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 82, 82, 128, 16, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 160, 160, 32, 32, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 160, 160, 32, 32, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 160, 160, 64, 128, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 160, 160, 64, 32, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 160, 160, 64, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 20, 20, 1024, 512, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 20, 20, 256, 256, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 20, 20, 256, 256, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 20, 20, 512, 256, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 20, 20, 512, 512, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 320, 320, 16, 32, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 320, 320, 32, 64, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 128, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 128, 128, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 256, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 256, 256, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 256, 256, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 256, 512, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 512, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 128, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 128, 128, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 128, 256, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 128, 256, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 128, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 256, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 64, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 64, 64, 3, 1, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 16, 20, 20, 512, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 16, 22, 22, 128, 128, 3, 1, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 16, 40, 40, 256, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 16, 42, 42, 128, 128, 3, 1, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 16, 80, 80, 128, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 16, 82, 82, 128, 128, 3, 1, '*')),
    ('cvb_train_focus_s2d', ('*', 16, 640, 640, '*')),
    ('cvb_train_focus_s2d', ('*', 64, 640, 640, '*')),
    ('cvb_train_pack_weights', ('*', 128, 128, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 128, 128, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 128, 256, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 128, 512, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 128, 64, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 16, 128, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 256, 128, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 256, 128, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 256, 256, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 256, 256, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 256, 512, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 32, 16, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 32, 32, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 32, 32, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 32, 64, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 512, 1024, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 512, 256, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 512, 512, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 64, 128, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 64, 256, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 64, 32, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 64, 64, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 64, 64, 3, '*', '*')),
    ('cvb_train_pred_conv', ('*', 16, 22, 22, 128, '*', 5, 16, '*', '*', 85, 0)),
    ('cvb_train_pred_conv', ('*', 16, 22, 22, 128, '*', 80, 128, '*', '*', 85, 5)),
    ('cvb_train_pred_conv', ('*', 16, 42, 42, 128, '*', 5, 16, '*', '*', 85, 0)),
    ('cvb_train_pred_conv', ('*', 16, 42, 42, 128, '*', 80, 128, '*', '*', 85, 5)),
    ('cvb_train_pred_conv', ('*', 16, 82, 82, 128, '*', 5, 16, '*', '*', 85, 0)),
    ('cvb_train_pred_conv', ('*', 16, 82, 82, 128, '*', 80, 128, '*', '*', 85, 5)),
    ('cvb_train_pred_conv', ('*', 64, 20, 20, 512, '*', 255, 256, '*', '*', 255, 0)),
    ('cvb_train_pred_conv', ('*', 64, 40, 40, 256, '*', 255, 256, '*', '*', 255, 0)),
    ('cvb_train_pred_conv', ('*', 64, 80, 80, 128, '*', 255, 256, '*', '*', 255, 0)),
    ('cvb_train_pred_grad', ('*', 16, 85, 22, 22, 0, 5, 16, '*', '*')),
    ('cvb_train_pred_grad', ('*', 16, 85, 22, 22, 5, 80, 128, '*', '*')),
    ('cvb_train_pred_grad', ('*', 16, 85, 42, 42, 0, 5, 16, '*', '*')),
    ('cvb_train_pred_grad', ('*', 16, 85, 42, 42, 5, 80, 128, '*', '*')),
    ('cvb_train_pred_grad', ('*', 16, 85, 82, 82, 0, 5, 16, '*', '*')),
    ('cvb_train_pred_grad', ('*', 16, 85, 82, 82, 5, 80, 128, '*', '*')),
    ('cvb_train_pred_grad', ('*', 64, 255, 20, 20, 0, 255, 256, '*', '*')),
    ('cvb_train_pred_grad', ('*', 64, 255, 40, 40, 0, 255, 256, '*', '*')),
    ('cvb_train_pred_grad', ('*', 64, 255, 80, 80, 0, 255, 256, '*', '*')),
    ('cvb_train_spp_pool_bwd', ('*', '*', 16, 20, 20, 256, '*')),
    ('cvb_train_spp_pool_fwd', ('*', 16, 20, 20, 256, '*', '*')),
    ('cvb_train_sppf_chain_bwd', ('*', '*', 64, 20, 20, 256, '*', '*')),
    ('cvb_train_sppf_chain_fwd', ('*', 64, 20, 20, 256, '*', '*')),
    ('cvb_train_upsample_cat_bwd', ('*', 16, 20, 20, 256, 256, '*', '*')),
    ('cvb_train_upsample_cat_bwd', ('*', 16, 40, 40, 128, 128, '*', '*')),
    ('cvb_train_upsample_cat_bwd', ('*', 64, 20, 20, 256, 256, '*', '*')),
    ('cvb_train_upsample_cat_bwd', ('*', 64, 40, 40, 128, 128, '*', '*')),
    ('cvb_train_upsample_cat_fwd', ('*', 16, 20, 20, 256, '*', 256, '*')),
    ('cvb_train_upsample_cat_fwd', ('*', 16, 40, 40, 128, '*', 128, '*')),
    ('cvb_train_upsample_cat_fwd', ('*', 64, 20, 20, 256, '*', 256, '*')),
    ('cvb_train_upsample_cat_fwd', ('*', 64, 40, 40, 128, '*', 128, '*')),
    ('cvb_train_yolov5_loss_bwd', ('*', (64, 255, 80, 80, 64, 255, 40, 40, 64, 255, 20, 20), (1.25, 1.625, 2.0, 3.75, 4.125, 2.875, 1.875, 3.8125, 3.875, 2.8125, 3.6875, 7.4375, 3.625, 2.8125, 4.875, 6.1875, 11.65625, 10.1875), (4.0, 1.0, 0.4), 3, 3, 80, '*', 741, (4.0, 0.05, 1.0, 0.5, 1.0), '*', '*', '*', '*', 1204736, '*', '*')),
    ('cvb_train_yolov5_loss_fwd', ('*', (64, 255, 80, 80, 64, 255, 40, 40, 64, 255, 20, 20), (1.25, 1.625, 2.0, 3.75, 4.125, 2.875, 1.875, 3.8125, 3.875, 2.8125, 3.6875, 7.4375, 3.625, 2.8125, 4.875, 6.1875, 11.65625, 10.1875), (4.0, 1.0, 0.4), 3, 3, 80, '*', 741, (4.0, 0.05, 1.0, 0.5, 1.0), '*', '*', '*', '*', '*', 1204736)),
    ('cvb_train_yolox_loss_bwd', ('*', (16, 85, 82, 82, 16, 85, 42, 42, 16, 85, 22, 22), (8.0, 16.0, 32.0), 3, 80, '*', 16, 17, '*', '*', '*', '*', '*')),
    ('cvb_train_yolox_loss_fwd', ('*', (16, 85, 82, 82, 16, 85, 42, 42, 16, 85, 22, 22), (8.0, 16.0, 32.0), 3, 80, '*', 16, 17, '*', '*', '*', '*', 5330176)),
]


# ------------------------------------------------------------------------------------------------ recording the launches of a step
def _signature(name, args):
    """(name, arguments): ints and floats as passed, '*' / None for a pointer / NULL, the contents of int / float arrays, '*' for an array
    of device pointers.  Every cvb_train_* launch takes the stream last; it is left out."""
    from cvpytorch_b200 import _lib
    sig = []
    for t, v in zip(_lib.SYMBOLS[name][1][:-1], args[:-1]):
        if t is ctypes.c_void_p:
            sig.append(None if v is None or getattr(v, 'value', v) is None else '*')
        elif t in (ctypes.c_int32, ctypes.c_int64, ctypes.c_size_t):
            sig.append(int(v))
        elif t is ctypes.c_float:
            sig.append(round(float(v), 7))
        elif t is ctypes.POINTER(ctypes.c_int32):
            sig.append(tuple(int(x) for x in v))
        elif t is ctypes.POINTER(ctypes.c_float):
            sig.append(tuple(round(float(x), 7) for x in v))
        else:
            sig.append('*')
    return name, tuple(sig)


class _Recorder:
    """Stands in for the loaded library: records the signature of every cvb_train_* launch and forwards every call."""

    def __init__(self, lib):
        self._lib, self.seen = lib, set()

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith('cvb_train_') or name.endswith('_workspace_bytes'):
            return fn

        def call(*args):
            self.seen.add(_signature(name, args))
            return fn(*args)
        return call


@pytest.fixture
def recorder(cuda, monkeypatch):
    from cvpytorch_b200 import _lib
    rec = _Recorder(_lib.lib())
    monkeypatch.setattr(_lib, 'lib', lambda: rec)  # (every wrapper calls _lib.lib() at call time)
    return rec


def _yolov5_targets(B, gen):
    """tools/bench_yolov5_train.py's targets: 2 to 20 rows (image, class, cx, cy, w, h) per image."""
    rows = []
    for b in range(B):
        n = int(torch.randint(2, 21, (1,), generator=gen))
        rows.append(torch.cat([torch.full((n, 1), float(b)), torch.randint(0, NC, (n, 1), generator=gen).float(), torch.rand((n, 2), generator=gen) * 0.8 + 0.1,
                               torch.rand((n, 2), generator=gen) * 0.4 + 0.02], 1))
    return torch.cat(rows, 0)


def _yolov5_step():
    """One YOLOv5-s training step (forward, loss, backward) at 64 x 3 x 640², the benchmark's images and targets."""
    from cvpytorch_b200 import synth
    gen = torch.Generator().manual_seed(2024)
    m = synth.build_yolov5s().cuda().train()
    x = torch.rand(V5_B, 3, SIZE, SIZE, generator=gen).cuda()
    gts = _yolov5_targets(V5_B, gen).cuda()
    m(x, gts, 'train')['loss'].backward()
    torch.cuda.synchronize()


def _yolox_step():
    """One YOLOX-s training step at 16 x 3 x 640²: 2 to 20 boxes (cx, cy, w, h in pixels) per image."""
    from cvpytorch_b200 import synth
    gen = torch.Generator().manual_seed(1031)
    m = synth.build_yolox().cuda().train()
    x = torch.randn(X_B, 3, SIZE, SIZE, generator=gen).cuda()
    targets = []
    for _ in range(X_B):
        n = int(torch.randint(2, 21, (1,), generator=gen))
        c = 32 + torch.rand(n, 2, generator=gen) * (SIZE - 64)
        wh = 16 + torch.rand(n, 2, generator=gen) * 200
        targets.append({'labels': torch.randint(0, NC, (n,), generator=gen).cuda(), 'boxes': torch.cat([c, wh], 1).cuda()})
    m(x, targets, 'train')['loss'].backward()
    torch.cuda.synchronize()


def _table(sigs):
    return '\n'.join(f'    {s!r},' for s in sorted(sigs, key=repr))


def test_launch_table_matches_the_steps(recorder):
    for step in (_yolov5_step, _yolox_step):
        step()
        torch.cuda.empty_cache()
    got, want = recorder.seen, set(LAUNCHES)
    assert len(want) == len(LAUNCHES), 'LAUNCHES lists a signature twice'
    assert got == want, (f'launches of the two steps differ from LAUNCHES: new {_table(got - want)}\nno longer launched {_table(want - got)}\n'
                         f'recorded table:\n{_table(got)}')


# ------------------------------------------------------------------------------------------------ operands and calls
def _gen(what):
    return torch.Generator(device='cuda').manual_seed(zlib.crc32(repr(what).encode()))


def _operand(shape, exact, g):
    """bf16 tensor: {-1, 0, 1} (exact) or unit Gaussian."""
    if exact:
        return torch.randint(-1, 2, shape, generator=g, device='cuda').to(torch.bfloat16)
    return torch.randn(shape, generator=g, device='cuda').to(torch.bfloat16)


def _weight(cout, cin, k, exact, g):
    """fp32 weight of bf16 values: {-1, 0, 1} or Gaussian / sqrt(fan-in)."""
    if exact:
        return torch.randint(-1, 2, (cout, cin, k, k), generator=g, device='cuda').float()
    return (torch.randn((cout, cin, k, k), generator=g, device='cuda') / (cin * k * k) ** 0.5).to(torch.bfloat16).float()


def _stat_prev(C, g):
    """BN statistics [4][C] of a producing layer with per-channel scale and shift (rows 2, 3: all the SiLU' epilogue reads)."""
    return torch.stack([torch.zeros(C, device='cuda'), torch.ones(C, device='cuda'), torch.rand(C, generator=g, device='cuda') + 0.5,
                        torch.randn(C, generator=g, device='cuda') * 0.5]).contiguous()


def _nan(shape, dtype):
    return torch.full(shape, NAN, dtype=dtype, device='cuda')


def _call(name, *args):
    from cvpytorch_b200 import _lib
    _lib.check(getattr(_lib.lib(), name)(*args, _lib._stream()), name)


def _p(t):
    from cvpytorch_b200 import _lib
    return _lib._p(t)


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _assert_equal(out, ref, what):
    """out == ref element by element (ref float64, out cast to float64; a NaN never matches); the message names the first mismatch."""
    out = out.detach().double()
    assert out.shape == ref.shape, (what, tuple(out.shape), tuple(ref.shape))
    bad = ~(out == ref)
    n = int(bad.sum())
    if n:
        idx = tuple(int(i) for i in torch.nonzero(bad)[0])
        raise AssertionError(f'{what}: {n} of {ref.numel()} elements differ; first at {idx}: out={float(out[idx])!r} ref={float(ref[idx])!r}')


def _bf16_rn(t):
    """bf16 round-to-nearest of float64 integers below 2^24 (exact in fp32, so there is one rounding), as float64."""
    return t.float().to(torch.bfloat16).double()


def _crop(x64, pad):
    """A negative padding crops the border (the backward-data of the padding-1 1x1 head stems)."""
    return (x64[:, :, -pad:x64.shape[2] + pad, -pad:x64.shape[3] + pad], 0) if pad < 0 else (x64, pad)


def _silu_epilogue(acc, acc_err, yp, stat):
    """float64 of acc * silu'(y_prev * s + t) and its bound: the epilogue's error and the bf16 store, plus acc_err (the accumulation error,
    0 with integer operands) through |silu'| <= 1.1."""
    z = _nchw(yp).double() * stat[2].double().view(1, -1, 1, 1) + stat[3].double().view(1, -1, 1, 1)
    ref = acc * R.silu_grad64(z)
    bound = (R.BF16_REL + 2 * R.U24) * ref.abs() + (1 + R.BF16_REL) * (1.1 * acc_err + (acc.abs() + acc_err) * R.silu_grad_err(z))
    return ref, bound


def _check_accumulated(out, ref, absref, gamma, silu, what):
    """A bf16 conv output (NHWC) against float64 ref / absref (NCHW).  exact (gamma None): bitwise bf16_rn(ref), or within the SiLU'
    epilogue's bound; Gaussian: |out - ref| <= 2^-8 |ref| + (1 + 2^-8) gamma * absref."""
    out = _nchw(out)
    if silu is not None:
        ref, bound = _silu_epilogue(ref, 0 if gamma is None else gamma * absref, *silu)
        R.check(out, ref, bound, what + " with the SiLU' epilogue")
    elif gamma is None:
        _assert_equal(out, _bf16_rn(ref), what)
    else:
        R.check(out, ref, R.BF16_REL * ref.abs() + (1 + R.BF16_REL) * gamma * absref, what)


# ------------------------------------------------------------------------------------------------ the checks, by entry point
def _conv(name, a, exact):
    """cvb_train_conv / cvb_train_conv_pad: forward, stride-1 backward-data (the same GEMM over dy with the rotated weights), padded
    head stems.  out[B, Ho, Wo, cout] = conv(x, W) (* silu'(z_prev) with y_prev)."""
    from cvpytorch_b200 import train as T
    _, B, H, W, cin, _, cout, k, s_or_p, _, y_prev, _ = a
    stride, pad = (s_or_p, k // 2) if name == 'cvb_train_conv' else (1, s_or_p)
    g = _gen((name, a, exact))
    x = _operand((B, H, W, cin), exact, g)
    w = _weight(cout, cin, k, exact, g)
    wf, _ = T.pack_weights(w)
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    out = _nan((B, Ho, Wo, cout), torch.bfloat16)
    silu = None
    if y_prev is not None:
        silu = (_operand((B, Ho, Wo, cout), False, g) * 2, _stat_prev(cout, g))
    _call(name, _p(x), B, H, W, cin, _p(wf), cout, k, s_or_p, _p(out), _p(silu and silu[0]), _p(silu and silu[1]))
    x64, p = _crop(_nchw(x).double(), pad)
    if exact:
        ref, absref = F.conv2d(x64, w.double(), None, stride, p), None
    else:
        ref, absref = R.conv_fwd(x64, w, stride, p)
    del x64
    _check_accumulated(out, ref, absref, None if exact else R.mma_gamma(k * k * T.kpad(cin)), silu, name)


def _dgrad_s2(name, a, exact):
    """cvb_train_conv_dgrad_s2: dx[B, H, W, cin] of the 3x3 / stride 2 / pad 1 conv, four parity launches."""
    from cvpytorch_b200 import train as T
    _, B, Ho, Wo, cout, _, cin, H, W, _, y_prev, _ = a
    g = _gen((name, a, exact))
    dy = _operand((B, Ho, Wo, cout), exact, g)
    w = _weight(cout, cin, 3, exact, g)
    _, wb = T.pack_weights(w)
    dx = _nan((B, H, W, cin), torch.bfloat16)
    silu = (_operand((B, H, W, cin), False, g) * 2, _stat_prev(cin, g)) if y_prev is not None else None
    _call(name, _p(dy), B, Ho, Wo, cout, _p(wb), cin, H, W, _p(dx), _p(silu and silu[0]), _p(silu and silu[1]))
    ref, absref = R.conv_dgrad(_nchw(dy), w, (B, cin, H, W), 2, 1)
    _check_accumulated(dx, ref, absref, None if exact else R.mma_gamma(4 * T.kpad(cout)), silu, name)


def _wgrad(name, a, exact):
    """cvb_train_conv_wgrad / _pad: dw[cout, k*k, cin] (fp32, split atomics into a zeroed buffer) = sum over pixels of x * dy."""
    _, _, B, H, W, cin, cout, k, s_or_p, _ = a
    stride, pad = (s_or_p, k // 2) if name == 'cvb_train_conv_wgrad' else (1, s_or_p)
    g = _gen((name, a, exact))
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    x, dy = _operand((B, H, W, cin), exact, g), _operand((B, Ho, Wo, cout), exact, g)
    dw = torch.zeros((cout, k * k, cin), dtype=torch.float32, device='cuda')
    _call(name, _p(x), _p(dy), B, H, W, cin, cout, k, s_or_p, _p(dw))
    dw = dw.view(cout, k, k, cin).permute(0, 3, 1, 2)
    x64, p = _crop(_nchw(x).double(), pad)
    ref, absref = R.conv_wgrad(x64, _nchw(dy), (cout, cin, k, k), stride, p)
    if exact:
        _assert_equal(dw, ref, name)
    else:
        R.check(dw, ref, R.wgrad_gamma(B, Ho, Wo, cin, cout, k, _sms()) * absref, name)


def _pred_conv(name, a, exact):
    """cvb_train_pred_conv: fp32 NCHW out[:, c_off:c_off + cout] = conv + bias, the other channels untouched."""
    from cvpytorch_b200 import train as T
    _, B, H, W, cin, _, cout, cout_pad, _, _, c_tot, c_off = a
    g = _gen((name, a, exact))
    x = _operand((B, H, W, cin), exact, g)
    w = _weight(cout, cin, 1, exact, g)
    bias = (torch.randint(-4, 5, (cout,), generator=g, device='cuda').float() if exact else torch.randn(cout, generator=g, device='cuda'))
    wf, _ = T.pack_weights(F.pad(w, (0, 0, 0, 0, 0, 0, 0, cout_pad - cout)))
    out = _nan((B, c_tot, H, W), torch.float32)
    _call(name, _p(x), B, H, W, cin, _p(wf), cout, cout_pad, _p(bias), _p(out), c_tot, c_off)
    yr, ya = R.conv_fwd(_nchw(x), w, 1, 0)
    ref = yr + bias.double().view(1, -1, 1, 1)
    if exact:
        _assert_equal(out[:, c_off:c_off + cout], ref, name)
    else:
        R.check(out[:, c_off:c_off + cout], ref, R.mma_gamma(T.kpad(cin)) * ya + 2 * R.U24 * (yr.abs() + bias.double().abs().view(1, -1, 1, 1)), name)
    assert torch.isnan(out[:, :c_off]).all() and torch.isnan(out[:, c_off + cout:]).all(), f'{name}: wrote outside channels [{c_off}, {c_off + cout})'


def _pred_grad(name, a, exact):
    """cvb_train_pred_grad: dy bf16 NHWC [B, h, w, cout_pad] = bf16(g[:, c_off:c_off + cout]), zero-padded; dbias = its fp32 sum."""
    _, B, c_tot, h, w, c_off, cout, cout_pad, _, _ = a
    g = _gen((name, a, exact))
    gr = (torch.randint(-1, 2, (B, c_tot, h, w), generator=g, device='cuda').float() if exact else torch.randn((B, c_tot, h, w), generator=g, device='cuda'))
    dy, db = _nan((B, h, w, cout_pad), torch.bfloat16), _nan((cout,), torch.float32)
    _call(name, _p(gr), B, c_tot, h, w, c_off, cout, cout_pad, _p(dy), _p(db))
    gs = gr[:, c_off:c_off + cout].double()
    _assert_equal(dy[..., :cout], _nhwc(gr[:, c_off:c_off + cout]).to(torch.bfloat16).double(), name + ' dy')
    assert not bool(dy[..., cout:].any()), f'{name}: the padding channels of dy are not zero'
    if exact:
        _assert_equal(db, gs.sum((0, 2, 3)), name + ' dbias')
    else:
        terms = B * -(-(h * w) // 256) + 8  # (one thread's pixels, then the 256-thread tree)
        R.check(db, gs.sum((0, 2, 3)), terms * R.U24 * gs.abs().sum((0, 2, 3)), name + ' dbias')


def _bn_inputs(npix, C, exact, g):
    """y [npix, C] bf16 (exact: a per-channel pivot + {-1, 0, 1} with y[0] = the pivot, so every pivoted sum is an integer below 2^24;
    else Gaussian channels with mean = 10 std), gamma, beta, running statistics."""
    if exact:
        pivot = torch.randint(-8, 9, (C,), generator=g, device='cuda').float() * 0.5
        d = torch.randint(-1, 2, (npix, C), generator=g, device='cuda').float()
        d[0] = 0
        y = (pivot + d).to(torch.bfloat16)
    else:
        std = torch.rand(C, generator=g, device='cuda') * 1.5 + 0.5
        y = ((torch.randn(npix, C, generator=g, device='cuda') + 10) * std).to(torch.bfloat16)
    gamma, beta = torch.rand(C, generator=g, device='cuda') + 0.5, torch.randn(C, generator=g, device='cuda') * 0.5
    return y, gamma, beta, torch.randn(C, generator=g, device='cuda'), torch.rand(C, generator=g, device='cuda') + 0.5


def _bn_stats(y, npix, C, gamma, beta, rm, rv, eps, mom):
    stat, scratch = _nan((4, C), torch.float32), _nan((2, C), torch.float32)
    _call('cvb_train_bn_stats', _p(y), npix, C, _p(gamma), _p(beta), eps, mom, _p(rm), _p(rv), _p(scratch), _p(stat))
    return stat


def _bn_gs(npix, C, exact):
    return EXACT_GS if exact else (R.red_chain(npix, C, _sms()) + 2) * R.U24


def _bn_stats_check(name, a, exact):
    _, npix, C, _, _, eps, mom, _, _, _, _ = a
    y, gamma, beta, rm0, rv0 = _bn_inputs(npix, C, exact, _gen((name, a, exact)))
    rm, rv = rm0.clone(), rv0.clone()
    stat = _bn_stats(y, npix, C, gamma, beta, rm, rv, eps, mom)
    R.bn_stats_check(y, gamma, beta, rm0, rv0, eps, mom, stat, rm, rv, _bn_gs(npix, C, exact))


def _bn_silu_fwd(name, a, exact):
    _, npix, C, _, _ = a
    y, gamma, beta, rm, rv = _bn_inputs(npix, C, exact, _gen((name, a, exact)))
    stat = _bn_stats(y, npix, C, gamma, beta, rm, rv, 1e-3, 0.03)
    out = _nan((npix, C), torch.bfloat16)
    _call(name, _p(y), npix, C, _p(stat), _p(out))
    R.bn_silu_fwd_check(y, stat, out)


def _bn_silu_bwd(name, a, exact):
    """g = d(loss)/d(a) (is_dz 0) or d(loss)/d(z) (is_dz 1, fed by the fused SiLU' epilogue).  exact: integer g makes sum dz exact for g = dz;
    with g = d(loss)/d(a), dz = g * silu'(z) is no integer and the sums keep their summation bound."""
    _, is_dz, _, npix, C, _, _, _, _ = a
    g = _gen((name, a, exact))
    y, gamma, beta, rm, rv = _bn_inputs(npix, C, exact, g)
    stat = _bn_stats(y, npix, C, gamma, beta, rm, rv, 1e-3, 0.03)
    da = _operand((npix, C), exact, g)
    sums, dy = _nan((2, C), torch.float32), _nan((npix, C), torch.bfloat16)
    _call(name, _p(da), is_dz, _p(y), npix, C, _p(stat), _p(gamma), _p(sums), _p(dy))
    gs = _bn_gs(npix, C, False)
    R.bn_silu_bwd_check(da, is_dz, y, gamma, stat, sums, dy, gs, gs_sum=0.0 if exact and is_dz else None)


def _focus_s2d(name, a, exact):
    _, B, H, W, _ = a
    img = torch.randn((B, 3, H, W), generator=_gen((name, a)), device='cuda')
    out = _nan((B, H // 2, W // 2, 16), torch.bfloat16)
    _call(name, _p(img), B, H, W, _p(out))
    ref = torch.cat((img[..., ::2, ::2], img[..., 1::2, ::2], img[..., ::2, 1::2], img[..., 1::2, 1::2]), 1)
    _assert_equal(out, F.pad(_nhwc(ref), (0, 4)).to(torch.bfloat16).double(), name)


def _pool_ref(a, chained):
    """float64 autograd reference of [a | pools]: the chained YOLOv5 SPPF (y_i = maxpool5(y_(i-1))) or YOLOX's parallel 5 / 9 / 13."""
    x = _nchw(a).double().requires_grad_(True)
    if chained:
        ys = [x]
        for _ in range(3):
            ys.append(F.max_pool2d(ys[-1], 5, 1, 2))
    else:
        ys = [x] + [F.max_pool2d(x, k, 1, k // 2) for k in (5, 9, 13)]
    return x, torch.cat(ys, 1)


def _pool(name, a, exact):
    """cvb_train_sppf_chain_* / cvb_train_spp_pool_*: forward bitwise; backward of integer gradients equal to bf16(the float64 sums), with
    autograd's routing of ties (bf16 values of a Gaussian tie often in a 13 x 13 window)."""
    chained = 'sppf_chain' in name
    B, H, W, C = a[1:5] if name.endswith('_fwd') else a[2:6]
    g = _gen((name, a))
    act = _operand((B, H, W, C), False, g)
    x, ref = _pool_ref(act, chained)
    if name.endswith('_fwd'):
        cat, idx = _nan((B, H, W, 4 * C), torch.bfloat16), torch.full((3, B, H, W, C), 255, dtype=torch.uint8, device='cuda')
        _call(name, _p(act), B, H, W, C, _p(cat), _p(idx))
        _assert_equal(_nchw(cat), ref.detach(), name)
        return
    from cvpytorch_b200 import train as T
    _, idx = (T.sppf_chain if chained else T.spp_pool)(act)
    gr = _operand((B, H, W, 4 * C), True, g)
    ref.backward(_nchw(gr).double())
    da = _nan((B, H, W, C), torch.bfloat16)
    if chained:
        _call(name, _p(gr), _p(idx), B, H, W, C, _p(_nan((2, B, H, W, C), torch.float32)), _p(da))
    else:
        _call(name, _p(gr), _p(idx), B, H, W, C, _p(da))
    _assert_equal(_nchw(da), _bf16_rn(x.grad), name)


def _upsample_cat(name, a, exact):
    """Forward bitwise; backward: db = g[..., Ca:] bitwise, da = bf16 of the 2x2 sums of integer gradients (exact in fp32)."""
    g = _gen((name, a))
    if name.endswith('_fwd'):
        _, B, h, w, Ca, _, Cb, _ = a
        x, y = _operand((B, h, w, Ca), False, g), _operand((B, 2 * h, 2 * w, Cb), False, g)
        cat = _nan((B, 2 * h, 2 * w, Ca + Cb), torch.bfloat16)
        _call(name, _p(x), B, h, w, Ca, _p(y), Cb, _p(cat))
        ref = torch.cat([F.interpolate(_nchw(x).double(), scale_factor=2, mode='nearest'), _nchw(y).double()], 1)
        _assert_equal(_nchw(cat), ref, name)
        return
    _, B, h, w, Ca, Cb, _, _ = a
    gr = _operand((B, 2 * h, 2 * w, Ca + Cb), True, g)
    da, db = _nan((B, h, w, Ca), torch.bfloat16), _nan((B, 2 * h, 2 * w, Cb), torch.bfloat16)
    _call(name, _p(gr), B, h, w, Ca, Cb, _p(da), _p(db))
    _assert_equal(db, gr[..., Ca:].double(), name + ' db')
    _assert_equal(_nchw(da), _bf16_rn(F.avg_pool2d(_nchw(gr[..., :Ca]).double(), 2) * 4), name + ' da')


def _pack_weights(name, a, exact):
    """[cout, cin, k, k] fp32 -> bf16 [cout, k*k, kpad(cin)] and the rotated [cin, k*k, kpad(cout)], zero K padding, bitwise."""
    from cvpytorch_b200 import train as T
    _, cout, cin, k, _, _ = a
    w = torch.randn((cout, cin, k, k), generator=_gen((name, a)), device='cuda')
    wf, wb = _nan((cout, k * k, T.kpad(cin)), torch.bfloat16), _nan((cin, k * k, T.kpad(cout)), torch.bfloat16)
    _call(name, _p(w), cout, cin, k, _p(wf), _p(wb))
    w16 = w.to(torch.bfloat16).double()
    ref_f = F.pad(w16.permute(0, 2, 3, 1).reshape(cout, k * k, cin), (0, T.kpad(cin) - cin))
    ref_b = F.pad(w16.flip(2, 3).permute(1, 2, 3, 0).reshape(cin, k * k, cout), (0, T.kpad(cout) - cout))
    _assert_equal(wf, ref_f, name + ' forward layout')
    _assert_equal(wb, ref_b, name + ' backward-data layout')


_LOSSES_CHECKED = set()


def _yolov5_loss(name, a, exact):
    """The recorded level shapes and target count against the oracle (test_yolov5_train_gpu._check: candidate lists exactly, loss terms
    within 1e-5, gradients within 1e-5 max-normalised); forward and backward of one step share the check."""
    import test_yolov5_train_gpu as V5
    shapes, anchors, nt = a[1], a[2], a[8]
    levels = [shapes[4 * i:4 * i + 4] for i in range(len(shapes) // 4)]
    assert anchors == tuple(round(v, 7) for v in np.array(V5.ANCHORS, dtype=np.float32).flatten().tolist()), anchors
    key = ('yolov5', shapes, nt)
    if key in _LOSSES_CHECKED:
        return
    g = torch.Generator().manual_seed(nt)
    preds = [(torch.randn(s, generator=g) * 1.5).cuda() for s in levels]
    V5._check(preds, V5._targets(levels[0][0], nt, NC, nt, awkward=False), NC)
    _LOSSES_CHECKED.add(key)


def _yolox_loss(name, a, exact):
    """The recorded level shapes and GT capacity against the oracle (test_yolox_loss_gpu._check: assignments equal in every image without a
    near-tie, loss terms and gradients within 1e-5); forward and backward share the check."""
    import test_yolox_loss_gpu as XL
    shapes, strides, B, max_gt = a[1], a[2], a[6], a[7]
    assert strides == tuple(float(s) for s in XL.STRIDES), strides
    key = ('yolox', shapes, max_gt)
    if key in _LOSSES_CHECKED:
        return
    H, W = (shapes[2] - 2) * XL.STRIDES[0], (shapes[3] - 2) * XL.STRIDES[0]
    counts = [2 + (7 * i) % (max_gt - 1) for i in range(B)]
    counts[-1] = max_gt
    preds, targets = XL._random_case(max_gt, B, H, W, NC, counts)
    assert [tuple(p.shape) for p in preds] == [shapes[4 * i:4 * i + 4] for i in range(len(preds))]
    compared = XL._check(preds, targets, NC, name)
    print('images compared (no near-tie):', compared, 'of', B)
    _LOSSES_CHECKED.add(key)


CHECKS = {'cvb_train_conv': _conv, 'cvb_train_conv_pad': _conv, 'cvb_train_conv_dgrad_s2': _dgrad_s2, 'cvb_train_conv_wgrad': _wgrad,
          'cvb_train_conv_wgrad_pad': _wgrad, 'cvb_train_pred_conv': _pred_conv, 'cvb_train_pred_grad': _pred_grad,
          'cvb_train_bn_stats': _bn_stats_check, 'cvb_train_bn_silu_fwd': _bn_silu_fwd, 'cvb_train_bn_silu_bwd': _bn_silu_bwd,
          'cvb_train_focus_s2d': _focus_s2d, 'cvb_train_sppf_chain_fwd': _pool, 'cvb_train_sppf_chain_bwd': _pool,
          'cvb_train_spp_pool_fwd': _pool, 'cvb_train_spp_pool_bwd': _pool, 'cvb_train_upsample_cat_fwd': _upsample_cat,
          'cvb_train_upsample_cat_bwd': _upsample_cat, 'cvb_train_pack_weights': _pack_weights,
          'cvb_train_yolov5_loss_fwd': _yolov5_loss, 'cvb_train_yolov5_loss_bwd': _yolov5_loss,
          'cvb_train_yolox_loss_fwd': _yolox_loss, 'cvb_train_yolox_loss_bwd': _yolox_loss}
# the element-wise and data-movement kernels are bitwise in both operand kinds, the losses have their oracle: one run each
ONE_KIND = ('cvb_train_focus_s2d', 'cvb_train_sppf_chain_fwd', 'cvb_train_sppf_chain_bwd', 'cvb_train_spp_pool_fwd', 'cvb_train_spp_pool_bwd',
            'cvb_train_upsample_cat_fwd', 'cvb_train_upsample_cat_bwd', 'cvb_train_pack_weights', 'cvb_train_yolov5_loss_fwd',
            'cvb_train_yolov5_loss_bwd', 'cvb_train_yolox_loss_fwd', 'cvb_train_yolox_loss_bwd')


def _id(sig):
    name, args = sig
    parts = ['NULL' if v is None else 'x'.join(map(str, v)) if isinstance(v, tuple) else str(v) for v in args if v != '*']
    return '-'.join([name[len('cvb_train_'):]] + parts)


def _run(sig):
    name, args = sig
    for exact in (True,) if name in ONE_KIND else (True, False):
        CHECKS[name](name, args, exact)
        torch.cuda.synchronize()
    torch.cuda.empty_cache()


# small shapes of the same entry points: the exactness the checks rely on, confirmed where a failure is cheap to read
SMALL = [('cvb_train_conv', ('*', 2, 16, 16, 64, '*', 64, 3, 1, '*', None, None)),
         ('cvb_train_conv', ('*', 2, 16, 16, 64, '*', 128, 3, 1, '*', '*', '*')),
         ('cvb_train_conv_dgrad_s2', ('*', 2, 8, 8, 64, '*', 32, 16, 16, '*', None, None)),
         ('cvb_train_conv_wgrad', ('*', '*', 2, 16, 16, 64, 64, 3, 1, '*')),
         ('cvb_train_conv_wgrad', ('*', '*', 16, 48, 48, 64, 64, 1, 1, '*')),
         ('cvb_train_pred_conv', ('*', 2, 10, 12, 64, '*', 80, 128, '*', '*', 85, 5)),
         ('cvb_train_bn_stats', ('*', 1000, 64, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
         ('cvb_train_bn_silu_bwd', ('*', 1, '*', 1000, 64, '*', '*', '*', '*'))]


@pytest.mark.parametrize('sig', SMALL, ids=[_id(s) for s in SMALL])
def test_small_shape_of_each_check(cuda, sig):
    _run(sig)


@pytest.mark.parametrize('sig', LAUNCHES, ids=[_id(s) for s in LAUNCHES])
def test_launch_at_its_real_shape(cuda, sig):
    _run(sig)


# ------------------------------------------------------------------------------------------------ the exact check has teeth
def test_exact_check_sees_a_lost_tile_and_swapped_parity_classes(cuda):
    """The YOLOv5-s stem backward-weight (64 x 320² pixels, 16 -> 32, 3x3): a reference with one 128-pixel tile of dy zeroed (the kernel's
    last tile, in the last images) differs from the kernel's dw, which equals the true reference.  The stage-1 stride-2 backward-data (dy 64 x 160² x 64
    -> dx 64 x 320² x 32): a reference with the parity classes (0, 0) and (1, 1) swapped differs from the kernel's dx.  Also reports whether
    the Gaussian check (b) would have seen the lost tile."""
    stem = ('cvb_train_conv_wgrad', ('*', '*', V5_B, 320, 320, 16, 32, 3, 1, '*'))
    down = ('cvb_train_conv_dgrad_s2', ('*', V5_B, 160, 160, 64, '*', 32, 320, 320, '*', None, None))
    assert stem in LAUNCHES and down in LAUNCHES
    B, H, W, cin, cout, k = stem[1][2:8]
    tw, th, nb = R.choose_box128(B, H, W)
    last = (slice((-(-B // nb) - 1) * nb, B), slice((-(-H // th) - 1) * th, H), slice((-(-W // tw) - 1) * tw, W))
    assert (last[0].stop - last[0].start) * (last[1].stop - last[1].start) * (last[2].stop - last[2].start) == 128, (tw, th, nb)

    def references(exact):
        """-> operands, float64 dw and |dw| reference, and the reference with the last tile of dy zeroed."""
        g = _gen(('teeth', exact))
        x, dy = _operand((B, H, W, cin), exact, g), _operand((B, H, W, cout), exact, g)
        ref, absref = R.conv_wgrad(_nchw(x), _nchw(dy), (cout, cin, k, k), 1, 1)
        dy_lost = dy.clone()
        dy_lost[last] = 0
        lost, _ = R.conv_wgrad(_nchw(x), _nchw(dy_lost), (cout, cin, k, k), 1, 1)
        return x, dy, ref, absref, lost

    x, dy, ref, _, lost = references(True)
    dw = torch.zeros((cout, k * k, cin), dtype=torch.float32, device='cuda')
    _call(stem[0], _p(x), _p(dy), B, H, W, cin, cout, k, 1, _p(dw))
    dw = dw.view(cout, k, k, cin).permute(0, 3, 1, 2).double()
    _assert_equal(dw, ref, 'stem backward-weight')
    n_diff = int((dw != lost).sum())
    print(f'lost tile: {n_diff} of {dw.numel()} dw elements differ from the reference without it, by up to {float((ref - lost).abs().max()):.0f}')
    assert n_diff > 0, 'the exact check does not see a lost 128-pixel tile'
    del x, dy, ref, lost, dw

    _, _, ref, absref, lost = references(False)
    bound = R.wgrad_gamma(B, H, W, cin, cout, k, _sms()) * absref
    caught = bool(((ref - lost).abs() > bound).any())
    print(f'Gaussian check (b) would {"" if caught else "NOT "}have caught the lost tile: largest change / bound '
          f'{float(((ref - lost).abs() / bound).max()):.3g}, bound {float(bound.min()):.3g} .. {float(bound.max()):.3g}')
    del ref, absref, lost, bound

    from cvpytorch_b200 import train as T
    _, B, Ho, Wo, co, _, ci, H, W, _, _, _ = down[1]
    g = _gen(('teeth', 'parity'))
    dy = _operand((B, Ho, Wo, co), True, g)
    w = _weight(co, ci, 3, True, g)
    dx = _nan((B, H, W, ci), torch.bfloat16)
    _call(down[0], _p(dy), B, Ho, Wo, co, _p(T.pack_weights(w)[1]), ci, H, W, _p(dx), None, None)
    ref, _ = R.conv_dgrad(_nchw(dy), w, (B, ci, H, W), 2, 1)
    ref = _bf16_rn(ref)
    _assert_equal(_nchw(dx), ref, 'stride-2 backward-data')
    swapped = ref.clone()
    swapped[:, :, 0::2, 0::2], swapped[:, :, 1::2, 1::2] = ref[:, :, 1::2, 1::2], ref[:, :, 0::2, 0::2]
    n_diff = int((_nchw(dx).double() != swapped).sum())
    print(f'swapped parity classes: {n_diff} of {dx.numel()} dx elements differ')
    assert n_diff > 0, 'the exact check does not see two swapped parity classes'
