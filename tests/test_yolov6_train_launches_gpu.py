"""Every training-kernel launch of the YOLOv6 training steps, at its real shape: one YOLOv6-s step at 64 x 3 x 640² (the batch of
coco_yolov6_s.yml, tools/bench_yolov6_train.py) and one YOLOv6-n step at 16 x 3 x 640² (its 16 / 32-wide blocks and the zero-padded
128-channel bifusion1.cv3), 80 classes and 2 to 20 targets per image.

The method is tests/test_train_launches_gpu.py's, whose helpers this file imports: LAUNCHES is the set of distinct cvb_train_* signatures of
the two steps, test_launch_table_matches_the_steps records both steps through a proxy of _lib.lib() and requires the recorded set to equal
LAUNCHES, and every signature then runs stand-alone into NaN-filled outputs, (a) with exact integer operands, where the kernel must equal
float64 (bf16 outputs bitwise bf16_rn of it), and (b) with Gaussian operands against the float64 bounds of fp64ref.  The convolutions (the
4c-column transposed-conv GEMMs and the zero-padded stride-2 centre-tap branches included), BatchNorm statistics, SiLU passes, pools,
prediction convs and weight packing use that file's checks.  The YOLOv6 passes:
  cvb_train_bn_relu_fwd      relu(fmaf(y, scale, shift)) rounded to bf16, bitwise in both operand kinds.
  cvb_train_bn_relu_bwd      fp64ref.bn_silu_bwd_check with g * [z > 0] as dz (z the same fp32 fma); sum dz exact with integer g.
  cvb_train_repvgg_fwd       relu((z3 + z1) [+ zid]) in fp32, each z_b one fma, rounded to bf16: bitwise in both operand kinds.
  cvb_train_repvgg_bwd       dz = g * [a > 0] from the forward's a; every branch's (dbeta, dgamma_b, dy_b) through bn_silu_bwd_check.
  cvb_train_convt_scatter    bf16(fp32(u) + bias) at the scattered pixel, bitwise.
  cvb_train_convt_gather     du bitwise (a permutation); dbias equal to the float64 sum with integer g, within its summation bound else.
The YOLOv6 loss runs its oracle check (test_yolov6_loss_gpu) at the step's batch, 640² and 80 classes."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fp64ref as R  # noqa: E402
import test_train_launches_gpu as TL  # noqa: E402
from test_train_launches_gpu import recorder  # noqa: E402,F401  (the recording fixture)
from test_yolov6_host import DICT, use_model  # noqa: E402  (conf/det/yolov6/coco_yolov6_{n,s}.yml USE_MODEL, 80 classes)

pytestmark = pytest.mark.gpu
SIZE, NC = 640, 80
STEPS = {'s': 64, 'n': 16}  # YOLOv6 width -> batch

LAUNCHES = [
    ('cvb_train_bn_relu_bwd', ('*', '*', 102400, 128, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_bwd', ('*', '*', 102400, 32, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_bwd', ('*', '*', 102400, 64, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_bwd', ('*', '*', 1638400, 64, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_bwd', ('*', '*', 25600, 128, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_bwd', ('*', '*', 25600, 256, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_bwd', ('*', '*', 25600, 32, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_bwd', ('*', '*', 25600, 512, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_bwd', ('*', '*', 25600, 64, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_bwd', ('*', '*', 409600, 128, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_bwd', ('*', '*', 409600, 32, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_bwd', ('*', '*', 409600, 64, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_bwd', ('*', '*', 6400, 128, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_bwd', ('*', '*', 6400, 256, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_bwd', ('*', '*', 6400, 64, '*', '*', '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 102400, 128, '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 102400, 32, '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 102400, 64, '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 1638400, 64, '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 25600, 128, '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 25600, 256, '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 25600, 32, '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 25600, 512, '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 25600, 64, '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 409600, 128, '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 409600, 32, '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 409600, 64, '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 6400, 128, '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 6400, 256, '*', '*')),
    ('cvb_train_bn_relu_fwd', ('*', 6400, 64, '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 102400, 128, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 102400, 32, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 25600, 256, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 25600, 64, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 409600, 64, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_bwd', ('*', 0, '*', 6400, 128, '*', '*', '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 102400, 128, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 102400, 32, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 25600, 256, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 25600, 64, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 409600, 64, '*', '*')),
    ('cvb_train_bn_silu_fwd', ('*', 6400, 128, '*', '*')),
    ('cvb_train_bn_stats', ('*', 102400, 128, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 102400, 256, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 102400, 32, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 102400, 64, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 1638400, 16, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 1638400, 64, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 25600, 128, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 25600, 256, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 25600, 32, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 25600, 512, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 25600, 64, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 409600, 128, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 409600, 32, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 409600, 64, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 6400, 128, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 6400, 256, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 6400, 64, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_bn_stats', ('*', 6553600, 32, '*', '*', 0.001, 0.03, '*', '*', '*', '*')),
    ('cvb_train_conv', ('*', 16, 160, 160, 32, '*', 32, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 160, 160, 32, '*', 32, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 160, 160, 32, '*', 32, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 160, 160, 32, '*', 64, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 128, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 128, '*', 128, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 128, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 128, '*', 512, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 16, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 256, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 256, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 256, '*', 256, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 256, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 512, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 20, 20, 64, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 320, 320, 16, '*', 16, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 320, 320, 16, '*', 32, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 128, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 128, '*', 128, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 128, '*', 256, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 128, '*', 32, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 128, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 16, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 192, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 32, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 32, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 64, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 64, '*', 192, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 64, '*', 32, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 64, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 64, '*', 64, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 40, 40, 64, '*', 64, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 128, '*', 32, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 16, '*', 32, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 32, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 32, '*', 32, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 32, '*', 32, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 32, '*', 32, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 32, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 64, '*', 128, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 64, '*', 32, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 64, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 64, '*', 64, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 16, 80, 80, 64, '*', 64, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 160, 160, 64, '*', 128, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 160, 160, 64, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 160, 160, 64, '*', 64, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 160, 160, 64, '*', 64, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 1024, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 128, '*', 512, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 16, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 256, '*', 1024, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 256, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 256, '*', 256, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 256, '*', 512, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 512, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 512, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 512, '*', 512, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 20, 20, 512, '*', 512, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 320, 320, 16, '*', 32, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 320, 320, 32, '*', 64, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 128, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 128, '*', 128, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 128, '*', 128, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 128, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 128, '*', 384, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 128, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 16, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 256, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 256, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 256, '*', 256, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 256, '*', 512, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 256, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 384, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 64, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 40, 40, 64, '*', 256, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 128, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 128, '*', 128, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 128, '*', 128, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 128, '*', 256, 3, 2, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 128, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 16, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 192, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 64, '*', 128, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 64, '*', 192, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 64, '*', 64, 1, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 64, '*', 64, 3, 1, '*', None, None)),
    ('cvb_train_conv', ('*', 64, 80, 80, 64, '*', 64, 3, 2, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 16, 160, 160, 32, '*', 16, 320, 320, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 16, 20, 20, 256, '*', 128, 40, 40, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 16, 20, 20, 64, '*', 64, 40, 40, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 16, 40, 40, 128, '*', 64, 80, 80, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 16, 40, 40, 32, '*', 32, 80, 80, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 16, 40, 40, 64, '*', 64, 80, 80, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 16, 80, 80, 32, '*', 32, 160, 160, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 16, 80, 80, 64, '*', 32, 160, 160, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 64, 160, 160, 64, '*', 32, 320, 320, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 64, 20, 20, 128, '*', 128, 40, 40, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 64, 20, 20, 512, '*', 256, 40, 40, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 64, 40, 40, 128, '*', 128, 80, 80, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 64, 40, 40, 256, '*', 128, 80, 80, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 64, 40, 40, 64, '*', 64, 80, 80, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 64, 80, 80, 128, '*', 64, 160, 160, '*', None, None)),
    ('cvb_train_conv_dgrad_s2', ('*', 64, 80, 80, 64, '*', 64, 160, 160, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 20, 20, 128, '*', 128, 1, 0, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 20, 20, 128, '*', 128, 3, 1, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 40, 40, 64, '*', 64, 1, 0, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 40, 40, 64, '*', 64, 3, 1, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 80, 80, 32, '*', 32, 1, 0, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 16, 80, 80, 32, '*', 32, 3, 1, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 64, 20, 20, 256, '*', 256, 1, 0, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 64, 20, 20, 256, '*', 256, 3, 1, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 64, 40, 40, 128, '*', 128, 1, 0, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 64, 40, 40, 128, '*', 128, 3, 1, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 64, 80, 80, 64, '*', 64, 1, 0, '*', None, None)),
    ('cvb_train_conv_pad', ('*', 64, 80, 80, 64, '*', 64, 3, 1, '*', None, None)),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 160, 160, 32, 32, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 160, 160, 32, 32, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 160, 160, 32, 32, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 160, 160, 32, 64, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 20, 20, 128, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 20, 20, 128, 128, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 20, 20, 128, 16, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 20, 20, 256, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 20, 20, 256, 256, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 20, 20, 256, 256, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 20, 20, 256, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 20, 20, 512, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 20, 20, 64, 256, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 320, 320, 16, 16, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 320, 320, 16, 32, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 128, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 128, 128, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 128, 256, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 128, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 192, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 32, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 64, 16, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 64, 32, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 64, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 64, 64, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 40, 40, 64, 64, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 128, 32, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 32, 16, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 32, 32, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 32, 32, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 32, 32, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 64, 128, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 64, 32, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 64, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 64, 64, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 16, 80, 80, 64, 64, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 160, 160, 64, 128, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 160, 160, 64, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 160, 160, 64, 64, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 160, 160, 64, 64, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 20, 20, 1024, 256, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 20, 20, 128, 512, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 20, 20, 256, 16, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 20, 20, 256, 256, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 20, 20, 256, 256, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 20, 20, 512, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 20, 20, 512, 256, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 20, 20, 512, 512, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 20, 20, 512, 512, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 320, 320, 16, 32, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 320, 320, 32, 64, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 128, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 128, 128, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 128, 128, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 128, 16, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 128, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 256, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 256, 256, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 256, 256, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 256, 512, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 384, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 40, 40, 64, 256, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 128, 128, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 128, 128, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 128, 128, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 128, 256, 3, 2, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 128, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 192, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 64, 16, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 64, 64, 1, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 64, 64, 3, 1, '*')),
    ('cvb_train_conv_wgrad', ('*', '*', 64, 80, 80, 64, 64, 3, 2, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 16, 20, 20, 128, 128, 1, 0, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 16, 20, 20, 128, 128, 3, 1, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 16, 40, 40, 64, 64, 1, 0, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 16, 40, 40, 64, 64, 3, 1, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 16, 80, 80, 32, 32, 1, 0, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 16, 80, 80, 32, 32, 3, 1, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 64, 20, 20, 256, 256, 1, 0, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 64, 20, 20, 256, 256, 3, 1, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 64, 40, 40, 128, 128, 1, 0, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 64, 40, 40, 128, 128, 3, 1, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 64, 80, 80, 64, 64, 1, 0, '*')),
    ('cvb_train_conv_wgrad_pad', ('*', '*', 64, 80, 80, 64, 64, 3, 1, '*')),
    ('cvb_train_convt_gather', ('*', 16, 20, 20, 64, '*', '*', '*')),
    ('cvb_train_convt_gather', ('*', 16, 40, 40, 32, '*', '*', '*')),
    ('cvb_train_convt_gather', ('*', 64, 20, 20, 128, '*', '*', '*')),
    ('cvb_train_convt_gather', ('*', 64, 40, 40, 64, '*', '*', '*')),
    ('cvb_train_convt_scatter', ('*', 16, 20, 20, 64, '*', '*')),
    ('cvb_train_convt_scatter', ('*', 16, 40, 40, 32, '*', '*')),
    ('cvb_train_convt_scatter', ('*', 64, 20, 20, 128, '*', '*')),
    ('cvb_train_convt_scatter', ('*', 64, 40, 40, 64, '*', '*')),
    ('cvb_train_focus_s2d', ('*', 16, 640, 640, '*')),
    ('cvb_train_focus_s2d', ('*', 64, 640, 640, '*')),
    ('cvb_train_pack_weights', ('*', 128, 128, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 128, 128, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 128, 256, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 128, 32, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 128, 384, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 128, 512, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 128, 64, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 128, 64, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 16, 128, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 16, 16, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 16, 256, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 16, 32, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 16, 64, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 256, 1024, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 256, 128, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 256, 256, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 256, 256, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 256, 512, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 256, 64, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 32, 128, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 32, 16, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 32, 32, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 32, 32, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 32, 64, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 512, 128, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 512, 256, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 512, 512, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 512, 512, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 64, 128, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 64, 192, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 64, 256, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 64, 32, 3, '*', '*')),
    ('cvb_train_pack_weights', ('*', 64, 64, 1, '*', '*')),
    ('cvb_train_pack_weights', ('*', 64, 64, 3, '*', '*')),
    ('cvb_train_pred_conv', ('*', 16, 20, 20, 128, '*', 4, 16, '*', '*', 4, 0)),
    ('cvb_train_pred_conv', ('*', 16, 20, 20, 128, '*', 80, 128, '*', '*', 80, 0)),
    ('cvb_train_pred_conv', ('*', 16, 40, 40, 64, '*', 4, 16, '*', '*', 4, 0)),
    ('cvb_train_pred_conv', ('*', 16, 40, 40, 64, '*', 80, 128, '*', '*', 80, 0)),
    ('cvb_train_pred_conv', ('*', 16, 80, 80, 32, '*', 4, 16, '*', '*', 4, 0)),
    ('cvb_train_pred_conv', ('*', 16, 80, 80, 32, '*', 80, 128, '*', '*', 80, 0)),
    ('cvb_train_pred_conv', ('*', 64, 20, 20, 256, '*', 4, 16, '*', '*', 4, 0)),
    ('cvb_train_pred_conv', ('*', 64, 20, 20, 256, '*', 80, 128, '*', '*', 80, 0)),
    ('cvb_train_pred_conv', ('*', 64, 40, 40, 128, '*', 4, 16, '*', '*', 4, 0)),
    ('cvb_train_pred_conv', ('*', 64, 40, 40, 128, '*', 80, 128, '*', '*', 80, 0)),
    ('cvb_train_pred_conv', ('*', 64, 80, 80, 64, '*', 4, 16, '*', '*', 4, 0)),
    ('cvb_train_pred_conv', ('*', 64, 80, 80, 64, '*', 80, 128, '*', '*', 80, 0)),
    ('cvb_train_pred_grad', ('*', 16, 4, 20, 20, 0, 4, 16, '*', '*')),
    ('cvb_train_pred_grad', ('*', 16, 4, 40, 40, 0, 4, 16, '*', '*')),
    ('cvb_train_pred_grad', ('*', 16, 4, 80, 80, 0, 4, 16, '*', '*')),
    ('cvb_train_pred_grad', ('*', 64, 4, 20, 20, 0, 4, 16, '*', '*')),
    ('cvb_train_pred_grad', ('*', 64, 4, 40, 40, 0, 4, 16, '*', '*')),
    ('cvb_train_pred_grad', ('*', 64, 4, 80, 80, 0, 4, 16, '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 102400, 128, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 102400, 256, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 102400, 32, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 102400, 64, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 1638400, 64, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 25600, 128, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 25600, 256, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 25600, 512, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 25600, 64, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 409600, 128, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 409600, 32, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 409600, 64, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 6400, 128, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 6400, 256, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', None, 102400, 256, '*', '*', None, '*', '*', None, '*', '*', '*', None)),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', None, 102400, 64, '*', '*', None, '*', '*', None, '*', '*', '*', None)),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', None, 1638400, 16, '*', '*', None, '*', '*', None, '*', '*', '*', None)),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', None, 1638400, 64, '*', '*', None, '*', '*', None, '*', '*', '*', None)),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', None, 25600, 128, '*', '*', None, '*', '*', None, '*', '*', '*', None)),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', None, 25600, 512, '*', '*', None, '*', '*', None, '*', '*', '*', None)),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', None, 409600, 128, '*', '*', None, '*', '*', None, '*', '*', '*', None)),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', None, 409600, 32, '*', '*', None, '*', '*', None, '*', '*', '*', None)),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', None, 6400, 256, '*', '*', None, '*', '*', None, '*', '*', '*', None)),
    ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', None, 6553600, 32, '*', '*', None, '*', '*', None, '*', '*', '*', None)),
    ('cvb_train_repvgg_fwd', ('*', '*', '*', 102400, 128, '*', '*', '*', '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', '*', 102400, 256, '*', '*', '*', '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', '*', 102400, 32, '*', '*', '*', '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', '*', 102400, 64, '*', '*', '*', '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', '*', 1638400, 64, '*', '*', '*', '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', '*', 25600, 128, '*', '*', '*', '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', '*', 25600, 256, '*', '*', '*', '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', '*', 25600, 512, '*', '*', '*', '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', '*', 25600, 64, '*', '*', '*', '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', '*', 409600, 128, '*', '*', '*', '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', '*', 409600, 32, '*', '*', '*', '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', '*', 409600, 64, '*', '*', '*', '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', '*', 6400, 128, '*', '*', '*', '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', '*', 6400, 256, '*', '*', '*', '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', None, 102400, 256, '*', '*', None, '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', None, 102400, 64, '*', '*', None, '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', None, 1638400, 16, '*', '*', None, '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', None, 1638400, 64, '*', '*', None, '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', None, 25600, 128, '*', '*', None, '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', None, 25600, 512, '*', '*', None, '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', None, 409600, 128, '*', '*', None, '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', None, 409600, 32, '*', '*', None, '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', None, 6400, 256, '*', '*', None, '*')),
    ('cvb_train_repvgg_fwd', ('*', '*', None, 6553600, 32, '*', '*', None, '*')),
    ('cvb_train_sppf_chain_bwd', ('*', '*', 16, 20, 20, 128, '*', '*')),
    ('cvb_train_sppf_chain_bwd', ('*', '*', 64, 20, 20, 256, '*', '*')),
    ('cvb_train_sppf_chain_fwd', ('*', 16, 20, 20, 128, '*', '*')),
    ('cvb_train_sppf_chain_fwd', ('*', 64, 20, 20, 256, '*', '*')),
    ('cvb_train_yolov6_loss_bwd', ('*', '*', '*', '*', '*', '*', '*', '*')),
    ('cvb_train_yolov6_loss_fwd', ('*', '*', '*', '*', 141, '*', '*', '*', '*', '*', '*', '*', '*', 3251968)),
    ('cvb_train_yolov6_loss_fwd', ('*', '*', '*', '*', 741, '*', '*', '*', '*', '*', '*', '*', '*', 13013504)),
]


def _step(stype):
    """One YOLOv6 training step (forward, loss, backward) at STEPS[stype] x 3 x 640², tools/bench_yolov5_train.py's targets."""
    from cvpytorch_b200 import yolov6_models as M
    gen = torch.Generator().manual_seed(2024)
    m = M.YOLOv6(DICT, use_model(stype)).cuda().train()
    B = STEPS[stype]
    x = torch.rand(B, 3, SIZE, SIZE, generator=gen).cuda()
    gts = TL._yolov5_targets(B, gen).cuda()
    m(x, gts, 'train')['loss'].backward()
    torch.cuda.synchronize()


def test_launch_table_matches_the_steps(recorder):  # noqa: F811
    for stype in STEPS:
        _step(stype)
        torch.cuda.empty_cache()
    got, want = recorder.seen, set(LAUNCHES)
    assert len(want) == len(LAUNCHES), 'LAUNCHES lists a signature twice'
    assert got == want, (f'launches of the two steps differ from LAUNCHES: new {TL._table(got - want)}\nno longer launched {TL._table(want - got)}\n'
                         f'recorded table:\n{TL._table(got)}')


# ------------------------------------------------------------------------------------------------ the YOLOv6 passes
def _stats(y, npix, C, g):
    """The kernel's batch statistics of y (cvb_train_bn_stats, checked on its own signature) and fp32 gamma."""
    gamma, beta = torch.rand(C, generator=g, device='cuda') + 0.5, torch.randn(C, generator=g, device='cuda') * 0.5
    return TL._bn_stats(y, npix, C, gamma, beta, torch.zeros(C, device='cuda'), torch.ones(C, device='cuda'), 1e-3, 0.03), gamma


def _z32(y, stat):
    """fp32 fmaf(y, scale, shift): the exact float64 product-sum, rounded once to fp32."""
    return (y.double() * stat[2].double() + stat[3].double()).float()


def _bn_relu_fwd(name, a, exact):
    _, npix, C, _, _ = a
    g = TL._gen((name, a, exact))
    y = TL._bn_inputs(npix, C, exact, g)[0]
    stat, _ = _stats(y, npix, C, g)
    out = TL._nan((npix, C), torch.bfloat16)
    TL._call(name, TL._p(y), npix, C, TL._p(stat), TL._p(out))
    TL._assert_equal(out, torch.relu(_z32(y, stat)).to(torch.bfloat16).double(), name)


def _bn_relu_bwd(name, a, exact):
    _, _, npix, C, _, _, _, _ = a
    g = TL._gen((name, a, exact))
    y = TL._bn_inputs(npix, C, exact, g)[0]
    stat, gamma = _stats(y, npix, C, g)
    da = TL._operand((npix, C), exact, g)
    sums, dy = TL._nan((2, C), torch.float32), TL._nan((npix, C), torch.bfloat16)
    TL._call(name, TL._p(da), TL._p(y), npix, C, TL._p(stat), TL._p(gamma), TL._p(sums), TL._p(dy))
    dz = (da.float() * (_z32(y, stat) > 0)).to(torch.bfloat16)  # (exact: a bf16 value times 0 or 1)
    gs = TL._bn_gs(npix, C, False)
    R.bn_silu_bwd_check(dz, 1, y, gamma, stat, sums, dy, gs, gs_sum=0.0 if exact else None)


def _repvgg_inputs(name, a, exact, ident, npix, C):
    g = TL._gen((name, a, exact))
    ys = [TL._bn_inputs(npix, C, exact, g)[0] for _ in range(3 if ident else 2)]
    st = [_stats(y, npix, C, g) for y in ys]
    return g, ys, st


def _repvgg_ref(ys, st):
    z = _z32(ys[0], st[0][0]) + _z32(ys[1], st[1][0])
    if len(ys) == 3:
        z = z + _z32(ys[2], st[2][0])
    return torch.relu(z).to(torch.bfloat16)


def _repvgg_fwd(name, a, exact):
    _, _, x, npix, C, _, _, _, _ = a
    _, ys, st = _repvgg_inputs(name, a, exact, x is not None, npix, C)
    out = TL._nan((npix, C), torch.bfloat16)
    xid = TL._p(ys[2]) if x is not None else None
    TL._call(name, TL._p(ys[0]), TL._p(ys[1]), xid, npix, C, TL._p(st[0][0]), TL._p(st[1][0]), TL._p(st[2][0]) if x is not None else None, TL._p(out))
    TL._assert_equal(out, _repvgg_ref(ys, st).double(), name)


def _repvgg_bwd(name, a, exact):
    x, npix, C = a[4], a[5], a[6]
    ident = x is not None
    g, ys, st = _repvgg_inputs(name, a, exact, ident, npix, C)
    act = _repvgg_ref(ys, st)  # (the forward's output: bitwise what cvb_train_repvgg_fwd writes)
    gr = TL._operand((npix, C), exact, g)
    sums = TL._nan((4, C), torch.float32)
    d = [TL._nan((npix, C), torch.bfloat16) for _ in range(3)]
    opt = lambda t: TL._p(t) if ident else None  # noqa: E731
    TL._call(name, TL._p(gr), TL._p(act), TL._p(ys[0]), TL._p(ys[1]), opt(ys[-1]), npix, C, TL._p(st[0][0]), TL._p(st[1][0]), opt(st[-1][0]),
             TL._p(st[0][1]), TL._p(st[1][1]), opt(st[-1][1]), TL._p(sums), TL._p(d[0]), TL._p(d[1]), opt(d[2]))
    dz = (gr.float() * (act.float() > 0)).to(torch.bfloat16)
    gs = TL._bn_gs(npix, C, False)
    for b in range(len(ys)):
        R.bn_silu_bwd_check(dz, 1, ys[b], st[b][1], st[b][0], torch.stack([sums[0], sums[1 + b]]), d[b], gs, gs_sum=0.0 if exact else None)
    if not ident:
        TL._assert_equal(sums[3], torch.zeros(C, dtype=torch.float64, device='cuda'), name + ' (no identity branch: dgamma_id row 0)')


def _convt_scatter(name, a, exact):
    _, B, h, w, C, _, _ = a
    g = TL._gen((name, a))
    u = TL._operand((B, h, w, 4 * C), False, g)
    bias = torch.randn(C, generator=g, device='cuda')
    out = TL._nan((B, 2 * h, 2 * w, C), torch.bfloat16)
    TL._call(name, TL._p(u), B, h, w, C, TL._p(bias), TL._p(out))
    ref = u.view(B, h, w, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B, 2 * h, 2 * w, C).float() + bias
    TL._assert_equal(out, ref.to(torch.bfloat16).double(), name)


def _convt_gather(name, a, exact):
    _, B, h, w, C, _, _, _ = a
    g = TL._gen((name, a, exact))
    gr = TL._operand((B, 2 * h, 2 * w, C), exact, g)
    du, db = TL._nan((B, h, w, 4 * C), torch.bfloat16), TL._nan((C,), torch.float32)
    TL._call(name, TL._p(gr), B, h, w, C, TL._p(TL._nan((256, C), torch.float32)), TL._p(du), TL._p(db))
    TL._assert_equal(du, gr.view(B, h, 2, w, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B, h, w, 4 * C).double(), name + ' du')
    ref = gr.double().sum((0, 1, 2))
    if exact:
        TL._assert_equal(db, ref, name + ' dbias')
    else:  # a lane's pixels in order, the lane tree, then the 256 partial sums in order
        npix, np_ = B * 4 * h * w, 256 // (C // 8)
        terms = -(-npix // (256 * np_)) + 9 + 256
        R.check(db, ref, terms * R.U24 * gr.double().abs().sum((0, 1, 2)), name + ' dbias')


_LOSSES_CHECKED = set()


def _yolov6_loss(name, a, exact):
    """The recorded GT count's step (its batch, 640², 80 classes, ATSS, GIoU) against the oracle: the test_yolov6_loss_gpu comparison."""
    import test_yolov6_loss_gpu as L6
    from oracle import yolov6_loss_oracle as LO
    if name.endswith('_bwd'):  # (the backward runs inside the forward's check)
        return
    nt = a[4]
    key = ('yolov6', nt)
    if key in _LOSSES_CHECKED:
        return
    B = 64 if nt > 16 * 20 else 16  # (the n step's 16 images hold at most 320 rows, the s step's 64 at least 128: about 700 on its seed)
    shapes, scores, distri, gt = L6._matrix_case(nt, B, SIZE, NC, 20, False)
    out, asg, grad = L6._run(shapes, scores, distri, gt, 'atss', 'giou', NC)
    d = distri.cuda().requires_grad_(True)
    o_out, o = LO.losses(shapes, scores.cuda(), d, gt.cuda(), 'atss', 'giou', NC)
    (o_out['iou'] + o_out['dfl'] + o_out['class']).backward()
    fg = o['fg']
    assert torch.equal(asg['fg'].bool(), fg) and torch.equal(asg['labels'].long(), o['labels'])
    ref = float(o_out['iou'].detach())
    assert abs(float(out[0]) - ref) <= 1e-6 * max(abs(ref), 1e-30)
    assert L6._gmax_err(grad, d.grad) <= 1e-5
    _LOSSES_CHECKED.add(key)


CHECKS = dict(TL.CHECKS, cvb_train_bn_relu_fwd=_bn_relu_fwd, cvb_train_bn_relu_bwd=_bn_relu_bwd, cvb_train_repvgg_fwd=_repvgg_fwd,
              cvb_train_repvgg_bwd=_repvgg_bwd, cvb_train_convt_scatter=_convt_scatter, cvb_train_convt_gather=_convt_gather,
              cvb_train_yolov6_loss_fwd=_yolov6_loss, cvb_train_yolov6_loss_bwd=_yolov6_loss)
ONE_KIND = TL.ONE_KIND + ('cvb_train_convt_scatter', 'cvb_train_yolov6_loss_fwd', 'cvb_train_yolov6_loss_bwd')


def _run(sig):
    name, args = sig
    for exact in (True,) if name in ONE_KIND else (True, False):
        CHECKS[name](name, args, exact)
        torch.cuda.synchronize()
    torch.cuda.empty_cache()


# small shapes of the new checks: the exactness they rely on, confirmed where a failure is cheap to read
SMALL = [('cvb_train_bn_relu_fwd', ('*', 1000, 64, '*', '*')),
         ('cvb_train_bn_relu_bwd', ('*', '*', 1000, 64, '*', '*', '*', '*')),
         ('cvb_train_repvgg_fwd', ('*', '*', '*', 1000, 32, '*', '*', '*', '*')),
         ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', '*', 1000, 32, '*', '*', '*', '*', '*', '*', '*', '*', '*', '*')),
         ('cvb_train_repvgg_bwd', ('*', '*', '*', '*', None, 1000, 192, '*', '*', None, '*', '*', None, '*', '*', '*', None)),
         ('cvb_train_convt_scatter', ('*', 2, 5, 7, 32, '*', '*')),
         ('cvb_train_convt_gather', ('*', 2, 5, 7, 192, '*', '*', '*'))]


@pytest.mark.parametrize('sig', SMALL, ids=[TL._id(s) for s in SMALL])
def test_small_shape_of_each_check(cuda, sig):
    _run(sig)


@pytest.mark.parametrize('sig', LAUNCHES, ids=[TL._id(s) for s in LAUNCHES])
def test_launch_at_its_real_shape(cuda, sig):
    _run(sig)
