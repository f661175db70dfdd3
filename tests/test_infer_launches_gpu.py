"""Every inference-kernel launch of the five benchmarked graphs, at its real shape: YOLOv5-s at 64 x 3 x 640² (fp32 input and the uint8-frame
stem, bench.py), YOLOX-s at 64 x 3 x 640², FCOS R50 at 32 x 3 x 800², DeepLabv3+ R50-D8 at 16 x 3 x 1024 x 2048 (bench.py --config) and
YOLOv6-s at 64 x 3 x 640² (tools/bench_yolov6.py).

LAUNCHES is the set of distinct signatures of those graphs' conv plans (cvb_conv_plan_create) and aux launches.  A view is resolved
against its graph's buffers into (format, buffer B, H, W, channel pitch, channel offset, channels, alias): alias is the index of an
earlier view of the same launch in the same buffer (-1: its own buffer), so in-place residuals and concat slices are rebuilt as the graph
has them.  A conv signature is every field that can change the plan: k, stride, pad, dilation, activation, output kind (with the fused
YOLO decode's na / no / anchors / stride / z_rows / z_off), block_n, w_window, residual placement and scale, and its four views.  The
NMS kernels, cvb_nms_workspace_reset and cvb_rescale_clip_boxes are left out: tests/test_nms_kernels_gpu.py checks them at their
capacity boundaries.  test_launch_table_matches_the_graphs records the five graphs through a proxy of _lib.lib() and requires the
recorded set to equal LAUNCHES, so a model change that adds a launch fails until its shape is listed here, and so checked.

Each conv signature then runs stand-alone through ops.ConvPlan into NaN-filled buffers (channels outside the output view must keep
their contents), twice:
(a) grid operands, the whole batch.  Activation hi in {-1, 0, 1}, lo = +-2^-12 on even channels; weight hi in {-1, 0, 1}, lo = +-2^-12 on
    odd input channels (so pack_conv_weights gives nonzero lo words and no lo * lo product, which the kernel drops, is ever nonzero);
    bias, residual and up-sampled partial on the same 2^-12 grid.  The test asserts that every |partial sum| (the float64 conv of the
    absolute operands plus the epilogue terms) stays below 2^24 grid units, with sparse operands on deep-K layers: then every fp32
    accumulation is exact in any order.  What is left is the kernel's round-toward-zero compensation: the hi * hi accumulator is multiplied
    by rz_gain = 1 + 1.9e-8 * chain (conv_tc.cu), which moves a result by at most (rz_gain - 1) |hi * hi sum|, bounded here with the
    longest chain any plan of the layer can have (block_n 256: three products per K step).  The bound is that term plus the epilogue's
    2^-19 relative (fp64ref.split_conv_reference); it has no accumulation term, so a lost, doubled or misplaced 128-pixel tile, or a lo
    plane read from the wrong address, in any image of the batch fails it (test_exact_check_sees_a_lost_tile_and_a_misread_lo_plane).
(b) Gaussian operands: fp64ref.split_conv_reference's element-wise bound and the single-layer budget on images 0 and B - 1, where
    end-of-batch addressing overflows if it does.
The fused YOLO head's z rows go through test_conv_plans_gpu.decode_reference with the pre-activation bound; rows outside the level stay NaN.

Each aux signature runs at its recorded shape and views against the references of test_aux_kernels_gpu.py: bit for bit for the layouts,
the stem space-to-depth (both variants), the max pools and depth-to-space, the element-wise bounds there for GroupNorm, the depthwise
conv, the average pool and the resizes, and the decode checks of the level shapes at B = 64 / 32.  test_depth_to_space2 covers the
kernel YOLOv6's BiFusion uses at its edges and refusals.

The float64 references run on the GPU in chunks of images, so every grid check runs at its full batch: on one H100 80GB (SXM; power
limit not recorded) the whole file took 50 s (pytest's count) with a peak of 54 GiB of device memory, reached while the DeepLab graph
is recorded; the stand-alone checks stay below 15 GiB."""
import ctypes
import os
import sys
import zlib

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fp64ref as R  # noqa: E402

pytestmark = pytest.mark.gpu
NAN = float('nan')
GRID = 2.0 ** -12      # the grid of check (a)'s operands
RZ_C = 1.9e-8          # conv_tc.cu: rz_gain = 1 + RZ_C * chain
CHUNK_ELEMS = 2 ** 27  # float64 elements of one reference chunk (1 GiB)

AUX = ('cvb_stem_s2d', 'cvb_stem_s2d_u8', 'cvb_maxpool3x3s2', 'cvb_sppf_pool', 'cvb_split_to_f32nhwc', 'cvb_groupnorm_relu', 'cvb_dwconv3x3',
       'cvb_global_avgpool', 'cvb_bilinear_resize', 'cvb_upsample_argmax', 'cvb_depth_to_space2', 'cvb_yolo_decode', 'cvb_yolox_decode',
       'cvb_fcos_decode', 'cvb_yolov6_decode')

# (entry point, fields, resolved views[, fused decode]): recorded from the five graphs (test_launch_table_matches_the_graphs prints the table)
LAUNCHES = [
    ('cvb_bilinear_resize', (('view', 0), ('view', 1)), (('split', 16, 1, 1, 512, 0, 512, -1), ('split', 16, 32, 64, 2560, 0, 512, -1))),
    ('cvb_bilinear_resize', (('view', 0), ('view', 1)), (('split', 16, 32, 64, 512, 0, 512, -1), ('split', 16, 256, 512, 576, 0, 512, -1))),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 16, 256, 512, 64, 0, 64, -1), ('split', 16, 256, 512, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 100, 100, 512, 0, 512, -1), ('split', 32, 100, 100, 256, 0, 256, -1), None, ('f32', 32, 50, 50, 256, 0, 256, -1)), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 200, 200, 64, 0, 64, -1), ('split', 32, 200, 200, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 25, 25, 2048, 0, 2048, -1), ('split', 32, 25, 25, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 50, 50, 1024, 0, 1024, -1), ('split', 32, 50, 50, 256, 0, 256, -1), None, ('f32', 32, 25, 25, 256, 0, 256, -1)), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 40, 40, 128, 64, 64, -1), ('split', 64, 40, 40, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 64, 20, 20, 256, 128, 128, -1), ('split', 64, 20, 20, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 40, 40, 256, 128, 128, -1), ('f32', 64, 40, 40, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 24), (('split', 16, 256, 512, 512, 0, 512, -1), ('f32', 16, 256, 512, 32, 0, 19, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 20, 20, 512, 256, 256, -1), ('f32', 64, 20, 20, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 8), (('split', 64, 20, 20, 512, 256, 256, -1), ('f32', 64, 20, 20, 32, 0, 4, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 8), (('split', 64, 22, 22, 128, 0, 128, -1), ('f32', 64, 22, 22, 32, 0, 5, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 8), (('split', 64, 40, 40, 256, 128, 128, -1), ('f32', 64, 40, 40, 32, 0, 4, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 8), (('split', 64, 42, 42, 128, 0, 128, -1), ('f32', 64, 42, 42, 32, 0, 5, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 8), (('split', 64, 80, 80, 128, 64, 64, -1), ('f32', 64, 80, 80, 32, 0, 4, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 8), (('split', 64, 82, 82, 128, 0, 128, -1), ('f32', 64, 82, 82, 32, 0, 5, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 80), (('split', 64, 20, 20, 512, 0, 256, -1), ('f32', 64, 20, 20, 96, 0, 80, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 80), (('split', 64, 22, 22, 128, 0, 128, -1), ('f32', 64, 22, 22, 96, 0, 80, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 80), (('split', 64, 40, 40, 256, 0, 128, -1), ('f32', 64, 40, 40, 96, 0, 80, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 80), (('split', 64, 42, 42, 128, 0, 128, -1), ('f32', 64, 42, 42, 96, 0, 80, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 80), (('split', 64, 80, 80, 128, 0, 64, -1), ('f32', 64, 80, 80, 96, 0, 80, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 80), (('split', 64, 82, 82, 128, 0, 128, -1), ('f32', 64, 82, 82, 96, 0, 80, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 2, 0, 0, 0, 1.0, 0, 0, 0, 0, 384), (('split', 64, 20, 20, 512, 0, 512, -1), ('z', 64, 20, 20, 384, 0, 384, -1), None, None), (3, 85, (116.0, 90.0, 156.0, 198.0, 373.0, 326.0), 32.0, 25200, 24000, True, 0.001, 1)),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 2, 0, 0, 0, 1.0, 0, 0, 0, 0, 384), (('split', 64, 40, 40, 256, 0, 256, -1), ('z', 64, 40, 40, 384, 0, 384, -1), None, None), (3, 85, (30.0, 61.0, 62.0, 45.0, 59.0, 119.0), 16.0, 25200, 19200, True, 0.001, 1)),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 0, 2, 0, 0, 0, 1.0, 0, 0, 0, 0, 384), (('split', 64, 80, 80, 128, 0, 128, -1), ('z', 64, 80, 80, 384, 0, 384, -1), None, None), (3, 85, (10.0, 13.0, 16.0, 30.0, 33.0, 23.0), 8.0, 25200, 0, True, 0.001, 1)),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 40, 40, 128, 0, 128, -1), ('split', 64, 40, 40, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 40, 40, 256, 0, 128, -1), ('split', 64, 40, 40, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 40, 40, 256, 0, 256, -1), ('split', 64, 40, 40, 256, 128, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 80, 80, 128, 0, 128, -1), ('split', 64, 80, 80, 128, 0, 128, -1), None, ('f32', 64, 40, 40, 128, 0, 128, -1)), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 80, 80, 128, 0, 128, -1), ('split', 64, 80, 80, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 20, 20, 256, 0, 256, -1), ('split', 64, 20, 20, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 20, 20, 512, 0, 256, -1), ('split', 64, 20, 20, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 20, 20, 512, 0, 512, -1), ('split', 64, 20, 20, 1024, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 20, 20, 512, 0, 512, -1), ('split', 64, 20, 20, 512, 256, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 40, 40, 256, 0, 256, -1), ('split', 64, 40, 40, 256, 0, 256, -1), None, ('f32', 64, 20, 20, 256, 0, 256, -1)), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 40, 40, 256, 0, 256, -1), ('split', 64, 40, 40, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 32), (('split', 64, 160, 160, 64, 0, 32, -1), ('split', 64, 160, 160, 32, 0, 32, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 64, 20, 20, 1024, 0, 1024, -1), ('split', 64, 20, 20, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 64, 20, 20, 512, 0, 512, -1), ('split', 64, 20, 20, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 160, 160, 64, 0, 64, -1), ('split', 64, 160, 160, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 80, 80, 128, 0, 64, -1), ('split', 64, 80, 80, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 80, 80, 64, 0, 64, -1), ('split', 64, 80, 80, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 16, 128, 256, 512, 0, 512, -1), ('split', 16, 128, 256, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 16, 256, 512, 256, 0, 256, -1), ('split', 16, 256, 512, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 32, 100, 100, 512, 0, 512, -1), ('split', 32, 100, 100, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 32, 200, 200, 256, 0, 256, -1), ('split', 32, 200, 200, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 20, 20, 512, 0, 512, -1), ('split', 64, 20, 20, 256, 128, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 40, 40, 256, 0, 256, -1), ('split', 64, 40, 40, 384, 128, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 40, 40, 384, 0, 384, -1), ('split', 64, 40, 40, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 80, 80, 128, 0, 128, -1), ('split', 64, 80, 80, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 16, 128, 256, 512, 0, 512, -1), ('split', 16, 128, 256, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 16, 64, 128, 1024, 0, 1024, -1), ('split', 16, 64, 128, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 100, 100, 512, 0, 512, -1), ('split', 32, 100, 100, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 50, 50, 1024, 0, 1024, -1), ('split', 32, 50, 50, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 20, 20, 1024, 0, 1024, -1), ('split', 64, 20, 20, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 20, 20, 256, 0, 256, -1), ('split', 64, 20, 20, 1024, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 48), (('split', 16, 256, 512, 256, 0, 256, -1), ('split', 16, 256, 512, 576, 512, 48, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 16, 1, 1, 2048, 0, 2048, -1), ('split', 16, 1, 1, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 16, 256, 512, 512, 0, 512, -1), ('split', 16, 256, 512, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 16, 256, 512, 576, 0, 576, -1), ('split', 16, 256, 512, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 16, 32, 64, 2048, 0, 2048, -1), ('split', 16, 32, 64, 2560, 1024, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 16, 32, 64, 2048, 0, 2048, -1), ('split', 16, 32, 64, 2560, 1536, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 16, 32, 64, 2048, 0, 2048, -1), ('split', 16, 32, 64, 2560, 2048, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 16, 32, 64, 2048, 0, 2048, -1), ('split', 16, 32, 64, 2560, 512, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 16, 32, 64, 2048, 0, 2048, -1), ('split', 16, 32, 64, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 16, 64, 128, 1024, 0, 1024, -1), ('split', 16, 64, 128, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 32, 25, 25, 2048, 0, 2048, -1), ('split', 32, 25, 25, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 32, 50, 50, 1024, 0, 1024, -1), ('split', 32, 50, 50, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 64, 20, 20, 512, 0, 512, -1), ('split', 64, 20, 20, 768, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 64, 20, 20, 768, 256, 512, -1), ('split', 64, 20, 20, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 16, 256, 512, 256, 0, 256, -1), ('split', 16, 256, 512, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 16, 256, 512, 64, 0, 64, -1), ('split', 16, 256, 512, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 32, 200, 200, 256, 0, 256, -1), ('split', 32, 200, 200, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 32, 200, 200, 64, 0, 64, -1), ('split', 32, 200, 200, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 160, 160, 64, 0, 64, -1), ('split', 64, 160, 160, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 40, 40, 128, 0, 128, -1), ('split', 64, 40, 40, 128, 64, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 80, 80, 128, 0, 128, -1), ('split', 64, 80, 80, 192, 64, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 80, 80, 192, 0, 192, -1), ('split', 64, 80, 80, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 1, 1.0, 0, 0, 0, 0, 1024), (('split', 16, 64, 128, 256, 0, 256, -1), ('split', 16, 64, 128, 1024, 0, 1024, -1), ('split', 16, 64, 128, 1024, 0, 1024, -1), None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 1, 1.0, 0, 0, 0, 0, 1024), (('split', 32, 50, 50, 256, 0, 256, -1), ('split', 32, 50, 50, 1024, 0, 1024, -1), ('split', 32, 50, 50, 1024, 0, 1024, -1), None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 1, 1.0, 0, 0, 0, 0, 2048), (('split', 16, 32, 64, 512, 0, 512, -1), ('split', 16, 32, 64, 2048, 0, 2048, -1), ('split', 16, 32, 64, 2048, 0, 2048, -1), None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 1, 1.0, 0, 0, 0, 0, 2048), (('split', 32, 25, 25, 512, 0, 512, -1), ('split', 32, 25, 25, 2048, 0, 2048, -1), ('split', 32, 25, 25, 2048, 0, 2048, -1), None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 1, 1.0, 0, 0, 0, 0, 256), (('split', 16, 256, 512, 64, 0, 64, -1), ('split', 16, 256, 512, 256, 0, 256, -1), ('split', 16, 256, 512, 256, 0, 256, -1), None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 1, 1.0, 0, 0, 0, 0, 256), (('split', 32, 200, 200, 64, 0, 64, -1), ('split', 32, 200, 200, 256, 0, 256, -1), ('split', 32, 200, 200, 256, 0, 256, -1), None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 1, 1.0, 0, 0, 0, 0, 512), (('split', 16, 128, 256, 128, 0, 128, -1), ('split', 16, 128, 256, 512, 0, 512, -1), ('split', 16, 128, 256, 512, 0, 512, -1), None), None),
    ('cvb_conv_plan_create', (1, 1, 0, 1, 2, 0, 0, 0, 1, 1.0, 0, 0, 0, 0, 512), (('split', 32, 100, 100, 128, 0, 128, -1), ('split', 32, 100, 100, 512, 0, 512, -1), ('split', 32, 100, 100, 512, 0, 512, -1), None), None),
    ('cvb_conv_plan_create', (1, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 20, 20, 512, 0, 512, -1), ('split', 64, 22, 22, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 40, 40, 256, 0, 256, -1), ('split', 64, 42, 42, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 80, 80, 128, 0, 128, -1), ('split', 64, 82, 82, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 2, 0, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 1024), (('split', 16, 128, 256, 512, 0, 512, -1), ('split', 16, 64, 128, 1024, 0, 1024, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 2, 0, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 1024), (('split', 32, 100, 100, 512, 0, 512, -1), ('split', 32, 50, 50, 1024, 0, 1024, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 2, 0, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 2048), (('split', 16, 64, 128, 1024, 0, 1024, -1), ('split', 16, 32, 64, 2048, 0, 2048, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 2, 0, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 2048), (('split', 32, 50, 50, 1024, 0, 1024, -1), ('split', 32, 25, 25, 2048, 0, 2048, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 2, 0, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 16, 256, 512, 256, 0, 256, -1), ('split', 16, 128, 256, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (1, 2, 0, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 32, 200, 200, 256, 0, 256, -1), ('split', 32, 100, 100, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (2, 1, 1, 1, 2, 0, 0, 4, 0, 1.0, 0, 0, 0, 0, 32), (('split', 16, 512, 1027, 16, 0, 16, -1), ('split', 16, 512, 1024, 32, 0, 32, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 100, 100, 256, 0, 256, -1), ('split', 32, 100, 100, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 13, 13, 256, 0, 256, -1), ('split', 32, 13, 13, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 25, 25, 256, 0, 256, -1), ('split', 32, 25, 25, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 50, 50, 256, 0, 256, -1), ('split', 32, 50, 50, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 7, 7, 256, 0, 256, -1), ('split', 32, 7, 7, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 8), (('split', 32, 100, 100, 256, 0, 256, -1), ('f32', 32, 100, 100, 32, 0, 5, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 8), (('split', 32, 13, 13, 256, 0, 256, -1), ('f32', 32, 13, 13, 32, 0, 5, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 8), (('split', 32, 25, 25, 256, 0, 256, -1), ('f32', 32, 25, 25, 32, 0, 5, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 8), (('split', 32, 50, 50, 256, 0, 256, -1), ('f32', 32, 50, 50, 32, 0, 5, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 8), (('split', 32, 7, 7, 256, 0, 256, -1), ('f32', 32, 7, 7, 32, 0, 5, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 80), (('split', 32, 100, 100, 256, 0, 256, -1), ('f32', 32, 100, 100, 96, 0, 80, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 80), (('split', 32, 13, 13, 256, 0, 256, -1), ('f32', 32, 13, 13, 96, 0, 80, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 80), (('split', 32, 25, 25, 256, 0, 256, -1), ('f32', 32, 25, 25, 96, 0, 80, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 80), (('split', 32, 50, 50, 256, 0, 256, -1), ('f32', 32, 50, 50, 96, 0, 80, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 0, 1, 0, 0, 0, 1.0, 0, 0, 0, 0, 80), (('split', 32, 7, 7, 256, 0, 256, -1), ('f32', 32, 7, 7, 96, 0, 80, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 22, 22, 256, 0, 128, -1), ('split', 64, 22, 22, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 22, 22, 256, 128, 128, -1), ('split', 64, 22, 22, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 40, 40, 128, 0, 128, -1), ('split', 64, 40, 40, 256, 0, 128, -1), ('split', 64, 40, 40, 256, 0, 128, 1), None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 40, 40, 128, 0, 128, -1), ('split', 64, 40, 40, 256, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 42, 42, 256, 0, 128, -1), ('split', 64, 42, 42, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 42, 42, 256, 128, 128, -1), ('split', 64, 42, 42, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 80, 80, 64, 0, 64, -1), ('split', 64, 80, 80, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 82, 82, 256, 0, 128, -1), ('split', 64, 82, 82, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 82, 82, 256, 128, 128, -1), ('split', 64, 82, 82, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 20, 20, 256, 0, 256, -1), ('split', 64, 20, 20, 512, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 22, 22, 128, 0, 128, -1), ('split', 64, 22, 22, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 40, 40, 128, 0, 128, -1), ('split', 64, 40, 40, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 42, 42, 128, 0, 128, -1), ('split', 64, 42, 42, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 82, 82, 128, 0, 128, -1), ('split', 64, 82, 82, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 32), (('split', 64, 160, 160, 32, 0, 32, -1), ('split', 64, 160, 160, 64, 0, 32, -1), ('split', 64, 160, 160, 64, 0, 32, 1), None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 64, 20, 20, 256, 0, 256, -1), ('split', 64, 20, 20, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 80, 80, 64, 0, 64, -1), ('split', 64, 80, 80, 128, 0, 64, -1), ('split', 64, 80, 80, 128, 0, 64, 1), None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 80, 80, 64, 0, 64, -1), ('split', 64, 80, 80, 128, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 1, 0, 0, 4, 0, 1.0, 0, 0, 0, 0, 32), (('split', 64, 320, 323, 16, 0, 16, -1), ('split', 64, 320, 320, 32, 0, 32, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 16, 128, 256, 128, 0, 128, -1), ('split', 16, 128, 256, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 32, 100, 100, 128, 0, 128, -1), ('split', 32, 100, 100, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 40, 40, 128, 0, 128, -1), ('split', 64, 40, 40, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 80, 80, 128, 0, 128, -1), ('split', 64, 80, 80, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 16, 64, 128, 256, 0, 256, -1), ('split', 16, 64, 128, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 50, 50, 256, 0, 256, -1), ('split', 32, 50, 50, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 20, 20, 256, 0, 256, -1), ('split', 64, 20, 20, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 20, 20, 256, 0, 256, -1), ('split', 64, 20, 20, 768, 512, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 20, 20, 768, 0, 256, -1), ('split', 64, 20, 20, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 40, 40, 256, 0, 256, -1), ('split', 64, 40, 40, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 32), (('split', 16, 512, 1024, 32, 0, 32, -1), ('split', 16, 512, 1024, 32, 0, 32, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 16, 32, 64, 2560, 0, 2560, -1), ('split', 16, 32, 64, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 16, 32, 64, 512, 0, 512, -1), ('split', 16, 32, 64, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 32, 25, 25, 512, 0, 512, -1), ('split', 32, 25, 25, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 64, 20, 20, 512, 0, 512, -1), ('split', 64, 20, 20, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 16, 256, 512, 64, 0, 64, -1), ('split', 16, 256, 512, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 16, 512, 1024, 32, 0, 32, -1), ('split', 16, 512, 1024, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 32, 200, 200, 64, 0, 64, -1), ('split', 32, 200, 200, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 160, 160, 64, 0, 64, -1), ('split', 64, 160, 160, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 80, 80, 64, 0, 64, -1), ('split', 64, 80, 80, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 1, 1, 1, 2, 0, 0, 4, 0, 1.0, 0, 0, 0, 0, 32), (('split', 64, 320, 323, 16, 0, 16, -1), ('split', 64, 320, 320, 32, 0, 32, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 13, 13, 256, 0, 256, -1), ('split', 32, 7, 7, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 25, 25, 256, 0, 256, -1), ('split', 32, 13, 13, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 160, 160, 64, 0, 64, -1), ('split', 64, 80, 80, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 80, 80, 128, 0, 128, -1), ('split', 64, 40, 40, 256, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 40, 40, 256, 0, 256, -1), ('split', 64, 20, 20, 512, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 80, 80, 128, 0, 128, -1), ('split', 64, 40, 40, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 64, 40, 40, 256, 0, 256, -1), ('split', 64, 20, 20, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 1, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 320, 320, 32, 0, 32, -1), ('split', 64, 160, 160, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 16, 256, 512, 128, 0, 128, -1), ('split', 16, 128, 256, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 32, 200, 200, 128, 0, 128, -1), ('split', 32, 100, 100, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 160, 160, 64, 0, 64, -1), ('split', 64, 80, 80, 128, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 40, 40, 128, 0, 128, -1), ('split', 64, 20, 20, 256, 0, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 128), (('split', 64, 80, 80, 128, 0, 128, -1), ('split', 64, 40, 40, 384, 256, 128, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 16, 128, 256, 256, 0, 256, -1), ('split', 16, 64, 128, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 100, 100, 256, 0, 256, -1), ('split', 32, 50, 50, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 32, 25, 25, 256, 0, 256, -1), ('split', 32, 13, 13, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 256), (('split', 64, 80, 80, 128, 0, 128, -1), ('split', 64, 40, 40, 256, 0, 256, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 16, 64, 128, 512, 0, 512, -1), ('split', 16, 32, 64, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 32, 50, 50, 512, 0, 512, -1), ('split', 32, 25, 25, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 512), (('split', 64, 40, 40, 256, 0, 256, -1), ('split', 64, 20, 20, 512, 0, 512, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 160, 160, 64, 0, 64, -1), ('split', 64, 80, 80, 192, 128, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 320, 320, 32, 0, 32, -1), ('split', 64, 160, 160, 64, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (3, 2, 1, 1, 2, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 64), (('split', 64, 80, 80, 64, 0, 64, -1), ('split', 64, 40, 40, 128, 0, 64, -1), None, None), None),
    ('cvb_conv_plan_create', (4, 1, 2, 1, 2, 0, 0, 4, 0, 1.0, 0, 0, 0, 0, 64), (('split', 32, 400, 403, 16, 0, 16, -1), ('split', 32, 400, 400, 64, 0, 64, -1), None, None), None),
    ('cvb_depth_to_space2', (('view', 0), ('view', 1)), (('split', 64, 20, 20, 512, 0, 512, -1), ('split', 64, 40, 40, 384, 0, 128, -1))),
    ('cvb_depth_to_space2', (('view', 0), ('view', 1)), (('split', 64, 40, 40, 256, 0, 256, -1), ('split', 64, 80, 80, 192, 0, 64, -1))),
    ('cvb_dwconv3x3', (('view', 0), '*', '*', 1, 1, ('view', 1)), (('split', 16, 256, 512, 512, 0, 512, -1), ('split', 16, 256, 512, 512, 0, 512, -1))),
    ('cvb_dwconv3x3', (('view', 0), '*', '*', 1, 1, ('view', 1)), (('split', 16, 256, 512, 576, 0, 576, -1), ('split', 16, 256, 512, 576, 0, 576, -1))),
    ('cvb_dwconv3x3', (('view', 0), '*', '*', 12, 1, ('view', 1)), (('split', 16, 32, 64, 2048, 0, 2048, -1), ('split', 16, 32, 64, 2048, 0, 2048, -1))),
    ('cvb_dwconv3x3', (('view', 0), '*', '*', 24, 1, ('view', 1)), (('split', 16, 32, 64, 2048, 0, 2048, -1), ('split', 16, 32, 64, 2048, 0, 2048, -1))),
    ('cvb_dwconv3x3', (('view', 0), '*', '*', 36, 1, ('view', 1)), (('split', 16, 32, 64, 2048, 0, 2048, -1), ('split', 16, 32, 64, 2048, 0, 2048, -1))),
    ('cvb_fcos_decode', (('view', 0), ('view', 1), 80, 128.0, 1.0, '*', '*', '*', 13343, 13294), (('f32', 32, 7, 7, 96, 0, 80, -1), ('f32', 32, 7, 7, 32, 0, 8, -1))),
    ('cvb_fcos_decode', (('view', 0), ('view', 1), 80, 16.0, 1.0, '*', '*', '*', 13343, 10000), (('f32', 32, 50, 50, 96, 0, 80, -1), ('f32', 32, 50, 50, 32, 0, 8, -1))),
    ('cvb_fcos_decode', (('view', 0), ('view', 1), 80, 32.0, 1.0, '*', '*', '*', 13343, 12500), (('f32', 32, 25, 25, 96, 0, 80, -1), ('f32', 32, 25, 25, 32, 0, 8, -1))),
    ('cvb_fcos_decode', (('view', 0), ('view', 1), 80, 64.0, 1.0, '*', '*', '*', 13343, 13125), (('f32', 32, 13, 13, 96, 0, 80, -1), ('f32', 32, 13, 13, 32, 0, 8, -1))),
    ('cvb_fcos_decode', (('view', 0), ('view', 1), 80, 8.0, 1.0, '*', '*', '*', 13343, 0), (('f32', 32, 100, 100, 96, 0, 80, -1), ('f32', 32, 100, 100, 32, 0, 8, -1))),
    ('cvb_global_avgpool', (('view', 0), ('view', 1)), (('split', 16, 32, 64, 2048, 0, 2048, -1), ('split', 16, 1, 1, 2048, 0, 2048, -1))),
    ('cvb_groupnorm_relu', (('view', 0), 32, '*', '*', 1e-05, 1, ('view', 1), '*', 16384), (('split', 32, 100, 100, 256, 0, 256, -1), ('split', 32, 100, 100, 256, 0, 256, -1))),
    ('cvb_groupnorm_relu', (('view', 0), 32, '*', '*', 1e-05, 1, ('view', 1), '*', 16384), (('split', 32, 13, 13, 256, 0, 256, -1), ('split', 32, 13, 13, 256, 0, 256, -1))),
    ('cvb_groupnorm_relu', (('view', 0), 32, '*', '*', 1e-05, 1, ('view', 1), '*', 16384), (('split', 32, 25, 25, 256, 0, 256, -1), ('split', 32, 25, 25, 256, 0, 256, -1))),
    ('cvb_groupnorm_relu', (('view', 0), 32, '*', '*', 1e-05, 1, ('view', 1), '*', 16384), (('split', 32, 50, 50, 256, 0, 256, -1), ('split', 32, 50, 50, 256, 0, 256, -1))),
    ('cvb_groupnorm_relu', (('view', 0), 32, '*', '*', 1e-05, 1, ('view', 1), '*', 16384), (('split', 32, 7, 7, 256, 0, 256, -1), ('split', 32, 7, 7, 256, 0, 256, -1))),
    ('cvb_maxpool3x3s2', (('view', 0), ('view', 1)), (('split', 16, 512, 1024, 64, 0, 64, -1), ('split', 16, 256, 512, 64, 0, 64, -1))),
    ('cvb_maxpool3x3s2', (('view', 0), ('view', 1)), (('split', 32, 400, 400, 64, 0, 64, -1), ('split', 32, 200, 200, 64, 0, 64, -1))),
    ('cvb_split_to_f32nhwc', (('view', 0), ('view', 1)), (('split', 32, 25, 25, 256, 0, 256, -1), ('f32', 32, 25, 25, 256, 0, 256, -1))),
    ('cvb_split_to_f32nhwc', (('view', 0), ('view', 1)), (('split', 32, 50, 50, 256, 0, 256, -1), ('f32', 32, 50, 50, 256, 0, 256, -1))),
    ('cvb_sppf_pool', (('view', 0), ('view', 1), ('view', 2), ('view', 3)), (('split', 64, 20, 20, 1024, 0, 256, -1), ('split', 64, 20, 20, 1024, 256, 256, 0), ('split', 64, 20, 20, 1024, 512, 256, 0), ('split', 64, 20, 20, 1024, 768, 256, 0))),
    ('cvb_stem_s2d', ('*', 16, 1024, 2048, ('view', 0), 1), (('split', 16, 512, 1027, 16, 0, 16, -1),)),
    ('cvb_stem_s2d', ('*', 32, 800, 800, ('view', 0), 2), (('split', 32, 400, 403, 16, 0, 16, -1),)),
    ('cvb_stem_s2d', ('*', 64, 640, 640, ('view', 0), 1), (('split', 64, 320, 323, 16, 0, 16, -1),)),
    ('cvb_stem_s2d_u8', ('*', 64, 640, 640, (0.406, 0.456, 0.485), (0.225, 0.224, 0.229), 1, ('view', 0), 1), (('split', 64, 320, 323, 16, 0, 16, -1),)),
    ('cvb_upsample_argmax', (('view', 0), 19, '*', 1024, 2048), (('f32', 16, 256, 512, 32, 0, 19, -1),)),
    ('cvb_yolov6_decode', (('view', 0), ('view', 1), 80, 16.0, '*', 8400, 6400, '*', 0.03, 1), (('f32', 64, 40, 40, 96, 0, 80, -1), ('f32', 64, 40, 40, 32, 0, 4, -1))),
    ('cvb_yolov6_decode', (('view', 0), ('view', 1), 80, 32.0, '*', 8400, 8000, '*', 0.03, 1), (('f32', 64, 20, 20, 96, 0, 80, -1), ('f32', 64, 20, 20, 32, 0, 4, -1))),
    ('cvb_yolov6_decode', (('view', 0), ('view', 1), 80, 8.0, '*', 8400, 0, '*', 0.03, 1), (('f32', 64, 80, 80, 96, 0, 80, -1), ('f32', 64, 80, 80, 32, 0, 4, -1))),
    ('cvb_yolox_decode', (('view', 0), ('view', 1), 80, 16.0, '*', 8972, 6724), (('f32', 64, 42, 42, 32, 0, 5, -1), ('f32', 64, 42, 42, 96, 0, 80, -1))),
    ('cvb_yolox_decode', (('view', 0), ('view', 1), 80, 32.0, '*', 8972, 8488), (('f32', 64, 22, 22, 32, 0, 5, -1), ('f32', 64, 22, 22, 96, 0, 80, -1))),
    ('cvb_yolox_decode', (('view', 0), ('view', 1), 80, 8.0, '*', 8972, 0), (('f32', 64, 82, 82, 32, 0, 5, -1), ('f32', 64, 82, 82, 96, 0, 80, -1))),
]


# ------------------------------------------------------------------------------------------------ recording the launches of a graph
def _view_raw(v):
    return None if not v.base else (int(v.base), v.B, v.H, v.W, v.C, v.c_pitch, int(v.plane_stride))


def _snapshot(name, args):
    """The launch's arguments with every view and the conv descriptor copied out (the caller's structs may be reused)."""
    from cvpytorch_b200 import _lib
    if name == 'cvb_conv_plan_create':
        d = args[0]._obj
        y = None
        if d.out_kind == _lib.CVB_OUT_YOLO:
            yy = d.yolo.contents
            y = (yy.na, yy.no, tuple(round(float(a), 4) for a in yy.anchors_px[:2 * yy.na]), float(yy.stride), int(yy.z_rows), int(yy.z_off),
                 bool(yy.nms_workspace), round(float(yy.conf_thres), 7), int(yy.multi_label))
        p = (d.kh, d.stride, d.pad, d.dilation, d.act, d.out_kind, d.block_n, d.w_window, d.residual_before_act, round(float(d.residual_scale), 7),
             d.no_resident, d.halo, d.schedule, d.sm_limit, d.cout_pad)
        return name, p, [_view_raw(d.inp), _view_raw(d.out), _view_raw(d.residual), _view_raw(d.up_partial)], y
    vals, views = [], []
    for t, v in zip(_lib.SYMBOLS[name][1][:-1], args[:-1]):
        if t is ctypes.POINTER(_lib.CvbView):
            vals.append(('view', len(views)))
            views.append(_view_raw(v._obj))
        elif t is ctypes.c_void_p:
            vals.append(None if v is None or getattr(v, 'value', v) is None else '*')
        elif t in (ctypes.c_int32, ctypes.c_int64, ctypes.c_size_t):
            vals.append(int(v))
        elif t is ctypes.c_float:
            vals.append(round(float(v), 7))
        else:
            vals.append(tuple(round(float(x), 7) for x in v))
    return name, tuple(vals), views, None


def _buffers(g):
    """(first byte, bytes, format, B, H, W, C) of every buffer the graph owns."""
    from cvpytorch_b200 import ops
    out = []
    for t in g.buffers:
        if isinstance(t, (ops.SplitTensor, ops.F32Tensor)):
            out.append((t.data.data_ptr(), t.data.numel() * t.data.element_size(), 'split' if isinstance(t, ops.SplitTensor) else 'f32',
                        t.B, t.H, t.W, t.C))
        elif torch.is_tensor(t):
            out.append((t.data_ptr(), t.numel() * t.element_size(), 'tensor', 0, 0, 0, 0))
    return out


def _resolve(views, bufs):
    """Raw views -> (format, B, H, W, pitch, c0, C, alias); the fused YOLO head's output (z) -> ('z', B, H, W, C, 0, C, -1)."""
    out, owners = [], []
    for v in views:
        if v is None:
            out.append(None)
            owners.append(None)
            continue
        base, B, H, W, C, pitch, ps = v
        hit = [b for b in bufs if b[0] <= base < b[0] + b[1]]
        assert len(hit) == 1, f'view {v} is not in exactly one buffer of the graph'
        p0, _, kind, bB, bH, bW, bC = hit[0]
        alias = owners.index(p0) if p0 in owners else -1
        owners.append(p0)
        if kind == 'tensor':
            out.append(('z', B, H, W, C, 0, C, -1))
            continue
        esz = 2 if kind == 'split' else 4
        assert (B, H, W, pitch) == (bB, bH, bW, bC) and (ps == 2 * B * H * W * pitch if kind == 'split' else ps == 0), (v, hit[0])
        out.append((kind, B, H, W, pitch, (base - p0) // esz, C, alias))
    return tuple(out)


class _Recorder:
    """Stands in for the loaded library: records every conv plan creation and aux launch and forwards every call."""

    def __init__(self, lib):
        self._lib, self.raw = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name != 'cvb_conv_plan_create' and name not in AUX:
            return fn

        def call(*args):
            self.raw.append(_snapshot(name, args))
            return fn(*args)
        return call


def _graphs():
    """(label, build-and-run) of the five benchmarked graphs: each returns the graph dict of the drop-in model, after one eager run."""
    from cvpytorch_b200 import synth

    def yolov5(u8):
        m = synth.build_yolov5s(calibrated=True).cuda()
        if u8:
            frames = torch.randint(0, 256, (64, 640, 640, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(5)).cuda()
            m.predict_frames(frames)
            return m._graph_for(frames)
        x = torch.randn(64, 3, 640, 640, generator=torch.Generator().manual_seed(5)).cuda()
        m.predict(x)
        return m._graph_for(x)

    def plain(build, B, H, W):
        def run():
            m = build().cuda()
            x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(B)).cuda()
            m.predict(x)
            return m._graph_for(x)
        return run

    def yolov6():
        import test_yolov6_gpu as T6
        m = T6.model('s')
        x = torch.randn(64, 3, 640, 640, generator=torch.Generator().manual_seed(1)).cuda()
        m.predict(x)
        return m._graph_for(x)

    return [('yolov5s', lambda: yolov5(False)), ('yolov5s_u8', lambda: yolov5(True)),
            ('yolox', plain(lambda: synth.build_yolox(calibrated=True), 64, 640, 640)),
            ('fcos', plain(lambda: synth.build_fcos(calibrated=True), 32, 800, 800)),
            ('deeplab', plain(lambda: synth.build_deeplab(calibrated=True), 16, 1024, 2048)),
            ('yolov6s', yolov6)]


def record_graphs(monkeypatch):
    """-> the set of signatures of the five graphs, one graph at a time (each freed before the next)."""
    from cvpytorch_b200 import _lib
    rec = _Recorder(_lib.lib())
    monkeypatch.setattr(_lib, 'lib', lambda: rec)  # (every wrapper calls _lib.lib() at call time)
    seen = set()
    for _, run in _graphs():
        rec.raw = []
        G = run()
        torch.cuda.synchronize()
        bufs = _buffers(G['g'])
        for name, fields, views, y in rec.raw:
            seen.add((name, fields, _resolve(views, bufs), y) if name == 'cvb_conv_plan_create' else (name, fields, _resolve(views, bufs)))
        del G, bufs
        rec.raw = []
        import gc
        gc.collect()
        torch.cuda.empty_cache()
    monkeypatch.undo()
    return seen


def _table(sigs):
    return '\n'.join(f'    {s!r},' for s in sorted(sigs, key=repr))


def test_launch_table_matches_the_graphs(cuda, monkeypatch):
    got, want = record_graphs(monkeypatch), set(LAUNCHES)
    assert len(want) == len(LAUNCHES), 'LAUNCHES lists a signature twice'
    assert got == want, (f'launches of the five graphs differ from LAUNCHES: new {_table(got - want)}\nno longer launched {_table(want - got)}\n'
                         f'recorded table:\n{_table(got)}')


def _views_of(sig):
    return [v for v in sig[2] if v is not None]


def test_launch_table_reaches_the_bench_shapes():
    """LAUNCHES has the shapes no other test reaches: a split16 plane stride >= 2^31 bytes (DeepLab), the YOLOv5 stem output at 64 x 320²,
    the FCOS GroupNorm heads at batch 32 and both depth-to-space shapes of YOLOv6-s."""
    views = [v for s in LAUNCHES for v in _views_of(s)]
    assert any(v[0] == 'split' and 2 * v[1] * v[2] * v[3] * v[4] >= 2 ** 31 for v in views)
    assert any(s[0] == 'cvb_conv_plan_create' and s[1][7] and s[2][1][1:4] == (64, 320, 320) for s in LAUNCHES)
    assert any(s[0] == 'cvb_groupnorm_relu' and s[2][0][1] == 32 for s in LAUNCHES)
    assert len({s[2] for s in LAUNCHES if s[0] == 'cvb_depth_to_space2'}) >= 2


# ------------------------------------------------------------------------------------------------ buffers and operands
def _gen(what):
    return torch.Generator(device='cuda').manual_seed(zlib.crc32(repr(what).encode()))


def _alloc(views):
    """NaN-filled buffers for resolved views (aliases share one) -> [(buffer, CvbView) or None]."""
    from cvpytorch_b200 import ops
    bufs, out = [], []
    for v in views:
        if v is None or v[0] == 'z':
            bufs.append(None)
            out.append(None)
            continue
        kind, B, H, W, pitch, c0, C, alias = v
        if alias >= 0:
            t = bufs[alias]
        else:
            t = (ops.SplitTensor if kind == 'split' else ops.F32Tensor)(B, H, W, pitch)
            t.data.fill_(NAN)
        bufs.append(t)
        out.append((t, t.view(c0, C)))
    return out


def _sl(v):
    return slice(v[5], v[5] + v[6])


def _chunks(B, per_image):
    n = max(1, CHUNK_ELEMS // max(1, per_image))
    return [slice(b, min(B, b + n)) for b in range(0, B, n)]


def _grid_planes(shape, density, lo_parity, g):
    """hi in {-1, 0, 1} (nonzero with probability `density`), lo = +-2^-12 on the channels of parity lo_parity (last dimension), fp16."""
    hi = (torch.rand(shape, generator=g, device='cuda') < density).half() * (torch.randint(0, 2, shape, generator=g, device='cuda').half() * 2 - 1)
    lo = (torch.randint(0, 2, shape, generator=g, device='cuda').half() * 2 - 1) * GRID
    lo[..., 1 - lo_parity::2] = 0
    return hi, lo


def _fill_split(t, view_c, gen_image):
    """Fills the split16 buffer t image by image (channels view_c of the last dimension) with gen_image(shape) -> (hi, lo)."""
    for b in range(t.B):
        hi, lo = gen_image((t.H, t.W, view_c.stop - view_c.start))
        t.data[0, b, ..., view_c] = hi
        t.data[1, b, ..., view_c] = lo


def _gauss_image(shape, g, scale=1.0):
    return R.split16(torch.randn(shape, generator=g, device='cuda') * scale)


def _outside(t, v):
    """The channels of buffer t outside view v (the 16-byte tail of an fp32 view excluded: the TMA store writes exact zeros there)."""
    end = v[5] + v[6]
    if t.data.dtype == torch.float32:
        end = -(-end * 4 // 16) * 16 // 4
    return t.data[..., :v[5]].clone(), t.data[..., end:].clone()


def _same(a, b):
    return torch.equal(torch.isnan(a), torch.isnan(b)) and bool(((a == b) | torch.isnan(a)).all())


# ------------------------------------------------------------------------------------------------ conv plans
def _conv_setup(sig, exact):
    """Buffers, weights and the plan of a conv signature, operands for check (a) (exact) or (b)."""
    from cvpytorch_b200 import ops
    _, p, views, y = sig
    k, s, pad, dil, act, out_kind, block_n, win, rfirst, rscale, no_res, halo, sched, sm_limit, cout_pad = p
    vin, vout, vres, vup = views
    g = _gen((sig, exact))
    bufs = _alloc(views)
    tin = bufs[0][0]
    C = vin[6]
    cout = y[0] * y[1] if y else vout[6]
    K = k * (win if win else k) * C
    density = min(2.0 / 3.0, (1500.0 / K) ** 0.5)
    if exact:
        _fill_split(tin, _sl(vin), lambda sh: _grid_planes(sh, density, 0, g))
    else:
        _fill_split(tin, _sl(vin), lambda sh: _gauss_image(sh, g))
    if exact:
        hi, lo = _grid_planes((cout, k, win or k, C), density, 1, g)
        w = (hi.double() + lo.double() * (hi != 0).double()).permute(0, 3, 1, 2)
        b = (torch.randint(-4, 5, (cout,), generator=g, device='cuda') + torch.randint(-8, 9, (cout,), generator=g, device='cuda') * GRID).double()
    else:
        w = torch.randn((cout, C, k, win or k), generator=g, device='cuda').double() / K ** 0.5
        b = torch.randn((cout,), generator=g, device='cuda').double() * 0.5
    w, b = w.cpu(), b.cpu()
    if y:
        wp, bp = ops.pack_yolo_head_weights(w, b, y[0], y[1])
    else:
        wp, bp = ops.pack_conv_weights(ops.window_weights(w, win) if win else w, b)
    if exact:
        assert bool(wp[1].any()), 'no weight has a nonzero lo word'
    if vres is not None:
        tr = bufs[2][0]
        if not (vres[7] == 0 and vres[5] == vin[5]):  # (a residual that is the input itself is filled already)
            if exact:
                _fill_split(tr, _sl(vres), lambda sh: (torch.randint(-2, 3, sh, generator=g, device='cuda').half(),
                                                       torch.randint(-4, 5, sh, generator=g, device='cuda').half() * GRID))
            else:
                _fill_split(tr, _sl(vres), lambda sh: _gauss_image(sh, g))
    if vup is not None:
        tu = bufs[3][0]
        shape = tu.data[..., _sl(vup)].shape
        if exact:
            tu.data[..., _sl(vup)] = (torch.randint(-4, 5, shape, generator=g, device='cuda') + torch.randint(-8, 9, shape, generator=g, device='cuda') * GRID).float()
        else:
            tu.data[..., _sl(vup)] = torch.randn(shape, generator=g, device='cuda')
    z = yd = ws = None
    if y:
        na, no, anchors, stride, z_rows, z_off, has_ws, conf, multi = y
        z = torch.full((vout[1], z_rows, no), NAN, device='cuda')
        ws = ops.NmsWorkspace(vout[1], z_rows, no - 5) if has_ws else None
        if ws is not None:
            ops.nms_reset(ws)
        yd = ops.yolo_decode_desc(na, no, torch.tensor(anchors).view(na, 2), stride, z, z_rows, z_off, ws, conf, bool(multi))
        out_view = ops.CvbView(z.data_ptr(), vout[1], vout[2], vout[3], na * 128, na * 128, 0)
    else:
        out_view = bufs[1][1]
    act_name = {0: None, 1: 'silu', 2: 'relu'}[act]
    plan = ops.ConvPlan(bufs[0][1], out_view, wp, bp, k, s, pad, dil, act_name, residual=bufs[2][1] if vres else None,
                        up_partial=bufs[3][1] if vup else None, block_n=block_n, sm_limit=sm_limit, w_window=win, no_resident=no_res,
                        residual_before_act=rfirst, halo=halo, residual_scale=rscale, yolo=yd, schedule=sched)
    return dict(bufs=bufs, wp=wp, bp=bp, plan=plan, z=z, ws=ws, act=act_name, k_tap=(win or k) * C, taps=k, cout=cout)


def _conv_run(sig, exact):
    """Runs the plan once; -> (setup, output view values as [B, H, W, C] planes / fp32, residual before the run)."""
    st = _conv_setup(sig, exact)
    _, p, views, y = sig
    vout, vres = views[1], views[2]
    res_before = None
    if vres is not None:
        res_before = st['bufs'][2][0].data[..., _sl(vres)].clone()
    outside = None if y else _outside(st['bufs'][1][0], vout)
    st['plan'].run()
    torch.cuda.synchronize()
    if outside is not None:
        after = _outside(st['bufs'][1][0], vout)
        for a, b_ in zip(outside, after):
            assert _same(a, b_), f'{_id(sig)}: the kernel wrote outside its output view'
        if vout[0] == 'f32':
            end = vout[5] + vout[6]
            tail = st['bufs'][1][0].data[..., end:-(-end * 4 // 16) * 16 // 4]
            assert bool((tail.isnan() | (tail == 0)).all()), f'{_id(sig)}: nonzero values after the view, up to its 16-byte boundary'
    st['res'] = res_before
    return st


def _conv_reference(sig, st, imgs, exact):
    """float64 reference of images `imgs` and its bound: (a) the grid bound (module docstring), (b) split_conv_reference."""
    _, p, views, y = sig
    k, s, pad, dil, act, out_kind, block_n, win, rfirst, rscale = p[:10]
    vin, vout, vres, vup = views
    tin = st['bufs'][0][0].data[:, imgs, ..., _sl(vin)]
    res = st['res'][:, imgs] if st['res'] is not None else None
    up = st['bufs'][3][0].data[imgs, ..., _sl(vup)] if vup is not None else None
    out_h = vout[2]
    if not exact:
        return R.split_conv_reference(tin, st['wp'], st['bp'], k, s, pad, dil, st['act'], residual=res, resid_first=rfirst, resid_scale=rscale,
                                      up=up, w_window=win, block_n=(128 if y else block_n), cout=(None if y else st['cout']), out_h=out_h)
    cout = st['wp'].shape[1] if y else st['cout']
    x = R.split64(tin)
    w = (st['wp'][0].double() + st['wp'][1].double())[:cout]
    (S, A), taps, k_tap = R.split_conv_sums([(x, w), (x.abs(), w.abs())], k, s, pad, dil, win, out_h)
    del x
    bias = st['bp'][:cout].double().view(1, -1, 1, 1)
    ref, terms = S + bias, A + bias.abs()
    Ho, Wo = ref.shape[2:]
    if up is not None:
        u = F.interpolate(up.double().permute(0, 3, 1, 2), scale_factor=2, mode='nearest')[:, :, :Ho, :Wo]
        ref, terms = ref + u, terms + u.abs()
    rsum = R.split64(res) * rscale if res is not None else torch.zeros_like(ref)
    if rfirst:
        ref, terms = ref + rsum, terms + rsum.abs()
    worst = float(terms.max()) / GRID
    assert worst < 2 ** 24, f'{_id(sig)}: a partial sum reaches {worst:.3g} grid units; the grid operands are not exact here'
    if st['act'] == 'silu':
        ref = F.silu(ref)
    elif st['act'] == 'relu':
        ref = F.relu(ref)
    if res is not None and not rfirst:
        ref = ref + rsum
    chain = 3 * taps * (-(-k_tap // 16))
    gain = (RZ_C * chain + 2.0 ** -23) * (S.abs() + 2.0 ** -11 * A)
    bound = R.SPLIT_REL * (ref.abs() + rsum.abs()) + (1.1 if st['act'] == 'silu' else 1.0) * gain + 1e-30
    if views[1][0] == 'split':
        bound = bound + R.SPLIT_OUT_ABS  # the lo word of a small output is an fp16 subnormal (fp64ref.split_out_bound)
    return ref, bound


def _conv_check(sig, st, imgs, exact, what):
    _, p, views, y = sig
    vout = views[1]
    B = vout[1]
    for c in imgs:
        ref, bound = _conv_reference(sig, st, c, exact)
        if y:
            _yolo_check(sig, st, c, ref, bound, what)
            continue
        buf = st['bufs'][1][0].data
        out = R.conv_out64(buf[:, c, ..., _sl(vout)] if vout[0] == 'split' else buf[c, ..., _sl(vout)])
        if exact:
            R.check(out, ref, bound, f'{what} images {c.start}..{c.stop - 1} of {B}')
            if vout[0] == 'split':
                _assert_split_format(buf[:, c, ..., _sl(vout)], what)
        else:
            R.check_conv(out, ref, bound, f'{what} images {c.start}..{c.stop - 1} of {B}')
        del ref, bound, out


def _assert_split_format(planes, what):
    """hi = fp16_rn(x), lo = fp16_rn(x - hi): |lo| is at most half an fp16 ulp of hi (2^-25 where hi is subnormal or zero), below the
    saturation at 65504.  Sees hi and lo swapped, which hi + lo alone cannot."""
    hi, lo = planes[0].float(), planes[1].float()
    half_ulp = torch.ldexp(torch.ones_like(hi), torch.frexp(hi).exponent - 12).clamp_min(2.0 ** -25)
    bad = (lo.abs() > half_ulp) & (hi.abs() < 65504)
    assert not bool(bad.any()), f'{what}: {int(bad.sum())} outputs are not in the split16 format (|lo| above half an ulp of hi)'


def _yolo_check(sig, st, c, ref, bound, what):
    import test_conv_plans_gpu as CP
    _, _, views, y = sig
    na, no, anchors, stride, z_rows, z_off, _, _, _ = y
    B, ny, nx = ref.shape[0], ref.shape[2], ref.shape[3]
    npix = ny * nx
    xr = ref.view(B, na, 128, npix).permute(0, 1, 3, 2)[..., :no]
    dx = bound.view(B, na, 128, npix).permute(0, 1, 3, 2)[..., :no]
    zref, zbound = CP.decode_reference(xr, dx, torch.tensor(anchors, dtype=torch.float64, device='cuda').view(na, 2), stride, nx)
    z = st['z'][c]
    CP._decode_check(z[:, z_off:z_off + na * npix].reshape(B, na, npix, no), zref, zbound, what)
    assert bool(z[:, :z_off].isnan().all()) and bool(z[:, z_off + na * npix:].isnan().all()), f'{what}: wrote outside its z rows'


def _conv(sig):
    vout = sig[2][1]
    B = vout[1]
    per_image = (sig[3][0] * 128 if sig[3] else vout[6]) * vout[2] * vout[3] * 4
    for exact in (True, False):
        st = _conv_run(sig, exact)
        imgs = _chunks(B, per_image) if exact else [slice(0, 1), slice(B - 1, B)]
        _conv_check(sig, st, imgs, exact, f'{_id(sig)} ({"grid" if exact else "Gaussian"})')
        del st
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ aux launches
def _args(sig):
    """Aux signature -> (argument values with the views in place of their ('view', i) markers, allocated (buffer, CvbView) per view)."""
    name, fields, views = sig
    bufs = _alloc(views)
    return [bufs[f[1]] if isinstance(f, tuple) and len(f) == 2 and f[0] == 'view' else f for f in fields], bufs


def _put(tv, v, g, scale=1.0):
    """Gaussian values into view v of buffer tv[0] (split16 or fp32), image by image."""
    if tv[0].data.dtype == torch.float32:
        for b in range(v[1]):
            tv[0].data[b, ..., _sl(v)] = torch.randn(tv[0].data[b, ..., _sl(v)].shape, generator=g, device='cuda') * scale
        return
    _fill_split(tv[0], _sl(v), lambda sh: _gauss_image(sh, g, scale))


def _get(tv, v, imgs):
    t = tv[0].data
    return t[0, imgs, ..., _sl(v)].double() + t[1, imgs, ..., _sl(v)].double() if t.dtype == torch.float16 else t[imgs, ..., _sl(v)].double()


def _check_outside(tv, v, before, what):
    for a, b in zip(before, _outside(tv[0], v)):
        assert _same(a, b), f'{what}: wrote outside its view'


def _bitwise(out, ref, what):
    import test_aux_kernels_gpu as AK
    AK._assert_same_bits(out, ref, what)


def _aux(sig):
    import test_aux_kernels_gpu as AK
    from cvpytorch_b200 import ops
    name, fields, views = sig
    if name in ('cvb_yolox_decode', 'cvb_fcos_decode', 'cvb_yolov6_decode', 'cvb_yolo_decode'):
        return _decode(sig)
    a, bufs = _args(sig)
    g = _gen(sig)
    what = _id(sig)
    if name in ('cvb_stem_s2d', 'cvb_stem_s2d_u8'):
        u8 = name.endswith('u8')
        _, B, H, W = a[:4]
        tv, pad_left = a[-2], a[-1]
        v = views[0]
        before = _outside(tv[0], v)
        cols = slice(pad_left, pad_left + W // 2)
        t = tv[0].data
        pad_before = (t[:, :, :, :pad_left].clone(), t[:, :, :, pad_left + W // 2:].clone())
        if u8:
            mean, std, rev = a[4], a[5], a[6]
            frame = torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8, generator=g, device='cuda')
            ops.stem_s2d(frame, tv[1], pad_left=pad_left, norm=dict(mean=mean, std=std, reverse_channels=bool(rev)))
        else:
            x = torch.randn((B, 3, H, W), generator=g, device='cuda') * 3
            ops.stem_s2d(x, tv[1], pad_left=pad_left)
        torch.cuda.synchronize()
        from oracle import yolov5_oracle as YO
        for c in _chunks(B, H * W * 16):
            xc = YO.input_transform(frame[c].cpu(), mean, std, reverse_channels=bool(rev)).cuda() if u8 else x[c]
            hi, lo = R.split16(AK._s2d_reference(xc))
            _bitwise(t[0, c, :, cols, _sl(v)], hi[..., :v[6]], f'{what} hi')
            _bitwise(t[1, c, :, cols, _sl(v)], lo[..., :v[6]], f'{what} lo')
        assert _same(pad_before[0], t[:, :, :, :pad_left]) and _same(pad_before[1], t[:, :, :, pad_left + W // 2:]), f'{what}: wrote into the pad columns'
        _check_outside(tv, v, before, what)
        return
    if name == 'cvb_depth_to_space2':
        src, dst = a
        _put(src, views[0], g)
        before = _outside(dst[0], views[1])
        ops.depth_to_space2(src[1], dst[1])
        torch.cuda.synchronize()
        for c in _chunks(views[1][1], views[1][2] * views[1][3] * views[1][6]):
            for plane in (0, 1):
                _bitwise(dst[0].data[plane, c, ..., _sl(views[1])], _d2s_reference(src[0].data[plane, c, ..., _sl(views[0])]), f'{what} plane {plane}')
        _check_outside(dst, views[1], before, what)
        return
    if name == 'cvb_sppf_pool':
        x, y1, y2, y3 = a
        _put(x, views[0], g, 4.0)
        befores = [_outside(t[0], v) for t, v in zip(a, views)]
        ops.sppf_pool(x[1], y1[1], y2[1], y3[1])
        torch.cuda.synchronize()
        B = views[0][1]
        for c in _chunks(B, 4 * views[0][2] * views[0][3] * views[0][6]):
            p = _get(x, views[0], c).permute(0, 3, 1, 2)
            for i in (1, 2, 3):
                p = F.max_pool2d(p, 5, 1, 2)
                _bitwise(_get(a[i], views[i], c), p.permute(0, 2, 3, 1), f'{what} y{i}')
        if views[1][7] < 0:
            for t, v, bf in zip(a, views, befores):
                _check_outside(t, v, bf, what)
        return
    x, y = bufs[0], (bufs[-1] if len(bufs) > 1 else None)
    vx, vy = views[0], views[-1]
    _put(x, vx, g, 5.0 if name != 'cvb_groupnorm_relu' else 3.0)
    if name == 'cvb_groupnorm_relu':  # GroupNorm inputs well off zero, as the FCOS heads see them
        t = x[0].data
        for b in range(vx[1]):
            v64 = t[0, b, ..., _sl(vx)].float() + t[1, b, ..., _sl(vx)].float() + 10
            t[0, b, ..., _sl(vx)], t[1, b, ..., _sl(vx)] = R.split16(v64)
    before = _outside(y[0], vy) if y is not None and vy[7] < 0 else None
    B = vx[1]
    if name == 'cvb_maxpool3x3s2':
        ops.maxpool3x3s2(x[1], y[1])
        torch.cuda.synchronize()
        for c in _chunks(B, vx[2] * vx[3] * vx[6]):
            ref = F.max_pool2d(_get(x, vx, c).permute(0, 3, 1, 2), 3, 2, 1)
            _bitwise(_get(y, vy, c), ref.permute(0, 2, 3, 1), what)
    elif name == 'cvb_split_to_f32nhwc':
        ops.split_to_f32(x[1], y[1])
        torch.cuda.synchronize()
        for c in _chunks(B, vx[2] * vx[3] * vx[6]):
            t = x[0].data
            _bitwise(y[0].data[c, ..., _sl(vy)], t[0, c, ..., _sl(vx)].float() + t[1, c, ..., _sl(vx)].float(), what)
    elif name == 'cvb_groupnorm_relu':
        groups, eps, relu = a[1], a[4], a[5]
        C = vx[6]
        gamma, beta = torch.rand(C, generator=g, device='cuda') + 0.5, torch.randn(C, generator=g, device='cuda')
        ops.groupnorm_relu(x[1], groups, gamma, beta, eps, y[1], ops.GroupNormWorkspace(B, groups), relu=bool(relu))
        torch.cuda.synchronize()
        for c in _chunks(B, 3 * vx[2] * vx[3] * C):
            ref, bound = R.groupnorm_reference(_get(x, vx, c).permute(0, 3, 1, 2), groups, gamma, beta, eps, bool(relu))
            R.check(_get(y, vy, c).permute(0, 3, 1, 2), ref, bound, what)
    elif name == 'cvb_dwconv3x3':
        dil, relu = a[3], a[4]
        C = vx[6]
        w9c, bias = ops.pack_dw_weights(torch.randn(C, 1, 3, 3, dtype=torch.float64), torch.randn(C, dtype=torch.float64))
        ops.dwconv3x3(x[1], w9c, bias, dil, y[1], bool(relu))
        torch.cuda.synchronize()
        wk, bk = w9c.double().t().reshape(C, 1, 3, 3), bias.double()
        for c in _chunks(B, 3 * vx[2] * vx[3] * C):
            xn = _get(x, vx, c).permute(0, 3, 1, 2)
            ref = F.conv2d(xn, wk, bk, 1, dil, dil, groups=C)
            absref = F.conv2d(xn.abs(), wk.abs(), bk.abs(), 1, dil, dil, groups=C)
            ref = F.relu(ref) if relu else ref
            # test_aux_kernels_gpu._dw_case: nine fmaf roundings from the bias, then the split16 store
            R.check(_get(y, vy, c).permute(0, 3, 1, 2), ref, 10 * R.U24 * absref + R.split_out_bound(ref), what)
    elif name == 'cvb_global_avgpool':
        ops.global_avgpool(x[1], y[1])
        torch.cuda.synchronize()
        npix = vx[2] * vx[3]
        xs = _get(x, vx, slice(0, B))
        ref = xs.mean((1, 2), keepdim=True)
        # test_aux_kernels_gpu.test_global_avgpool's bound
        bound = R.gamma_n(-(-npix // 256) + 7) * xs.abs().mean((1, 2), keepdim=True) + R.U24 * ref.abs() + R.split_out_bound(ref)
        R.check(_get(y, vy, slice(0, B)), ref, bound, what)
    elif name == 'cvb_bilinear_resize':
        ops.bilinear_resize(x[1], y[1])
        torch.cuda.synchronize()
        for c in _chunks(B, 8 * vy[2] * vy[3] * vy[6]):
            wts, vals = AK._bilinear_terms(_get(x, vx, c), vy[2], vy[3])
            ref = (wts * vals).sum(0)
            R.check(_get(y, vy, c), ref, R.gamma_n(4) * (wts * vals).abs().sum(0) + R.split_out_bound(ref), what)
            del wts, vals
    elif name == 'cvb_upsample_argmax':
        nc, Ho, Wo = a[1], a[3], a[4]
        labels = torch.full((B, Ho, Wo), -1, dtype=torch.int64, device='cuda')
        ops.upsample_argmax(x[1], nc, labels)
        torch.cuda.synchronize()
        for c in _chunks(B, 8 * Ho * Wo * nc):
            wts, vals = AK._bilinear_terms(_get(x, vx, c), Ho, Wo)
            ref = (wts * vals).sum(0)
            bnd = R.gamma_n(4) * (wts * vals).abs().sum(0)
            del wts, vals
            best = ref.max(-1, keepdim=True).values
            second = torch.where(ref == best, torch.full_like(ref, float('-inf')), ref).max(-1).values
            decided = (best[..., 0] - second) > 2 * bnd.max(-1).values
            lab = labels[c]
            assert bool(((lab >= 0) & (lab < nc)).all()), what
            bad = decided & (lab != ref.argmax(-1))
            assert not bool(bad.any()), f'{what}: {int(bad.sum())} labels differ from the float64 argmax where the gap exceeds the bound'
    else:
        raise AssertionError(f'no check for {name}')
    if before is not None:
        _check_outside(y, vy, before, what)


def _d2s_reference(src):
    """[B, h, w, 4c] (channel (py*2+px)*c + o) -> [B, 2h, 2w, c] (pixel (2y+py, 2x+px)) (ops.depth_to_space2)."""
    B, h, w, C4 = src.shape
    c = C4 // 4
    return src.view(B, h, w, 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(B, 2 * h, 2 * w, c)


_DECODES_CHECKED = set()


def _decode(sig):
    """The decodes at their level shapes and batch, through the decode checks of test_aux_kernels_gpu / test_yolov6_gpu / test_conv_plans_gpu."""
    import test_aux_kernels_gpu as AK
    name, fields, views = sig
    v = views[0]
    B, H, W = v[1], v[2], v[3]
    if name == 'cvb_yolox_decode':
        AK._yolox_case(fields[2], B, H, W, fields[3])
    elif name == 'cvb_fcos_decode':
        AK._fcos_case(fields[2], B, H, W, fields[3], fields[4])
    elif name == 'cvb_yolov6_decode':
        _yolov6_decode_case(fields[2], B, H, W, fields[3], fields[9])
    else:
        raise AssertionError(f'{name}: the graphs fuse the YOLOv5 decode into the head conv; add a check when a graph launches it')


def _yolov6_decode_case(nc, B, H, W, stride, multi):
    """cvb_yolov6_decode of one level against the oracle (test_yolov6_gpu.test_decode_kernel_against_oracle): box and objectness bit for
    bit, class scores within 1e-6 (sigmoid_fast); rows outside the level stay NaN."""
    from cvpytorch_b200 import ops
    from oracle import yolov6_oracle as V6
    g = torch.Generator().manual_seed(nc * 1000 + H)
    cls = torch.randn(B, H, W, nc, generator=g) * 2 - 3
    reg = torch.rand(B, H, W, 4, generator=g) * 4
    off = 3
    A = off + H * W + 2
    z = torch.full((B, A, nc + 5), NAN, device='cuda')
    cv, rv = ops.CvbView(), ops.CvbView()
    ct, rt = cls.cuda(), reg.cuda()
    for vv, t in ((cv, ct), (rv, rt)):
        vv.base, vv.B, vv.H, vv.W, vv.C, vv.c_pitch, vv.plane_stride = t.data_ptr(), B, H, W, t.shape[3], t.shape[3], 0
    ops.yolov6_decode(cv, rv, nc, stride, z, A, off, None, 0.001, bool(multi))
    torch.cuda.synchronize()
    zo = V6.detect(torch.sigmoid(cls).reshape(B, -1, nc), reg.reshape(B, -1, 4), [(H, W)], strides=(stride,))
    zc = z[:, off:off + H * W].cpu()
    assert torch.equal(zc[..., :5], zo[..., :5]), f'yolov6_decode {B}x{H}x{W}: box / objectness differ from the oracle'
    assert float((zc[..., 5:] - zo[..., 5:]).abs().max()) < 1e-6
    assert bool(z[:, :off].isnan().all()) and bool(z[:, off + H * W:].isnan().all()), 'yolov6_decode wrote outside its rows'


# ------------------------------------------------------------------------------------------------ the launch tests
def _id(sig):
    name = sig[0][len('cvb_'):]
    if name == 'conv_plan_create':
        p, views, y = sig[1], sig[2], sig[3]
        vin, vout = views[0], views[1]
        parts = [f'conv{p[0]}x{p[0]}s{p[1]}d{p[3]}', f'{vin[1]}x{vin[2]}x{vin[3]}x{vin[6]}', f'{vout[2]}x{vout[3]}x{vout[6]}',
                 {0: 'none', 1: 'silu', 2: 'relu'}[p[4]]]
        parts += ['res'] if views[2] else []
        parts += ['up'] if views[3] else []
        parts += [f'win{p[7]}'] if p[7] else []
        parts += [f'yolo{y[5]}'] if y else []
        parts += [f'bn{p[6]}'] if p[6] else []
        parts += [f'in@{vin[5]}/{vin[4]}', f'out@{vout[5]}/{vout[4]}']
        return '-'.join(parts)
    v = sig[2][0]
    return '-'.join([name, 'x'.join(map(str, v[1:4])), f'c{v[6]}@{v[5]}/{v[4]}'] + [str(f) for f in sig[1] if isinstance(f, (int, float))])


@pytest.mark.parametrize('sig', LAUNCHES, ids=[_id(s) for s in LAUNCHES])
def test_launch_at_its_real_shape(cuda, sig):
    (_conv if sig[0] == 'cvb_conv_plan_create' else _aux)(sig)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ depth-to-space at its edges
@pytest.mark.parametrize('B,h,w', [(3, 1, 5), (1, 4, 1), (3, 5, 7), (2, 6, 4)])
@pytest.mark.parametrize('C', [8, 128])
def test_depth_to_space2(cuda, B, h, w, C):
    """A bitwise permutation: src a channel slice (c0 = 8) of a wider buffer, dst a channel slice of a wider NaN-filled buffer like the
    cv3 input concat of BiFusion; every other channel of both buffers keeps its bits."""
    from cvpytorch_b200 import ops
    g = _gen(('d2s', B, h, w, C))
    src = ops.SplitTensor(B, h, w, 4 * C + 16)
    src.data.copy_(torch.randn(src.data.shape, generator=g, device='cuda').half())
    dst = ops.SplitTensor(B, 2 * h, 2 * w, 3 * C)
    dst.data.fill_(NAN)
    src0 = src.data.clone()
    ops.depth_to_space2(src.view(8, 4 * C), dst.view(C, C))
    torch.cuda.synchronize()
    for plane in (0, 1):
        _bitwise(dst.data[plane, ..., C:2 * C], _d2s_reference(src0[plane, ..., 8:8 + 4 * C]), f'depth_to_space2 plane {plane}')
    assert bool(dst.data[..., :C].isnan().all()) and bool(dst.data[..., 2 * C:].isnan().all()), 'depth_to_space2 wrote outside its dst slice'
    assert torch.equal(src.data.view(torch.int16), src0.view(torch.int16)), 'depth_to_space2 changed its source'


def test_depth_to_space2_refusals(cuda):
    """cvb_depth_to_space2 refuses C not a multiple of 8, src not 4 x dst channels, sizes not doubled, fp32 views and misalignment."""
    from cvpytorch_b200 import ops
    from cvpytorch_b200._lib import CvbError
    src = ops.SplitTensor(2, 3, 4, 64)
    dst = ops.SplitTensor(2, 6, 8, 32)
    ok = (src.view(0, 32), dst.view(0, 8))
    ops.depth_to_space2(*ok)
    f32 = ops.F32Tensor(2, 6, 8, 16)

    def shifted(v, nbytes):
        v2 = ops.CvbView()
        v2.base, v2.B, v2.H, v2.W, v2.C, v2.c_pitch, v2.plane_stride = v.base + nbytes, v.B, v.H, v.W, v.C, v.c_pitch, v.plane_stride
        return v2

    def reshaped(v, **kw):
        v2 = shifted(v, 0)
        for k_, val in kw.items():
            setattr(v2, k_, val)
        return v2

    bad = {'C not a multiple of 8': (reshaped(ok[0], C=16), reshaped(ok[1], C=4)),
           'src not 4 x dst channels': (src.view(0, 24), dst.view(0, 8)),
           'sizes not doubled': (ok[0], reshaped(ok[1], W=7)),
           'fp32 dst': (ok[0], f32.view(0, 8)),
           'misaligned base': (shifted(ok[0], 2), ok[1]),
           'misaligned pitch': (reshaped(ok[0], c_pitch=36), ok[1])}
    for what, (s, d) in bad.items():
        with pytest.raises(CvbError):
            ops.depth_to_space2(s, d)
        print(f'refused: {what}')


# ------------------------------------------------------------------------------------------------ the exact check has teeth
def test_exact_check_sees_a_lost_tile_and_a_misread_lo_plane(cuda):
    """The YOLOv5-s stem conv (64 x 320² x 32 outputs, row-window loader) under check (a): its output passes; the same output with one
    128-pixel tile of the last image zeroed, with the lo words of one pixel row read from the next row, or with one 8-channel slice
    shifted by a pixel is rejected, and hi and lo swapped on one pixel row fail the split16 format check."""
    stems = [s for s in LAUNCHES if s[0] == 'cvb_conv_plan_create' and s[1][7] and s[2][1][1:4] == (64, 320, 320)]
    assert stems
    sig = stems[0]
    vout = sig[2][1]
    B = vout[1]
    st = _conv_run(sig, True)
    last = slice(B - 1, B)
    ref, bound = _conv_reference(sig, st, last, True)
    buf = st['bufs'][1][0].data[:, last, ..., _sl(vout)]

    def rejected(d):
        try:
            R.check(R.conv_out64(d), ref, bound, 'perturbed')
        except AssertionError:
            return True
        return False
    R.check(R.conv_out64(buf), ref, bound, 'stem conv, last image')
    lost = buf.clone()
    lost[:, :, 96:104, 0:16] = 0  # one 8 x 16 pixel tile
    misread = buf.clone()
    misread[1, :, 7] = buf[1, :, 8]  # the lo words of pixel row 7 read from row 8
    swapped = buf.clone()
    swapped[0, :, 7], swapped[1, :, 7] = buf[1, :, 7], buf[0, :, 7]
    shifted = buf.clone()
    shifted[..., 8:16] = torch.roll(buf[..., 8:16], 1, dims=3)
    for what, d in (('lost tile', lost), ('lo plane misread on one row', misread), ('channel slice shifted', shifted)):
        assert rejected(d), f'check (a) accepts the output with a {what}'
    _assert_split_format(buf, 'stem conv, last image')
    with pytest.raises(AssertionError):
        _assert_split_format(swapped, 'hi / lo swapped on one row')
