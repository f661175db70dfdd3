"""One small launch of every kernel family (every conv_tc_kernel<BLOCK_N, BLOCK_K, OUT> instantiation the planner can select, both
activation loaders, residual / up-partial epilogues, the aux kernels, decode, the three NMS pipelines), for
  compute-sanitizer --tool memcheck  python tools/sanitize_kernels.py
  compute-sanitizer --tool racecheck python tools/sanitize_kernels.py
Shapes are tiny (the sanitizer serialises everything).  Results are compared loosely against torch only to make sure the launches ran."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from cvpytorch_b200 import models as M  # noqa: E402
from cvpytorch_b200 import ops  # noqa: E402
from oracle import nms_oracle as NO  # noqa: E402
from oracle import yolox_oracle as XO  # noqa: E402
import test_conv_gpu as T  # noqa: E402
import test_nms_kernels_gpu as TN  # noqa: E402

torch.backends.cudnn.allow_tf32 = False  # the torch fp32 reference must not run on TF32 tensor cores
torch.backends.cuda.matmul.allow_tf32 = False

n = 0


def conv(*a, **k):
    global n
    err = T._run_conv(*a, **k)
    if err >= 2e-5:
        print('NUMERIC MISMATCH', a, k, err)
    n += 1


# (cin, cout, k, s, p, B, H, W): every (BLOCK_N, BLOCK_K) pair through cin / cout / block_n choices
for cin in (16, 32, 64):           # BLOCK_K 16 / 32 / 64
    for bn in (32, 64, 128, 256):
        conv(cin, max(bn, 32), 1, 1, 0, 1, 16, 16, block_n=bn)
        conv(cin, max(bn, 32), 1, 1, 0, 1, 16, 16, block_n=bn, act=None, f32_out=True)
for halo in (-1, 1, 2):
    conv(32, 32, 3, 1, 1, 1, 16, 24, halo=halo)
    conv(64, 64, 3, 1, 1, 1, 16, 24, halo=halo, residual=True)
    conv(64, 128, 3, 2, 1, 1, 16, 24, halo=halo)
    conv(128, 128, 3, 1, 1, 1, 16, 16, halo=halo, no_resident=1)
conv(128, 128, 1, 1, 0, 1, 16, 16, up=True)
conv(64, 64, 1, 1, 0, 2, 20, 20, residual=True)
print('conv launches ok:', n)

# aux kernels
x = torch.randn(1, 3, 64, 64, device='cuda')
t = ops.SplitTensor(1, 32, 35, 16)
ops.stem_s2d(x, t.view())
p = ops.SplitTensor(1, 20, 20, 256)
ops.nchw_to_split(torch.randn(1, 64, 20, 20, device='cuda'), p.view(0, 64))
ops.sppf_pool(p.view(0, 64), p.view(64, 64), p.view(128, 64), p.view(192, 64))
ops.split_to_nchw(p.view())
# one channel-slice case per aux kernel: inputs and outputs are slices of wider buffers, 24 channels = a partial 32-channel slab
q = ops.SplitTensor(1, 9, 13, 64)
ops.nchw_to_split(torch.randn(1, 24, 9, 13, device='cuda'), q.view(8, 24))
ops.split_to_nchw(q.view(8, 24))
f = ops.F32Tensor(1, 9, 13, 40)
ops.split_to_f32(q.view(8, 24), f.view(8, 24))
ops.f32nhwc_to_nchw(f.view(4, 24))
ops.stem_s2d(x, ops.SplitTensor(1, 32, 35, 16).view(), pad_left=2)
ops.maxpool3x3s2(q.view(8, 24), ops.SplitTensor(1, 5, 7, 40).view(16, 24))
d = ops.SplitTensor(1, 9, 13, 48)
w9c, bias = ops.pack_dw_weights(torch.randn(24, 1, 3, 3, dtype=torch.float64), torch.randn(24, dtype=torch.float64))
for dil in (1, 6):
    ops.dwconv3x3(q.view(8, 24), w9c, bias, dil, d.view(16, 24), True)
gp = ops.SplitTensor(1, 1, 1, 40)
ops.global_avgpool(q.view(8, 24), gp.view(16, 24))
r = ops.SplitTensor(1, 17, 23, 64)
ops.bilinear_resize(q.view(8, 24), r.view(24, 24))
ops.bilinear_resize(gp.view(16, 24), r.view(40, 24))
ops.groupnorm_relu(q.view(8, 24), 3, torch.ones(24, device='cuda'), torch.zeros(24, device='cuda'), 1e-5, d.view(16, 24),
                   ops.GroupNormWorkspace(1, 3), relu=False)
lg = ops.F32Tensor(1, 9, 13, 24)
ops.upsample_argmax(lg.view(0, 19), 19, torch.zeros((1, 17, 23), dtype=torch.int64, device='cuda'))
ro = ops.F32Tensor(1, 9, 13, 8)
ops.yolox_decode(ro.view(0, 5), lg.view(0, 19), 19, 8.0, ops.YoloxWorkspace(1, 9 * 13 + 8), 4)
ops.fcos_decode(lg.view(0, 19), ro.view(0, 5), 19, 8.0, 1.0, ops.FcosWorkspace(1, 9 * 13 + 8), 4)
torch.cuda.synchronize()
print('aux kernels ok')

# YOLOv5 decode + NMS (both phases) on a small stress tensor
pred = torch.from_numpy(NO.make_stress_prediction(1, A=25200, regime='typical', seed=2)).cuda()
M.non_max_suppression(pred, 0.001, 0.6, multi_label=True)
pred = torch.from_numpy(NO.make_stress_prediction(1, A=25200, regime='capped', seed=3)).cuda()
M.non_max_suppression(pred, 0.001, 0.6, multi_label=True)
# full path with the sort's grid-wide steps: 9000 candidates whose top ~3k keep fewer than max_det boxes
wsb = ops.NmsWorkspace(1, 9000, 4)
ops.yolo_nms(torch.from_numpy(TN.big_scene(9000)[None]).cuda(), wsb)
torch.cuda.synchronize()
assert int(TN.ws_regions(wsb)['cntB'][0]) == 9000 and int(wsb.status[0]) == 0
print('yolo nms ok')

# YOLOX post-process
rec = XO.make_stress_records(regime='typical', seed=2)
ws = ops.YoloxWorkspace(1, rec.shape[0])
ops.yolox_nms(ws, 0.01, 0.65, cand=torch.from_numpy(rec[None]).cuda().contiguous())
# 1001 candidates > vanilla_above: per-class chains of kept boxes
rec = TN._switch_scene(1001)
ws = ops.YoloxWorkspace(1, rec.shape[0])
ops.yolox_nms(ws, 0.01, 0.65, vanilla_above=1000, cand=torch.from_numpy(rec[None]).cuda().contiguous())
torch.cuda.synchronize()
assert int(ws.count[0]) == 1001
print('yolox nms ok')

# FCOS NMS
B, N = 1, 4096
g = torch.Generator().manual_seed(0)
sc = torch.rand(B, N, generator=g).cuda()
cl = torch.randint(1, 81, (B, N), generator=g, dtype=torch.int32).cuda()
xy = torch.rand(B, N, 2, generator=g) * 700
wh = torch.rand(B, N, 2, generator=g) * 90 + 4
bx = torch.cat([xy, xy + wh], 2).cuda().contiguous()
fw = ops.FcosWorkspace(B, N)
ops.fcos_nms(fw, 0.05, 0.6, scores=sc, classes=cl, boxes=bx)
# more locations than the 4096 keys of the selection
fs, fc, fb = TN.fcos_scene(6000)
fw = ops.FcosWorkspace(1, 6000)
ops.fcos_nms(fw, 0.05, 0.6, scores=torch.from_numpy(fs[None]).cuda(), classes=torch.from_numpy(fc[None].astype('int32')).cuda(),
             boxes=torch.from_numpy(fb[None]).cuda())
torch.cuda.synchronize()
assert int(fw.out_count[0]) == 1000 and int(fw.status[0]) == 0
print('fcos nms ok')

# whole model at a tiny size (every graph step incl. the fused decode histogram path)
from cvpytorch_b200 import synth  # noqa: E402
m = synth.build_yolov5s(True)
m.predict(torch.randn(1, 3, 64, 64, device='cuda'))
torch.cuda.synchronize()
print('model ok')

# fused detect head: 1x1 conv with the YOLOv5 decode as its epilogue (CVB_OUT_YOLO; bulk-store and generic copy-out paths)
for (Bh, ny, nx, cinh, na, nc, zo) in ((1, 12, 20, 64, 3, 80, 4), (1, 7, 13, 32, 3, 80, 3), (1, 9, 16, 96, 2, 3, 8)):
    no = nc + 5
    tin = ops.SplitTensor(Bh, ny, nx, cinh)
    ops.nchw_to_split(torch.randn(Bh, cinh, ny, nx, device='cuda'), tin.view())
    wh_ = (torch.randn(na * no, cinh, 1, 1) * (2.5 / cinh ** 0.5)).double()
    bh_ = (torch.randn(na * no) * 0.5).double()
    A = na * ny * nx + zo + 7
    wsh = ops.NmsWorkspace(Bh, A, nc)
    ops.nms_reset(wsh)
    zh = torch.zeros(Bh, A, no, device='cuda')
    wy, by = ops.pack_yolo_head_weights(wh_, bh_, na, no)
    yd = ops.yolo_decode_desc(na, no, torch.tensor([[10., 13.], [16., 30.], [33., 23.]][:na]), 8.0, zh, A, zo, wsh, 0.05, True)
    ops.ConvPlan(tin.view(), ops.CvbView(zh.data_ptr(), Bh, ny, nx, na * 128, na * 128, 0), wy, by, 1, 1, 0, 1, None, yolo=yd).run()
    ops.yolo_nms(zh, wsh, 0.05, 0.6, True, hist_ready=True)
torch.cuda.synchronize()
print('fused head ok')

# training kernels (SURVEY 8 f-3): conv forward / backward-data (+ SiLU' epilogue) / backward-weight, BatchNorm + SiLU passes, one C3 step
from cvpytorch_b200 import train as TR  # noqa: E402
for (Bt, Ht, Wt, ci, co, kk) in ((1, 8, 16, 64, 64, 1), (2, 9, 7, 128, 64, 3), (1, 8, 8, 64, 128, 3)):
    xt = torch.randn(Bt, Ht, Wt, ci, device='cuda').to(torch.bfloat16)
    dyt = torch.randn(Bt, Ht, Wt, co, device='cuda').to(torch.bfloat16)
    wf_, wb_ = TR.pack_weights(torch.randn(co, ci, kk, kk, device='cuda') * 0.05)
    TR.conv(xt, wf_, co, kk)
    TR.conv(dyt, wb_, ci, kk)
    TR.conv_wgrad(xt, dyt, kk)
for (Bt, Ht, Wt, ci, co) in ((1, 9, 14, 64, 64), (2, 8, 8, 64, 128)):  # stride 2: parity maps, four backward-data sub-convolutions
    xt = torch.randn(Bt, Ht, Wt, ci, device='cuda').to(torch.bfloat16)
    wf_, wb_ = TR.pack_weights(torch.randn(co, ci, 3, 3, device='cuda') * 0.05)
    yt = TR.conv(xt, wf_, co, 3, stride=2)
    TR.conv_dgrad_s2(yt, wb_, ci, Ht, Wt)
    TR.conv_wgrad(xt, yt, 3, stride=2)
mt = TR.CSPLayer(128, 128, n=1).cuda().train()
xt = torch.randn(1, 128, 8, 8, device='cuda', requires_grad=True)
mt(xt).sum().backward()
torch.cuda.synchronize()
print('training kernels ok')

# segmentation loss: forward + backward at x4, a non-integer ratio with a strided int32 label view, a downsample, a footprint larger than
# one shared-memory block (1 x 1 -> 200 x 300), an all-ignored batch and an out-of-range label
from cvpytorch_b200 import seg_train as ST  # noqa: E402
for (Bs, Cs, hs, ws_, Hs, Ws, dt) in ((2, 19, 8, 12, 32, 48, torch.uint8), (1, 5, 13, 29, 40, 61, torch.int32), (1, 3, 20, 28, 9, 11, torch.int64),
                                      (1, 2, 1, 1, 200, 300, torch.uint8)):
    ps = torch.randn(Bs, Cs, hs, ws_, device='cuda', requires_grad=True)
    ts = torch.randint(0, Cs, (Bs, Hs, Ws + 3), device='cuda').to(dt)[:, :, 1:Ws + 1]
    ST.CrossEntropyLoss2d()(ps, ts).backward()
    ST.CrossEntropyLoss2d()(ps, torch.full_like(ts, 255)).backward()
    ts[0, 0, 0] = Cs
    ST.CrossEntropyLoss2d()(ps, ts).backward()
torch.cuda.synchronize()
print('segmentation loss ok')
