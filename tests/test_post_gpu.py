"""Decode + batched NMS kernels (through the C ABI) against the oracle.
NMS: kept candidate indices / rows must be BIT-EXACT vs oracle.nms_oracle (pinned to the reference's
non_max_suppression + torchvision.ops.nms by tests/test_oracle_golden.py)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _nms_case(pred, conf=0.001, iou=0.6, multi_label=True, max_det=300):
    from cvpytorch_b200 import ops
    from oracle import nms_oracle as NO
    B, A, no = pred.shape
    ws = ops.NmsWorkspace(B, A, no - 5, max_det=max_det)
    det, idx, cnt = ops.yolo_nms(torch.from_numpy(pred).cuda(), ws, conf, iou, multi_label)
    torch.cuda.synchronize()
    assert int(ws.status[0]) == 0, 'candidate capacity overflow'
    det, idx, cnt = det.cpu().numpy(), idx.cpu().numpy(), cnt.cpu().numpy()
    ref = NO.non_max_suppression(pred, conf, iou, multi_label=multi_label, max_det=max_det)
    for b in range(B):
        rd, ri = ref[b]
        assert cnt[b] == rd.shape[0], f'image {b}: kept {cnt[b]} vs oracle {rd.shape[0]}'
        assert np.array_equal(idx[b, :cnt[b]].astype(np.int64), ri), f'image {b}: kept indices differ'
        assert np.array_equal(det[b, :cnt[b]], rd), f'image {b}: detection rows differ'


@pytest.mark.parametrize('regime', ['few', 'sparse', 'typical', 'capped'])
@pytest.mark.parametrize('multi_label', [True, False])
def test_nms_stress(cuda, regime, multi_label):
    from oracle import nms_oracle as NO
    pred = NO.make_stress_prediction(3, regime=regime, seed=2)
    _nms_case(pred, multi_label=multi_label)


def test_nms_empty_and_single(cuda):
    pred = np.zeros((2, 1000, 85), np.float32)  # no candidates at all
    _nms_case(pred)
    pred[1, 7, :4] = [100, 100, 50, 60]
    pred[1, 7, 4] = 0.9
    pred[1, 7, 5 + 3] = 0.8
    _nms_case(pred)


def test_nms_score_ties_and_iou_edge(cuda):
    """ties: equal scores keep candidate-index order; IoU == float32(0.6) is suppressed (double comparison)."""
    pred = np.zeros((1, 64, 85), np.float32)
    # two boxes with inter/union = 3/5 -> float32(0.6): second one must be suppressed at iou_thres=0.6
    pred[0, 0, :5] = [2.5, 0.5, 5, 1, 0.9]
    pred[0, 1, :5] = [1.5, 0.5, 3, 1, 0.8]
    pred[0, :2, 5] = 1.0
    # exact score ties, far apart
    for k in range(10):
        pred[0, 10 + k, :5] = [100 + 30 * k, 300, 20, 20, 0.5]
        pred[0, 10 + k, 5 + 7] = 0.5
    _nms_case(pred)


def test_nms_other_thresholds(cuda):
    from oracle import nms_oracle as NO
    pred = NO.make_stress_prediction(2, regime='typical', seed=4)
    _nms_case(pred, conf=0.25, iou=0.45, multi_label=False)
    _nms_case(pred, conf=0.05, iou=0.7, multi_label=True, max_det=100)


def test_nms_full_path_with_global_sort_steps(cuda):
    """Image 0: 10 000 copies of one box with distinct scores above a 20 x 20 grid of disjoint boxes.  The top ~3k candidates keep
    one box, so the image takes the full top-max_nms path, and its 10 400 candidates (> 2 x 4096) need the sort's grid-wide
    steps.  Image 1 holds the grid only and is finished by the top ~3k candidates."""
    pred = np.zeros((2, 10400, 85), np.float32)
    pred[0, :10000, :5] = [320, 320, 100, 100, 1.0]
    pred[0, :10000, 5] = np.linspace(0.5, 0.9, 10000, dtype=np.float32)
    gy, gx = np.divmod(np.arange(400), 20)
    pred[:, 10000:, 0] = 16 + 32 * gx
    pred[:, 10000:, 1] = 16 + 32 * gy
    pred[:, 10000:, 2:4] = 20
    pred[:, 10000:, 4] = 1.0
    pred[:, 10000:, 6] = np.linspace(0.1, 0.4, 400, dtype=np.float32)
    _nms_case(pred)


def test_output_side_rescale_clip_and_confusion_matrix(cuda):
    """SURVEY.md 8(f) rank 2: device-side box rescale/clip == the reference's numpy lines (yolov5.py:274-281) bit for bit;
    device confusion matrix == eval_segmentation.py:52-57 (np.bincount) exactly."""
    from cvpytorch_b200 import ops
    rng = np.random.default_rng(3)
    B, M = 5, 300
    rows = rng.uniform(-50, 700, size=(B, M, 6)).astype(np.float32)
    cnt = np.array([300, 0, 17, 299, 1], np.int32)
    pads = rng.uniform(0, 40, size=(B, 2)).astype(np.float32)
    scales = rng.uniform(0.3, 2.0, size=(B, 2)).astype(np.float32)
    wh = np.array([[640, 480], [1280, 720], [333, 500], [640, 640], [50, 60]], np.float32)
    out = ops.rescale_clip_boxes(torch.from_numpy(rows.copy()).cuda(), torch.from_numpy(cnt).cuda(), torch.from_numpy(pads).cuda(),
                                 torch.from_numpy(scales).cuda(), torch.from_numpy(wh).cuda()).cpu().numpy()
    for b in range(B):
        k = int(cnt[b])
        bb = rows[b, :k, :4].copy()              # the reference's lines, numpy float32
        bb[:, [0, 2]] -= pads[b, 1]
        bb[:, [1, 3]] -= pads[b, 0]
        bb[:, [0, 2]] /= scales[b, 1]
        bb[:, [1, 3]] /= scales[b, 0]
        bb[:, [0, 2]] = bb[:, [0, 2]].clip(0, np.array(int(wh[b, 0])))
        bb[:, [1, 3]] = bb[:, [1, 3]].clip(0, np.array(int(wh[b, 1])))
        assert np.array_equal(out[b, :k, :4], bb), b
        assert np.array_equal(out[b, k:], rows[b, k:]) and np.array_equal(out[b, :, 4:], rows[b, :, 4:])   # nothing else touched
    # confusion matrix with ignore labels (255, -1) and accumulation over two updates
    nc = 19
    gt = rng.integers(-1, 21, size=(3, 97, 131)).astype(np.int64)
    gt[gt == 20] = 255
    pr = rng.integers(0, nc, size=gt.shape).astype(np.int64)
    cm = ops.confusion_matrix(torch.from_numpy(gt).cuda(), torch.from_numpy(pr).cuda(), nc)
    cm = ops.confusion_matrix(torch.from_numpy(gt[:1]).cuda(), torch.from_numpy(pr[:1]).cuda(), nc, out=cm)

    def ref_matrix(g, p):
        mask = (g >= 0) & (g < nc)
        return np.bincount(nc * g[mask].astype('int') + p[mask], minlength=nc ** 2).reshape(nc, nc)
    assert np.array_equal(cm.cpu().numpy(), ref_matrix(gt, pr) + ref_matrix(gt[:1], pr[:1]))


def test_letterbox_on_device_equals_reference_resize(cuda):
    """cvb_letterbox_u8 (frames of different sizes in one launch) == the reference's Resize(keep_ratio=True) fixture, bit for bit
    (tests/golden/letterbox.npz: cv2.resize INTER_LINEAR + copyMakeBorder through the reference's own class), pads / scales included."""
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_oracle_golden import _letterbox_cases
    from cvpytorch_b200 import ops
    cases = _letterbox_cases()
    for size in sorted({c[1] for c in cases}):
        group = [c for c in cases if c[1] == size]
        frames = [torch.from_numpy(c[0]).cuda() for c in group]
        out, pads, scales = ops.letterbox_frames(frames, size=size, fill=(114, 114, 114))
        torch.cuda.synchronize()
        for i, (frame, _, p, s, check) in enumerate(group):
            assert check(out[i].cpu().numpy()), (size, frame.shape)
            assert tuple(int(v) for v in pads[i]) == p and abs(float(scales[i, 0]) - s) < 1e-6 * s


def test_letterbox_feeds_predict_frames(cuda):
    """camera frames of two sizes -> device letterbox -> YOLOv5.predict_frames == the reference-order pipeline on the oracle-letterboxed batch"""
    from cvpytorch_b200 import ops, synth
    from oracle import io_oracle as IO
    m = synth.build_yolov5s(True)
    rng = np.random.default_rng(9)
    frames = [rng.integers(0, 256, size=(96, 128, 3), dtype=np.uint8), rng.integers(0, 256, size=(150, 100, 3), dtype=np.uint8)]
    lb, pads, scales = ops.letterbox_frames([torch.from_numpy(f).cuda() for f in frames], size=(128, 128))
    ref = np.stack([IO.letterbox(f, (128, 128))[0] for f in frames])
    assert np.array_equal(lb.cpu().numpy(), ref)
    d0, i0, c0 = [t.clone() for t in m.predict_frames(lb)]
    d1, i1, c1 = m.predict_frames(torch.from_numpy(ref).cuda())
    assert torch.equal(c0, c1) and torch.equal(i0, i1) and torch.equal(d0, d1)


def test_coco_pack_on_device(cuda):
    from cvpytorch_b200 import ops
    from oracle import io_oracle as IO
    g = torch.Generator().manual_seed(12)
    B, M = 5, 300
    xy = torch.rand(B, M, 2, generator=g) * 500
    wh = torch.rand(B, M, 2, generator=g) * 120
    rows = torch.cat([xy, xy + wh, torch.rand(B, M, 1, generator=g), torch.randint(0, 80, (B, M, 1), generator=g).float()], 2).contiguous()
    count = torch.tensor([300, 0, 17, 1, 250], dtype=torch.int32)
    image_ids = [581929, 42, 139, 7, 100000]
    id2cat = list(range(1, 81))
    rec_ids, rec_box, total = ops.coco_pack(rows.cuda(), count.cuda(), image_ids, id2cat)
    torch.cuda.synchronize()
    n = int(total[0])
    ids, cats, xywh, sc = IO.coco_records(rows[:, :, :4].numpy(), rows[:, :, 4].numpy(), rows[:, :, 5].numpy(), count.tolist(), image_ids, id2cat)
    assert n == int(count.sum()) == ids.shape[0]
    assert np.array_equal(rec_ids[:n, 0].cpu().numpy(), ids) and np.array_equal(rec_ids[:n, 1].cpu().numpy(), cats)
    assert np.array_equal(rec_box[:n, :4].cpu().numpy(), xywh) and np.array_equal(rec_box[:n, 4].cpu().numpy(), sc)


def _ws_regions(ws, B, A):
    """(histogram u32 [B,16384], rowmax f32 [B,A]) views of an NmsWorkspace (layout: csrc/internal.h)."""
    al = lambda x, a: (x + a - 1) // a * a
    head = al(B * 16384 * 4, 256) + 6 * al(B * 4, 256)
    rm_off = head + B * (65536 + 4096) * 8
    off = ws.ws_ptr - ws.ws.data_ptr()
    raw = ws.ws[off:]
    hist = raw[:B * 16384 * 4].view(torch.int32).view(B, 16384)
    rowmax = raw[rm_off:rm_off + B * A * 4].view(torch.float32).view(B, A)
    return hist, rowmax


@pytest.mark.parametrize('B,ny,nx,cin,na,nc,z_off,multi', [
    (2, 12, 20, 64, 3, 80, 4, True),     # vector copy-out path (16-byte aligned runs)
    (3, 7, 13, 32, 3, 80, 3, False),     # odd map, misaligned z rows -> scalar copy-out, best-class histogram
    (2, 20, 20, 128, 3, 80, 0, True),    # the 20x20 level geometry (tile 20x6)
    (2, 9, 16, 96, 2, 3, 8, True),       # small `no` (8), two anchors
    (1, 80, 80, 128, 3, 80, 0, True),    # 80x80 level: tile 16x8, several tiles per CTA
])
def test_fused_head_conv_decode_equals_conv_then_decode(cuda, B, ny, nx, cin, na, nc, z_off, multi):
    """CVB_OUT_YOLO (decode as the conv epilogue) == fp32-out conv + cvb_yolo_decode, bit for bit: z rows, NMS histogram and per-row
    best scores; then the NMS that consumes them returns identical rows."""
    from cvpytorch_b200 import ops
    no = nc + 5
    g = torch.Generator().manual_seed(11 + cin + nx)
    x = torch.randn(B, cin, ny, nx, generator=g)
    w = (torch.randn(na * no, cin, 1, 1, generator=g) * (2.5 / cin ** 0.5)).double()
    b = (torch.randn(na * no, generator=g) * 0.5).double()
    tin = ops.SplitTensor(B, ny, nx, cin)
    ops.nchw_to_split(x.cuda(), tin.view())
    anchors_px = torch.tensor([[10., 13.], [16., 30.], [33., 23.]][:na])
    A = na * ny * nx + z_off + 7
    conf = 0.05
    # (a) two steps
    ws_a = ops.NmsWorkspace(B, A, nc)
    ops.nms_reset(ws_a)
    z_a = torch.zeros(B, A, no, device='cuda')
    cp = (na * no + 31) // 32 * 32
    raw = ops.F32Tensor(B, ny, nx, cp)
    wp, bp = ops.pack_conv_weights(w, b)
    ops.ConvPlan(tin.view(), raw.view(0, na * no), wp, bp, 1, 1, 0, 1, None).run()
    ops.yolo_decode(raw.view(0, na * no), na, no, anchors_px.cuda().contiguous(), 8.0, z_a, A, z_off, None, ws_a, conf, multi)
    # (b) fused
    ws_b = ops.NmsWorkspace(B, A, nc)
    ops.nms_reset(ws_b)
    z_b = torch.zeros(B, A, no, device='cuda')
    wy, by = ops.pack_yolo_head_weights(w, b, na, no)
    y = ops.yolo_decode_desc(na, no, anchors_px, 8.0, z_b, A, z_off, ws_b, conf, multi)
    ops.ConvPlan(tin.view(), ops.CvbView(z_b.data_ptr(), B, ny, nx, na * 128, na * 128, 0), wy, by, 1, 1, 0, 1, None, yolo=y).run()
    torch.cuda.synchronize()
    bad = (z_a != z_b).nonzero()
    assert bad.shape[0] == 0, (bad.shape[0], bad[:8].tolist(), bad[-4:].tolist())
    assert float(z_b[:, :z_off].abs().max() if z_off else 0.0) == 0.0 and float(z_b[:, z_off + na * ny * nx:].abs().max()) == 0.0
    ha, ra = _ws_regions(ws_a, B, A)
    hb, rb = _ws_regions(ws_b, B, A)
    assert int(ha.sum()) > 0
    assert torch.equal(ha, hb)
    assert torch.equal(ra[:, z_off:z_off + na * ny * nx], rb[:, z_off:z_off + na * ny * nx])
    da = [t.clone() for t in ops.yolo_nms(z_a, ws_a, conf, 0.6, multi, hist_ready=True)]
    db = [t.clone() for t in ops.yolo_nms(z_b, ws_b, conf, 0.6, multi, hist_ready=True)]
    torch.cuda.synchronize()
    for ta, tb in zip(da, db):
        assert torch.equal(ta, tb)
    assert int(da[2].sum()) > 0


def test_predict_fused_decode_equals_unfused(cuda, monkeypatch):
    """model.predict with the decode fused into the head convs (default) == the conv + cvb_yolo_decode graph (CVB_FUSED_DECODE=0)."""
    from cvpytorch_b200 import synth
    torch.manual_seed(5)
    x = torch.randn(3, 3, 160, 192).cuda()
    m1 = synth.build_yolov5s(calibrated=True)
    det1, idx1, cnt1 = [t.clone() for t in m1.predict(x)]
    z1 = m1._graph_for(x)['z'].clone()
    n1 = m1._graph_for(x)['g'].n_convs
    monkeypatch.setenv('CVB_FUSED_DECODE', '0')
    m2 = synth.build_yolov5s(calibrated=True)
    det2, idx2, cnt2 = [t.clone() for t in m2.predict(x)]
    z2 = m2._graph_for(x)['z'].clone()
    torch.cuda.synchronize()
    assert n1 == m2._graph_for(x)['g'].n_convs
    assert sum(1 for s in m1._graph_for(x)['g'].steps if s[0] == 'fn') + 3 == sum(1 for s in m2._graph_for(x)['g'].steps if s[0] == 'fn')
    assert torch.equal(z1, z2) and torch.equal(cnt1, cnt2) and torch.equal(idx1, idx2) and torch.equal(det1, det2)
    assert int(cnt1.sum()) > 0
