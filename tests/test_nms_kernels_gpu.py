"""The three NMS pipelines of csrc/nms.cu (two-phase YOLOv5 NMS, single-CTA YOLOX batched_nms, single-CTA FCOS top-k + NMS)
against oracle.nms_oracle / yolox_oracle / fcos_oracle at every capacity boundary, sort size, tie pattern and limit.

Rows, indices and counts are compared with np.array_equal: these kernels have no tolerance.  Inputs are constructed, not drawn:
scores come from bit patterns (histogram bin = fp32 bits >> 17), so the sort size, the threshold bin and the phase that finishes
an image are chosen by the test, and each test asserts from the workspace (`done` / `cnt` / `total` / `tbin`, `status`,
`det_count`) that it reached the path it is named after."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_post_gpu import _ws_regions  # noqa: E402

pytestmark = pytest.mark.gpu

BINS, CAP_B, CAP_A = 16384, 65536, 4096  # csrc/internal.h: kNmsBins, kNmsCap, kNmsCapA


# ------------------------------------------------------------------------------------------------ input builders
def ladder(spec, tie=1):
    """Scores in descending order from spec = [(histogram bin, count), ...]: bit pattern (bin << 17) | low, with distinct low bits
    inside a bin; with tie > 1 every `tie` consecutive candidates of a bin share one bit pattern."""
    parts = []
    for b, c in sorted(spec, reverse=True):
        step = max(1, (1 << 17) // c)
        low = ((c - 1 - np.arange(c)) // tie) * step
        parts.append((np.uint32(b) << np.uint32(17)) | low.astype(np.uint32))
    return np.concatenate(parts).view(np.float32)


def top_bin(scores, target):
    """The bin of the target-th best score, 0 when there are fewer: what top_bin_search must return."""
    bins = np.sort(np.asarray(scores, np.float32).view(np.uint32) >> 17)[::-1]
    return int(bins[target - 1]) if bins.size >= target else 0


def grid_xywh(k, cols=80):
    """Disjoint 20 x 20 boxes on a pitch of 32, numbered row by row."""
    gy, gx = np.divmod(np.asarray(k), cols)
    return np.stack([16 + 32 * gx, 16 + 32 * gy, 20 + 0 * gx, 20 + 0 * gx], -1).astype(np.float32)


def xyxy(xywh):
    xywh = np.asarray(xywh, np.float32)
    return np.concatenate([xywh[:, :2] - xywh[:, 2:] / 2, xywh[:, :2] + xywh[:, 2:] / 2], 1)


STACK = np.array([3000, 3000, 100, 100], np.float32)  # clear of grid_xywh(k < 6400)


def stack_and_grid(n, grid_ranks):
    """n boxes: one stack of identical boxes (all but the best of a class suppressed), disjoint grid boxes at `grid_ranks`."""
    boxes = np.tile(STACK, (n, 1))
    boxes[grid_ranks] = grid_xywh(np.arange(len(grid_ranks)))
    return boxes


def yolo_scene(scores, boxes, nc=4, A=None, cls=None):
    """One YOLOv5 image [A, 5 + nc]: the candidate of rank r (scores descending) has box boxes[r] (xywh), class cls[r] (default
    r % nc), objectness 1 and sits alone on an anchor row.  Rows are a fixed permutation of the ranks, so the order in which the
    kernels emit keys has nothing to do with the score order."""
    n = len(scores)
    A = A or n
    assert n <= A and np.gcd(7919, A) == 1
    r = np.arange(n)
    row = (r * 7919 + 13) % A
    pred = np.zeros((A, 5 + nc), np.float32)
    pred[row, :4] = boxes
    pred[row, 4] = 1.0
    pred[row, 5 + (r % nc if cls is None else cls)] = scores
    return pred


HEAD = [(8100 - i, 100) for i in range(32)]  # 3200 candidates, 100 per bin: the top 31 bins (3100) are phase A's key set


def big_scene(n, A=None, nc=4):
    """n candidates whose top ~3k keep fewer than max_det boxes, so the image needs the full path: 3200 in HEAD, the rest in fat
    bins below, one stack plus 250 grid boxes spread over all ranks (any misplaced key changes the kept list or the max_nms cut)."""
    rest, spec, b = n - 3200, list(HEAD), 8000
    while rest > 0:
        spec.append((b, min(rest, 65536)))
        rest, b = rest - 65536, b - 1
    return yolo_scene(ladder(spec), stack_and_grid(n, np.arange(7, n, max(n // 250, 1))[:250]), nc, A)


# ------------------------------------------------------------------------------------------------ YOLOv5 harness
def ws_regions(ws):
    """Views of every region of an NmsWorkspace: the histogram and rowmax of test_post_gpu._ws_regions, and the per-image slots and
    key arrays between them (carve_ws in csrc/nms.cu)."""
    B = ws.B
    al = lambda x, a: (x + a - 1) // a * a
    hist_bytes, slot = al(B * BINS * 4, 256), al(B * 4, 256)
    head = hist_bytes + 6 * slot
    raw = ws.ws[ws.ws_ptr - ws.ws.data_ptr():]
    r = dict(zip(('hist', 'rowmax'), _ws_regions(ws, B, ws.A)))
    for i, name in enumerate(('cntB', 'tbinB', 'cntA', 'tbinA', 'done', 'total')):
        r[name] = raw[hist_bytes + i * slot:hist_bytes + i * slot + B * 4].view(torch.int32)
    r['keysB'] = raw[head:head + B * CAP_B * 8].view(torch.int64).view(B, CAP_B)
    r['keysA'] = raw[head + B * CAP_B * 8:head + B * (CAP_B + CAP_A) * 8].view(torch.int64).view(B, CAP_A)
    return r


def run_yolo(pred, conf=0.001, iou=0.6, multi_label=True, max_det=300, max_nms=30000, ws=None, status=0):
    """cvb_yolo_nms on pred [B, A, 5 + nc] == the oracle, bit for bit (unless a capacity overflow is expected).  Returns the
    per-image phase state of the workspace, the status word and the kept counts."""
    from cvpytorch_b200 import ops
    from oracle import nms_oracle as NO
    B, A, no = pred.shape
    ws = ws or ops.NmsWorkspace(B, A, no - 5, max_det=max_det)
    det, idx, cnt = ops.yolo_nms(torch.from_numpy(pred).cuda(), ws, conf, iou, multi_label, max_nms=max_nms)
    torch.cuda.synchronize()
    reg = ws_regions(ws)
    st = {k: reg[k].cpu().numpy().astype(np.int64) for k in ('cntA', 'tbinA', 'cntB', 'tbinB', 'done', 'total')}
    st['status'], st['count'] = int(ws.status[0]), cnt.cpu().numpy().copy()
    assert st['status'] == status
    if status == 0:
        det, idx = det.cpu().numpy(), idx.cpu().numpy()
        ref = NO.non_max_suppression(pred, conf, iou, multi_label=multi_label, max_det=ws.max_det, max_nms=max_nms)
        for b in range(B):
            rd, ri = ref[b]
            k = st['count'][b]
            assert k == rd.shape[0], f'image {b}: kept {k} vs oracle {rd.shape[0]}'
            assert np.array_equal(idx[b, :k].astype(np.int64), ri), f'image {b}: kept indices differ'
            assert np.array_equal(det[b, :k], rd), f'image {b}: detection rows differ'
            assert (idx[b, k:] == -1).all() and not det[b, k:].any(), f'image {b}: rows past the count are not cleared'
    return st


# ------------------------------------------------------------------------------------------------ 1. sort sizes
@pytest.mark.parametrize('n', [4097, 8192, 8193, 16384, 32768, 32769, 65536])
def test_yolov5_phase_b_sort_size(cuda, n):
    """npad = 8192 (n = npad / 2 + 1 and n = npad) ... 65536 (n = 65536 is also the exact key capacity: no overflow status)."""
    st = run_yolo(big_scene(n)[None])
    assert st['cntA'][0] == 3100 and st['done'][0] == 0, 'phase A must run and leave the image to phase B'
    assert st['cntB'][0] == n == st['total'][0] and st['count'][0] < 300


def test_yolov5_phase_b_images_of_different_sort_size(cuda):
    """npad 16384, 65536 and 8192 next to an image phase A finished, in one cooperative sort."""
    A = 65536
    first = yolo_scene(ladder([(8100, 500)]), grid_xywh(np.arange(500)), A=A)  # 500 disjoint boxes: max_det in phase A
    st = run_yolo(np.stack([big_scene(9000, A), big_scene(40000, A), first, big_scene(65536, A), big_scene(5000, A)]))
    assert st['done'].tolist() == [0, 0, 1, 0, 0] and st['cntB'].tolist() == [9000, 40000, 0, 65536, 5000]
    assert st['count'][2] == 300


def test_yolov5_phase_b_more_sort_chunks_than_ctas(cuda):
    """10 images x 16 chunks of 4096 keys: more work items than the cooperative grid has CTAs, each CTA loops."""
    ns = [65536, 61441, 65536, 65000, 65536, 63000, 65536, 61441, 65536, 64000]
    st = run_yolo(np.stack([big_scene(n, 65536) for n in ns]))
    assert not st['done'].any() and st['cntB'].tolist() == ns
    assert sum((n + 4095) // 4096 for n in ns) > torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ 2. phase A -> phase B
@pytest.mark.parametrize('boxes,below,kept', [('stack', 2000, 144), ('stack', 0, 104), ('grid', 0, 300)])
def test_yolov5_phase_a_overflows_on_fat_threshold_bin(cuda, boxes, below, kept):
    """The bin that crosses 3072 holds 3000: 5000 keys > 4096, so phase A's key set is incomplete and it must give up without
    raising the status -- also when it counted every candidate of the image (below = 0), and when 4096 arbitrary keys of
    disjoint boxes would reach max_det ('grid')."""
    scores = ladder([(8100, 2000), (8090, 3000), (8000, below)][:3 if below else 2])
    n = 5000 + below
    st = run_yolo(yolo_scene(scores, stack_and_grid(n, np.arange(5, n, 50) if boxes == 'stack' else np.arange(n)))[None])
    assert st['tbinA'][0] == 8090 and st['cntA'][0] == 5000 > CAP_A and st['done'][0] == 0
    assert st['tbinB'][0] == 0 and st['cntB'][0] == n == st['total'][0] and st['count'][0] == kept


def test_yolov5_phase_a_final_when_it_saw_every_candidate(cuda):
    scores = ladder([(8100 - i, 100) for i in range(20)])
    st = run_yolo(yolo_scene(scores, np.tile(STACK, (2000, 1)))[None])
    assert st['cntA'][0] == 2000 == st['total'][0] and st['done'][0] == 1 and st['cntB'][0] == 0
    assert st['count'][0] == 4  # the best of each class


def test_yolov5_phase_a_final_at_max_det(cuda):
    scores = ladder([(8100 - i, 100) for i in range(100)])
    st = run_yolo(yolo_scene(scores, stack_and_grid(10000, np.arange(400)))[None])
    assert st['cntA'][0] == 3100 < st['total'][0] == 10000 and st['done'][0] == 1 and st['cntB'][0] == 0
    assert st['count'][0] == 300


@pytest.mark.parametrize('max_nms', [1, 100, 3071, 3072, 3500, 4096, 4097])
def test_yolov5_max_nms(cuda, max_nms):
    """Below 3072 max_nms is phase A's target too; from 3072 to 4096 and above it cuts inside / past phase A's key set."""
    scores = ladder([(8100 - i, 100) for i in range(60)])
    st = run_yolo(yolo_scene(scores, stack_and_grid(6000, np.arange(3, 6000, 37)))[None], max_nms=max_nms)
    assert st['tbinA'][0] == top_bin(scores, min(max_nms, 3072)) and st['tbinB'][0] == top_bin(scores, max_nms)
    assert st['done'][0] == 0 and st['cntB'][0] == (max_nms + 99) // 100 * 100
    assert st['count'][0] == min(max_nms, 4) + len(range(3, max_nms, 37))


def test_yolov5_max_nms_cuts_inside_a_run_of_equal_scores(cuda):
    """90 stacked boxes above 40 disjoint boxes of one score; max_nms = 100 admits the 10 tied boxes of lowest candidate id."""
    scores = np.concatenate([ladder([(8100, 90)]), np.full(40, 0.25, np.float32)])
    pred = yolo_scene(scores, stack_and_grid(130, np.arange(90, 130)), A=131)
    st = run_yolo(pred[None], max_nms=100)
    assert st['cntA'][0] == 130 == st['total'][0] and st['done'][0] == 1 and st['count'][0] == 4 + 10


# ------------------------------------------------------------------------------------------------ 3. capacity
def test_yolov5_one_key_past_capacity_raises_status(cuda):
    st = run_yolo(yolo_scene(ladder([(8000, 65537)]), np.tile(STACK, (65537, 1)))[None], status=1)
    assert st['cntB'][0] == 65537 > CAP_B and st['tbinB'][0] == 8000


def test_yolov5_more_candidates_than_capacity_below_the_threshold_bin(cuda):
    """93 200 candidates, but the bins from the threshold bin up hold 43 200: no overflow, exact result."""
    n = 93200
    scores = ladder(HEAD + [(8000, 40000), (7900, 50000)])
    st = run_yolo(yolo_scene(scores, stack_and_grid(n, np.arange(7, n, 300)))[None])
    assert st['total'][0] == n > CAP_B and st['tbinB'][0] == 8000 and st['cntB'][0] == 43200 and st['done'][0] == 0


# ------------------------------------------------------------------------------------------------ 4. top_bin_search
def _bin_case(t, at, above=((1, 50), (40, 50), (400, 50)), below=((1, 300), (33, 200))):
    return [(t + d, c) for d, c in above] + [(t, at)] + [(t - d, c) for d, c in below]


@pytest.mark.parametrize('name,spec,tbin,cnt', [
    ('lane_edge_512', _bin_case(7680, 100), 7680, 250),       # lowest bin of a lane of the top-down scan
    ('lane_top_511', _bin_case(7679, 100), 7679, 250),        # highest bin of the next lane
    ('segment_edge_32', _bin_case(7712, 100), 7712, 250),
    ('segment_top_31', _bin_case(7711, 100), 7711, 250),
    ('target_met_at_bin_edge', _bin_case(7700, 50), 7700, 200),
    ('top_populated_bin', [(8100, 300), (8000, 300)], 8100, 300),
    ('fewer_than_target', [(8100, 100), (7680, 50)], 0, 150),
])
def test_yolov5_threshold_bin(cuda, name, spec, tbin, cnt):
    scores = ladder(spec)
    n = len(scores)
    st = run_yolo(yolo_scene(scores, stack_and_grid(n, np.arange(2, n, 9)))[None], max_nms=200)
    assert tbin == top_bin(scores, 200)
    assert st['tbinA'][0] == tbin and st['cntA'][0] == cnt and st['total'][0] == n
    if cnt == n:
        assert st['done'][0] == 1
    else:
        assert st['done'][0] == 0 and st['tbinB'][0] == tbin and st['cntB'][0] == cnt


# ------------------------------------------------------------------------------------------------ 5. class counts
@pytest.mark.parametrize('multi_label', [True, False])
@pytest.mark.parametrize('nc', [1, 2, 31, 32, 33, 96, 97, 200])
def test_yolov5_class_count_sweep(cuda, nc, multi_label):
    from oracle import nms_oracle as NO
    pred = NO.make_stress_prediction(1 + nc % 3, A=3000, nc=nc, regime='capped', seed=nc)
    conf, iou = [(0.001, 0.6), (0.05, 0.45), (0.25, 0.7)][nc % 3]
    st = run_yolo(pred, conf=conf, iou=iou, multi_label=multi_label)
    assert (st['count'] > 0).all() and (st['total'] > 300).all()


@pytest.mark.parametrize('nc', [96, 97, 128, 200, 320])
def test_yolov5_every_class_of_every_row_is_a_candidate(cuda, nc):
    """70 disjoint boxes on neighbouring rows with every class above conf: each 64-row batch fills the emit stage completely
    (nc = 320 is the largest stage there is), and the best scores belong to the highest classes."""
    rows = 70
    pred = np.zeros((1, 100, 5 + nc), np.float32)
    pred[0, :rows, :4] = grid_xywh(np.arange(rows))
    pred[0, :rows, 4] = 1.0
    c, r = np.meshgrid(np.arange(nc), np.arange(rows))
    pred[0, :rows, 5:] = (0.1 + 0.8 * (c * rows + r) / (nc * rows)).astype(np.float32)
    st = run_yolo(pred)
    assert st['total'][0] == rows * nc and st['count'][0] == 300


def test_yolov5_best_class_ties_take_the_first_maximum(cuda):
    """multi_label off: equal class scores in one lane (5, 37), across lanes (40, 5), three ways, and after a smaller value."""
    ties = [(5, 37), (40, 5), (70, 6, 38), (79, 0), (33, 32, 31)]
    pred = np.zeros((1, 64, 85), np.float32)
    for i, t in enumerate(ties):
        pred[0, 3 * i, :5] = [*grid_xywh(i), 0.5 + 0.0625 * i]
        pred[0, 3 * i, 5:] = 0.25
        pred[0, 3 * i, 5 + np.array(t)] = 0.75
    from cvpytorch_b200 import ops
    ws = ops.NmsWorkspace(1, 64, 80)
    st = run_yolo(pred, multi_label=False, ws=ws)
    assert st['count'][0] == len(ties)
    assert sorted(ws.det[0, :len(ties), 5].cpu().tolist()) == sorted(float(min(t)) for t in ties)


# ------------------------------------------------------------------------------------------------ 6. greedy chunks
@pytest.mark.parametrize('max_det', [1, 511, 512, 513, 4096])
def test_yolov5_max_det(cuda, max_det):
    """5000 candidates in score order: ranks 0..599 are disjoint (512 survivors fill the first chunk and the kept list crosses
    into the second), and from rank 600 every tenth repeats a box kept 597 ranks -- one or two chunks -- earlier."""
    n, nc = 5000, 3
    r = np.arange(n)
    dup = (r >= 600) & (r % 10 == 3)
    src = np.where(dup, r - 597, r)  # 597 = 3 * 199: same class; r - 597 = 6 (mod 10) is never a repeat itself
    st = run_yolo(yolo_scene(ladder([(8100 - i, 100) for i in range(50)]), grid_xywh(src), nc)[None], max_det=max_det)
    assert st['count'][0] == max_det
    if max_det <= 513:
        assert st['done'][0] == 1 and st['cntB'][0] == 0
    else:
        assert st['done'][0] == 0 and st['cntB'][0] == n  # phase A's 3100 keys cannot hold 4096 boxes


def test_yolov5_iou_equal_to_threshold(cuda):
    """IoU 3/5 = float32(0.6) exceeds the double 0.6 (suppressed) but not the double float32(0.6); IoU 1/2 never exceeds 0.5."""
    pred = np.zeros((1, 16, 85), np.float32)
    pred[0, 0, :5] = [2.5, 0.5, 5, 1, 0.9]
    pred[0, 1, :5] = [1.5, 0.5, 3, 1, 0.8]
    pred[0, 2, :5] = [102, 100.5, 4, 1, 0.7]
    pred[0, 3, :5] = [101, 100.5, 2, 1, 0.6]
    pred[0, :4, 5] = 1.0
    for iou, kept in ((0.6, 3), (float(np.float32(0.6)), 4), (0.5, 3), (np.nextafter(0.5, 0), 2)):
        assert run_yolo(pred, iou=iou)['count'][0] == kept, iou


# ------------------------------------------------------------------------------------------------ 9. workspace reuse
def _bytes(*tensors):
    return [t.cpu().numpy().tobytes() for t in tensors]


def _thrice_identical(call, outputs):
    """The same call twice and once more as a CUDA-graph replay writes identical bytes to the cleared `outputs` (the order in
    which keys are emitted depends on atomics; the result must not)."""
    def run(launch):
        for t in outputs:
            t.zero_()
        launch()
        torch.cuda.synchronize()
        return _bytes(*outputs)

    first = run(call)
    assert run(call) == first
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call()
    assert run(g.replay) == first


def test_yolov5_workspace_reuse_and_replay(cuda):
    from cvpytorch_b200 import ops
    A = 65536
    ws = ops.NmsWorkspace(2, A, 4)
    big = np.stack([big_scene(65536, A), big_scene(40000, A)])
    tiny = np.stack([yolo_scene(ladder([(8100, 5)]), grid_xywh(np.arange(5)), A=A), np.zeros((A, 9), np.float32)])
    assert run_yolo(big, ws=ws)['done'].tolist() == [0, 0]
    st = run_yolo(tiny, ws=ws)  # stale keys, flags and kept-box scratch of the large set must not show
    assert st['done'].tolist() == [1, 1] and st['count'].tolist() == [5, 0] and st['cntB'].tolist() == [0, 0]
    assert run_yolo(big, ws=ws)['cntB'].tolist() == [65536, 40000]
    p = torch.from_numpy(big).cuda()
    _thrice_identical(lambda: ops.yolo_nms(p, ws), (ws.packed, ws.status))


# ------------------------------------------------------------------------------------------------ argument validation
def test_yolov5_rejected_arguments(cuda):
    from cvpytorch_b200 import ops
    from cvpytorch_b200._lib import CvbError

    def call(nc=4, max_det=300, shift=0, **kw):
        ws = ops.NmsWorkspace(1, 8, nc, max_det=max_det)
        ws.ws_ptr += shift
        ops.yolo_nms(torch.zeros((1, 8, 5 + nc), device='cuda'), ws, **kw)
        torch.cuda.synchronize()

    call(max_det=4096)
    call(nc=320)
    with pytest.raises(CvbError, match='nms: bad limits'):
        call(max_det=4097)
    with pytest.raises(CvbError, match='nms: bad limits'):
        call(max_nms=0)
    with pytest.raises(CvbError, match=r'nms: too many classes \(321\)'):
        call(nc=321)
    with pytest.raises(CvbError, match='nms: workspace must be 256-byte aligned'):
        call(shift=16)

    # a decode level must write inside z's rows: [z_off, z_off + rows) within [0, z_rows), rows = na * ny * nx (YOLOv5) or ny * nx (YOLOv6)
    na, no, ny, nx, A = 3, 85, 4, 5, 60
    anchors = torch.tensor([[10., 13.], [16., 30.], [33., 23.]])
    z = torch.zeros((1, A + 1, no), device='cuda')
    raw = ops.F32Tensor(1, ny, nx, 256)
    for off in (-1, 1):
        with pytest.raises(CvbError, match=rf"yolo_decode: level rows \[{off}, {off + A}\) outside z's {A} rows"):
            ops.yolo_decode(raw.view(0, na * no), na, no, anchors.cuda(), 8.0, z, A, off, None, None, 0.05, True)
    ops.yolo_decode(raw.view(0, na * no), na, no, anchors.cuda(), 8.0, z, A + 1, 1, None, None, 0.05, True)
    cls, reg = ops.F32Tensor(1, ny, nx, 96), ops.F32Tensor(1, ny, nx, 32)
    with pytest.raises(CvbError, match=r"yolov6_decode: level rows \[1, 21\) outside z's 20 rows"):
        ops.yolov6_decode(cls.view(0, 80), reg.view(0, 4), 80, 8.0, z[:, :20].contiguous(), 20, 1)
    tin = ops.SplitTensor(1, ny, nx, 64)
    wy, by = ops.pack_yolo_head_weights(torch.zeros(na * no, 64, 1, 1, dtype=torch.float64), torch.zeros(na * no, dtype=torch.float64), na, no)
    for off in (-1, 1):
        y = ops.yolo_decode_desc(na, no, anchors, 8.0, z, A, off)
        with pytest.raises(CvbError, match=rf"conv\(yolo\): level rows \[{off}, {off + A}\) outside z's {A} rows"):
            ops.ConvPlan(tin.view(), ops.CvbView(z.data_ptr(), 1, ny, nx, na * 128, na * 128, 0), wy, by, 1, yolo=y)
    ops.ConvPlan(tin.view(), ops.CvbView(z.data_ptr(), 1, ny, nx, na * 128, na * 128, 0), wy, by, 1, yolo=ops.yolo_decode_desc(
        na, no, anchors, 8.0, z, A + 1, 1))
    torch.cuda.synchronize()


# ================================================================================================ YOLOX
def xrec(boxes, scores, cls, A=None):
    """Candidate records [A, 8] of one image: objectness 1, class_conf = score, so obj * class_conf is the score bit for bit."""
    n = len(scores)
    rec = np.zeros((A or n, 8), np.float32)
    rec[:n, :4], rec[:n, 4], rec[:n, 5], rec[:n, 6], rec[:n, 7] = boxes, 1.0, scores, cls, scores
    return rec


def scattered(scores):
    """Distinct scores in a fixed non-monotone order: the location index says nothing about the rank."""
    scores = np.asarray(scores, np.float32)
    return scores[(np.arange(len(scores)) * 7919 + 13) % len(scores)] if np.gcd(7919, len(scores)) == 1 else scores[::-1].copy()


def run_yolox(recs, conf=0.01, iou=0.65, vanilla_above=1000, ws=None):
    from cvpytorch_b200 import ops
    from oracle import yolox_oracle as XO
    recs = np.asarray(recs, np.float32)
    B, A, _ = recs.shape
    ws = ws or ops.YoloxWorkspace(B, A)
    det, cnt = ops.yolox_nms(ws, conf, iou, vanilla_above, cand=torch.from_numpy(recs).cuda())
    torch.cuda.synchronize()
    det, cnt = det.cpu().numpy(), cnt.cpu().numpy().copy()
    for b in range(B):
        rows, _ = XO.nms_records(recs[b], conf, iou, vanilla_above)
        assert cnt[b] == rows.shape[0], f'image {b}: kept {cnt[b]} vs oracle {rows.shape[0]}'
        assert np.array_equal(det[b, :cnt[b]], rows), f'image {b}: rows differ'
    return cnt


def _switch_scene(n):
    """n candidates: n - 2 disjoint boxes of class 0, a class-1 box P that holds the largest coordinate m, and a class-2 box
    Q = P - (m + 1) with negative coordinates.  With the coordinate trick Q + 2 (m + 1) lands exactly on P + (m + 1) and is
    suppressed; class by class on the raw boxes it is kept."""
    boxes = np.concatenate([xyxy(grid_xywh(np.arange(n - 2))), [[2950, 2950, 3050, 3050], [-101, -101, -1, -1]]]).astype(np.float32)
    scores = scattered(ladder([(8100 - i, 50) for i in range(n // 50 + 1)])[:n])
    cls = np.concatenate([np.zeros(n - 2), [1, 2]])
    return xrec(boxes, scores, cls, A=n + 24)


@pytest.mark.parametrize('n,kept', [(1000, 999), (1001, 1001)])
def test_yolox_coordinate_trick_up_to_vanilla_above_then_per_class(cuda, n, kept):
    assert run_yolox(_switch_scene(n)[None], vanilla_above=1000)[0] == kept
    assert run_yolox(_switch_scene(n)[None], vanilla_above=n - 1)[0] == n  # the same set one past its own limit: per class
    assert run_yolox(_switch_scene(n)[None], vanilla_above=n)[0] == n - 1


def test_yolox_vanilla_classes_that_share_a_chain(cuda):
    """Per-class mode: classes 5, 1029, 2053, 3077 hash to one chain of kept boxes.  One box X carries all four, in the first
    chunk (3077 beside 5) and after 600 disjoint boxes (1029, 2053, and a second class-5 copy that the chain walk must drop)."""
    X = [2950, 2950, 3050, 3050]
    boxes = np.concatenate([[X, X], xyxy(grid_xywh(np.arange(600))), [X, X, X]]).astype(np.float32)
    cls = np.concatenate([[5, 3077], np.full(600, 7), [1029, 5, 2053]])
    rec = xrec(boxes, ladder([(8100, 605)]), cls)
    assert run_yolox(rec[None], vanilla_above=10)[0] == 604


@pytest.mark.parametrize('vanilla_above', [1000, 100000])
def test_yolox_one_class_holds_everything(cuda, vanilla_above):
    """2000 candidates of class 3; past rank 700 every third repeats the box 700 ranks (one or two chunks) earlier, which is never
    a repeat itself (r - 700 = 2 mod 3)."""
    r = np.arange(2000)
    src = np.where((r >= 700) & (r % 3 == 0), r - 700, r)
    rec = xrec(xyxy(grid_xywh(src)), ladder([(8100 - i, 100) for i in range(20)]), np.full(2000, 3))
    assert run_yolox(rec[None], vanilla_above=vanilla_above)[0] == len(np.unique(src))


def test_yolox_score_equal_to_conf_is_a_candidate(cuda):
    below = np.nextafter(np.float32(0.25), np.float32(0))
    scores = np.array([0.25, below, 0.5, 0.25, below, 0.2500001], np.float32)
    rec = xrec(xyxy(grid_xywh(np.arange(6))), scores, np.arange(6))
    assert run_yolox(rec[None], conf=0.25)[0] == 4


@pytest.mark.parametrize('vanilla_above', [1000, 100000])
@pytest.mark.parametrize('A', [1, 2, 511, 512, 513, 16384])
def test_yolox_every_location_passes(cuda, A, vanilla_above):
    """All A locations are candidates (16384 fills the key array); boxes repeat with period 2048, classes with period 4."""
    k = np.arange(A)
    scores = scattered(ladder([(8100 - i, 128) for i in range(128)])[:A])
    rec = xrec(xyxy(grid_xywh(k % 2048, 128)), scores, (k % 2048) % 4)
    assert run_yolox(rec[None], vanilla_above=vanilla_above)[0] == min(A, 2048)


def test_yolox_equal_scores_across_classes(cuda):
    """Runs of 8 equal scores over 4 classes, the boxes in identical pairs: of a tied same-class pair the lower location wins."""
    k = np.arange(64)
    rec = xrec(xyxy(grid_xywh(k // 2)), ladder([(8100, 64)], tie=8), (k // 2) % 4)
    for vanilla_above in (10, 1000):
        det_n = run_yolox(rec[None], vanilla_above=vanilla_above)
        assert det_n[0] == 32


def test_yolox_workspace_reuse_and_replay(cuda):
    from cvpytorch_b200 import ops
    A = 4096
    k = np.arange(A)
    big = xrec(xyxy(grid_xywh(k % 1500, 128)), scattered(ladder([(8100 - i, 128) for i in range(32)])), (k % 1500) % 4)
    tiny = xrec(xyxy(grid_xywh(np.arange(3))), ladder([(8100, 3)]), np.arange(3), A=A)
    ws = ops.YoloxWorkspace(2, A)
    assert run_yolox(np.stack([big, big[::-1]]), ws=ws).tolist() == [1500, 1500]
    assert run_yolox(np.stack([tiny, np.zeros_like(tiny)]), ws=ws).tolist() == [3, 0]
    c = torch.from_numpy(np.stack([big, tiny])).cuda()
    _thrice_identical(lambda: ops.yolox_nms(ws, 0.01, 0.65, cand=c), (ws.det, ws.count))


def test_yolox_rejected_arguments(cuda):
    from cvpytorch_b200 import ops
    from cvpytorch_b200._lib import CvbError
    with pytest.raises(CvbError, match=r'yolox_nms: at most 16384 locations per image \(got 16385\)'):
        ops.yolox_nms(ops.YoloxWorkspace(1, 16385), 0.01, 0.65)
    ws = ops.YoloxWorkspace(1, 64)
    with pytest.raises(CvbError, match='yolox_nms: candidate records must be 16-byte aligned'):
        ops.yolox_nms(ws, 0.01, 0.65, cand=torch.zeros(64 * 8 + 1, device='cuda')[1:].view(1, 64, 8))


# ================================================================================================ FCOS
def run_fcos(s, c, b, score_thres=0.05, iou_thres=0.6, topk=1000, ws=None, status=0):
    """cvb_fcos_nms on scores [B, N], classes [B, N] (1-based), boxes [B, N, 4] == the oracle's post_process, bit for bit."""
    from cvpytorch_b200 import ops
    from oracle import fcos_oracle as FO
    s, c, b = np.asarray(s, np.float32), np.asarray(c, np.int32), np.asarray(b, np.float32)
    B, N = s.shape
    ws = ws or ops.FcosWorkspace(B, N, topk)
    out = ops.fcos_nms(ws, score_thres, iou_thres, torch.from_numpy(s).cuda(), torch.from_numpy(c).cuda(), torch.from_numpy(b).cuda())
    torch.cuda.synchronize()
    assert int(ws.status[0]) == status
    osc, ocl, obx, oloc, ocnt = (t.cpu().numpy() for t in out)
    if status == 0:
        for i in range(B):
            rs, rc, rb, rl = FO.post_process(s[i], c[i], b[i], score_thres, iou_thres, ws.topk)
            k = ocnt[i]
            assert k == rs.shape[0], f'image {i}: kept {k} vs oracle {rs.shape[0]}'
            assert np.array_equal(oloc[i, :k].astype(np.int64), rl), f'image {i}: kept locations differ'
            assert np.array_equal(osc[i, :k], rs) and np.array_equal(ocl[i, :k], rc) and np.array_equal(obx[i, :k], rb)
            assert (oloc[i, k:] == -1).all() and not osc[i, k:].any()
    return ocnt.copy()


def fcos_scene(N, scores=None, period=6000, ncls=5):
    """N locations with scattered distinct scores; boxes are disjoint and repeat with `period`, classes (1-based) with ncls."""
    k = np.arange(N)
    s = scattered(ladder([(8100 - i, 200) for i in range((N + 199) // 200)])[:N] if scores is None else scores)
    return s, 1 + (k % period) % ncls, xyxy(grid_xywh(k % period))


@pytest.mark.parametrize('topk', [1, 7, 1000, 2048])
def test_fcos_topk(cuda, topk):
    """N = 20000 > the 4096 keys of the selection; every score passes the threshold, so topk candidates reach the NMS."""
    s, c, b = fcos_scene(20000)
    cnt = run_fcos(s[None], c[None], b[None], topk=topk)
    assert 0 < cnt[0] <= topk and (topk > 7 or cnt[0] == topk)


@pytest.mark.parametrize('N', [1, 300])
def test_fcos_fewer_locations_than_topk(cuda, N):
    s, c, b = fcos_scene(N, period=200)
    assert run_fcos(s[None], c[None], b[None])[0] == min(N, 200)


def test_fcos_score_equal_to_threshold_is_a_candidate(cuda):
    below = np.nextafter(np.float32(0.25), np.float32(0))
    s = np.array([0.25, below, 0.5, 0.25, below, 0.2500001, 0.0, 0.1], np.float32)
    assert run_fcos(s[None], np.ones((1, 8)), xyxy(grid_xywh(np.arange(8)))[None], score_thres=0.25)[0] == 4


def test_fcos_iou_equal_to_threshold_is_kept(cuda):
    """Boxes (0,0,9,4) and (5,0,14,4): '+1' areas 50 each, intersection 16, IoU = 16/84 in float32."""
    thr = float(np.float32(16) / (np.float32(50) + np.float32(50) - np.float32(16)))
    b = np.array([[[0, 0, 9, 4], [5, 0, 14, 4]]], np.float32)
    s, c = np.array([[0.9, 0.8]], np.float32), np.zeros((1, 2))
    assert run_fcos(s, c, b, iou_thres=thr)[0] == 2
    assert run_fcos(s, c, b, iou_thres=float(np.nextafter(np.float32(thr), np.float32(0))))[0] == 1


def test_fcos_class_offset_from_the_candidates_only(cuda):
    """P (class 1) holds the candidates' largest coordinate m = 200, Q = P - 201 (class 2) lands on it once the class offsets are
    added and is suppressed.  A box below the score threshold and one outside the top-k carry larger coordinates."""
    b = np.array([[[150, 150, 200, 200], [-51, -51, -1, -1], [0, 0, 5000, 5000], [0, 0, 7000, 7000]]], np.float32)
    s, c = np.array([[0.9, 0.8, 0.01, 0.7]], np.float32), np.array([[1, 2, 3, 4]])
    assert run_fcos(s, c, b, topk=3)[0] == 3  # 0.7 is the third candidate: m = 7000, Q is clear of P
    assert run_fcos(s, c, b, topk=2)[0] == 1  # candidates P and Q only
    s[0, 3] = 0.02
    assert run_fcos(s, c, b, topk=3)[0] == 1  # neither large box passes the score threshold


@pytest.mark.parametrize('fat,status', [(3196, 0), (3197, 1)])
def test_fcos_selection_capacity(cuda, fat, status):
    """900 scores above a threshold bin of `fat` scores in runs of 16 equal ones: 4096 selected keys fit, 4097 raise the status.
    topk = 1000 cuts inside a run, where the lower location wins."""
    s = ladder([(8100, 900), (8000, fat), (7900, 2000)], tie=16)
    s, c, b = fcos_scene(len(s), s, period=len(s))
    cnt = run_fcos(s[None], c[None], b[None], status=status)
    assert status or cnt[0] == 1000


@pytest.mark.parametrize('N,status', [(4096, 0), (4097, 1)])
def test_fcos_equal_scores_are_one_fat_threshold_bin(cuda, N, status):
    """A map of equal scores (here 0, below the score threshold) is selected whole: one location past 4096 raises the status."""
    assert run_fcos(np.zeros((1, N)), np.ones((1, N)), xyxy(grid_xywh(np.arange(N)))[None], status=status)[0] == 0


def test_fcos_nan_negative_and_negative_zero_scores(cuda):
    """NaN and negative scores are never selected; -0.0 is the score 0: it passes a threshold of 0 in location order with +0.0
    and sorts below every positive score."""
    N = 3000
    s, c, b = fcos_scene(N)
    s[5::60] = -0.0
    s[7::60] = 0.0
    s[11::60] = np.nan
    s[13::60] = -0.5
    s[17::60] = -np.inf
    assert run_fcos(s[None], c[None], b[None])[0] == 1000  # 50 scores of -0.0 must not displace the top 1000
    few = slice(0, 600)  # fewer than topk: the zeros are candidates at threshold 0
    assert run_fcos(s[None, few], c[None, few], b[None, few], score_thres=0.0)[0] == 600 - 30
    assert run_fcos(s[None, few], c[None, few], b[None, few], score_thres=0.05)[0] == 600 - 50


def test_fcos_workspace_reuse_and_replay(cuda):
    from cvpytorch_b200 import ops
    N = 8000
    s, c, b = fcos_scene(N, period=N)
    ws = ops.FcosWorkspace(2, N, 1000)
    assert run_fcos(np.stack([s, s[::-1]]), np.stack([c, c]), np.stack([b, b]), ws=ws).tolist() == [1000, 1000]
    s2 = np.full((2, N), -1.0, np.float32)  # (N equal scores of 0 would be one fat threshold bin: a capacity overflow)
    s2[0, [5, 4000, 7999]] = [0.5, 0.75, 0.625]
    assert run_fcos(s2, np.stack([c, c]), np.stack([b, b]), ws=ws).tolist() == [3, 0]
    ts, tc, tb = torch.from_numpy(np.stack([s, s2[0]])).cuda(), torch.from_numpy(np.stack([c, c]).astype(np.int32)).cuda(), \
        torch.from_numpy(np.stack([b, b])).cuda()
    _thrice_identical(lambda: ops.fcos_nms(ws, 0.05, 0.6, ts, tc, tb),
                      (ws.out_scores, ws.out_classes, ws.out_boxes, ws.out_loc, ws.out_count, ws.status))


def test_fcos_rejected_arguments(cuda):
    from cvpytorch_b200 import ops
    from cvpytorch_b200._lib import CvbError
    ok, big, ws = ops.FcosWorkspace(1, 64, 2048), ops.FcosWorkspace(1, 64, 2049), ops.FcosWorkspace(1, 64, 10)
    ops.fcos_nms(ok)
    with pytest.raises(CvbError, match=r'fcos_nms: bad sizes \(topk <= 2048\)'):
        ops.fcos_nms(big)
    with pytest.raises(CvbError, match='fcos_nms: box arrays must be 16-byte aligned'):
        ops.fcos_nms(ws, boxes=torch.zeros(64 * 4 + 1, device='cuda')[1:].view(1, 64, 4))
    torch.cuda.synchronize()
