"""COCO box mAP without a GPU: hand-derived cases against the COCOeval oracle (each with its derivation), the optional comparison with
pycocotools, the drop-in CocoEvaluator's refusals before any launch, the host checks of the C ABI, and the record rules (the rank merge and
the within-batch "last wins")."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import coco_eval_oracle as O  # noqa: E402

ONE = 1 / (1 + np.spacing(1))  # precision of a lone true positive: tp / (tp + fp + 2^-52)


def _one(x):
    # a statistic is np.mean over many entries equal to ONE: the pairwise sum may round it by an ulp
    return abs(x - ONE) <= 2e-16


def _gt(anns, cats=(1,), images=(1,)):
    out = {'images': [{'id': i} for i in images], 'categories': [{'id': c} for c in cats], 'annotations': []}
    for n, a in enumerate(anns):
        box = a['bbox']
        out['annotations'].append(dict(id=a.get('id', n + 1), image_id=a.get('image_id', 1), category_id=a.get('category_id', 1), bbox=box,
                                       area=a.get('area', box[2] * box[3]), iscrowd=a.get('iscrowd', 0)))
    return out


def _run(gt, results, img_ids=(1,)):
    return O.coco_eval(gt, [(r[0], r[1], r[2], r[3]) for r in results], list(img_ids))


def test_parameters_are_cocoeval_defaults():
    assert O.IOU_THRS.tolist()[0] == .5 and O.IOU_THRS.tolist()[5] == .75 and len(O.IOU_THRS) == 10
    assert len(O.REC_THRS) == 101 and O.REC_THRS[0] == 0 and O.REC_THRS[-1] == 1
    assert O.AREA_RNG == [[0, 1e10], [0, 1024], [1024, 9216], [9216, 1e10]] and O.MAX_DETS == [1, 10, 100]


def test_identical_detection_scores_one_over_one_plus_eps():
    # tp = 1, fp = 0: pr = 1 / (1 + 2^-52) = 0.9999999999999998 at every recall threshold (rc = 1); the box is 10x10 (small), so
    # medium / large have no ground truth and stay -1
    r = _run(_gt([{'bbox': [0, 0, 10, 10]}]), [(1, 1, [0, 0, 10, 10], .9)])
    assert ONE == 0.9999999999999998
    s = r['stats']
    assert np.all(r['precision'][:, :, 0, :2, :] == ONE) and np.all(r['precision'][:, :, 0, 2:, :] == -1)
    assert all(_one(x) for x in s[:4])
    assert s[4] == s[5] == -1 and s[10] == s[11] == -1
    assert s[6] == s[7] == s[8] == s[9] == 1.0


def test_false_positive_ranked_first_gives_exactly_one_half():
    # scores .9 (miss), .8 (hit): tp = [0, 1], fp = [1, 1]; pr = [0, 1 / (2 + 2^-52)] and 2 + 2^-52 rounds to 2, so pr[1] = .5; the
    # envelope lifts pr[0] to .5 and every recall threshold reads .5
    r = _run(_gt([{'bbox': [0, 0, 10, 10]}]), [(1, 1, [50, 50, 10, 10], .9), (1, 1, [0, 0, 10, 10], .8)])
    assert r['stats'][0] == r['stats'][1] == .5
    assert np.all(r['precision'][:, :, 0, 0, 2] == .5)


def test_iou_exactly_half_matches_only_at_the_first_threshold():
    # [0,0,10,10] vs [0,0,10,5]: w*h = 50, union 100 + 50 - 50 = 100, IoU = .5 exactly: matched at t = .5 only
    r = _run(_gt([{'bbox': [0, 0, 10, 10]}]), [(1, 1, [0, 0, 10, 5], .9)])
    assert O.bb_iou([[0, 0, 10, 5]], [[0, 0, 10, 10]], [False])[0, 0] == .5
    s = r['stats']
    assert _one(s[1]) and s[2] == 0
    assert s[0] == pytest.approx(.1, abs=1e-15)
    m = r['evals'][1, 0, 1]['dtMatches'][:, 0]
    assert m[0] == 1 and not m[1:].any()


def test_detection_on_a_crowd_is_ignored_not_a_false_positive():
    # the crowd ground truth matches both of its detections (it is never used up) and both take its ignore flag, so they count in
    # neither tp nor fp and the lone true positive keeps AP = 1 / (1 + eps)
    gt = _gt([{'bbox': [0, 0, 10, 10], 'id': 7}, {'bbox': [100, 100, 50, 50], 'iscrowd': 1, 'id': 9}])
    r = _run(gt, [(1, 1, [100, 100, 50, 50], .95), (1, 1, [110, 110, 20, 20], .93), (1, 1, [0, 0, 10, 10], .9)])
    e = r['evals'][1, 0, 1]
    assert (e['dtMatches'][0] == [9, 9, 7]).all()
    assert e['dtIgnore'][0].tolist() == [True, True, False]
    assert _one(r['stats'][0])
    # crowd IoU divides by the detection area: 20x20 inside 50x50 -> 1
    assert O.bb_iou([[110, 110, 20, 20]], [[100, 100, 50, 50]], [True])[0, 0] == 1.0
    # without the crowd flag the second detection on it is a false positive
    r2 = _run(_gt([{'bbox': [0, 0, 10, 10]}, {'bbox': [100, 100, 50, 50]}]),
              [(1, 1, [100, 100, 50, 50], .95), (1, 1, [110, 110, 20, 20], .93), (1, 1, [0, 0, 10, 10], .9)])
    assert r2['stats'][0] < .99


def test_ground_truth_of_area_exactly_1024_is_small_and_medium():
    # area bounds are inclusive: 1024 lies in [0, 1024] and in [1024, 9216]
    r = _run(_gt([{'bbox': [0, 0, 32, 32], 'area': 1024.0}]), [(1, 1, [0, 0, 32, 32], .9)])
    assert _one(r['stats'][3]) and _one(r['stats'][4]) and r['stats'][5] == -1
    # the area field, not the box, decides: a 32x32 box whose area says 9217 is large only, and the detection (area 1024) that matches
    # it counts in 'large' although its own area is outside the range
    r = _run(_gt([{'bbox': [0, 0, 32, 32], 'area': 9217.0}]), [(1, 1, [0, 0, 32, 32], .9)])
    assert r['stats'][3] == r['stats'][4] == -1 and _one(r['stats'][5])
    # an unmatched detection outside the range is ignored there: a miss of area 1024 leaves 'large' untouched
    r = _run(_gt([{'bbox': [0, 0, 32, 32], 'area': 9217.0}]), [(1, 1, [500, 0, 32, 32], .95), (1, 1, [0, 0, 32, 32], .9)])
    assert _one(r['stats'][5]) and r['stats'][0] < .99


def test_last_of_two_tied_ground_truths_wins():
    # [2.5,0,10,10] overlaps [0,0,10,10] and [5,0,10,10] by 75 each, union 125: equal IoU .6, the later ground truth is taken
    gt = _gt([{'bbox': [0, 0, 10, 10], 'id': 3}, {'bbox': [5, 0, 10, 10], 'id': 4}])
    iou = O.bb_iou([[2.5, 0, 10, 10]], [[0, 0, 10, 10], [5, 0, 10, 10]], [False, False])
    assert iou[0, 0] == iou[0, 1]
    r = _run(gt, [(1, 1, [2.5, 0, 10, 10], .9)])
    assert r['evals'][1, 0, 1]['dtMatches'][0, 0] == 4


def test_ignore_field_is_overwritten_by_iscrowd_and_images_come_from_the_update():
    # an 'ignore' key does not make a ground truth ignored; an image that was never passed to update does not count its ground truth
    gt = _gt([{'bbox': [0, 0, 10, 10]}, {'bbox': [0, 0, 10, 10], 'image_id': 2}], images=(1, 2))
    gt['annotations'][0]['ignore'] = 1
    r = _run(gt, [(1, 1, [0, 0, 10, 10], .9)], img_ids=(1,))
    assert _one(r['stats'][0])
    r = _run(gt, [(1, 1, [0, 0, 10, 10], .9)], img_ids=(1, 2))
    assert r['stats'][8] == .5


def test_more_than_100_detections_are_cut_after_the_score_sort():
    gt = _gt([{'bbox': [0, 0, 10, 10]}])
    res = [(1, 1, [200 + i, 0, 10, 10], .5) for i in range(120)] + [(1, 1, [0, 0, 10, 10], .4)]
    r = _run(gt, res)
    assert len(r['evals'][1, 0, 1]['dtScores']) == 100 and r['stats'][0] == 0
    # ties keep input order (mergesort): the first 100 of the .5 detections survive
    assert r['evals'][1, 0, 1]['dtOrder'].tolist() == list(range(100))


def test_pycocotools_agrees_with_the_oracle():
    pytest.importorskip('pycocotools')
    from pycocotools.coco import COCO
    from pycocotools.cocoeval import COCOeval
    gt, results, img_ids = random_case(np.random.default_rng(5), n_img=12, n_cat=4)
    coco = COCO()
    coco.dataset = gt
    coco.createIndex()
    dt = coco.loadRes([dict(image_id=i, category_id=c, bbox=b, score=s) for i, c, b, s in results])
    E = COCOeval(coco, dt, 'bbox')
    E.params.imgIds = img_ids
    E.evaluate()
    E.accumulate()
    E.summarize()
    r = O.coco_eval(gt, results, img_ids)
    assert np.array_equal(E.eval['precision'], r['precision']) and np.array_equal(E.eval['recall'], r['recall'])
    assert np.allclose(E.stats, r['stats'], rtol=0, atol=1e-12)


def random_case(rng, n_img, n_cat, dets_per_img=30, crowd=0.1):
    """A seeded COCO-format GT and result records on an integer grid (exact-threshold IoUs happen), with score ties."""
    cats = sorted(rng.choice(np.arange(1, 4 * n_cat), n_cat, replace=False).tolist())
    gt = {'images': [{'id': int(i)} for i in range(1, n_img + 1)], 'categories': [{'id': int(c)} for c in cats], 'annotations': []}
    aid = 1
    results = []
    for img in range(1, n_img + 1):
        boxes = []
        for _ in range(int(rng.integers(0, 8))):
            x, y = rng.integers(0, 200, 2)
            w, h = rng.integers(1, 120, 2)
            c = int(rng.choice(cats))
            area = float(w * h) if rng.random() > .2 else float(rng.choice([1024, 9216, w * h + .5]))
            gt['annotations'].append(dict(id=aid, image_id=img, category_id=c, bbox=[float(x), float(y), float(w), float(h)], area=area,
                                          iscrowd=int(rng.random() < crowd)))
            boxes.append((c, x, y, w, h))
            aid += 1
        for _ in range(int(rng.integers(0, dets_per_img))):
            if boxes and rng.random() < .7:
                c, x, y, w, h = boxes[int(rng.integers(len(boxes)))]
                x, y = x + int(rng.integers(-4, 5)), y + int(rng.integers(-4, 5))
                w, h = max(1, w + int(rng.integers(-4, 5))), max(1, h + int(rng.integers(-4, 5)))
            else:
                c, x, y, w, h = int(rng.choice(cats)), *rng.integers(0, 200, 2), *rng.integers(1, 120, 2)
            results.append((img, int(c), [float(x), float(y), float(w), float(h)], float(np.float32(rng.integers(1, 20) / 20))))
    return gt, results, list(range(1, n_img + 1))


# ----------------------------------------------------------------------------------------------- drop-in refusals and record rules
class _Coco:
    def __init__(self, d):
        self.dataset = d


class _Dataset:
    def __init__(self, gt, id2category=None):
        self.coco = _Coco(gt)
        if id2category is not None:
            self.id2category = id2category


def _out(boxes, scores, labels):
    return {'boxes': torch.tensor(boxes, dtype=torch.float32).reshape(-1, 4), 'scores': torch.tensor(scores, dtype=torch.float32),
            'labels': torch.tensor(labels, dtype=torch.float32)}


def test_refusals_are_raised_before_any_launch():
    from cvpytorch_b200.coco_eval import CocoEvaluator
    gt = _gt([{'bbox': [0, 0, 10, 10]}], cats=(1, 3))
    for types in (['segm'], ['bbox', 'segm'], ['keypoints'], []):
        with pytest.raises(NotImplementedError):
            CocoEvaluator(_Dataset(gt), types)
    bad = _gt([{'bbox': [0, 0, 10, 10], 'id': 0}])
    with pytest.raises(ValueError, match='> 0'):
        CocoEvaluator(_Dataset(bad), ['bbox'])
    ev = CocoEvaluator(_Dataset(gt, {0: 1, 1: 3}), ['bbox'])
    assert ev.evaluate() is None  # no update: the reference returns None as well
    with pytest.raises(AssertionError, match='coco set'):
        ev.update([{'image_id': torch.tensor(42)}], [_out([[0, 0, 5, 5]], [.5], [0])])
    with pytest.raises(KeyError):
        ev.update([{'image_id': torch.tensor(1)}], [_out([[0, 0, 5, 5], [1, 1, 4, 4]], [.5, .4], [0, 2])])
    with pytest.raises(KeyError):
        ev.update([{'image_id': torch.tensor(1)}], [_out([[0, 0, 5, 5]], [.5], [0.5])])
    with pytest.raises(ValueError, match='NaN'):
        ev.update([{'image_id': torch.tensor(1)}], [_out([[0, 0, 5, 5]], [float('nan')], [0])])
    assert ev.count == 0 and not ev._seen and not ev._chunks
    assert ev.evaluate() is None
    # an unknown image without detections is not an error (the reference's loadRes only checks result records)
    ev.update([{'image_id': torch.tensor(42)}], [_out([], [], [])])
    assert ev.count == 1 and not ev._images
    assert ev.metric_names == O.METRIC_NAMES


def test_within_batch_last_wins_and_rank_merge_first_wins():
    from cvpytorch_b200.coco_eval import batch_outputs, merge_rank_images
    assert batch_outputs([{'image_id': torch.tensor(v)} for v in (3, 5, 3, 7, 5)]) == [(3, 2), (5, 4), (7, 3)]
    ranks = [[1, 2, 3], [2, 4], [4, 5, 1], []]
    assert merge_rank_images(ranks) == [[1, 2, 3], [4], [5], []]
    # the same rule as the oracle's merge of the reference's gathered records
    recs = [(list(r), [(i, 1, [0, 0, 1, 1], float(n)) for i in r]) for n, r in enumerate(ranks)]
    imgs, merged = O.merge_updates(recs)
    kept = merge_rank_images(ranks)
    assert imgs == sorted(i for k in kept for i in k)
    assert merged == [x for n, k in enumerate(kept) for x in recs[n][1] if x[0] in k]
    # the oracle's restatement of one update keys the batch by image id and converts boxes in fp32
    targets = [{'image_id': 1}, {'image_id': 1}]
    outs = [{'boxes': np.array([[0, 0, 1, 1]], np.float32), 'scores': np.array([.1], np.float32), 'labels': np.array([0.])},
            {'boxes': np.array([[.1, .2, 1.3, 1.7]], np.float32), 'scores': np.array([.7], np.float32), 'labels': np.array([1.])}]
    ids, recs = O.batch_records(targets, outs, {0: 5, 1: 6})
    assert ids == [1] and len(recs) == 1 and recs[0][1] == 6
    assert recs[0][2][2] == float(np.float32(1.3) - np.float32(.1)) and recs[0][3] == float(np.float32(.7))


def test_summary_lines_follow_pycocotools():
    from cvpytorch_b200.coco_eval import summary_lines
    lines = summary_lines([.5] * 6 + [-1] * 6)
    assert lines[0] == ' Average Precision  (AP) @[ IoU=0.50:0.95 | area=   all | maxDets=100 ] = 0.500'
    assert lines[2] == ' Average Precision  (AP) @[ IoU=0.75      | area=   all | maxDets=100 ] = 0.500'
    assert lines[6] == ' Average Recall     (AR) @[ IoU=0.50:0.95 | area=   all | maxDets=  1 ] = -1.000'


# ----------------------------------------------------------------------------------------------- C ABI host checks
def _call(lib, params, *, gt=256, det=256, out=256, ws=256, ws_bytes=1 << 30):
    v = ctypes.c_void_p
    return lib.cvb_coco_eval_bbox(params, v(gt), v(gt), v(gt), v(gt), v(out), v(det), v(det), v(det), v(det), v(det), v(out), v(out), v(out),
                                  v(ws), ws_bytes, None)


def test_c_abi_rejects_bad_sizes_and_pointers():
    from cvpytorch_b200 import _lib
    lib = _lib.lib()

    def params(n_images=10, n_cats=3, n_gt=5, n_det=7):
        return ctypes.byref(_lib.CvbCocoEvalParams(n_images, n_cats, n_gt, n_det))
    assert _call(lib, None) != 0 and b'null params' in lib.cvb_last_error_string()
    for kw, msg in ((dict(n_images=0), b'n_images'), (dict(n_images=_lib.CVB_COCO_MAX_IMAGES + 1), b'n_images'), (dict(n_cats=0), b'n_cats'),
                    (dict(n_cats=_lib.CVB_COCO_MAX_CATS + 1), b'n_cats'), (dict(n_gt=-1), b'n_gt'), (dict(n_gt=_lib.CVB_COCO_MAX_GT + 1), b'n_gt'),
                    (dict(n_det=-1), b'n_det'), (dict(n_det=_lib.CVB_COCO_MAX_DETS + 1), b'n_det')):
        assert _call(lib, params(**kw)) != 0 and msg in lib.cvb_last_error_string(), kw
    assert _call(lib, params(), out=0) != 0 and b'null pointer' in lib.cvb_last_error_string()
    assert _call(lib, params(), gt=0) != 0 and b'ground-truth' in lib.cvb_last_error_string()
    assert _call(lib, params(), det=0) != 0 and b'detection' in lib.cvb_last_error_string()
    assert _call(lib, params(), ws=0) != 0
    assert _call(lib, params(), ws=256 + 8) != 0 and b'aligned' in lib.cvb_last_error_string()
    assert lib.cvb_coco_eval_workspace_bytes(-1, 0, 1) == 0 and lib.cvb_coco_eval_workspace_bytes(0, 0, 0) == 0
    assert lib.cvb_coco_eval_workspace_bytes(_lib.CVB_COCO_MAX_DETS + 1, 0, 1) == 0
    # LVIS fits: 1 203 categories, 20 k images
    assert _lib.CVB_COCO_MAX_CATS >= 1203 and _lib.CVB_COCO_MAX_IMAGES >= 20000
    assert _lib.CVB_COCO_MAX_CATS * _lib.CVB_COCO_MAX_IMAGES < 2 ** 32 - 1  # the (category, image) key stays below the drop key


def test_ops_refuses_sizes_beyond_the_limits_before_any_launch():
    from cvpytorch_b200 import _lib, ops
    e = torch.zeros(0)
    with pytest.raises(_lib.CvbError, match='categories'):
        ops.coco_eval_bbox(e, e, e, e, torch.zeros(3, dtype=torch.uint8), e, e, e, e, _lib.CVB_COCO_MAX_CATS + 1, O.IOU_THRS, O.REC_THRS)
    with pytest.raises(_lib.CvbError, match='CUDA'):
        ops.coco_eval_bbox(e, e, e, e, torch.zeros(3, dtype=torch.uint8), e, e, e, e, 80, O.IOU_THRS, O.REC_THRS)
