"""COCO box mAP (pycocotools COCOeval, iouType='bbox', default parameters) restated in numpy from the algorithm, plus the record rules of
the reference CocoEvaluator wrapper (src/evaluator/eval_coco.py).  The oracle of cvpytorch_b200/coco_eval.py and csrc/coco_eval.cu.

evaluate():   per (category, area range, image) match records: detections stable-sorted by -score and cut to 100, ground truths
              stable-sorted by their ignore flag, one greedy scan per IoU threshold.
accumulate(): precision [T, R, K, A, M] and recall [T, K, A, M] (-1 where a category has no non-ignored ground truth).
summarize():  the 12 statistics of COCOeval.summarize, in METRIC_NAMES order.
"""
import numpy as np

IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ['all', 'small', 'medium', 'large']
METRIC_NAMES = ['mAP', 'AP_50', 'AP_75', 'AP_small', 'AP_medium', 'AP_large',
                'Recall_1', 'Recall_10', 'Recall_100', 'Recall_small', 'Recall_medium', 'Recall_large']
# (is AP, IoU threshold or None, area label, maxDets) of each statistic
STAT_SPECS = [(1, None, 'all', 100), (1, .5, 'all', 100), (1, .75, 'all', 100), (1, None, 'small', 100), (1, None, 'medium', 100),
              (1, None, 'large', 100), (0, None, 'all', 1), (0, None, 'all', 10), (0, None, 'all', 100), (0, None, 'small', 100),
              (0, None, 'medium', 100), (0, None, 'large', 100)]


def bb_iou(d, g, crowd):
    """IoU [D, G] of xywh float64 boxes d [D, 4] and g [G, 4]; a crowd ground truth divides by the detection's area alone."""
    d = np.asarray(d, np.float64).reshape(-1, 4)
    g = np.asarray(g, np.float64).reshape(-1, 4)
    w = np.minimum((d[:, 0] + d[:, 2])[:, None], (g[:, 0] + g[:, 2])[None]) - np.maximum(d[:, 0][:, None], g[:, 0][None])
    h = np.minimum((d[:, 1] + d[:, 3])[:, None], (g[:, 1] + g[:, 3])[None]) - np.maximum(d[:, 1][:, None], g[:, 1][None])
    inter = w * h
    da = (d[:, 2] * d[:, 3])[:, None]
    ga = (g[:, 2] * g[:, 3])[None]
    u = np.where(np.asarray(crowd, bool)[None], da, (da + ga) - inter)
    ok = (w > 0) & (h > 0)
    with np.errstate(divide='ignore', invalid='ignore'):
        return np.where(ok, inter / np.where(ok, u, 1.0), 0.0)


def _gt_index(gt):
    """Ground truths grouped per (image id, category id) in annotation order, as (box, area, crowd, id) lists."""
    out = {}
    for a in gt['annotations']:
        out.setdefault((a['image_id'], a['category_id']), []).append(
            (list(map(float, a['bbox'])), float(a['area']), bool(a.get('iscrowd', 0)), a['id']))
    return out


def cat_ids(gt):
    return sorted({c['id'] for c in gt['categories']})


def evaluate(gt, results, img_ids):
    """results: (image_id, category_id, [x, y, w, h], score) records; img_ids: the evaluated images.  Returns
    {(category id, area index, image id): record or None}; a record holds dtMatches [T, D] (matched ground-truth id, 0 when unmatched),
    dtIgnore [T, D], gtIgnore [G] (in the ignore-sorted order), dtScores [D] and dtOrder [D] (indices into `results`)."""
    cats = cat_ids(gt)
    imgs = set(img_ids)
    gts = _gt_index(gt)
    dts = {}
    for i, (img, cat, box, score) in enumerate(results):
        if img in imgs and cat in cats:
            dts.setdefault((img, cat), []).append((list(map(float, box)), float(score), i))
    T = len(IOU_THRS)
    out = {}
    for cat in cats:
        for img in sorted(imgs):
            g = gts.get((img, cat), [])
            d = dts.get((img, cat), [])
            order = np.argsort([-x[1] for x in d], kind='mergesort')[:MAX_DETS[-1]]
            d = [d[i] for i in order]
            crowd = np.array([x[2] for x in g], bool)
            ious = bb_iou([x[0] for x in d], [x[0] for x in g], crowd) if len(g) and len(d) else np.zeros((len(d), len(g)))
            for ai, rng in enumerate(AREA_RNG):
                if not g and not d:
                    out[cat, ai, img] = None
                    continue
                ig = np.array([x[2] or x[1] < rng[0] or x[1] > rng[1] for x in g], bool)
                gi = np.argsort(ig, kind='mergesort')
                gIg, gCrowd, gIds = ig[gi], crowd[gi], [g[i][3] for i in gi]
                io = ious[:, gi]
                gtm = np.zeros((T, len(g)), np.int64)
                dtm = np.zeros((T, len(d)), np.int64)
                dtIg = np.zeros((T, len(d)), bool)
                for ti, t in enumerate(IOU_THRS):
                    for di in range(len(d)):
                        best, m = min([t, 1 - 1e-10]), -1
                        for gj in range(len(g)):
                            if gtm[ti, gj] > 0 and not gCrowd[gj]:
                                continue
                            if m > -1 and not gIg[m] and gIg[gj]:
                                break
                            if io[di, gj] < best:
                                continue
                            best, m = io[di, gj], gj
                        if m == -1:
                            continue
                        dtIg[ti, di] = gIg[m]
                        dtm[ti, di] = gIds[m]
                        gtm[ti, m] = di + 1
                darea = np.array([x[0][2] * x[0][3] for x in d], np.float64)
                outside = (darea < rng[0]) | (darea > rng[1])
                dtIg = dtIg | ((dtm == 0) & outside[None])
                out[cat, ai, img] = dict(dtMatches=dtm, dtIgnore=dtIg, gtIgnore=gIg, dtScores=np.array([x[1] for x in d], np.float64),
                                         dtOrder=np.array([x[2] for x in d], np.int64))
    return out


def accumulate(evals, cats, img_ids):
    T, R, K, A, M = len(IOU_THRS), len(REC_THRS), len(cats), len(AREA_RNG), len(MAX_DETS)
    precision = -np.ones((T, R, K, A, M))
    recall = -np.ones((T, K, A, M))
    imgs = sorted(set(img_ids))
    for k, cat in enumerate(cats):
        for a in range(A):
            E = [evals[cat, a, i] for i in imgs]
            E = [e for e in E if e is not None]
            if not E:
                continue
            gtIg = np.concatenate([e['gtIgnore'] for e in E])
            npig = np.count_nonzero(gtIg == 0)
            if npig == 0:
                continue
            for m, maxDet in enumerate(MAX_DETS):
                scores = np.concatenate([e['dtScores'][0:maxDet] for e in E])
                inds = np.argsort(-scores, kind='mergesort')
                dtm = np.concatenate([e['dtMatches'][:, 0:maxDet] for e in E], axis=1)[:, inds]
                dtIg = np.concatenate([e['dtIgnore'][:, 0:maxDet] for e in E], axis=1)[:, inds]
                tps = np.logical_and(dtm, np.logical_not(dtIg))
                fps = np.logical_and(np.logical_not(dtm), np.logical_not(dtIg))
                tp_sum = np.cumsum(tps, axis=1).astype(dtype=float)
                fp_sum = np.cumsum(fps, axis=1).astype(dtype=float)
                for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                    nd = len(tp)
                    rc = tp / npig
                    pr = (tp / (fp + tp + np.spacing(1))).tolist()
                    recall[t, k, a, m] = rc[-1] if nd else 0
                    for i in range(nd - 1, 0, -1):  # precision envelope: suffix maximum
                        if pr[i] > pr[i - 1]:
                            pr[i - 1] = pr[i]
                    q = np.zeros((R,))
                    for ri, pi in enumerate(np.searchsorted(rc, REC_THRS, side='left')):
                        if pi >= nd:
                            break
                        q[ri] = pr[pi]
                    precision[t, :, k, a, m] = q
    return precision, recall


def summarize(precision, recall):
    stats = np.zeros(12)
    for n, (ap, thr, area, maxDet) in enumerate(STAT_SPECS):
        a, m = AREA_LBL.index(area), MAX_DETS.index(maxDet)
        s = precision if ap else recall
        if thr is not None:
            s = s[np.where(thr == IOU_THRS)[0]]
        s = s[:, :, :, a, m] if ap else s[:, :, a, m]
        stats[n] = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
    return stats


def coco_eval(gt, results, img_ids):
    """The whole bbox evaluation: {'evals', 'precision', 'recall', 'stats'}."""
    evals = evaluate(gt, results, img_ids)
    precision, recall = accumulate(evals, cat_ids(gt), img_ids)
    return dict(evals=evals, precision=precision, recall=recall, stats=summarize(precision, recall))


# ------------------------------------------------------------------------------- the reference wrapper's record rules
def batch_records(targets, outputs, id2category=None):
    """One CocoEvaluator.update: (evaluated image ids, result records).  The batch is keyed by image id, so a repeated image keeps its
    last output; boxes go xyxy -> xywh in the outputs' dtype and only then become Python floats."""
    preds = {int(t['image_id']): o for t, o in zip(targets, outputs)}
    recs = []
    for img, p in preds.items():
        b = p['boxes']
        xywh = np.stack([b[:, 0], b[:, 1], b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]], 1) if len(b) else np.zeros((0, 4), b.dtype)
        labels = np.asarray(p['labels']).tolist()
        if id2category is not None:
            labels = [id2category[l] for l in labels]
        recs += [(img, labels[k], xywh[k].tolist(), float(p['scores'][k])) for k in range(len(xywh))]
    return sorted(preds), recs


def merge_updates(updates):
    """updates: (image ids, records) of every update of every rank, in rank order and update order.  The first evaluation of an image
    wins.  Returns (sorted image ids, records)."""
    seen, recs = set(), []
    for img_ids, r in updates:
        new = set(img_ids) - seen
        seen |= new
        recs += [x for x in r if x[0] in new]
    return sorted(seen), recs
