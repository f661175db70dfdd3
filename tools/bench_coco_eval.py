"""Benchmark of the COCO box mAP drop-in (cvpytorch_b200.coco_eval.CocoEvaluator, csrc/coco_eval.cu) on a seeded COCO-val-sized set:
5 000 images, about 36 k ground truths over 80 non-contiguous category ids (some crowd), 300 detections per image with score ties, fed
as host fp32 outputs in batches of 64, as the drop-in models' val forward returns them.  Writes nothing; one JSON line with the card's
name and power limit read in the same call.  Single GPU.

  python tools/bench_coco_eval.py [--images 5000] [--dets 300] [--repeats 5] [--no-oracle]

  update_s          all update() calls (host outputs into the device buffers), host clock ending in a device synchronise;
  evaluate_s        evaluate() after one warm-up evaluate(), host clock ending in a device synchronise (median and all repeats);
  oracle_s          the numpy COCOeval restatement (oracle/coco_eval_oracle.py) on the same records, on the host;
  stats_max_abs_diff / precision_equal / recall_equal: the device against the oracle."""
import argparse
import contextlib
import io
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_darknet_train import _card  # noqa: E402


class _Coco:
    def __init__(self, d):
        self.dataset = d


class _Dataset:
    def __init__(self, gt, id2category):
        self.coco = _Coco(gt)
        self.id2category = id2category


def make_set(n_img, dets, seed=2024):
    rng = np.random.default_rng(seed)
    cat_ids = [1 + i + (i // 10) * 2 for i in range(80)]  # non-contiguous, as COCO's 1..90
    gt = {'images': [{'id': 1000 + i} for i in range(n_img)], 'categories': [{'id': c} for c in cat_ids], 'annotations': []}
    outs = []
    for i in range(n_img):
        ng = int(rng.integers(0, 15))
        xy = rng.uniform(0, 560, (ng, 2))
        wh = np.exp(rng.uniform(np.log(4), np.log(400), (ng, 2)))
        cats = rng.integers(0, 80, ng)
        for k in range(ng):
            gt['annotations'].append(dict(id=len(gt['annotations']) + 1, image_id=1000 + i, category_id=cat_ids[cats[k]],
                                          bbox=[float(v) for v in (*xy[k], *wh[k])], area=float(wh[k, 0] * wh[k, 1] * .8),
                                          iscrowd=int(rng.random() < .01)))
        # detections: jittered copies of the ground truths plus background boxes, scores on a coarse grid (ties)
        src = rng.integers(0, max(ng, 1), dets)
        hit = (rng.random(dets) < .3) & (ng > 0)
        base = np.where(hit[:, None], np.concatenate([xy, xy + wh], 1)[src] if ng else 0, 0)
        bg = np.sort(rng.uniform(0, 640, (dets, 2, 2)), axis=1).reshape(dets, 4)[:, [0, 2, 1, 3]]
        boxes = np.where(hit[:, None], base + rng.normal(0, 3, (dets, 4)), bg).astype(np.float32)
        labels = np.where(hit, cats[src] if ng else 0, rng.integers(0, 80, dets)).astype(np.float32)
        scores = (rng.integers(1, 1000, dets) / 1000).astype(np.float32)
        outs.append({'boxes': torch.from_numpy(boxes), 'scores': torch.from_numpy(scores), 'labels': torch.from_numpy(labels)})
    return gt, {k: c for k, c in enumerate(cat_ids)}, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=5000)
    ap.add_argument('--dets', type=int, default=300)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--no-oracle', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_coco_eval.py needs a CUDA device')
    from cvpytorch_b200.coco_eval import CocoEvaluator
    from oracle import coco_eval_oracle as O
    gt, id2category, outs = make_set(args.images, args.dets)
    ev = CocoEvaluator(_Dataset(gt, id2category), ['bbox'])
    ids = [img['id'] for img in gt['images']]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for b in range(0, len(ids), 64):
        ev.update([{'image_id': torch.tensor(i)} for i in ids[b:b + 64]], outs[b:b + 64])
    torch.cuda.synchronize()
    update_s = time.perf_counter() - t0
    quiet = contextlib.redirect_stdout(io.StringIO())
    with quiet:
        ev.evaluate()  # warm-up: module load, GT upload
    times = []
    for _ in range(args.repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            ev.evaluate()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    res = {'bench': 'coco_eval', 'card': _card(torch.cuda.current_device()), 'images': args.images, 'ground_truths': len(gt['annotations']),
           'detections': args.images * args.dets, 'update_s': round(update_s, 3), 'evaluate_s': round(statistics.median(times), 4),
           'evaluate_s_all': [round(t, 4) for t in times], 'stats': [float(x) for x in ev.stats]}
    if not args.no_oracle:
        t0 = time.perf_counter()
        recs = []
        for b in range(0, len(ids), 64):
            targets = [{'image_id': i} for i in ids[b:b + 64]]
            recs.append(O.batch_records(targets, [{k: v.numpy() for k, v in o.items()} for o in outs[b:b + 64]], id2category))
        img_ids, records = O.merge_updates(recs)
        ref = O.coco_eval(gt, records, img_ids)
        res['oracle_s'] = round(time.perf_counter() - t0, 1)
        res['stats_max_abs_diff'] = float(np.abs(ev.stats - ref['stats']).max())
        res['precision_equal'] = bool(np.array_equal(ev.eval['precision'].cpu().numpy(), ref['precision']))
        res['recall_equal'] = bool(np.array_equal(ev.eval['recall'].cpu().numpy(), ref['recall']))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
