"""COCO box mAP on the H100 against the COCOeval oracle: bitwise-equal match / ignore masks, precision and recall, and stats within 1e-12
(the means' summation order), over seeded sweeps, the drop-in CocoEvaluator's record rules, and the YOLOv5-s val forward end to end."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import coco_eval_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu


class _Coco:
    def __init__(self, d):
        self.dataset = d


class _Dataset:
    def __init__(self, gt, id2category=None):
        self.coco = _Coco(gt)
        if id2category is not None:
            self.id2category = id2category


def make_case(seed, n_img=40, n_cat=6, dets=(0, 40), gts=(0, 8), crowd=.1, unused_cats=2, big_segment=0, neg_zero=False):
    """Seeded GT and result records on an integer grid: IoUs land exactly on thresholds, areas hit 1024 / 9216, scores tie inside and
    across images.  big_segment > 0 gives image 1 that many ground truths and 3x as many detections of one category."""
    rng = np.random.default_rng(seed)
    cats = sorted(rng.choice(np.arange(1, 8 * (n_cat + unused_cats)), n_cat + unused_cats, replace=False).tolist())
    used = cats[:n_cat]
    gt = {'images': [{'id': int(i)} for i in range(1, n_img + 1)], 'categories': [{'id': int(c)} for c in cats], 'annotations': []}
    results = []
    aid = 1
    for img in range(1, n_img + 1):
        boxes = []
        ng = int(rng.integers(*gts)) if img != 1 or not big_segment else big_segment
        for _ in range(ng):
            c = used[0] if img == 1 and big_segment else int(rng.choice(used))
            x, y = (int(v) for v in rng.integers(0, 300, 2))
            w, h = (int(v) for v in rng.integers(1, 130, 2))
            area = float(w * h) if rng.random() > .3 else float(rng.choice([1024, 9216, 1023.5, 9216.5]))
            gt['annotations'].append(dict(id=aid, image_id=img, category_id=c, bbox=[float(x), float(y), float(w), float(h)], area=area,
                                          iscrowd=int(rng.random() < crowd)))
            boxes.append((c, x, y, w, h))
            aid += 1
        nd = int(rng.integers(*dets)) if img != 1 or not big_segment else 3 * big_segment
        for _ in range(nd):
            if boxes and rng.random() < .75:
                c, x, y, w, h = boxes[int(rng.integers(len(boxes)))]
                # integer shifts: many IoUs are ratios of small integers, some exactly .5 / .75
                x, y = x + int(rng.integers(-3, 4)), y + int(rng.integers(-3, 4))
                w, h = max(1, w + int(rng.integers(-3, 4))), max(1, h + int(rng.integers(-3, 4)))
            else:
                c = int(rng.choice(cats + [99999]))  # a category the GT does not list is never evaluated
                x, y, w, h = (int(v) for v in (*rng.integers(0, 300, 2), *rng.integers(1, 130, 2)))
            s = float(np.float32(rng.integers(0, 12) / 11))
            if neg_zero and s == 0 and rng.random() < .5:
                s = -0.0
            results.append((img, int(c), [float(x), float(y), float(w), float(h)], s))
    return gt, results


def device_eval(gt, results, img_ids, dev):
    from cvpytorch_b200 import ops
    from cvpytorch_b200.coco_eval import CocoEvaluator
    ev = CocoEvaluator(_Dataset(gt), ['bbox'])
    g = {k: torch.from_numpy(v).to(dev) for k, v in ev._gt_host.items()}
    ci = {c: k for k, c in enumerate(ev.cat_ids)}
    det_img = torch.tensor([ev._img_index[r[0]] for r in results], dtype=torch.int32).to(dev)
    det_cat = torch.tensor([ci.get(r[1], -1) for r in results], dtype=torch.int32).to(dev)
    det_score = torch.tensor([r[3] for r in results], dtype=torch.float32).to(dev)
    det_box = torch.tensor([r[2] for r in results], dtype=torch.float64).reshape(-1, 4).to(dev)
    evaluated = torch.zeros(len(ev.img_ids), dtype=torch.uint8)
    evaluated[[ev._img_index[i] for i in img_ids]] = 1
    P, R, S, M = ops.coco_eval_bbox(g['key'], g['box'], g['area'], g['crowd'], evaluated.to(dev), det_img, det_cat, det_score, det_box,
                                    len(ev.cat_ids), O.IOU_THRS, O.REC_THRS)
    return P.cpu().numpy(), R.cpu().numpy(), S.cpu().numpy(), M.cpu().numpy().view(np.uint32)


def assert_matches_oracle(gt, results, img_ids, dev):
    P, R, S, M = device_eval(gt, results, img_ids, dev)
    ref = O.coco_eval(gt, results, img_ids)
    want = np.zeros((len(results), 4), np.uint32)
    for (cat, a, img), e in ref['evals'].items():
        if e is None:
            continue
        for d, o in enumerate(e['dtOrder']):
            bits = sum(int(e['dtMatches'][t, d] > 0) << t for t in range(10)) | sum(int(e['dtIgnore'][t, d]) << (16 + t) for t in range(10))
            want[o, a] = bits
    assert np.array_equal(M, want), np.argwhere(M != want)[:5]
    assert np.array_equal(P, ref['precision']), np.argwhere(P != ref['precision'])[:5]
    assert np.array_equal(R, ref['recall'])
    assert np.allclose(S, ref['stats'], rtol=0, atol=1e-12), (S, ref['stats'])
    return ref


SWEEPS = {
    'mixed': dict(seed=1),
    'empty_images': dict(seed=2, dets=(0, 3), gts=(0, 3)),
    'dense_over_100': dict(seed=3, n_img=6, n_cat=1, unused_cats=1, dets=(90, 260), gts=(2, 12)),
    'crowds': dict(seed=4, crowd=.5, dets=(10, 60)),
    'big_segment': dict(seed=5, n_img=5, big_segment=75),
    'neg_zero_ties': dict(seed=6, neg_zero=True, dets=(20, 80)),
    'many_cats': dict(seed=7, n_img=60, n_cat=40, unused_cats=10, dets=(0, 120), gts=(0, 20)),
}


@pytest.mark.parametrize('name', list(SWEEPS))
def test_device_matches_oracle(cuda, name):
    gt, results = make_case(**SWEEPS[name])
    n_img = len(gt['images'])
    assert_matches_oracle(gt, results, list(range(1, n_img + 1)), cuda)
    # a subset of the images: the others' ground truths do not count
    assert_matches_oracle(gt, [r for r in results if r[0] % 3], [i for i in range(1, n_img + 1) if i % 3], cuda)


def test_no_detections_and_no_ground_truth(cuda):
    gt, results = make_case(8, n_img=5)
    ref = assert_matches_oracle(gt, [], [1, 2, 3], cuda)
    assert (ref['stats'][ref['stats'] != -1] == 0).all()
    gt['annotations'] = []
    ref = assert_matches_oracle(gt, results, [1, 2, 3, 4, 5], cuda)
    assert (ref['stats'] == -1).all()


def test_coco_val_sized(cuda):
    # 5 000 images, about 36 k ground truths over 80 non-contiguous categories
    gt, results = make_case(9, n_img=5000, n_cat=80, unused_cats=0, dets=(0, 100), gts=(0, 15), crowd=.01)
    assert 30000 < len(gt['annotations']) < 40000
    assert_matches_oracle(gt, results, list(range(1, 5001)), cuda)


# ------------------------------------------------------------------------------------------------- drop-in CocoEvaluator
def _outputs(rng, gt, img_ids, labels_of, device, n=(0, 30)):
    """Model-style outputs: xyxy fp32 boxes with fractional corners (the fp32 xywh conversion rounds), fp32 scores with ties."""
    by_img = {}
    for a in gt['annotations']:
        by_img.setdefault(a['image_id'], []).append(a)
    outs = []
    for img in img_ids:
        rows = []
        for _ in range(int(rng.integers(*n))):
            anns = by_img.get(img)
            if anns and rng.random() < .7:
                a = anns[int(rng.integers(len(anns)))]
                x, y, w, h = a['bbox']
                lab = labels_of[a['category_id']]
            else:
                x, y, w, h = (float(v) for v in rng.uniform(0, 300, 4))
                lab = int(rng.integers(0, len(labels_of)))
            j = rng.normal(0, 1.5, 4)
            rows.append([x + j[0] + .1, y + j[1] + .3, x + w + j[2] + .7, y + h + j[3] + .9, float(rng.integers(1, 9) / 9), float(lab)])
        r = torch.tensor(rows, dtype=torch.float32).reshape(-1, 6)
        outs.append({'boxes': r[:, :4].contiguous().to(device), 'scores': r[:, 4].contiguous().to(device), 'labels': r[:, 5].contiguous().to(device)})
    return outs


@pytest.mark.parametrize('where', ['host', 'cuda'])
def test_evaluator_updates_match_the_reference_rules(cuda, where):
    from cvpytorch_b200.coco_eval import CocoEvaluator
    gt, _ = make_case(10, n_img=30, n_cat=5, unused_cats=0)
    cats = [c['id'] for c in gt['categories']]
    id2category = {i: c for i, c in enumerate(cats)}
    labels_of = {c: i for i, c in id2category.items()}
    ev = CocoEvaluator(_Dataset(gt, id2category), ['bbox'])
    rng = np.random.default_rng(11)
    dev = cuda if where == 'cuda' else torch.device('cpu')
    batches = [[1, 2, 3, 2], [4, 5, 1], [6, 7, 8, 9, 10], [3, 11, 11], list(range(12, 31))]  # repeats inside and across updates
    updates = []
    for ids in batches:
        outs = _outputs(rng, gt, ids, labels_of, dev)
        targets = [{'image_id': torch.tensor(i)} for i in ids]
        ev.update(targets, outs)
        updates.append(O.batch_records(targets, [{k: v.cpu().numpy() for k, v in o.items()} for o in outs], id2category))
    img_ids, recs = O.merge_updates(updates)
    ref = O.coco_eval(gt, recs, img_ids)
    res = ev.evaluate()
    assert np.array_equal(ev.eval['precision'].cpu().numpy(), ref['precision'])
    assert np.array_equal(ev.eval['recall'].cpu().numpy(), ref['recall'])
    assert np.allclose(ev.stats, ref['stats'], rtol=0, atol=1e-12)
    assert list(res) == ['performance'] + ['bbox_' + k for k in O.METRIC_NAMES] and res['performance'] == res['bbox_mAP']
    ev.reset()
    assert ev.evaluate() is None


def test_cuda_outputs_with_an_unknown_label_raise_at_evaluate(cuda):
    from cvpytorch_b200.coco_eval import CocoEvaluator
    gt, _ = make_case(12, n_img=3)
    ev = CocoEvaluator(_Dataset(gt, {0: gt['categories'][0]['id']}), ['bbox'])
    o = {'boxes': torch.tensor([[0., 0., 5., 5.]], device=cuda), 'scores': torch.tensor([.5], device=cuda),
         'labels': torch.tensor([3.], device=cuda)}
    ev.update([{'image_id': torch.tensor(1)}], [o])
    with pytest.raises(KeyError):
        ev.evaluate()


def test_yolov5s_val_forward_end_to_end(cuda):
    """The synthetic calibrated YOLOv5-s val forward on seeded images, scored by the drop-in against the oracle on the same outputs."""
    from cvpytorch_b200 import synth
    from cvpytorch_b200.coco_eval import CocoEvaluator
    model = synth.build_yolov5s(calibrated=True, device=cuda)
    cat_ids = [1 + 2 * i + (i // 10) for i in range(80)]  # non-contiguous, as COCO's
    id2category = {i: c for i, c in enumerate(cat_ids)}
    rng = np.random.default_rng(13)
    g = torch.Generator().manual_seed(13)
    gt = {'images': [{'id': 100 + i} for i in range(8)], 'categories': [{'id': c} for c in cat_ids], 'annotations': []}
    for i in range(8):
        for _ in range(int(rng.integers(1, 10))):
            x, y = rng.uniform(0, 200, 2)
            w, h = rng.uniform(4, 120, 2)
            gt['annotations'].append(dict(id=len(gt['annotations']) + 1, image_id=100 + i, category_id=int(rng.choice(cat_ids)),
                                          bbox=[float(x), float(y), float(w), float(h)], area=float(w * h), iscrowd=int(rng.random() < .05)))
    ev = CocoEvaluator(_Dataset(gt, id2category), ['bbox'])
    updates = []
    n_det = 0
    with torch.no_grad():
        for b in range(2):
            imgs = torch.rand((4, 3, 256, 256), generator=g).to(cuda)
            targets = [{'image_id': torch.tensor(100 + 4 * b + i)} for i in range(4)]
            _, outs = model(imgs, targets, 'val')
            n_det += sum(o['scores'].numel() for o in outs)
            ev.update(targets, outs)
            updates.append(O.batch_records(targets, [{k: v.numpy() for k, v in o.items()} for o in outs], id2category))
    assert n_det > 0
    img_ids, recs = O.merge_updates(updates)
    ref = O.coco_eval(gt, recs, img_ids)
    ev.evaluate()
    assert np.array_equal(ev.eval['precision'].cpu().numpy(), ref['precision'])
    assert np.array_equal(ev.eval['recall'].cpu().numpy(), ref['recall'])
    assert np.allclose(ev.stats, ref['stats'], rtol=0, atol=1e-12)
