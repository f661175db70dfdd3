"""Drop-in for src/evaluator/eval_coco.py CocoEvaluator (iou_types ['bbox']): COCO box mAP with pycocotools' numbers, computed on the
H100 (csrc/coco_eval.cu), without pycocotools.

The ground truth is read from dataset.coco.dataset, the raw COCO dict.  Detections accumulate in device buffers across update() calls;
evaluate() merges the ranks under an initialised process group, runs matching, accumulation and the summary on the device, prints
pycocotools' 12-line summary and returns the reference's dict.  Record rules follow the reference: within one update a repeated image keeps
its last output, across updates and ranks the first evaluation of an image wins, labels map through dataset.id2category when it exists,
and boxes go xyxy -> xywh in the outputs' dtype before they are widened to float64.
"""
import numpy as np
import torch
import torch.distributed as dist

from . import ops

IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
METRIC_NAMES = ['mAP', 'AP_50', 'AP_75', 'AP_small', 'AP_medium', 'AP_large',
                'Recall_1', 'Recall_10', 'Recall_100', 'Recall_small', 'Recall_medium', 'Recall_large']
# (title, IoU, area, maxDets) of each line of COCOeval.summarize()
_SUMMARY = [(1, None, 'all', 100), (1, .5, 'all', 100), (1, .75, 'all', 100), (1, None, 'small', 100), (1, None, 'medium', 100),
            (1, None, 'large', 100), (0, None, 'all', 1), (0, None, 'all', 10), (0, None, 'all', 100), (0, None, 'small', 100),
            (0, None, 'medium', 100), (0, None, 'large', 100)]
_MISSING, _DROPPED = -2, -1  # category lookup: a label with no id2category entry / a category the ground truth does not list


def batch_outputs(targets):
    """One update's (image id, output index) pairs: the batch is keyed by image id, so a repeated image keeps its last output (at the
    position of its first appearance)."""
    pairs = {}
    for i, t in enumerate(targets):
        pairs[int(t['image_id'])] = i
    return list(pairs.items())


def merge_rank_images(rank_images):
    """Each rank's evaluated image ids in update order (unique within a rank) -> each rank's images that count.  Ranks are merged in
    order and the first evaluation of an image wins, as the reference's np.unique(..., return_index=True) over the gathered lists."""
    seen, kept = set(), []
    for imgs in rank_images:
        k = [i for i in imgs if i not in seen]
        seen.update(k)
        kept.append(k)
    return kept


def summary_lines(stats):
    """pycocotools COCOeval.summarize()'s 12 lines."""
    lines = []
    for s, (ap, thr, area, max_det) in zip(stats, _SUMMARY):
        title, kind = ('Average Precision', '(AP)') if ap else ('Average Recall', '(AR)')
        iou = f'{IOU_THRS[0]:0.2f}:{IOU_THRS[-1]:0.2f}' if thr is None else f'{thr:0.2f}'
        lines.append(f' {title:<18} {kind} @[ IoU={iou:<9} | area={area:>6s} | maxDets={max_det:>3d} ] = {s:0.3f}')
    return lines


class CocoEvaluator:
    def __init__(self, dataset, iou_types):
        assert isinstance(iou_types, (list, tuple))
        if list(iou_types) != ['bbox']:
            raise NotImplementedError(f'CocoEvaluator (H100): iou_types {list(iou_types)!r}; only ["bbox"] is implemented')
        self.dataset = dataset
        self.iou_types = list(iou_types)
        self.metric_names = list(METRIC_NAMES)
        gt = dataset.coco.dataset
        self._known_images = {img['id'] for img in gt.get('images', [])}
        anns = gt.get('annotations', [])
        self.cat_ids = sorted({c['id'] for c in gt.get('categories', [])})
        if not self.cat_ids:
            raise ValueError('CocoEvaluator: the ground truth lists no categories')
        self.img_ids = np.array(sorted(self._known_images | {a['image_id'] for a in anns}), dtype=np.int64)
        self._img_index = {int(i): n for n, i in enumerate(self.img_ids)}
        cat_index = {c: k for k, c in enumerate(self.cat_ids)}
        anns = [a for a in anns if a['category_id'] in cat_index]
        bad = [a['id'] for a in anns if not a['id'] > 0]
        if bad:
            raise ValueError(f'CocoEvaluator: annotation ids must be > 0 (COCOeval uses 0 for "unmatched"); got {bad[:5]}')
        n_img = len(self.img_ids)
        key = np.array([cat_index[a['category_id']] * n_img + self._img_index[a['image_id']] for a in anns], dtype=np.int64)
        order = np.argsort(key, kind='stable')
        self._gt_host = dict(key=key[order].astype(np.int32),
                             box=np.array([[float(v) for v in a['bbox']] for a in anns], dtype=np.float64).reshape(-1, 4)[order],
                             area=np.array([float(a['area']) for a in anns], dtype=np.float64)[order],
                             crowd=np.array([1 if a.get('iscrowd', 0) else 0 for a in anns], dtype=np.uint8)[order])
        # label -> category index, over the integer labels 0 .. len - 1
        if hasattr(dataset, 'id2category'):
            m = dataset.id2category
            m = dict(m) if isinstance(m, dict) else dict(enumerate(m))
            labels = [int(k) for k in m if float(k) == int(k) and int(k) >= 0]
            lut = np.full(max(labels, default=-1) + 1, _MISSING, dtype=np.int32)
            for k in labels:
                lut[k] = cat_index.get(m[k], _DROPPED)
            self._outside = _MISSING
        else:
            lut = np.full(max(max(self.cat_ids), -1) + 1, _DROPPED, dtype=np.int32)
            for c, k in cat_index.items():
                if c >= 0:
                    lut[c] = k
            self._outside = _DROPPED
        self._lut_host = torch.from_numpy(lut)
        self._gt = None
        self._lut = {}
        self.reset()

    def reset(self):
        self.count = 0
        self._seen = set()
        self._images = []  # image indices evaluated on this rank, in update order
        self._chunks = []  # per update (image index, category index, score, xywh float64) device tensors
        self._flags = None  # CUDA outputs: [missing label, NaN score] counts, checked before evaluation
        self.eval = {}
        self.stats = None

    # ------------------------------------------------------------------------------------------------- update
    def _categories(self, labels, device):
        lut = self._lut_host if device.type == 'cpu' else self._lut.setdefault(device, self._lut_host.to(device))
        lab = labels.reshape(-1).to(torch.float64)
        ok = (lab == torch.floor(lab)) & (lab >= 0) & (lab < lut.numel())
        idx = torch.where(ok, lab, torch.zeros_like(lab)).to(torch.int64)
        return torch.where(ok, lut[idx], torch.full_like(idx, self._outside, dtype=torch.int32))

    def update(self, targets, outputs):
        outputs = list(outputs)
        plan = []
        for img_id, i in batch_outputs(targets):
            if img_id in self._seen:
                continue  # the first evaluation of an image wins
            o = outputs[i]
            boxes, scores, labels = o['boxes'], o['scores'], o['labels']
            n = scores.numel()
            if tuple(boxes.shape) != (n, 4) or labels.numel() != n:
                raise ValueError(f'CocoEvaluator.update: image {img_id}: boxes {tuple(boxes.shape)}, scores {tuple(scores.shape)}, '
                                 f'labels {tuple(labels.shape)}')
            if n and img_id not in self._known_images:
                raise AssertionError(f'Results do not correspond to current coco set (image id {img_id})')
            cats = None
            if not scores.is_cuda:
                if n and bool(torch.isnan(scores).any()):
                    raise ValueError(f'CocoEvaluator.update: image {img_id} has NaN scores')
                cats = self._categories(labels, labels.device)
                if bool((cats == _MISSING).any()):
                    bad = labels.reshape(-1)[cats == _MISSING][0].item()
                    raise KeyError(bad)  # dataset.id2category[label], as the reference's lookup raises
            plan.append((img_id, o, cats))
        for img_id, o, cats in plan:
            self._seen.add(img_id)
            if img_id not in self._img_index:
                continue  # no detections and no ground truth: nothing to count
            idx = self._img_index[img_id]
            self._images.append(idx)
            boxes, scores, labels = o['boxes'], o['scores'].reshape(-1), o['labels']
            if scores.numel() == 0:
                continue
            dev = scores.device if scores.is_cuda else torch.device('cuda', torch.cuda.current_device())
            if cats is None:
                cats = self._categories(labels, dev)
                flags = torch.stack([(cats == _MISSING).sum(), torch.isnan(scores).sum()])
                self._flags = flags if self._flags is None else self._flags + flags
            xywh = torch.stack((boxes[:, 0], boxes[:, 1], boxes[:, 2] - boxes[:, 0], boxes[:, 3] - boxes[:, 1]), 1)
            self._chunks.append((torch.full((scores.numel(),), idx, dtype=torch.int32, device=dev), cats.to(dev, torch.int32),
                                 scores.to(dev, torch.float32), xywh.to(torch.float64).to(dev)))
        self.count += 1

    # ------------------------------------------------------------------------------------------------- evaluate
    def _device(self):
        for c in self._chunks:
            return c[0].device
        return torch.device('cuda', torch.cuda.current_device())

    def _local(self, dev):
        if self._chunks:
            return [torch.cat([c[j] for c in self._chunks]) for j in range(4)]
        return [torch.zeros((0,), dtype=torch.int32, device=dev), torch.zeros((0,), dtype=torch.int32, device=dev),
                torch.zeros((0,), dtype=torch.float32, device=dev), torch.zeros((0, 4), dtype=torch.float64, device=dev)]

    def synchronize_between_processes(self):
        """Merges every rank's records (one size exchange and one all_gather_into_tensor of padded float64 rows) into self._merged:
        (evaluated image indices, detections).  Without a process group of more than one rank the local records are used."""
        if self._flags is not None:
            missing, nan = (int(v) for v in self._flags.cpu())
            if missing:
                raise KeyError('CocoEvaluator: a label has no dataset.id2category entry')
            if nan:
                raise ValueError('CocoEvaluator: NaN detection scores')
        dev = self._device()
        img, cat, score, box = self._local(dev)
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
            self._merged = (list(self._images), (img, cat, score, box))
            return
        world = dist.get_world_size()
        n_img, n_det = len(self._images), img.numel()
        sizes = torch.zeros((world * 2,), dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(sizes, torch.tensor([n_img, n_det], dtype=torch.int64, device=dev))
        sizes = sizes.view(world, 2).cpu().tolist()
        rows = max(a + b for a, b in sizes)
        mine = torch.zeros((rows, 7), dtype=torch.float64, device=dev)
        mine[:n_img, 0] = torch.tensor(self._images, dtype=torch.float64, device=dev)
        mine[n_img:n_img + n_det] = torch.cat([img[:, None].double(), cat[:, None].double(), score[:, None].double(), box], 1)
        gathered = torch.empty((world * rows, 7), dtype=torch.float64, device=dev).view(world, rows, 7)
        dist.all_gather_into_tensor(gathered.view(world * rows, 7), mine)
        max_img = max(a for a, _ in sizes)
        img_cols = gathered[:, :max_img, 0].cpu().to(torch.int64)
        kept = merge_rank_images([img_cols[r, :sizes[r][0]].tolist() for r in range(world)])
        dets = []
        for r, (ni, nd) in enumerate(sizes):
            d = gathered[r, ni:ni + nd]
            mask = torch.zeros((len(self.img_ids),), dtype=torch.bool, device=dev)
            if kept[r]:
                mask[torch.tensor(kept[r], dtype=torch.int64, device=dev)] = True
            dets.append(d[mask[d[:, 0].to(torch.int64)]])
        d = torch.cat(dets)
        self._merged = ([i for k in kept for i in k], (d[:, 0].to(torch.int32).contiguous(), d[:, 1].to(torch.int32).contiguous(),
                                                       d[:, 2].to(torch.float32).contiguous(), d[:, 3:7].contiguous()))

    def accumulate(self):
        """Matching, accumulation and the 12 statistics on the device; one 96-byte copy brings the statistics back."""
        images, (img, cat, score, box) = self._merged
        dev = img.device
        if self._gt is None or self._gt['key'].device != dev:
            self._gt = {k: torch.from_numpy(v).to(dev) for k, v in self._gt_host.items()}
        evaluated = torch.zeros((len(self.img_ids),), dtype=torch.uint8)
        evaluated[images] = 1
        g = self._gt
        precision, recall, stats, masks = ops.coco_eval_bbox(g['key'], g['box'], g['area'], g['crowd'], evaluated.to(dev), img, cat, score, box,
                                                             len(self.cat_ids), IOU_THRS, REC_THRS)
        self.eval = {'precision': precision, 'recall': recall, 'det_masks': masks}
        self.stats = stats.cpu().numpy()

    def summarize(self):
        print('IoU metric: bbox')
        for line in summary_lines(self.stats):
            print(line)

    def evaluate(self):
        if self.count < 1:
            return None
        self.synchronize_between_processes()
        self.accumulate()
        self.summarize()
        performances = {'performance': 0}
        for k, v in zip(self.metric_names, self.stats):
            performances['bbox_' + k] = v
            if k == 'mAP':
                performances['performance'] += v
        return performances
