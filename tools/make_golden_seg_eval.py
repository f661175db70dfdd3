"""Writes tests/golden/seg_eval.npz: the reference's SegmentationEvaluator (src/evaluator/eval_segmentation.py) run on the CPU over small
stored cases.

  CVPYTORCH_REFERENCE=<reference checkout> python tools/make_golden_seg_eval.py

src/evaluator/__init__.py imports eval_coco, which needs pycocotools and torch._six, so eval_segmentation.py is loaded by file path inside
a stand-in package that provides its relative `base_evaluator` import.  Each case starts from a fresh evaluator and runs a sequence of
update / reset / evaluate steps; the fixture stores the inputs, whether each update raised, and each evaluate()'s metrics and matrix.
Before writing, oracle/seg_eval_oracle.py must reproduce every outcome bitwise (NaN for NaN)."""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import seg_eval_oracle as SO  # noqa: E402

REF = os.environ.get('CVPYTORCH_REFERENCE', '')


def load_reference():
    pkg_dir = os.path.join(REF, 'src', 'evaluator')
    pkg = types.ModuleType('_ref_evaluator')
    pkg.__path__ = [pkg_dir]
    sys.modules['_ref_evaluator'] = pkg
    mods = {}
    for name in ('base_evaluator', 'eval_segmentation'):
        spec = importlib.util.spec_from_file_location(f'_ref_evaluator.{name}', os.path.join(pkg_dir, f'{name}.py'))
        mods[name] = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = mods[name]
        spec.loader.exec_module(mods[name])
    return mods['eval_segmentation'].SegmentationEvaluator


class _Dataset:
    def __init__(self, nc):
        self.num_classes = nc
        self.dictionary = [{f'c{i}': 1.0} for i in range(nc)]


class _TorchInputs:
    """Hands the reference torch tensors, as the trainer does."""

    def __init__(self, ev):
        self.ev = ev

    def update(self, gt, pred):
        self.ev.update(torch.from_numpy(gt), torch.from_numpy(pred))

    def reset(self):
        self.ev.reset()

    def evaluate(self):
        return self.ev.evaluate()

    @property
    def confusion_matrix(self):
        return self.ev.confusion_matrix


def _maps(nc, shape, seed, gt_dtype, pred_dtype, agree=.7):
    """Seeded label maps: gt in [0, nc) with 10 % ignore pixels (255 for uint8; -1, 255 or nc for wider types), pred equal to gt where
    they agree and uniform in [0, nc) elsewhere."""
    rng = np.random.default_rng(seed)
    gt = rng.integers(0, nc, shape)
    pred = np.where(rng.random(shape) < agree, gt, rng.integers(0, nc, shape))
    drop = rng.random(shape) < .1
    gt = np.where(drop, 255 if np.dtype(gt_dtype) == np.uint8 else rng.choice([-1, 255, nc], shape), gt)
    return gt.astype(gt_dtype), pred.astype(pred_dtype)


def cases():
    """name -> (nc, steps); a step is ('u', gt, pred), ('r',) or ('e',)."""
    c = {}
    # the ones-initialised first update (uint8 targets with 255 ignores), then updates after reset() (int64 targets with negatives)
    g0, p0 = _maps(5, (2, 6, 7), 1, np.uint8, np.int64)
    g1, p1 = _maps(5, (1, 9, 5), 2, np.int64, np.int64)
    g2, p2 = _maps(5, (3, 4, 4), 3, np.int64, np.int32)
    c['first_then_reset'] = (5, [('u', g0, p0), ('e',), ('r',), ('u', g1, p1), ('e',), ('u', g2, p2), ('e',)])
    # class 3 in neither map (NaN IoU and Acc), class 4 only in the predictions (IoU 0, Acc NaN)
    g = np.array([[0, 1, 2, 0], [1, 2, 0, 255]], np.uint8)
    p = np.array([[0, 4, 2, 1], [1, 2, 4, 3]], np.uint8)
    c['absent_classes'] = (5, [('r',), ('u', g, p), ('e',)])
    # every pixel ignored: Acc = 0 / 0 = NaN, mAcc and mIoU the nanmean of all NaN, FWIoU = 0.0 (no class with freq > 0)
    g = np.full((2, 3), 255, np.uint8)
    c['all_ignored'] = (4, [('r',), ('u', g, np.zeros((2, 3), np.int64)), ('e',)])
    # out-of-range predictions whose flat index is in range alias into a neighbouring row: nc = 3, gt 0 / pred 3 -> (1, 0),
    # gt 2 / pred -1 -> (1, 2), gt 1 / pred 5 -> (2, 2)
    c['aliasing'] = (3, [('r',), ('u', np.array([0, 2, 1, 0, 2, 1], np.int64), np.array([3, -1, 1, 0, 2, 5], np.int64)), ('e',)])
    # a flat index < 0 (np.bincount raises) and one >= nc² (the reshape raises), each after a valid update
    c['error_negative'] = (3, [('r',), ('u', np.array([1, 2], np.int64), np.array([1, 2], np.int64)),
                               ('u', np.array([0, 1], np.int64), np.array([-1, 0], np.int64)), ('e',)])
    c['error_overflow'] = (3, [('r',), ('u', np.array([1, 2], np.uint8), np.array([1, 2], np.int32)),
                               ('u', np.array([2, 1], np.uint8), np.array([3, 0], np.int32)), ('e',)])
    # no update: evaluate() is None, before and after reset()
    c['count_zero'] = (4, [('e',), ('r',), ('e',)])
    # Cityscapes' 19 classes and ADE20K's 150
    g, p = _maps(19, (2, 24, 40), 4, np.uint8, np.int64, agree=.8)
    g2, p2 = _maps(19, (1, 17, 33), 5, np.int32, np.uint8)
    c['nc19'] = (19, [('r',), ('u', g, p), ('u', g2, p2), ('e',)])
    g, p = _maps(150, (1, 40, 60), 6, np.int64, np.int32, agree=.5)
    c['nc150'] = (150, [('r',), ('u', g, p), ('e',)])
    return c


def same(a, b):
    """Bitwise equal, or both NaN."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


def main():
    Ref = load_reference()
    res = {}
    for name, (nc, steps) in cases().items():
        ref = SO.run_case(_TorchInputs(Ref(_Dataset(nc))), steps)
        ora = SO.run_case(SO.Evaluator(nc), steps)
        for i, (r, o) in enumerate(zip(ref, ora)):
            if isinstance(r, tuple):
                assert isinstance(o, tuple) and same(r[1], o[1]), (name, i)
                for k in SO.METRICS:
                    assert type(r[0][k]) is np.float64 and type(o[0][k]) is np.float64 and same(r[0][k], o[0][k]), (name, i, k)
            else:
                assert r == o, (name, i, r, o)
        res.update(SO.fixture_arrays(name, nc, steps, ref))
        print(name, [r if not isinstance(r, tuple) else {k: float(v) for k, v in r[0].items()} for r in ref])
    path = os.path.join(ROOT, 'tests', 'golden', 'seg_eval.npz')
    np.savez_compressed(path, **res)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
