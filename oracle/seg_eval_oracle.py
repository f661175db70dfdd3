"""numpy restatement of the reference's segmentation evaluator (src/evaluator/eval_segmentation.py SegmentationEvaluator).

  update:   pixels with 0 <= gt < nc; flat = nc * gt + pred in int64 (wrapping); bincount(flat, minlength=nc²).reshape(nc, nc) is added to
            the float64 matrix.  A flat index < 0 makes np.bincount raise, one >= nc² makes the reshape raise: confusion_update reports
            them as the error bits ERR_NEGATIVE / ERR_OVERFLOW, together with the counts of the flat indices inside [0, nc²).
  state:    np.ones((nc, nc)) after __init__, np.zeros((nc, nc)) after reset(); evaluate() is None while count < 1.
  metrics:  Acc, mAcc, mIoU, FWIoU and performance (= mIoU), float64, with 0 / 0 = NaN, nanmean and FWIoU over freq > 0.

tests/golden/seg_eval.npz (tools/make_golden_seg_eval.py) pins this restatement to the reference evaluator on the CPU.
"""
import warnings

import numpy as np

ERR_NEGATIVE, ERR_OVERFLOW = 1, 2


def confusion_update(gt, pred, nc):
    """(int64 [nc, nc] counts of the flat indices inside [0, nc²), error bits) for one pair of label maps."""
    gt, pred = np.asarray(gt).reshape(-1), np.asarray(pred).reshape(-1)
    mask = (gt >= 0) & (gt < nc)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')  # int64 overflow wraps, as in the reference's expression
        flat = np.int64(nc) * gt[mask].astype(np.int64) + pred[mask].astype(np.int64)
    err = (ERR_NEGATIVE if (flat < 0).any() else 0) | (ERR_OVERFLOW if (flat >= nc * nc).any() else 0)
    ok = flat[(flat >= 0) & (flat < nc * nc)]
    return np.bincount(ok, minlength=nc * nc).reshape(nc, nc), err


def metrics(cm):
    """The reference's four metrics of a float64 confusion matrix, as np.float64 values."""
    with np.errstate(divide='ignore', invalid='ignore'):
        acc = np.diag(cm).sum() / cm.sum()
        macc = np.nanmean(np.diag(cm) / cm.sum(axis=1))
        iu = np.diag(cm) / (np.sum(cm, axis=1) + np.sum(cm, axis=0) - np.diag(cm))
        miou = np.nanmean(iu)
        freq = np.sum(cm, axis=1) / np.sum(cm)
        fwiou = (freq[freq > 0] * iu[freq > 0]).sum()
    return {'Acc': acc, 'mAcc': macc, 'mIoU': miou, 'FWIoU': fwiou, 'performance': miou}


class Evaluator:
    """The reference evaluator's state machine.  An update with error bits raises ValueError, as the reference's does, and leaves the
    matrix and count unchanged."""

    def __init__(self, nc):
        self.nc = nc
        self.confusion_matrix = np.ones((nc, nc))
        self.count = 0

    def update(self, gt, pred):
        assert np.shape(gt) == np.shape(pred)
        counts, err = confusion_update(gt, pred, self.nc)
        if err:
            raise ValueError(f'flat index outside [0, nc²): error bits {err}')
        self.confusion_matrix += counts
        self.count += 1

    def reset(self):
        self.confusion_matrix = np.zeros((self.nc, self.nc))
        self.count = 0

    def evaluate(self):
        if self.count < 1:
            return None
        return metrics(self.confusion_matrix)


def run_case(evaluator, steps):
    """Runs a case's steps on an evaluator with the reference's surface; returns one entry per step: 'ok' for an update that did not
    raise, 'raises' for one that did, None for reset, and evaluate()'s result (None or the metrics dict with a copy of the matrix)."""
    out = []
    for st in steps:
        if st[0] == 'u':
            try:
                evaluator.update(st[1], st[2])
                out.append('ok')
            except ValueError:
                out.append('raises')
        elif st[0] == 'r':
            evaluator.reset()
            out.append(None)
        else:
            r = evaluator.evaluate()
            out.append(None if r is None else (r, np.array(evaluator.confusion_matrix, dtype=np.float64)))
    return out


METRICS = ('Acc', 'mAcc', 'mIoU', 'FWIoU', 'performance')


def fixture_arrays(name, nc, steps, outcomes):
    """The npz entries of one case: its nc, step kinds and inputs, and per step 'ok' / 'raises' / 'none' / 'metrics' with the metrics
    (float64, METRICS order) and the matrix of every evaluate() that returned them."""
    res = {f'{name}__nc': np.array(nc), f'{name}__kinds': np.array([st[0] for st in steps])}
    status = []
    for i, (st, o) in enumerate(zip(steps, outcomes)):
        if st[0] == 'u':
            res[f'{name}__gt{i}'], res[f'{name}__pred{i}'] = st[1], st[2]
            status.append(o)
        elif st[0] == 'r':
            status.append('none')
        elif o is None:
            status.append('none')
        else:
            status.append('metrics')
            res[f'{name}__metrics{i}'] = np.array([o[0][k] for k in METRICS], dtype=np.float64)
            res[f'{name}__cm{i}'] = o[1]
    res[f'{name}__status'] = np.array(status)
    return res


def load_fixture(path):
    """name -> (nc, steps, expected): steps as fixture_arrays took them, expected[i] = 'ok' / 'raises' for updates, None for resets and
    for evaluate() calls that returned None, else (metrics dict of np.float64, float64 matrix)."""
    z = np.load(path)
    names = sorted({k.split('__')[0] for k in z.files})
    cases = {}
    for name in names:
        kinds, status = z[f'{name}__kinds'].tolist(), z[f'{name}__status'].tolist()
        steps, expected = [], []
        for i, (k, s) in enumerate(zip(kinds, status)):
            if k == 'u':
                steps.append(('u', z[f'{name}__gt{i}'], z[f'{name}__pred{i}']))
                expected.append(s)
            else:
                steps.append((k,))
                expected.append(None if s == 'none' else
                                (dict(zip(METRICS, (np.float64(v) for v in z[f'{name}__metrics{i}']))), z[f'{name}__cm{i}']))
        cases[name] = (int(z[f'{name}__nc']), steps, expected)
    return cases
