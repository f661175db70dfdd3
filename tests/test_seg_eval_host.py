"""Segmentation mIoU without a GPU: the numpy oracle against the reference evaluator's fixture (bitwise, NaN for NaN), the C ABI's
refusals before any launch, and the drop-in SegmentationEvaluator's refusals and its None before any update."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import seg_eval_oracle as SO  # noqa: E402

GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'seg_eval.npz')


def same(a, b):
    """Bitwise equal, or both NaN."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


class _Dataset:
    def __init__(self, nc):
        self.num_classes = nc
        self.dictionary = [{f'c{i}': 1.0} for i in range(nc)]


@pytest.mark.filterwarnings('ignore:Mean of empty slice')
def test_oracle_reproduces_reference_fixture():
    cases = SO.load_fixture(GOLDEN)
    assert {'first_then_reset', 'absent_classes', 'all_ignored', 'aliasing', 'error_negative', 'error_overflow', 'count_zero', 'nc19',
            'nc150'} <= set(cases)
    for name, (nc, steps, expected) in cases.items():
        got = SO.run_case(SO.Evaluator(nc), steps)
        for i, (g, e) in enumerate(zip(got, expected)):
            if isinstance(e, tuple):
                assert same(g[1], e[1]), (name, i)
                for k in SO.METRICS:
                    assert type(g[0][k]) is np.float64 and same(g[0][k], e[0][k]), (name, i, k)
            else:
                assert g == e, (name, i)


def test_fixture_covers_the_edges():
    cases = SO.load_fixture(GOLDEN)
    # ones-initialised matrix: the first evaluate() counts 1 in every bin on top of the pixels
    nc, steps, exp = cases['first_then_reset']
    g, p = steps[0][1], steps[0][2]
    assert g.dtype == np.uint8 and (g == 255).any() and np.array_equal(exp[1][1], 1 + SO.confusion_update(g, p, nc)[0])
    assert steps[3][1].dtype == np.int64 and (steps[3][1] < 0).any()
    m = cases['all_ignored'][2][2][0]
    assert np.isnan(m['Acc']) and np.isnan(m['mIoU']) and m['FWIoU'] == 0.0
    # class 3 in no counted pixel (NaN IoU and Acc); class 4 only in the predictions (IoU 0, Acc NaN)
    m, cm = cases['absent_classes'][2][2]
    assert cm[3].sum() == 0 and cm[:, 3].sum() == 0 and cm[4].sum() == 0 and cm[:, 4].sum() == 2
    assert not np.isnan(m['mIoU']) and not np.isnan(m['mAcc'])
    # nc = 3: gt 0 / pred 3 counts at (1, 0), gt 2 / pred -1 at (1, 2)
    assert np.array_equal(cases['aliasing'][2][2][1], [[1, 0, 0], [1, 1, 1], [0, 0, 2]])
    assert cases['error_negative'][2][2] == 'raises' and cases['error_overflow'][2][2] == 'raises'
    assert cases['count_zero'][2] == [None, None, None]
    assert cases['nc19'][0] == 19 and cases['nc150'][0] == 150


def test_oracle_error_bits_and_wrap():
    assert SO.confusion_update(np.array([0]), np.array([-1]), 3)[1] == SO.ERR_NEGATIVE
    assert SO.confusion_update(np.array([2]), np.array([3]), 3)[1] == SO.ERR_OVERFLOW
    assert SO.confusion_update(np.array([0, 2]), np.array([-1, 3]), 3)[1] == SO.ERR_NEGATIVE | SO.ERR_OVERFLOW
    # nc * gt + pred wraps in int64 as the reference's expression does: a huge prediction turns negative
    cm, err = SO.confusion_update(np.array([2], np.int64), np.array([np.iinfo(np.int64).max], np.int64), 3)
    assert err == SO.ERR_NEGATIVE and cm.sum() == 0
    cm, err = SO.confusion_update(np.array([255, -1, 3], np.int64), np.array([9, 9, 9], np.int64), 3)
    assert err == 0 and cm.sum() == 0


def _err(L, rc, text):
    assert rc != 0
    assert text in L.cvb_last_error_string(), L.cvb_last_error_string()


def test_c_abi_rejects_bad_arguments():
    """cvb_seg_confusion_update checks nc, n, the dtype codes, null and misaligned pointers on the host, before any launch."""
    from cvpytorch_b200 import _lib
    L = _lib.lib()
    nc_max = L.cvb_seg_confusion_nc_max()
    assert nc_max == 241  # (nc_max + 1)² uint32 bins would not fit the 227 KB of opt-in shared memory
    assert nc_max * nc_max * 4 <= 232448 < (nc_max + 1) ** 2 * 4
    p = ctypes.c_void_p(4096)

    def call(gt=p, gd=_lib.CVB_SEG_I64, pred=p, pd=_lib.CVB_SEG_I64, n=16, nc=19, matrix=p, err=p):
        return L.cvb_seg_confusion_update(gt, gd, pred, pd, n, nc, matrix, err, None)
    _err(L, call(nc=0), b'nc must be in [1, 241]')
    _err(L, call(nc=nc_max + 1), b'nc must be in [1, 241]')
    _err(L, call(nc=-3), b'nc must be in [1, 241]')
    _err(L, call(n=-1), b'n must be in [0, 2^31 - 1]')
    _err(L, call(n=1 << 31), b'n must be in [0, 2^31 - 1]')
    for gd, pd in ((3, 2), (2, -1), (7, 7)):
        _err(L, call(gd=gd, pd=pd), b'unknown dtype code')
    _err(L, call(gt=None), b'null pointer')
    _err(L, call(pred=None), b'null pointer')
    _err(L, call(matrix=None), b'null pointer')
    _err(L, call(err=None), b'null pointer')
    _err(L, call(gt=ctypes.c_void_p(4097)), b'not aligned to their element size')
    _err(L, call(pred=ctypes.c_void_p(4100), pd=_lib.CVB_SEG_I64), b'not aligned to their element size')
    _err(L, call(pred=ctypes.c_void_p(4098), pd=_lib.CVB_SEG_I32), b'not aligned to their element size')
    _err(L, call(matrix=ctypes.c_void_p(4100)), b'matrix must be 8-byte')
    _err(L, call(err=ctypes.c_void_p(4098)), b'err 4-byte aligned')
    # n = 0 is a no-op that needs no pointers
    assert call(gt=None, pred=None, matrix=None, err=None, n=0) == 0


def test_drop_in_refuses_cpu_float_and_bad_shapes():
    from cvpytorch_b200 import _lib
    from cvpytorch_b200.seg_eval import SegmentationEvaluator
    ev = SegmentationEvaluator(_Dataset(19))
    assert ev.num_class == 19 and len(ev.dictionary) == 19 and ev.count == 0
    g = torch.zeros((2, 4, 4), dtype=torch.int64)
    with pytest.raises(_lib.CvbError, match='CUDA tensor'):
        ev.update(g, g)
    with pytest.raises(AssertionError):
        ev.update(g, g[:, :3])
    with pytest.raises(_lib.CvbError, match='CUDA tensor'):
        ev.update(g.float(), g.float())  # a CPU tensor is refused before its dtype is looked at
    assert ev.count == 0 and ev.evaluate() is None
    from cvpytorch_b200 import ops
    with pytest.raises(ValueError, match='num_classes'):
        SegmentationEvaluator(_Dataset(ops.seg_nc_max() + 1))


def test_drop_in_states_before_any_update():
    """evaluate() is None before any update; the matrix reads as the reference's np.ones after __init__ and np.zeros after reset()."""
    from cvpytorch_b200.seg_eval import SegmentationEvaluator
    ev = SegmentationEvaluator(_Dataset(7))
    assert ev.evaluate() is None
    cm = ev.confusion_matrix
    assert cm.dtype == np.float64 and np.array_equal(cm, np.ones((7, 7)))
    ev.reset()
    assert ev.evaluate() is None and np.array_equal(ev.confusion_matrix, np.zeros((7, 7)))
    with pytest.raises(AttributeError):
        ev.confusion_matrix = np.zeros((7, 7))

