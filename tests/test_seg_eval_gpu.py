"""Segmentation confusion matrix on the H100 against the numpy oracle: the device matrix and error bits bitwise equal over every gt × pred
dtype pair, sizes around the vector width, misaligned views, nc from 1 to NC_MAX, one-bin contention and a 16 × 1024 × 2048 batch; the
drop-in SegmentationEvaluator on the reference fixture (metrics bitwise, np.float64), its error state, no host sync in update(), and the
DeepLabv3+ val forward end to end.  Large label maps come from a closed-form integer formula of the pixel index."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import seg_eval_oracle as SO  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'seg_eval.npz')
DTYPES = {np.uint8: torch.uint8, np.int32: torch.int32, np.int64: torch.int64}


class _Dataset:
    def __init__(self, nc):
        self.num_classes = nc
        self.dictionary = [{f'c{i}': 1.0} for i in range(nc)]


def same(a, b):
    """Bitwise equal, or both NaN."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


def labels(n, nc, dtype, start=0, bad=True):
    """(gt, pred) of n pixels from a closed-form hash of the pixel index: gt in [0, nc + 2) with about 8 % ignore pixels (255, or -1 for
    signed types), pred equal to gt on about 60 % of the pixels and in [0, nc) elsewhere.  With bad=True a few predictions are nc or -1,
    so some flat indices alias and some leave [0, nc²)."""
    i = np.arange(start, start + n, dtype=np.int64)
    h = ((i * 2654435761) & 0xFFFFFFFF) >> 4
    gt = h % (nc + 2)
    gt = np.where(h % 13 == 0, 255 if dtype == np.uint8 else -1, gt)
    pred = np.where((h >> 7) % 5 < 3, gt % nc, (h >> 11) % nc)
    if bad:
        pred = np.where((h >> 13) % 211 == 0, nc, pred)
        pred = np.where((h >> 17) % 223 == 0, -1, pred)
    return gt, pred


def device_count(gt, pred, nc, offsets=(0, 0)):
    """Runs ops.seg_confusion_update on CUDA copies of gt / pred placed at the given element offsets of larger buffers."""
    from cvpytorch_b200 import ops
    views = []
    for a, off in zip((gt, pred), offsets):
        buf = torch.zeros(a.size + off + 8, dtype=DTYPES[a.dtype.type], device='cuda')
        v = buf[off:off + a.size].view(a.shape)
        v.copy_(torch.from_numpy(np.ascontiguousarray(a)))
        views.append(v)
    matrix = torch.zeros((nc, nc), dtype=torch.int64, device='cuda').view(torch.uint64)
    err = torch.zeros(1, dtype=torch.int32, device='cuda')
    ops.seg_confusion_update(views[0], views[1], nc, matrix, err)
    return matrix.cpu().numpy(), int(err.cpu()[0])


def check(gt, pred, nc, offsets=(0, 0)):
    m, e = device_count(gt, pred, nc, offsets)
    ref, ref_err = SO.confusion_update(gt, pred, nc)
    assert np.array_equal(m.astype(np.int64), ref) and m.dtype == np.uint64, (nc, gt.dtype, pred.dtype, gt.size, offsets)
    assert e == ref_err, (nc, gt.dtype, pred.dtype, gt.size, offsets, e, ref_err)
    return ref_err


@pytest.mark.parametrize('gd', [np.uint8, np.int32, np.int64])
@pytest.mark.parametrize('pd', [np.uint8, np.int32, np.int64])
def test_matrix_every_dtype_pair(cuda, gd, pd):
    """Every gt × pred dtype pair: n = 0, 1, odd and not a multiple of 16, contiguous views at odd element offsets (the vector path
    starts late, or never when the two maps cannot be aligned together), nc = 1, 2, 19, 150 and NC_MAX; the error bits too."""
    from cvpytorch_b200 import ops
    errs = set()
    for nc in (1, 2, 19, 150, ops.seg_nc_max()):
        for n, offsets in ((0, (0, 0)), (1, (0, 0)), (15, (0, 0)), (17, (1, 0)), (1000, (0, 0)), (4099, (3, 3)), (65537, (1, 5)),
                           (65535, (2, 1)), (250001, (0, 7))):
            gt, pred = labels(n, nc, gd, start=n * 7 + nc)
            errs.add(check(gt.astype(gd), pred.astype(pd), nc, offsets))
    assert len(errs) > 1  # both clean and flagged launches ran


def test_contention_every_pixel_in_one_bin(cuda):
    from cvpytorch_b200 import ops
    n = 3 * 1024 * 1024 + 5
    for nc in (1, 19, 150, ops.seg_nc_max()):
        for gd, pd in ((np.uint8, np.uint8), (np.int64, np.int64)):
            b = nc // 2
            m, e = device_count(np.full(n, b, gd), np.full(n, b, pd), nc)
            assert e == 0 and m[b, b] == n and m.sum() == n


def test_batch_16x1024x2048(cuda):
    nc = 19
    gt, pred = labels(16 * 1024 * 2048, nc, np.uint8, bad=False)
    gt, pred = gt.astype(np.uint8).reshape(16, 1024, 2048), pred.astype(np.int64).reshape(16, 1024, 2048)
    assert check(gt, pred, nc) == 0


def test_launches_split_above_the_per_call_limit(cuda, monkeypatch):
    from cvpytorch_b200 import _lib
    monkeypatch.setattr(_lib, 'CVB_SEG_MAX_N', 1000)
    gt, pred = labels(4567, 19, np.int64)
    n0 = _lib.launch_count()
    check(gt, pred, 19, (1, 0))
    assert _lib.launch_count() - n0 == 5


def _run_fixture_case(nc, steps, expected):
    from cvpytorch_b200.seg_eval import SegmentationEvaluator
    ev = SegmentationEvaluator(_Dataset(nc))
    pending = False
    for i, (st, exp) in enumerate(zip(steps, expected)):
        if st[0] == 'u':
            ev.update(torch.from_numpy(st[1]).cuda(), torch.from_numpy(st[2]).cuda())
            pending |= exp == 'raises'
        elif st[0] == 'r':
            ev.reset()
            pending = False
        elif pending:
            # the reference raised inside the offending update; the drop-in raises here, and keeps raising until reset()
            with pytest.raises(ValueError, match='flat index'):
                ev.evaluate()
            with pytest.raises(ValueError, match='flat index'):
                ev.evaluate()
        elif exp is None:
            assert ev.evaluate() is None
        else:
            got = ev.evaluate()
            assert list(got) == list(exp[0])
            for k in SO.METRICS:
                assert type(got[k]) is np.float64 and same(got[k], exp[0][k]), (i, k, got[k], exp[0][k])
            cm = ev.confusion_matrix
            assert cm.dtype == np.float64 and same(cm, exp[1])
    return ev


@pytest.mark.filterwarnings('ignore:Mean of empty slice')
def test_drop_in_reproduces_reference_fixture(cuda):
    """Every fixture case through the drop-in on CUDA tensors of the stored dtypes: matrices and metrics bitwise the reference's."""
    for name, (nc, steps, expected) in SO.load_fixture(GOLDEN).items():
        _run_fixture_case(nc, steps, expected)


def test_error_state_until_reset(cuda):
    from cvpytorch_b200.seg_eval import SegmentationEvaluator
    nc = 3
    for pred, bits in (([-1, 0], 'no negative'), ([0, 3], '>= nc²'), ([-1, 3], r'\) and a flat index')):
        ev = SegmentationEvaluator(_Dataset(nc))
        ev.update(torch.tensor([0, 2], device='cuda'), torch.tensor(pred, device='cuda'))
        for _ in range(2):
            with pytest.raises(ValueError, match=bits):
                ev.evaluate()
        ev.update(torch.tensor([1], device='cuda'), torch.tensor([1], device='cuda'))
        with pytest.raises(ValueError):
            ev.evaluate()
        ev.reset()
        assert ev.evaluate() is None
        ev.update(torch.tensor([1, 2], device='cuda'), torch.tensor([1, 0], device='cuda'))
        r = ev.evaluate()
        assert r['Acc'] == 0.5 and np.array_equal(ev.confusion_matrix, [[0, 0, 0], [0, 1, 0], [1, 0, 0]])


def test_update_checks(cuda):
    from cvpytorch_b200 import _lib
    from cvpytorch_b200.seg_eval import SegmentationEvaluator
    ev = SegmentationEvaluator(_Dataset(19))
    g = torch.zeros((2, 8, 8), dtype=torch.int64, device='cuda')
    with pytest.raises(AssertionError):
        ev.update(g, g[:, :, :7])
    with pytest.raises(AssertionError):
        ev.update(g, g.view(2, 64))
    for bad in (torch.float32, torch.float16, torch.bool, torch.int16):
        with pytest.raises(TypeError, match='uint8, int32 or int64'):
            ev.update(g, g.to(bad))
    with pytest.raises(_lib.CvbError, match='CUDA tensor'):
        ev.update(g, g.cpu())
    assert ev.count == 0 and ev.evaluate() is None


def test_update_makes_no_host_sync(cuda):
    """The first update allocates the matrix on the labels' device; neither it nor later updates, non-contiguous inputs included,
    synchronise the host."""
    from cvpytorch_b200.seg_eval import SegmentationEvaluator
    nc = 19
    gt, pred = labels(2 * 96 * 128, nc, np.uint8, bad=False)
    g = torch.from_numpy(gt.astype(np.uint8).reshape(2, 96, 128)).cuda()
    p = torch.from_numpy(pred.astype(np.int64).reshape(2, 128, 96)).cuda().transpose(1, 2)  # non-contiguous
    ev = SegmentationEvaluator(_Dataset(nc))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for _ in range(3):
            ev.update(g, p)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    ref = SO.Evaluator(nc)
    for _ in range(3):
        ref.update(g.cpu().numpy(), p.cpu().numpy())
    assert same(ev.confusion_matrix, ref.confusion_matrix) and ev.count == 3
    got, exp = ev.evaluate(), ref.evaluate()
    assert all(same(got[k], exp[k]) for k in SO.METRICS)


def test_deeplab_val_forward_end_to_end(cuda):
    """EncoderDecoder(mode='val') on a seeded 256×512 image with 19 classes feeds the drop-in; the oracle scores the same label maps
    copied to the host."""
    from cvpytorch_b200 import synth
    from cvpytorch_b200.seg_eval import SegmentationEvaluator
    model = synth.build_deeplab(True)
    g = torch.Generator().manual_seed(7)
    ev, ref = SegmentationEvaluator(_Dataset(19)), SO.Evaluator(19)
    ev.reset()
    ref.reset()
    for b in range(2):
        imgs = torch.randn((1, 3, 256, 512), generator=g).cuda()
        gt, _ = labels(256 * 512, 19, np.int64, start=b * 131072, bad=False)
        targets = torch.from_numpy(gt.reshape(1, 256, 512)).cuda()
        preds = model(imgs, targets, mode='val')
        assert preds.shape == targets.shape and preds.dtype == torch.int64
        ev.update(targets, preds)
        ref.update(targets.cpu().numpy(), preds.cpu().numpy())
    assert same(ev.confusion_matrix, ref.confusion_matrix)
    got, exp = ev.evaluate(), ref.evaluate()
    assert len(np.unique(preds.cpu().numpy())) > 1
    for k in SO.METRICS:
        assert type(got[k]) is np.float64 and same(got[k], exp[k]), k
