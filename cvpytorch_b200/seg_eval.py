"""Drop-in for src/evaluator/eval_segmentation.py SegmentationEvaluator: the confusion matrix is counted on the H100
(csrc/seg_eval.cu) and the metrics are the reference's float64 numpy formulas.

update() launches one kernel on the current stream and does not sync the host; the matrix lives on the device of the first update.
evaluate() copies the matrix and the error word to the host once.  Divergences from the reference:
  * A flat index nc * gt + pred outside [0, nc²) makes the reference raise inside update() (np.bincount / reshape) and crash the trainer.
    Here the kernel flags it, and the next evaluate() raises ValueError; the evaluator stays in error until reset(), because the host
    cannot see the flag without a sync.  Flat indices inside [0, nc²) alias into a neighbouring row exactly as in the reference.
  * Float and bool label maps are refused (the reference truncates them with astype('int')), and so are CPU tensors: there is no
    fallback.
Like the reference there is no cross-rank merge: each rank scores what it saw.
"""
import numpy as np
import torch

from . import _lib, ops


def metrics(confusion_matrix):
    """The reference's Acc, mAcc, mIoU, FWIoU and performance (= mIoU) of a float64 confusion matrix, as np.float64, with its nan
    semantics (0 / 0 is NaN, nanmean, FWIoU over the classes with freq > 0)."""
    cm = confusion_matrix
    with np.errstate(divide='ignore', invalid='ignore'):
        diag, rows, cols = np.diag(cm), np.sum(cm, axis=1), np.sum(cm, axis=0)
        acc = diag.sum() / cm.sum()
        macc = np.nanmean(diag / cm.sum(axis=1))
        iu = diag / (rows + cols - diag)
        miou = np.nanmean(iu)
        freq = rows / np.sum(cm)
        fwiou = (freq[freq > 0] * iu[freq > 0]).sum()
    return {'Acc': acc, 'mAcc': macc, 'mIoU': miou, 'FWIoU': fwiou, 'performance': miou}


class SegmentationEvaluator:
    def __init__(self, dataset):
        self.dataset = dataset
        self.num_class = dataset.num_classes
        self.dictionary = dataset.dictionary
        if not 1 <= self.num_class <= ops.seg_nc_max():
            raise ValueError(f'SegmentationEvaluator (H100): num_classes must be in [1, {ops.seg_nc_max()}], got {self.num_class}')
        self.count = 0
        self._start = 1  # the reference starts from np.ones in __init__ and from np.zeros after reset()
        self._buf = None

    def reset(self):
        self.count = 0
        self._start = 0
        self._buf = None

    def _views(self):
        """The device buffer: nc² uint64 counts followed by the int32 error word, so that evaluate() needs one copy."""
        nc2 = self.num_class * self.num_class
        return self._buf[:nc2].view(torch.uint64).view(self.num_class, self.num_class), self._buf[nc2:].view(torch.int32)

    def update(self, gt_image, pre_image):
        assert gt_image.shape == pre_image.shape
        for name, t in (('gt_image', gt_image), ('pre_image', pre_image)):
            if not isinstance(t, torch.Tensor) or not t.is_cuda:
                raise _lib.CvbError(f'SegmentationEvaluator.update: {name} must be a CUDA tensor (the H100 path has no CPU fallback)')
            if t.dtype not in ops.SEG_DTYPES:
                raise TypeError(f'SegmentationEvaluator.update: {name} is {t.dtype}; label maps must be uint8, int32 or int64')
        if gt_image.device != pre_image.device:
            raise _lib.CvbError(f'SegmentationEvaluator.update: gt_image on {gt_image.device}, pre_image on {pre_image.device}')
        if self._buf is None:
            nc2 = self.num_class * self.num_class
            self._buf = torch.full((nc2 + 1,), self._start, dtype=torch.int64, device=gt_image.device)
            self._buf[nc2:] = 0
        elif self._buf.device != gt_image.device:
            raise _lib.CvbError(f'SegmentationEvaluator.update: the confusion matrix lives on {self._buf.device}, the labels on '
                                f'{gt_image.device}')
        matrix, err = self._views()
        ops.seg_confusion_update(gt_image.detach(), pre_image.detach(), self.num_class, matrix, err)
        self.count += 1

    def _host(self):
        nc = self.num_class
        if self._buf is None:
            return np.full((nc, nc), float(self._start)), 0
        h = self._buf.cpu().numpy()
        return h[:nc * nc].view(np.uint64).reshape(nc, nc).astype(np.float64), int(h[nc * nc:].view(np.int32)[0])

    @property
    def confusion_matrix(self):
        """A host float64 copy of the matrix, as the reference's attribute holds it.  Reading it syncs the host with the device."""
        return self._host()[0]

    def evaluate(self):
        if self.count < 1:
            return None
        cm, err = self._host()
        if err:
            why = []
            if err & _lib.CVB_SEG_ERR_NEGATIVE:
                why.append('a flat index nc * gt + pred < 0 (np.bincount: "no negative elements")')
            if err & _lib.CVB_SEG_ERR_OVERFLOW:
                why.append(f'a flat index nc * gt + pred >= nc² = {self.num_class ** 2} (the reshape to [nc, nc] fails)')
            raise ValueError('SegmentationEvaluator: an update since the last reset() had ' + ' and '.join(why) + '; reset() clears it')
        return metrics(cm)
