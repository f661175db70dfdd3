"""Drop-in for the reference's model EMA (src/utils/ema.py): ``ModelEMA`` with the same constructor, attributes and methods, whose ``update``
runs every floating state_dict entry in ONE kernel launch (csrc/ema.cu, ``cvb_ema_update``) instead of three ATen launches per entry.

The result is bitwise the reference's on the same GPU: the kernel rounds ``item * decay``, ``src * (1 - decay)`` and their sum to fp32
one by one, with the decay computed on the host in Python double as the reference's lambda does.  What the kernel cannot run raises, with no
fallback: CPU tensors or tensors on different devices (CvbError); floating entries that are not fp32, not contiguous, shaped differently
in the model and the EMA, or overlapping another entry in memory (NotImplementedError); a floating EMA key missing from the model (KeyError,
as the reference raises).

The device table of (ema, src, numel) entries is built on the first update and reused while every entry's tensors keep their address,
dtype, shape and contiguity; ``.to()``, ``load_state_dict`` into replaced tensors, or ``convert_sync_batchnorm`` on either model is seen at
the next update, which rebuilds the table.
"""
import math
from copy import deepcopy

import torch
import torch.nn as nn

from . import _lib
from ._lib import _stream


def is_parallel(model):
    """True if model is a DataParallel / DistributedDataParallel wrapper (src/utils/ema.py is_parallel)."""
    return type(model) in (nn.parallel.DataParallel, nn.parallel.DistributedDataParallel)


def de_parallel(model):
    return model.module if is_parallel(model) else model


def copy_attr(a, b, include=(), exclude=()):
    """Sets on a every public attribute of b's __dict__ (only those in include, if given; none in exclude)."""
    for k, item in b.__dict__.items():
        if (len(include) and k not in include) or k.startswith('_') or k in exclude:
            continue
        setattr(a, k, item)


def _overlap(pairs):
    """The first (key, key) whose memory overlaps where an EMA tensor is one of the two, or None.  Source tensors may overlap each other."""
    spans = []
    for k, e, s in pairs:
        if e.numel():
            spans.append((e.data_ptr(), e.data_ptr() + 4 * e.numel(), True, k))
            spans.append((s.data_ptr(), s.data_ptr() + 4 * s.numel(), False, k))
    spans.sort(key=lambda t: t[0])
    end_all = end_ema = (-1, None)
    for start, end, is_ema, k in spans:
        if start < end_ema[0]:
            return end_ema[1], k
        if is_ema and start < end_all[0]:
            return end_all[1], k
        end_all = max(end_all, (end, k))
        if is_ema:
            end_ema = max(end_ema, (end, k))
    return None


class ModelEMA:
    """Model exponential moving average of everything in the model's state_dict (parameters and buffers), as src/utils/ema.py ModelEMA.

    ema: a deepcopy of the model (of model.module under DataParallel / DistributedDataParallel), in eval mode, parameters without grad.
    updates: the number of updates so far (a host int).  decay(x): decay * (1 - exp(-x / 2000)), the decay of update x."""

    def __init__(self, model, decay=0.9999, updates=0):
        self.ema = deepcopy(de_parallel(model)).eval()
        self.updates = updates
        self.decay = lambda x: decay * (1 - math.exp(-x / 2000))
        for p in self.ema.parameters():
            p.requires_grad_(False)
        self._sig = None    # what the table was built from: per entry (addresses, dtypes, shapes, contiguity)
        self._table = None  # (device table, entry count)

    def _pairs(self, model):
        src = de_parallel(model).state_dict(keep_vars=True)
        return [(k, e, src[k]) for k, e in self.ema.state_dict(keep_vars=True).items() if e.dtype.is_floating_point]

    def _build(self, pairs):
        for k, e, s in pairs:
            if e.dtype != torch.float32 or s.dtype != torch.float32:
                raise NotImplementedError(f'ModelEMA (H100): {k} is {e.dtype} in the EMA and {s.dtype} in the model; only fp32 entries are updated')
            if not (e.is_contiguous() and s.is_contiguous()):
                raise NotImplementedError(f'ModelEMA (H100): {k} is not contiguous in the EMA or the model')
            if e.shape != s.shape:
                raise NotImplementedError(f'ModelEMA (H100): {k} has shape {tuple(e.shape)} in the EMA and {tuple(s.shape)} in the model')
        clash = _overlap(pairs)
        if clash:
            raise NotImplementedError(f'ModelEMA (H100): {clash[0]} and {clash[1]} share memory with an EMA tensor (the reference would update it '
                                      'twice or read it after its update)')
        for k, e, s in pairs:
            if not (e.is_cuda and s.is_cuda):
                raise _lib.CvbError(f'ModelEMA: {k} is on the CPU; the H100 EMA update has no CPU fallback')
        devices = {t.device for _, e, s in pairs for t in (e, s)}
        if len(devices) > 1:
            raise _lib.CvbError(f'ModelEMA: the EMA and the model must live on one device (found {sorted(map(str, devices))})')
        entries = (_lib.CvbEmaEntry * len(pairs))(*[_lib.CvbEmaEntry(e.data_ptr(), s.data_ptr(), e.numel()) for _, e, s in pairs])
        dev = devices.pop()
        with torch.cuda.device(dev):
            table = torch.empty((len(pairs) * _lib.CVB_EMA_TABLE_ENTRY_BYTES,), dtype=torch.uint8, device=dev)
            _lib.check(_lib.lib().cvb_ema_table_upload(entries, len(pairs), table.data_ptr(), _stream()), 'cvb_ema_table_upload')
        return table, len(pairs)

    def update(self, model):
        """One EMA step: updates += 1, then every floating entry e of the EMA's state_dict becomes e * d + (1 - d) * model's entry, d =
        decay(updates), in one kernel launch on the tensors' device's current stream."""
        with torch.no_grad():
            self.updates += 1
            d = self.decay(self.updates)
            pairs = self._pairs(model)
            if not pairs:
                return
            sig = [(e.data_ptr(), s.data_ptr(), e.dtype, s.dtype, e.shape, s.shape, e.is_contiguous(), s.is_contiguous()) for _, e, s in pairs]
            if sig != self._sig:
                self._sig, self._table = None, None
                self._table = self._build(pairs)
                self._sig = sig
            table, n = self._table
            with torch.cuda.device(table.device):
                _lib.check(_lib.lib().cvb_ema_update(table.data_ptr(), n, d, 1 - d, _stream()), 'cvb_ema_update')

    def update_attr(self, model, include=(), exclude=('process_group', 'reducer')):
        copy_attr(self.ema, model, include, exclude)
