"""Drop-in for the trainer's optimiser (src/optimizers/__init__.py build_optimizer with OPTIMIZER.TYPE 'SGD'): ``SGD``, a
``torch.optim.SGD`` whose ``step()`` updates every parameter of every group in ONE kernel launch (csrc/sgd.cu, ``cvb_sgd_step``) and never
synchronises the host, instead of a Python loop of foreach launches per group.

Under ``torch.amp.GradScaler`` the step takes the scaler's ``grad_scale`` and ``found_inf`` on the device (``_step_supports_amp_scaling``):
the kernel unscales the gradients as it reads them and does nothing when ``found_inf`` is set, so ``scaler.step(opt)`` skips its
``found_inf.item()``.  After an explicit ``scaler.unscale_(opt)`` (gradient clipping) only ``found_inf`` is passed.  Params, momentum
buffers and the scaler's scale are bitwise those of ``torch.optim.SGD`` + ``GradScaler`` on the same GPU.

Whether a parameter's momentum buffer holds a value is kept on the device (a skipped first step creates none in the reference, and the host
cannot know about the skip without a sync).  ``state`` holds a ``momentum_buffer`` for every parameter with momentum that has had a
gradient at a step; ``state_dict()`` reads the flags (one sync) and emits ``momentum_buffer`` exactly where the reference has one, so the
state dicts of this class and of ``torch.optim.SGD`` load into each other.

The contents of ``p.grad`` after ``step()`` are not part of the contract (the trainer zeroes them next): this step leaves them as they
were, while the reference leaves them unscaled, and overwritten by the Nesterov term in groups without weight decay.

What the kernel cannot run raises before any launch, with no fallback: ``dampening != 0``, ``maximize``, ``fused``, ``differentiable``,
tensor hyper-parameters, sparse gradients, params or gradients that are not fp32 or not contiguous, a gradient shaped unlike its param,
params that overlap in memory, and more than ``CVB_SGD_MAX_GROUPS`` groups (NotImplementedError); CPU tensors, or params, gradients,
``grad_scale`` and ``found_inf`` on more than one device (CvbError).

The device table of (param, grad, momentum buffer, flags) entries is rebuilt when any entry's tensors change address, dtype, shape or
device, when a group's momentum turns on or off, or when the set of params with a gradient changes; ``table_builds`` counts the builds.
"""
import torch

from . import _lib
from ._lib import _p, _stream


def _refuse(group, gi):
    for key, bad in (('dampening', group['dampening'] != 0), ('maximize', group['maximize']), ('fused', group['fused']),
                     ('differentiable', group['differentiable'])):
        if bad:
            raise NotImplementedError(f'SGD (H100): group {gi} sets {key}={group[key]!r}; the one-launch step has no such path')
    for key in ('lr', 'momentum', 'weight_decay'):
        if isinstance(group[key], torch.Tensor):
            raise NotImplementedError(f'SGD (H100): group {gi} has a tensor {key}; the step takes Python numbers by value')


def _check_entry(p, g):
    if p.dtype != torch.float32 or g.dtype != torch.float32:
        raise NotImplementedError(f'SGD (H100): a param of {p.dtype} with a gradient of {g.dtype}; only fp32 is stepped')
    if not (p.is_contiguous() and g.is_contiguous()):
        raise NotImplementedError('SGD (H100): a param or its gradient is not contiguous')
    if p.shape != g.shape:
        raise NotImplementedError(f'SGD (H100): a gradient of shape {tuple(g.shape)} for a param of shape {tuple(p.shape)}')


def _overlapping(params):
    """True if two params share memory (the reference would step it twice)."""
    spans = sorted((p.data_ptr(), p.data_ptr() + 4 * p.numel()) for p in params if p.numel())
    end = -1
    for start, stop in spans:
        if start < end:
            return True
        end = max(end, stop)
    return False


def _flag_count(numel):
    return max(1, -(-numel // _lib.CVB_SGD_CHUNK))


class SGD(torch.optim.SGD):
    """torch.optim.SGD with the same constructor, param_groups, state, state_dict / load_state_dict, add_param_group and zero_grad, whose
    step() is one kernel launch on the current stream of the params' device."""

    _step_supports_amp_scaling = True

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._flags = {}  # param -> (its momentum buffer, int32 device flags: 1 per CVB_SGD_CHUNK elements where the buffer holds a value)
        self._checked = None  # the (param, grad) signature last checked
        self._sig = None      # what the table was built from: that signature and the momentum buffers' addresses
        self._table = None    # (device table, entry count)
        self.table_builds = 0

    def _momentum_buffer(self, p):
        """The param's buffer and its flags.  A buffer this optimiser did not allocate (load_state_dict, or state set by hand) holds a value."""
        state = self.state[p]
        buf = state.get('momentum_buffer')
        known = self._flags.get(p)
        if known is not None and known[0] is buf:
            return known
        if buf is None:
            buf = state['momentum_buffer'] = torch.empty_like(p, memory_format=torch.contiguous_format)
            flags = torch.zeros(_flag_count(p.numel()), dtype=torch.int32, device=p.device)
        else:
            if buf.dtype != torch.float32 or not buf.is_contiguous() or buf.shape != p.shape or buf.device != p.device:
                raise NotImplementedError('SGD (H100): a loaded momentum_buffer is not an fp32 contiguous tensor shaped as its param')
            flags = torch.ones(_flag_count(p.numel()), dtype=torch.int32, device=p.device)
        self._flags[p] = (buf, flags)
        return buf, flags

    @staticmethod
    def _check(entries, grad_scale, found_inf):
        for p, g, _, _ in entries:
            _check_entry(p, g)
        if _overlapping([p for p, _, _, _ in entries]):
            raise NotImplementedError('SGD (H100): two params share memory (the reference would step it twice)')
        devices = {t.device for p, g, _, _ in entries for t in (p, g)} | {t.device for t in (grad_scale, found_inf) if t is not None}
        if any(d.type != 'cuda' for d in devices):
            raise _lib.CvbError('SGD: a param, gradient or GradScaler tensor is on the CPU; the H100 step has no CPU fallback')
        if len(devices) > 1:
            raise _lib.CvbError(f'SGD: params, gradients, grad_scale and found_inf must live on one device (found {sorted(map(str, devices))})')

    def _build(self, entries, n_groups):
        rows = []
        for p, g, gi, mom in entries:
            buf, flags = self._flags[p] if mom else (None, None)
            rows.append(_lib.CvbSgdEntry(p.data_ptr(), g.data_ptr(), buf.data_ptr() if buf is not None else None,
                                         flags.data_ptr() if flags is not None else None, p.numel(), gi))
        dev = entries[0][0].device
        with torch.cuda.device(dev):
            table = torch.empty((len(rows) * _lib.CVB_SGD_TABLE_ENTRY_BYTES,), dtype=torch.uint8, device=dev)
            _lib.check(_lib.lib().cvb_sgd_table_upload((_lib.CvbSgdEntry * len(rows))(*rows), len(rows), n_groups, table.data_ptr(),
                                                       _stream()), 'cvb_sgd_table_upload')
        self.table_builds += 1
        return table, len(rows)

    @torch.no_grad()
    def step(self, closure=None):
        """One SGD step over every param with a gradient, in one launch; with GradScaler's grad_scale / found_inf when it set them."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        groups = self.param_groups
        if len(groups) > _lib.CVB_SGD_MAX_GROUPS:
            raise NotImplementedError(f'SGD (H100): {len(groups)} param groups; the step passes at most {_lib.CVB_SGD_MAX_GROUPS} by value')
        entries, sig, hyper = [], [], []
        for gi, group in enumerate(groups):
            _refuse(group, gi)
            mom = group['momentum'] != 0
            hyper.append(_lib.CvbSgdGroup(group['lr'], group['weight_decay'], group['momentum'],
                                          (_lib.CVB_SGD_NESTEROV if group['nesterov'] else 0) |
                                          (_lib.CVB_SGD_WEIGHT_DECAY if group['weight_decay'] != 0 else 0) |
                                          (_lib.CVB_SGD_MOMENTUM if mom else 0)))
            for p in group['params']:
                g = p.grad
                if g is None:
                    continue
                if g.is_sparse:
                    raise NotImplementedError('SGD (H100): sparse gradients are not stepped')
                entries.append((p, g, gi, mom))
                sig.append((p.data_ptr(), g.data_ptr(), p.dtype, g.dtype, p.shape, g.shape, p.device, g.device, p.is_contiguous(),
                            g.is_contiguous(), gi, mom))
        if not entries:
            return loss
        grad_scale, found_inf = getattr(self, 'grad_scale', None), getattr(self, 'found_inf', None)
        if sig != self._checked:
            self._checked = None
            self._check(entries, grad_scale, found_inf)
            self._checked = sig
        for t in (grad_scale, found_inf):
            if t is not None and t.device != entries[0][0].device:
                raise _lib.CvbError(f'SGD: grad_scale / found_inf on {t.device}, the params on {entries[0][0].device}')
        bufs = [self._momentum_buffer(p)[0].data_ptr() if mom else None for p, _, _, mom in entries]
        if (sig, bufs) != self._sig:
            self._sig, self._table = None, None
            self._table = self._build(entries, len(groups))
            self._sig = (sig, bufs)
        table, n = self._table
        with torch.cuda.device(table.device):
            _lib.check(_lib.lib().cvb_sgd_step(table.data_ptr(), n, (_lib.CvbSgdGroup * len(hyper))(*hyper), len(hyper),
                                               _p(grad_scale), _p(found_inf), _stream()), 'cvb_sgd_step')
        return loss

    def state_dict(self):
        """torch.optim.SGD's state dict, with a momentum_buffer only where a step that was not skipped has written it (one sync)."""
        sd = super().state_dict()
        params = [p for group in self.param_groups for p in group['params']]
        held = [(i, self._flags[p][1]) for i, p in enumerate(params) if p in self._flags and self._flags[p][0] is self.state[p].get('momentum_buffer')]
        unset = {i for (i, _), v in zip(held, torch.cat([f[:1] for _, f in held]).tolist() if held else []) if not v}
        for i in unset:
            st = {k: v for k, v in sd['state'][i].items() if k != 'momentum_buffer'}
            if st:
                sd['state'][i] = st
            else:
                del sd['state'][i]
        return sd
