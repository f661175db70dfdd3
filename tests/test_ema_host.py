"""The model EMA drop-in without a GPU: the oracle against tests/golden/ema.npz, the decay / updates bookkeeping and the .ema copy, the host
checks of the C ABI, every refusal of ModelEMA.update, and deepcopy / pickle of drop-in models whose graph caches hold C handles."""
import copy
import ctypes
import os
import pickle
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _fixture_state(f, prefix):
    return {k[len(prefix):]: torch.from_numpy(f[k].copy()) for k in f.files if k.startswith(prefix)}


def test_oracle_reproduces_the_reference_fixture_bit_for_bit():
    from oracle import ema_oracle as O
    f = np.load(os.path.join(ROOT, 'tests', 'golden', 'ema.npz'))
    for name, start, n in O.SCENARIOS:
        ema = _fixture_state(f, f'{name}:init:')
        assert 'num_batches_tracked' in ''.join(ema)
        for i in range(n):
            assert int(f[f'{name}:updates{i}']) == start + i + 1
            d = O.decay_at(start + i + 1)
            assert d == float(f[f'{name}:decay{i}'])
            O.update_(ema, _fixture_state(f, f'{name}:src{i}:'), d)
            want = _fixture_state(f, f'{name}:ema{i}:')
            assert list(ema) == list(want)
            for k in want:
                assert torch.equal(ema[k], want[k]), (name, i, k)


def test_decay_updates_and_the_ema_copy_follow_the_reference():
    from cvpytorch_b200.ema import ModelEMA
    from oracle import ema_oracle as O
    model = O.fixture_model().train()
    for decay, updates in ((0.9999, 0), (0.999, 1234), (0.5, 10 ** 6)):
        mine, ref = ModelEMA(model, decay=decay, updates=updates), O.ModelEMA(model, decay=decay, updates=updates)
        assert mine.updates == ref.updates == updates and isinstance(mine.updates, int)
        for x in (0, 1, 2, 1999, 2000, 12345, 10 ** 7):
            assert mine.decay(x) == ref.decay(x)
        assert not mine.ema.training and all(not m.training for m in mine.ema.modules())
        assert all(not p.requires_grad for p in mine.ema.parameters())
        assert mine.ema is not model and all(a is not b for a, b in zip(mine.ema.parameters(), model.parameters()))
        assert all(torch.equal(a, b) for a, b in zip(mine.ema.state_dict().values(), model.state_dict().values()))
    assert model.training and all(p.requires_grad for p in model.parameters())
    # DataParallel wraps: the EMA copies the inner module
    assert type(ModelEMA(nn.DataParallel(model)).ema) is nn.Sequential

    ema = ModelEMA(model)
    model.custom, model._private, model.process_group = 3, 4, 5
    ema.update_attr(model)
    assert ema.ema.custom == 3 and not hasattr(ema.ema, '_private') and not hasattr(ema.ema, 'process_group')
    model.other = 6
    ema.update_attr(model, include=('other',))
    assert ema.ema.other == 6


def test_c_abi_rejects_bad_arguments_before_touching_the_device():
    from cvpytorch_b200 import _lib
    L = _lib.lib()
    table, odd = ctypes.c_void_p(256), ctypes.c_void_p(264)

    def rejects(rc, what):
        assert rc != 0
        assert what in L.cvb_last_error_string()

    def entries(*rows):
        return (_lib.CvbEmaEntry * len(rows))(*[_lib.CvbEmaEntry(*r) for r in rows])

    good = entries((256, 512, 10))
    rejects(L.cvb_ema_table_upload(None, 1, table, None), b'null pointer')
    rejects(L.cvb_ema_table_upload(good, 1, None, None), b'null pointer')
    for n in (0, -1):
        rejects(L.cvb_ema_table_upload(good, n, table, None), b'n_entries must be > 0')
    rejects(L.cvb_ema_table_upload(good, 1, odd, None), b'16-byte aligned')
    rejects(L.cvb_ema_table_upload(entries((256, 512, 10), (256, 512, -1)), 2, table, None), b'entry 1 has numel -1 < 0')
    rejects(L.cvb_ema_table_upload(entries((None, 512, 10)), 1, table, None), b'entry 0 has a null pointer')
    rejects(L.cvb_ema_table_upload(entries((256, 512, 0), (256, None, 3)), 2, table, None), b'entry 1 has a null pointer')
    rejects(L.cvb_ema_update(None, 1, 0.5, 0.5, None), b'null pointer')
    for n in (0, -3):
        rejects(L.cvb_ema_update(table, n, 0.5, 0.5, None), b'n_entries must be > 0')
    rejects(L.cvb_ema_update(odd, 1, 0.5, 0.5, None), b'16-byte aligned')


def test_update_refusals():
    """Every refusal of ModelEMA.update raises before any launch; the tensors stay as they were."""
    from cvpytorch_b200 import _lib
    from cvpytorch_b200.ema import ModelEMA
    from oracle import ema_oracle as O

    def attempt(model, ema_edit=None, exc=NotImplementedError, match=''):
        ema = ModelEMA(model)
        if ema_edit:
            ema_edit(ema.ema)
        before = {k: v.clone() for k, v in ema.ema.state_dict().items()}
        with pytest.raises(exc, match=match):
            ema.update(model)
        assert all(torch.equal(v, before[k]) for k, v in ema.ema.state_dict().items())

    attempt(O.fixture_model(), exc=_lib.CvbError, match='no CPU fallback')
    attempt(O.fixture_model().double(), match='only fp32')
    attempt(O.fixture_model(), ema_edit=lambda e: setattr(e[0].weight, 'data', e[0].weight.data.transpose(2, 3)), match='not contiguous')
    tied = O.fixture_model()
    tied[3].weight = nn.Parameter(torch.zeros(8, 8, 1, 1))
    tied[3].bias = nn.Parameter(torch.zeros(8))
    tied[1].weight = tied[3].bias  # one tensor under two keys: the reference would update it twice
    attempt(tied, match='share memory')
    missing = O.fixture_model()
    ema = ModelEMA(missing)
    ema.ema.add_module('extra', nn.Linear(2, 2))
    with pytest.raises(KeyError):
        ema.update(missing)
    shaped = O.fixture_model()
    attempt(shaped, ema_edit=lambda e: setattr(e[3], 'bias', nn.Parameter(torch.zeros(6))), match='has shape')


class _Plan:
    """Stands in for an ops.ConvPlan: a ctypes pointer, which copy.deepcopy and pickle refuse."""

    def __init__(self):
        self.handle = ctypes.c_void_p(5)


@pytest.mark.parametrize('kind', ['yolox', 'yolov5'])
def test_deepcopy_and_pickle_of_a_model_that_has_run(kind):
    from cvpytorch_b200 import models as M, synth, yolox_models as XM
    dictionary = [{f'c{i}': 1.0} for i in range(80)]
    m = (XM.YOLOX(dictionary=dictionary, model_cfg=dict(synth.YOLOX_CFG)) if kind == 'yolox' else
         M.YOLOv5(dictionary, dict(synth.YOLOV5S_CFG)))
    with pytest.raises(ValueError, match='pickled'):
        copy.deepcopy(_Plan())
    plan, sub = _Plan(), _Plan()
    m._graphs[((1, 3, 64, 64), 0)] = {'plans': [plan]}
    m.backbone._graphs[((1, 3, 64, 64), 0)] = sub
    bound = (('train modules',), [])
    m.__dict__['_train_modules'] = bound
    for c in (copy.deepcopy(m), pickle.loads(pickle.dumps(m))):
        assert c._graphs == {} and c.backbone._graphs == {} and c._train_modules is None
        assert set(c.__dict__) == set(m.__dict__)
        sd, csd = m.state_dict(), c.state_dict()
        assert list(sd) == list(csd) and all(torch.equal(sd[k], csd[k]) for k in sd)
        assert all(a is not b for a, b in zip(c.parameters(), m.parameters()))
    assert m._graphs[((1, 3, 64, 64), 0)]['plans'][0] is plan and m.backbone._graphs[((1, 3, 64, 64), 0)] is sub
    assert m._train_modules is bound
