"""tests/golden/ema.npz: the REFERENCE's ModelEMA (src/utils/ema.py) on the CPU over oracle/ema_oracle.fixture_model().

  CVPYTORCH_REFERENCE=<reference checkout> python tools/make_golden_ema.py

For each of oracle/ema_oracle.SCENARIOS (name, updates at construction, n updates): the model's state is drawn from SEED + scenario index,
the reference ModelEMA is built over it, and before each of the n updates the model gets a new "trained" state (the previous one plus
seeded noise, num_batches_tracked advanced).  Stored, per scenario s and step i: `s:init:<key>` (the model at construction),
`s:src{i}:<key>` (the model at update i), `s:ema{i}:<key>` (the reference EMA after update i), `s:decay{i}` and `s:updates{i}`, plus the
seeds.  The reference's tensor-times-scalar ops round the same way on the CPU and the GPU, so the expected states are exact on both."""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ema_oracle as O  # noqa: E402

SEED = 4242


def _reference_ema():
    ref = os.environ.get('CVPYTORCH_REFERENCE', '')
    spec = importlib.util.spec_from_file_location('ref_ema', os.path.join(ref, 'src', 'utils', 'ema.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.ModelEMA


def _state(model, g, base=None):
    """A seeded state: base + noise (or noise alone), positive running_var, num_batches_tracked one step further."""
    sd = {}
    for k, v in model.state_dict().items():
        if not v.dtype.is_floating_point:
            sd[k] = v + 1
            continue
        noise = torch.randn(v.shape, generator=g) * 0.5
        sd[k] = (base[k] + 0.1 * noise) if base is not None else noise
        if k.endswith('running_var'):
            sd[k] = sd[k].abs() + 0.1
    return sd


def main():
    RefEMA = _reference_ema()
    out = {'seed': np.array([SEED])}
    for si, (name, start, n) in enumerate(O.SCENARIOS):
        g = torch.Generator().manual_seed(SEED + si)
        model = O.fixture_model()
        model.load_state_dict(_state(model, g))
        ref, ora = RefEMA(model, updates=start), O.ModelEMA(model, updates=start)
        out.update({f'{name}:init:{k}': v.numpy().copy() for k, v in model.state_dict().items()})
        for i in range(n):
            model.load_state_dict(_state(model, g, model.state_dict()))
            ref.update(model)
            ora.update(model)
            assert ref.updates == ora.updates == start + i + 1 and ref.decay(ref.updates) == ora.decay(ora.updates)
            for k, v in ref.ema.state_dict().items():  # the oracle restatement must reproduce the reference before the fixture is written
                assert torch.equal(v, ora.ema.state_dict()[k]), (name, i, k)
            out.update({f'{name}:src{i}:{k}': v.numpy().copy() for k, v in model.state_dict().items()})
            out.update({f'{name}:ema{i}:{k}': v.numpy().copy() for k, v in ref.ema.state_dict().items()})
            out[f'{name}:decay{i}'] = np.array(ref.decay(ref.updates), dtype=np.float64)
            out[f'{name}:updates{i}'] = np.array(ref.updates)
        print(name, 'updates', start + 1, '..', start + n, 'decays', [float(out[f'{name}:decay{i}']) for i in range(n)])
    np.savez_compressed(os.path.join(ROOT, 'tests/golden/ema.npz'), **out)


if __name__ == '__main__':
    main()
