"""Whole-backbone training (cvpytorch_b200.train.CSPDarknet, Focus, SPPF) without a GPU: the oracle against the reference fixture, the
drop-in's module tree, the configurations it refuses, and the host-side argument checks of the new and widened C entry points."""
import ast
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def test_darknet_train_oracle_reproduces_reference_fixture():
    """oracle/darknet_train_oracle.py (functional Focus, SPPF, CSPDarknet, torch.autograd) vs the reference's own CSPDarknet in fp32:
    outputs, every parameter gradient and the running statistics after the step, <= 1e-5.  The parameters, image and output gradients
    are regenerated from the fixture's seeds; the key list is the reference's and must equal the training drop-in's."""
    from oracle import darknet_train_oracle as DO
    g = np.load(os.path.join(GOLD, 'darknet_train.npz'))
    keys, sd, x, Gs, oc = DO.fixture_inputs(g)
    outs, grads, stats = DO.train_step(x, Gs, sd, subtype='cspdark_n', out_channels=oc)
    errs = {f'y{i}': _rel(o, g[f'y{i}']) for i, o in enumerate(outs)}
    for k, v in grads.items():
        errs['grad ' + k] = _rel(v, g[f'grad_{k}'])
    for k, v in stats.items():
        errs['after ' + k] = _rel(v, g[f'after_{k}'])
    from cvpytorch_b200 import train as T
    assert list(T.CSPDarknet('cspdark_n', out_channels=oc).state_dict().keys()) == keys
    assert len([k for k in errs if k.startswith('grad ')]) == sum(1 for k in keys if 'running_' not in k and 'num_batches' not in k)
    worst = max(errs, key=errs.get)
    assert errs[worst] <= 1e-5, (worst, errs[worst])


def test_training_csp_darknet_keys_match_reference_and_inference_module():
    """CSPDarknet('cspdark_s'): the 210 backbone.* keys and shapes of tests/golden/yolox_keys.npz (dumped from the reference) and those of
    the inference drop-in; every BatchNorm has eps 1e-3 and momentum 0.03."""
    from cvpytorch_b200 import train as T, yolox_models as Y
    g = np.load(os.path.join(GOLD, 'yolox_keys.npz'))
    ref = {str(k)[len('backbone.'):]: tuple(ast.literal_eval(str(s))) for k, s in zip(g['keys'], g['shapes']) if str(k).startswith('backbone.')}
    m = T.CSPDarknet('cspdark_s')
    sd = m.state_dict()
    assert len(sd) == 210
    got = {k: tuple(v.shape) for k, v in sd.items()}
    assert got == {k: ref[k] for k in got} and set(got) == set(ref)
    inf = {k: tuple(v.shape) for k, v in Y.CSPDarknet('cspdark_s').state_dict().items()}
    assert list(got) == list(inf) and got == inf
    bns = [mod for mod in m.modules() if isinstance(mod, torch.nn.BatchNorm2d)]
    assert len(bns) == 35 and all(b.eps == 1e-3 and b.momentum == 0.03 for b in bns)
    assert m.out_channels == [128, 256, 512]


@pytest.mark.parametrize('kw', [dict(subtype='cspdark_t'), dict(subtype='cspdark_m'), dict(subtype='cspdark_x'), dict(depthwise=True),
                                dict(norm_eval=True), dict(frozen_stages=0), dict(spp_ksizes=(3, 5, 7)), dict(spp_ksizes=5)])
def test_training_csp_darknet_refuses_unsupported_configurations(kw):
    from cvpytorch_b200 import train as T
    with pytest.raises(NotImplementedError):
        T.CSPDarknet(**kw)


def test_training_csp_darknet_supported_widths_and_cpu_refusal():
    from cvpytorch_b200 import _lib, train as T
    for sub in ('cspdark_n', 'cspdark_s', 'cspdark_l'):
        T.CSPDarknet(sub)
    T.BaseConv(16, 32, 3, 1)
    T.BaseConv(32, 64, 3, 2)
    for c in (24, 48, 96):
        with pytest.raises(NotImplementedError):
            T.BaseConv(c, 64, 1, 1)
        with pytest.raises(NotImplementedError):
            T.BaseConv(64, c, 1, 1)
    m = T.CSPDarknet('cspdark_n').train()
    with pytest.raises(_lib.CvbError):
        m(torch.zeros(1, 3, 64, 64))  # CPU tensor: no fallback
    m.eval()
    with pytest.raises(RuntimeError):
        m(torch.zeros(1, 3, 64, 64))


def test_training_c_abi_narrow_widths_focus_and_pool_arguments():
    """Widths 24, 48 and 96 stay rejected by every training convolution entry point; the Focus kernel rejects odd H or W, the pool kernels
    C % 8 != 0 -- on the host, before the device is touched."""
    from cvpytorch_b200 import _lib
    L = _lib.lib()
    one = ctypes.c_void_p(16)
    for c in (24, 48, 96):
        assert L.cvb_train_conv(one, 1, 8, 8, c, one, 64, 1, 1, one, None, None, None) != 0
        assert b'multiples of 64' in L.cvb_last_error_string()
        assert L.cvb_train_conv(one, 1, 8, 8, 64, one, c, 3, 1, one, None, None, None) != 0
        assert b'multiples of 64' in L.cvb_last_error_string()
        assert L.cvb_train_conv_wgrad(one, one, 1, 8, 8, c, 32, 3, 1, one, None) != 0
        assert b'multiples of 64' in L.cvb_last_error_string()
        assert L.cvb_train_conv_dgrad_s2(one, 1, 4, 4, 32, one, c, 8, 8, one, None, None, None) != 0
        assert b'multiples of 64' in L.cvb_last_error_string()
        assert L.cvb_train_pack_weights(one, c, 16, 3, one, one, None) != 0
        assert b'multiples of 64' in L.cvb_last_error_string()
    for H, W in ((7, 8), (8, 9)):
        assert L.cvb_train_focus_s2d(one, 1, H, W, one, None) != 0
        assert b'even' in L.cvb_last_error_string()
    for C in (4, 12, 20):
        assert L.cvb_train_spp_pool_fwd(one, 1, 8, 8, C, one, one, None) != 0
        assert b'multiple of 8' in L.cvb_last_error_string()
        assert L.cvb_train_spp_pool_bwd(one, one, 1, 8, 8, C, one, None) != 0
        assert b'multiple of 8' in L.cvb_last_error_string()
