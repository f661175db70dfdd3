"""The YOLOv6 oracle (oracle/yolov6_oracle.py) against the reference's own outputs (tests/golden/yolov6_*.npz, tools/make_golden_yolov6.py):
network, decode and NMS; and the claim the H100 path rests on -- on objectness-1 predictions the YOLOv6 NMS keeps exactly the rows and
scores of the YOLOv5 NMS (oracle.nms_oracle)."""
import os

import numpy as np
import pytest
import torch

from oracle import nms_oracle as NO
from oracle import yolov6_oracle as V6

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
SEEDS = {'n': 606, 's': 616}
NMS_CASES = [('few', 0.03), ('typical', 0.03), ('typical', 0.25), ('capped', 0.03)]


def _keys():
    return np.load(os.path.join(GOLD, 'yolov6_keys.npz'))


def keys_shapes(stype):
    k = _keys()
    return [(str(a), tuple(int(t) for t in s.split(',')) if s else ()) for a, s in zip(k[f'{stype}_keys'], k[f'{stype}_shapes'])]


def seeded(stype):
    return V6.seeded_state_dict(keys_shapes(stype), SEEDS[stype])


def test_key_lists():
    k = _keys()
    for stype, params in (('n', 5058239), ('s', 20147343)):
        keys = list(k[f'{stype}_keys'])
        assert len(keys) == 757 and int(k[f'{stype}_params']) == params
        assert 'loss.0.proj' in keys and 'head.proj' in keys and 'head.proj_conv.weight' in keys
        assert {x.split('.')[0] for x in keys} == {'backbone', 'neck', 'head', 'loss'}
    # the two LOSS sections differ: n sets reg_max 0, s keeps the default 16
    sn, ss = dict(keys_shapes('n')), dict(keys_shapes('s'))
    assert sn['loss.0.proj'] == (1,) and ss['loss.0.proj'] == (17,)


def oracle_tensors(z, d):
    return dict([(f'backbone_{i}', t) for i, t in enumerate(d['backbone'])] + [(f'neck_{i}', t) for i, t in enumerate(d['neck'])] +
                [(f'stems_{i}', t) for i, t in enumerate(d['stems'])] + [('cls', d['cls']), ('reg', d['reg']), ('z', z)])


def sample_err(t, f, key):
    """error of t's fixture samples against the reference's, relative to the reference tensor's max|t|"""
    return float((V6.subsample(t).double() - torch.from_numpy(f[key + '_sample']).double()).abs().max() / float(f[key + '_max']))


@pytest.mark.parametrize('stype', ['n', 's'])
def test_oracle_forward_128(stype):
    f = np.load(os.path.join(GOLD, 'yolov6_fwd128.npz'))
    z, d = V6.forward(V6.fixture_input(V6.FWD_SEED, V6.FWD_SHAPE), seeded(stype))
    for name, t in oracle_tensors(z, d).items():
        assert sample_err(t, f, f'{stype}_{name}') < 1e-5, name
        assert abs(float(t.abs().max()) / float(f[f'{stype}_{name}_max']) - 1) < 1e-5, name
    assert V6.rel_err(d['reg'], f[f'{stype}_reg']) < 1e-5


def test_oracle_decode_exact():
    """On the reference's own distances the oracle decode reproduces the reference's box and objectness columns bit for bit."""
    f = np.load(os.path.join(GOLD, 'yolov6_fwd128.npz'))
    for stype in ('n', 's'):
        reg = torch.from_numpy(f[f'{stype}_reg'])
        z = V6.detect(torch.zeros(reg.shape[:2] + (80,)), reg, [(16, 16), (8, 8), (4, 4)])
        assert np.array_equal(z[..., :5].numpy(), f[f'{stype}_z_box'])


def test_oracle_nms_320():
    """The oracle NMS on the reference's 320² z (its boxes and candidate scores) gives the reference's rows; the oracle network's z matches."""
    p = np.load(os.path.join(GOLD, 'yolov6_post320.npz'))
    zs = V6.dense_from_candidates(p['boxes'], p['rows'], p['classes'], p['scores'], 80)
    det, _ = V6.non_max_suppression(zs, 0.03, 0.65)[0]
    assert det.shape[0] > 0 and np.array_equal(det, p['det'])
    z, _ = V6.forward(V6.fixture_input(V6.POST_SEED, V6.POST_SHAPE), seeded('s'))
    assert float((z[..., :4] - torch.from_numpy(p['boxes'])).abs().max()) < 1e-5 * float(p['z_max'])
    r = torch.from_numpy(p['rows'].astype(np.int64))
    got = z[r[:, 0], r[:, 1], torch.from_numpy(p['classes'].astype(np.int64)) + 5]
    assert float((got - torch.from_numpy(p['scores'])).abs().max()) < 1e-5 * float(p['z_max'])


def test_oracle_nms_stress():
    g = np.load(os.path.join(GOLD, 'yolov6_nms.npz'))
    for k, (regime, conf) in enumerate(NMS_CASES):
        pred = NO.make_stress_prediction(2, A=4200, nc=20, regime=regime, seed=40 + k)
        pred[:, :, 4] = 1.0
        for b, (det, _) in enumerate(V6.non_max_suppression(pred, conf, 0.65)):
            assert np.array_equal(det, g[f'case{k}_det{b}']), (regime, conf, b)


@pytest.mark.parametrize('k', range(len(NMS_CASES)))
def test_yolov6_nms_equals_yolov5_nms_on_objectness_one(k):
    """obj = 1: YOLOv6's extra `max cls > conf` filter only drops rows without a class above conf, and cls *= 1 is exact, so the YOLOv5 NMS
    (the device kernel's semantics) keeps the same rows, scores and indices."""
    regime, conf = NMS_CASES[k]
    pred = NO.make_stress_prediction(2, A=4200, nc=20, regime=regime, seed=40 + k)
    pred[:, :, 4] = 1.0
    for (d6, i6), (d5, i5) in zip(V6.non_max_suppression(pred, conf, 0.65), NO.non_max_suppression(pred, conf, 0.65, multi_label=True)):
        assert np.array_equal(d6, d5) and np.array_equal(i6, i5)
    p = np.load(os.path.join(GOLD, 'yolov6_post320.npz'))
    z = V6.dense_from_candidates(p['boxes'], p['rows'], p['classes'], p['scores'], 80)
    for (d6, i6), (d5, i5) in zip(V6.non_max_suppression(z, 0.03, 0.65), NO.non_max_suppression(z, 0.03, 0.65, multi_label=True)):
        assert np.array_equal(d6, d5) and np.array_equal(i6, i5)
