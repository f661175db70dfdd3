"""SyncBatchNorm through the YOLOv6 training step: the RepVGG blocks (cvb_train_repvgg_bwd_reduce / _apply, one record per branch) and the
BatchNorm + ReLU ConvModules (cvb_train_bn_relu_bwd_reduce / _apply), the halves of the fused backward entries with a collective between.

Kernel level, one GPU, no collective: the shards of test_sync_bn_gpu.SHARDS (1 to 8 of them, shards of 1 and 2 pixels among them), each
branch's record from cvb_train_bn_partial, stacked and merged; each shard's reduce, the sums added in rank order in fp32 (what all_reduce
does), each shard's apply.  Against float64 of the whole tensor with fp64ref.bn_silu_bwd_check (dz = g * [a > 0] or g * [z > 0], exact in
bf16), whose summation bound gs covers the largest shard's addition chain plus one fp32 addition per shard; each shard's own sums against
its own chain.  The split fed the fused entry's own sums and count = npix equals the fused entry bitwise.  Every (npix, C, identity)
signature of the YOLOv6-s (64 x 640²) and YOLOv6-n (16 x 640²) steps runs through test_yolov6_train_launches_gpu's checks with the fused
entry replaced by its reduce -> apply split (a world of one), exact integer operands and Gaussian ones.

Module level, two ranks (gloo) sharing one GPU: YOLOv6-n and YOLOv5-s converted with convert_sync_batchnorm, each rank one image of a
2-image batch, against the oracle's fp32 step on the whole batch with the YOLOv6 / YOLOv5 network tests' rule (3 x the bf16-autocast error
+ 1e-2, max-normalised).  With per-rank statistics (the unconverted YOLOv6-n) the rule fails: the largest ratio was 8.7, with 132 entries
outside.  Measured on one H100 80GB HBM3 (SXM, 700 W power limit), the largest error / (3 x autocast error + 1e-2) was 0.814 for YOLOv6-n
in two runs and 0.436 for YOLOv5-s in one run.  The YOLOv6-n margin is the thinner one.

Trainer level: the reference trainer's step on a converted YOLOv6-n under DDP over two ranks.  The reference discards its class loss, so
head.cls_convs / head.cls_preds get no gradient; a plain DDP(model) then raises "Expected to have finished reduction in the prior iteration"
on its second step (confirmed on the CPU with gloo and oracle/yolov6_train_oracle.py), so the model is wrapped with
find_unused_parameters=True, as the reference's own YOLOv6 model would have to be."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fp64ref as R  # noqa: E402
import test_train_launches_gpu as TL  # noqa: E402
import test_yolov6_train_launches_gpu as L6  # noqa: E402
from test_sync_bn_gpu import SHARDS, _rank_main, _run_rank, _spawn  # noqa: E402
from test_yolov6_host import DICT, use_model  # noqa: E402
from test_yolov6_train_gpu import _batch, _modules, _randomise, _rel  # noqa: E402

pytestmark = pytest.mark.gpu
N_SYNC_BN = 128  # BatchNorms of YOLOv6-n / -s after conversion: 100 in 35 RepVGG blocks, 19 ReLU ConvModules, 9 SiLU head ConvModules


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _merged(ys, sizes, g):
    """Each shard of y [npix, C] -> its cvb_train_bn_partial record; the records merged -> (stat [4, C], fp32 gamma, count fp64 [1])."""
    from cvpytorch_b200 import _lib, train as T
    L = _lib.lib()
    C = ys.shape[1]
    recs = torch.empty((len(sizes), 2 * C + 1), dtype=torch.float64, device='cuda')
    scratch = torch.empty(2, C, device='cuda')
    for i, part in enumerate(torch.split(ys, sizes)):
        _lib.check(L.cvb_train_bn_partial(T._p(part), part.shape[0], C, T._p(scratch), T._p(recs[i]), T._stream()), 'partial')
    gamma, beta = torch.rand(C, generator=g, device='cuda') + 0.5, torch.randn(C, generator=g, device='cuda') * 0.5
    stat, count = torch.empty(4, C, device='cuda'), torch.empty(1, dtype=torch.float64, device='cuda')
    _lib.check(L.cvb_train_bn_merge(T._p(recs), len(sizes), C, T._p(gamma), T._p(beta), 1e-3, 0.03, None, None, T._p(stat), T._p(count), T._stream()),
               'merge')
    return stat, gamma, count


def _shard_sums_check(sums, dz, xhats, sizes, C, tag):
    """Each shard's sums [k][C] (row 0 = sum dz, rows 1.. = sum dz * xhat_b) against float64 with that shard's own chain bound."""
    u = R.U24
    bounds = np.cumsum([0] + sizes).tolist()
    for i, (a, b) in enumerate(zip(bounds, bounds[1:])):
        gs = (R.red_chain(b - a, C, _sms()) + 2) * u
        R.check(sums[i][0], dz[a:b].sum(0), gs * dz[a:b].abs().sum(0), f'{tag} shard {i} sum dz')
        for row, xh in xhats.items():
            dzx = dz[a:b] * xh[a:b]
            R.check(sums[i][row], dzx.sum(0), (gs + 3 * u) * dzx.abs().sum(0), f'{tag} shard {i} sums[{row}]')


def _total_gs(sizes, C):
    """Summation bound of the rank-ordered fp32 sum of the shards' sums: the longest shard chain plus one addition per shard."""
    return max((R.red_chain(n, C, _sms()) + 2) * R.U24 for n in sizes) + len(sizes) * R.U24


@pytest.mark.parametrize('shift', [0, 100])
@pytest.mark.parametrize('ident', [False, True])
@pytest.mark.parametrize('shards', list(SHARDS))
@pytest.mark.parametrize('C', [16, 32, 64, 128, 256, 512])
def test_repvgg_split_backward_vs_float64(cuda, C, shards, ident, shift):
    from cvpytorch_b200 import _lib, train as T
    L = _lib.lib()
    sizes = SHARDS[shards]
    npix = sum(sizes)
    g = torch.Generator(device='cuda').manual_seed(C * 1000 + npix + shift + ident)
    nb = 3 if ident else 2
    ys = [((torch.randn(npix, C, generator=g, device='cuda') * (1 + b) + shift) * (torch.rand(C, generator=g, device='cuda') + 0.5)).bfloat16()
          for b in range(nb)]
    st = [_merged(y, sizes, g) for y in ys]
    count = st[0][2]
    gout = torch.randn(npix, C, generator=g, device='cuda').bfloat16()
    P = T._p
    parts = [list(torch.split(t, sizes)) for t in ys + [gout]]
    opt = lambda t: P(t) if ident else None  # noqa: E731
    acts, sums = [], []
    for r in range(len(sizes)):
        y3, y1, xr, gr = parts[0][r], parts[1][r], parts[-2][r], parts[-1][r]
        a = torch.empty_like(y3)
        _lib.check(L.cvb_train_repvgg_fwd(P(y3), P(y1), opt(xr), y3.shape[0], C, P(st[0][0]), P(st[1][0]), opt(st[-1][0]), P(a), T._stream()), 'fwd')
        s = torch.full((4, C), float('nan'), device='cuda')
        _lib.check(L.cvb_train_repvgg_bwd_reduce(P(gr), P(a), P(y3), P(y1), opt(xr), y3.shape[0], C, P(st[0][0]), P(st[1][0]), opt(st[-1][0]), P(s),
                                                 T._stream()), 'reduce')
        acts.append(a)
        sums.append(s)
    total = torch.stack(sums).sum(0)  # (the all-reduce: fp32 additions in rank order)
    ds = [[torch.full_like(p, float('nan')) for p in parts[0]] for _ in range(3)]
    for r in range(len(sizes)):
        y3, y1, xr, gr = parts[0][r], parts[1][r], parts[-2][r], parts[-1][r]
        _lib.check(L.cvb_train_repvgg_bwd_apply(P(gr), P(acts[r]), P(y3), P(y1), opt(xr), y3.shape[0], C, P(st[0][0]), P(st[1][0]), opt(st[-1][0]),
                                                P(st[0][1]), P(st[1][1]), opt(st[-1][1]), P(total), P(count), P(ds[0][r]), P(ds[1][r]), opt(ds[2][r]),
                                                T._stream()), 'apply')
    torch.cuda.synchronize()
    assert float(count) == npix
    dz = (gout.float() * (torch.cat(acts).float() > 0)).to(torch.bfloat16)
    xhats = {1 + b: (ys[b].double() - st[b][0][0].double()) * st[b][0][1].double() for b in range(nb)}
    _shard_sums_check(sums, dz.double(), xhats, sizes, C, 'repvgg')
    if not ident:
        assert all(torch.equal(s[3], torch.zeros_like(s[3])) for s in sums)
    gs = _total_gs(sizes, C)
    r = {}
    for b in range(nb):
        r[b] = R.bn_silu_bwd_check(dz, 1, ys[b], st[b][1], st[b][0], torch.stack([total[0], total[1 + b]]), torch.cat(ds[b]), gs)
    print('worst error / bound', {b: {k: round(v, 3) for k, v in rb.items()} for b, rb in r.items()})


@pytest.mark.parametrize('shift', [0, 100])
@pytest.mark.parametrize('shards', list(SHARDS))
@pytest.mark.parametrize('C', [16, 32, 64, 128, 256, 512])
def test_bn_relu_split_backward_vs_float64(cuda, C, shards, shift):
    from cvpytorch_b200 import _lib, train as T
    L = _lib.lib()
    sizes = SHARDS[shards]
    npix = sum(sizes)
    g = torch.Generator(device='cuda').manual_seed(C * 1000 + npix + shift + 7)
    y = ((torch.randn(npix, C, generator=g, device='cuda') + shift) * (torch.rand(C, generator=g, device='cuda') + 0.5)).bfloat16()
    stat, gamma, count = _merged(y, sizes, g)
    gout = torch.randn(npix, C, generator=g, device='cuda').bfloat16()
    P = T._p
    yp, gp = list(torch.split(y, sizes)), list(torch.split(gout, sizes))
    sums = [torch.full((2, C), float('nan'), device='cuda') for _ in sizes]
    for ys, gs_, s in zip(yp, gp, sums):
        _lib.check(L.cvb_train_bn_relu_bwd_reduce(P(gs_), P(ys), ys.shape[0], C, P(stat), P(s), T._stream()), 'reduce')
    total = torch.stack(sums).sum(0)
    dys = [torch.full_like(p, float('nan')) for p in yp]
    for ys, gs_, d in zip(yp, gp, dys):
        _lib.check(L.cvb_train_bn_relu_bwd_apply(P(gs_), P(ys), ys.shape[0], C, P(stat), P(gamma), P(total), P(count), P(d), T._stream()), 'apply')
    torch.cuda.synchronize()
    dz = (gout.float() * (L6._z32(y, stat) > 0)).to(torch.bfloat16)  # (the forward's fp32 fma decides the mask)
    xhat = (y.double() - stat[0].double()) * stat[1].double()
    _shard_sums_check(sums, dz.double(), {1: xhat}, sizes, C, 'bn_relu')
    r = R.bn_silu_bwd_check(dz, 1, y, gamma, stat, total, torch.cat(dys), _total_gs(sizes, C))
    print('worst error / bound', {k: round(v, 3) for k, v in r.items()})


@pytest.mark.parametrize('ident', [False, True])
@pytest.mark.parametrize('C', [16, 64, 512])
def test_split_apply_equals_the_fused_entry_bitwise(cuda, C, ident):
    """The apply halves fed the fused entry's own sums and count = npix write the fused entry's dy bit for bit (same fp32 expressions, the
    same fp32 1 / N), for the RepVGG backward and BatchNorm + ReLU."""
    from cvpytorch_b200 import _lib, train as T
    L, P = _lib.lib(), T._p
    npix = 3 * 37 * 41
    g = torch.Generator(device='cuda').manual_seed(C + ident)
    ys = [((torch.randn(npix, C, generator=g, device='cuda') + i) * (1 + i)).bfloat16() for i in range(3)]
    gb = [(torch.rand(C, generator=g, device='cuda') + 0.5, torch.randn(C, generator=g, device='cuda') * 0.3) for _ in range(3)]
    st = [T.bn_stats(ys[i], *gb[i], torch.zeros(C, device='cuda'), torch.ones(C, device='cuda'), 1e-3, 0.03) for i in range(3)]
    gout = torch.randn(npix, C, generator=g, device='cuda').bfloat16()
    count = torch.full((1,), float(npix), dtype=torch.float64, device='cuda')
    opt = lambda t: P(t) if ident else None  # noqa: E731
    a = torch.empty_like(ys[0])
    _lib.check(L.cvb_train_repvgg_fwd(P(ys[0]), P(ys[1]), opt(ys[2]), npix, C, P(st[0][0]), P(st[1][0]), opt(st[2][0]), P(a), T._stream()), 'fwd')
    sums = torch.empty(4, C, device='cuda')
    fused = [torch.empty_like(a) for _ in range(3)]
    split = [torch.full_like(a, float('nan')) for _ in range(3)]
    common = (P(gout), P(a), P(ys[0]), P(ys[1]), opt(ys[2]), npix, C, P(st[0][0]), P(st[1][0]), opt(st[2][0]), P(st[0][1]), P(st[1][1]), opt(st[2][1]))
    _lib.check(L.cvb_train_repvgg_bwd(*common, P(sums), P(fused[0]), P(fused[1]), opt(fused[2]), T._stream()), 'fused')
    _lib.check(L.cvb_train_repvgg_bwd_apply(*common, P(sums), P(count), P(split[0]), P(split[1]), opt(split[2]), T._stream()), 'apply')
    for b in range(3 if ident else 2):
        assert torch.equal(fused[b], split[b]), b
    s2, dy_f, dy_s = torch.empty(2, C, device='cuda'), torch.empty_like(a), torch.full_like(a, float('nan'))
    _lib.check(L.cvb_train_bn_relu_bwd(P(gout), P(ys[0]), npix, C, P(st[0][0]), P(st[0][1]), P(s2), P(dy_f), T._stream()), 'relu fused')
    _lib.check(L.cvb_train_bn_relu_bwd_apply(P(gout), P(ys[0]), npix, C, P(st[0][0]), P(st[0][1]), P(s2), P(count), P(dy_s), T._stream()), 'relu apply')
    assert torch.equal(dy_f, dy_s)


# ------------------------------------------------------------------------------------------------ every real shape
class _SplitLib:
    """The loaded library with cvb_train_repvgg_bwd and cvb_train_bn_relu_bwd replaced by their reduce -> apply halves in a world of one
    (count = npix on the device), so that test_yolov6_train_launches_gpu's checks of the fused entries check the split."""

    def __init__(self, lib):
        self._lib, self._counts = lib, []

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def _count(self, npix):
        c = torch.full((1,), float(npix), dtype=torch.float64, device='cuda')
        self._counts.append(c)  # (kept until the check has synchronised)
        return c.data_ptr()

    def cvb_train_repvgg_bwd(self, g, a, y3, y1, x, npix, C, s3, s1, sid, g3, g1, gid, sums, dy3, dy1, dxid, stream):
        rc = self._lib.cvb_train_repvgg_bwd_reduce(g, a, y3, y1, x, npix, C, s3, s1, sid, sums, stream)
        return rc or self._lib.cvb_train_repvgg_bwd_apply(g, a, y3, y1, x, npix, C, s3, s1, sid, g3, g1, gid, sums, self._count(npix), dy3, dy1, dxid,
                                                          stream)

    def cvb_train_bn_relu_bwd(self, g, y, npix, C, stat, gamma, sums, dy, stream):
        rc = self._lib.cvb_train_bn_relu_bwd_reduce(g, y, npix, C, stat, sums, stream)
        return rc or self._lib.cvb_train_bn_relu_bwd_apply(g, y, npix, C, stat, gamma, sums, self._count(npix), dy, stream)


SPLIT_SIGS = [s for s in L6.LAUNCHES if s[0] in ('cvb_train_repvgg_bwd', 'cvb_train_bn_relu_bwd')]


@pytest.mark.parametrize('sig', SPLIT_SIGS, ids=[TL._id(s) for s in SPLIT_SIGS])
def test_split_at_every_real_shape(cuda, monkeypatch, sig):
    from cvpytorch_b200 import _lib
    split = _SplitLib(_lib.lib())
    monkeypatch.setattr(_lib, 'lib', lambda: split)
    L6._run(sig)


# ------------------------------------------------------------------------------------------------ ranks on one GPU (gloo)
def _family(name):
    """-> (model on cuda in train mode, images [2, ...], stand-in output gradients, oracle(x, state) -> outputs, state prefixes).  Seeded,
    so that every rank's process and the parent build the same weights."""
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(6)
    if name == 'yolov6_n':
        from oracle import yolov6_train_oracle as O
        m = _modules('n')
        _randomise(m, 5)
        x = torch.rand((2, 3, 64, 96), generator=g).cuda()
        A = 8 * 12 + 4 * 6 + 2 * 3
        Gs = [torch.randn((2, A, 3), generator=g).cuda(), torch.randn((2, A, 4), generator=g).cuda()]
        return m, x, Gs, lambda x_, sd: list(O.network(x_, sd)[1:]), ('backbone.', 'neck.', 'head.')
    from oracle import yolov5_train_oracle as O
    from test_yolov5_train_gpu import _model
    m = _model()
    x = torch.rand((2, 3, 128, 128), generator=g).cuda()
    Gs = [torch.randn((2, 255, 128 // s, 128 // s), generator=g).cuda() for s in (8, 16, 32)]
    return m, x, Gs, O.network, ('backbone.', 'neck.', 'detect.')


def _outputs(name, mods, x):
    a, b, c = mods
    outs = c.forward_nhwc(b.forward_nhwc(a.forward_nhwc(x)))
    return list(outs[1:]) if name == 'yolov6_n' else list(outs)


def _family_rank(rank, world, name, sync):
    """One training step of the network on this rank's image -> CPU {outputs, parameter gradients, running statistics}."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    m, x, Gs, _, prefixes = _family(name)
    if sync:
        m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m)
    mods = m._training_modules()
    n_sync = sum(isinstance(b, torch.nn.SyncBatchNorm) for tm in mods for b in tm.modules())
    part = slice(rank, rank + 1)
    outs = _outputs(name, mods, x[part])
    sum((o.float() * G[part]).sum() for o, G in zip(outs, Gs)).backward()
    res = {f'y{i}': o.detach().float() for i, o in enumerate(outs)}
    res.update({'grad_' + k: p.grad for k, p in m.named_parameters() if p.grad is not None})
    res.update({'after_' + k: v for k, v in m.state_dict().items() if 'running_' in k and k.startswith(prefixes)})
    return res, n_sync


def _two_ranks_vs_oracle(name, sync):
    """-> (the entries outside 3 x autocast error + 1e-2, the largest error / (3 x autocast error + 1e-2), running statistics bitwise equal
    across ranks, SyncBatchNorm layers)."""
    (r0, n0), (r1, _) = _spawn(_rank_main, 2, _family_rank, name, sync)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    m, x, Gs, oracle, prefixes = _family(name)
    state = {k: v.detach().clone() for k, v in m.state_dict().items() if k.startswith(prefixes)}
    nograd = ('running_', 'num_batches_tracked', 'proj', 'anchors')

    def oracle_step(autocast):
        sd = {k: v.clone().requires_grad_(v.dtype.is_floating_point and not any(s in k for s in nograd)) for k, v in state.items()}
        with torch.autocast('cuda', dtype=torch.bfloat16, enabled=autocast):
            outs = oracle(x, sd)
        sum((o.float() * G).sum() for o, G in zip(outs, Gs)).backward()
        r = {f'y{i}': o.detach().float().cpu() for i, o in enumerate(outs)}
        r.update({'grad_' + k: v.grad.cpu() for k, v in sd.items() if v.grad is not None})
        r.update({'after_' + k: v.cpu() for k, v in sd.items() if 'running_' in k})
        return r
    ref, auto = oracle_step(False), oracle_step(True)
    stats = [k for k in r0 if k.startswith('after_')]
    same = bool(stats) and all(torch.equal(r0[k], r1[k]) for k in stats)
    got = {k: r0[k] + r1[k] for k in r0 if k.startswith('grad_')}
    got.update({k: r0[k] for k in stats})
    ref_c, auto_c = {k: ref[k] for k in got}, {k: auto[k] for k in got}
    for rank, res in enumerate((r0, r1)):
        for k in (k for k in res if k.startswith('y')):
            got[f'rank{rank} {k}'], ref_c[f'rank{rank} {k}'], auto_c[f'rank{rank} {k}'] = res[k], ref[k][rank:rank + 1], auto[k][rank:rank + 1]
    assert set(got) == set(ref_c) and len(got) > len(stats)
    errs = {k: _rel(got[k], ref_c[k]) for k in got}
    au = {k: _rel(auto_c[k], ref_c[k]) for k in got}
    ratio = {k: errs[k] / (3 * au[k] + 1e-2) for k in got}
    bad = {k: (errs[k], au[k]) for k in got if ratio[k] > 1}
    return bad, max(ratio.values()), same, n0


def test_yolov6_two_ranks_match_the_full_batch_step(cuda):
    """YOLOv6-n converted (128 SyncBatchNorm layers), two gloo ranks on one GPU, one of 2 images each: each rank's head outputs match its
    half of the oracle's fp32 step, the sum of the ranks' gradients matches the oracle's, the running statistics match the oracle's and are
    bitwise equal across ranks.  With per-rank statistics the same comparison fails."""
    bad, worst, same, n_sync = _two_ranks_vs_oracle('yolov6_n', True)
    print('YOLOv6-n, synced: largest error / (3 x autocast error + 1e-2)', round(worst, 3))
    assert n_sync == N_SYNC_BN
    assert same and not bad, bad
    bad, worst, same, n_sync = _two_ranks_vs_oracle('yolov6_n', False)
    print('YOLOv6-n, per-rank statistics: largest ratio', round(worst, 3), len(bad), 'entries outside')
    assert n_sync == 0 and bad and not same


def test_yolov5_two_ranks_match_the_full_batch_step(cuda):
    """YOLOv5-s converted (its BaseConv-style layers sync through train._conv_bn_silu), two gloo ranks at 128², against
    oracle/yolov5_train_oracle.py's fp32 step on both images, with the YOLOv5 network tests' rule."""
    bad, worst, same, n_sync = _two_ranks_vs_oracle('yolov5_s', True)
    print('YOLOv5-s, synced: largest error / (3 x autocast error + 1e-2)', round(worst, 3), n_sync, 'SyncBatchNorm layers')
    assert n_sync > 0
    assert same and not bad, bad


class _SeqRecorder(TL._Recorder):
    """The launch recorder, keeping every cvb_train_* launch in order."""

    def __init__(self, lib):
        super().__init__(lib)
        self.seq = []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith('cvb_train_') or name.endswith('_workspace_bytes'):
            return fn

        def call(*args):
            self.seq.append(TL._signature(name, args))
            return fn(*args)
        return call


def _world_of_one_rank(rank, world):
    """The launches of one YOLOv6-n training step (model forward 'train' + backward), unconverted and converted in a world of one, and the
    collectives the converted step issued."""
    import torch.distributed as dist
    from cvpytorch_b200 import _lib
    plain = _modules('n')
    _randomise(plain, 3)
    synced = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(plain))
    imgs, targets = _batch(B=2, size=128, nc=3)
    calls = []
    real = {k: getattr(dist, k) for k in ('all_gather_into_tensor', 'all_reduce')}
    for k, fn in real.items():
        setattr(dist, k, lambda *a, _k=k, _fn=fn, **kw: (calls.append(_k), _fn(*a, **kw))[1])
    load = _lib.lib
    seqs = []
    try:
        for m in (plain, synced):
            rec = _SeqRecorder(load())
            _lib.lib = lambda: rec
            m(imgs, targets, 'train')['loss'].backward()
            torch.cuda.synchronize()
            _lib.lib = load
            seqs.append(rec.seq)
    finally:
        _lib.lib = load
        for k, fn in real.items():
            setattr(dist, k, fn)
    n_sync = sum(isinstance(b, torch.nn.SyncBatchNorm) for b in synced.modules())
    return {'same': seqs[0] == seqs[1], 'n': len(seqs[0]), 'collectives': len(calls), 'n_sync': n_sync}


def test_world_of_one_takes_the_local_path(cuda):
    """A converted YOLOv6-n in a one-rank process group issues exactly the launch sequence of the unconverted model, and no collective."""
    r = _spawn(_rank_main, 1, _world_of_one_rank)[0]
    assert r['n_sync'] >= N_SYNC_BN and r['n'] > 0
    assert r['same'] and r['collectives'] == 0, r


# ------------------------------------------------------------------------------------------------ the reference trainer's step under DDP
def _trainer_rank(rank, world, iters):
    """YOLOv6-n, convert_sync_batchnorm, DDP; the reference trainer's step on this rank's image of a fixed 2-image batch."""
    from torch.nn.parallel import DistributedDataParallel as DDP
    from cvpytorch_b200 import yolov6_models as M
    m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(M.YOLOv6(DICT, use_model('n')).cuda().train())
    assert sum(isinstance(b, torch.nn.SyncBatchNorm) for tm in m._training_modules() for b in tm.modules()) == N_SYNC_BN
    # broadcast_buffers off: the running statistics must agree without rank 0's copy; find_unused_parameters: the class branch gets no
    # gradient (the reference discards its class loss)
    ddp = DDP(m, device_ids=[0], broadcast_buffers=False, find_unused_parameters=True)
    imgs, targets = _batch(B=2, size=320)
    imgs, targets = imgs[rank:rank + 1], targets[rank:rank + 1]
    params = list(m.parameters())
    opt = torch.optim.SGD(params, lr=0.01, momentum=0.9)
    scaler = torch.amp.GradScaler('cuda', enabled=True)
    hist = []
    for _ in range(iters):
        with torch.autocast('cuda', enabled=True):
            losses = ddp(imgs, targets, 'train')
        scaler.scale(losses['loss']).backward()
        scaler.unscale_(opt)
        torch.nn.utils.clip_grad_norm_(params, 10.0)
        scaler.step(opt)
        scaler.update()
        opt.zero_grad(set_to_none=True)
        hist.append(float(losses['loss'].detach()))
    sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    m.eval()
    with torch.no_grad():
        got, _, cnt = m.predict(imgs)
        got, cnt = got.clone(), cnt.clone()
    fresh = M.YOLOv6(DICT, use_model('n'))
    fresh.load_state_dict(m.state_dict(), strict=True)
    fresh.cuda().eval()
    with torch.no_grad():
        want, _, wcnt = fresh.predict(imgs)
    return hist, sd, bool(torch.equal(cnt, wcnt) and torch.equal(got, want))


def test_trainer_steps_under_ddp(cuda):
    """Two gloo ranks on one GPU, one image each, 10 steps of autocast + GradScaler + clip + SGD: the loss falls on both ranks, parameters
    and running statistics stay bitwise identical across ranks, and eval() serves the trained weights as a fresh YOLOv6 loaded with the
    trained state_dict."""
    (h0, sd0, ok0), (h1, sd1, ok1) = _spawn(_rank_main, 2, _trainer_rank, 10)
    print('loss rank 0', [round(v, 4) for v in h0], 'rank 1', [round(v, 4) for v in h1])
    for hist in (h0, h1):
        assert all(np.isfinite(hist)) and np.mean(hist[-3:]) < hist[0], hist
    assert ok0 and ok1
    assert list(sd0) == list(sd1)
    diff = [k for k in sd0 if not torch.equal(sd0[k], sd1[k])]
    assert not diff, diff


def _graph_rank(rank, world):
    """The converted YOLOv6-n step (model forward 'train', backward, gradient all-reduce, SGD) with NCCL, one GPU per rank, captured as one
    CUDA graph and replayed."""
    import torch.distributed as dist
    from cvpytorch_b200 import yolov6_models as M
    torch.cuda.set_device(rank)
    m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(M.YOLOv6(DICT, use_model('n')).cuda().train())
    imgs, targets = _batch(B=2, size=128)
    imgs, targets = imgs[rank:rank + 1].cuda(), targets[rank:rank + 1]
    gt = m.pack_targets(imgs, targets)
    params = [p for p in m.parameters() if p.requires_grad]
    opt = torch.optim.SGD(params, lr=0.01, momentum=0.9)

    def step():
        loss = m(imgs, gt, 'train')['loss']
        loss.backward()
        for p in params:
            if p.grad is not None:
                dist.all_reduce(p.grad)
                p.grad /= world
        opt.step()
        opt.zero_grad(set_to_none=False)
        return loss
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_loss = step()
    hist = []
    for _ in range(12):
        graph.replay()
        hist.append(float(static_loss.detach()))
    stats = {k: v.detach().cpu().clone() for k, v in m.state_dict().items() if 'running_' in k}
    return hist, stats


def _nccl_main(rank, world, store, q):
    _run_rank(rank, world, store, q, 'nccl', rank, _graph_rank)


def test_step_captured_as_cuda_graph_nccl(cuda):
    """NCCL, two GPUs: the synced YOLOv6-n step captured as one CUDA graph and replayed: the loss falls, and the running statistics are
    bitwise equal across ranks."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    (h0, s0), (h1, s1) = _spawn(_nccl_main, 2)
    print('graph loss', [round(v, 4) for v in h0])
    for hist in (h0, h1):
        assert all(np.isfinite(hist)) and hist[-1] < hist[0], hist
    assert all(torch.equal(s0[k], s1[k]) for k in s0)
