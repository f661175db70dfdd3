"""SyncBatchNorm on the H100 training kernels: BatchNorm statistics over every rank's pixels (cvb_train_bn_partial / _merge,
cvb_train_bn_silu_bwd_reduce / _apply; train._conv_bn_silu and train._bn_silu_backward with a process group).

Kernel level, one GPU, no collective: a bf16 tensor is split into unequal shards (1 to 8 of them, shards of 1 and 2 pixels among them), each
shard's record comes from cvb_train_bn_partial, the records are stacked as all_gather_into_tensor lays them out and merged.  Against float64
of the whole tensor with the bounds of test_train_gpu.py::test_bn_statistics_silu_forward_backward_vs_float64: each shard's summation bound
(its own addition chain), carried through the merge (the fp64 merge itself adds nothing at these scales).

Module level, two ranks (gloo) sharing one GPU: YOLOX-n converted with convert_sync_batchnorm, each rank one image of a 2-image batch, against
the oracle's fp32 step on the whole batch with test_yolox_train_gpu.py's rule (FACTOR x the bf16-autocast error + FLOOR).  With per-rank
statistics (the behaviour without this feature) the two ranks' running statistics already differ, and the test fails there.  Measured on
one H100 80GB HBM3 (SXM, 700 W power limit): the largest kernel / autocast error ratio was 1.997-2.046 over six runs, against 1.953-1.972
for the single-GPU step on the same batch (FACTOR = 3); runs differ because the backward reductions add with atomics in no fixed order.

Trainer level: the reference trainer's step (autocast + GradScaler + clip + SGD) on a converted, DDP-wrapped YOLOX over two ranks."""
import os
import queue
import sys
import time
import traceback

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fp64ref as R  # noqa: E402
from test_yolox_train_gpu import _compare, _leaves, _network_models, _network_state, _oracle_named  # noqa: E402

pytestmark = pytest.mark.gpu
SHARDS = {'1': [1000], '2': [1, 2], '3': [2, 5000, 1], '8': [1, 2, 129, 7, 4096, 3, 102401, 64]}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize('shift', [0, 10, 100])
@pytest.mark.parametrize('shards', list(SHARDS))
@pytest.mark.parametrize('C', [8, 24, 64, 192, 1024, 2048])
def test_sync_bn_merged_statistics_and_backward_vs_float64(cuda, C, shards, shift):
    from cvpytorch_b200 import _lib, train as T
    L, u = _lib.lib(), R.U24
    sizes = SHARDS[shards]
    npix = sum(sizes)
    g = torch.Generator(device='cuda').manual_seed(C * 1000 + npix + shift)
    kw = dict(generator=g, device='cuda')
    std = torch.rand(C, **kw) * 1.5 + 0.5
    y = ((torch.randn(npix, C, **kw) + shift) * std).to(torch.bfloat16)
    gamma, beta = torch.rand(C, **kw) + 0.5, torch.randn(C, **kw) * 0.5
    rm0, rv0 = torch.randn(C, **kw), torch.rand(C, **kw) + 0.5
    eps, mom = 1e-3, 0.1
    parts = list(torch.split(y, sizes))
    recs = torch.empty((len(sizes), 2 * C + 1), dtype=torch.float64, device='cuda')
    scratch = torch.empty(2, C, device='cuda')
    for i, ys in enumerate(parts):
        _lib.check(L.cvb_train_bn_partial(T._p(ys), ys.shape[0], C, T._p(scratch), T._p(recs[i]), T._stream()), 'partial')
    rm, rv = rm0.clone(), rv0.clone()
    stat, count = torch.empty(4, C, device='cuda'), torch.empty(1, dtype=torch.float64, device='cuda')
    _lib.check(L.cvb_train_bn_merge(T._p(recs), len(sizes), C, T._p(gamma), T._p(beta), eps, mom, T._p(rm), T._p(rv), T._p(stat), T._p(count),
                                    T._stream()), 'merge')
    da = torch.randn(npix, C, **kw).to(torch.bfloat16)
    gparts = list(torch.split(da, sizes))
    sums = {is_dz: [torch.empty(2, C, device='cuda') for _ in sizes] for is_dz in (0, 1)}
    dys = {is_dz: [torch.empty_like(p) for p in parts] for is_dz in (0, 1)}
    total = {}
    for is_dz in (0, 1):
        for ys, gs_, s in zip(parts, gparts, sums[is_dz]):
            _lib.check(L.cvb_train_bn_silu_bwd_reduce(T._p(gs_), is_dz, T._p(ys), ys.shape[0], C, T._p(stat), T._p(s), T._stream()), 'reduce')
        total[is_dz] = torch.stack(sums[is_dz]).sum(0)  # (the all-reduce: fp32 additions in rank order)
        for ys, gs_, d in zip(parts, gparts, dys[is_dz]):
            _lib.check(L.cvb_train_bn_silu_bwd_apply(T._p(gs_), is_dz, T._p(ys), ys.shape[0], C, T._p(stat), T._p(gamma), T._p(total[is_dz]), T._p(count),
                                                     T._p(d), T._stream()), 'apply')
    torch.cuda.synchronize()
    assert float(count) == npix
    r = {}

    # statistics: each shard sums d = y - (its first pixel) with its own chain bound gs; the merge recombines (mean, M2) exactly in fp64
    y64, n = y.double(), float(npix)
    mean, var = y64.mean(0), y64.var(0, unbiased=False)
    e_mean, e_m2 = torch.zeros_like(mean), torch.zeros_like(mean)
    for ys in parts:
        ys64, ns = ys.double(), ys.shape[0]
        gs = (R.red_chain(ns, C, _sms()) + 2) * u
        d = ys64 - ys64[0]
        d_abs, d_sq, d_mean = d.abs().sum(0), (d * d).sum(0), d.mean(0)
        e_ms = gs * d_abs / ns
        e_mean += e_ms * ns / n
        e_m2 += gs * d_sq + 2 * d_mean.abs() * gs * d_abs + 2 * ns * (ys64.mean(0) - mean).abs() * e_ms
    e_mean += u * mean.abs()
    e_var = e_m2 / n + 1e-12 * (var + mean * mean)
    rstd = 1 / torch.sqrt(var + eps)
    e_rstd = rstd * (0.5 * e_var / (var + eps) + 2 * u)
    g64, b64 = gamma.double(), beta.double()
    scale = g64 * rstd
    e_scale = g64 * e_rstd + u * scale
    e_shift = mean.abs() * e_scale + scale * e_mean + 2 * u * ((mean * scale).abs() + b64.abs())
    r['mean'] = R.check(stat[0], mean, e_mean, 'mean')
    r['rstd'] = R.check(stat[1], rstd, e_rstd, 'rstd')
    r['scale'] = R.check(stat[2], scale, e_scale, 'scale')
    r['shift'] = R.check(stat[3], b64 - mean * scale, e_shift, 'shift')
    m = float(np.float32(mom))
    var_unb = var * n / max(n - 1, 1)
    rm_ref, rv_ref = (1 - m) * rm0.double() + m * mean, (1 - m) * rv0.double() + m * var_unb
    r['running_mean'] = R.check(rm, rm_ref, m * e_mean + 4 * u * ((1 - m) * rm0.double().abs() + m * mean.abs()), 'running_mean')
    r['running_var'] = R.check(rv, rv_ref, m * (e_var * n / max(n - 1, 1) + u * var_unb) + 4 * u * rv_ref, 'running_var')

    # backward with the merged statistics: per-shard sums (= that shard's dbeta / dgamma), their sum over shards, dy with 1 / N from the device
    xhat = (y64 - stat[0].double()) * stat[1].double()
    z = y64 * stat[2].double() + stat[3].double()
    g64d = da.double()
    bounds = torch.tensor([0] + sizes).cumsum(0).tolist()
    for is_dz in (0, 1):
        if is_dz:
            dz, e_dz = g64d, torch.zeros_like(g64d)
        else:
            dz = g64d * R.silu_grad64(z)
            e_dz = g64d.abs() * R.silu_grad_err(z) + u * dz.abs()
        tag = ' (g = dz)' if is_dz else ''
        e_tot0, e_tot1 = 0, 0
        for i, (a, b) in enumerate(zip(bounds, bounds[1:])):
            gs = (R.red_chain(b - a, C, _sms()) + 2) * u
            dzs, dzxs = dz[a:b], dz[a:b] * xhat[a:b]
            e0 = gs * dzs.abs().sum(0) + e_dz[a:b].sum(0)
            e1 = (gs + 3 * u) * dzxs.abs().sum(0) + (e_dz[a:b] * xhat[a:b].abs()).sum(0)
            r[f'shard {i} dbeta' + tag] = R.check(sums[is_dz][i][0], dzs.sum(0), e0, 'dbeta' + tag)
            r[f'shard {i} dgamma' + tag] = R.check(sums[is_dz][i][1], dzxs.sum(0), e1, 'dgamma' + tag)
            e_tot0, e_tot1 = e_tot0 + e0, e_tot1 + e1
        k = len(sizes) * u  # the fp32 additions across shards
        r['sum dz' + tag] = R.check(total[is_dz][0], dz.sum(0), e_tot0 + k * dz.abs().sum(0), 'sum dz' + tag)
        r['sum dz*xhat' + tag] = R.check(total[is_dz][1], (dz * xhat).sum(0), e_tot1 + k * (dz * xhat).abs().sum(0), 'sum dz*xhat' + tag)
        S0, S1 = total[is_dz][0].double() / n, total[is_dz][1].double() / n
        gr = (g64 * stat[1].double()).abs()
        dy_ref = g64 * stat[1].double() * (dz - S0 - xhat * S1)
        bound = R.BF16_REL * dy_ref.abs() + (1 + R.BF16_REL) * gr * (e_dz + 8 * u * (dz.abs() + S0.abs() + (xhat * S1).abs()))
        r['dy' + tag] = R.check(torch.cat(dys[is_dz]), dy_ref, bound, 'dy' + tag)
        del dz, e_dz, dy_ref, bound
    print('worst error / bound', {k_: round(v, 3) for k_, v in r.items()})


# ------------------------------------------------------------------------------------------------ ranks on one GPU (gloo)
def _spawn(target, world, *args, timeout=900):
    """Runs target(rank, world, store, q, *args) in `world` spawned processes; -> the results they put on q, ordered by rank.
    Each rank puts exactly one message, ('ok', result) or ('error', traceback), before its process-group teardown, so a teardown failure
    cannot stand in for another rank's result; it shows as that rank's exit code, reported on its own.  The ranks rendezvous through a
    file store in a fresh directory (no port to race for).  The parent's cached GPU memory (the float64 kernel tests before this one hold
    several GB) is returned to the device first, since the ranks share it.  A timeout fails the test; no process outlives it."""
    import gc
    import tempfile
    import torch.multiprocessing as mp
    gc.collect()
    torch.cuda.empty_cache()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    with tempfile.TemporaryDirectory() as tmp:
        store = 'file://' + os.path.join(tmp, 'store')
        procs = [ctx.Process(target=target, args=(r, world, store, q) + args) for r in range(world)]
        for p in procs:
            p.start()
        res = {}
        deadline = time.monotonic() + timeout
        try:
            while len(res) < world:
                try:
                    rank, status, value = q.get(timeout=5)
                    res[rank] = (status, value)
                except queue.Empty:
                    gone = {r: p.exitcode for r, p in enumerate(procs) if r not in res and p.exitcode is not None}
                    assert not gone, f'ranks {sorted(gone)} exited without a result, exit codes {gone}'
                    assert time.monotonic() < deadline, f'no result from ranks {sorted(set(range(world)) - set(res))} after {timeout} s'
            for p in procs:
                p.join(120)
        finally:
            for p in procs:
                if p.is_alive():
                    p.terminate()
                    p.join(30)
    errs = {r: v for r, (s, v) in res.items() if s != 'ok'}
    assert not errs, f'rank {min(errs)} failed:\n{errs[min(errs)]}'
    codes = {r: p.exitcode for r, p in enumerate(procs)}
    assert all(c == 0 for c in codes.values()), f'every rank delivered its result, but the exit codes are {codes} (process-group teardown)'
    return [_map(res[r][1], torch.from_numpy, np.ndarray) for r in range(world)]


def _map(obj, fn, kind):
    """fn applied to every `kind` leaf of nested dicts / lists / tuples.  Results cross the queue as numpy arrays: a CPU tensor would travel
    as a shared-memory handle that dies with the rank's process."""
    if isinstance(obj, kind):
        return fn(obj)
    if isinstance(obj, dict):
        return {k: _map(v, fn, kind) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_map(v, fn, kind) for v in obj)
    return obj


def _run_rank(rank, world, store, q, backend, device, body, *args):
    """init, body, ONE message on q, then teardown (whose failure only sets the exit code)."""
    import torch.distributed as dist
    try:
        torch.cuda.set_device(device)
        dist.init_process_group(backend, init_method=store, rank=rank, world_size=world)
        out = body(rank, world, *args)
        torch.cuda.synchronize()
        msg = (rank, 'ok', _map(out, lambda t: t.detach().cpu().numpy(), torch.Tensor))
    except Exception:  # noqa: BLE001  (the traceback fails the test in the parent)
        msg = (rank, 'error', traceback.format_exc())
    q.put(msg)
    if msg[1] == 'ok':  # (after a failure the other ranks may be inside a collective: no barrier)
        dist.barrier()
        dist.destroy_process_group()


def _rank_main(rank, world, store, q, body, *args):
    """gloo, every rank on cuda:0."""
    _run_rank(rank, world, store, q, 'gloo', 0, body, *args)


def _synced_network(sub, seed):
    sd = _network_state(sub, seed)
    mods = dict(zip(('backbone.', 'neck.', 'head.'), _network_models(sub)))
    for pre, m in mods.items():
        m.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)})
        mods[pre] = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m).cuda().train()
    return sd, mods


def _network_inputs(B=2):
    """The batch of test_yolox_train_gpu.py::test_backbone_neck_head_training_step_vs_oracle[cspdark_n] (same seed and state), whose margin
    under FACTOR / FLOOR is known; a 4-image batch of another seed puts the stem's BatchNorm weight gradient, a nearly cancelling sum at
    the end of the whole backward, at 0.92 max-normalised error against autocast's 0.29 in some runs."""
    g = torch.Generator().manual_seed(13)
    x = torch.randn(B, 3, 128, 160, generator=g)
    Gs = [torch.randn(B, 85, 128 // s + 2, 160 // s + 2, generator=g) for s in (8, 16, 32)]
    return x, Gs


def _network_rank(rank, world, seed):
    """One training step of the converted YOLOX-n on this rank's slice of the batch -> CPU {outputs, parameter gradients, running stats}."""
    sd, mods = _synced_network('cspdark_n', seed)
    assert sum(isinstance(m, torch.nn.SyncBatchNorm) for mod in mods.values() for m in mod.modules()) == 74
    x, Gs = _network_inputs()
    per = x.shape[0] // world
    part = slice(rank * per, (rank + 1) * per)
    bb, nk, hd = mods.values()
    outs = hd.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(x[part].cuda())))
    sum((o * G[part].cuda()).sum() for o, G in zip(outs, Gs)).backward()
    res = {f'y{i}': o.detach().cpu() for i, o in enumerate(outs)}
    for pre, m in mods.items():
        res.update({'grad_' + pre + k: p.grad.cpu() for k, p in m.named_parameters()})
        res.update({'after_' + pre + k: v.cpu() for k, v in m.state_dict().items() if 'running_' in k})
    return res


def test_sync_bn_two_ranks_match_the_full_batch_step(cuda):
    """YOLOX-n (backbone + neck + head, 74 SyncBatchNorm layers), two gloo ranks on one GPU, one of 2 images each: every rank's head outputs
    match its half of the oracle's fp32 step on both images, the sum of the ranks' parameter gradients matches the oracle's gradients, and
    the running statistics are bitwise equal across ranks and match the oracle's."""
    from oracle import yolox_train_oracle as XO
    seed = 7 + len('cspdark_n')
    r0, r1 = _spawn(_rank_main, 2, _network_rank, seed)
    sd = _network_state('cspdark_n', seed)
    x, Gs = _network_inputs()

    def oracle_step(autocast):
        sdt = _leaves(sd, 'cuda')
        with torch.autocast('cuda', dtype=torch.bfloat16, enabled=autocast):
            outs = XO.network(x.cuda(), sdt, 'cspdark_n')
        sum((o.float() * G.cuda()).sum() for o, G in zip(outs, Gs)).backward()
        return _oracle_named([o.float().detach().cpu() for o in outs], [], {k: v.grad.cpu() for k, v in sdt.items() if v.requires_grad},
                             {k: v.cpu() for k, v in sdt.items() if 'running_' in k})
    ref, auto = oracle_step(False), oracle_step(True)
    stats = [k for k in r0 if k.startswith('after_')]
    assert stats and all(torch.equal(r0[k], r1[k]) for k in stats)
    got = {k: r0[k] + r1[k] for k in r0 if k.startswith('grad_')}
    got.update({k: r0[k] for k in stats})
    ref_c, auto_c = {k: ref[k] for k in got}, {k: auto[k] for k in got}
    for rank, res in enumerate((r0, r1)):
        per = x.shape[0] // 2
        part = slice(rank * per, (rank + 1) * per)
        for i in range(3):
            got[f'rank{rank} y{i}'] = res[f'y{i}']
            ref_c[f'rank{rank} y{i}'], auto_c[f'rank{rank} y{i}'] = ref[f'y{i}'][part], auto[f'y{i}'][part]
    _compare(got, ref_c, auto_c)


def _csp_step(m, x, G):
    y = m(x.clone())
    (y.float() * G).sum().backward()
    out = {'y': y.detach().clone()}
    out.update({'grad_' + k: p.grad.clone() for k, p in m.named_parameters()})
    out.update({k: v.clone() for k, v in m.state_dict().items()})
    m.zero_grad(set_to_none=True)
    return out


def _world_of_one_rank(rank, world):
    """A CSPLayer on 2 x 8 x 8 pixels (every reduction runs in one CTA, so a step is bitwise reproducible): the unconverted module, and the
    converted one in a world of one, step for step."""
    import copy
    from cvpytorch_b200 import train as T
    torch.manual_seed(3)
    plain = T.CSPLayer(64, 64, n=1).cuda().train()
    synced = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(plain))
    x = torch.randn(2, 64, 8, 8, device='cuda')
    G = torch.randn(2, 64, 8, 8, device='cuda')
    steps = [(_csp_step(plain, x, G), _csp_step(synced, x, G)) for _ in range(2)]
    return [{k: bool(torch.equal(a[k], b[k])) for k in a} for a, b in steps]


def test_sync_bn_world_of_one_is_the_local_path_bitwise(cuda):
    """nn.SyncBatchNorm layers without a process group and in a world of one run the local statistics: outputs, gradients and running
    statistics bitwise equal to the unconverted module's over two steps."""
    import copy
    from cvpytorch_b200 import train as T
    torch.manual_seed(3)
    plain = T.CSPLayer(64, 64, n=1).cuda().train()
    synced = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(plain))
    x = torch.randn(2, 64, 8, 8, device='cuda')
    G = torch.randn(2, 64, 8, 8, device='cuda')
    for _ in range(2):
        a, b = _csp_step(plain, x, G), _csp_step(synced, x, G)
        assert all(torch.equal(a[k], b[k]) for k in a), [k for k in a if not torch.equal(a[k], b[k])]
    for step in _spawn(_rank_main, 1, _world_of_one_rank)[0]:
        assert all(step.values()), [k for k, v in step.items() if not v]


# ------------------------------------------------------------------------------------------------ the reference trainer's step under DDP
def _trainer_rank(rank, world, iters):
    """YOLOX-s (synthetic state), convert_sync_batchnorm, DDP; the reference trainer's step on this rank's image of a fixed 2-image batch."""
    from torch.nn.parallel import DistributedDataParallel as DDP
    from cvpytorch_b200 import synth, yolox_models as XM
    from test_yolox_loss_gpu import _batch, _model
    m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_model())
    assert sum(isinstance(b, torch.nn.SyncBatchNorm) for b in m.modules()) == 74
    ddp = DDP(m, device_ids=[0], broadcast_buffers=False)  # (the running statistics must agree without rank 0's copy)
    imgs, targets = _batch()
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
        _, got = m(imgs, None, 'val')
    fresh = XM.YOLOX(dictionary=[{f'c{i}': 1.0} for i in range(80)], model_cfg=dict(synth.YOLOX_CFG))
    fresh.load_state_dict(m.state_dict(), strict=True)
    fresh.cuda().eval()
    with torch.no_grad():
        _, want = fresh(imgs, None, 'val')
    handoff = all(torch.equal(a[k], b[k]) for a, b in zip(got, want) for k in ('boxes', 'labels', 'scores'))
    return hist, sd, handoff


def test_sync_bn_trainer_steps_under_ddp(cuda):
    """Two gloo ranks on one GPU, one image each: the loss falls on both ranks, parameters and running statistics stay bitwise identical across
    ranks over the whole run (DDP's buffer broadcast is off, so every step's running statistics come from each rank's own merge), and
    eval() + 'val' equals a fresh eval YOLOX loaded with the trained state_dict."""
    (h0, sd0, ok0), (h1, sd1, ok1) = _spawn(_rank_main, 2, _trainer_rank, 10)
    print('loss rank 0', [round(v, 4) for v in h0], 'rank 1', [round(v, 4) for v in h1])
    for hist in (h0, h1):
        assert all(np.isfinite(hist)) and np.mean(hist[-3:]) < hist[0], hist
    assert ok0 and ok1
    assert list(sd0) == list(sd1)
    diff = [k for k in sd0 if not torch.equal(sd0[k], sd1[k])]
    assert not diff, diff


def _graph_rank(rank, world):
    """The converted YOLOX-n step with NCCL, one GPU per rank, captured as one CUDA graph and replayed."""
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    _, mods = _synced_network('cspdark_n', 9)
    bb, nk, hd = mods.values()
    params = [p for m in mods.values() for p in m.parameters()]
    opt = torch.optim.SGD(params, lr=0.05, momentum=0.9)
    g = torch.Generator().manual_seed(6 + rank)
    x = torch.randn(2, 3, 128, 128, generator=g).cuda()
    targets = [(torch.randn(2, 85, 128 // s + 2, 128 // s + 2, generator=g) * 0.1).cuda() for s in (8, 16, 32)]

    def step():
        outs = hd.forward_nhwc(nk.forward_nhwc(bb.forward_nhwc(x)))
        loss = sum((o - t).pow(2).mean() for o, t in zip(outs, targets))
        loss.backward()
        for p in params:
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
    stats = {k: v.detach().cpu().clone() for m in mods.values() for k, v in m.state_dict().items() if 'running_' in k}
    return hist, stats


def _nccl_main(rank, world, store, q):
    """NCCL, rank r on cuda:r."""
    _run_rank(rank, world, store, q, 'nccl', rank, _graph_rank)


def test_sync_bn_step_captured_as_cuda_graph_nccl(cuda):
    """NCCL, two GPUs: the synced step (74 all-gathers forward, 74 all-reduces backward, the gradient all-reduce, SGD) captured as one CUDA
    graph and replayed: the loss falls, the running statistics are bitwise equal across ranks."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    (h0, s0), (h1, s1) = _spawn(_nccl_main, 2)
    print('graph loss', [round(v, 4) for v in h0])
    for hist in (h0, h1):
        assert all(np.isfinite(hist)) and hist[-1] < 0.8 * hist[0], hist
    assert all(torch.equal(s0[k], s1[k]) for k in s0)
