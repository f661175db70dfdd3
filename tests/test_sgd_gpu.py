"""The one-launch SGD on the H100 (csrc/sgd.cu, cvpytorch_b200.optim.SGD) against torch.optim.SGD + torch.amp.GradScaler on the same GPU,
bit for bit after every step: params, momentum buffers and the scaler's scale.  Both arms see cloned, identical gradients.  Covers the
reference's YOLOX-s and YOLOv5-s groups with a warm-up and a cosine lr, every hyper-parameter branch, awkward sizes and misaligned views,
overflow skips (first step, mid-run, after unscale_ + clipping), params without a gradient, replaced tensors, add_param_group, state_dict
round trips with torch.optim.SGD, launch counts, the absence of host syncs, CUDA-graph replay and the trainer's step on a drop-in YOLOX."""
import copy
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

DICT80 = [{f'c{i}': 1.0} for i in range(80)]


def _model(name):
    from cvpytorch_b200 import models as M, synth, yolox_models as XM
    return XM.YOLOX(dictionary=DICT80, model_cfg=dict(synth.YOLOX_CFG)) if name == 'yolox_s' else M.YOLOv5(DICT80, dict(synth.YOLOV5S_CFG))


class Twins:
    """The drop-in and torch.optim.SGD over two copies of the same params, each with its own GradScaler (or none)."""

    def __init__(self, params, make_groups, scaler_kw=None):
        from cvpytorch_b200.optim import SGD
        self.mine = [torch.nn.Parameter(p.detach().clone().cuda()) for p in params]
        self.ref = [torch.nn.Parameter(p.detach().clone().cuda()) for p in params]
        self.opt = SGD(make_groups(self.mine))
        self.ref_opt = torch.optim.SGD(make_groups(self.ref))
        self.scalers = None
        if scaler_kw is not None:
            self.scalers = (torch.amp.GradScaler('cuda', **scaler_kw), torch.amp.GradScaler('cuda', **scaler_kw))

    def step(self, grads, clip=None):
        """grads: one tensor or None per param (cloned into both arms)."""
        for arm, opt, scaler in ((self.mine, self.opt, self.scalers and self.scalers[0]), (self.ref, self.ref_opt, self.scalers and self.scalers[1])):
            for p, g in zip(arm, grads):
                p.grad = None if g is None else g.clone()
            if scaler is None:
                opt.step()
                continue
            scaler.scale(torch.ones((), device='cuda'))  # as scaler.scale(loss) in the trainer: the scale exists from here on
            if clip is not None:
                scaler.unscale_(opt)
                torch.nn.utils.clip_grad_norm_(arm, clip)
            scaler.step(opt)
            scaler.update()
        self.check()

    def check(self):
        for i, (a, b) in enumerate(zip(self.mine, self.ref)):
            assert torch.equal(a, b), f'param {i}: max diff {(a - b).abs().max().item()}'
            rb = self.ref_opt.state.get(b, {}).get('momentum_buffer')
            if rb is not None:
                assert torch.equal(self.opt.state[a]['momentum_buffer'], rb), f'momentum buffer {i}'
        if self.scalers:
            assert self.scalers[0].get_scale() == self.scalers[1].get_scale()

    def check_state_dicts(self):
        a, b = self.opt.state_dict(), self.ref_opt.state_dict()
        assert a['param_groups'] == b['param_groups']
        assert sorted(a['state']) == sorted(b['state'])
        for k, v in b['state'].items():
            assert set(a['state'][k]) == set(v)
            assert all(torch.equal(a['state'][k][n], t) for n, t in v.items())


def _grads(params, g, scale=1.0, none=(), inf=()):
    out = []
    for i, p in enumerate(params):
        if i in none:
            out.append(None)
            continue
        t = (torch.randn(p.shape, generator=g) * scale).cuda()
        if i in inf and t.numel():
            t.view(-1)[t.numel() // 2] = float('inf')
        out.append(t)
    return out


@pytest.mark.parametrize('name', ['yolox_s', 'yolov5_s'])
def test_reference_groups_with_warmup_and_cosine_lr(cuda, name):
    """The groups build_optimizer makes for the model, GradScaler at a non-power-of-two scale, lr rewritten every warm-up step, then a
    CosineAnnealingLR; an overflow on the first step (no buffer is created) and one mid-run."""
    from oracle import optim_oracle as O
    cfg = O.CONFIGS[name]
    model = _model(name)
    params = [g['params'][0] for g in O.param_groups(model, cfg)]
    pos = {id(p): i for i, p in enumerate(params)}

    def groups(ps):
        return [dict(g, params=[ps[pos[id(g['params'][0])]]]) for g in O.param_groups(model, cfg)]
    tw = Twins(params, groups, dict(init_scale=3000.0, growth_interval=3))
    g = torch.Generator().manual_seed(11)
    for it in range(1, 7):
        for opt in (tw.opt, tw.ref_opt):
            for pg in opt.param_groups:
                pg['lr'] = O.warmup_lr(it, cfg)
        tw.step(_grads(params, g, 3000.0, inf={0, 7} if it in (1, 4) else ()))
        if it == 1:
            tw.check_state_dicts()
            assert not tw.opt.state_dict()['state']
    scheds = [torch.optim.lr_scheduler.CosineAnnealingLR(o, T_max=10, eta_min=1e-4) for o in (tw.opt, tw.ref_opt)]
    for _ in range(6):
        tw.step(_grads(params, g, tw.scalers[0].get_scale()))
        for s in scheds:
            s.step()
    tw.check_state_dicts()


@pytest.mark.parametrize('momentum,nesterov,wd', [(0.0, False, 0.0), (0.0, False, 5e-4), (0.9, False, 0.0), (0.9, False, 1e-4),
                                                  (0.937, True, 0.0), (0.949, True, 5e-4)])
def test_hyper_parameter_branches_in_multi_tensor_groups(cuda, momentum, nesterov, wd):
    shapes = [(64, 32, 3, 3), (64,), (7,), (4097,), (300, 50)]
    g = torch.Generator().manual_seed(3)
    params = [torch.randn(s, generator=g) for s in shapes]

    def groups(ps):
        return [{'params': ps[:3], 'lr': 0.02, 'momentum': momentum, 'nesterov': nesterov, 'weight_decay': wd},
                {'params': ps[3:], 'lr': 0.005, 'momentum': 0.9, 'weight_decay': 1e-3}]
    tw = Twins(params, groups)
    for _ in range(5):
        tw.step(_grads(params, g))
    tw.check_state_dicts()


def test_awkward_sizes_and_misaligned_views(cuda):
    """0, 1, 3 and 4k + 1 elements, several 4096-element chunks, and params / gradients at every 4-byte offset."""
    from cvpytorch_b200.optim import SGD
    sizes = [0, 1, 3, 5, 4097, 4096 * 3 + 1, 100003]
    g = torch.Generator().manual_seed(8)
    params = [torch.randn(n, generator=g) for n in sizes]

    def groups(ps):
        return [{'params': ps, 'lr': 0.03, 'momentum': 0.9, 'nesterov': True, 'weight_decay': 1e-4}]
    tw = Twins(params, groups, dict(init_scale=1000.0))
    for _ in range(3):
        tw.step(_grads(params, g, 1000.0))
    tw.check_state_dicts()
    for off in range(4):
        for n in (5, 4097, 9000):
            base, gbase = torch.zeros(n + 8, device='cuda'), torch.zeros(n + 8, device='cuda')
            p = torch.nn.Parameter(base[off:off + n])
            p.data.copy_(torch.randn(n, generator=g).cuda())
            ref = torch.nn.Parameter(p.detach().clone())
            opt, ref_opt = SGD([p], lr=0.1, momentum=0.9, weight_decay=5e-4), torch.optim.SGD([ref], lr=0.1, momentum=0.9, weight_decay=5e-4)
            for _ in range(3):
                gv = gbase[(3 - off):(3 - off) + n]
                gv.copy_(torch.randn(n, generator=g).cuda())
                p.grad, ref.grad = gv, gv.clone()
                opt.step()
                ref_opt.step()
                assert torch.equal(p, ref) and torch.equal(opt.state[p]['momentum_buffer'], ref_opt.state[ref]['momentum_buffer'])
            assert torch.equal(base[:off], torch.zeros(off, device='cuda')) and torch.equal(base[off + n:], torch.zeros(8 - off, device='cuda'))


def test_overflow_skips_and_clipping(cuda):
    """inf on the first step (no buffer; the next applied step copies), twice in a row mid-run, and after unscale_ + clip_grad_norm_."""
    g = torch.Generator().manual_seed(9)
    params = [torch.randn(s, generator=g) for s in [(32, 16, 3, 3), (32,), (5000,), (3,)]]

    def groups(ps):
        return [{'params': ps[:2], 'lr': 0.01, 'momentum': 0.937, 'nesterov': True, 'weight_decay': 5e-4},
                {'params': ps[2:], 'lr': 0.02, 'momentum': 0.9}]
    tw = Twins(params, groups, dict(init_scale=2.0 ** 16 * 0.75, growth_interval=2))
    tw.step(_grads(params, g, 1e4, inf={1}))
    tw.check_state_dicts()
    tw.step(_grads(params, g, 1e4, none={2}))          # params 0, 1, 3 get their first buffers; 2 has none yet
    tw.check_state_dicts()
    tw.step(_grads(params, g, 1e4, inf={3}))
    tw.step(_grads(params, g, 1e4, inf={0}))
    tw.step(_grads(params, g, 1e4))                    # param 2's first applied step
    tw.check_state_dicts()
    for i in range(4):
        tw.step(_grads(params, g, 1e4, inf={2} if i == 1 else ()), clip=1.0)
    tw.check_state_dicts()


def test_replaced_tensors_add_param_group_and_no_grad(cuda):
    g = torch.Generator().manual_seed(12)
    params = [torch.randn(s, generator=g) for s in [(40, 3), (40,), (9,)]]

    def groups(ps):
        return [{'params': ps, 'lr': 0.05, 'momentum': 0.9, 'weight_decay': 1e-4}]
    tw = Twins(params, groups, dict(init_scale=512.0))
    tw.step(_grads(params, g, 512.0))
    tw.step(_grads(params, g, 512.0, none={0}))
    for arm in (tw.mine, tw.ref):                      # a new storage for one param (as .to() or load_state_dict(assign=True) give)
        arm[1].data = arm[1].data.clone()
    tw.step(_grads(params, g, 512.0))
    extra = [torch.randn(s, generator=g) for s in [(17,), (6, 6)]]
    for arm, opt in ((tw.mine, tw.opt), (tw.ref, tw.ref_opt)):
        new = [torch.nn.Parameter(e.clone().cuda()) for e in extra]
        arm.extend(new)
        opt.add_param_group({'params': new, 'lr': 0.2, 'momentum': 0.95, 'nesterov': True})
    allp = params + extra
    for _ in range(3):
        tw.step(_grads(allp, g, 512.0))
    tw.check_state_dicts()


def test_state_dict_round_trips_with_torch_sgd(cuda):
    from cvpytorch_b200.optim import SGD
    g = torch.Generator().manual_seed(13)
    params = [torch.randn(s, generator=g) for s in [(30, 4), (30,), (4100,)]]

    def groups(ps):
        return [{'params': ps[:2], 'lr': 0.01, 'momentum': 0.9, 'nesterov': True}, {'params': ps[2:], 'lr': 0.03, 'momentum': 0.9}]
    tw = Twins(params, groups, dict(init_scale=100.0))
    tw.step(_grads(params, g, 100.0, inf={0}))
    tw.step(_grads(params, g, 100.0, none={2}))
    tw.check_state_dicts()
    # swap the arms: the drop-in continues from torch's state dict and torch from the drop-in's
    mine_sd, ref_sd = copy.deepcopy(tw.opt.state_dict()), copy.deepcopy(tw.ref_opt.state_dict())
    assert 2 not in mine_sd['state']
    tw.opt, tw.ref_opt = SGD(groups(tw.mine)), torch.optim.SGD(groups(tw.ref))
    tw.opt.load_state_dict(ref_sd)
    tw.ref_opt.load_state_dict(mine_sd)
    for _ in range(3):
        tw.step(_grads(params, g, 100.0))
    tw.check_state_dicts()


def test_one_launch_per_step_and_no_host_sync(cuda):
    from cvpytorch_b200 import _lib
    from cvpytorch_b200.optim import SGD
    g = torch.Generator().manual_seed(14)
    ps = [torch.nn.Parameter(torch.randn(s, generator=g).cuda()) for s in [(64, 64, 3, 3), (64,), (3,), (0,)]]
    opt = SGD([{'params': ps[:2], 'weight_decay': 5e-4}, {'params': ps[2:]}], lr=0.01, momentum=0.9, nesterov=True)
    scaler = torch.amp.GradScaler('cuda', init_scale=1024.0)
    for i in range(4):
        for p in ps:
            p.grad = torch.randn(p.shape, generator=g).cuda()
        scaler.scale(torch.ones((), device='cuda'))
        n0 = _lib.launch_count()
        if i == 0:
            scaler.step(opt)
            scaler.update()
        else:
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode('error')
            try:
                scaler.step(opt)
                scaler.update()
            finally:
                torch.cuda.set_sync_debug_mode('default')
        assert _lib.launch_count() == n0 + 1
    opt.zero_grad(set_to_none=True)
    n0 = _lib.launch_count()
    opt.step()
    assert _lib.launch_count() == n0


def test_cuda_graph_replay_matches_eager_torch(cuda):
    """A scaler-free step() captured after one eager step replays bitwise like eager torch.optim.SGD."""
    from cvpytorch_b200.optim import SGD
    g = torch.Generator().manual_seed(15)
    shapes = [(128, 64, 3, 3), (128,), (5,), (10001,)]
    init = [torch.randn(s, generator=g) for s in shapes]
    mine = [torch.nn.Parameter(t.clone().cuda()) for t in init]
    ref = [torch.nn.Parameter(t.clone().cuda()) for t in init]
    kw = dict(lr=0.01, momentum=0.937, nesterov=True, weight_decay=5e-4)
    opt, ref_opt = SGD(mine, **kw), torch.optim.SGD(ref, **kw)
    static = [torch.randn(s, generator=g).cuda() for s in shapes]
    for p, r, s in zip(mine, ref, static):
        p.grad, r.grad = s, s.clone()
    opt.step()
    ref_opt.step()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            opt.step()
    torch.cuda.current_stream().wait_stream(side)
    for _ in range(4):
        for p, r, s in zip(mine, ref, static):
            s.copy_(torch.randn(s.shape, generator=g).cuda())
            r.grad = s.clone()
        graph.replay()
        ref_opt.step()
        torch.cuda.synchronize()
        for p, r in zip(mine, ref):
            assert torch.equal(p, r) and torch.equal(opt.state[p]['momentum_buffer'], ref_opt.state[r]['momentum_buffer'])


def test_device_refusals(cuda):
    from cvpytorch_b200 import _lib
    from cvpytorch_b200.optim import SGD
    a, b = torch.nn.Parameter(torch.randn(4, device='cuda')), torch.nn.Parameter(torch.randn(4))
    a.grad, b.grad = torch.randn(4, device='cuda'), torch.randn(4)
    with pytest.raises(_lib.CvbError, match='CPU'):
        SGD([a, b], lr=0.1).step()
    c = torch.nn.Parameter(torch.randn(4, device='cuda'))
    c.grad = torch.randn(4, device='cuda')
    opt = SGD([c], lr=0.1)
    opt.found_inf = torch.zeros(())
    with pytest.raises(_lib.CvbError, match='CPU'):
        opt.step()


def test_trainer_step_on_drop_in_yolox(cuda):
    """run_step of the reference trainer (autocast, scaler.scale(loss).backward(), scaler.step, scaler.update, zero_grad(set_to_none=True),
    ema.update) on a drop-in YOLOX with the reference's groups; torch.optim.SGD + its own GradScaler steps a shadow copy of the params on
    clones of the same gradients."""
    from cvpytorch_b200.ema import ModelEMA
    from cvpytorch_b200.optim import SGD
    from oracle import optim_oracle as O
    cfg = O.CONFIGS['yolox_s']
    model = _model('yolox_s').cuda().train()
    groups = O.param_groups(model, cfg)
    shadow = {id(gr['params'][0]): torch.nn.Parameter(gr['params'][0].detach().clone()) for gr in groups}
    opt = SGD(groups)
    ref_opt = torch.optim.SGD([dict(gr, params=[shadow[id(gr['params'][0])]]) for gr in O.param_groups(model, cfg)])
    scaler, ref_scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 12), torch.amp.GradScaler('cuda', init_scale=2.0 ** 12)
    ema = ModelEMA(model)
    g = torch.Generator().manual_seed(77)
    imgs = torch.randn(2, 3, 128, 128, generator=g).cuda()
    targets = [{'labels': torch.randint(0, 80, (3 + b,), generator=g).cuda(),
                'boxes': torch.cat([20 + torch.rand(3 + b, 2, generator=g) * 88, 16 + torch.rand(3 + b, 2, generator=g) * 40], 1).cuda()}
               for b in range(2)]
    for it in range(1, 5):
        for o in (opt, ref_opt):
            for pg in o.param_groups:
                pg['lr'] = O.warmup_lr(it, cfg)
        with torch.autocast('cuda', enabled=True):
            losses = model(imgs, targets, 'train')
        scaler.scale(losses['loss']).backward()
        ref_scaler.scale(losses['loss'].detach())  # the shadow arm's scaler sees the same loss
        for gr in groups:
            p = gr['params'][0]
            shadow[id(p)].grad = None if p.grad is None else p.grad.clone()
        ref_scaler.step(ref_opt)
        ref_scaler.update()
        scaler.step(opt)
        scaler.update()
        opt.zero_grad(set_to_none=True)
        ema.update(model)
        assert scaler.get_scale() == ref_scaler.get_scale()
        for gr in groups:
            p = gr['params'][0]
            assert torch.equal(p, shadow[id(p)])
