"""Every plan family of the fused conv kernel (csrc/conv_tc.cu) and every A/B knob path against float64, element by element.

A case table (CASES) spans the planner's plan space: block_n, K chunk, resident / streamed weights, CTAs per SM, classic / halo
loaders, row-window stems, dilation, both schedules, every epilogue, ragged edges, channel-slice views and grid shapes.  Each case runs
once into a NaN-filled output and is checked against fp64ref.split_conv_reference with
  (a) the element-wise bound |out - ref| <= bound (derived there from the kernel's arithmetic), and
  (b) max|out - ref| / max|ref| < 2e-5, the single-layer budget (tighter than (a) on deep-K layers);
channels of the output buffer outside the view must stay NaN.

`CVB_PLAN_DEBUG=1` makes the library print one `[cvb plan]` line per plan, and it and most knobs are read once per process, so child
processes of this file (`python tests/test_conv_plans_gpu.py --plans | --run OUT`) create the plans or run the cases under a knob:
  - test_plan_coverage parses the default plans and requires every plan dimension of the table (COVERAGE) to occur;
  - test_knob_* compare a knob's outputs with the default ones (bitwise where the K order of every element is unchanged, else the
    float64 bound) and require the plan lines to show that the knob took effect.
The YOLOv5 decode paths (fused CVB_OUT_YOLO epilogue, the stand-alone yolo_decode_kernel) are checked against the decode formula in
float64, and their NMS histogram / per-row best score against what the NMS recomputes from their own z.  test_*_teeth show that the
checks reject subtly wrong outputs.
"""
import math
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import fp64ref  # noqa: E402
from test_post_gpu import _ws_regions  # noqa: E402

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------------------- cases
class Case:
    """One conv layer with seeded inputs (CPU generator: identical in every process)."""

    def __init__(self, name, cin=64, cout=64, k=1, s=1, p=None, dil=1, B=2, H=16, W=16, act='silu', residual=False, resid_first=0,
                 resid_scale=1.0, up=False, f32=False, block_n=0, no_resident=0, sm_limit=0, halo=0, schedule=0, in_c0=0, in_pitch=None,
                 out_c0=0, out_pitch=None, stem=None, seed=0):
        self.name, self.cin, self.cout, self.s, self.dil, self.B, self.H, self.W = name, cin, cout, s, dil, B, H, W
        self.act, self.residual, self.resid_first, self.resid_scale, self.up, self.f32 = act, residual, resid_first, resid_scale, up, f32
        self.block_n, self.no_resident, self.sm_limit, self.halo, self.schedule = block_n, no_resident, sm_limit, halo, schedule
        self.in_c0, self.in_pitch, self.out_c0, self.stem, self.seed = in_c0, in_pitch or cin, out_c0, stem, seed
        self.out_pitch = out_pitch or (cout + 7) // 8 * 8
        if stem:  # row-window stems: the YOLOv5 6x6/s2/p2 (3 filter rows, pad_left 1), the ResNet 7x7/s2/p3 (4 filter rows, pad_left 2)
            self.k, self.p, self.win = (3, 1, 4) if stem == 'yolov5' else (4, 2, 4)
            self.cin = 16
            self.Ho, self.Wo = H // 2, W // 2
        else:
            self.k, self.win = k, 0
            self.p = k // 2 * dil if p is None else p
            self.Ho = (H + 2 * self.p - dil * (k - 1) - 1) // s + 1
            self.Wo = (W + 2 * self.p - dil * (k - 1) - 1) // s + 1
        self._t = None

    def tensors(self):
        if self._t is not None:
            return self._t
        from cvpytorch_b200 import ops
        g = torch.Generator().manual_seed(self.seed)
        B, H, W, cout = self.B, self.H, self.W, self.cout
        t = {}
        if self.stem:
            from cvpytorch_b200.fcos_models import resnet_stem_weights_to_s2d
            kk = 6 if self.stem == 'yolov5' else 7
            x = torch.randn(B, 3, H, W, generator=g)
            w = torch.randn(cout, 3, kk, kk, generator=g) / (3 * kk * kk) ** 0.5
            b = torch.randn(cout, generator=g) * 0.5
            t['tin'] = ops.SplitTensor(B, H // 2, W // 2 + 3, 16)
            ops.stem_s2d(x.cuda().contiguous(), t['tin'].view(), pad_left=1 if self.stem == 'yolov5' else 2)
            w3 = ops.stem_weights_to_s2d(w.double()) if self.stem == 'yolov5' else resnet_stem_weights_to_s2d(w.double())
            t['wp'], t['bp'] = ops.pack_conv_weights(ops.window_weights(w3, 4), b.double())
            t['orig'] = (x, w, b, 2, 2 if self.stem == 'yolov5' else 3)
        else:
            x = torch.randn(B, self.in_pitch, H, W, generator=g)
            w = torch.randn(cout, self.cin, self.k, self.k, generator=g) / (self.cin * self.k * self.k) ** 0.5
            b = torch.randn(cout, generator=g) * 0.5
            t['tin'] = ops.SplitTensor(B, H, W, self.in_pitch)
            ops.nchw_to_split(x.cuda(), t['tin'].view())
            t['wp'], t['bp'] = ops.pack_conv_weights(w.double(), b.double())
        t['res'] = t['up'] = None
        if self.residual:
            t['res'] = ops.SplitTensor(B, self.Ho, self.Wo, cout)
            ops.nchw_to_split(torch.randn(B, cout, self.Ho, self.Wo, generator=g).cuda(), t['res'].view())
        if self.up:
            t['up'] = ops.F32Tensor(B, (self.Ho + 1) // 2, (self.Wo + 1) // 2, cout)
            t['up'].data.copy_(torch.randn(B, (self.Ho + 1) // 2, (self.Wo + 1) // 2, cout, generator=g))
        t['out'] = (ops.F32Tensor if self.f32 else ops.SplitTensor)(B, self.Ho, self.Wo, self.out_pitch)
        self._t = t
        return t

    def plan(self):
        from cvpytorch_b200 import ops
        t = self.tensors()
        inp = t['tin'].view() if self.stem else t['tin'].view(self.in_c0, self.cin)
        return ops.ConvPlan(inp, t['out'].view(self.out_c0, self.cout), t['wp'], t['bp'], self.k, self.s, self.p, self.dil, self.act,
                            residual=t['res'].view() if t['res'] else None, up_partial=t['up'].view() if t['up'] else None,
                            block_n=self.block_n, sm_limit=self.sm_limit, w_window=self.win, no_resident=self.no_resident,
                            residual_before_act=self.resid_first, halo=self.halo, residual_scale=self.resid_scale, schedule=self.schedule)

    def run(self):
        """-> the whole output buffer after one run of the plan (filled with NaN before)."""
        t = self.tensors()
        plan = self.plan()
        t['out'].data.fill_(float('nan'))
        plan.run()
        torch.cuda.synchronize()
        return t['out'].data.clone()

    def view_of(self, buf):
        return buf[..., self.out_c0:self.out_c0 + self.cout]

    def reference(self):
        t = self.tensors()
        if 'ref' not in t:
            tin = t['tin'].data if self.stem else t['tin'].data[..., self.in_c0:self.in_c0 + self.cin]
            t['ref'] = fp64ref.split_conv_reference(tin, t['wp'], t['bp'], self.k, self.s, self.p, self.dil, self.act, residual=t['res'],
                                                    resid_first=self.resid_first, resid_scale=self.resid_scale,
                                                    up=t['up'].data if t['up'] else None, w_window=self.win, block_n=self.block_n,
                                                    cout=self.cout, out_h=self.Ho)
        return t['ref']

    def check(self, buf, what=''):
        """Checks (a) and (b) on the output buffer, and that nothing outside the output view was written.  -> worst error / bound.

        The output tile's TMA store writes whole 16-byte units of a pixel's channels: an fp32 view whose width is not a multiple of 4
        (85, 255) also gets the zero-padded weight rows' outputs, exact zeros, in the channels up to its next 16-byte boundary.  Views
        start on 16-byte boundaries, so those channels belong to no other view."""
        rest = buf.clone()
        end = self.out_c0 + self.cout
        pad_end = -(-end * buf.element_size() // 16) * 16 // buf.element_size()
        rest[..., self.out_c0:end] = float('nan')
        tail = rest[..., end:pad_end]
        assert bool((tail.isnan() | (tail == 0)).all()), f'{self.name}: nonzero values after the view, up to its 16-byte boundary'
        rest[..., end:pad_end] = float('nan')
        written = (~rest.isnan()).nonzero()
        assert written.numel() == 0, f'{self.name}: the kernel wrote outside its output view, channels {written[:, -1].unique().tolist()}'
        ref, bound = self.reference()
        return fp64ref.check_conv(fp64ref.conv_out64(self.view_of(buf)), ref, bound, f'{self.name}{what}')


# (name, kwargs).  Comments: the plan the case is there for (test_plan_coverage checks the table keeps covering every dimension).
CASES = [Case(n, **kw) for n, kw in [
    # block_n x K chunk, resident / streamed, CTAs per SM, classic loader
    ('bn32_bk16_cin16_1x1', dict(cin=16, cout=32, B=2, H=24, W=24)),
    ('bn32_bk32_cin96_3x3_classic_cout24', dict(cin=96, cout=24, k=3, B=2, H=16, W=20, halo=-1)),
    ('bn32_bk64_1x1_streamed', dict(cin=128, cout=32, B=2, H=24, W=24, no_resident=1)),
    ('bn64_bk16_cin48_3x3_ragged_batch3', dict(cin=48, cout=64, k=3, B=3, H=13, W=19, halo=-1)),
    ('bn64_bk32_cin32_1x1', dict(cin=32, cout=64, B=2, H=20, W=20)),
    ('bn64_bk64_1x1_cout40', dict(cin=64, cout=40, B=2, H=24, W=24)),
    ('bn64_pingpong_1x1_tma_residual', dict(cin=16, cout=64, B=1, H=40, W=40, residual=True)),
    ('bn128_bk64_3x3_pingpong', dict(cin=128, cout=128, k=3, B=2, H=20, W=20)),
    ('bn128_3x3_tma_residual_cooperative', dict(cin=64, cout=128, k=3, B=2, H=24, W=24, residual=True)),
    ('bn128_1x1_streamed_two_ntiles', dict(cin=128, cout=256, B=2, H=20, W=20, no_resident=1)),
    ('bn256_1x1', dict(cin=64, cout=256, B=2, H=16, W=16, block_n=256)),
    ('bn256_3x3_stride2', dict(cin=64, cout=256, k=3, s=2, B=2, H=17, W=23, block_n=256)),
    ('deep_k_3x3_cin512_classic', dict(cin=512, cout=64, k=3, B=1, H=16, W=16, halo=-1)),
    ('classic_stride2_odd_map', dict(cin=64, cout=64, k=3, s=2, B=1, H=13, W=19, halo=-1)),
    # halo loader
    ('halo1_cin32_3x3', dict(cin=32, cout=32, k=3, B=2, H=32, W=32, halo=1)),
    ('halo1_stride2_parity', dict(cin=32, cout=64, k=3, s=2, B=2, H=33, W=30, halo=1)),
    ('halo2_cin64_3x3_ragged', dict(cin=64, cout=64, k=3, B=1, H=13, W=19, halo=2)),
    ('halo2_stride2_parity_odd_map', dict(cin=128, cout=128, k=3, s=2, B=1, H=26, W=38, halo=2)),
    ('halo2_tma_residual', dict(cin=64, cout=64, k=3, B=2, H=24, W=24, residual=True, halo=2)),
    ('halo2_per_thread_residual_f32', dict(cin=64, cout=64, k=3, B=2, H=24, W=24, residual=True, act=None, f32=True, halo=2)),
    ('halo_auto_cin64_3x3', dict(cin=64, cout=64, k=3, B=2, H=24, W=24)),
    ('halo_auto_cin32_3x3_s2', dict(cin=32, cout=32, k=3, s=2, B=2, H=33, W=30)),
    # row-window stems
    ('stem_yolov5_160', dict(stem='yolov5', cout=32, B=2, H=160, W=160)),
    ('stem_yolov5_classic', dict(stem='yolov5', cout=32, B=1, H=64, W=96, halo=-1)),
    ('stem_yolov5_halo_kskip', dict(stem='yolov5', cout=32, B=2, H=64, W=96, halo=2)),
    ('stem_resnet', dict(stem='resnet', cout=64, act='relu', B=2, H=64, W=96)),
    # dilation
    ('dilation2', dict(cin=64, cout=64, k=3, dil=2, B=1, H=24, W=24)),
    ('deeplab_aspp_dilation12', dict(cin=128, cout=128, k=3, dil=12, act='relu', B=1, H=33, W=33)),
    # epilogues
    ('relu_residual_before_act', dict(cin=64, cout=256, act='relu', residual=True, resid_first=1, B=2, H=20, W=20)),
    ('scaled_residual_up_partial', dict(cin=128, cout=128, residual=True, resid_scale=0.75, up=True, B=2, H=18, W=22)),
    ('classic_per_thread_residual_f32', dict(cin=64, cout=64, k=3, residual=True, act=None, f32=True, B=2, H=16, W=16, halo=-1)),
    ('relu_3x3', dict(cin=64, cout=64, k=3, act='relu', B=2, H=16, W=16, halo=-1)),
    ('act_none_split_out', dict(cin=64, cout=64, act=None, B=2, H=16, W=16)),
    ('f32_out_cout85', dict(cin=64, cout=85, act=None, f32=True, B=2, H=16, W=16)),
    # ragged edges, channel slices, grid
    ('batch5_small_map', dict(cin=64, cout=64, B=5, H=7, W=9)),
    ('channel_slice_views_3x3', dict(cin=64, cout=64, k=3, B=2, H=16, W=20, in_c0=32, in_pitch=128, out_c0=64, out_pitch=192, halo=-1)),
    ('channel_slice_views_halo', dict(cin=32, cout=32, k=3, B=2, H=16, W=16, in_c0=64, in_pitch=128, out_c0=32, out_pitch=96, halo=2)),
    ('single_tile', dict(cin=64, cout=128, k=3, B=1, H=8, W=8)),
    ('odd_tiles_per_cta', dict(cin=128, cout=128, k=3, B=2, H=20, W=28, sm_limit=3)),
    ('many_tiles_3x3', dict(cin=64, cout=64, k=3, B=4, H=80, W=80, halo=-1)),
    # real layers of the bench models at small batch
    ('yolov5_3x3s2_64_128_80', dict(cin=64, cout=128, k=3, s=2, B=2, H=80, W=80)),
    ('yolov5_head_256_255_f32', dict(cin=256, cout=255, act=None, f32=True, B=1, H=40, W=40)),
    ('fcos_tower_3x3_256', dict(cin=256, cout=256, k=3, act=None, B=1, H=20, W=24)),
]]
BY_NAME = {c.name: c for c in CASES}
assert len(BY_NAME) == len(CASES)


# ------------------------------------------------------------------------------------------------- plan lines and child processes
def parse_plan_line(line):
    """'[cvb plan] cin=64 ... schedule=pingpong epi=1 pdl=0' -> {'cin': 64, ..., 'schedule': 'pingpong', ...}"""
    f = {}
    for k, v in re.findall(r'(\S+?)=(\S+)', line):
        f[k] = int(v) if re.fullmatch(r'-?\d+', v) else v
    return f


def parse_child_stderr(text):
    """-> [(entry label, plan fields)], one per plan, from the `[case] <label>` marker printed before each plan creation."""
    out, label = [], None
    for line in text.splitlines():
        if line.startswith('[case] '):
            label = line[7:].strip()
        elif line.startswith('[cvb plan] '):
            out.append((label, parse_plan_line(line)))
    return out


# CVB_HALO* knobs are read at every plan creation: (label, env, cases) variants of the auto-halo cases.  Two CTAs per SM need
# block_n <= 64 and a ring that fits half the shared memory: only the 32-channel layer has such a halo plan.
HALO_ENV_CASES = ['halo_auto_cin64_3x3', 'halo_auto_cin32_3x3_s2']
HALO_ENVS = [
    ('halo0', {'CVB_HALO': '0'}, HALO_ENV_CASES),
    ('halo1', {'CVB_HALO': '1'}, HALO_ENV_CASES),
    ('halo2', {'CVB_HALO': '2'}, HALO_ENV_CASES),
    ('halo2_bk32', {'CVB_HALO': '2', 'CVB_HALO_BK': '32'}, HALO_ENV_CASES),
    ('halo2_streamed', {'CVB_HALO': '2', 'CVB_HALO_RES': '0'}, HALO_ENV_CASES),
    ('halo2_ctas1', {'CVB_HALO': '2', 'CVB_HALO_CTAS': '1'}, HALO_ENV_CASES),
    ('halo2_ctas2', {'CVB_HALO': '2', 'CVB_HALO_CTAS': '2'}, ['halo_auto_cin32_3x3_s2']),
]
HALO_RUNS = [(n, label, env) for label, env, names in HALO_ENVS for n in names]
HALO_KEYS = ('CVB_HALO', 'CVB_HALO_BK', 'CVB_HALO_RES', 'CVB_HALO_CTAS')


def _set_env(env):
    for k in HALO_KEYS:
        os.environ.pop(k, None)
    os.environ.update(env)


def pdl_chain():
    """Four dependent layers run back to back with ops.run_plans: A -> B (3x3), B -> C (1x1), C -> B with residual A (B was the previous
    layer's input: write after read), B -> D (3x3).  Every layer reads the previous one's output (read after write).  -> (B, D)."""
    from cvpytorch_b200 import ops
    g = torch.Generator().manual_seed(21)
    Bn, H, W = 2, 24, 24
    bufs = {n: ops.SplitTensor(Bn, H, W, c) for n, c in (('A', 64), ('B', 64), ('C', 128), ('D', 64))}
    ops.nchw_to_split(torch.randn(Bn, 64, H, W, generator=g).cuda(), bufs['A'].view())
    plans = []
    for src, dst, cin, cout, k, act, res in (('A', 'B', 64, 64, 3, 'silu', None), ('B', 'C', 64, 128, 1, 'silu', None),
                                             ('C', 'B', 128, 64, 1, 'silu', 'A'), ('B', 'D', 64, 64, 3, 'relu', None)):
        w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
        wp, bp = ops.pack_conv_weights(w.double(), (torch.randn(cout, generator=g) * 0.5).double())
        plans.append(ops.ConvPlan(bufs[src].view(), bufs[dst].view(), wp, bp, k, 1, k // 2, 1, act,
                                  residual=bufs[res].view() if res else None))
    ops.run_plans(plans)
    torch.cuda.synchronize()
    return bufs['B'].data.clone(), bufs['D'].data.clone()


def _child_main(argv):
    """--plans: create the plan of every case (and the CVB_HALO* variants); --run OUT: run every case and the PDL chain, save outputs."""
    torch.cuda.init()
    if argv[0] == '--plans':
        for c in CASES:
            print(f'[case] {c.name}', file=sys.stderr, flush=True)
            c.plan()
        for n, label, env in HALO_RUNS:
            _set_env(env)
            print(f'[case] {n}@{label}', file=sys.stderr, flush=True)
            BY_NAME[n].plan()
        _set_env({})
    else:
        outs = {}
        for c in CASES:
            print(f'[case] {c.name}', file=sys.stderr, flush=True)
            outs[c.name] = c.run().cpu()
        print('[case] pdl_chain', file=sys.stderr, flush=True)
        outs['pdl_chain'] = tuple(t.cpu() for t in pdl_chain())
        torch.save(outs, argv[1])


CHILD_KNOBS = {
    'epi_spec0': {'CVB_EPI_SPEC': '0'},
    'resid_tma0': {'CVB_RESID_TMA': '0'},
    'bk_smalln32': {'CVB_BK_SMALLN': '32'},
    'bk_smalln16': {'CVB_BK_SMALLN': '16'},
    'split_n128_0': {'CVB_SPLIT_N128': '0'},
    'ctas_per_sm1': {'CVB_CTAS_PER_SM': '1'},
    'pdl1': {'CVB_PDL': '1'},
}
CHILD_TIMEOUT = 300


@pytest.fixture(scope='module')
def children(cuda, tmp_path_factory):
    """Starts one child per knob (and one that only creates the default plans) at once, waits for all of them -> {knob: (plans, outputs
    path)}.  Every child has exited when this returns."""
    tmp = tmp_path_factory.mktemp('conv_plans')
    base = {k: v for k, v in os.environ.items() if not k.startswith('CVB_')}
    base['CVB_PLAN_DEBUG'] = '1'
    procs, logs = {}, {}
    jobs = [('plans', ['--plans'], {})] + [(knob, ['--run', str(tmp / f'{knob}.pt')], env) for knob, env in CHILD_KNOBS.items()]
    try:
        for knob, args, env in jobs:
            logs[knob] = open(tmp / f'{knob}.log', 'w')
            procs[knob] = subprocess.Popen([sys.executable, os.path.abspath(__file__)] + args, env={**base, **env}, cwd=ROOT,
                                           stdout=subprocess.DEVNULL, stderr=logs[knob])
        res = {}
        for knob, p in procs.items():
            p.wait(timeout=CHILD_TIMEOUT)
            logs[knob].close()
            err = (tmp / f'{knob}.log').read_text()
            assert p.returncode == 0, f'child {knob} failed ({p.returncode}):\n{err[-3000:]}'
            res[knob] = (parse_child_stderr(err), tmp / f'{knob}.pt')
    finally:
        for p in procs.values():
            if p.poll() is None:
                p.kill()
                p.wait()
        for f in logs.values():
            f.close()
    return res


@pytest.fixture(scope='module')
def default_plans(children):
    """{case name (or name@halo-variant): plan fields} of the default knobs."""
    d = dict(children['plans'][0])
    assert len(d) == len(CASES) + len(HALO_RUNS), sorted(d)
    return d


@pytest.fixture(scope='module')
def default_outputs(cuda):
    """Every case run in this process (default knobs) -> {name: whole output buffer}."""
    return {c.name: c.run() for c in CASES}


# --------------------------------------------------------------------------------------------------------------- the plan matrix
@pytest.mark.parametrize('name', [c.name for c in CASES])
def test_conv_plan_matrix(default_outputs, name):
    c = BY_NAME[name]
    r = c.check(default_outputs[name])
    print(f'{name}: worst error / bound {r:.3f}')


@pytest.mark.parametrize('name', ['stem_yolov5_160', 'stem_resnet'])
def test_stem_window_packing(cuda, name):
    """The row-window reference (window-packed weights over the padded space-to-depth input) equals the original 6x6/s2/p2 or 7x7/s2/p3
    conv in float64 up to the hi / lo rounding of inputs and weights (2^-22 relative each): the packing is the stem."""
    c = BY_NAME[name]
    t = c.tensors()
    x, w, b, s, p = t['orig']
    x64, w64 = x.double().cuda(), w.double().cuda()
    orig = F.conv2d(x64, w64, b.double().cuda(), s, p)
    absorig = F.conv2d(x64.abs(), w64.abs(), b.double().cuda().abs(), s, p)
    orig = F.silu(orig) if c.act == 'silu' else F.relu(orig)
    ref, _ = c.reference()
    fp64ref.check(ref, orig, 1.1 * 2.0 ** -20 * absorig + 1e-30, f'{name}: window packing')


# ------------------------------------------------------------------------------------------------------------------ plan coverage
def _tiles_per_cta_odd(f):
    return f['grid'] < f['tiles'] and math.ceil(f['tiles'] / f['grid']) % 2 == 1


def _ragged(c):
    return c.Ho % 8 != 0 or c.Wo % 8 != 0


# (plan dimension, predicate on (case, plan fields)).  When a planner change moves a case off one of these, update CASES.
COVERAGE = [
    ('block_n 32', lambda c, f: f['bn'] == 32),
    ('block_n 64', lambda c, f: f['bn'] == 64),
    ('block_n 128', lambda c, f: f['bn'] == 128),
    ('block_n 256', lambda c, f: f['bn'] == 256),
    ('K chunk 16 (cin 16 or 48)', lambda c, f: f['bk'] == 16 and f['cin'] in (16, 48)),
    ('K chunk 32 (cin 32 or 96)', lambda c, f: f['bk'] == 32 and f['cin'] in (32, 96)),
    ('K chunk 64', lambda c, f: f['bk'] == 64),
    ('resident weights', lambda c, f: f['resident'] == 1),
    ('streamed weights', lambda c, f: f['resident'] == 0),
    ('one CTA per SM', lambda c, f: f['ctas/sm'] == 1),
    ('two CTAs per SM', lambda c, f: f['ctas/sm'] == 2),
    ('two CTAs per SM, classic loader', lambda c, f: f['ctas/sm'] == 2 and f['halo'] == 0),
    ('classic loader', lambda c, f: f['halo'] == 0 and f['k'] != '1x1'),
    ('classic loader, stride 2', lambda c, f: f['halo'] == 0 and c.s == 2),
    ('halo mode 1', lambda c, f: f['halo'] == 1),
    ('halo mode 2', lambda c, f: f['halo'] == 2),
    ('halo loader, stride 2 (parity maps)', lambda c, f: f['halo'] > 0 and c.s == 2),
    ('YOLOv5 row-window stem, kskip 1', lambda c, f: c.stem == 'yolov5' and f['kskip'] == 1),
    ('ResNet row-window stem, kskip 0', lambda c, f: c.stem == 'resnet' and f['kskip'] == 0),
    ('row-window stem, classic loader', lambda c, f: c.stem is not None and f['halo'] == 0),
    ('dilation 2', lambda c, f: c.dil == 2),
    ('large dilation', lambda c, f: c.dil >= 12),
    ('cooperative schedule', lambda c, f: f['schedule'] == 'cooperative'),
    ('ping-pong schedule', lambda c, f: f['schedule'] == 'pingpong'),
    ('ping-pong, narrow n-tile', lambda c, f: f['schedule'] == 'pingpong' and f['bn'] <= 64),
    ('SiLU', lambda c, f: c.act == 'silu'),
    ('ReLU', lambda c, f: c.act == 'relu'),
    ('no activation', lambda c, f: c.act is None),
    ('specialised SiLU epilogue', lambda c, f: f['epi'] == 1),
    ('specialised SiLU + residual epilogue', lambda c, f: f['epi'] == 2),
    ('specialised ReLU epilogue', lambda c, f: f['epi'] == 3),
    ('specialised ReLU(x + residual) epilogue', lambda c, f: f['epi'] == 4),
    ('TMA residual', lambda c, f: c.residual and f['resid_tma'] == 1),
    ('per-thread residual, classic loader', lambda c, f: c.residual and f['resid_tma'] == 0 and f['halo'] == 0),
    ('per-thread residual, halo loader', lambda c, f: c.residual and f['resid_tma'] == 0 and f['halo'] > 0),
    ('residual before the activation', lambda c, f: c.resid_first == 1),
    ('scaled residual', lambda c, f: c.residual and c.resid_scale != 1.0),
    ('up-sampled partial', lambda c, f: c.up),
    ('f32 out', lambda c, f: c.f32),
    ('map not a multiple of the box', lambda c, f: _ragged(c)),
    ('batch not a multiple of the box', lambda c, f: c.B in (3, 5)),
    ('cout not a multiple of 8 (f32 out)', lambda c, f: c.f32 and c.cout % 8 != 0),
    ('cout below the n-tile, block_n 64', lambda c, f: f['bn'] == 64 and c.cout < 64),
    ('cout below the n-tile, block_n 32', lambda c, f: f['bn'] == 32 and c.cout < 32),
    ('channel-slice input and output, classic', lambda c, f: c.in_c0 > 0 and c.out_c0 > 0 and f['halo'] == 0),
    ('channel-slice input and output, halo', lambda c, f: c.in_c0 > 0 and c.out_c0 > 0 and f['halo'] > 0),
    ('more tiles than CTAs', lambda c, f: f['tiles'] > f['grid']),
    ('fewer tiles than CTAs', lambda c, f: f['tiles'] == f['grid'] and c.sm_limit == 0 and f['tiles'] < 100),
    ('sm_limit with an odd number of tiles per CTA', lambda c, f: c.sm_limit > 0 and _tiles_per_cta_odd(f)),
]


def test_plan_coverage(default_plans):
    """Every plan dimension of COVERAGE occurs in the default plans of CASES."""
    for name in BY_NAME:
        f = default_plans[name]
        print(f"{name}: bn={f['bn']} bk={f['bk']} stages={f['stages']} resident={f['resident']} ctas/sm={f['ctas/sm']} "
              f"resid_tma={f['resid_tma']} halo={f['halo']} kskip={f['kskip']} {f['schedule']} epi={f['epi']} grid={f['grid']} "
              f"tiles={f['tiles']}")
    missing = [dim for dim, pred in COVERAGE if not any(pred(c, default_plans[c.name]) for c in CASES)]
    assert not missing, f'plan dimensions no case of CASES reaches any more: {missing}'


# ------------------------------------------------------------------------------------------------------------------ A/B knob paths
def _same_k_order(d, k):
    """Two plans of one layer chain every element's K steps in the same order: both classic (tap-major, `it = tap * chunks + ck`), or
    the same halo mode and K chunk (chunk-major over the copies)."""
    return (d['halo'] == 0 and k['halo'] == 0) or (d['halo'] == k['halo'] and d['bk'] == k['bk'])


def _knob_compare(children, default_plans, default_outputs, knob):
    """Child outputs under `knob` vs the default: bitwise where the K order is unchanged, else the float64 bound.  -> (default plans,
    knob plans, names compared bitwise)."""
    plans, path = children[knob]
    kp = dict(plans)
    outs = torch.load(path)
    bitwise = []
    for c in CASES:
        d, k = default_plans[c.name], kp[c.name]
        got = outs[c.name].cuda()
        if _same_k_order(d, k):
            a, b = c.view_of(default_outputs[c.name]), c.view_of(got)
            bits = torch.int32 if c.f32 else torch.int16
            assert torch.equal(a.contiguous().view(bits), b.contiguous().view(bits)), (
                f'{knob}: {c.name} differs from the default plan although the K order is the same\n  default {d}\n  {knob} {k}')
            bitwise.append(c.name)
        else:
            r = c.check(got, f' under {knob}')
            print(f'{knob}: {c.name} on another loader: worst error / bound {r:.3f}')
    assert bitwise
    return kp, bitwise


def test_knob_generic_epilogue(children, default_plans, default_outputs):
    """CVB_EPI_SPEC=0: the generic epilogue on the SiLU / ReLU hot modes gives bitwise-equal outputs."""
    kp, _ = _knob_compare(children, default_plans, default_outputs, 'epi_spec0')
    spec = [n for n in BY_NAME if default_plans[n]['epi'] != 0]
    assert spec and all(kp[n]['epi'] == 0 for n in spec), [(n, kp[n]['epi']) for n in spec]


def test_knob_per_thread_residual(children, default_plans, default_outputs):
    """CVB_RESID_TMA=0: per-thread residual loads give bitwise-equal outputs."""
    kp, _ = _knob_compare(children, default_plans, default_outputs, 'resid_tma0')
    tma = [n for n in BY_NAME if default_plans[n]['resid_tma'] == 1]
    assert tma and all(kp[n]['resid_tma'] == 0 for n in tma), [(n, kp[n]['resid_tma']) for n in tma]


@pytest.mark.parametrize('bk', [32, 16])
def test_knob_half_k_chunks(children, default_plans, default_outputs, bk):
    """CVB_BK_SMALLN=32 / 16: narrower K chunks of the narrow 1x1 plans on 64-channel inputs keep every element's K order."""
    kp, _ = _knob_compare(children, default_plans, default_outputs, f'bk_smalln{bk}')
    changed = [n for n in BY_NAME if default_plans[n]['bk'] != bk and kp[n]['bk'] == bk]
    assert changed, f'CVB_BK_SMALLN={bk} changed no plan'


def test_knob_split_n128_off(children, default_plans, default_outputs):
    """CVB_SPLIT_N128=0: the 128 -> 128 1x1 layer with an up-sampled partial as one 128-wide tile instead of two 64-wide ones."""
    kp, _ = _knob_compare(children, default_plans, default_outputs, 'split_n128_0')
    split = [n for n in BY_NAME if default_plans[n]['bn'] == 64 and BY_NAME[n].cout == 128 and BY_NAME[n].block_n == 0]
    assert split and all(kp[n]['bn'] == 128 for n in split), [(n, kp[n]['bn']) for n in split]


def test_knob_one_cta_per_sm(children, default_plans, default_outputs):
    """CVB_CTAS_PER_SM=1: bitwise equal on the classic-loader plans; the layers that thereby leave the halo loader (chunk-major K order)
    are checked against the float64 bound."""
    kp, bitwise = _knob_compare(children, default_plans, default_outputs, 'ctas_per_sm1')
    two = [n for n in BY_NAME if default_plans[n]['ctas/sm'] == 2]
    assert two and all(kp[n]['ctas/sm'] == 1 for n in two), [(n, kp[n]['ctas/sm']) for n in two]
    assert any(default_plans[n]['halo'] == 0 for n in two if n in bitwise), 'no classic two-CTA plan compared bitwise'


def test_knob_programmatic_dependent_launch(children, default_plans, default_outputs):
    """CVB_PDL=1: every case, and a chain of four dependent layers through ops.run_plans (read after write and write after read between
    consecutive layers), bitwise equal to the default launches."""
    kp, _ = _knob_compare(children, default_plans, default_outputs, 'pdl1')
    assert all(f['pdl'] == 1 for f in kp.values()) and all(f['pdl'] == 0 for f in default_plans.values())
    ref = pdl_chain()
    got = torch.load(children['pdl1'][1])['pdl_chain']
    for r, g in zip(ref, got):
        assert bool(torch.isfinite(r).all())
        assert torch.equal(r.cpu().view(torch.int16), g.view(torch.int16))


@pytest.mark.parametrize('name,label,env', HALO_RUNS, ids=[f'{n}-{label}' for n, label, _ in HALO_RUNS])
def test_knob_halo(default_plans, monkeypatch, name, label, env):
    """CVB_HALO / CVB_HALO_BK / CVB_HALO_RES / CVB_HALO_CTAS (read at every plan creation): the plan takes the requested loader, K chunk,
    residency and CTAs per SM, and its output stays within the float64 bound."""
    f = default_plans[f'{name}@{label}']
    mode = int(env['CVB_HALO'])
    assert f['halo'] == mode, f
    if 'CVB_HALO_BK' in env:
        assert f['bk'] == int(env['CVB_HALO_BK']), f
    if 'CVB_HALO_RES' in env:
        assert f['resident'] == 0, f
    if 'CVB_HALO_CTAS' in env:
        assert f['ctas/sm'] == int(env['CVB_HALO_CTAS']), f
    for k in HALO_KEYS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    c = BY_NAME[name]
    r = c.check(c.run(), f' under {env}')
    print(f'{name} {env}: worst error / bound {r:.3f}')


# ------------------------------------------------------------------------------------------------------------------------- teeth
def _rejected(fn):
    try:
        fn()
    except AssertionError:
        return True
    return False


@pytest.mark.parametrize('name', ['bn64_bk64_1x1_cout40', 'halo2_cin64_3x3_ragged', 'stem_yolov5_160', 'f32_out_cout85',
                                  'bn256_3x3_stride2'])
def test_conv_checks_teeth(default_outputs, name):
    """Each of the matrix's checks rejects a subtly wrong output: one element moved by twice its own bound, one element left NaN."""
    c = BY_NAME[name]
    ref, bound = c.reference()
    out = fp64ref.conv_out64(c.view_of(default_outputs[name]))
    fp64ref.check_conv(out, ref, bound, name)
    idx = tuple(int(i) for i in torch.unravel_index(torch.argmax(ref.abs()).cpu(), ref.shape))
    moved = out.clone()
    e = float(moved[idx] - ref[idx])
    moved[idx] += (1.0 if e >= 0 else -1.0) * 2 * float(bound[idx])
    assert _rejected(lambda: fp64ref.check(moved, ref, bound, name))
    nan = out.clone()
    nan[idx] = float('nan')
    assert _rejected(lambda: fp64ref.check(nan, ref, bound, name))
    assert _rejected(lambda: fp64ref.check_conv(nan, ref, bound, name))


def test_conv_checks_teeth_lost_lo_plane(cuda):
    """A short-K SiLU layer (1x1, cin 64) whose outputs with |y| < 0.25 lose their lo plane (errors up to half an fp16 ulp, 2^-14 at
    most) is rejected by the element-wise bound (a), while the max-normalised check (b) alone accepts it: what (a) adds."""
    c = Case('short_k_silu', cin=64, cout=64, B=2, H=32, W=32)
    buf = c.run()
    c.check(buf)
    ref, bound = c.reference()
    small = buf[0].abs() < 0.25
    bad = buf.clone()
    bad[1][small] = 0
    out = fp64ref.conv_out64(bad)
    assert float((out - ref).abs().max()) > 0
    assert fp64ref.max_rel(out, ref) < fp64ref.LAYER_BUDGET, 'check (b) alone rejects the lost lo plane already'
    assert _rejected(lambda: fp64ref.check(out, ref, bound, 'lost lo plane'))


# ----------------------------------------------------------------------------------------------------------- YOLOv5 decode paths
def sigmoid_fast_rel_err(z):
    """Relative error of sigmoid_fast(z) = rcp.approx(1 + ex2.approx(z * -log2 e)) (csrc/internal.h): ex2.approx of the rounded
    product is __expf(-z), within 2 + floor(1.173 |z|) ulps (CUDA programming guide, intrinsic functions); 1 + e rounds once
    (2^-24); rcp.approx is within one ulp (2^-23).  An error eta of e moves sigma by sigma (1 - sigma) eta <= sigma eta."""
    return (2 + 1.173 * z.abs()) * fp64ref.U23 + fp64ref.U24 + fp64ref.U23


def decode_reference(x, dx, anchors, stride, nx):
    """float64 YOLOv5 decode (oracle/yolov5_oracle.py) of pre-activations x [B, na, npix, no] known to within dx (element-wise) ->
    (z, bound), both [B, na, npix, no].

      y  = sigmoid(x):            |y^ - y| <= e_y = dx / 4 + r (y + dx / 4),  r = sigmoid_fast_rel_err(|x| + dx)   (sigmoid' <= 1/4)
      xy = (2 y - 0.5 + grid) s:  2 y^ is exact; three fp32 roundings of values <= (|2y - 0.5| + grid + 2 e_y) s
                                   -> 2 e_y s + 3 u (|2 y - 0.5| + grid + 2 e_y) s
      wh = (2 y)^2 a:             |4 y^2 - 4 y^^2| <= (8 y + 4 e_y) e_y, two fp32 roundings of values <= 4 (y + e_y)^2 a
      obj, cls = y:               e_y
    u = 2^-24; a tiny absolute 2^-120 covers the flush to zero of ex2 / rcp at |x| > 87."""
    u = fp64ref.U24
    y = torch.sigmoid(x)
    r = sigmoid_fast_rel_err(x.abs() + dx)
    ey = dx / 4 + r * (y + dx / 4) + 2.0 ** -120
    npix = x.shape[2]
    pix = torch.arange(npix, device=x.device)
    gx, gy = (pix % nx).double(), (pix // nx).double()
    z, bound = y.clone(), ey.clone()
    for j, gr in ((0, gx), (1, gy)):
        g = gr.view(1, 1, -1)
        z[..., j] = (2 * y[..., j] - 0.5 + g) * stride
        bound[..., j] = 2 * ey[..., j] * stride + 3 * u * ((2 * y[..., j] - 0.5).abs() + g + 2 * ey[..., j]) * stride
    for j in (2, 3):
        a = anchors[:, j - 2].view(1, -1, 1)
        z[..., j] = (2 * y[..., j]) ** 2 * a
        bound[..., j] = ((8 * y[..., j] + 4 * ey[..., j]) * ey[..., j] + 2 * u * 4 * (y[..., j] + ey[..., j]) ** 2) * a
    return z, bound


def nms_consistency(z, hist, rowmax, conf, multi, what):
    """The NMS histogram and per-row best score equal what the NMS recomputes from the decoded rows z [B, rows, no] (fp32): score =
    fp32(cls * obj); rowmax = the best score if it is > conf, else 0; histogram bin = fp32 bits >> 17 clamped to 16383, of every score
    > conf (multi-label) or of every rowmax > conf (best class)."""
    sc = z[..., 5:] * z[..., 4:5]  # fp32 products, rounded to nearest as the kernels' __fmul_rn
    best = sc.max(-1).values
    rm = torch.where(best > conf, best, torch.zeros_like(best))
    assert torch.equal(rowmax, rm), f'{what}: rowmax differs in {int((rowmax != rm).sum())} rows'
    B = z.shape[0]
    ref = torch.zeros(B, 16384, dtype=torch.int64, device=z.device)
    for b in range(B):
        v = sc[b][sc[b] > conf] if multi else rm[b][rm[b] > conf]
        bins = (v.view(torch.int32).long() >> 17).clamp(max=16383)
        ref[b] = torch.bincount(bins, minlength=16384)
    assert int(ref.sum()) > 0, f'{what}: no candidate above conf; the case tests nothing'
    assert torch.equal(hist.long(), ref), f'{what}: histogram differs in {int((hist.long() != ref).sum())} bins'


def _decode_check(z, zref, zbound, what):
    r = fp64ref.check(z, zref, zbound, what)
    print(f'{what}: worst error / bound {r:.3f}')
    return r


@pytest.mark.parametrize('no,multi', [(85, True), (85, False), (64, True)])
def test_fused_decode_vs_formula(cuda, no, multi):
    """The fused CVB_OUT_YOLO epilogue against the float64 decode of the float64 conv (pre-activation bound of
    fp64ref.split_conv_reference, block_n 128), and its histogram / rowmax against its own z."""
    from cvpytorch_b200 import ops
    B, ny, nx, cin, na, z_off, stride = 2, 12, 20, 64, 3, 3, 16.0
    g = torch.Generator().manual_seed(40 + no)
    x = torch.randn(B, cin, ny, nx, generator=g)
    w = (torch.randn(na * no, cin, 1, 1, generator=g) * (2.5 / cin ** 0.5)).double()
    b = (torch.randn(na * no, generator=g) * 0.5).double()
    tin = ops.SplitTensor(B, ny, nx, cin)
    ops.nchw_to_split(x.cuda(), tin.view())
    anchors = torch.tensor([[10., 13.], [16., 30.], [33., 23.]])
    A, conf = na * ny * nx + z_off + 5, 0.05
    ws = ops.NmsWorkspace(B, A, no - 5)
    ops.nms_reset(ws)
    z = torch.full((B, A, no), float('nan'), device='cuda')
    wy, by = ops.pack_yolo_head_weights(w, b, na, no)
    y = ops.yolo_decode_desc(na, no, anchors, stride, z, A, z_off, ws, conf, multi)
    ops.ConvPlan(tin.view(), ops.CvbView(z.data_ptr(), B, ny, nx, na * 128, na * 128, 0), wy, by, 1, 1, 0, 1, None, yolo=y).run()
    torch.cuda.synchronize()
    ref, bound = fp64ref.split_conv_reference(tin, wy, by, 1, act=None, block_n=128)  # [B, na*128, ny, nx]
    npix = ny * nx
    xr = ref.view(B, na, 128, npix).permute(0, 1, 3, 2)[..., :no]
    dx = bound.view(B, na, 128, npix).permute(0, 1, 3, 2)[..., :no]
    zref, zbound = decode_reference(xr, dx, anchors.double().cuda(), stride, nx)
    zl = z[:, z_off:z_off + na * npix]
    _decode_check(zl.view(B, na, npix, no), zref, zbound, f'fused decode no={no}')
    assert bool(z[:, :z_off].isnan().all()) and bool(z[:, z_off + na * npix:].isnan().all()), 'fused decode wrote outside its z rows'
    hist, rowmax = _ws_regions(ws, B, A)
    torch.cuda.synchronize()
    nms_consistency(zl, hist, rowmax[:, z_off:z_off + na * npix], conf, multi and no - 5 > 1, f'fused decode no={no}')


DECODE_CASES = [  # (no, multi, hist, na, nx, xperm)
    (64, True, True, 3, 13, False), (85, True, True, 3, 13, False), (85, False, True, 3, 13, False), (96, True, True, 3, 13, False),
    (96, False, True, 3, 13, False), (85, True, False, 3, 13, False),
    (85, True, False, 3, 13, True),    # xperm: the raw rows of the want_raw graph
    (85, True, True, 3, 13, True),     # xperm and the histogram
    (8, True, True, 2, 13, False),     # small no, two anchors
    (6, False, True, 3, 13, False),    # one class
    (85, True, True, 3, 1, False),     # nx = 1
    (6, False, True, 1, 20800, False),  # pix * nx >= 2^32: real division instead of the multiply-high
]


def _decode_id(c):
    no, multi, hist, na, nx, xperm = c
    return f'{no}-{multi}-{hist}' + (f'-na{na}' if na != 3 else '') + (f'-nx{nx}' if nx != 13 else '') + ('-xperm' if xperm else '')


@pytest.mark.parametrize('no,multi,hist,na,nx,xperm', DECODE_CASES, ids=[_decode_id(c) for c in DECODE_CASES])
def test_fast_decode_vs_formula(cuda, no, multi, hist, na, nx, xperm):
    """yolo_decode_kernel (cvb_yolo_decode) against the float64 decode of its own fp32 input (dx = 0), also max-normalised within
    5e-6; its xperm rows equal the permuted raw tensor bit for bit; its histogram / rowmax (both variants) against its own z."""
    from cvpytorch_b200 import ops
    B, ny, z_off, stride = 2, 10, 2, 8.0
    g = torch.Generator().manual_seed(60 + no)
    pitch = (na * no + 7) // 8 * 8
    raw = ops.F32Tensor(B, ny, nx, pitch)
    raw.data.copy_(torch.randn(B, ny, nx, pitch, generator=g) * 3)
    anchors = torch.tensor([[10., 13.], [16., 30.], [33., 23.]])[:na]
    A, conf = na * ny * nx + z_off + 3, 0.05
    ws = ops.NmsWorkspace(B, A, no - 5)
    ops.nms_reset(ws)
    z = torch.full((B, A, no), float('nan'), device='cuda')
    xp = torch.full((B, na, ny, nx, no), float('nan'), device='cuda') if xperm else None
    ops.yolo_decode(raw.view(0, na * no), na, no, anchors.cuda().contiguous(), stride, z, A, z_off, xp, ws if hist else None, conf, multi)
    torch.cuda.synchronize()
    npix = ny * nx
    xr = raw.data[..., :na * no].view(B, npix, na, no).permute(0, 2, 1, 3)
    if xperm:
        assert torch.equal(xp.view(B, na, npix, no), xr), 'xperm is not the permuted raw tensor'
    xr = xr.double()
    zref, zbound = decode_reference(xr, torch.zeros_like(xr), anchors.double().cuda(), stride, nx)
    zl = z[:, z_off:z_off + na * npix]
    _decode_check(zl.view(B, na, npix, no), zref, zbound, f'decode no={no}')
    assert fp64ref.max_rel(zl.view(B, na, npix, no), zref) < 5e-6
    assert bool(z[:, :z_off].isnan().all()) and bool(z[:, z_off + na * npix:].isnan().all()), 'decode wrote outside its z rows'
    if hist:
        h, rowmax = _ws_regions(ws, B, A)
        nms_consistency(zl, h, rowmax[:, z_off:z_off + na * npix], conf, multi and no - 5 > 1, f'decode no={no}')


@pytest.mark.parametrize('producer', ['yolov6_decode', 'count_pass'])
@pytest.mark.parametrize('nc,multi', [(80, True), (80, False), (1, True), (1, False)])
def test_prepass_producers_vs_z(cuda, producer, nc, multi):
    """The histogram / rowmax of the other two producers of the NMS pre-pass against their own z: cvb_yolov6_decode and the NMS counting
    pass (yolo_nms with hist_ready=False).  With one class both multi_label values must build the best-class pre-pass (the reference's
    multi_label &= nc > 1, applied by the C entry points), and the counting pass's NMS rows equal the oracle's for both."""
    from cvpytorch_b200 import ops
    from oracle import nms_oracle as NO
    B, ny, nx, z_off, conf = 2, 10, 13, 2, 0.05
    no, A = nc + 5, ny * nx + z_off + 3
    g = torch.Generator().manual_seed(90 + nc)
    ws = ops.NmsWorkspace(B, A, nc)
    if producer == 'yolov6_decode':
        cls, reg = ops.F32Tensor(B, ny, nx, (nc + 31) // 32 * 32), ops.F32Tensor(B, ny, nx, 32)
        cls.data.copy_(torch.randn(cls.data.shape, generator=g) * 3)
        reg.data.copy_(torch.rand(reg.data.shape, generator=g) * 4)
        z = torch.full((B, A, no), float('nan'), device='cuda')
        ops.nms_reset(ws)
        ops.yolov6_decode(cls.view(0, nc), reg.view(0, 4), nc, 8.0, z, A, z_off, ws, conf, multi)
        rows = slice(z_off, z_off + ny * nx)
    else:
        z = torch.rand(B, A, no, generator=g)
        z[..., :2] *= 640
        z[..., 2:4] *= 64
        z = z.cuda()
        det, idx, cnt = ops.yolo_nms(z, ws, conf, 0.6, multi)
        rows = slice(0, A)
    torch.cuda.synchronize()
    h, rowmax = _ws_regions(ws, B, A)
    nms_consistency(z[:, rows], h, rowmax[:, rows], conf, multi and nc > 1, f'{producer} nc={nc} multi={multi}')
    if producer == 'count_pass':
        assert int(ws.status[0]) == 0
        ref = NO.non_max_suppression(z.cpu().numpy(), conf, 0.6, multi_label=multi)
        for b in range(B):
            k = int(cnt[b])
            assert k == ref[b][0].shape[0] and torch.equal(idx[b, :k].cpu().long(), torch.from_numpy(ref[b][1]))
            assert torch.equal(det[b, :k].cpu(), torch.from_numpy(ref[b][0]))


def test_decode_checks_teeth(cuda):
    """The decode checks reject one z element moved by twice its bound, one NaN, and a histogram count or a rowmax off by one step."""
    from cvpytorch_b200 import ops
    B, ny, nx, na, no, stride = 1, 6, 7, 3, 85, 8.0
    g = torch.Generator().manual_seed(77)
    raw = ops.F32Tensor(B, ny, nx, 256)
    raw.data.copy_(torch.randn(B, ny, nx, 256, generator=g) * 3)
    anchors = torch.tensor([[10., 13.], [16., 30.], [33., 23.]])
    A, conf = na * ny * nx, 0.05
    ws = ops.NmsWorkspace(B, A, no - 5)
    ops.nms_reset(ws)
    z = torch.zeros(B, A, no, device='cuda')
    ops.yolo_decode(raw.view(0, na * no), na, no, anchors.cuda().contiguous(), stride, z, A, 0, None, ws, conf, True)
    torch.cuda.synchronize()
    xr = raw.data[..., :na * no].double().view(B, ny * nx, na, no).permute(0, 2, 1, 3)
    zref, zbound = decode_reference(xr, torch.zeros_like(xr), anchors.double().cuda(), stride, nx)
    zz = z.view(B, na, ny * nx, no).double()
    fp64ref.check(zz, zref, zbound, 'decode')
    for j in (0, 2, 4, 40):
        moved = zz.clone()
        moved[0, 1, 5, j] += 2 * float(zbound[0, 1, 5, j]) * (1 if float(moved[0, 1, 5, j] - zref[0, 1, 5, j]) >= 0 else -1)
        assert _rejected(lambda: fp64ref.check(moved, zref, zbound, 'decode'))
    nan = zz.clone()
    nan[0, 2, 3, 7] = float('nan')
    assert _rejected(lambda: fp64ref.check(nan, zref, zbound, 'decode'))
    h, rowmax = _ws_regions(ws, B, A)
    nms_consistency(z, h, rowmax, conf, True, 'decode')
    hb = h.clone()
    i = int(torch.nonzero(hb[0])[0])
    hb[0, i] += 1
    assert _rejected(lambda: nms_consistency(z, hb, rowmax, conf, True, 'decode'))
    rb = rowmax.clone()
    j = int(torch.nonzero(rb[0])[0])
    rb[0, j] = torch.nextafter(rb[0, j], torch.tensor(2.0, device='cuda'))
    assert _rejected(lambda: nms_consistency(z, h, rb, conf, True, 'decode'))


if __name__ == '__main__':
    _child_main(sys.argv[1:])
