"""CPU suite, part 2: host-side logic (state_dict surface, BN folding, weight packing, stem re-formulation, factories,
C-ABI export list, loud failure without CUDA) and the world_size-2 gloo test of the detection all-gather."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden')


def test_state_dict_keys_equal_reference():
    from cvpytorch_b200 import synth
    g = np.load(os.path.join(GOLD, 'yolov5s_keys.npz'))
    t = synth.template_state_dict()
    assert list(t.keys()) == list(g['keys'])
    assert [str(tuple(v.shape)) for v in t.values()] == list(g['shapes'])
    assert sum(v.numel() for k, v in t.items() if not k.endswith('num_batches_tracked') and not k.endswith('running_mean')
               and not k.endswith('running_var') and not k.endswith('anchors')) == 7235389  # SURVEY.md §3.5


def test_fold_conv_bn_matches_batchnorm():
    """Algebra of src/utils/fuse.py:33-54 (the reference's only numeric self-check, :67-80, prints this error)."""
    from cvpytorch_b200 import ops
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 8, 9, 9, generator=g)
    w = torch.randn(16, 8, 3, 3, generator=g)
    gamma, beta = torch.rand(16, generator=g) + 0.5, torch.randn(16, generator=g)
    mean, var = torch.randn(16, generator=g), torch.rand(16, generator=g) + 0.1
    ref = F.batch_norm(F.conv2d(x, w, None, 1, 1), mean, var, gamma, beta, False, 0.0, 1e-3)
    w64, b64 = ops.fold_conv_bn(w, None, (gamma, beta, mean, var, 1e-3))
    got = F.conv2d(x.double(), w64, b64, 1, 1)
    assert float((got - ref.double()).abs().max() / ref.abs().max()) < 2e-6  # fp32 rounding of the reference itself


def test_pack_weights_layout_and_split_precision():
    from cvpytorch_b200 import ops
    g = torch.Generator().manual_seed(1)
    w = torch.randn(10, 16, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(10, generator=g, dtype=torch.float64)
    packed, bias = ops.pack_conv_weights(w, b, device='cpu')
    assert packed.shape == (2, 16, 3 * 3 * 16) and packed.dtype == torch.float16 and bias.shape == (16,)
    rec = (packed[0].double() + packed[1].double()).reshape(16, 3, 3, 16)[:10].permute(0, 3, 1, 2)
    assert float((rec - w).abs().max() / w.abs().max()) < 2 ** -20  # hi+lo carries ~22 mantissa bits
    assert float(packed[:, 10:].abs().max()) == 0.0 and torch.equal(bias[:10], b.float())


def test_stem_space_to_depth_equivalence():
    """6x6/s2/p2 conv == 3x3/s1/p1 conv over the 2x2 space-to-depth input (channel = (dy*2+dx)*3+c)."""
    from cvpytorch_b200 import ops
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1, 3, 16, 20, generator=g, dtype=torch.float64)
    w = torch.randn(4, 3, 6, 6, generator=g, dtype=torch.float64)
    ref = F.conv2d(x, w, None, 2, 2)
    s2d = torch.zeros(1, 16, 8, 10, dtype=torch.float64)
    for dy in range(2):
        for dx in range(2):
            for c in range(3):
                s2d[:, (dy * 2 + dx) * 3 + c] = x[:, c, dy::2, dx::2]
    got = F.conv2d(s2d, ops.stem_weights_to_s2d(w), None, 1, 1)
    assert float((got - ref).abs().max()) < 1e-12


def test_factories_follow_reference_contract():
    """The build_* factories of all four model families: an unknown name raises NotImplementedError, and the cfg is deep-copied,
    not consumed (not even the 'depth_mul' / 'width_mul' keys YOLOv5's build_backbone drops)."""
    from copy import deepcopy

    from cvpytorch_b200 import fcos_models as FM
    from cvpytorch_b200 import models as M
    from cvpytorch_b200 import seg_models as SM
    from cvpytorch_b200 import synth
    from cvpytorch_b200 import yolox_models as XM
    for build in (M.build_backbone, M.build_neck, M.build_detect, XM.build_backbone, XM.build_neck, XM.build_head, FM.build_backbone,
                  FM.build_neck, FM.build_head, FM.build_detect, SM.build_backbone, SM.build_head):
        with pytest.raises(NotImplementedError):
            build({'name': 'NoSuchModule'})
    cfg = {'name': 'YOLOv5Detect', 'in_channels': [256, 512, 1024], 'width_mul': 0.5, 'anchors': M.YOLOv5.anchors, 'num_classes': 80}
    d = M.build_detect(cfg)
    assert 'name' in cfg and d.m[0].weight.shape == (255, 128, 1, 1)
    bias = d.m[0].bias.view(3, 85)
    assert abs(float(bias[0, 4]) - np.log(8 / (640 / 8) ** 2)) < 1.0  # prior added on top of the default init
    for build, cfg in ((M.build_backbone, {**synth.YOLOV5S_CFG['BACKBONE'], 'depth_mul': 0.33, 'width_mul': 0.5}),
                       (M.build_detect, cfg),
                       (XM.build_neck, {**synth.YOLOX_CFG['NECK'], 'depth_mul': 0.33, 'width_mul': 0.5}),
                       (FM.build_detect, synth.FCOS_CFG['DETECT']),
                       (SM.build_head, synth.DEEPLAB_CFG['HEAD'])):
        before = deepcopy(cfg)
        build(cfg)
        assert cfg == before, cfg['name']


def test_standalone_dropins_reject_cpu_input_and_training_without_caching():
    """Every drop-in that runs on its own -- the 3 backbones, the 7 components, the bricks, the yolo_blocks blocks and the 5 models'
    'val' forward, on a tensor and on a list of images -- raises CvbError on CPU tensors and RuntimeError in training mode (that check
    first), and caches no graph.  The models' other modes: 'infer' returns None (the detectors) or runs the graph (EncoderDecoder), 'train'
    in eval mode names .train() (the YOLO trainers; YOLOv6 refuses CPU images first) or is refused (FCOS, EncoderDecoder), and an unknown
    mode raises RuntimeError."""
    from test_yolov6_host import use_model

    from cvpytorch_b200 import _lib, synth
    from cvpytorch_b200 import fcos_models as FM
    from cvpytorch_b200 import models as M
    from cvpytorch_b200 import seg_models as SM
    from cvpytorch_b200 import yolo_blocks as YB
    from cvpytorch_b200 import yolov6_models as Y6
    from cvpytorch_b200 import yolox_models as XM
    from cvpytorch_b200.modules import Conv, ConvModule
    cls80 = [{f'c{i}': 1.0} for i in range(80)]
    v5, yx, v6 = M.YOLOv5(cls80, dict(synth.YOLOV5S_CFG)), XM.YOLOX(cls80, dict(synth.YOLOX_CFG)), Y6.YOLOv6(cls80, use_model('n'))
    fc, dl = FM.FCOS(cls80, dict(synth.FCOS_CFG)), SM.EncoderDecoder([{f'c{i}': 1.0} for i in range(19)], dict(synth.DEEPLAB_CFG))
    models = (v5, yx, v6, fc, dl)
    img = torch.zeros(1, 3, 64, 64)
    maps = lambda *cs: [torch.zeros(1, c, 8 >> i, 8 >> i) for i, c in enumerate(cs)]  # noqa: E731
    x = torch.zeros(1, 32, 8, 8)
    inputs = [(v5.backbone, img), (yx.backbone, img), (fc.backbone, img),
              (v5.neck, maps(128, 256, 512)), (v5.detect, maps(128, 256, 512)), (yx.neck, maps(128, 256, 512)), (yx.head, maps(128, 256, 512)),
              (fc.neck, maps(512, 1024, 2048)), (fc.head, maps(256, 256, 256, 256)), (dl.head, maps(256, 2048)),
              (ConvModule(24, 32, 3, padding=1, norm_cfg=dict(type='BN')), torch.zeros(1, 24, 8, 8)), (Conv(24, 32, 3), torch.zeros(1, 24, 8, 8)),
              (YB.RepVGGBlock(32, 32), x), (YB.BottleRep(32, 32), x), (YB.RepBlock(32, 32, n=2), x), (YB.Conv_C3(32, 32), x),
              (YB.BepC3(32, 32, n=2), x), (YB.EELAN(32, 16, 32), x)]
    calls = ([(m, lambda m=m, t=t: m(t)) for m, t in inputs] + [(m, lambda m=m: m(img, None, 'val')) for m in models]
             + [(m, lambda m=m: m([img[0], img[0]], None, 'val')) for m in models])
    for m, call in calls:
        m.eval()
        with pytest.raises(_lib.CvbError):
            call()
        assert m._graphs == {}, type(m).__name__
        m.train()
        with pytest.raises(RuntimeError) as e:
            call()
        assert not isinstance(e.value, _lib.CvbError), type(m).__name__
        assert m._graphs == {}, type(m).__name__
    for m in models:
        m.eval()
        with pytest.raises(RuntimeError, match='unknown mode'):
            m(img, None, 'bogus')
    assert all(m(img, None, 'infer') is None for m in (v5, yx, v6, fc))
    with pytest.raises(_lib.CvbError):
        dl(img, None, 'infer')  # the label map of the cached graph
    for m in (v5, yx):
        with pytest.raises(RuntimeError, match=r'\.train\(\)'):
            m(img, None, 'train')
    with pytest.raises(NotImplementedError, match='no CPU fallback'):
        v6(img, None, 'train')
    for m in (fc, dl):
        for mode in (True, False):
            with pytest.raises(RuntimeError, match='training stays on the reference'):
                m.train(mode)(img, None, 'train')
    assert all(m._graphs == {} for m in models)


def test_models_name_a_missing_config_section():
    """A dict or attribute model_cfg without a required section fails at construction with a KeyError that names the section."""
    from types import SimpleNamespace

    from test_yolov6_host import use_model

    from cvpytorch_b200 import fcos_models as FM, models as M, seg_models as SM, synth, yolov6_models as Y6, yolox_models as XM
    cls80 = [{f'c{i}': 1.0} for i in range(80)]
    for cls, cfg, key in ((M.YOLOv5, synth.YOLOV5S_CFG, 'NECK'), (XM.YOLOX, synth.YOLOX_CFG, 'HEAD'), (Y6.YOLOv6, use_model('n'), 'DETECT'),
                          (FM.FCOS, synth.FCOS_CFG, 'BACKBONE'), (SM.EncoderDecoder, synth.DEEPLAB_CFG, 'HEAD')):
        rest = {k: v for k, v in cfg.items() if k != key}
        for model_cfg in (rest, SimpleNamespace(**rest)):
            with pytest.raises(KeyError, match=key):
                cls(cls80, model_cfg)


def test_model_surface_and_loud_failure_without_cuda():
    from cvpytorch_b200 import _lib, synth
    m = synth.build_yolov5s(calibrated=True)
    assert tuple(m.dummy_input.shape) == (1, 3, 640, 640) and m.conf_thres == 0.001 and m.iou_thres == 0.6
    assert m(torch.zeros(1, 3, 64, 64), None, 'infer') is None  # reference returns None in 'infer' mode
    with pytest.raises(_lib.CvbError):
        m(torch.zeros(1, 3, 64, 64), None, 'val')  # CPU tensor: no fallback
    m.train()
    with pytest.raises(RuntimeError):
        m.backbone(torch.zeros(1, 3, 64, 64))
    with pytest.raises(RuntimeError):
        m.backbone.stage1[1](torch.zeros(1, 64, 8, 8))  # fused-path block is not executable stand-alone


def test_c_abi_library_exports_every_declared_symbol():
    from cvpytorch_b200 import _lib
    header = open(os.path.join(ROOT, 'include', 'cvb200.h')).read()
    declared = set(re.findall(r'\b(cvb_[a-z0-9_]+)\s*\(', header))
    assert declared == set(_lib.SYMBOLS.keys()), declared ^ set(_lib.SYMBOLS.keys())
    assert os.path.exists(_lib.LIB_PATH), 'libcvb200.so not built (python -c "import __graft_entry__ as g; g.build()")'
    h = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(h, name), name
    assert _lib.lib().cvb_version() == 100
    assert _lib.lib().cvb_nms_workspace_bytes(2, 25200, 80) > 2 * 65536 * 8


def test_shard_range_covers_batch():
    from cvpytorch_b200.dist import shard_range
    for gb, w in ((64, 8), (64, 3), (5, 8)):
        spans = [shard_range(gb, r, w) for r in range(w)]
        assert spans[0][0] == 0 and spans[-1][1] == gb and all(a[1] == b[0] for a, b in zip(spans, spans[1:]))


def _free_port():
    import socket
    with socket.socket() as sk:
        sk.bind(('127.0.0.1', 0))
        return sk.getsockname()[1]


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist
    from cvpytorch_b200.dist import all_gather_detections
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    B, M = 3, 7
    det = torch.full((B, M, 6), float(rank)) + torch.arange(B).view(B, 1, 1)
    idx = (torch.arange(B * M, dtype=torch.int32).view(B, M) + 1000 * rank)
    cnt = torch.tensor([rank + 1, 0, M], dtype=torch.int32)
    d, i, c = all_gather_detections(det, idx, cnt)
    q.put((rank, d.clone(), i.clone(), c.clone()))
    dist.barrier()
    dist.destroy_process_group()


def test_all_gather_detections_gloo_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(2)]
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    for rank, d, i, c in res:
        assert d.shape == (6, 7, 6) and i.shape == (6, 7) and c.tolist() == [1, 0, 7, 2, 0, 7]
        assert float(d[0, 0, 0]) == 0.0 and float(d[3, 0, 0]) == 1.0 and float(d[5, 0, 0]) == 3.0
        assert int(i[3, 0]) == 1000 and int(i[0, 6]) == 6


def _gloo_worker_packed(rank, world, port, q):
    """the wire format the NMS kernels write (ops.NmsWorkspace.packed: [det B*M*6 | idx B*M | count B], views of ONE flat buffer)"""
    import torch.distributed as dist
    from cvpytorch_b200.dist import all_gather_packed, packed_len, unpack_gathered
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    B, M = 3, 7
    packed = torch.zeros(packed_len(B, M))
    det = packed[:B * M * 6].view(B, M, 6)
    idx = packed[B * M * 6:B * M * 7].view(torch.int32).view(B, M)
    cnt = packed[B * M * 7:].view(torch.int32)
    det.copy_(torch.full((B, M, 6), float(rank)) + torch.arange(B).view(B, 1, 1))
    idx.copy_(torch.arange(B * M, dtype=torch.int32).view(B, M) + 1000 * rank)
    cnt.copy_(torch.tensor([rank + 1, 0, M], dtype=torch.int32))
    out = torch.empty((world, packed.numel()))
    all_gather_packed(packed, out)
    d, i, c = unpack_gathered(out, B, M)
    q.put((rank, d.clone(), i.clone(), c.clone()))
    dist.barrier()
    dist.destroy_process_group()


def test_all_gather_packed_gloo_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker_packed, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(2)]
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    for rank, d, i, c in res:
        assert d.shape == (6, 7, 6) and i.shape == (6, 7) and c.tolist() == [1, 0, 7, 2, 0, 7]
        assert float(d[0, 0, 0]) == 0.0 and float(d[3, 0, 0]) == 1.0 and float(d[5, 0, 0]) == 3.0
        assert int(i[3, 0]) == 1000 and int(i[0, 6]) == 6


def _gloo_worker_fcos_seg(rank, world, port, q):
    import torch.distributed as dist
    from cvpytorch_b200.dist import all_gather_fcos_detections, all_gather_label_maps
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    B, K = 2, 5
    scores = torch.arange(B * K, dtype=torch.float32).view(B, K) + 100 * rank
    classes = torch.arange(B * K, dtype=torch.int64).view(B, K) % 80 + 1
    boxes = torch.arange(B * K * 4, dtype=torch.float32).view(B, K, 4) + 0.5 * rank
    counts = torch.tensor([K, rank], dtype=torch.int32)
    s, c, bx, n = all_gather_fcos_detections(scores, classes, boxes, counts)
    lab = (torch.arange(B * 4 * 6).view(B, 4, 6) % 19 + rank).to(torch.int64)
    g = all_gather_label_maps(lab)
    q.put((rank, s.clone(), c.clone(), bx.clone(), n.clone(), g.clone()))
    dist.barrier()
    dist.destroy_process_group()


def test_all_gather_fcos_and_label_maps_gloo_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker_fcos_seg, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(2)]
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    for rank, s, c, bx, n, g in res:
        assert s.shape == (4, 5) and c.dtype == torch.int32 and bx.shape == (4, 5, 4) and n.tolist() == [5, 0, 5, 1]
        assert float(s[0, 0]) == 0.0 and float(s[2, 0]) == 100.0 and float(bx[2, 0, 0]) == 0.5 and int(c[3, 4]) == 10
        assert g.dtype == torch.int64 and g.shape == (4, 4, 6) and int(g[0, 0, 1]) == 1 and int(g[2, 0, 1]) == 2


def test_yolox_factories_and_contract_on_cpu():
    from cvpytorch_b200 import _lib, synth
    from cvpytorch_b200 import yolox_models as XM
    with pytest.raises(NotImplementedError):
        XM.build_backbone({'name': 'NoSuchBackbone'})
    with pytest.raises(NotImplementedError):
        XM.build_head({'name': 'NoSuchHead'})
    # the reference YAML's (unbuildable) backbone name is accepted and mapped onto the composite that runs
    cfg = dict(synth.YOLOX_CFG)
    cfg['BACKBONE'] = {'name': 'CspDarkNet', 'out_stages': [2, 3, 4], 'output_stride': 32, 'pretrained': False}
    m = XM.YOLOX(dictionary=[{f'c{i}': 1.0} for i in range(80)], model_cfg=cfg)
    assert list(m.state_dict().keys()) == list(synth.yolox_template_state_dict().keys())
    m.load_state_dict(synth.yolox_state_dict(calibrated=True), strict=True)
    m.eval()
    assert m.dummy_input.shape == (1, 3, 640, 640) and m.conf_thr == 0.01 and m.nms_thr == 0.65
    assert m(torch.zeros(1, 3, 64, 64), None, 'infer') is None
    with pytest.raises(_lib.CvbError):
        m(torch.zeros(1, 3, 64, 64), None, 'val')  # CPU tensor: no fallback
    with pytest.raises(RuntimeError):
        m(torch.zeros(1, 3, 64, 64), None, 'train')
    # Focus weight re-ordering: reference patch order (tl, bl, tr, br) -> loader order (tl, tr, bl, br), 4 zero pad channels
    w = torch.arange(2 * 12 * 9, dtype=torch.float64).view(2, 12, 3, 3)
    w16 = XM.focus_weights_to_s2d(w)
    assert torch.equal(w16[:, 0:3], w[:, 0:3]) and torch.equal(w16[:, 3:6], w[:, 6:9]) and torch.equal(w16[:, 6:9], w[:, 3:6])
    assert torch.equal(w16[:, 9:12], w[:, 9:12]) and float(w16[:, 12:].abs().max()) == 0.0


def test_focus_and_window_formulation_equivalence():
    """YOLOX Focus (yolo_modules.py:29-37: cat(tl, bl, tr, br) -> 3x3 conv) == 3x3 conv over the loader's space-to-depth tensor with
    focus_weights_to_s2d, and the row-window re-formulation used on the device (ops.window_weights: the three taps of a filter row laid
    side by side over 4 adjacent pixels, one zero-padded) gives the same result."""
    from cvpytorch_b200 import ops
    from cvpytorch_b200.yolox_models import focus_weights_to_s2d
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 3, 12, 16, generator=g, dtype=torch.float64)
    w = torch.randn(5, 12, 3, 3, generator=g, dtype=torch.float64)
    ref = F.conv2d(torch.cat((x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]), 1), w, None, 1, 1)
    s2d = torch.zeros(2, 16, 6, 8, dtype=torch.float64)
    for dy in range(2):
        for dx in range(2):
            for c in range(3):
                s2d[:, (dy * 2 + dx) * 3 + c] = x[:, c, dy::2, dx::2]
    w16 = focus_weights_to_s2d(w)
    assert float((F.conv2d(s2d, w16, None, 1, 1) - ref).abs().max()) < 1e-12
    # row-window form: input padded by one zero column on the left and two on the right (W + 3 columns), window of 4 pixels
    ww = ops.window_weights(w16, 4)                       # [O, 4*16, 3, 1], k = kx*16 + c
    xp = F.pad(s2d, (1, 2, 0, 0))                          # columns -1 .. W+1
    win = torch.stack([xp[..., j:j + 8] for j in range(4)], 1).reshape(2, 64, 6, 8)   # channel = kx*16 + c of pixel (w - 1 + kx)
    got = F.conv2d(win, ww, None, 1, (1, 0))
    assert float((got - ref).abs().max()) < 1e-12


def test_brick_registration_hook():
    """cvpytorch_b200.bricks.register() against a stand-in with the reference registry's interface
    (src/utils/registry.py:293-346: register_module(name=, module=), KeyError on duplicates)."""
    import types

    from cvpytorch_b200 import bricks

    class Registry:
        def __init__(self):
            self.module_dict = {}

        def register_module(self, name=None, force=False, module=None):
            if name in self.module_dict and not force:
                raise KeyError(f'{name} is already registered')
            self.module_dict[name] = module

        def get(self, k):
            return self.module_dict.get(k)

    reg = types.SimpleNamespace(CONV_LAYERS=Registry(), PLUGIN_LAYERS=Registry())
    bricks.register(reg)
    bricks.register(reg)  # idempotent
    assert reg.CONV_LAYERS.get('B200Conv2d') is bricks.B200Conv2d and reg.PLUGIN_LAYERS.get('B200ConvModule') is bricks.B200ConvModule
    m = reg.PLUGIN_LAYERS.get('B200ConvModule')(16, 32, 3, padding=1, conv_cfg=dict(type='B200Conv2d'), norm_cfg=dict(type='BN'), act_cfg=dict(type='SiLU'))
    assert set(m.state_dict().keys()) == {'conv.weight', 'bn.weight', 'bn.bias', 'bn.running_mean', 'bn.running_var', 'bn.num_batches_tracked'}
    with pytest.raises(Exception):
        m.eval()(torch.zeros(1, 16, 8, 8))  # CPU tensor: no fallback


def test_training_dropin_mirrors_reference_block_and_fails_loudly_on_cpu():
    """cvpytorch_b200.train.CSPLayer has the reference block's parameter names (tests/golden/c3_train.npz key list, dumped from the reference)
    and no CPU fallback."""
    from cvpytorch_b200 import _lib, train as T
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'c3_train.npz'))
    m = T.CSPLayer(128, 128, n=2)
    assert list(m.state_dict().keys()) == [str(k) for k in g['c3_n2_keys']]
    m.train()
    with pytest.raises(_lib.CvbError):
        m(torch.zeros(1, 128, 8, 8))
    m.eval()
    with pytest.raises(RuntimeError):
        m.conv1(torch.zeros(1, 8, 8, 128, dtype=torch.bfloat16))
    with pytest.raises(NotImplementedError):
        T.BaseConv(48, 64, 1, 1)
    with pytest.raises(NotImplementedError):
        T.BaseConv(64, 64, 1, 2)  # stride 2 only with ksize 3


def test_training_c_abi_rejects_bad_arguments_before_touching_the_device():
    """cvb_train_* entry points validate their arguments on the host (no GPU needed) and report through cvb_last_error_string()."""
    import ctypes
    from cvpytorch_b200 import _lib
    L = _lib.lib()
    one = ctypes.c_void_p(16)  # any non-null, 16-byte aligned value: the checks below fail before it is dereferenced
    assert L.cvb_train_conv(one, 1, 8, 8, 48, one, 64, 1, 1, one, None, None, None) != 0      # cin not a multiple of 64
    assert b'multiples of 64' in L.cvb_last_error_string()
    assert L.cvb_train_conv(one, 1, 8, 8, 64, one, 64, 1, 2, one, None, None, None) != 0      # stride 2 needs k = 3
    assert b'stride' in L.cvb_last_error_string()
    assert L.cvb_train_conv(one, 1, 8, 8, 64, one, 64, 3, 1, one, one, None, None) != 0       # SiLU' epilogue needs both operands
    assert L.cvb_train_conv_wgrad(one, one, 1, 8, 8, 64, 96, 3, 1, one, None) != 0           # cout not a multiple of 64
    assert b'multiples of 64' in L.cvb_last_error_string()
    assert L.cvb_train_conv_dgrad_s2(one, 1, 5, 5, 64, one, 64, 8, 8, one, None, None, None) != 0  # Ho != (H - 1) / 2 + 1
    assert b'geometry' in L.cvb_last_error_string()
    assert L.cvb_train_pack_weights(one, 64, 64, 5, one, one, None) != 0                      # k in {1, 3}


def test_fp64_reference_helpers_and_wgrad_split_geometry():
    """tests/fp64ref.py (the float64 references and element-wise bound of the training-kernel tests) on CPU tensors: the references agree
    with torch.autograd in float64, the bound accepts a bf16-rounded result and names the element it rejects, and the backward-weight
    split that test_train_gpu.py's docstring states for its per > 1 cases."""
    import sys
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import fp64ref as R
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 64, 5, 7, generator=g).to(torch.bfloat16).double().requires_grad_(True)
    w = torch.randn(32, 64, 3, 3, generator=g).to(torch.bfloat16).double().requires_grad_(True)
    yr, ya = R.conv_fwd(x.detach(), w.detach(), 2, 1)
    dy = torch.randn(yr.shape, generator=g).to(torch.bfloat16).double()
    F.conv2d(x, w, None, 2, 1).backward(dy)
    dxr, _ = R.conv_dgrad(dy, w.detach(), x.shape, 2, 1)
    dwr, dwa = R.conv_wgrad(x.detach(), dy, w.shape, 2, 1)
    assert torch.allclose(dxr, x.grad, rtol=1e-12, atol=1e-12) and torch.allclose(dwr, w.grad, rtol=1e-12, atol=1e-12)
    assert bool((ya >= yr.abs()).all()) and bool((dwa >= dwr.abs()).all())
    bound = R.BF16_REL * yr.abs() + R.mma_gamma(9 * 64) * ya
    assert R.check(yr.float().to(torch.bfloat16), yr, bound, 'bf16-rounded') <= 1.0
    bad = yr.clone()
    bad[1, 3, 2, 1] += 1.5 * bound[1, 3, 2, 1]
    with pytest.raises(AssertionError, match=r'at \(1, 3, 2, 1\)'):
        R.check(bad, yr, bound, 'perturbed')
    assert R.choose_box128(16, 48, 48) == (16, 1, 8) and R.wgrad_split(16, 48, 48, 64, 64, 1, 132) == (288, 264, 2)
    assert R.choose_box128(16, 40, 40) == (8, 1, 16) and R.wgrad_split(16, 40, 40, 64, 64, 3, 132) == (200, 29, 7)
    assert R.wgrad_split(2, 10, 10, 64, 192, 3, 132)[1:] == (3, 1)  # cout 192: three 64-wide blocks, no split beyond the 3 tiles
