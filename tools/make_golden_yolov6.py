"""Generates the YOLOv6 fixtures under tests/golden/ by running the REFERENCE ($CVPYTORCH_REFERENCE) on CPU, composed by hand:
YOLOv6EfficientRep -> YOLOv6RepBiPAN -> YOLOv6Effidehead -> YOLOv6Detect -> non_max_suppression (src/models/yolov6.py), with the
subtype / widths the USE_MODEL sections of conf/det/yolov6/coco_yolov6_{n,s}.yml give (the s YAML route itself fails in build_detect).
Weights and BN statistics: oracle.yolov6_oracle.seeded_state_dict(keys, seed), so that the tests regenerate them from the seed.

  yolov6_keys.npz    state_dict keys / shapes of the model (backbone. / neck. / head. / loss.0.proj, as YOLODetector) for n and s
  yolov6_fwd128.npz  per-module outputs at 2x3x128x128 for n and s (input: oracle.yolov6_oracle.fixture_input(FWD_SEED, FWD_SHAPE)):
                     backbone (4 stages), neck (3), head (stems, cls scores, reg) and z, each as max|t| and oracle.yolov6_oracle.subsample(t);
                     reg and the box / objectness columns of z in full
  yolov6_post320.npz s at 1x3x320x320 (fixture_input(POST_SEED, POST_SHAPE)): z as its boxes and the class scores above conf 0.03
                     (oracle.yolov6_oracle.sparse_candidates, all the NMS reads) and the NMS rows (conf 0.03, iou 0.65, multi-label,
                     max_det 300)
  yolov6_nms.npz     the reference NMS on seeded objectness-1 predictions (oracle.nms_oracle.make_stress_prediction, column 4 = 1.0)
Only samples of the large tensors are stored; the tests compare the device's full tensors with the oracle, which the samples pin.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import ref_shim  # noqa: E402
from oracle import nms_oracle as NO  # noqa: E402
from oracle import yolov6_oracle as V6  # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
torch.set_num_threads(8)
SEEDS = {'n': 606, 's': 616}
NECK = dict(in_channels=[128, 256, 512, 1024], mid_channels=[128, 128, 256], out_channels=[128, 256, 512], num_blocks=[12, 12, 12, 12])
NMS_CASES = [('few', 0.03), ('typical', 0.03), ('typical', 0.25), ('capped', 0.03)]


def build_reference(stype):
    ref_shim.install()
    from src.losses.det.yolov6_loss import YOLOv6Loss
    from src.models.backbones import build_backbone
    from src.models.detects.yolov6_detect import YOLOv6Detect
    from src.models.heads import build_head
    from src.models.necks import build_neck
    sub = f'yolov6_{stype}'
    m = torch.nn.Module()  # SingleStageDetector's attribute order: backbone, neck, head, detect, loss
    m.backbone = build_backbone({'name': 'YOLOv6EfficientRep', 'subtype': sub, 'out_stages': [1, 2, 3, 4], 'output_stride': 32, 'pretrained': False})
    m.neck = build_neck(dict(NECK, name='YOLOv6RepBiPAN', subtype=sub))
    m.head = build_head({'name': 'YOLOv6Effidehead', 'subtype': sub, 'num_classes': 80, 'in_channels': [128, 256, 512], 'use_dfl': False,
                         'fuse_ab': False})
    m.detect = YOLOv6Detect(subtype=sub, in_channels=[128, 256, 512])
    loss_kw = dict(num_classes=80, use_dfl=False, reg_max=0, iou_type='siou') if stype == 'n' else dict(num_classes=80)  # the two LOSS sections
    m.loss = torch.nn.ModuleList([YOLOv6Loss(**loss_kw)])
    return m.eval()


def ref_forward(m, x):
    with torch.no_grad():
        b = m.backbone(x)
        n = m.neck(b)
        feats, cls, reg = m.head(list(n))
        z = m.detect((feats, cls, reg))
    return b, n, feats, cls, reg, z


def main():
    keys, fwd = {}, {}
    for stype in ('n', 's'):
        m = build_reference(stype)
        sd = m.state_dict()
        keys[f'{stype}_keys'] = np.array(list(sd.keys()))
        keys[f'{stype}_shapes'] = np.array([','.join(str(s) for s in v.shape) for v in sd.values()])
        keys[f'{stype}_params'] = np.array(sum(p.numel() for p in m.parameters()))
        m.load_state_dict(V6.seeded_state_dict([(k, v.shape) for k, v in sd.items()], SEEDS[stype]), strict=True)
        x = V6.fixture_input(V6.FWD_SEED, V6.FWD_SHAPE)
        b, n, feats, cls, reg, z = ref_forward(m, x)
        named = [(f'backbone_{i}', t) for i, t in enumerate(b)] + [(f'neck_{i}', t) for i, t in enumerate(n)] + \
            [(f'stems_{i}', t) for i, t in enumerate(feats)] + [('cls', cls), ('reg', reg), ('z', z)]
        for name, t in named:
            fwd[f'{stype}_{name}_max'] = np.array(float(t.abs().max()), np.float32)
            fwd[f'{stype}_{name}_sample'] = V6.subsample(t).numpy()
        fwd[f'{stype}_reg'], fwd[f'{stype}_z_box'] = reg.numpy(), z[..., :5].numpy()
        zo, _ = V6.forward(x, m.state_dict())
        assert V6.rel_err(zo, z) < 1e-5, 'oracle network differs from the reference'
        print(stype, 'params', int(keys[f'{stype}_params']), 'keys', len(sd), 'z', tuple(z.shape), 'neck max', [float(t.abs().max()) for t in n])
        if stype == 's':
            from src.models.yolov6 import non_max_suppression
            x3 = V6.fixture_input(V6.POST_SEED, V6.POST_SHAPE)
            z3 = ref_forward(m, x3)[-1]
            preds = non_max_suppression(z3.clone(), 0.03, 0.65, multi_label=True)
            boxes, rows, classes, scores = V6.sparse_candidates(z3.numpy(), 0.03)
            post = dict(boxes=boxes, rows=rows, classes=classes, scores=scores, z_max=np.array(float(z3.abs().max()), np.float32),
                        det=preds[0].numpy())
            assert np.array_equal(V6.non_max_suppression(z3.numpy(), 0.03, 0.65)[0][0], post['det']), 'oracle NMS differs from the reference'
            zs = V6.dense_from_candidates(boxes, rows, classes, scores, 80)
            assert np.array_equal(V6.non_max_suppression(zs, 0.03, 0.65)[0][0], post['det']), 'candidate rows lose NMS information'
            print('s 320: z', tuple(z3.shape), 'kept', preds[0].shape[0])
            np.savez_compressed(os.path.join(GOLD, 'yolov6_post320.npz'), **post)
            nms = {}
            for k, (regime, conf) in enumerate(NMS_CASES):
                p = NO.make_stress_prediction(2, A=4200, nc=20, regime=regime, seed=40 + k)
                p[:, :, 4] = 1.0
                for b_, (d, (do, _)) in enumerate(zip(non_max_suppression(torch.from_numpy(p), conf, 0.65, multi_label=True),
                                                      V6.non_max_suppression(p, conf, 0.65))):
                    assert np.array_equal(do, d.numpy()), ('oracle NMS differs from the reference', regime, conf)
                    nms[f'case{k}_det{b_}'] = d.numpy()
                print('nms', regime, conf, [int(d.shape[0]) for d in non_max_suppression(torch.from_numpy(p), conf, 0.65, multi_label=True)])
            np.savez_compressed(os.path.join(GOLD, 'yolov6_nms.npz'), **nms)
    np.savez_compressed(os.path.join(GOLD, 'yolov6_keys.npz'), **keys)
    np.savez_compressed(os.path.join(GOLD, 'yolov6_fwd128.npz'), **fwd)
    for f in ('yolov6_keys', 'yolov6_fwd128', 'yolov6_post320', 'yolov6_nms'):
        print(f, os.path.getsize(os.path.join(GOLD, f + '.npz')))


if __name__ == '__main__':
    main()
