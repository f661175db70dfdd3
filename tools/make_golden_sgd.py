"""tests/golden/sgd_groups.npz: the REFERENCE's build_optimizer (src/optimizers/__init__.py) on the reference's YOLOX-s (SURVEY §3.5
composite: CSPDarknet yolox_s + YOLOXNeck + YOLOXHead) and YOLOv5-s (tools/ref_shim.build_yolov5s) models, with each YAML's OPTIMIZER
section (conf/det/yolox/coco_yolox_s.yml, conf/det/yolov5/coco_yolov5_s.yml).

  CVPYTORCH_REFERENCE=<reference checkout> python tools/make_golden_sgd.py

Stored per model m: `m:names` (the parameter name of each group's one tensor, in group order), `m:lr`, `m:weight_decay`, `m:momentum`
(float64) and `m:nesterov` (bool).  Before writing, oracle/optim_oracle.param_groups must give the same groups on the same reference model,
and its CONFIGS must equal what the YAML loader produced."""
import importlib
import os
import sys

import numpy as np
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import ref_shim  # noqa: E402
from oracle import optim_oracle as O  # noqa: E402

YAMLS = {'yolox_s': 'conf/det/yolox/coco_yolox_s.yml', 'yolov5_s': 'conf/det/yolov5/coco_yolov5_s.yml'}


def _models():
    ref_shim.install()
    from src.models.backbones import build_backbone
    bb = build_backbone({'name': 'CSPDarknet', 'subtype': 'yolox_s', 'out_stages': [2, 3, 4]})
    nk = importlib.import_module('src.models.necks.yolox_neck').YOLOXNeck('yolox_s', [256, 512, 1024], depth_mul=.33, width_mul=.5)
    hd = importlib.import_module('src.models.heads.yolox_head').YOLOXHead(num_classes=80, subtype='yolox_s', in_channels=[256, 512, 1024],
                                                                          depth_mul=.33, width_mul=.5)
    yolox = nn.Module()
    yolox.backbone, yolox.neck, yolox.head = bb, nk, hd
    bb5, nk5, dt5, _ = ref_shim.build_yolov5s()
    yolov5 = nn.Module()
    yolov5.backbone, yolov5.neck, yolov5.detect = bb5, nk5, dt5
    return {'yolox_s': yolox, 'yolov5_s': yolov5}


def _plain(c):
    return {k: _plain(v) for k, v in c.items()} if hasattr(c, 'items') else c


def main():
    models = _models()
    from src.optimizers import build_optimizer
    from src.utils.config import CommonConfiguration
    out = {}
    for name, model in models.items():
        cfg = CommonConfiguration.from_yaml(os.path.join(ref_shim.REF, YAMLS[name]))
        mine = O.CONFIGS[name]
        assert (cfg.INIT_LR, cfg.BACKBONE_LR, cfg.WARMUP.ITERS, cfg.WARMUP.FACTOR) == (mine['INIT_LR'], mine['BACKBONE_LR'],
                                                                                       mine['WARMUP']['ITERS'], mine['WARMUP']['FACTOR'])
        assert _plain(cfg.OPTIMIZER) == dict(mine['OPTIMIZER'], TYPE='SGD'), _plain(cfg.OPTIMIZER)
        ref = build_optimizer(cfg, model).param_groups
        ora = O.param_groups(model, mine)
        assert len(ref) == len(ora)
        for a, b in zip(ref, ora):
            assert len(a['params']) == 1 and a['params'][0] is b['params'][0]
            assert all(a[k] == b[k] for k in ('lr', 'weight_decay', 'momentum', 'nesterov'))
        assert len({id(g['params'][0]) for g in ref}) == len(ref) == len(list(model.parameters()))
        out[f'{name}:names'] = np.array(O.group_names(model, ref))
        for k in ('lr', 'weight_decay', 'momentum'):
            out[f'{name}:{k}'] = np.array([g[k] for g in ref], dtype=np.float64)
        out[f'{name}:nesterov'] = np.array([g['nesterov'] for g in ref], dtype=bool)
        print(name, len(ref), 'groups')
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'sgd_groups.npz'), **out)


if __name__ == '__main__':
    main()
