"""Torch restatement of the reference trainer's parameter grouping (src/optimizers/__init__.py build_optimizer), written from the algorithm:
one group per parameter tensor, in named_modules() order.

  param_groups(model, cfg)  -> the list of group dicts build_optimizer hands to torch.optim.SGD ({'params': [p], 'lr', 'momentum',
                               'weight_decay', 'nesterov'}), per module:
                                 * a module with an nn.Parameter `bias`: a group for the bias with BIAS_PARAMS;
                                 * then a normalisation layer (an nn class whose name contains 'Norm'): a group for its weight with BIAS_PARAMS;
                                 * otherwise a module with an nn.Parameter `weight`: a group for the weight with WEIGHT_PARAMS.
                               lr is BACKBONE_LR for modules whose name contains 'backbone' (when BACKBONE_LR is set), INIT_LR otherwise,
                               times BIAS_LR_MULTIPLIER (or 1.0) whenever the module has a `bias` attribute, even None.
  group_names(model, groups) -> the parameter name of each group's tensor
  CONFIGS                   -> the optimiser settings of the two YOLO configs (conf/det/yolox/coco_yolox_s.yml, conf/det/yolov5/coco_yolov5_s.yml)
  warmup_lr(it, cfg)        -> the linear warm-up lr of iteration `it` (src/lr_schedulers/warmup.py), which the trainer writes into every group
"""
import torch.nn as nn

CONFIGS = {
    'yolox_s': {'INIT_LR': 0.01, 'BACKBONE_LR': 0.01, 'WARMUP': {'ITERS': 10000, 'FACTOR': 0.05},
                'OPTIMIZER': {'WEIGHT_PARAMS': {'momentum': 0.9, 'weight_decay': 0.0005, 'nesterov': True},
                              'BIAS_PARAMS': {'momentum': 0.9, 'weight_decay': 0, 'nesterov': True}, 'BIAS_LR_MULTIPLIER': 1}},
    'yolov5_s': {'INIT_LR': 0.01, 'BACKBONE_LR': 0.01, 'WARMUP': {'ITERS': 5500, 'FACTOR': 0.1},
                 'OPTIMIZER': {'WEIGHT_PARAMS': {'momentum': 0.937, 'weight_decay': 0.0005, 'nesterov': True},
                               'BIAS_PARAMS': {'momentum': 0.937, 'weight_decay': 0, 'nesterov': True}, 'BIAS_LR_MULTIPLIER': 1}},
}

_NORMS = tuple(v for k, v in nn.__dict__.items() if 'Norm' in k)


def param_groups(model, cfg):
    opt = cfg['OPTIMIZER']
    groups = []

    def add(module_name, module, p, args):
        lr = cfg['BACKBONE_LR'] if 'backbone' in module_name and cfg['BACKBONE_LR'] is not None else cfg['INIT_LR']
        if hasattr(module, 'bias'):
            lr *= opt['BIAS_LR_MULTIPLIER'] or 1.0
        groups.append({'params': [p], 'lr': lr, **args})

    for k, v in model.named_modules():
        if hasattr(v, 'bias') and isinstance(v.bias, nn.Parameter):
            add(k, v, v.bias, opt['BIAS_PARAMS'])
        if isinstance(v, _NORMS):
            add(k, v, v.weight, opt['BIAS_PARAMS'])
        elif hasattr(v, 'weight') and isinstance(v.weight, nn.Parameter):
            add(k, v, v.weight, opt['WEIGHT_PARAMS'])
    return groups


def group_names(model, groups):
    name = {id(p): n for n, p in model.named_parameters()}
    return [name[id(g['params'][0])] for g in groups]


def warmup_lr(it, cfg):
    alpha = it / cfg['WARMUP']['ITERS']
    return cfg['INIT_LR'] * (cfg['WARMUP']['FACTOR'] * (1.0 - alpha) + alpha)
