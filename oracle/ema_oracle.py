"""Torch restatement of the reference's model EMA (src/utils/ema.py ModelEMA.__init__ / update), written from the algorithm: eager ATen ops in
the reference's order, so on a given device it gives the reference's bits.

  decay_at(updates, decay=0.9999) -> the decay of update number `updates` (Python double, as the reference's lambda)
  update_(ema_sd, src_sd, d)       -> one step in place over the floating entries of ema_sd: e *= d; e += (1 - d) * src
  ModelEMA(model, decay, updates)  -> .ema / .updates / .decay / .update(model), the reference's surface on top of the two
  fixture_model()                  -> the small conv / BN model of tests/golden/ema.npz (tools/make_golden_ema.py)
  SCENARIOS                        -> (name, updates at construction, number of updates) of that fixture
"""
import math
from copy import deepcopy

import torch
import torch.nn as nn

# a fresh EMA (decay ~ 5e-4 at the first update), one resumed mid-ramp and one resumed where the decay has reached 0.9999
SCENARIOS = (('fresh', 0, 6), ('mid', 1500, 3), ('late', 200000, 4))


def decay_at(updates, decay=0.9999):
    return decay * (1 - math.exp(-updates / 2000))


def update_(ema_sd, src_sd, d):
    for k, e in ema_sd.items():
        if e.dtype.is_floating_point:
            e *= d
            e += (1 - d) * src_sd[k].detach()


def _bare(model):
    return model.module if type(model) in (nn.parallel.DataParallel, nn.parallel.DistributedDataParallel) else model


class ModelEMA:
    def __init__(self, model, decay=0.9999, updates=0):
        self.ema = deepcopy(_bare(model)).eval()
        self.updates = updates
        self.decay = lambda x: decay_at(x, decay)
        for p in self.ema.parameters():
            p.requires_grad_(False)

    def update(self, model):
        with torch.no_grad():
            self.updates += 1
            update_(self.ema.state_dict(), _bare(model).state_dict(), self.decay(self.updates))


def fixture_model():
    """conv 3x3 (no bias) -> BatchNorm (with num_batches_tracked) -> SiLU -> conv 1x1 (bias)."""
    return nn.Sequential(nn.Conv2d(3, 8, 3, padding=1, bias=False), nn.BatchNorm2d(8), nn.SiLU(), nn.Conv2d(8, 5, 1))
