"""CPU/GPU torch restatement of the two remaining loss terms of the reference's training step - TEST INFRASTRUCTURE, not product
code.  Restates, citing the reference's train.py:
  train.py:114-122  object-accumulation loss on the objects-only render's acc (clamp, entropy inside obj_bound, -log(1 - a) outside)
  train.py:124-132  LiDAR depth loss: |depth / (acc + 1e-10) - lidar| on (lidar > 0) & mask, mean of the int(0.95 n) smallest
Pinned by tests/golden/callsite/train_losses.npz, which the reference's own train.py lines produced
(tests/golden/make_train_loss_golden.py).  These are the reference's lines, so they keep its host synchronisation
(boolean index, host-side k for torch.topk).
"""
from __future__ import annotations

import torch


def obj_acc_loss(acc_obj, obj_bound, weight=1.0):
    a = torch.clamp(acc_obj, min=1e-6, max=1.0 - 1e-6)
    return weight * torch.where(obj_bound, -(a * torch.log(a) + (1.0 - a) * torch.log(1.0 - a)), -torch.log(1.0 - a)).mean()


def lidar_depth_loss(depth, acc, lidar_depth, mask=None, weight=1.0, keep=0.95):
    depth_mask = lidar_depth > 0.0
    if mask is not None:
        depth_mask = torch.logical_and(depth_mask, mask)
    expected_depth = depth / (acc + 1e-10)
    err = torch.abs(expected_depth[depth_mask] - lidar_depth[depth_mask])
    err, _ = torch.topk(err, int(keep * err.size(0)), largest=False)
    return weight * err.mean()
