"""Times the LiDAR depth loss (train.py:124-132) and the object-accumulation loss (train.py:114-122) at 1920x1280: the reference's
torch lines (tests/train_loss_oracle.py, on the GPU) against the fused losses.lidar_depth_loss / losses.obj_acc_loss, at 5 % and
100 % LiDAR density.  CUDA events, median of 50 calls after 5 warm-up calls; `fwd` is the value alone (inputs without gradient),
`fwd_bwd` the value and backward into depth / acc.  Prints one JSON line with the GPU name and its enforced power limit.
python tools/loss_bench.py"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import train_loss_oracle as TO  # noqa: E402
from street_gaussians_b200 import losses  # noqa: E402

H, W = 1280, 1920


def power_limit_w():
    try:
        import pynvml
        pynvml.nvmlInit()
        return pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())) / 1000.0
    except Exception:
        try:
            out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                                  str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
            return float(out.strip().splitlines()[0])
        except Exception:
            return None


def time_ms(fn, iters=50, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def inputs(density, seed=0):
    g = torch.Generator().manual_seed(seed)
    acc = torch.rand(1, H, W, generator=g)
    z = 2.0 + 78.0 * torch.rand(1, H, W, generator=g)
    depth = acc * z * (1.0 + 0.01 * torch.randn(1, H, W, generator=g))
    lidar = torch.where(torch.rand(1, H, W, generator=g) < density, z + 0.5 * torch.randn(1, H, W, generator=g), torch.zeros_like(z))
    mask = torch.rand(1, H, W, generator=g) > 0.1
    return depth.cuda(), acc.cuda(), lidar.clamp_min(0.0).cuda(), mask.cuda()


def bench_pair(make_call, leaves):
    """make_call(tensors) -> loss; times the value alone and value + backward."""
    rec = {}
    plain = [t.detach() for t in leaves]
    rec["fwd_ms"] = time_ms(lambda: make_call(plain))
    grad = [t.detach().clone().requires_grad_(True) for t in leaves]

    def fwd_bwd():
        for t in grad:
            t.grad = None
        make_call(grad).backward()

    rec["fwd_bwd_ms"] = time_ms(fwd_bwd)
    rec["value"] = float(make_call(plain))
    return rec


def main():
    assert torch.cuda.is_available(), "tools/loss_bench.py needs a CUDA device"
    dev = torch.cuda.current_device()
    out = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), H=H, W=W, lidar={}, obj={})
    for density in (0.05, 1.0):
        depth, acc, lidar, mask = inputs(density)
        rec = {}
        for label, fn in (("reference", TO.lidar_depth_loss), ("fused", losses.lidar_depth_loss)):
            rec[label] = bench_pair(lambda t, fn=fn: fn(t[0], t[1], lidar, mask, 0.1), [depth, acc])
        rec["speedup_fwd_bwd"] = rec["reference"]["fwd_bwd_ms"] / rec["fused"]["fwd_bwd_ms"]
        out["lidar"][f"density_{density:g}"] = rec
    g = torch.Generator().manual_seed(1)
    acc_obj = torch.rand(1, H, W, generator=g).cuda()
    bound = (torch.rand(1, H, W, generator=g) > 0.5).cuda()
    for label, fn in (("reference", TO.obj_acc_loss), ("fused", losses.obj_acc_loss)):
        out["obj"][label] = bench_pair(lambda t, fn=fn: fn(t[0], bound, 0.1), [acc_obj])
    out["obj"]["speedup_fwd_bwd"] = out["obj"]["reference"]["fwd_bwd_ms"] / out["obj"]["fused"]["fwd_bwd_ms"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
