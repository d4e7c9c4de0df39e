"""CPU: the torch restatement of the object-accumulation and LiDAR depth losses (tests/train_loss_oracle.py) against values and
gradients that the reference's own train.py:114-122 / :124-132 produced (tests/golden/callsite/train_losses.npz,
tests/golden/make_train_loss_golden.py)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_train_loss_golden import case  # noqa: E402  (pure-torch input generator; the reference is read only in its main())
import train_loss_oracle as TO  # noqa: E402
from test_losses_cpu import rel  # noqa: E402

TRAIN_FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "callsite", "train_losses.npz")


def test_fixture_covers_the_reference_blocks():
    z = np.load(TRAIN_FIX)
    assert list(z["lines_lambda_reg"]) == [114, 122] and list(z["lines_lambda_depth_lidar"]) == [125, 132]
    c = case(0)
    n = int(((c["lidar_depth"] > 0) & c["mask"]).sum())
    assert 0.2 * c["mask"].numel() < n < 0.3 * c["mask"].numel()  # ~30 % LiDAR density, thinned by the mask


def test_train_loss_oracle_matches_reference_lines():
    z = np.load(TRAIN_FIX)
    for seed in (0, 1):
        c = case(seed)
        k = f"s{seed}_"
        depth = c["depth"].clone().requires_grad_(True)
        acc = c["acc"].clone().requires_grad_(True)
        v = TO.lidar_depth_loss(depth, acc, c["lidar_depth"], c["mask"])
        v.backward()
        assert abs(float(v.detach()) - float(z[k + "lidar"])) <= 1e-6 * abs(float(z[k + "lidar"]))
        assert rel(depth.grad.numpy(), z[k + "g_depth"]) <= 1e-6 and rel(acc.grad.numpy(), z[k + "g_acc"]) <= 1e-6
        a = c["acc_obj"].clone().requires_grad_(True)
        v = TO.obj_acc_loss(a, c["obj_bound"])
        v.backward()
        assert abs(float(v.detach()) - float(z[k + "obj"])) <= 1e-6 * abs(float(z[k + "obj"]))
        assert rel(a.grad.numpy(), z[k + "g_acc_obj"]) <= 1e-6


def test_lidar_and_obj_entry_points_validate_before_touching_cuda():
    """Argument errors of sgr_lidar_depth_loss / sgr_obj_acc_loss come back as error codes with a message; no CUDA call is made."""
    import ctypes as C

    from street_gaussians_b200 import _capi
    L = _capi.lib()
    err = lambda: L.sgr_last_error().decode()
    N = 1280 * 1920
    nbytes = L.sgr_lidar_depth_loss_scratch_bytes(N)
    assert nbytes >= 4 * N and L.sgr_lidar_depth_loss_scratch_bytes(0) == 0 and L.sgr_lidar_depth_loss_scratch_bytes(1 << 31) == 0
    p = C.c_void_p(256)  # never dereferenced: every call below fails validation
    for keep in (0.0, -0.5, 1.5, float("nan")):
        assert L.sgr_lidar_depth_loss(N, p, p, p, None, keep, 1.0, None, None, p, p, nbytes, None) == -1 and "keep" in err()
    assert L.sgr_lidar_depth_loss(1 << 31, p, p, p, None, 0.95, 1.0, None, None, p, p, nbytes, None) == -1 and "2^31" in err()
    assert L.sgr_lidar_depth_loss(N, None, p, p, None, 0.95, 1.0, None, None, p, p, nbytes, None) == -1 and "NULL" in err()
    assert L.sgr_lidar_depth_loss(N, p, p, p, None, 0.95, 1.0, None, None, p, p, nbytes - 1, None) == -3 and "scratch" in err()
    assert L.sgr_obj_acc_loss(N, p, None, 1.0, None, p, p, None) == -1 and "NULL" in err()
    assert L.sgr_obj_acc_loss(0, p, p, 1.0, None, p, p, None) == -1 and "positive" in err()
