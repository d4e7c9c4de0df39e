"""CPU: the torch restatement of the tracked actor poses (tests/actor_pose_oracle.py) against what the reference's own ActorPose and
parse_camera computed (tests/golden/callsite/actor_pose.npz), the float64 tier and its bounds, the reference's quirk on the second
frame's rotation, which outputs the tie rule decides, the host-side track table and the argument checks of the C entries."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import actor_pose_case as AC
import actor_pose_oracle as AO
import refharness as H
import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi
from street_gaussians_b200.actor_pose import track_table

FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "callsite", "actor_pose.npz")
NAMES = [c["name"] for c in AC.CASES]
# At opt_rots = 0 the slerp's two ends are the same quaternion: the stubbed reference's autograd multiplies the zero gradient of the
# small-angle branch by acos'(1) = -inf and returns NaN; the project returns the branch's finite gradient.  Values still compare.
NAN_GRAD_CASES = {"zero"}


def fixture():
    z = np.load(FIX)
    meta = AC.metadata()
    T = AO.Table(z["tracklets"], z["timestamps"], meta["camera_timestamps"], meta["obj_meta"])
    return z, meta, T


def inputs(z, case, dtype=torch.float32, device="cpu"):
    tr = torch.from_numpy(z["tracklets"]).to(device)
    ot = orr = None
    if case["opt_track"]:
        ot = torch.from_numpy(z[f"params_{case['params']}_trans"]).to(device=device, dtype=dtype).requires_grad_(True)
        orr = torch.from_numpy(z[f"params_{case['params']}_rots"]).to(device=device, dtype=dtype).requires_grad_(True)
    ego = torch.from_numpy(AC.ego_pose(case["ego"])).to(device)
    return tr[..., 1:4], tr[..., 4:8], ot, orr, ego


def close(a, b, tol):
    """max |a - b| / max(1, |b|) per element."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float((np.abs(a - b) / np.maximum(1.0, np.abs(b))).max()) <= tol


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-12))


def run_oracle(z, T, case, dtype=torch.float32, tie="first", finite=False):
    in_t, in_r, ot, orr, ego = inputs(z, case, dtype)
    vis = [int(v) for v in z[f"{case['name']}_visible"]]
    p = AO.poses(T, vis, float(case["t"]), case["cam"], case["is_val"], ego, in_t, in_r, ot, orr, dtype=dtype, tie=tie, finite=finite)
    if ot is not None:
        (p * torch.from_numpy(z[f"{case['name']}_w"]).to(dtype)).sum().backward()
    return p, ot, orr


def test_fixture_covers_what_it_claims():
    z, meta, T = fixture()
    counts = {tid: len(T.idx[tid]) for tid in T.idx}
    assert 2 in counts.values() and max(counts.values()) > 32
    cols = {tid: set(T.idx[tid][:, 1].tolist()) for tid in T.idx}
    assert len(cols[0]) > 1 and len(cols[2]) > 1                       # tracks that change column
    steps = np.diff(z["timestamps"])
    assert len(set(steps.tolist())) > 1 and z["timestamps"][0] > 1e9    # non-uniform, large float64 timestamps
    tie = AC.BY_NAME["tie"]
    assert tie["t"] in z["timestamps"]                                 # on a tracklet timestamp, with a tie for the second entry
    k = int(np.where(z["timestamps"] == tie["t"])[0][0])
    assert z["timestamps"][k] - z["timestamps"][k - 1] == z["timestamps"][k + 1] - z["timestamps"][k]
    mid = AC.BY_NAME["midway"]["t"]                                     # midway between two entries: a tie for the nearest
    assert mid - z["timestamps"][k] == z["timestamps"][k + 1] - mid
    # the val case has an actor with fewer than two training timestamps of its camera in its span (actor_pose.py:127)
    m = meta["obj_meta"][1]
    ct = np.asarray(meta["camera_timestamps"][0]["train_timestamps"])
    assert 1 in z["val_visible"] and int(((ct >= m["start_timestamp"]) & (ct <= m["end_timestamp"])).sum()) < 2
    # every branch of matrix_to_quaternion
    branches = set()
    for name in AC.EGO:
        R = torch.from_numpy(AC.ego_pose(name))[:3, :3]
        x = torch.stack([1 + R[0, 0] + R[1, 1] + R[2, 2], 1 + R[0, 0] - R[1, 1] - R[2, 2], 1 - R[0, 0] + R[1, 1] - R[2, 2], 1 - R[0, 0] - R[1, 1] + R[2, 2]])
        branches.add(int(torch.argmax(x)))
    assert branches == {0, 1, 2, 3}


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_fixture(name):
    z, _, T = fixture()
    case = AC.BY_NAME[name]
    p, ot, orr = run_oracle(z, T, case)
    assert close(p.detach().numpy(), z[f"{name}_poses"], 1e-6)
    vis = [int(v) for v in z[f"{name}_visible"]]
    idft = AO.idft_rows(T, vis, case["frame"], int(z["fourier_dim"]), float(z["fourier_scale"]))
    assert close(idft.numpy(), z[f"{name}_idft"], 1e-6)
    if ot is None:
        assert f"{name}_dtrans" not in z
        return
    assert rel(ot.grad.numpy(), z[f"{name}_dtrans"]) < 2e-5
    if name in NAN_GRAD_CASES:
        assert np.isnan(z[f"{name}_drots"]).any()                     # the stubbed reference's NaN, see NAN_GRAD_CASES
        _, _, orr_f = run_oracle(z, T, case, finite=True)
        assert torch.isfinite(orr_f.grad).all()
    else:
        assert rel(orr.grad.numpy(), z[f"{name}_drots"]) < 2e-5


@pytest.mark.parametrize("name", NAMES)
def test_fp32_lines_inside_float64_bounds(name):
    z, _, T = fixture()
    case = AC.BY_NAME[name]
    p, ot, orr = run_oracle(z, T, case, finite=True)
    in_t, in_r, ot0, orr0, ego = inputs(z, case)
    w = torch.from_numpy(z[f"{name}_w"])
    vis = [int(v) for v in z[f"{name}_visible"]]
    r = AO.bounds(T, vis, float(case["t"]), case["cam"], case["is_val"], ego, in_t, in_r, ot0, orr0, w)
    assert bool(((p.detach().double() - r["poses"]).abs() <= r["b_poses"]).all())
    if ot is not None:
        assert bool(((ot.grad.double() - r["dtrans"]).abs() <= r["b_dtrans"]).all())
        assert bool(((orr.grad.double() - r["drots"]).abs() <= r["b_drots"]).all())


def test_second_frame_rotation_is_never_read_with_opt_track():
    """actor_pose.py:145-150: with opt_track the slerp runs between q1 (x) theta1 and q1 (x) theta1 (x) theta2, theta2 taken at
    (frame_ind1, column_ind2); input_rots of the second frame does not enter.  Without opt_track it does."""
    z, _, T = fixture()
    for name in ("train_mid", "no_opt"):
        case = AC.BY_NAME[name]
        in_t, in_r, ot, orr, ego = inputs(z, case)
        vis = [int(v) for v in z[f"{name}_visible"]]
        info = []
        p = AO.poses(T, vis, float(case["t"]), case["cam"], case["is_val"], ego, in_t, in_r, ot, orr, info=info)
        second = [r[2] for r in info if isinstance(r, tuple) and r[0] == "rows"]
        firsts = {r[1] for r in info if isinstance(r, tuple) and r[0] == "rows"}
        bumped = in_r.clone()
        for f, c in second:
            if (f, c) not in firsts:
                bumped[f, c] = torch.tensor([0.3, -0.5, 0.7, 0.1])
        q = AO.poses(T, vis, float(case["t"]), case["cam"], case["is_val"], ego, in_t, bumped, ot, orr)
        assert torch.equal(p, q) == case["opt_track"], name
    if H.available() and not torch.cuda.is_available():  # the same on the reference's own ActorPose
        ns = H.load()
        ns.cfg.model.nsg.opt_track = True
        from lib.models.actor_pose import ActorPose
        meta = AC.metadata()
        ap = ActorPose(meta["obj_tracklets"], meta["tracklet_timestamps"], meta["camera_timestamps"], {k: dict(v) for k, v in meta["obj_meta"].items()})
        ap.opt_rots.data.copy_(torch.from_numpy(z["params_seeded_rots"]))
        cam = AC.camera(ns, AC.BY_NAME["train_mid"])
        before = ap.get_tracking_rotation(0, cam).detach().clone()
        ap.input_rots[14] = torch.tensor([0.3, -0.5, 0.7, 0.1])  # frame 14 is the second-nearest entry of track 0
        ap.input_rots[12] = torch.tensor([0.3, -0.5, 0.7, 0.1])
        assert torch.equal(ap.get_tracking_rotation(0, cam), before)


def test_tie_rule_decides_only_the_tie_cases():
    """`midway` ties for the nearest entry of track 3: the rule picks the frame whose rotation and opt_rots row the slerp starts from
    (the quirk of actor_pose.py:148-150), so the rotation depends on it while the translation, symmetric in the two ends, does not.
    `tie` ties for the second-nearest entries of tracks 0 and 3: the rule picks the second end of the interpolation (and the rows
    that receive theta2's and trans2's gradient).  No other case has a tie.  The fixture holds the rule's side."""
    z, _, T = fixture()
    for name in NAMES:
        case = AC.BY_NAME[name]
        a, ota, orra = run_oracle(z, T, case, finite=True)
        b, otb, orrb = run_oracle(z, T, case, tie="last", finite=True)
        if name in ("midway", "tie"):
            assert not close(b.detach().numpy(), z[f"{name}_poses"], 1e-4), name
            assert not torch.equal(ota.grad != 0, otb.grad != 0) or not torch.equal(orra.grad != 0, orrb.grad != 0), name
            if name == "midway":
                assert close(b[:, 4:].detach().numpy(), z["midway_poses"][:, 4:], 1e-6)
        else:
            assert torch.equal(a, b), name
            if ota is not None:
                assert torch.equal(ota.grad, otb.grad) and torch.equal(orra.grad, orrb.grad), name


def test_track_table_layout():
    meta = AC.metadata()
    tab = track_table(meta["obj_tracklets"], meta["tracklet_timestamps"], meta["camera_timestamps"], meta["obj_meta"])
    assert tab["track_ids"] == [0, 1, 2, 3] and list(tab["counts"]) == [38, 2, 19, 8]
    off = tab["track_off"]
    for k, (frames, col) in AC.TRACKS.items():
        fc = tab["entry_fc"][off[k]:off[k + 1]]
        assert [tuple(x) for x in fc] == [(f, col(f)) for f in frames]
        assert np.array_equal(tab["entry_ts"][off[k]:off[k + 1]], meta["tracklet_timestamps"][list(frames)])
    assert list(tab["cam_off"]) == [0, 20, 34] and tab["cam_ts"].dtype == np.float64
    assert tab["track_frames"][2].tolist() == [5, 25]


def test_entries_validate_before_touching_cuda():
    L = _capi.lib()
    err = lambda: L.sgr_last_error().decode()
    ok = C.c_void_p(1 << 20)
    tab = [4, 4, ok, ok, ok, ok, ok, 2, ok, ok, ok, ok]
    slots = (C.c_int32 * 2)(0, 4)
    assert L.sgr_actor_pose_forward(*tab, 2, slots, 0.0, 0, 0, ok, None, None, 0, 1.0, 1, ok, None, None) == -1 and "outside [0, 4)" in err()
    slots = (C.c_int32 * 2)(0, 3)
    assert L.sgr_actor_pose_forward(*tab, 2, slots, 0.0, 0, 0, ok, ok, None, 0, 1.0, 1, ok, None, None) == -1 and "both opt_trans" in err()
    assert L.sgr_actor_pose_forward(*tab, 2, slots, 0.0, 5, 1, ok, ok, ok, 0, 1.0, 1, ok, None, None) == -1 and "camera 5" in err()
    assert L.sgr_actor_pose_forward(*tab, 2, slots, 0.0, 0, 0, ok, None, None, 0, 1.0, 9, ok, ok, None) == -1 and "fourier_dim" in err()
    assert L.sgr_actor_pose_forward(*tab, 0, None, 0.0, 0, 0, ok, None, None, 0, 1.0, 1, None, None, None) == 0
    assert L.sgr_actor_pose_backward(*tab, 2, slots, 0.0, 0, 0, ok, None, None, ok, ok, ok, ok, 1 << 20, None) == -1 and "no parameters" in err()
    assert L.sgr_actor_pose_backward(*tab, 2, slots, 0.0, 0, 0, ok, ok, ok, ok, ok, ok, ok, 16, None) == -1 and "scratch" in err()
    assert L.sgr_actor_pose_scratch_bytes(8) >= 8 * 4 * 24


def test_module_needs_cuda():
    meta = AC.metadata()
    with pytest.raises(_capi.SgrError, match="no CPU fallback"):
        sgb.ActorPose(meta["obj_tracklets"], meta["tracklet_timestamps"], meta["camera_timestamps"], meta["obj_meta"], device="cpu")
