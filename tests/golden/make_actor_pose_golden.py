"""Generates tests/golden/callsite/actor_pose.npz: the tracked actor poses the reference's UNMODIFIED ActorPose
(lib/models/actor_pose.py) gives StreetGaussianModel.parse_camera (street_gaussian_model.py:219-274), the IDFT rows of
gaussian_model_actor.py:71-77, and the gradients autograd sends back to opt_trans / opt_rots for a seeded linear functional of the
poses.  Run on a CPU-only machine with a reference checkout (tests/refharness.py):
    python tests/golden/make_actor_pose_golden.py
The model comes from refharness.make_street_model with its tracklets replaced by the ones below (tests/actor_pose_case.py), on
non-uniform float64 timestamps near 1.6e9 s.  roma is stubbed by the harness's textbook slerp (DESIGN.md §5).  The reference's
np.argsort runs in numpy's stable kind, which is the project's tie rule (nearer first, then the earlier entry): numpy's default kind
is not stable, so without this the order among ties would be whatever numpy's sort implementation gives.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import actor_pose_case as AC  # noqa: E402
import refharness as H  # noqa: E402


def _stable_argsort():
    """np.argsort in its stable kind, counting the calls where numpy's default kind orders the first two differently.  The default
    (introsort, or a SIMD sort where the CPU has one) is not stable, so on a tie the reference's choice is numpy's; the fixture is
    written with the project's rule (nearer first, then the earlier entry), which is the stable order."""
    orig = np.argsort
    seen = {"ties": 0, "differ": 0}

    def argsort(a, *args, **kw):
        s = orig(a, kind="stable")
        if len(a) > 2 and np.sum(a == a[s[1]]) > 1:
            seen["ties"] += 1
        seen["differ"] += int(list(orig(a)[:2]) != list(s[:2]))
        return s

    return orig, argsort, seen


def main():
    ns = H.load()
    cfg = ns.cfg
    cfg.mode = "train"
    C = int(cfg.model.gaussian.fourier_dim)
    scale = float(cfg.model.gaussian.fourier_scale)
    meta = AC.metadata()
    fx = dict(tracklets=meta["obj_tracklets"], timestamps=meta["tracklet_timestamps"], fourier_dim=np.int32(C), fourier_scale=np.float64(scale),
              track_ids=np.array(list(meta["obj_meta"].keys()), np.int32))
    for c, v in meta["camera_timestamps"].items():
        fx[f"cam{c}_train"] = np.asarray(v["train_timestamps"], np.float64)
    for k, v in meta["obj_meta"].items():
        fx[f"meta{k}"] = np.array([v["start_frame"], v["end_frame"], v["start_timestamp"], v["end_timestamp"]], np.float64)
    params = AC.params()
    for name, (ot, orr) in params.items():
        fx[f"params_{name}_trans"], fx[f"params_{name}_rots"] = ot, orr
    orig, argsort, seen = _stable_argsort()
    np.argsort = argsort
    try:
        for case in AC.CASES:
            cfg.model.nsg.opt_track = case["opt_track"]
            model = H.make_street_model(ns, n_bkgd=64, n_obj=len(meta["obj_meta"]), per_obj=4, num_frames=AC.F, seed=1)
            from lib.models.actor_pose import ActorPose
            model.actor_pose = ActorPose(meta["obj_tracklets"], meta["tracklet_timestamps"], meta["camera_timestamps"],
                                         {k: dict(v) for k, v in meta["obj_meta"].items()})
            for name in model.obj_list:
                om = getattr(model, name)
                m = meta["obj_meta"][om.track_id]
                om.start_frame, om.end_frame = m["start_frame"], m["end_frame"]
            ap = model.actor_pose
            if case["opt_track"]:
                ot, orr = params[case["params"]]
                ap.opt_trans.data.copy_(torch.from_numpy(ot))
                ap.opt_rots.data.copy_(torch.from_numpy(orr))
            cam = AC.camera(ns, case)
            model.set_visibility(["background"] + model.obj_list)
            model.parse_camera(cam)                                               # street_gaussian_model.py:219-284
            vis = [getattr(model, n).track_id for n in model.graph_obj_list]
            assert vis == AC.visible(case), (case["name"], vis)
            n_bkgd = model.graph_gaussian_range["background"][1]
            rows = [model.graph_gaussian_range[n][0] - n_bkgd for n in model.graph_obj_list]  # obj_rots / obj_trans hold the actors only
            poses = torch.cat([model.obj_rots[rows], model.obj_trans[rows]], 1)   # [n_act, 7]
            w = torch.from_numpy(AC.functional(case, len(vis)))
            nm = case["name"]
            fx[f"{nm}_visible"] = np.array(vis, np.int32)
            fx[f"{nm}_poses"] = poses.detach().numpy().astype(np.float32)
            fx[f"{nm}_w"] = w.numpy()
            idft = []
            for n in model.graph_obj_list:                                        # gaussian_model_actor.py:71-75
                om = getattr(model, n)
                normalized_frame = (model.frame - om.start_frame) / (om.end_frame - om.start_frame)
                idft.append(ns.sh_utils.IDFT(om.fourier_scale * normalized_frame, om.fourier_dim)[0])
            fx[f"{nm}_idft"] = torch.stack(idft).numpy().astype(np.float32)
            if case["opt_track"]:
                (poses * w).sum().backward()
                fx[f"{nm}_dtrans"] = ap.opt_trans.grad.numpy().astype(np.float32)
                fx[f"{nm}_drots"] = ap.opt_rots.grad.numpy().astype(np.float32)
            print(nm, "visible", vis, "finite grads", bool(np.isfinite(fx.get(f"{nm}_drots", np.zeros(1))).all()))
    finally:
        np.argsort = orig
    assert seen["ties"] > 0, "no case has a tie for the second-nearest entry"
    fx["cases"] = np.array([c["name"] for c in AC.CASES])
    os.makedirs(os.path.join(HERE, "callsite"), exist_ok=True)
    path = os.path.join(HERE, "callsite", "actor_pose.npz")
    np.savez_compressed(path, **fx)
    print("wrote", path, os.path.getsize(path), "bytes; ties:", seen["ties"], "calls where numpy's default argsort differs:", seen["differ"])


if __name__ == "__main__":
    main()
