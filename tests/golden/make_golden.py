"""Generates tests/golden/*.npz: seeded inputs + the outputs/gradients of the UNMODIFIED reference CUDA rasterizer
(oracle/_ref, built by oracle/build_ref.sh from /root/reference sources) on those inputs.  Must run on a GPU box:

    gpurun -- 'python tests/golden/make_golden.py'      (files come back through gpurun_out/golden/, then are copied here)
    python tests/golden/make_golden.py --only waymo_K --only scale_mod    (just those cases; the other files stay byte-identical)

These fixtures are the pin for the CPU oracle (tests/test_oracle_cpu.py) and a second, box-independent reference for the
CUDA parity tests (tests/test_parity_gpu.py).  The reference ships no golden vectors of its own (SURVEY.md §4)."""
import argparse
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import camera64_case  # noqa: E402
import util  # noqa: E402
from street_gaussians_b200 import synthetic  # noqa: E402

CASES = {
    "sh3_pose": dict(gen=lambda: synthetic.make_scene(P=1500, width=160, height=96, sh_degree=3, seed=101, pose=True, scale_med=0.06)),
    "sh1_whitebg": dict(gen=lambda: synthetic.make_scene(P=1200, width=112, height=80, sh_degree=1, seed=102, pose=True, scale_med=0.05,
                                                          bg=(1.0, 1.0, 1.0))),
    "smoke_script": dict(gen=lambda: synthetic.smoke_script_scene(num_points=1500, width=311, height=94, seed=103)),
    "semantics3": dict(gen=lambda: synthetic.make_scene(P=1000, width=96, height=64, sh_degree=2, seed=104, pose=True, scale_med=0.06,
                                                         semantics=3)),
    "colors_precomp": dict(gen=lambda: synthetic.make_scene(P=1000, width=96, height=64, sh_degree=0, seed=105, pose=True, scale_med=0.06),
                           colors_precomp=True),
    # a Waymo frame's camera (tests/camera64_case.py C2): K-projection with the principal point off centre, swapped FoVs
    "waymo_K": dict(gen=lambda: synthetic.make_scene(P=800, width=96, height=64, sh_degree=3, seed=106, pose=True, scale_med=0.06,
                                                     intrinsics=camera64_case.intrinsics("C2", 96, 64))),
    # scale_modifier != 1: the backward reports the gradient w.r.t. modifier * scale
    "scale_mod": dict(gen=lambda: synthetic.make_scene(P=1000, width=96, height=64, sh_degree=2, seed=107, pose=True, scale_med=0.06,
                                                       scale_modifier=0.6)),
    # active degree 1 of 16 stored coefficients (finite, non-zero beyond the first 4)
    "active_sh": dict(gen=lambda: synthetic.make_scene(P=1000, width=96, height=64, sh_degree=1, sh_coeffs=16, seed=108, pose=True,
                                                       scale_med=0.06)),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", action="append", choices=sorted(CASES), help="generate this case only (repeatable)")
    only = ap.parse_args().only
    out_dirs = [HERE, os.path.join(ROOT, "gpurun_out", "golden")]
    for d in out_dirs:
        os.makedirs(d, exist_ok=True)
    ref = util.load_ref()
    for name, spec in CASES.items():
        if only and name not in only:
            continue
        scene = spec["gen"]()
        use_cp = bool(spec.get("colors_precomp"))
        if use_cp:
            gen = torch.Generator().manual_seed(7)
            scene["colors_precomp"] = torch.rand(scene["means3D"].shape[0], 3, generator=gen)
        r = util.run_api(ref, scene, use_colors_precomp=use_cp)
        cam = scene["cam"]
        z = {k: np.asarray(cam[k]) for k in ("image_height", "image_width", "tanfovx", "tanfovy", "scale_modifier", "sh_degree")}
        for k in ("bg", "viewmatrix", "projmatrix", "campos"):
            z[k] = cam[k].numpy()
        for k in ("means3D", "shs", "opacities", "scales", "rotations", "semantics", "colors_precomp", "grad_color", "grad_depth",
                  "grad_alpha", "grad_semantic"):
            if k in scene and not (use_cp and k == "shs"):
                z["in_" + k] = scene[k].numpy()
        for k, v in r.items():
            if v is not None:
                z["ref_" + k] = v
        for d in out_dirs:
            np.savez_compressed(os.path.join(d, name + ".npz"), **z)
        print(name, "visible", int((r["radii"] > 0).sum()), "of", scene["means3D"].shape[0])


if __name__ == "__main__":
    main()
