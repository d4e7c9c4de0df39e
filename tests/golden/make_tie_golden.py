"""Generates tests/golden/live/ties.npz: what the UNMODIFIED reference CUDA rasterizer (oracle/_ref, built by oracle/build_ref.sh)
computes for the two seeded tie scenes of tests/test_depth_ties_gpu.py (tests/tie_case.py: the tie groups and the clone scene).
Must run on a GPU with oracle/_ref present:

    python tests/golden/make_tie_golden.py [OUT_DIR]      (default: tests/golden/live)

The inputs are not stored: both scenes are rebuilt from their seeds on the CPU.  The scenes are small, so every output is stored
whole, per scene prefix <name>_: radii, depth_bits (the view depth of every Gaussian, from the reference's GeometryState), the
color / depth / alpha images and every gradient (g_means3D, g_means2D, g_shs, g_opacities, g_scales, g_rotations)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import util  # noqa: E402
import test_parity_gpu as T  # noqa: E402
import test_depth_ties_gpu as D  # noqa: E402


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "live")
    os.makedirs(out, exist_ok=True)
    ref = util.load_ref()
    z = {}
    for name, c in D.golden_scenes().items():
        sc = c["scene"]
        r = util.run_api(ref, sc)
        P = sc["means3D"].shape[0]
        _, _, radii, geom = T.reference_geometry(ref, sc)
        g = T._parse_ref_geom(geom, P)
        assert (radii.cpu().numpy() == r["radii"]).all()
        z[f"{name}_radii"] = r["radii"]
        z[f"{name}_depth_bits"] = g["depth"].view(np.int32).copy()
        for k in ("color", "depth", "alpha", "g_means3D", "g_means2D", "g_shs", "g_opacities", "g_scales", "g_rotations"):
            z[f"{name}_{k}"] = r[k]
        torch.cuda.empty_cache()
    path = os.path.join(out, "ties.npz")
    np.savez_compressed(path, **z)
    print(path, os.path.getsize(path), "bytes", flush=True)


if __name__ == "__main__":
    main()
