"""Generates tests/golden/live/thresholds.npz: what the UNMODIFIED reference CUDA rasterizer (oracle/_ref, built by
oracle/build_ref.sh) renders for the near-threshold scenes of tests/threshold_case.golden_scenes() — rings of pixels on
alpha = 1/255, splats centred on a pixel, needles of conic condition number up to 1e6.  Must run on a GPU with oracle/_ref:

    python tests/golden/make_threshold_golden.py [OUT_DIR]      (default: tests/golden/live)

The inputs are not stored (they are regenerated from seeds on the CPU).  Per scene <name>: <name>/radii, <name>/color [3, H, W],
<name>/alpha [H, W] and the reference's GeometryState records decoded by test_parity_gpu._parse_ref_geom: <name>/xy [P, 2],
<name>/conic_opacity [P, 4], <name>/depth [P], <name>/rgb [P, 3]; the images are small (at most 128 x 96)."""
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
import threshold_case as TC  # noqa: E402


def reference_forward(ref, scene):
    """The reference's forward entry point (rasterize_points.cu) on one scene: colour, alpha, radii and decoded records."""
    dev, P = "cuda", scene["means3D"].shape[0]
    st = util.settings_from(ref, scene["cam"], dev)
    args = (st.bg, scene["means3D"].to(dev), torch.Tensor([]), torch.zeros(P, 0, device=dev), scene["opacities"].to(dev),
            scene["scales"].to(dev), scene["rotations"].to(dev), st.scale_modifier, torch.Tensor([]), st.viewmatrix, st.projmatrix,
            st.tanfovx, st.tanfovy, st.image_height, st.image_width, scene["shs"].to(dev), st.sh_degree, st.campos, False, False)
    n_ref, color, depth, alpha, sem, radii, geom, binning, img = ref._C.rasterize_gaussians(*args)
    torch.cuda.synchronize()
    g = T._parse_ref_geom(geom, P)
    return dict(radii=radii.cpu().numpy(), color=color.cpu().numpy(), alpha=alpha.reshape(color.shape[1:]).cpu().numpy(),
                xy=g["xy"].copy(), conic_opacity=g["conic_opacity"].copy(), depth=g["depth"].copy(), rgb=g["rgb"].copy())


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "live")
    os.makedirs(out, exist_ok=True)
    ref = util.load_ref()
    z = {}
    for name, scene in TC.golden_scenes().items():
        for k, v in reference_forward(ref, scene).items():
            z[f"{name}/{k}"] = v
    path = os.path.join(out, "thresholds.npz")
    np.savez_compressed(path, **z)
    print("thresholds", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
