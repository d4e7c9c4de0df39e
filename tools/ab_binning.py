"""Renders the same seeded frames through two builds of libsgr.so in one process and asserts that they bin and render alike:
    python tools/ab_binning.py OLD.so NEW.so [--configs C,B,E]
For every frame, in exact and in bounded mode (and bounded with an overflowing capacity): equal `ranges`, vals_out[:E], status
words, images and grad2d, all bit for bit; plus the layered forward (objects-only / background-only layers) of a small scene."""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import util  # noqa: E402
import street_gaussians_b200 as sgb  # noqa: E402
from street_gaussians_b200 import _capi, synthetic  # noqa: E402
from street_gaussians_b200 import rasterizer as R  # noqa: E402

DEV = "cuda"


def use(lib):
    _capi._lib = None
    _capi.LIB_PATH = os.path.abspath(lib)
    _capi.lib()


def frame(scene, band, capacity):
    cam = scene["cam"]
    st = util.settings_from(sgb, cam, DEV)
    dv = lambda k: scene[k].to(DEV) if scene.get(k) is not None else None
    P = scene["means3D"].shape[0]
    cap = sgb.InstanceCapacity(initial=capacity) if capacity else None
    with torch.no_grad():
        col, rad, dep, alp, sem, fst, tens = R._forward_impl(dv("means3D"), dv("shs"), dv("colors_precomp"), dv("semantics"),
                                                            dv("opacities"), dv("scales"), dv("rotations"), dv("cov3D_precomp"), st,
                                                            band, cap)
        H, W = cam["image_height"], cam["image_width"]
        g2d, _ = R._backward_blend_impl(st, band, fst, tens, alp, scene["grad_color"].to(DEV), scene["grad_depth"].to(DEV),
                                        scene["grad_alpha"].to(DEV), torch.zeros(0, H, W, device=DEV))
    torch.cuda.synchronize()
    v = R.state_views(st, fst, P)
    E = int(v["status"][_capi.STATUS_EMITTED])
    lst = v["vals_out"][:E].clone() if E else torch.zeros(0, dtype=torch.int32, device=DEV)
    return dict(status=v["status"][:5].clone(), ranges=v["ranges"].clone(), list=lst, color=col, depth=dep, alpha=alp, radii=rad,
                grad2d=g2d), E


def layered(scene):
    cam = scene["cam"]
    st = util.settings_from(sgb, cam, DEV)
    P = scene["means3D"].shape[0]
    kw = {k: scene[k].to(DEV) for k in ("means3D", "opacities", "shs", "scales", "rotations")}
    with torch.no_grad():
        out = sgb.GaussianRasterizer(st).forward_layers(means2D=None, layers=[sgb.RenderLayer(P // 2, P, (1.0, 1.0, 1.0)),
                                                                                  sgb.RenderLayer(0, P // 2, (0.0, 0.0, 0.0))], **kw)
    torch.cuda.synchronize()
    flat = []
    for o in out:
        if isinstance(o, torch.Tensor):
            flat.append(o.clone())
        elif isinstance(o, (tuple, list)):
            for x in o:
                flat.extend(y.clone() for y in (x if isinstance(x, (tuple, list)) else (x,)) if isinstance(y, torch.Tensor))
    return flat


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--configs", default="C,B,E")
    args = ap.parse_args()
    scenes = [(c, synthetic.make_config(c, seed=0)) for c in args.configs.split(",") if c]
    scenes += [("small_sh3", synthetic.make_scene(P=3000, width=208, height=120, sh_degree=3, seed=7, pose=True, scale_med=0.08)),
               ("60k_720p", synthetic.make_scene(P=60_000, width=1280, height=720, sh_degree=1, seed=3, pose=True)),
               ("smoke_A", synthetic.smoke_script_scene(10000, 256, 256, seed=0)),
               # 313 x 250 tiles: the tile radix sort on 32-bit tile ids
               ("5000x4000", synthetic.make_scene(P=200_000, width=5000, height=4000, sh_degree=0, seed=2, scale_med=0.02))]
    bad = 0
    for name, sc in scenes:
        rows = (sc["cam"]["image_height"] + 15) // 16
        res = {}
        for lib in (args.old, args.new):
            use(lib)
            r, E = frame(sc, None, None)
            res.setdefault("exact", []).append(r)
            for label, band, cap in (("bounded", None, int(E * 1.25) + 4096), ("overflow", None, max(E // 3, 1)),
                                     ("cyclic", R.TileRowBand(1, rows, 3), int(E * 1.25) + 4096)):
                res.setdefault(label, []).append(frame(sc, band, cap)[0])
            if sc["means3D"].shape[0] <= 100_000:
                res.setdefault("layers", []).append(dict(enumerate(layered(sc))))
        for label, (a, b) in res.items():
            diff = [k for k in a if k != "grad2d" and not torch.equal(a[k], b[k])]
            note = ""
            if "grad2d" in a and not torch.equal(a["grad2d"], b["grad2d"]):
                # blend_bwd accumulates grad2d with float atomics, whose order may differ from run to run even with identical lists
                rel = float((a["grad2d"] - b["grad2d"]).abs().max() / a["grad2d"].abs().max().clamp(min=1e-30))
                note = f" (grad2d differs by float-atomic order: max rel {rel:.2e})"
                if rel > 1e-5:
                    diff.append("grad2d")
            print(f"{name:10s} {label:9s} E={int(a['status'][_capi.STATUS_EMITTED]) if 'status' in a else '-':>9} {'OK' if not diff else 'DIFF ' + ','.join(map(str, diff))}{note}",
                  flush=True)
            bad += bool(diff)
        del res
        torch.cuda.empty_cache()
    print("ALL EQUAL" if bad == 0 else f"{bad} cases differ")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
