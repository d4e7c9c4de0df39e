"""Regenerates tests/golden/callsite/densify.npz from the reference's UNMODIFIED StreetGaussianModel.densify_and_prune (the
background's and the actors' densify_and_prune, lib/models/gaussian_model_bkgd.py:74-114 and gaussian_model_actor.py:204-261), run
on the CPU through tests/refharness.py.  Needs a reference checkout (SGR_REFERENCE_DIR); the fixture is committed.

The model is a real StreetGaussianModel (a background and two actors, SH degree 1, fourier_dim 5) whose optimizers have taken two
Adam steps on seeded gradients, so that the moments are non-zero.  Its densification statistics are seeded, random_initialization is
False on the actors, and a few Gaussians are planted: big ones inside and outside 2 * sphere_radius, and actor points next to the
faces of the tracking box.  torch.normal is replaced by mean + z * std with z from a seeded generator (torch's own definition of
normal(mean, std)), and every z is recorded and stored in the per-parent layout of oracle/densify_oracle.py.

    python tests/golden/make_densify_golden.py
"""
from __future__ import annotations

import io
import os
import sys
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import refharness as RH  # noqa: E402
from oracle import densify_oracle as DO  # noqa: E402

OUT = os.path.join(HERE, "callsite", "densify.npz")
NAMES = dict(xyz="_xyz", f_dc="_features_dc", f_rest="_features_rest", opacity="_opacity", scaling="_scaling", rotation="_rotation",
             semantic="_semantic")
MIN_OPACITY, MAX_GRAD = 0.005, 2e-4


def write_npz(path, arrays):
    """np.savez_compressed with a fixed timestamp, so that the file is byte-for-byte reproducible."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    torch.manual_seed(0)
    ns = RH.load()
    cfg = ns.cfg
    model = RH.make_street_model(ns, n_bkgd=600, n_obj=2, per_obj=200, seed=11)
    model.training_setup()
    g = torch.Generator().manual_seed(5)
    names = list(model.model_name_id.keys())
    out = {"min_opacity": np.float64(MIN_OPACITY), "max_grad": np.float64(MAX_GRAD), "names": np.array(names)}
    for k, name in enumerate(names):
        sub = getattr(model, name)
        for _ in range(2):  # two Adam steps on seeded gradients: non-zero moments, step == 2
            for p in (getattr(sub, a) for a in NAMES.values()):
                p.grad = torch.randn(p.shape, generator=g) * 1e-2
            sub.optimizer.step()
        n = sub._xyz.shape[0]
        with torch.no_grad():
            denom = torch.randint(0, 5, (n, 1), generator=g).float()
            accum = denom * torch.rand(n, 2, generator=g) * torch.tensor([6e-4, 1.6e-3]) * 1.2
            opac = sub._opacity.data
            low = torch.rand(n, generator=g) < 0.05
            opac[low] = -6.0
            if k == 0:  # big Gaussians: 0..4 inside 2 * sphere_radius (pruned), 5..9 outside (kept); no densification of either
                sub._scaling.data[:10] = torch.log(torch.tensor([3.0, 0.5, 0.5]))
                sub._xyz.data[:5] = torch.tensor([0.0, 0.0, 10.0])
                sub._xyz.data[5:10] = torch.tensor([50.0, 5.0, 20.0])
                accum[:10] = 0.0
                opac[:10] = 2.0
            else:       # actor points 0.05 inside a face of the tracking box, with scales whose samples may cross it
                sub.random_initialization = False
                hi = torch.as_tensor(sub.max_xyz).float().reshape(-1)
                for r in range(12):
                    a = r % 3
                    sub._xyz.data[r] = 0.0
                    sub._xyz.data[r, a] = (1 if r % 2 else -1) * (float(hi[a]) - 0.05)
                    sub._scaling.data[r] = float(np.log(0.02))
                    opac[r] = 2.0
        sub.xyz_gradient_accum = accum
        sub.denom = denom
        sub.max_radii2D = torch.rand(n, generator=g) * 30
        pre = {a: getattr(sub, attr).detach().clone() for a, attr in NAMES.items()}
        st = {a: sub.optimizer.state[getattr(sub, attr)] for a, attr in NAMES.items()}
        kind = "background" if k == 0 else "actor"
        col = int(bool(cfg.optim.get("densify_grad_abs_bkgd" if k == 0 else "densify_grad_abs_obj", False)))
        thr = float(cfg.optim.get("densify_grad_threshold_bkgd" if k == 0 else "densify_grad_threshold_obj", MAX_GRAD))
        extent = sub.scene_radius if k == 0 else sub.extent
        p = f"m{k}_"
        out[p + "kind"] = np.array(kind)
        out[p + "grad_col"], out[p + "grad_threshold"] = np.int64(col), np.float64(thr)
        out[p + "extent"] = extent.numpy().astype(np.float32)
        out[p + "percent_dense"], out[p + "percent_big_ws"] = np.float64(sub.percent_dense), np.float64(sub.percent_big_ws)
        if k == 0:
            out[p + "sphere_center"], out[p + "sphere_radius"] = sub.sphere_center.numpy(), sub.sphere_radius.numpy()
        else:
            out[p + "min_xyz"] = torch.as_tensor(sub.min_xyz).float().numpy()
            out[p + "max_xyz"] = torch.as_tensor(sub.max_xyz).float().numpy()
        for a in NAMES:
            out[p + "in_" + a] = pre[a].numpy()
            out[p + "in_exp_avg_" + a] = st[a]["exp_avg"].numpy().copy()
            out[p + "in_exp_avg_sq_" + a] = st[a]["exp_avg_sq"].numpy().copy()
            out[p + "in_step_" + a] = np.float64(float(st[a]["step"]))
        out[p + "in_xyz_gradient_accum"], out[p + "in_denom"] = accum.numpy(), denom.numpy()
        out[p + "in_max_radii2D"] = sub.max_radii2D.numpy()

    drawn = []
    orig = torch.normal
    zg = torch.Generator().manual_seed(17)

    def normal(mean, std, *a, **kw):
        z = torch.randn(torch.broadcast_shapes(mean.shape, std.shape), generator=zg)
        drawn.append(z)
        return mean + z * std

    torch.normal = normal
    try:
        model.densify_and_prune(max_grad=MAX_GRAD, min_opacity=MIN_OPACITY, prune_big_points=True)
    finally:
        torch.normal = orig
    # draws per model in call order: background split; then per actor split, box
    it = iter(drawn)
    for k, name in enumerate(names):
        sub = getattr(model, name)
        p = f"m{k}_"
        t = {a: torch.from_numpy(out[p + "in_" + a]) for a in NAMES}
        t["xyz_gradient_accum"], t["denom"] = torch.from_numpy(out[p + "in_xyz_gradient_accum"]), torch.from_numpy(out[p + "in_denom"])
        _, clone, split = DO.decisions(t, int(out[p + "grad_col"]), float(out[p + "grad_threshold"]), torch.from_numpy(out[p + "extent"]),
                                       float(out[p + "percent_dense"]))
        z_split = next(it)
        z_box = next(it) if k > 0 else None
        out[p + "draws"] = DO.reference_draws_to_layout(t["xyz"].shape[0], z_split, z_box, clone, split).numpy()
        for a, attr in NAMES.items():
            prm = getattr(sub, attr)
            st = sub.optimizer.state[prm]
            out[p + "out_" + a] = prm.detach().numpy()
            out[p + "out_exp_avg_" + a] = st["exp_avg"].numpy()
            out[p + "out_exp_avg_sq_" + a] = st["exp_avg_sq"].numpy()
            out[p + "out_step_" + a] = np.float64(float(st["step"]))
        for s in ("xyz_gradient_accum", "denom", "max_radii2D"):
            out[p + "out_" + s] = getattr(sub, s).numpy()
        sc = dict(sub.scalar_dict)
        out[p + "scalar_keys"] = np.array(sorted(sc))
        out[p + "scalar_values"] = np.array([int(sc[s]) for s in sorted(sc)], dtype=np.int64)
    assert next(it, None) is None
    write_npz(OUT, out)
    print(OUT, os.path.getsize(OUT), "bytes;", {n: dict(getattr(model, n).scalar_dict) for n in names})


if __name__ == "__main__":
    main()
