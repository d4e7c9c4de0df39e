"""Loads tests/golden/callsite/densify.npz (tests/golden/make_densify_golden.py) into per-model inputs for the oracle
(oracle/densify_oracle.py) and for street_gaussians_b200.training.densify_and_prune."""
from __future__ import annotations

import os
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "callsite", "densify.npz")
NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "semantic")
ATTR = dict(xyz="_xyz", f_dc="_features_dc", f_rest="_features_rest", opacity="_opacity", scaling="_scaling", rotation="_rotation",
            semantic="_semantic")


def load():
    z = np.load(FIXTURE)
    models = []
    k = 0
    while f"m{k}_kind" in z:
        p = f"m{k}_"
        g = lambda s: torch.from_numpy(np.array(z[p + s]))
        m = dict(kind=str(z[p + "kind"]), grad_col=int(z[p + "grad_col"]), grad_threshold=float(z[p + "grad_threshold"]),
                 extent=g("extent"), percent_dense=float(z[p + "percent_dense"]), percent_big_ws=float(z[p + "percent_big_ws"]),
                 draws=g("draws"))
        if m["kind"] == "background":
            m["sphere_center"], m["sphere_radius"] = g("sphere_center"), g("sphere_radius")
        else:
            m["min_xyz"], m["max_xyz"] = g("min_xyz"), g("max_xyz")
        for io in ("in", "out"):
            m[io] = {a: g(f"{io}_{a}") for a in NAMES}
            m[io]["exp_avg"] = {a: g(f"{io}_exp_avg_{a}") for a in NAMES}
            m[io]["exp_avg_sq"] = {a: g(f"{io}_exp_avg_sq_{a}") for a in NAMES}
            m[io]["step"] = {a: float(z[p + f"{io}_step_{a}"]) for a in NAMES}
            for s in ("xyz_gradient_accum", "denom", "max_radii2D"):
                m[io][s] = g(f"{io}_{s}")
        m["scalars"] = dict(zip([str(s) for s in z[p + "scalar_keys"]], [int(v) for v in z[p + "scalar_values"]]))
        models.append(m)
        k += 1
    return models, float(z["min_opacity"])


def oracle_kwargs(m, min_opacity, prune_big_points=True):
    kw = dict(grad_threshold=m["grad_threshold"], grad_col=m["grad_col"], extent=m["extent"], percent_dense=m["percent_dense"],
              percent_big_ws=m["percent_big_ws"], min_opacity=min_opacity, prune_big_points=prune_big_points)
    if m["kind"] == "background":
        kw.update(sphere_center=m["sphere_center"], sphere_radius=m["sphere_radius"])
    else:
        kw.update(min_xyz=m["min_xyz"], max_xyz=m["max_xyz"])
    return kw


def product_model(m, device, io="in"):
    """A model object with the reference's attribute names, as densify_and_prune reads it."""
    ns = types.SimpleNamespace()
    d = m[io]
    for a in NAMES:
        setattr(ns, ATTR[a], torch.nn.Parameter(d[a].clone().to(device)))
    for s in ("xyz_gradient_accum", "denom", "max_radii2D"):
        setattr(ns, s, d[s].clone().to(device))
    ns.percent_dense, ns.percent_big_ws = m["percent_dense"], m["percent_big_ws"]
    if m["kind"] == "background":
        ns.scene_radius = m["extent"].to(device)
        ns.sphere_center, ns.sphere_radius = m["sphere_center"].to(device), m["sphere_radius"].to(device)
    else:
        ns.extent = m["extent"].to(device)
        ns.min_xyz, ns.max_xyz = m["min_xyz"].to(device), m["max_xyz"].to(device)
    return ns
