"""street_gaussians_b200 — H100-native (sm_90a) differentiable Gaussian-splatting rasterizer.

Drop-in for the one hot path of zju3dv/street_gaussians (SURVEY.md §8): ``submodules/diff-gaussian-rasterization`` and
``simple-knn``'s ``distCUDA2``, behind the reference's own Python API.  ``install_shims()`` makes
``import diff_gaussian_rasterization`` / ``from simple_knn._C import distCUDA2`` resolve to this package so
lib/utils/camera_utils.py:13 and lib/models/gaussian_model.py:5 run unchanged.
"""
from __future__ import annotations

import os
import sys

from .rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, InstanceCapacity, RenderLayer, TileRowBand,  # noqa: F401
                         distCUDA2, rasterize_gaussians)

from .composer import compose  # noqa: E402,F401
from .corrections import color_correct, color_correction_reg_loss  # noqa: E402,F401
from .sky import sky_composite  # noqa: E402,F401
from .actor_pose import ActorPose  # noqa: E402,F401
from .features import compose_semantics, finish_features, gaussian_normals  # noqa: E402,F401
from .metrics import ViewMetrics  # noqa: E402,F401
from . import band_losses, corrections, features, losses, metrics, sky, training  # noqa: E402,F401

__all__ = ["compose", "ActorPose", "color_correct", "color_correction_reg_loss", "sky_composite", "gaussian_normals", "compose_semantics",
           "finish_features", "ViewMetrics", "GaussianRasterizationSettings", "GaussianRasterizer", "TileRowBand", "InstanceCapacity", "RenderLayer", "rasterize_gaussians", "distCUDA2",
           "install_shims"]

_SHIMS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "shims")


def install_shims() -> str:
    """Put the import-compatible shim packages (diff_gaussian_rasterization, simple_knn) first on sys.path."""
    if _SHIMS not in sys.path:
        sys.path.insert(0, _SHIMS)
    for name in ("diff_gaussian_rasterization", "simple_knn", "simple_knn._C"):
        mod = sys.modules.get(name)
        if mod is not None and not getattr(mod, "__file__", "").startswith(_SHIMS):
            del sys.modules[name]
    return _SHIMS
