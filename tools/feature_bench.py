"""Times the renderer's feature channels at config C (1.5 M background + 8 x 50 k vehicle Gaussians, 1920x1280, SH degree 3).
CUDA events around each call, median and p10-p90 of STEPS after WARMUP, the arms alternating call by call in one process.
  (a) each operation, forward + backward, against the reference's torch lines on the same GPU:
      gaussian_normals   vs GaussianModel.get_normals on the composed rows (tests/feature_oracle.normals64 in fp32), and vs the
                         reference's per-model lines with the actors' normals rotated by their pose and renormalised
                         (street_gaussian_model.py:459-480 with torch.nn.functional spelt right: as shipped they raise)
      compose_semantics  vs StreetGaussianModel.get_semantic (K = 19, both modes)
      finish_features    vs render_kernel's split and finishing (S = 3 + 19, both modes)
      plus the device time of each feature kernel (torch.profiler)
  (b) compose -> rasterize -> finish -> loss -> backward with S = 0, S = 3 (normals) and S = 3 + K (normals + semantics, K = 19)
Prints one JSON line with the GPU name and its enforced power limit.
python tools/feature_bench.py"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from layer_bench import events_ms  # noqa: E402
from loss_bench import power_limit_w  # noqa: E402
import feature_oracle as FO  # noqa: E402
import street_gaussians_b200 as sgb  # noqa: E402
from street_gaussians_b200 import synthetic  # noqa: E402

DEV = "cuda"
K = 19
STEPS = int(os.environ.get("FEATURE_BENCH_STEPS", 30))
WARMUP = int(os.environ.get("FEATURE_BENCH_WARMUP", 5))
KERNELS = ("gaussian_normals_fwd_kernel", "gaussian_normals_bwd_kernel", "semantic_softmax_fwd_kernel", "semantic_softmax_bwd_kernel",
           "semantic_actor_fwd_kernel", "semantic_actor_bwd_kernel", "finish_features_fwd_kernel", "finish_features_bwd_kernel")


def timed(calls, iters=STEPS, warmup=WARMUP):
    ts = [[] for _ in calls]
    for it in range(warmup + iters):
        for k, fn in enumerate(calls):
            t = events_ms(fn)
            if it >= warmup:
                ts[k].append(t)
    return [dict(median_ms=float(np.median(t)), p10_ms=float(np.percentile(t, 10)), p90_ms=float(np.percentile(t, 90))) for t in ts]


def kernel_us(fn, calls=5):
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        name = ev.key.split("(")[0].split("::")[-1].split("<")[0]
        if name in KERNELS:
            out[name] = out.get(name, 0.0) + ev.device_time_total / calls
    return out


def quat_mat(q):
    return FO.quaternion_to_matrix(q.reshape(1, 4))[0]


def main():
    assert torch.cuda.is_available(), "tools/feature_bench.py needs a CUDA device"
    out = dict(gpu=torch.cuda.get_device_name(), power_limit_w=power_limit_w(), steps=STEPS, warmup=WARMUP, K=K)
    sc = synthetic.make_config("C", seed=0, with_raw=True)
    raw, cam = sc["raw"], sc["cam"]
    H, W = cam["image_height"], cam["image_width"]
    n_act = raw["poses"].shape[0]
    poses, idft = raw["poses"].to(DEV), raw["idft"].to(DEV)
    labels = [(3 * a + 1) % K for a in range(n_act)]
    g = torch.Generator().manual_seed(0)
    models = []
    for k, m in enumerate(raw["models"]):
        d = {key: v.to(DEV).requires_grad_(True) for key, v in m.items()}
        d["semantic"] = torch.randn(int(m["xyz"].shape[0]), K if k == 0 else 1, generator=g).to(DEV).requires_grad_(True)
        models.append(d)
    leaves = [v for m in models for v in m.values()]
    centre = cam["campos"].to(DEV)
    with torch.no_grad():
        xyz, rot, scale, opac, sh = sgb.compose(models, poses, idft)
    P = int(xyz.shape[0])
    out["P"] = P

    # ---- (a) each operation, forward + backward
    rot_leaf = rot.clone().requires_grad_(True)
    up_n = torch.randn(P, 3, device=DEV)

    def zero():
        for x in leaves + [rot_leaf]:
            x.grad = None

    def n_ours():
        zero()
        sgb.gaussian_normals(xyz, rot_leaf, scale, centre).backward(up_n)

    def n_torch():
        zero()
        FO.normals64(xyz, rot_leaf, scale, centre)["n"].backward(up_n)

    def n_reference_models():
        """The reference's per-model lines: get_normals per sub-model on its own rows; the actors' normals turned by their pose and
        renormalised (street_gaussian_model.py:466-477, torch.nn.functional spelt right)."""
        zero()
        parts = []
        for k, m in enumerate(models):
            r = torch.nn.functional.normalize(m["rotation"])
            nk = FO.normals64(m["xyz"], r, torch.exp(m["scaling"]), centre)["n"]
            if k > 0:
                nk = torch.nn.functional.normalize(nk @ quat_mat(poses[k - 1, :4]).T)
            parts.append(nk)
        torch.cat(parts, 0).backward(up_n)

    ops = {}
    t = timed([n_ours, n_torch, n_reference_models])
    ops["gaussian_normals"] = dict(fused=t[0], reference_lines_composed_rows=t[1], reference_lines_per_model_actor_typo_fixed=t[2],
                                   kernel_us=kernel_us(n_ours))
    up_s = torch.randn(P, K, device=DEV)
    for mode in ("logits", "probabilities"):
        def s_ours():
            zero()
            sgb.compose_semantics(models, labels, mode).backward(up_s)

        def s_torch():
            zero()
            FO.semantics64(models[0]["semantic"], [m["semantic"] for m in models[1:]], labels, mode).backward(up_s)

        t = timed([s_ours, s_torch])
        ops[f"compose_semantics_{mode}"] = dict(fused=t[0], reference_lines=t[1], kernel_us=kernel_us(s_ours))
    feat = torch.rand(3 + K, H, W, device=DEV).requires_grad_(True)
    gn, gs = torch.randn(3, H, W, device=DEV), torch.randn(K, H, W, device=DEV)
    for mode in ("logits", "probabilities"):
        def f_ours():
            feat.grad = None
            n, s = sgb.finish_features(feat, 3, mode)
            torch.autograd.backward([n, s], [gn, gs])

        def f_torch():
            feat.grad = None
            n, s = FO.finish64(feat, 3, mode)
            torch.autograd.backward([n, s], [gn, gs])

        t = timed([f_ours, f_torch])
        ops[f"finish_features_{mode}"] = dict(fused=t[0], reference_lines=t[1], kernel_us=kernel_us(f_ours))
    out["operations"] = ops

    # ---- (b) the composed step with S = 0, 3 and 3 + K
    st = sgb.GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=cam["tanfovx"], tanfovy=cam["tanfovy"], bg=torch.zeros(3, device=DEV),
                                           scale_modifier=1.0, viewmatrix=cam["viewmatrix"].to(DEV), projmatrix=cam["projmatrix"].to(DEV),
                                           sh_degree=cam["sh_degree"], campos=cam["campos"].to(DEV), prefiltered=False, debug=False)
    rast = sgb.GaussianRasterizer(st)
    gt = torch.rand(3, H, W, device=DEV)
    gt_n, gt_s = torch.randn(3, H, W, device=DEV), torch.randn(K, H, W, device=DEV)
    losses = {}

    def step(S):
        def go():
            zero()
            x, r, s, o, f = sgb.compose(models, poses, idft)
            m2d = torch.zeros_like(x, requires_grad=True)
            feats = None
            if S:
                parts = [sgb.gaussian_normals(x, r, s, centre)]
                if S > 3:
                    parts.append(sgb.compose_semantics(models, labels, "probabilities"))
                feats = torch.cat(parts, -1)
            res = rast(means3D=x, means2D=m2d, opacities=o, shs=f, scales=s, rotations=r, semantics=feats)
            loss = (res[0] - gt).abs().mean()
            if S:
                n_img, s_img = sgb.finish_features(res[4], 3, "probabilities")
                loss = loss + (n_img * gt_n).mean()
                if s_img is not None:
                    loss = loss + (s_img * gt_s).mean()
            loss.backward()
            losses.setdefault(S, []).append(loss.detach())
        return go

    arms = (0, 3, 3 + K)
    t = timed([step(S) for S in arms], iters=max(STEPS, 20))
    for S in arms:
        assert bool(torch.isfinite(torch.stack(losses[S])).all()), f"S = {S}: non-finite loss"
    out["composed_step_config_C"] = {f"S={S}": tt for S, tt in zip(arms, t)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
