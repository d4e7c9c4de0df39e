#!/usr/bin/env bash
# compute-sanitizer (memcheck + racecheck + synccheck) over one small forward+backward of every kernel family.
# Run under gpurun; logs land in gpurun_out/sanitizer_*.log
set -u
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
cat > /tmp/san_case.py <<'PY'
import sys, os
sys.path.insert(0, os.getcwd()); sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
import torch, util
import street_gaussians_b200 as sgb
from street_gaussians_b200 import synthetic
from street_gaussians_b200.sharded import cyclic_band
for kw, extra in ((dict(P=4000, width=208, height=120, sh_degree=3, seed=21, pose=True, scale_med=0.06), {}),
                  (dict(P=1500, width=128, height=80, sh_degree=2, seed=25, pose=True, scale_med=0.3, semantics=5), {}),
                  (dict(P=3000, width=160, height=112, sh_degree=1, seed=26, pose=True, scale_med=0.06), dict(band=cyclic_band(112, 1, 3)))):
    sc = synthetic.make_scene(**kw)
    r = util.run_api(sgb, sc, rasterizer_kwargs=extra)
    print("ok", kw["P"], float(abs(r["color"]).sum()), float(abs(r["g_means3D"]).sum()))
print(float(sgb.distCUDA2(torch.rand(3000, 3, device="cuda")).sum()))
# round-2 kernels: the fused Gaussian-sharded step (world = 1: project+scatter, count / compacted depth order, chain rule with the gather),
# the composer, the losses, the densification statistics and the multi-tensor Adam
import compose_case as CC
from street_gaussians_b200 import sharded as SH, losses, training
dev = torch.device("cuda")
sc = synthetic.make_scene(P=3000, width=160, height=96, sh_degree=3, seed=1, pose=True)
st = util.settings_from(sgb, sc["cam"], dev)
lt = SH._local_tensors(sc["means3D"].to(dev), sc["shs"].to(dev), None, None, sc["opacities"].to(dev), sc["scales"].to(dev), sc["rotations"].to(dev), None)
up = [sc[k].to(dev) for k in ("grad_color", "grad_depth", "grad_alpha")]
with torch.no_grad():
    for gcap in (3000, 700, -1):
        ws = SH.PeerWorkspace.emulate(st, 3000, 1, dev)[0]
        col, dep, alp, _ = SH.sharded_forward_raw(st, None, ws, lt, 3000, 500_000, gcap)
        g = SH.sharded_backward_raw(st, None, ws, lt, 3000, 500_000, alp, *up)
        print("fused ok", gcap, float(col.abs().sum()), float(g[0].abs().sum()))
models = [{k: v.to(dev).requires_grad_(True) for k, v in m.items()} for m in CC.make_case(3, 1001, [37, 0, 501], 16, 5)]
poses = torch.randn(3, 7, device=dev, requires_grad=True)
out = sgb.compose(models, poses, torch.randn(3, 5, device=dev), torch.rand(538, device=dev) < 0.5, torch.tensor([0.0, 0.0, 1.0, 0.0], device=dev))
sum(o.sum() for o in out).backward()
print("compose ok", float(out[0].abs().sum()), float(poses.grad.abs().sum()))
# the corrected composer (background pose correction, 40 actors: two segment groups) and the colour correction with its regularisation
models = [{k: v.to(dev).requires_grad_(True) for k, v in m.items()} for m in CC.make_case(4, 777, [13] * 40, 9, 3)]
poses = torch.randn(40, 7, device=dev, requires_grad=True)
corr = (torch.tensor([0.9, 0.1, -0.2, 0.3], device=dev, requires_grad=True), torch.randn(3, device=dev, requires_grad=True))
out = sgb.compose(models, poses, torch.randn(40, 3, device=dev), torch.rand(520, device=dev) < 0.5, torch.tensor([0.0, 0.0, 1.0, 0.0], device=dev),
                  pose_correction=corr)
sum(o.sum() for o in out).backward()
aff = (torch.eye(4, device=dev)[:3] + 0.1).requires_grad_(True)
for hw in ((70, 93), (64, 96)):
    img = torch.rand(3, *hw, device=dev, requires_grad=True)
    (sgb.color_correct(img, aff).sum() + sgb.color_correction_reg_loss(aff, aff * 0.5, 0.1)).backward()
print("corrections ok", float(corr[0].grad.abs().sum()), float(aff.grad.abs().sum()))
img = torch.rand(3, 70, 93, device=dev, requires_grad=True)
l = losses.photometric_loss(img, torch.rand(3, 70, 93, device=dev), torch.rand(1, 70, 93, device=dev) > 0.3) + losses.sky_loss(img[:1], torch.rand(1, 70, 93, device=dev) > 0.5)
l.backward()
print("loss ok", float(l), float(img.grad.abs().sum()))
stats = [dict(max_radii2D=torch.zeros(n, device=dev), xyz_gradient_accum=torch.zeros(n, 2, device=dev), denom=torch.zeros(n, 1, device=dev)) for n in (1001, 37, 0, 501)]
training.add_densification_stats(stats, torch.randint(-1, 9, (1539,), device=dev, dtype=torch.int32), torch.randn(1539, 3, device=dev))
ps = [torch.nn.Parameter(torch.randn(n, device=dev)) for n in (5, 70001, 12)]
opt = training.FusedAdam([dict(params=[p], lr=1e-3) for p in ps], eps=1e-15)
for p in ps:
    p.grad = torch.randn_like(p)
opt.step()
print("stats/adam ok", float(stats[0]["denom"].sum()), float(ps[1].abs().sum()))
PY
for tool in memcheck racecheck synccheck; do
  timeout 600 compute-sanitizer --tool $tool --print-limit 20 python /tmp/san_case.py > gpurun_out/sanitizer_$tool.log 2>&1
  echo "== $tool rc=$? =="; grep -E "ERROR SUMMARY|RACECHECK SUMMARY|ok |Error|hazard" gpurun_out/sanitizer_$tool.log | head -12
done
