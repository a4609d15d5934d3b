"""Cost and gain of the learned background (DESIGN §4.16).  Needs a GPU.  Every JSON line carries the card and its power limit, read in
the same run.
  (a) cost: the median time (CUDA events) of a 4096-ray eval render (tetra_nerf settings) on the 301,875-tetrahedra Delaunay mesh and of
      an 8192-ray fused training step (forward + backward, map gradient included) on the 2,020,866-tetrahedra mesh, each without and
      with a 256 x 512 map, in the default and the deterministic mode;
  (b) quality: surface_scene on a 45k-point mesh, viewed so that about half of each view leaves the mesh, rendered over a known map
      (a sky gradient with a few coloured patches) is the target.  From a random field and a fresh MLP, Adam trains the field, the MLP
      and, in one arm, a white-initialised map, against the constant white background in the other arm.  Held-out PSNR on all rays and
      on the rays with accumulation < 0.5."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (str(ROOT), str(ROOT / "tetra-nerf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import oracle as orc  # noqa: E402
from tetranerf.b200 import synthetic as syn  # noqa: E402

DEV = torch.device("cuda:0")


def _gpu():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else "unknown"


def _timed(fn, n, warm):
    ts = []
    for i in range(warm + n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        if i >= warm:
            ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def sky_map(H: int) -> torch.Tensor:
    """f32[H,2H,3] on the CPU: a blue-to-orange gradient in latitude with three coloured patches"""
    v = (torch.arange(H, dtype=torch.float32) + 0.5) / H  # 0 at the zenith, 1 at the nadir
    m = torch.empty((H, 2 * H, 3))
    m[..., 0] = (0.25 + 0.7 * v)[:, None]
    m[..., 1] = (0.45 + 0.25 * v)[:, None]
    m[..., 2] = (0.95 - 0.75 * v)[:, None]
    W = 2 * H
    for (j, i, c) in ((H // 4, W // 8, (1.0, 0.1, 0.1)), (H // 2, W // 2, (0.1, 0.9, 0.2)), (3 * H // 4, 3 * W // 4, (0.9, 0.9, 0.1))):
        m[max(0, j - H // 8):j + H // 8 + 1, max(0, i - W // 16):i + W // 16 + 1] = torch.tensor(c)
    return m


def view_rays(R: int, seed: int):
    """camera_rays' bundle, its targets spread over [-0.5, 1.5]^3, so about half of the rays leave the unit-cube mesh"""
    rng = np.random.default_rng(seed)
    o = (np.array([0.5, -1.5, 0.5]) + 0.05 * rng.standard_normal((R, 3))).astype(np.float32)
    d = (-0.5 + 2.0 * rng.random((R, 3))).astype(np.float32) - o
    return o, (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


def train_arm(mesh, steps: int, H: int, seed: int, rays: int, learn_map: bool, target_map: torch.Tensor, lr: float = 1e-2):
    """trains field + MLP (+ the map when learn_map) on `rays` fixed rays against the target rendered over target_map -> metrics"""
    from tetranerf import cpp
    from tetranerf.b200.render import PARAM_ORDER, FusedRenderer, FusedTrainRender, RenderSettings

    V, C = mesh
    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV))
    fr = FusedRenderer(tr)
    st = RenderSettings(num_samples=64, num_fine_samples=64, use_biased_sampler=True)
    f_t, p_t = syn.surface_scene(V, 30, orc.init_mlp_params(0))
    fr.set_field(torch.from_numpy(f_t).to(DEV))
    fr.set_weights(p_t)
    fr.set_background(target_map.to(DEV).contiguous())
    o, d = view_rays(rays, seed)
    oh, dh = view_rays(rays, seed + 1000)
    o, d, oh, dh = (torch.from_numpy(x).to(DEV) for x in (o, d, oh, dh))
    with torch.no_grad():
        target, target_h = fr.render(o, d, st)["rgb"].clone(), fr.render(oh, dh, st)["rgb"].clone()
    field = torch.from_numpy(syn.random_field(len(V), 64, seed=seed + 3)).to(DEV).mul_(0.1).requires_grad_(True)
    params = {k: v.to(DEV).clone().requires_grad_(True) for k, v in orc.init_mlp_params(seed + 1).items()}
    bg = torch.ones((H, 2 * H, 3), device=DEV, requires_grad=learn_map)
    fr.set_background(bg.detach() if learn_map else None)
    opt = torch.optim.Adam([field, *params.values()] + ([bg] if learn_map else []), lr=lr)

    def held_out():
        with torch.no_grad():
            fr.set_field(field.detach().contiguous())
            fr.set_weights(params)
            out = fr.render(oh, dh, st)
        err = ((out["rgb"] - target_h) ** 2).mean(1)
        low = out["accumulation"][:, 0] < 0.5
        miss = ~out["ray_mask"]
        psnr = lambda e: float(-10 * torch.log10(e.mean().clamp_min(1e-12)))  # noqa: E731
        return {"psnr_all": psnr(err), "psnr_acc_below_half": psnr(err[low]), "miss_mse": float(err[miss].mean()),
                "share_acc_below_half": float(low.float().mean()), "share_miss": float(miss.float().mean())}

    before = held_out()
    for _ in range(steps):
        fr.set_field(field.detach().contiguous())
        fr.set_weights(params)
        extra = (bg,) if learn_map else ()
        rgb, acc, _, _ = FusedTrainRender.apply(fr, st, False, o, d, None, None, field, *[params[n] for n in PARAM_ORDER], *extra)
        loss = torch.nn.functional.mse_loss(rgb, target)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
    after = held_out()
    return {"learn_map": learn_map, "steps": steps, "H": H, **{f"{k}_before": v for k, v in before.items()},
            **{f"{k}_after": v for k, v in after.items()}}


def cost(gpu, n, warm):
    from tetranerf import cpp
    from tetranerf.b200.render import FusedRenderer, RenderSettings

    st = RenderSettings.tetra_nerf()
    bg = torch.rand((256, 512, 3), generator=torch.Generator().manual_seed(0)).to(DEV)
    for points, R, what in ((45000, 4096, "eval"), (300000, 8192, "train")):
        V, C = syn.delaunay_mesh(points, seed=0)
        tr = cpp.TetrahedraTracer(DEV)
        tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(C).to(DEV))
        fr = FusedRenderer(tr)
        fr.set_field(torch.from_numpy(syn.random_field(len(V), 64, seed=3)).to(DEV))
        fr.set_weights(orc.init_mlp_params(0))
        o, d = view_rays(R, 5)
        o, d = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
        g_rgb = torch.full((R, 3), 1e-3, device=DEV)
        for det in ((False,) if what == "eval" else (False, True)):
            for use_map in (False, True, False, True):  # alternating, twice
                fr.set_background(bg if use_map else None)
                torch.use_deterministic_algorithms(det)
                if what == "eval":
                    fn = lambda: fr.render(o, d, st)  # noqa: E731
                else:
                    def fn():
                        _, s = fr.train_forward_saved(o, d, st)
                        fr.train_backward_saved(s, g_rgb, None, len(V), grad_background=use_map)
                ms = _timed(fn, n, warm)
                torch.use_deterministic_algorithms(False)
                print(json.dumps({"arm": "cost", "what": what, "tetrahedra": len(C), "rays": R, "map": use_map, "deterministic": det,
                                  "median_ms": round(ms, 4), "gpu": gpu}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--warm", type=int, default=5)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--skip-cost", action="store_true")
    args = ap.parse_args()
    gpu = _gpu()
    if not args.skip_cost:
        cost(gpu, args.n, args.warm)
    mesh = syn.delaunay_mesh(45000, seed=0)
    target = sky_map(32)
    for learn in (False, True):
        r = train_arm(mesh, args.steps, 32, 0, 8192, learn, target)
        print(json.dumps({"arm": "quality", **{k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items()}, "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
