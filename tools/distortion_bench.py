"""Cost of the distortion loss (DESIGN §4.11) on bench.py's --mode train workload: the 300k-point mesh (~2.0 M tetrahedra), 8192 rays,
tetra_nerf settings, the model's own field initialisation, training steps (forward + get_loss_dict + backward + RAdam step) through
TetrahedraNerf with distortion_loss_mult = 0 and > 0, alternating, in the default and the deterministic mode.  Prints one JSON line per
mode with the median step times (CUDA events) and the peak device memory of each; then one line with the kernel times of k_distortion
and k_composite_bwd (torch.profiler, a run of its own), and one line with nerfstudio's O(S^2) formula in torch on the same weights (forward
+ backward time and peak memory) beside the O(S) torch form of the unfused path.  Every line carries the card, its power limit and
clocks, read in the same run.  Needs a GPU."""
from __future__ import annotations

import argparse
import json
import os
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
from tetranerf.nerfstudio import model as tnm  # noqa: E402


def ns_distortion(weights, sdist):
    """nerfstudio 0.3.x losses.distortion_loss per ray, as written there: the [R, S, S] pairwise form"""
    midpoints = (sdist[..., 1:] + sdist[..., :-1]) / 2
    dut = torch.abs(midpoints[..., :, None] - midpoints[..., None, :])
    w = weights[..., 0]
    loss_inter = torch.sum(w[..., :, None] * w[..., None, :] * dut, dim=(-1, -2))
    loss_intra = torch.sum(w**2 * (sdist[..., 1:] - sdist[..., :-1]), dim=-1) / 3
    return loss_inter + loss_intra


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--points", type=int, default=300000)
    ap.add_argument("--mult", type=float, default=0.01)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("distortion_bench needs a GPU")
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    V, C = syn.delaunay_mesh(a.points, seed=0)
    field = syn.random_field(len(V), 64, seed=3, kind="init")
    params = orc.init_mlp_params(0)
    R = a.rays
    o, d = syn.camera_rays(R, seed=5000)
    o, d = torch.from_numpy(o).to(dev), torch.from_numpy(d).to(dev)
    target = torch.from_numpy(np.random.default_rng(9000).random((R, 3), dtype=np.float32)).to(dev)
    os.environ["TETRANERF_B200_UNFUSED_TRAIN"] = "0"

    def make(mult):
        cfg = tnm.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), num_samples=128, num_fine_samples=128,
                                       use_biased_sampler=True, distortion_loss_mult=mult)
        m = tnm.TetrahedraNerf(cfg)
        sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C), "tetrahedra_field": torch.from_numpy(field)}
        sd.update(params)
        m.load_state_dict(sd, strict=False)
        m = m.to(dev).train()
        opt = torch.optim.RAdam(m.parameters(), lr=1e-3)
        init = [p.detach().clone() for p in m.parameters()]

        def step():
            with torch.no_grad():  # every step from the same state, as bench.py
                for p, p0 in zip(m.parameters(), init):
                    p.copy_(p0)
            opt.state.clear()
            out = m(tnm.RayBundle(origins=o, directions=d))
            loss = sum(m.get_loss_dict(out, {"image": target}).values())
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            return out

        return m, step

    models = {0.0: make(0.0), a.mult: make(a.mult)}
    for mode in ("default", "deterministic"):
        torch.use_deterministic_algorithms(mode == "deterministic")
        times = {k: [] for k in models}
        peak = {}
        for it in range(a.warmup + a.iters):
            for k, (_, step) in models.items():
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats(dev)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                step()
                e1.record()
                e1.synchronize()
                peak[k] = max(peak.get(k, 0), torch.cuda.max_memory_allocated(dev))
                if it >= a.warmup:
                    times[k].append(e0.elapsed_time(e1))
        torch.use_deterministic_algorithms(False)
        t0, t1 = float(np.median(times[0.0])), float(np.median(times[a.mult]))
        print(json.dumps({"case": "train_step", "mode": mode, "rays": R, "tetrahedra": len(C), "step_ms_mult0": round(t0, 3),
                          f"step_ms_mult{a.mult}": round(t1, 3), "extra_ms": round(t1 - t0, 3),
                          "step_ms_spread_mult0": [round(float(np.min(times[0.0])), 3), round(float(np.max(times[0.0])), 3)],
                          f"step_ms_spread_mult{a.mult}": [round(float(np.min(times[a.mult])), 3), round(float(np.max(times[a.mult])), 3)],
                          "peak_mem_gb_mult0": round(peak[0.0] / 1e9, 3), f"peak_mem_gb_mult{a.mult}": round(peak[a.mult] / 1e9, 3),
                          "gpu": gpu}), flush=True)

    # kernel times: torch.profiler over a few steps with the distortion, default mode
    from torch.profiler import ProfilerActivity, profile

    _, step = models[a.mult]
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            step()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        for name in ("k_distortion", "k_composite_bwd"):
            if name in ev.key:
                t = kern.setdefault(name, [0.0, 0])
                t[0] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
                t[1] += ev.count
    print(json.dumps({"case": "kernels", "mode": "default", "rays": R,
                      **{f"{n}_us": round(t[0] / max(t[1], 1), 2) for n, t in kern.items()},
                      **{f"{n}_calls": t[1] for n, t in kern.items()}, "gpu": gpu}), flush=True)

    # nerfstudio's O(S^2) formula against the O(S) form, on the weights and spacing bins of one fused training forward
    m, _ = models[a.mult]
    fr = m._fused_renderer()
    from tetranerf.b200.render import RenderSettings

    st = RenderSettings(512, 128, 128, True, float(m.collider.far_plane), (1.0, 1.0, 1.0))
    with torch.no_grad():
        out, state = fr.train_forward_saved(o, d, st)
        d_kernel = fr.train_distortion(state)
    S2 = st.num_samples + st.num_fine_samples + 1
    blob, off = state.blob, [256]

    def take(nbytes):  # the layout of saved_layout in tn_render.cu: 256-byte aligned arrays after the header
        t = blob[off[0]:off[0] + nbytes]
        off[0] += (nbytes + 255) // 256 * 256
        return t

    n = int(take(16).view(torch.int32)[0])
    ray_list = take(4 * R).view(torch.int32)[:n].long()
    eb = take(4 * R * (S2 + 1)).view(torch.float32).view(R, S2 + 1)[:n]
    sb = take(4 * R * (S2 + 1)).view(torch.float32).view(R, S2 + 1)[:n]
    take(16 * R * S2)
    take(12 * R * S2)
    sig = take(16 * R * S2).view(torch.float32).view(R, S2, 4)[:n, :, 0]
    x = (eb[:, 1:] - eb[:, :-1]) * sig
    weights = torch.nan_to_num((1 - torch.exp(-x)) * torch.exp(-(torch.cumsum(x, -1) - x)))[..., None].contiguous()
    sdist = sb.contiguous()
    res = {"case": "formula", "rays": n, "samples_per_ray": S2}
    for name, fn in (("nerfstudio_O(S^2)", ns_distortion), ("prefix_sum_O(S)", lambda w, s: tnm.distortion_per_ray(w, s)[..., 0])):
        ts = []
        for it in range(a.warmup + a.iters):
            w = weights.clone().requires_grad_(True)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            base = torch.cuda.memory_allocated(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            val = fn(w, sdist)
            val.sum().backward()
            e1.record()
            e1.synchronize()
            if it >= a.warmup:
                ts.append(e0.elapsed_time(e1))
        res[f"{name}_fwd_bwd_ms"] = round(float(np.median(ts)), 3)
        res[f"{name}_peak_extra_gb"] = round((torch.cuda.max_memory_allocated(dev) - base) / 1e9, 3)
        got = torch.zeros(R, device=dev).index_copy(0, ray_list, val.detach().float())
        res[f"{name}_max_rel_diff_to_kernel"] = float(((got - d_kernel[:, 0]).abs().max() / d_kernel.abs().max()).item())
    res["gpu"] = gpu
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
