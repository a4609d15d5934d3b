"""Cost and gain of the field smoothness loss (DESIGN §4.15).  Needs a GPU.  Every JSON line carries the card and its power limit, read
in the same run.
  (a) on Delaunay meshes of 45k and 300k points (301,875 and 2,020,866 tetrahedra): the vertex adjacency's build time (the first call
      after a load; median over reloads) and the device bytes it keeps; the median time of one loss-and-gradient call (CUDA events)
      against the torch edge-list formulation (gather, square, sum, autograd backward with index_add) and that one's peak torch memory;
  (b) the median time of an 8192-ray fused training step (forward + losses + backward + RAdam step, CUDA events) on the 2.02 M
      tetrahedra mesh, without and with the loss, in the default and the deterministic mode;
  (c) quality from sparse supervision: surface_scene rendered on a 45k-point mesh is the target; the field alone (MLP held fixed) is
      trained with RAdam on that same dense mesh from a U(-1e-4, 1e-4) start, on a few thousand fixed training rays; held-out PSNR for
      each field_smoothness_mult."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
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


def _model(V, Cc, field, params, **cfg):
    from tetranerf.nerfstudio import model as M

    config = M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(Cc), **cfg)
    m = M.TetrahedraNerf(config)
    sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(Cc), "tetrahedra_field": torch.from_numpy(field)}
    sd.update(params)
    m.load_state_dict(sd, strict=False)
    return m.to(DEV), M


def _train_step(m, M, opt, bundle, image):
    opt.zero_grad(set_to_none=True)
    loss = sum(m.get_loss_dict(m(bundle), {"image": image}).values())
    loss.backward()
    opt.step()


def _torch_edges(cells):
    """the unique undirected edges of the cells on the device -> (i, j) int64[E] each"""
    c = cells.long()
    a = torch.cat([c[:, i] for i, j in ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))])
    b = torch.cat([c[:, j] for i, j in ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))])
    key = torch.unique(torch.minimum(a, b) * (1 << 32) + torch.maximum(a, b))
    return key >> 32, key & 0xFFFFFFFF


def kernel_cost(points, gpu):
    from tetranerf import cpp
    from tetranerf.b200.render import FusedRenderer

    V, Cc = syn.delaunay_mesh(points, seed=0)
    xyz, cells = torch.from_numpy(V).to(DEV), torch.from_numpy(Cc).to(DEV)
    field = torch.from_numpy(syn.random_field(len(V), 64, seed=3)).to(DEV)
    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(xyz, cells)
    fr = FusedRenderer(tr)
    fr.set_field(field)
    torch.cuda.synchronize()
    before = cpp._lib.tn_debug_device_bytes()
    fr.field_smoothness(1.0)
    kept = cpp._lib.tn_debug_device_bytes() - before
    builds = []
    for _ in range(5):  # the first call after each load builds the adjacency (and synchronises)
        tr.load_tetrahedra(xyz, cells)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fr.field_smoothness(1.0)
        torch.cuda.synchronize()
        builds.append((time.perf_counter() - t0) * 1e3)
    t_build = float(np.median(builds))
    t_fused = _timed(lambda: fr.field_smoothness(1.0, grad=True), 50, 5)
    _, E, _ = fr.field_smoothness(1.0)
    i, j = _torch_edges(cells)
    assert len(i) == E
    f = field.clone().requires_grad_(True)

    def edge_list():
        f.grad = None
        d = f[:, i] - f[:, j]
        ((d * d).sum() * (1.0 / (E * 64))).backward()

    edge_list()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t_torch = _timed(edge_list, 20, 3)
    peak = torch.cuda.max_memory_allocated() - base
    print(json.dumps({"bench": "field_smoothness_kernel", "gpu": gpu, "tetrahedra": len(Cc), "vertices": len(V), "edges": E,
                      "csr_build_ms": round(t_build, 3), "csr_bytes": int(kept), "loss_and_grad_ms": round(t_fused, 4),
                      "torch_edge_list_ms": round(t_torch, 3), "torch_edge_list_peak_MB": round(peak / 1e6, 1),
                      "speedup": round(t_torch / t_fused, 2)}), flush=True)


def train_step_cost(points, gpu):
    V, Cc = syn.delaunay_mesh(points, seed=0)
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    o, d = syn.camera_rays(8192, seed=3)
    image = torch.rand((8192, 3), generator=torch.Generator().manual_seed(1)).to(DEV)
    res = {}
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        try:
            for mult in (0.0, 1.0):
                m, M = _model(V, Cc, field, params, num_samples=128, num_fine_samples=128, use_biased_sampler=True, field_smoothness_mult=mult)
                bundle = M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV))
                opt = torch.optim.RAdam(list(m.parameters()), lr=1e-3)
                m.train()
                res[f"{'deterministic' if det else 'default'}_{'with' if mult else 'without'}_ms"] = round(
                    _timed(lambda: _train_step(m, M, opt, bundle, image), 10, 3), 3)
                del m, opt
                torch.cuda.empty_cache()
        finally:
            torch.use_deterministic_algorithms(False)
    print(json.dumps({"bench": "field_smoothness_train_step", "gpu": gpu, "tetrahedra": len(Cc), "rays": 8192, "num_samples": 128,
                      "num_fine_samples": 128, **res}), flush=True)


def quality(gpu, steps, mults, train_rays):
    from tetranerf import cpp
    from tetranerf.b200.render import FusedRenderer, RenderSettings

    V, Cc = syn.delaunay_mesh(45_000, seed=0)
    ft, params = syn.surface_scene(V, 100, orc.init_mlp_params(0), noise=0.0)
    st = RenderSettings(num_samples=64, num_fine_samples=64)
    tr = cpp.TetrahedraTracer(DEV)
    tr.load_tetrahedra(torch.from_numpy(V).to(DEV), torch.from_numpy(Cc).to(DEV))
    fr = FusedRenderer(tr)
    fr.set_field(torch.from_numpy(ft).to(DEV))
    fr.set_weights(params)
    fr.set_mlp_precision(3)

    def rays(n, seed):
        o, d = syn.camera_rays(n, seed=seed)
        o, d = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
        return o, d, fr.render(o, d, st)["rgb"].clone()

    batch = 1024
    train = [rays(batch, 100 + k) for k in range(max(1, train_rays // batch))]
    held = rays(16384, 7)
    f0 = np.random.default_rng(0).uniform(-1e-4, 1e-4, (64, len(V))).astype(np.float32)
    arms = {}
    t0 = time.perf_counter()
    for mult in mults:
        torch.manual_seed(0)
        m, M = _model(V, Cc, f0, params, num_samples=64, num_fine_samples=64, field_smoothness_mult=mult)
        for n, p in m.named_parameters():
            p.requires_grad_(n == "tetrahedra_field")
        opt = torch.optim.RAdam([m.tetrahedra_field], lr=1e-2)
        m.train()
        for s in range(steps):
            o, d, img = train[s % len(train)]
            _train_step(m, M, opt, M.RayBundle(origins=o, directions=d), img)
        m.eval()
        with torch.no_grad():
            got = m(M.RayBundle(origins=held[0], directions=held[1]))["rgb"]
        arms[str(mult)] = round(float(10 * torch.log10(1.0 / torch.mean((got - held[2]) ** 2))), 3)
    print(json.dumps({"bench": "field_smoothness_quality", "gpu": gpu, "vertices": len(V), "tetrahedra": len(Cc), "steps": steps,
                      "train_rays": len(train) * batch, "heldout_rays": 16384, "psnr_by_mult": arms,
                      "seconds": round(time.perf_counter() - t0, 1)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="*", default=[45_000, 300_000])
    ap.add_argument("--train-points", type=int, default=300_000)
    ap.add_argument("--quality-steps", type=int, default=1500)
    ap.add_argument("--quality-mults", type=float, nargs="*", default=[0.0, 1.0, 10.0, 100.0])
    ap.add_argument("--train-rays", type=int, default=4096)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("field_smoothness_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    for n in a.points:
        kernel_cost(n, gpu)
    if a.train_points > 0:
        train_step_cost(a.train_points, gpu)
    if a.quality_steps > 0:
        quality(gpu, a.quality_steps, a.quality_mults, a.train_rays)


if __name__ == "__main__":
    main()
