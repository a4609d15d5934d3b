"""Cost and effect of the fold guard of a vertex step (TetrahedraTracer.guard_vertex_step, DESIGN §4.17).  Prints JSON lines:
  * "guard": its time (median over --iters calls, CUDA events around the synchronous call), rounds and limited / frozen vertices on the
    45k- and 300k-point Delaunay meshes (0.30 M and 2.02 M tetrahedra), for a step that folds nothing (a 1 % affine motion), a smooth one
    of 0.1 median edge lengths (folds some faces) and independent noise of 0.15 edge lengths (folds thousands), with the faces each folds
    unguarded;
  * "train_step": bench.py --mode train's workload (8192 rays, 2.02 M tetrahedra, tetra_nerf settings, a random field) trained in its
    vertices with Adam, one line per --train-lr: forward + backward with the vertex gradient + step + refit, without and with the guard
    before the refit, two tracers, alternating which runs first.  Quartiles of the step times, of the paired per-iteration difference and
    of the guard call timed on its own, how many timed steps each arm's refit kept the walk on, and the paired difference over the steps
    in which both arms walked: there it is the guard's own cost.  At 0.01 edge lengths the unguarded arm folds and loses the walk, and
    the difference over all steps is the net effect;
  * "aggressive": surface_scene on the 45k-point mesh, only the vertices trained through FusedTrainRender from 8 views at 64 x 64 with
    Adam at --lr edge lengths for --steps steps, from a guarded smooth displacement of 0.1 edge lengths, without and with the guard:
    the folded faces at the end, whether the walk is on, trace time at 8192 and 65,536 rays, and the PSNR of 4 held-out views against
    the render at the true positions.
with the card and its power limit.  Needs a GPU."""
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
from tetranerf import cpp  # noqa: E402
from tetranerf.b200 import synthetic as syn  # noqa: E402
from tetranerf.b200.render import PARAM_ORDER, FusedRenderer, FusedTrainRender, RenderSettings  # noqa: E402


def _time(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def _edge(V, C):
    return float(np.median(np.linalg.norm(V[C[:, 1]] - V[C[:, 0]], axis=-1)))


def _steps(V, edge):
    A = np.array([[1.01, 0.01, 0.0], [0.0, 0.99, 0.01], [0.01, 0.0, 1.0]])
    X = V.astype(np.float64)
    smooth = np.stack([np.sin(6.0 * X[:, 1] + 1.0), np.sin(6.0 * X[:, 2] + 2.0), np.sin(6.0 * X[:, 0] + 3.0)], -1)
    return {"none": (X @ A.T + 0.05).astype(np.float32), "some": (V + 0.1 * edge * smooth).astype(np.float32),
            "many": (V + 0.15 * edge * np.random.default_rng(3).standard_normal(V.shape)).astype(np.float32)}


def _views(dev, n, first, count, ring=1.6):
    u = torch.linspace(-0.25, 0.25, n, device=dev)
    uu, vv = torch.meshgrid(u, u, indexing="xy")
    os_, ds = [], []
    for k in range(first, first + count):
        a = 2 * np.pi * k / 8 + (0.0 if k < 8 else np.pi / 8)
        cam = torch.tensor([0.5 + ring * np.cos(a), 0.5 + ring * np.sin(a), 0.5 + 0.3 * (-1) ** k], device=dev, dtype=torch.float32)
        fwd = torch.tensor([0.5, 0.5, 0.5], device=dev) - cam
        fwd = fwd / fwd.norm()
        right = torch.linalg.cross(fwd, torch.tensor([0.0, 0.0, 1.0], device=dev))
        right = right / right.norm()
        up = torch.linalg.cross(right, fwd)
        dirs = fwd + uu.reshape(-1, 1) * right + vv.reshape(-1, 1) * up
        os_.append(cam.expand(n * n, 3))
        ds.append(dirs / dirs.norm(dim=-1, keepdim=True))
    return torch.cat(os_).contiguous(), torch.cat(ds).contiguous()


def _faces(xyz, C, dev):
    tr = cpp.TetrahedraTracer(dev)
    tr.load_tetrahedra(xyz, torch.from_numpy(C).to(dev))
    return tr.get_faces()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--lr", type=float, default=0.05, help="aggressive arm: Adam learning rate in median edge lengths")
    ap.add_argument("--train-lr", type=float, nargs="+", default=[1e-5, 0.01],
                    help="train_step: Adam learning rates in median edge lengths, one JSON line each")
    ap.add_argument("--skip", default="", help="comma-separated parts to skip: guard, train_step, aggressive")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vertex_fold_guard_bench needs a GPU")
    skip = set(filter(None, a.skip.split(",")))
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    meshes = {n: syn.delaunay_mesh(n, seed=0) for n in (45_000, 300_000)}

    if "guard" not in skip:
        for npts, (V, C) in meshes.items():
            edge = _edge(V, C)
            tr = cpp.TetrahedraTracer(dev)
            xyz, cells = torch.from_numpy(V).to(dev), torch.from_numpy(C).to(dev)
            tr.load_tetrahedra(xyz, cells)
            for kind, P in _steps(V, edge).items():
                P1 = torch.from_numpy(P).to(dev)
                unguarded, _ = tr.update_vertices(P1)
                tr.update_vertices(xyz)
                new = P1.clone()
                ts, counts = [], None
                for it in range(a.warmup + a.iters):
                    new.copy_(P1)
                    torch.cuda.synchronize()
                    t = _time(lambda: tr.guard_vertex_step(xyz, new))
                    counts = tr.guard_vertex_step(xyz, new.copy_(P1))
                    if it >= a.warmup:
                        ts.append(t)
                folded, walkable = tr.update_vertices(new)
                tr.update_vertices(xyz)
                print(json.dumps({"what": "guard", "tetrahedra": len(C), "step": kind, "unguarded_folded_faces": unguarded,
                                  "guard_ms": round(float(np.median(ts)), 3), "limited": counts[0], "frozen": counts[1], "rounds": counts[2],
                                  "guarded_folded_faces": folded, "walkable": walkable, "iters": a.iters, "gpu": q}), flush=True)

    if "train_step" not in skip:
        V, C = meshes[300_000]
        edge = _edge(V, C)
        st = RenderSettings.tetra_nerf()
        o, d = (torch.from_numpy(x).to(dev) for x in syn.camera_rays(a.rays, seed=5000))
        g = torch.Generator().manual_seed(9)
        jc, jf = torch.rand((a.rays, st.num_samples + 1), generator=g).to(dev), torch.rand((a.rays, st.num_fine_samples + 1), generator=g).to(dev)
        target = torch.rand((a.rays, 3), generator=g).to(dev)
        field = torch.from_numpy(syn.random_field(len(V), 64, seed=3, kind="init")).to(dev)
        for lr in a.train_lr:
            arms = {}
            for guard in (False, True):
                tr = cpp.TetrahedraTracer(dev)
                xyz = torch.nn.Parameter(torch.from_numpy(V).to(dev))
                tr.load_tetrahedra(xyz.detach(), torch.from_numpy(C).to(dev))
                fr = FusedRenderer(tr)
                fr.set_field(field)
                fr.set_weights(orc.init_mlp_params(0))
                arms[guard] = (tr, fr, xyz, xyz.detach().clone(), torch.optim.Adam([xyz], lr=lr * edge))
            log = {False: [], True: []}  # per timed step: (step ms, guard-call ms, folded faces after the refit, walk on, guard counts)

            def step(guard):
                tr, fr, xyz, prev, opt = arms[guard]
                out, state = fr.train_forward_saved(o, d, st, jc, jf)
                g_rgb = (2.0 * (out["rgb"] - target) / (3 * a.rays)).contiguous()
                *_, gv = fr.train_backward_saved(state, g_rgb, None, len(V), True, grad_vertices=True)
                xyz.grad = gv
                opt.step()
                res = {"guard_ms": 0.0, "counts": (0, 0, 0)}
                if guard:  # the guard call on its own: synchronous, so its events span its kernels and its read-backs
                    def call():
                        res["counts"] = tr.guard_vertex_step(prev, xyz.detach())
                    res["guard_ms"] = _time(call)
                res["folded"], res["walk"] = tr.update_vertices(xyz.detach())
                prev.copy_(xyz.detach())
                return res

            for it in range(a.warmup + a.iters):
                for guard in ((False, True) if it % 2 == 0 else (True, False)):  # alternate which arm runs first
                    box = {}
                    t = _time(lambda: box.update(step(guard)))
                    if it >= a.warmup:
                        log[guard].append((t, box["guard_ms"], box["folded"], box["walk"], box["counts"]))

            def q3(x):
                return [round(float(v), 3) for v in np.percentile(x, [25, 50, 75])]

            plain, guarded = np.array([r[0] for r in log[False]]), np.array([r[0] for r in log[True]])
            # the iterations in which both arms traced on the walk: there the difference is the guard alone
            both = (guarded - plain)[np.array([r[3] for r in log[False]]) & np.array([r[3] for r in log[True]])]
            print(json.dumps({"what": "train_step", "rays": a.rays, "tetrahedra": len(C), "lr_edges": lr, "iters": a.iters,
                              "step_ms_p25_p50_p75": q3(plain), "step_ms_with_guard_p25_p50_p75": q3(guarded),
                              "paired_extra_ms_p25_p50_p75": q3(guarded - plain),
                              "paired_extra_ms_both_walking_p25_p50_p75": q3(both) if len(both) else None, "steps_both_walking": len(both),
                              "guard_call_ms_p25_p50_p75": q3([r[1] for r in log[True]]),
                              "guard_rounds_max": max(r[4][2] for r in log[True]), "guard_limited_max": max(r[4][0] for r in log[True]),
                              "timed_steps_walking": sum(r[3] for r in log[False]), "timed_steps_walking_with_guard": sum(r[3] for r in log[True]),
                              "folded_faces_max": max(r[2] for r in log[False]), "folded_faces_max_with_guard": max(r[2] for r in log[True]),
                              "gpu": q}), flush=True)

    if "aggressive" not in skip:
        V, C = meshes[45_000]
        edge = _edge(V, C)
        field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
        st = RenderSettings.tetra_nerf()
        f = torch.from_numpy(field).to(dev)
        ot, dt = _views(dev, 64, 0, 8)
        oh, dh = _views(dev, 64, 8, 4)
        to, td = (torch.from_numpy(x).to(dev) for x in syn.camera_rays(65536, seed=77))
        true = torch.from_numpy(V).to(dev)
        # both arms start from the same valid displacement: a smooth 0.1 edge lengths on the interior vertices, guarded from the true positions
        X = V.astype(np.float64)
        noise = 0.1 * edge * np.stack([np.sin(6.0 * X[:, 1] + 1.0), np.sin(6.0 * X[:, 2] + 2.0), np.sin(6.0 * X[:, 0] + 3.0)], -1)
        tri, tt = (t.cpu().numpy() for t in _faces(true, C, dev))
        noise[np.unique(tri[tt[:, 1] < 0])] = 0
        start = torch.from_numpy((V + noise).astype(np.float32)).to(dev)
        g0 = cpp.TetrahedraTracer(dev)
        g0.load_tetrahedra(true, torch.from_numpy(C).to(dev))
        g0.guard_vertex_step(true, start)
        for guard in (False, True):
            tr = cpp.TetrahedraTracer(dev)
            tr.load_tetrahedra(true.clone(), torch.from_numpy(C).to(dev))
            fr = FusedRenderer(tr)
            fr.set_field(f)
            fr.set_weights(params)
            ps = [params[n].to(dev) for n in PARAM_ORDER]
            with torch.no_grad():
                target = FusedTrainRender.apply(fr, st, False, ot, dt, None, None, f, *ps)[0].clone()
                held = FusedTrainRender.apply(fr, st, False, oh, dh, None, None, f, *ps)[0].clone()
            xyz = torch.nn.Parameter(start.clone())
            tr.update_vertices(xyz.detach())
            prev = xyz.detach().clone()
            opt = torch.optim.Adam([xyz], lr=a.lr * edge)
            losses, max_rounds, warn_folds = [], 0, 0
            for _ in range(a.steps):
                opt.zero_grad()
                loss = torch.nn.functional.mse_loss(FusedTrainRender.apply(fr, st, False, ot, dt, None, None, f, *ps, xyz)[0], target)
                loss.backward()
                opt.step()
                if guard:
                    max_rounds = max(max_rounds, tr.guard_vertex_step(prev, xyz.detach())[2])
                folded, walkable = tr.update_vertices(xyz.detach())
                warn_folds = max(warn_folds, folded)
                prev.copy_(xyz.detach())
                losses.append(loss.item())
            with torch.no_grad():
                pred = FusedTrainRender.apply(fr, st, False, oh, dh, None, None, f, *ps, xyz)[0]
            mse = torch.mean((pred.clamp(0, 1) - held.clamp(0, 1)) ** 2).item()
            tt = {}
            for R in (8192, 65536):
                oo, dd = to[:R].contiguous(), td[:R].contiguous()
                ts = []
                for it in range(a.warmup + a.iters):
                    t = _time(lambda: tr.trace_rays(oo, dd, st.max_intersected_triangles))
                    if it >= a.warmup:
                        ts.append(t)
                tt[R] = round(float(np.median(ts)), 3)
            tr.synchronize()
            print(json.dumps({"what": "aggressive", "guard": guard, "tetrahedra": len(C), "steps": a.steps, "lr_edges": a.lr,
                              "train_loss_first": losses[0], "train_loss_last": losses[-1], "position_error_mean": (xyz.detach() - true).norm(dim=-1).mean().item(), "folded_faces_at_end": folded,
                              "most_folded_faces": warn_folds, "walkable": walkable, "max_guard_rounds": max_rounds,
                              "trace_ms_8192": tt[8192], "trace_ms_65536": tt[65536],
                              "heldout_psnr": round(-10.0 * float(np.log10(max(mse, 1e-20))), 3), "gpu": q}), flush=True)


if __name__ == "__main__":
    main()
