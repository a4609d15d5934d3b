"""Oracle of occupancy sampling on the fused paths -- TEST INFRASTRUCTURE ONLY.

Definition (DESIGN.md §4.13).  A trace record k of a ray (t_in_k, t_out_k, cell_k) is *skipped* when cell_k is a tetrahedron with
occ[cell_k] < threshold (exactly the records whose matched samples occupancy culling culls), *kept* otherwise -- gap records (cell = -1)
included.  With both kinds on a ray, its coarse bin edges are placed in the kept records only:
  * biased sampler: map_from_real_distances_to_biased_with_bounds over the kept records -- u = (e - near) / (far - near) of today's
    euclidean edge e, i = min(floor(u n_kept), n_kept - 1), frac = u n_kept - i, edge = t_in + len frac of the i-th kept record;
  * uniform sampler: x = b L with L the total kept length and b today's spacing edge; the last kept record i whose kept-length prefix
    P_i is <= x; edge = t_in + (x - P_i).
Each edge is clamped to its record's t_out (rounding never leaves the record), the edges take a running maximum (sorted bins), and the
spacing bins are (edge - near) / (far - near) with near / far over ALL records.  A ray with no skipped or no kept record keeps today's bins.

`place_coarse_bins` restates the kernel's float32 arithmetic (its prefix sum in the warp-scan order of `smem_scan_add`).  `render` /
`render_train` are oracle/occupancy.py's culled render / training render with these coarse bins."""
from __future__ import annotations

import contextlib

import numpy as np
import torch

from . import occupancy as ocu
from . import oracle as orc

_today_coarse_bins = orc.coarse_bins  # (placed() patches orc.coarse_bins)


def kept_records(num_visited, visited_cells, occ, threshold) -> np.ndarray:
    """bool [R, M]: record k < num_visited[r] of ray r is kept (not in a tetrahedron with occ < threshold)"""
    num = np.asarray(num_visited).astype(np.int64)
    cells = np.asarray(visited_cells).view(np.int32).astype(np.int64)
    occ = np.asarray(occ.cpu() if torch.is_tensor(occ) else occ, dtype=np.float32)
    inside = np.arange(cells.shape[1])[None, :] < num[:, None]
    tet = cells >= 0
    skipped = tet & (occ[np.where(tet, cells, 0)] < np.float32(threshold))
    return inside & ~skipped


def warp_scan_add(a: np.ndarray) -> np.ndarray:
    """inclusive float32 prefix sum along the last axis in the order of smem_scan_add: a Hillis-Steele scan per 32-element chunk,
    plus the running carry of the chunks before"""
    a = np.asarray(a, dtype=np.float32)
    out = np.empty_like(a)
    carry = np.zeros(a.shape[:-1], np.float32)
    for base in range(0, a.shape[-1], 32):
        v = np.zeros(a.shape[:-1] + (32,), np.float32)
        w = a[..., base:base + 32]
        v[..., :w.shape[-1]] = w
        o = 1
        while o < 32:
            nv = v.copy()
            nv[..., o:] = v[..., o:] + v[..., :-o]
            v = nv
            o <<= 1
        v = v + carry[..., None]
        out[..., base:base + 32] = v[..., :w.shape[-1]]
        carry = v[..., 31]
    return out


def place_coarse_bins(cfg, nears, fars, num_visited, hit_distances, kept, t_rand=None):
    """oracle.coarse_bins with the coarse edges of every ray that has both skipped and kept records placed in its kept records (float32,
    the kernel's arithmetic); kept bool [R, M] as kept_records.  Returns (euclidean_bins [R,S+1], spacing_bins [R,S+1])."""
    euclid, sbins = _today_coarse_bins(cfg, nears, fars, num_visited, hit_distances, t_rand)
    euclid, sbins = euclid.clone(), sbins.clone()
    S = cfg.num_samples
    b = torch.linspace(0.0, 1.0, S + 1)[None, ...]
    if t_rand is not None:  # the spacing edges before the biased mapping, as oracle.coarse_bins forms them
        centers = (b[..., 1:] + b[..., :-1]) / 2.0
        upper, lower = torch.cat([centers, b[..., -1:]], -1), torch.cat([b[..., :1], centers], -1)
        b = lower + (upper - lower) * t_rand
    b = b.expand(len(euclid), -1).numpy().astype(np.float32)
    hd = np.asarray(hit_distances, dtype=np.float32)
    num = np.asarray(num_visited).astype(np.int64)
    near_np, far_np = np.asarray(nears, np.float32)[:, 0], np.asarray(fars, np.float32)[:, 0]
    for r in range(len(euclid)):
        n = int(num[r])
        idx = np.nonzero(kept[r, :n])[0]
        nk = len(idx)
        if nk == 0 or nk == n:
            continue
        near, far = near_np[r], far_np[r]
        t_in, t_out = hd[r, idx, 0], hd[r, idx, 1]
        length = np.maximum(t_out - t_in, np.float32(0))
        br = b[r]
        if cfg.use_biased_sampler:
            uni = (br * far + (np.float32(1) - br) * near - near) / (far - near)
            rest = uni * np.float32(nk)
            iv = np.maximum(np.minimum(np.floor(rest), np.float32(nk - 1)), np.float32(0))
            rest = rest - iv
            i = iv.astype(np.int64)
            off = length[i] * rest
        else:
            cum = warp_scan_add(np.concatenate([[np.float32(0)], length]).astype(np.float32))
            x = br * cum[nk]
            # last i in [0, nk) with cum[i] <= x (cum[0] = 0 <= x)
            i = np.searchsorted(cum[1:nk], x, side="right")
            off = x - cum[i]
        e = np.minimum(t_in[i] + off, np.maximum(t_in[i], t_out[i])).astype(np.float32)
        e = np.maximum.accumulate(e)
        euclid[r] = torch.from_numpy(e)
        sbins[r] = torch.from_numpy((e - near) / (far - near))
    return euclid, sbins


@contextlib.contextmanager
def placed(mesh, origins, directions, cfg, occupancy, nthreads: int = 0):
    """inside: oracle.coarse_bins places the bins of the (non-empty, in ray order) rays of this batch by `occupancy` = (occ, threshold)"""
    o = np.asarray(origins, np.float32).reshape(-1, 3)
    d = np.asarray(directions, np.float32).reshape(-1, 3)
    tr = mesh.trace_rays(o, d, cfg.max_intersected_triangles, nthreads=nthreads)
    m = tr["num_visited_cells"] > 0
    kept = kept_records(tr["num_visited_cells"][m], tr["visited_cells"][m], *occupancy)
    orc.coarse_bins = lambda cfg_, nears, fars, nv, hd, t_rand=None: place_coarse_bins(cfg_, nears, fars, nv, hd, kept, t_rand)
    try:
        yield kept
    finally:
        orc.coarse_bins = _today_coarse_bins


def render(mesh, field, params, origins, directions, cfg, occupancy, nthreads: int = 0):
    """oracle/occupancy.render (culling by `occupancy` = (occ, threshold)) with the placed coarse bins; aux as there plus "kept"."""
    with placed(mesh, origins, directions, cfg, occupancy, nthreads) as kept:
        out = ocu.render(mesh, field, params, origins, directions, cfg, occupancy=occupancy, nthreads=nthreads)
    out["aux"]["kept"] = kept
    return out


def render_train(mesh, field, params, origins, directions, cfg, jitter_coarse=None, jitter_fine=None, use_gradient_scaling: bool = False,
                 occupancy=None, fine_euclid=None, nthreads: int = 0):
    """oracle/occupancy.render_train with the placed coarse bins (differentiable; the bins are constants)."""
    with placed(mesh, origins, directions, cfg, occupancy, nthreads):
        return ocu.render_train(mesh, field, params, origins, directions, cfg, jitter_coarse, jitter_fine,
                                use_gradient_scaling=use_gradient_scaling, occupancy=occupancy, fine_euclid=fine_euclid, nthreads=nthreads)
