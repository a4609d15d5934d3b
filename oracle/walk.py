"""CPU restatement of the trace's adjacency walk (csrc/tn_walk.cu, k_walk) -- TEST INFRASTRUCTURE ONLY.

The walk's control flow in numpy, all rays in lockstep, with the fp32 triangle test of the oracle library (bit-exact with the kernels):
  * hull entry: the smallest (t bits, face id) key over the hull faces and the number of hull hits; a ray that hits no hull face misses
    the mesh (no records), one with a hull-hit count other than two goes to the exact stage;
  * step loop: from the entry face, the three other faces of the tetrahedron in their stored windings; zero or several exit faces send the
    ray to the exact stage, one is the next entry face.  A step with t_out <= t_in, or two crossings shorter than eps in a row, make the
    ray non-generic; a generic ray writes one record per crossing of at least eps; the hit cap (M - 1 faces) sends it to the exact stage;
  * routes: GENERIC rays keep the walk's own records, KEYS rays (non-generic) the pairing of the walk's (t, face) keys by the oracle's
    sort + post-process, EXACT rays the oracle's all-hits trace.

What the walk cannot do is see a face its chain of tetrahedra never reaches.  Comparing `walk_trace` with `OracleMesh.trace_rays` on a
mesh therefore measures exactly that: on a mesh whose every line crossing lies on the chain from the hull entry, the two are equal.
"""
from __future__ import annotations

from typing import Dict

import numpy as np

from oracle import oracle as orc
from oracle.vertex_grads import face_tables

GENERIC, KEYS, EXACT, MISS = 0, 1, 2, 3
ROUTES = ("generic", "keys", "exact", "miss")
EPS = np.float32(1e-6)  # TN_EPS
EMPTY = -1


class WalkTables:
    """the tables of a walkable load, in the reference's face numbering: tri [F,3] (stored windings), tt [F,2], the face id of every slot
    slot_face [T,4] (slot j = the face opposite local vertex j) and the neighbour across it nbr [T,4] (-1 = hull)"""

    def __init__(self, cells):
        c = np.asarray(cells, dtype=np.int64)
        self.tri, self.tt = face_tables(c)
        T = len(c)
        key = np.sort(np.stack([c[:, [(j + 1) % 4, (j + 2) % 4, (j + 3) % 4]] for j in range(4)], 1), -1).reshape(-1, 3)
        fkey = np.sort(self.tri, -1)
        # face id of every slot: look the sorted triple up among the sorted face triples
        order = np.lexsort((fkey[:, 2], fkey[:, 1], fkey[:, 0]))
        sk = fkey[order]
        pos = np.searchsorted(_pack(sk), _pack(key))
        self.slot_face = order[pos].reshape(T, 4)
        assert np.array_equal(np.sort(self.tri[self.slot_face.reshape(-1)], -1), key)
        owners = self.tt[self.slot_face]  # [T,4,2]
        me = np.arange(T)[:, None]
        self.nbr = np.where(owners[..., 0] == me, owners[..., 1], owners[..., 0])
        self.hull_faces = np.nonzero(self.tt[:, 1] < 0)[0]


def _pack(k):
    k = np.asarray(k, dtype=np.int64)
    return (k[:, 0] << 42) | (k[:, 1] << 21) | k[:, 2]


def _keys(t, face):
    return (np.asarray(t, np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.asarray(face).astype(np.uint64)


def walk_trace(xyz, cells, origins, directions, M: int, tables: WalkTables = None, mesh: orc.OracleMesh = None,
               nthreads: int = 0, walk_one_hull_hit: bool = False) -> Dict[str, np.ndarray]:
    """-> the trace_rays dictionary the walk path produces (OracleMesh.trace_rays' keys, dense tails as the tracer writes them) plus
    "route" i32[R] (GENERIC / KEYS / EXACT / MISS) and "hull_hits" i32[R].  walk_one_hull_hit: rays with a single hull hit walk instead of
    going to the exact stage at once (the `hullhits > 2` form of the hull-hit test)"""
    X = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
    o = np.ascontiguousarray(origins, dtype=np.float32).reshape(-1, 3)
    d = np.ascontiguousarray(directions, dtype=np.float32).reshape(-1, 3)
    R = len(o)
    tb = tables if tables is not None else WalkTables(cells)
    tri, slot_face, nbr = tb.tri, tb.slot_face, tb.nbr

    # ---- hull entry ----
    HF = tb.hull_faces
    best = np.full(R, np.iinfo(np.uint64).max, np.uint64)
    bu, bv = np.zeros(R, np.float32), np.zeros(R, np.float32)
    hull_hits = np.zeros(R, np.int64)
    chunk = max(1, (1 << 21) // max(len(HF), 1))
    for r0 in range(0, R, chunk):
        rr = np.arange(r0, min(R, r0 + chunk))
        ray = np.repeat(rr, len(HF))
        f = np.tile(HF, len(rr))
        hit, tuv = orc.ray_tri_pairs(X, o, d, ray, tri[f], nthreads)
        ray, f, tuv = ray[hit], f[hit], tuv[hit]
        np.add.at(hull_hits, ray, 1)
        k = _keys(tuv[:, 0], f)
        srt = np.lexsort((k, ray))
        ray, k, tuv = ray[srt], k[srt], tuv[srt]
        first = np.ones(len(ray), bool)
        first[1:] = ray[1:] != ray[:-1]
        best[ray[first]] = k[first]
        bu[ray[first]], bv[ray[first]] = tuv[first, 1], tuv[first, 2]
    route = np.full(R, MISS, np.int32)
    walking = (hull_hits == 2) | (walk_one_hull_hit & (hull_hits == 1))
    route[(hull_hits > 0) & ~walking] = EXACT
    route[walking] = GENERIC

    # ---- walk, all live rays in lockstep ----
    fin = (best & np.uint64(0xFFFFFFFF)).astype(np.int64)
    t_in = (best >> np.uint64(32)).astype(np.uint32).view(np.float32)
    u_in, v_in = bu.copy(), bv.copy()
    c = np.where(walking, tb.tt[np.where(walking, fin, 0), 0], -1)  # a hull face's only owner
    generic = walking.copy()
    prev_small = np.zeros(R, bool)
    nfaces = np.where(walking, 1, 0)
    nrec = np.zeros(R, np.int64)
    kt = np.zeros((R, M), np.float32)  # the walk's keys (t, face) and the (u, v) of each crossing, in walk order
    kf = np.zeros((R, M), np.int64)
    kuv = np.zeros((R, M, 2), np.float32)
    kt[:, 0], kf[:, 0], kuv[:, 0, 0], kuv[:, 0, 1] = t_in, fin, bu, bv
    num = np.zeros(R, np.int32)
    cells_out = np.full((R, M), EMPTY, np.int32)
    bary = np.zeros((R, M, 2, 3), np.float32)
    dist = np.zeros((R, M, 2), np.float32)
    verts = np.full((R, M, 4), EMPTY, np.int32)
    one = np.float32(1.0)
    while walking.any():
        rays = np.nonzero(walking)[0]
        cr = c[rays]
        sf = slot_face[cr]  # [n,4]
        jin = np.full(len(rays), 3)
        for j in (2, 1, 0):  # the first slot holding the entry face (k_walk: 0, then 1, then 2, else 3)
            jin = np.where(sf[:, j] == fin[rays], j, jin)
        ray = np.repeat(rays, 4)
        hit, tuv = orc.ray_tri_pairs(X, o, d, ray, tri[sf.reshape(-1)], nthreads)
        hit = hit.reshape(-1, 4) & (np.arange(4)[None, :] != jin[:, None])
        tuv = tuv.reshape(-1, 4, 3)
        hits = hit.sum(1)
        jout = 3 - np.argmax(hit[:, ::-1], 1)  # the last hit slot (k_walk keeps the last one; irrelevant unless hits == 1)
        stop_exact = hits != 1
        route[rays[stop_exact]] = EXACT
        walking[rays[stop_exact]] = False
        ok = ~stop_exact
        rays, cr, jout, sf, tuv = rays[ok], cr[ok], jout[ok], sf[ok], tuv[ok]
        n = np.arange(len(rays))
        t_out, u_out, v_out = tuv[n, jout, 0], tuv[n, jout, 1], tuv[n, jout, 2]
        fout = sf[n, jout]
        small = np.abs(t_out - t_in[rays]) < EPS
        generic[rays] &= (t_out > t_in[rays]) & ~(small & prev_small[rays])
        prev_small[rays] = small
        rec = generic[rays] & ~small
        # record: combine_indices of (entry face, exit face), the oracle's layout
        i = np.nonzero(rec)[0]
        r, g = rays[i], nrec[rays[i]]
        e, x = tri[fin[r]], tri[fout[i]]
        r2 = np.stack([(one - u_out[i]) - v_out[i], u_out[i], v_out[i]], 1)
        match = e[:, None, :] == x[:, :, None]  # [n, exit vertex q, entry vertex m]
        o2 = np.zeros((len(i), 3), np.float32)
        for q in range(3):
            for m in range(3):
                o2[:, m] = np.where(match[:, q, m], r2[:, q], o2[:, m])
        lone = x[np.arange(len(i)), np.argmax(~match.any(2), 1)]
        cells_out[r, g] = cr[i]
        verts[r, g] = np.stack([lone, e[:, 0], e[:, 1], e[:, 2]], 1)
        bary[r, g, 0] = np.stack([(one - u_in[r]) - v_in[r], u_in[r], v_in[r]], 1)
        bary[r, g, 1] = o2
        dist[r, g] = np.stack([t_in[r], t_out[i]], 1)
        nrec[r] += 1
        kt[rays, nfaces[rays]], kf[rays, nfaces[rays]] = t_out, fout
        kuv[rays, nfaces[rays]] = np.stack([u_out, v_out], 1)
        nfaces[rays] += 1
        nxt = nbr[cr, jout]
        left = nxt < 0
        walking[rays[left]] = False
        capped = ~left & (nfaces[rays] >= M - 1)
        route[rays[capped]] = EXACT
        walking[rays[capped]] = False
        go = ~left & ~capped
        gr = rays[go]
        c[gr], fin[gr] = nxt[go], fout[go]
        t_in[gr], u_in[gr], v_in[gr] = t_out[go], u_out[go], v_out[go]
    route[(route == GENERIC) & ~generic] = KEYS

    # ---- finish: generic rays keep their records, the others go through the oracle ----
    num[route == GENERIC] = nrec[route == GENERIC]
    if mesh is None:
        mesh = orc.OracleMesh(X, cells)
    for r in np.nonzero(route == KEYS)[0]:
        k = nfaces[r]
        n, cc, b, dd, vv = mesh.post_process_one(kf[r, :k], kt[r, :k], kuv[r, :k], M)
        num[r], cells_out[r], bary[r], dist[r], verts[r] = n, cc, b, dd, vv
    ex = np.nonzero(route == EXACT)[0]
    if len(ex):
        ref = mesh.trace_rays(o[ex], d[ex], M, nthreads=nthreads)
        num[ex], cells_out[ex], bary[ex] = ref["num_visited_cells"], ref["visited_cells"], ref["barycentric_coordinates"]
        dist[ex], verts[ex] = ref["hit_distances"], ref["vertex_indices"]
    return {"num_visited_cells": num, "visited_cells": cells_out, "barycentric_coordinates": bary, "vertex_indices": verts,
            "hit_distances": dist, "route": route, "hull_hits": hull_hits.astype(np.int32)}


def differing_rays(a: Dict[str, np.ndarray], b: Dict[str, np.ndarray]) -> np.ndarray:
    """ray ids on which two trace_rays dictionaries differ in any bit"""
    bad = np.zeros(len(a["num_visited_cells"]), bool)
    for k in ("num_visited_cells", "visited_cells", "barycentric_coordinates", "vertex_indices", "hit_distances"):
        x, y = np.asarray(a[k]), np.asarray(b[k])
        x, y = x.view(np.uint32).reshape(len(bad), -1), y.view(np.uint32).reshape(len(bad), -1)
        bad |= (x != y).any(1)
    return np.nonzero(bad)[0]
