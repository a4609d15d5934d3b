"""float64 restatement of the surface extraction (tn_surface_extract, DESIGN.md §4.6) -- TEST INFRASTRUCTURE ONLY.  It never imports the
CUDA package.

The definition, on the tracer's mesh (positions x_v, tetrahedra), the field F[:, v] and a level tau > 0:
  * vertex v is inside when sigma(F[:, v]) >= tau, sigma = density_head(mlp_base(.)) (the renderer's density, no GradientScaler);
  * every mesh edge (a, b), a < b, with one end inside and one outside gives one output vertex; vertices are ordered by (a, b);
  * along the edge f(s) = (1 - s) F_a + s F_b at the point (1 - s) x_a + s x_b; the crossing is bracketed by 63 evaluations at s = i/64,
    then 63 inside the first bracket whose end differs from a's side, and placed by linear interpolation in the final 1/4096 bracket;
  * faces by marching tetrahedra (the case table of `tet_faces`), ordered by tetrahedron, normals from inside to outside;
  * vertex normals: normalised sums of the unnormalised face normals; colours: the colour head at f(s) seen along -normal.
`surface` takes the density and colour as functions, so the CPU tests can drive it with a density that is linear in the features;
`extract` is the network's.  Given `positions` / `normals` (the kernel's), colours are evaluated there instead of at its own."""
from __future__ import annotations

from typing import Callable, Dict, Optional

import numpy as np
import torch

from oracle import oracle as orc

ROUND = 64  # samples per refinement round (63 inside the bracket + its known end)


def orient(xyz, q0, q1, q2, q3) -> np.ndarray:
    """det(x_q1 - x_q0, x_q2 - x_q0, x_q3 - x_q0) in float64, in the operation order of the kernel's `orient`"""
    x = np.asarray(xyz, dtype=np.float32).astype(np.float64)
    a, b, c = x[q1] - x[q0], x[q2] - x[q0], x[q3] - x[q0]
    t1 = b[..., 1] * c[..., 2] - b[..., 2] * c[..., 1]
    t2 = b[..., 0] * c[..., 2] - b[..., 2] * c[..., 0]
    t3 = b[..., 0] * c[..., 1] - b[..., 1] * c[..., 0]
    return a[..., 0] * t1 - a[..., 1] * t2 + a[..., 2] * t3


def tet_faces(xyz, cell, inside):
    """marching tetrahedra on one tetrahedron (4 vertex ids, their inside flags) -> list of triangles, each three edges (x, y), x < y.
    With the inside ids i0 < i1 < ... and outside ids o0 < o1 < ...:
      1 inside: (i,o0), (i,o1), (i,o2)                     -- last two swapped iff det(o0-i, o1-i, o2-i) < 0
      3 inside: (i0,o), (i1,o), (i2,o)                     -- swapped iff det(i0-o, i1-o, i2-o) > 0
      2 inside: (i0,o0), (i0,o1), (i1,o1) and (i0,o0), (i1,o1), (i1,o0)   -- swapped iff det(i1-i0, o0-i0, o1-i0) < 0
    so that every normal points from the inside vertices to the outside ones."""
    v = np.sort(np.asarray(cell, dtype=np.int64))
    ins = np.asarray(inside, dtype=bool)[np.argsort(np.asarray(cell, dtype=np.int64), kind="stable")]
    I, O = [int(x) for x in v[ins]], [int(x) for x in v[~ins]]

    def e(x, y):
        return (min(x, y), max(x, y))

    if len(I) == 1:
        tris = [[e(I[0], O[0]), e(I[0], O[1]), e(I[0], O[2])]]
        flip = orient(xyz, I[0], O[0], O[1], O[2]) < 0
    elif len(I) == 3:
        tris = [[e(I[0], O[0]), e(I[1], O[0]), e(I[2], O[0])]]
        flip = orient(xyz, O[0], I[0], I[1], I[2]) > 0
    elif len(I) == 2:
        a, b, c, d = e(I[0], O[0]), e(I[0], O[1]), e(I[1], O[1]), e(I[1], O[0])
        tris = [[a, b, c], [a, c, d]]
        flip = orient(xyz, I[0], I[1], O[0], O[1]) < 0
    else:
        return []
    return [[t[0], t[2], t[1]] if flip else t for t in tris]


def crossing(sigma_along: Callable[[np.ndarray], np.ndarray], level: float, sig_a, sig_b) -> np.ndarray:
    """the crossing parameter s of E edges.  sigma_along(s f64[E, k]) -> sigma f64[E, k] on each edge; sig_a / sig_b the endpoint
    densities.  Two rounds: 63 evaluations inside the current bracket (s0 + i step, step 1/64 then 1/4096), the new bracket ends at the
    smallest i whose side differs from a's; then linear interpolation in the last bracket."""
    sig_a, sig_b = np.asarray(sig_a, np.float64), np.asarray(sig_b, np.float64)
    E = len(sig_a)
    ins_a = sig_a >= level
    s0, lo, hi = np.zeros(E), sig_a.copy(), sig_b.copy()
    r = np.arange(E)
    for step in (1.0 / ROUND, 1.0 / ROUND**2):
        s = s0[:, None] + np.arange(1, ROUND) * step
        full = np.concatenate([lo[:, None], sigma_along(s), hi[:, None]], axis=1)  # samples 0..64
        flip = (full[:, 1:] >= level) != ins_a[:, None]
        i = np.argmax(flip, axis=1) + 1
        s0, lo, hi = s0 + (i - 1) * step, full[r, i - 1], full[r, i]
    t = np.clip((level - lo) / (hi - lo), 0.0, 1.0)
    return s0 + t * (1.0 / ROUND**2)


def surface(xyz, cells, feats, level: float, sigma_fn, color_fn=None, positions=None, normals=None, chunk: int = 512) -> Dict[str, np.ndarray]:
    """the extraction on features feats f64[V, C] with density sigma_fn(f [..., C]) -> [...] and colour color_fn(f [N, C], dirs [N, 3])
    -> [N, 3].  -> edges i64[N,2], s, vertices, normals, colors (None without color_fn), faces i64[F,3], face_tetrahedra, vertex_sigma
    f64[V], area f64[N] (the area of the faces around each vertex)."""
    xyz = np.asarray(xyz, dtype=np.float32).reshape(-1, 3)
    cells = np.asarray(cells, dtype=np.int64).reshape(-1, 4)
    feats = np.asarray(feats, dtype=np.float64)
    V = len(xyz)
    vsig = np.asarray(sigma_fn(feats), dtype=np.float64)
    inside = vsig >= level
    n_in = inside[cells].sum(1)
    tri_edges, ftet = [], []
    for t in np.nonzero((n_in > 0) & (n_in < 4))[0]:
        for tri in tet_faces(xyz, cells[t], inside[cells[t]]):
            tri_edges.append(tri)
            ftet.append(t)
    tri_edges = np.asarray(tri_edges, dtype=np.int64).reshape(-1, 3, 2)
    keys = tri_edges[..., 0] * V + tri_edges[..., 1]
    ukeys = np.unique(keys)
    edges = np.stack([ukeys // V, ukeys % V], 1)
    faces = np.searchsorted(ukeys, keys)
    a, b = edges[:, 0], edges[:, 1]
    x64 = xyz.astype(np.float64)
    if positions is None:
        s = np.empty(len(edges))
        for c0 in range(0, len(edges), chunk):
            ea, eb = a[c0:c0 + chunk], b[c0:c0 + chunk]
            Fa, Fb = feats[ea][:, None, :], feats[eb][:, None, :]
            s[c0:c0 + chunk] = crossing(lambda ss: np.asarray(sigma_fn((1.0 - ss)[..., None] * Fa + ss[..., None] * Fb)), level, vsig[ea], vsig[eb])
        pos = (1.0 - s)[:, None] * x64[a] + s[:, None] * x64[b]
    else:  # the given points' parameters along their edges
        pos = np.asarray(positions, dtype=np.float64).reshape(-1, 3)
        d = x64[b] - x64[a]
        s = np.sum((pos - x64[a]) * d, 1) / np.sum(d * d, 1)
    p = pos[faces]
    fn = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    acc = np.zeros((len(edges), 3))
    area = np.zeros(len(edges))
    for k in range(3):
        np.add.at(acc, faces[:, k], fn)
        np.add.at(area, faces[:, k], 0.5 * np.linalg.norm(fn, axis=1))
    ln = np.linalg.norm(acc, axis=1, keepdims=True)
    nrm = np.divide(acc, ln, out=np.zeros_like(acc), where=ln > 0)
    view = nrm if normals is None else np.asarray(normals, dtype=np.float64).reshape(-1, 3)
    colors = None
    if color_fn is not None and len(edges):
        f = (1.0 - s)[:, None] * feats[a] + s[:, None] * feats[b]
        colors = np.asarray(color_fn(f, -view), dtype=np.float64)
    return {"edges": edges, "s": s, "vertices": pos, "normals": nrm, "colors": colors, "faces": faces, "face_tetrahedra": np.asarray(ftet, np.int64),
            "vertex_sigma": vsig, "area": area}


def network(params):
    """(sigma_fn, color_fn) of the MLP parameters ({PARAM_ORDER name: tensor}) in float64, on numpy arrays"""
    P = {k: v.detach().to(torch.float64) for k, v in params.items()}

    def sigma_fn(f):
        with torch.no_grad():
            x = torch.from_numpy(np.ascontiguousarray(f, dtype=np.float64))
            return orc.density_head(P, orc.mlp_base(P, x))[..., 0].numpy()

    def color_fn(f, dirs):
        with torch.no_grad():
            x = torch.from_numpy(np.ascontiguousarray(f, dtype=np.float64))
            d = torch.from_numpy(np.ascontiguousarray(dirs, dtype=np.float64))
            return orc.color_head(P, orc.mlp_base(P, x), orc.nerf_encoding_dirs(d)).numpy()

    return sigma_fn, color_fn


def extract(xyz, cells, field, params, level: float, positions=None, normals=None) -> Dict[str, np.ndarray]:
    """the surface of the network `params` on field f32[64, V] (feature-major, as tn_render_set_field takes it)"""
    sigma_fn, color_fn = network(params)
    return surface(xyz, cells, np.asarray(field, dtype=np.float64).T, level, sigma_fn, color_fn, positions, normals)


def topology(faces, n_vertices: int) -> Dict:
    """closedness and components of a triangle mesh: `directed_once` (every directed edge appears exactly once and its reverse too: a
    closed, consistently oriented surface), `components` (list of (vertices, edges, faces, Euler characteristic) per connected component
    of the faces)"""
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    de = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = de[:, 0] * n_vertices + de[:, 1]
    rkey = de[:, 1] * n_vertices + de[:, 0]
    uk, cnt = np.unique(key, return_counts=True)
    directed_once = bool((cnt == 1).all()) and bool(np.isin(rkey, uk).all())
    parent = np.arange(n_vertices)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for u, w in de:
        ru, rw = find(u), find(w)
        if ru != rw:
            parent[ru] = rw
    used = np.unique(f)
    root = np.array([find(x) for x in range(n_vertices)])
    comps = []
    und = np.unique(np.sort(de, axis=1), axis=0)
    for r in np.unique(root[used]):
        nv = int(np.sum(root[used] == r))
        ne = int(np.sum(root[und[:, 0]] == r))
        nf = int(np.sum(root[f[:, 0]] == r))
        comps.append((nv, ne, nf, nv - ne + nf))
    return {"directed_once": directed_once, "components": comps}
