"""Oracle of the learned background (tn_render_set_background, DESIGN.md §4.16) -- TEST INFRASTRUCTURE ONLY.

In float64 numpy, from the definition.  B [H,W,3], W = 2H; for a direction d, n = d / |d|:
    u = W (atan2(n_y, n_x) / 2 pi + 1/2) - 1/2,  columns modulo W
    v = H (1 - n_z) / 2 - 1/2, clamped to [0, H - 1]
    i0 = floor(u), fu = u - i0;  j0 = floor(v), j1 = min(j0 + 1, H - 1), fv = v - j0
    bg(d) = lerp(lerp(B[j0,i0], B[j0,i0+1], fu), lerp(B[j1,i0], B[j1,i0+1], fu), fv),  lerp(a, b, t) = a + t (b - a)
Per ray, with w_j, c_j the weights and colours of its samples and acc = sum_j w_j:
    rgb = sum_j w_j c_j + (1 - acc) bg(d) on rays with hits,  rgb = bg(d) on empty rays (eval mode clamps every pixel to [0, 1])
Gradients, with s = grad_rgb (1 - acc) per ray (grad_rgb on empty rays):
    dL/dB   = s scattered to the four texels with the bilinear weights (1 - fu)(1 - fv), fu (1 - fv), (1 - fu) fv, fu fv
    dL/dw_j = grad_rgb . (c_j - bg(d)) + grad_acc
    dL/dd  += (d bg / d d)^T s, with the u-derivative taken as 0 where n_x^2 + n_y^2 < POLE_EPS (u is undefined at the poles)."""
from __future__ import annotations

import numpy as np

POLE_EPS = 1e-8


def taps(H: int, W: int, d):
    """-> dict of the lookup's intermediate quantities for directions d [R,3] (float64)"""
    d = np.asarray(d, dtype=np.float64).reshape(-1, 3)
    ln = np.linalg.norm(d, axis=1)
    n = d / ln[:, None]
    u = W * (np.arctan2(n[:, 1], n[:, 0]) / (2 * np.pi) + 0.5) - 0.5
    v_raw = H * (1 - n[:, 2]) / 2 - 0.5
    v = np.clip(v_raw, 0.0, H - 1)
    fi, fj = np.floor(u), np.floor(v)
    i0 = np.mod(fi.astype(np.int64), W)
    i1 = np.mod(i0 + 1, W)
    j0 = np.minimum(fj.astype(np.int64), H - 1)
    j1 = np.minimum(j0 + 1, H - 1)
    return {"n": n, "len": ln, "u": u, "v": v, "v_in": (v_raw >= 0) & (v_raw <= H - 1), "fu": u - fi, "fv": v - fj,
            "tex": np.stack([j0 * W + i0, j0 * W + i1, j1 * W + i0, j1 * W + i1], 1)}


def _lerp(a, b, t):
    return a + t * (b - a)


def lookup(B, d) -> np.ndarray:
    """bg(d) -> [R,3] float64"""
    B = np.asarray(B, dtype=np.float64)
    H, W = B.shape[:2]
    t = taps(H, W, d)
    f = B.reshape(-1, 3)[t["tex"]]  # [R,4,3]
    fu, fv = t["fu"][:, None], t["fv"][:, None]
    return _lerp(_lerp(f[:, 0], f[:, 1], fu), _lerp(f[:, 2], f[:, 3], fu), fv)


def composite(comp, acc, ray_mask, B, d, train: bool) -> np.ndarray:
    """rgb per ray from the samples' composited colour comp [R,3] and accumulation acc [R] (ignored on empty rays)"""
    bg = lookup(B, d)
    comp = np.asarray(comp, dtype=np.float64).reshape(-1, 3)
    acc = np.asarray(acc, dtype=np.float64).reshape(-1, 1)
    m = np.asarray(ray_mask, dtype=bool).reshape(-1, 1)
    rgb = np.where(m, comp + (1 - acc) * bg, bg)
    return rgb if train else np.clip(rgb, 0.0, 1.0)


def weights_s(grad_rgb, acc, ray_mask) -> np.ndarray:
    """s = grad_rgb (1 - acc) per ray, grad_rgb on empty rays -> [R,3]"""
    g = np.asarray(grad_rgb, dtype=np.float64).reshape(-1, 3)
    a = np.where(np.asarray(ray_mask, dtype=bool), np.asarray(acc, dtype=np.float64).reshape(-1), 0.0)
    return g * (1 - a)[:, None]


def grad_map(H: int, W: int, d, s) -> np.ndarray:
    """dL/dB [H,W,3] for per-ray weights s [R,3]"""
    t = taps(H, W, d)
    fu, fv = t["fu"], t["fv"]
    w = np.stack([(1 - fu) * (1 - fv), fu * (1 - fv), (1 - fu) * fv, fu * fv], 1)  # [R,4]
    out = np.zeros((H * W, 3))
    s = np.asarray(s, dtype=np.float64).reshape(-1, 3)
    for k in range(4):
        np.add.at(out, t["tex"][:, k], w[:, k:k + 1] * s)
    return out.reshape(H, W, 3)


def grad_direction(B, d, s) -> np.ndarray:
    """(d bg / d d)^T s -> [R,3], with the pole convention of the module docstring"""
    B = np.asarray(B, dtype=np.float64)
    H, W = B.shape[:2]
    t = taps(H, W, d)
    f = B.reshape(-1, 3)[t["tex"]]
    fu, fv = t["fu"][:, None], t["fv"][:, None]
    s = np.asarray(s, dtype=np.float64).reshape(-1, 3)
    gu = np.sum(s * ((1 - fv) * (f[:, 1] - f[:, 0]) + fv * (f[:, 3] - f[:, 2])), 1)
    gv = np.sum(s * (_lerp(f[:, 2], f[:, 3], fu) - _lerp(f[:, 0], f[:, 1], fu)), 1)
    n = t["n"]
    rho2 = n[:, 0] ** 2 + n[:, 1] ** 2
    k = np.where(rho2 >= POLE_EPS, gu * W / (2 * np.pi) / np.maximum(rho2, POLE_EPS), 0.0)
    gn = np.stack([-k * n[:, 1], k * n[:, 0], np.where(t["v_in"], -gv * H / 2, 0.0)], 1)
    gn = gn - np.sum(gn * n, 1, keepdims=True) * n
    return gn / t["len"][:, None]
