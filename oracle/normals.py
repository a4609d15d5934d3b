"""Float64 oracle of the normal map of the fused render -- TEST INFRASTRUCTURE ONLY.

Definition (DESIGN.md §4.7).  For one sample matched to the tetrahedron with vertex ids (v0, v1, v2, v3) (the vi order of the fused
render and of find_visited_cells) and weights (b0, b1, b2) on v1, v2, v3 (w0 = 1 - sum b on v0):
  f = F_v0 + sum_k b_k (F_vk - F_v0),  pre = wd . mlp_base(f) + bd,  sigma = softplus(pre)
  g = d pre / d f in R^64 (reverse chain through the three Linear + ReLU layers; a ReLU passes gradient where its pre-activation > 0)
  q_k = g . (F_vk - F_v0),  E = [x_v1 - x_v0 | x_v2 - x_v0 | x_v3 - x_v0],  grad_x pre = E^-T q = cof(E) q / det(E)
  n = -grad / max(|grad|, 1e-12)  (nerfstudio Field.get_normals = -normalize(grad sigma); softplus' > 0), 0 for unmatched samples and
  det(E) = 0;  pixel N = sum_i w_i n_i, then N / sqrt(max(|N|^2, 1e-20))  (nerfstudio NormalsRenderer(normalize=True)).

`emulate_grad_pre` repeats the reverse chain with the operand rounding of the tensor-core kernel (f16w2 / bf16x3), which predicts the
per-sample error of each precision without a GPU."""
from __future__ import annotations

from typing import Dict

import numpy as np

_LAYERS = ("mlp_base.layers.0", "mlp_base.layers.1", "mlp_base.layers.2")


def _p64(params) -> Dict[str, np.ndarray]:
    return {k: np.asarray(v.detach().cpu().numpy() if hasattr(v, "detach") else v, dtype=np.float64) for k, v in params.items()}


def features(vi, bary, field) -> np.ndarray:
    """f = F_v0 + sum_k b_k (F_vk - F_v0) in float64: vi [N,4] (negative / 0xFFFFFFFF = unmatched -> 0), bary [N,3], field [64,V]"""
    vi = np.asarray(vi).astype(np.int64).reshape(-1, 4)
    b = np.asarray(bary, dtype=np.float64).reshape(-1, 3)
    F = np.asarray(field, dtype=np.float64).T
    ok = (vi[:, 0] >= 0) & (vi[:, 0] < len(F))
    v = np.where(ok[:, None], vi, 0)
    f = F[v[:, 0]] + sum(b[:, k:k + 1] * (F[v[:, k + 1]] - F[v[:, 0]]) for k in range(3))
    return np.where(ok[:, None], f, 0.0)


def forward(params, f) -> Dict[str, list]:
    """mlp_base in float64: the layer inputs a_0 = f, a_1, a_2, a_3 and pre-activations z_1..z_3, and the density pre-activation"""
    P = _p64(params)
    a, z = [np.asarray(f, dtype=np.float64)], []
    for name in _LAYERS:
        z.append(a[-1] @ P[f"{name}.weight"].T + P[f"{name}.bias"])
        a.append(np.maximum(z[-1], 0.0))
    pre = a[-1] @ P["field_output_density.net.weight"][0] + P["field_output_density.net.bias"][0]
    return {"a": a, "z": z, "pre": pre}


def mask_ambiguous(params, fw, kappa: float) -> np.ndarray:
    """samples with a hidden pre-activation inside the band |z| <= kappa (sum_k |W_k a_k| + |b|), where an implementation that rounds
    its operands at relative precision ~kappa may see the other sign (and so another ReLU mask)"""
    P = _p64(params)
    amb = np.zeros(len(fw["pre"]), dtype=bool)
    for l, name in enumerate(_LAYERS):
        scale = np.abs(fw["a"][l]) @ np.abs(P[f"{name}.weight"]).T + np.abs(P[f"{name}.bias"])
        amb |= ((np.abs(fw["z"][l]) <= kappa * scale) & (scale > 0)).any(-1)  # (a unit with no inputs and no bias is exactly 0 everywhere)
    return amb


def feature_grad(params, fw) -> np.ndarray:
    """g = d pre / d f [N,64]"""
    P = _p64(params)
    d = (fw["z"][2] > 0) * P["field_output_density.net.weight"][0]
    d = (d @ P["mlp_base.layers.2.weight"]) * (fw["z"][1] > 0)
    d = (d @ P["mlp_base.layers.1.weight"]) * (fw["z"][0] > 0)
    return d @ P["mlp_base.layers.0.weight"]


def solve(vi, g, field, xyz, g_is_f32_diff: bool = False) -> Dict[str, np.ndarray]:
    """q, cof(E), det(E) and grad_x pre = cof(E) q / det(E) from the feature gradient g [N,64] (0 for unmatched samples and det = 0).
    g_is_f32_diff: form F_vk - F_v0 in float32 first, as the kernel does"""
    vi = np.asarray(vi).astype(np.int64).reshape(-1, 4)
    ok = (vi[:, 0] >= 0) & (vi[:, 0] < np.asarray(field).shape[1])
    v = np.where(ok[:, None], vi, 0)
    F = np.asarray(field, dtype=np.float32).T
    X = np.asarray(xyz, dtype=np.float32).astype(np.float64).reshape(-1, 3)
    if g_is_f32_diff:
        dF = [(F[v[:, k]] - F[v[:, 0]]).astype(np.float64) for k in (1, 2, 3)]
    else:
        dF = [F[v[:, k]].astype(np.float64) - F[v[:, 0]].astype(np.float64) for k in (1, 2, 3)]
    q = np.stack([np.sum(g * d, -1) for d in dF], -1)
    e = [X[v[:, k]] - X[v[:, 0]] for k in (1, 2, 3)]
    cof = np.stack([np.cross(e[1], e[2]), np.cross(e[2], e[0]), np.cross(e[0], e[1])], -1)  # columns
    det = np.sum(e[0] * cof[..., 0], -1)
    good = ok & (det != 0)
    grad = np.einsum("nij,nj->ni", cof, q) / np.where(good, det, 1.0)[:, None]
    grad[~good] = 0.0
    q[~ok] = 0.0
    return {"grad": grad, "q": q, "cof": cof, "det": det, "matched": ok}


def grad_pre(vi, bary, xyz, field, params, kappa: float = 0.0) -> Dict[str, np.ndarray]:
    """grad_x pre of every sample in float64 (plus q, cof, det, the feature gradient and, for kappa > 0, the mask-ambiguity flags)"""
    fw = forward(params, features(vi, bary, field))
    g = feature_grad(params, fw)
    out = solve(vi, g, field, xyz)
    out.update(g=g, pre=fw["pre"])
    if kappa > 0:
        out["ambiguous"] = mask_ambiguous(params, fw, kappa)
    return out


def sample_normals(grad) -> np.ndarray:
    grad = np.asarray(grad, dtype=np.float64)
    return -grad / np.maximum(np.linalg.norm(grad, axis=-1, keepdims=True), 1e-12)


def composite(weights, normals):
    """NormalsRenderer: weights [R,S], sample normals [R,S,3] -> (sum w n [R,3], normalised [R,3])"""
    n = np.sum(np.asarray(weights, dtype=np.float64)[..., None] * np.asarray(normals, dtype=np.float64), axis=-2)
    return n, n / np.sqrt(np.maximum(np.sum(n * n, -1, keepdims=True), 1e-20))


# ---- operand rounding of the tensor-core reverse chain ---------------------------------------------------------------------------------
def _bf16(x) -> np.ndarray:
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return (r & 0xFFFFFFFF).astype(np.uint32).view(np.float32).astype(np.float64)


def _f16(x) -> np.ndarray:
    return np.clip(np.asarray(x, dtype=np.float32), -65504.0, 65504.0).astype(np.float16).astype(np.float64)


def _split(x, prec):
    """operand halves (hi, lo) of the kernel: bf16 hi / lo (prec 3) or fp16 hi / lo (prec 2)"""
    rnd = _bf16 if prec == 3 else _f16
    x32 = np.asarray(x, dtype=np.float32)
    hi = rnd(x32)
    return hi, rnd(x32.astype(np.float64) - hi)


def _product(a, W, prec):
    """a [N,K] (fp32 cotangent) times W [K,M] as the MMAs form it: bf16x3 a_hi W_hi + a_lo W_hi + a_hi W_lo; f16w2 fp16(a) (W_hi + W_lo)"""
    wh, wl = _split(W, prec)
    if prec == 3:
        ah, al = _split(a, 3)
        out = ah @ wh + al @ wh + ah @ wl
    else:
        af = _f16(a)
        out = af @ wh + af @ wl
    return out.astype(np.float32).astype(np.float64)  # fp32 accumulator


def emulate_feature_grad(params, fw, prec: int) -> np.ndarray:
    """g as k_mlp_normals<prec> forms it, with the float64 masks: the seed m3 * wd 2^-e, max |wd 2^-e| in [2^7, 2^8) (exact), every
    cotangent rounded to the operand format before each of the three products, fp32 accumulators; the power of two undone"""
    P = {k: np.asarray(v, dtype=np.float32) for k, v in _p64(params).items()}
    wd = P["field_output_density.net.weight"][0]
    e = np.frexp(np.max(np.abs(wd)))[1] - 8
    d = (fw["z"][2] > 0) * np.ldexp(wd.astype(np.float64), -e)
    d = _product(d, P["mlp_base.layers.2.weight"], prec) * (fw["z"][1] > 0)
    d = _product(d, P["mlp_base.layers.1.weight"], prec) * (fw["z"][0] > 0)
    return np.ldexp(_product(d, P["mlp_base.layers.0.weight"], prec), e)


def emulate_grad_pre(vi, bary, xyz, field, params, prec: int) -> np.ndarray:
    fw = forward(params, features(vi, bary, field))
    return solve(vi, emulate_feature_grad(params, fw, prec), field, xyz, g_is_f32_diff=True)["grad"]


def error_measure(grad, ref) -> np.ndarray:
    """|grad - ref_grad| / (|cof E|_F |q| / |det E|): the per-sample error relative to what the solve can amplify (holds in slivers);
    ref = the dict of grad_pre.  0 where the reference is 0 (unmatched, det = 0) and the gradient is too."""
    bound = np.linalg.norm(ref["cof"], axis=(-2, -1)) * np.linalg.norm(ref["q"], axis=-1) / np.where(ref["det"] != 0, np.abs(ref["det"]), 1.0)
    diff = np.linalg.norm(np.asarray(grad, dtype=np.float64) - ref["grad"], axis=-1)
    return np.where(bound > 0, diff / np.where(bound > 0, bound, 1.0), np.where(diff > 0, np.inf, 0.0))
