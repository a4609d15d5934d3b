"""VERDICT r1 item 4: is there a cheaper operand split than bf16x3 (3 MMAs per product) that holds the 1e-4 per-sample bar?
CPU emulation of the fused MLP's arithmetic (exact products of the split operands, fp32 accumulation) on the bench's field /
weights: per-sample density and colour against float64; then the same on the opaque surface network of synthetic.surface_scene, where
f16w2's error turns out relative to the activations (density ~4e-4 |sigma|).  Run: python tools/split_accuracy.py"""
import os, sys
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [R, R + "/tetra-nerf_b200"]
import numpy as np, torch
from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn

torch.manual_seed(0)
params = {k: (v.double() if torch.is_tensor(v) else torch.as_tensor(v).double()) for k, v in orc.init_mlp_params(0).items()}
names = list(params)
N = 20000
rng = np.random.default_rng(0)
field = torch.from_numpy(syn.random_field(4000, 64, seed=3, kind="normal")).double()
if field.shape[0] == 64: field = field.T.contiguous()  # [V,64]
idx = torch.from_numpy(rng.integers(0, 4000, (N, 4)))
b = torch.from_numpy(rng.dirichlet(np.ones(4), N))
x0 = (field[idx] * b[..., None]).sum(1)                       # [N,64] interpolated features
dirs = torch.from_numpy(rng.standard_normal((N, 3))); dirs = dirs / dirs.norm(dim=1, keepdim=True)


def split(t, dt, terms):
    hi = t.float().to(dt).double()
    if terms == 1:
        return [hi]
    lo = (t - hi).float().to(dt).double()
    return [hi, lo]


def linear(a, w, bias, scheme):
    """scheme: None (float64) or (dtype, products) with products a list of (a_term, w_term) index pairs"""
    if scheme is None:
        return a @ w.T + bias
    dt, prods = scheme
    A, W = split(a, dt, 2), split(w, dt, 2)
    acc = torch.zeros(a.shape[0], w.shape[0], dtype=torch.float32)
    for ia, iw in prods:
        acc = acc + (A[ia] @ W[iw].T).float()                 # products exact (<= 22 bit), sum rounded to fp32 once per term
    return acc.double() + bias


def mlp(scheme, p=params, x=x0):
    h = x
    for l in range(3):
        h = torch.relu(linear(h, p[f"mlp_base.layers.{l}.weight"], p[f"mlp_base.layers.{l}.bias"], scheme))
    # the heads are fp32 FMAs in the kernel, the direction part of mlp_head is a per-ray fp32 bias: only the 128 hidden inputs of
    # mlp_head go through the tensor cores
    sigma = torch.nn.functional.softplus(h @ p["field_output_density.net.weight"].T + p["field_output_density.net.bias"])
    enc = orc.nerf_encoding_dirs(dirs.float()).double()
    w4 = p["mlp_head.layers.0.weight"]
    ne = enc.shape[1]
    hh = torch.relu(linear(h, w4[:, ne:], p["mlp_head.layers.0.bias"] + enc @ w4[:, :ne].T, scheme))
    rgb = torch.sigmoid(hh @ p["field_output_color.net.weight"].T + p["field_output_color.net.bias"])
    return sigma, rgb


bf, fp = torch.bfloat16, torch.float16
SCHEMES = {
    "bf16x3 (training / reference mode): hi.hi + lo.hi + hi.lo": (bf, [(0, 0), (1, 0), (0, 1)]),
    "fp16x3: hi.hi + lo.hi + hi.lo": (fp, [(0, 0), (1, 0), (0, 1)]),
    "fp16x2: (a_hi + a_lo).w_hi": (fp, [(0, 0), (1, 0)]),
    "f16w2 (inference default): a_hi.(w_hi + w_lo)": (fp, [(0, 0), (0, 1)]),
    "bf16x2: (a_hi + a_lo).w_hi": (bf, [(0, 0), (1, 0)]),
    "fp16x1": (fp, [(0, 0)]),
}


def surface_inputs(sharpness):
    """(params, interpolated features) of synthetic.surface_scene(sharpness) on 4000 random points, in float64"""
    pts = np.random.default_rng(1).random((4000, 3))
    fld, p = syn.surface_scene(pts, sharpness, orc.init_mlp_params(0))
    f = torch.from_numpy(fld).double().T.contiguous()
    return {k: v.double() for k, v in p.items()}, (f[idx] * b[..., None]).sum(1)


def errors(p=params, x=x0):
    """{scheme: (max |sigma err|, max |colour err|, 99.9th percentiles, max |sigma err| / sigma where sigma > 1)} against float64"""
    ref_s, ref_c = mlp(None, p, x)
    out = {}
    big = ref_s > 1.0
    for name, sc in SCHEMES.items():
        s, c = mlp(sc, p, x)
        out[name] = ((s - ref_s).abs().max().item(), (c - ref_c).abs().max().item(),
                     (s - ref_s).abs().flatten().quantile(0.999).item(), (c - ref_c).abs().flatten().quantile(0.999).item(),
                     ((s - ref_s).abs()[big] / ref_s[big]).max().item() if bool(big.any()) else 0.0)
    return out


if __name__ == "__main__":
    print(f"{N} samples; max / 99.9th-percentile absolute error against float64 (bar: 1e-4 per sample)")
    for name, (es, ec, qs, qc, _) in errors().items():
        print(f"{name:58s} sigma {es:.2e} / {qs:.2e}   colour {ec:.2e} / {qc:.2e}")
    for k in (10, 100, 1000):
        print(f"surface network, sharpness {k}: max |sigma err|, relative where sigma > 1, max |colour err|")
        for name, (es, ec, _, _, rel) in errors(*surface_inputs(k)).items():
            print(f"  {name:56s} sigma {es:.2e} (relative {rel:.2e})   colour {ec:.2e}")
