"""Writing the surface of `TetrahedraNerf.extract_surface` / `FusedRenderer.extract_surface` to disk."""
from __future__ import annotations

from pathlib import Path
from typing import Dict, Union

import numpy as np


def _host(x) -> np.ndarray:
    return x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)


def write_ply(path: Union[str, Path], surface: Dict) -> None:
    """binary little-endian PLY: per vertex float x, y, z, nx, ny, nz and uchar red, green, blue (colours in [0,1] -> round(255 c)); per
    face a uchar-counted list of int vertex indices.  `surface`: the dict of extract_surface (tensors or arrays)."""
    v = _host(surface["vertices"]).astype("<f4").reshape(-1, 3)
    n = _host(surface["normals"]).astype("<f4").reshape(-1, 3)
    c = np.clip(np.rint(_host(surface["colors"]).astype(np.float64).reshape(-1, 3) * 255.0), 0, 255).astype(np.uint8)
    f = _host(surface["faces"]).astype("<i4").reshape(-1, 3)
    vert = np.empty(len(v), dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"), ("red", "u1"),
                                   ("green", "u1"), ("blue", "u1")])
    for i, k in enumerate("xyz"):
        vert[k] = v[:, i]
        vert["n" + k] = n[:, i]
    for i, k in enumerate(("red", "green", "blue")):
        vert[k] = c[:, i]
    face = np.empty(len(f), dtype=[("n", "u1"), ("v", "<i4", (3,))])
    face["n"] = 3
    face["v"] = f
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {len(v)}\n"
              "property float x\nproperty float y\nproperty float z\nproperty float nx\nproperty float ny\nproperty float nz\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\n"
              f"element face {len(f)}\n"
              "property list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(vert.tobytes())
        fh.write(face.tobytes())


def read_ply(path: Union[str, Path]) -> Dict[str, np.ndarray]:
    """reads back what write_ply wrote (that layout only) -> vertices, normals f32[N,3], colors u8[N,3], faces i32[F,3]"""
    data = Path(path).read_bytes()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    lines = data[:end].decode("ascii").splitlines()
    if lines[:2] != ["ply", "format binary_little_endian 1.0"]:
        raise ValueError(f"{path}: not a binary little-endian PLY")
    nv = int(next(ln for ln in lines if ln.startswith("element vertex")).split()[-1])
    nf = int(next(ln for ln in lines if ln.startswith("element face")).split()[-1])
    vt = np.dtype([("p", "<f4", (6,)), ("c", "u1", (3,))])
    ft = np.dtype([("n", "u1"), ("v", "<i4", (3,))])
    vert = np.frombuffer(data, dtype=vt, count=nv, offset=end)
    face = np.frombuffer(data, dtype=ft, count=nf, offset=end + nv * vt.itemsize)
    if nf and not (face["n"] == 3).all():
        raise ValueError(f"{path}: faces that are not triangles")
    return {"vertices": vert["p"][:, :3].copy(), "normals": vert["p"][:, 3:].copy(), "colors": vert["c"].copy(), "faces": face["v"].copy()}
