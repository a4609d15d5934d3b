"""torchrun --nproc-per-node N tools/peer_gather_check.py [--background] : the fused peer-store pixel gather (tn_render_set_gather) against
the 1-GPU render of the whole batch, bit for bit, on every rank; also the NCCL all_gather path (tetranerf.b200.distributed.sharded_render).
--background: every render composites over the same N(0,1) background map (FusedRenderer.set_background, DESIGN §4.16), so the gathered
pixels of the active rays and of the rays that miss the mesh come from the map lookup inside the pixel-writing kernels."""
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tetra-nerf_b200")]
import numpy as np
import torch
import torch.distributed as dist

import bench
from tetranerf import cpp
from tetranerf.b200 import synthetic as syn
from tetranerf.b200.distributed import shard_bounds, sharded_render
from tetranerf.b200.render import FusedRenderer, RenderSettings
from tetranerf.utils.extension import tetranerf_cpp_extension as ext


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dev = torch.device("cuda", lr)
    dist.init_process_group("nccl", device_id=dev)
    V, C = syn.delaunay_mesh(4000, seed=0)
    field = syn.random_field(len(V), 64, seed=3)
    params = bench.mlp_params()
    Rper = 1024
    R = Rper * world
    o, d = syn.camera_rays(R, seed=77)
    o[5] = [5, 5, 5]; d[5] = [1, 0, 0]
    if "--background" in sys.argv:  # a miss in every rank's shard, looking elsewhere on the map
        for r in range(world):
            o[r * Rper + 7] = [-4, 0.5, 0.5]; d[r * Rper + 7] = [-0.8, 0.2, 0.56]
    tr = cpp.TetrahedraTracer(dev)
    tr.load_tetrahedra(torch.from_numpy(V).to(dev), torch.from_numpy(C).to(dev))
    fr = FusedRenderer(tr)
    fr.set_field(torch.from_numpy(field).to(dev))
    fr.set_weights(params)
    if "--background" in sys.argv:  # the same map on every rank (seeded on the CPU)
        fr.set_background(torch.randn((8, 16, 3), generator=torch.Generator().manual_seed(5)).to(dev))
    st = RenderSettings.tetra_nerf()
    do, dd = torch.from_numpy(o).to(dev), torch.from_numpy(d).to(dev)
    whole = {k: v.clone() for k, v in fr.render(do, dd, st).items()}  # every rank renders the whole batch itself: the reference result
    # ---- NCCL path ----
    got = sharded_render(lambda a, b: fr.render(a, b, st), do, dd)
    for k in ("rgb", "accumulation", "depth", "ray_mask"):
        assert torch.equal(got[k], whole[k]), f"rank {rank}: NCCL gather differs in {k}"
    # ---- fused peer-store path ----
    gathered = bench.setup_peer_gather(ext._lib, tr, dist, dev, world, rank, Rper)
    lo, hi = shard_bounds(R, rank, world)
    assert (lo, hi) == (rank * Rper, (rank + 1) * Rper)
    fr.render(do[lo:hi].contiguous(), dd[lo:hi].contiguous(), st)
    torch.cuda.synchronize(dev)
    dist.barrier()  # every rank's kernels have completed: their peer stores have been performed
    torch.cuda.synchronize(dev)
    assert torch.equal(gathered[:, 0:3], whole["rgb"]), f"rank {rank}: fused gather rgb differs"
    assert torch.equal(gathered[:, 3:4], whole["accumulation"]) and torch.equal(gathered[:, 4:5], whole["depth"])
    assert torch.equal(gathered[:, 5] > 0.5, whole["ray_mask"])
    dist.barrier()
    if rank == 0:
        bg = ", over a background map" if "--background" in sys.argv else ""
        print(f"peer_gather_check ok: world {world}, {R} rays{bg}, fused peer-store gather == NCCL gather == 1-GPU render (bitwise)")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
