"""trace-only sweep: warp-per-ray BVH gather vs adjacency walks, through the fused renderer's per-kernel timings"""
import os, sys, json
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [R, R + "/tetra-nerf_b200"]
import numpy as np, torch, bench
from tetranerf import cpp
from tetranerf.b200 import synthetic as syn
from tetranerf.b200.render import FusedRenderer, RenderSettings

# each implementation of trace_rays forced through the setters: (walk_min_rays, solo range, quad range, spec max rays)
NEVER, ALWAYS = (1, 0), (0, 2**32 - 1)
FORMS = {
    "bvh": (2**32 - 1, NEVER, NEVER, 0),                       # warp-per-ray all-hits BVH gather
    "walk": (0, NEVER, NEVER, 0),                              # 32 rays per warp
    "walk_solo": (2**32 - 1, ALWAYS, NEVER, 2**32 - 1),        # 1 ray per warp, speculative record loads
    "walk_quad_pf": (2**32 - 1, NEVER, ALWAYS, 0),             # 8 rays per warp, prefetched record loads
    "walk_quad": (2**32 - 1, NEVER, ALWAYS, 2**32 - 1),        # 8 rays per warp, speculative record loads
}
dev = torch.device("cuda:0")
V, C, field = bench.make_workload()
tr = cpp.TetrahedraTracer(dev); dV, dC = torch.from_numpy(V).to(dev), torch.from_numpy(C).to(dev); tr.load_tetrahedra(dV, dC)
fr = FusedRenderer(tr); fr.set_field(torch.from_numpy(field).to(dev)); fr.set_weights(bench.mlp_params()); fr.set_profiling(True)
st = RenderSettings.tetra_nerf()
for name, (min_rays, solo, quad, spec) in FORMS.items():
    tr.set_walk_min_rays(min_rays); tr.set_walk_solo_range(*solo); tr.set_walk_quad_range(*quad); tr.set_walk_quad_spec_max_rays(spec)
    res = {}
    for n in (1024, 2048, 4096, 8192, 16384, 32768, 65536):
        o, d = syn.camera_rays(n, seed=3); o, d = torch.from_numpy(o).to(dev), torch.from_numpy(d).to(dev)
        for _ in range(2): fr.render(o, d, st)
        t = []
        for _ in range(4):
            fr.render(o, d, st); t.append(fr.kernel_timings_ms())
        res[n] = {k: round(float(np.median([x[k] for x in t])), 4) for k in t[0]}
    print(name, json.dumps(res), flush=True)
