"""GPU: the fused training op keeps per-call saved state (FusedRenderer.train_forward_saved / train_backward_saved, FusedTrainRender), so
it composes like any autograd op: two forwards before one backward, an eval render between forward and backward, backwards in any
order, retain_graph.  A backward after an in-place change of its inputs or after set_field / set_weights raises; a graph dropped without
its backward frees its saved state."""
import pytest
import torch

from oracle import oracle as orc
from tetranerf.b200 import synthetic as syn
from test_gpu_train import DEV, GRAD_TOL, _oracle_grads, _setup

pytestmark = pytest.mark.gpu


def _settings():
    from tetranerf.b200.render import RenderSettings

    return RenderSettings.tetra_nerf(), orc.RenderConfig.tetra_nerf()


def _batch(nrays, ray_seed, seed, st, empty_ray=None):
    """rays, jitters and target of one call: (numpy o, d, CPU jc, jf, target) and the same on the GPU"""
    o, d = syn.camera_rays(nrays, seed=ray_seed)
    if empty_ray is not None:
        o[empty_ray] = [5, 5, 5]; d[empty_ray] = [1, 0, 0]
    g = torch.Generator().manual_seed(seed)
    jc = torch.rand((nrays, st.num_samples + 1), generator=g)
    jf = torch.rand((nrays, st.num_fine_samples + 1), generator=g)
    target = torch.rand((nrays, 3), generator=g)
    cpu = (o, d, jc, jf, target)
    return cpu, (torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), jc.to(DEV), jf.to(DEV), target.to(DEV))


class _Step:
    """a renderer plus leaf tensors for tetrahedra_field and the twelve MLP parameters"""

    def __init__(self, V, C, field):
        from tetranerf.b200.render import PARAM_ORDER

        self.tr, self.fr, params = _setup(V, C, field)
        self.field = torch.from_numpy(field).to(DEV).requires_grad_(True)
        self.params = [params[n].detach().to(DEV).clone().requires_grad_(True) for n in PARAM_ORDER]

    def forward(self, st, batch, gs=False):
        """-> the loss of one FusedTrainRender call (the loss of test_gpu_train: MSE + 0.05 mean accumulation)"""
        from tetranerf.b200.render import FusedTrainRender

        o, d, jc, jf, target = batch
        rgb, acc, _, _ = FusedTrainRender.apply(self.fr, st, gs, o, d, jc, jf, self.field, *self.params)
        return torch.nn.functional.mse_loss(rgb, target) + 0.05 * acc.mean()

    def take_grads(self):
        """-> [field gradient, twelve parameter gradients], cloned; resets them"""
        torch.cuda.synchronize()
        out = [t.grad.clone() for t in [self.field] + self.params]
        for t in [self.field] + self.params:
            t.grad = None
        return out

    def alone(self, st, batch, gs=False):
        self.forward(st, batch, gs).backward()
        return self.take_grads()


def _names():
    from tetranerf.b200.render import PARAM_ORDER

    return ["tetrahedra_field"] + PARAM_ORDER


@pytest.mark.parametrize("det", [True, False], ids=["deterministic", "default"])
def test_two_forwards_one_backward(medium_mesh, monkeypatch, det):
    """forward A (700 rays), forward B (1200 other rays and jitters), one backward of a loss of both = g_A + g_B, where g_A and g_B each
    come from forward -> backward alone; bitwise in deterministic mode (IEEE addition commutes, so the order in which autograd runs the two
    nodes does not matter).  The default mode sums with float atomics, so two runs of the same backward already differ by ~1e-6 of the
    largest entry (tetrahedra_field): it gets the run-to-run bar of test_fused_train_step_is_repeatable_and_many_tiles, 1e-5."""
    if det:
        monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1")
    else:
        monkeypatch.delenv("TETRANERF_B200_DETERMINISTIC", raising=False)
    V, C = medium_mesh
    st, _ = _settings()
    s = _Step(V, C, syn.random_field(len(V), 64, seed=3))
    _, a = _batch(700, 12, 6, st)
    _, b = _batch(1200, 31, 7, st)
    ga = s.alone(st, a)
    gb = s.alone(st, b)
    (s.forward(st, a) + s.forward(st, b)).backward()
    g = s.take_grads()
    for n, x, y, z in zip(_names(), g, ga, gb):
        assert torch.isfinite(x).all(), n
        if det:
            assert torch.equal(x, y + z), n
        else:
            err = (x - (y + z)).abs().max().item() / (y + z).abs().max().item()
            print(f"  {n:34s} |g - (g_A + g_B)| / max: {err:.2e}")
            assert err <= 1e-5, (n, err)


def test_two_forwards_meet_the_float64_bar(small_mesh, monkeypatch):
    """the sum of two calls against the float64 oracle differentiated on both calls, per tensor in units of its largest entry:
    max |g - g_f64| <= max(2e-4, 6 max |g_torch_f32 - g_f64|) (the end-to-end bar of test_gpu_train.py)"""
    monkeypatch.delenv("TETRANERF_B200_DETERMINISTIC", raising=False)
    V, C = small_mesh
    st, oc = _settings()
    field = syn.random_field(len(V), 64, seed=3)
    s = _Step(V, C, field)
    ca, a = _batch(300, 11, 5, st, empty_ray=5)
    cb, b = _batch(200, 17, 9, st)
    gs = True
    (s.forward(st, a, gs) + s.forward(st, b, gs)).backward()
    g = s.take_grads()
    params = orc.init_mlp_params(0)
    mesh = orc.OracleMesh(V, C)
    ref = {}
    for dtype in (torch.float32, torch.float64):
        tot = None
        for o, d, jc, jf, target in (ca, cb):
            _, gf, gp = _oracle_grads(V, C, field, params, o, d, oc, jc, jf, target, gs, mesh, dtype=dtype)
            one = [gf] + [gp[n] for n in _names()[1:]]
            tot = one if tot is None else [x + y for x, y in zip(tot, one)]
        ref[dtype] = [t.detach().double() for t in tot]
    failures = []
    for n, x, f32, f64 in zip(_names(), g, ref[torch.float32], ref[torch.float64]):
        x = x.detach().cpu().double()
        scale = f64.abs().max().item()
        err = (x - f64).abs().max().item() / scale
        noise = (f32 - f64).abs().max().item() / scale
        print(f"  {n:34s} max|g| {scale:.3e}  kernel vs f64: {err:.2e}   torch-f32 vs f64: {noise:.2e}")
        if not err <= max(2 * GRAD_TOL, 6 * noise):
            failures.append((n, err, noise))
    assert not failures, failures


def test_interleaved_eval_render_and_reversed_backwards(medium_mesh, monkeypatch):
    """forward A, an eval render, forward B, backward B, backward A: bitwise the gradients of one backward of both"""
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1")
    V, C = medium_mesh
    st, _ = _settings()
    s = _Step(V, C, syn.random_field(len(V), 64, seed=3))
    _, a = _batch(700, 12, 6, st)
    _, b = _batch(1200, 31, 7, st)
    (s.forward(st, a) + s.forward(st, b)).backward()
    g = s.take_grads()
    la = s.forward(st, a)
    eo, ed = (torch.from_numpy(x).to(DEV) for x in syn.camera_rays(2000, seed=40))
    s.fr.render(eo, ed, st)  # more rays than either training call: the tracer's own buffers grow
    lb = s.forward(st, b)
    lb.backward()
    la.backward()
    for n, x, y in zip(_names(), s.take_grads(), g):
        assert torch.equal(x, y), n


def test_retain_graph_twice_gives_twice_the_gradient(medium_mesh, monkeypatch):
    monkeypatch.setenv("TETRANERF_B200_DETERMINISTIC", "1")
    V, C = medium_mesh
    st, _ = _settings()
    s = _Step(V, C, syn.random_field(len(V), 64, seed=3))
    _, a = _batch(700, 12, 6, st)
    g1 = s.alone(st, a)
    loss = s.forward(st, a)
    loss.backward(retain_graph=True)
    loss.backward()
    for n, x, y in zip(_names(), s.take_grads(), g1):
        assert torch.equal(x, 2 * y), n


@pytest.mark.parametrize("change", ["field_in_place", "weight_in_place", "set_field", "set_weights"])
def test_backward_after_a_change_raises(small_mesh, change):
    from tetranerf.b200.render import PARAM_ORDER

    V, C = small_mesh
    st, _ = _settings()
    s = _Step(V, C, syn.random_field(len(V), 64, seed=3))
    _, a = _batch(200, 11, 5, st)
    loss = s.forward(st, a)
    if change == "field_in_place":
        with torch.no_grad():
            s.field.mul_(1.0)
    elif change == "weight_in_place":
        with torch.no_grad():
            s.params[2].add_(0.0)
    elif change == "set_field":
        s.fr.set_field(s.field.detach())
    else:
        s.fr.set_weights({n: p.detach() for n, p in zip(PARAM_ORDER, s.params)})
    with pytest.raises(RuntimeError):
        loss.backward()
    torch.cuda.synchronize()
    # a forward after the change trains again
    s.alone(st, a)


def test_backward_checks_the_gradient_shape(small_mesh):
    V, C = small_mesh
    st, _ = _settings()
    s = _Step(V, C, syn.random_field(len(V), 64, seed=3))
    _, (o, d, jc, jf, _) = _batch(200, 11, 5, st)
    out, state = s.fr.train_forward_saved(o, d, st, jc, jf)
    assert state.R == 200 and state.blob.numel() == s.fr.train_saved_bytes(200, st)
    with pytest.raises(RuntimeError, match="200 rays"):
        s.fr.train_backward_saved(state, torch.zeros((199, 3), device=DEV), None, len(V))
    gf, gp = s.fr.train_backward_saved(state, torch.zeros((200, 3), device=DEV), None, len(V))
    torch.cuda.synchronize()
    assert not gf.any() and not any(t.any() for t in gp.values())


def test_dropped_graph_frees_its_saved_state(small_mesh):
    V, C = small_mesh
    st, _ = _settings()
    s = _Step(V, C, syn.random_field(len(V), 64, seed=3))
    _, a = _batch(700, 12, 6, st)
    s.alone(st, a)  # warm-up: the tracer's workspace exists, torch's cache holds blocks of these sizes
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(DEV)
    loss = s.forward(st, a)
    held = torch.cuda.memory_allocated(DEV) - before
    assert held >= s.fr.train_saved_bytes(700, st)
    del loss
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(DEV) == before
    print(f"saved state of 700 rays: {s.fr.train_saved_bytes(700, st) / 2**20:.1f} MiB; at 8192 rays x 257 fine samples: "
          f"{s.fr.train_saved_bytes(8192, st) / 2**20:.1f} MiB")


def test_model_two_training_calls_fused_vs_unfused(small_mesh, monkeypatch):
    """TetrahedraNerf in training mode: two get_outputs calls, a summed MSE loss, one backward; fused against the unfused op sequence
    with the bar of test_model_training_path_fused_vs_unfused (stratified draws off so both consume the same bins)"""
    from tetranerf.nerfstudio import model as M

    V, C = small_mesh
    field = syn.random_field(len(V), 64, seed=3)
    rays = [syn.camera_rays(256, seed=14), syn.camera_rays(180, seed=15)]
    targets = [torch.rand((len(o), 3), generator=torch.Generator().manual_seed(3 + i)).to(DEV) for i, (o, _) in enumerate(rays)]
    grads = {}
    for mode in ("fused", "unfused"):
        monkeypatch.setenv("TETRANERF_B200_UNFUSED_TRAIN", "1" if mode == "unfused" else "0")
        cfg = M.TetrahedraNerfConfig(num_tetrahedra_vertices=len(V), num_tetrahedra_cells=len(C), num_samples=64, num_fine_samples=64,
                                     use_biased_sampler=True, use_gradient_scaling=True)
        m = M.TetrahedraNerf(cfg)
        sd = {"tetrahedra_vertices": torch.from_numpy(V), "tetrahedra_cells": torch.from_numpy(C), "tetrahedra_field": torch.from_numpy(field)}
        sd.update(orc.init_mlp_params(0))
        m.load_state_dict(sd, strict=False)
        m = m.to(DEV).train()
        m.sampler_uniform.train_stratified = False
        m.sampler_pdf.train_stratified = False
        loss, rgbs = 0.0, []
        for (o, d), target in zip(rays, targets):
            out = m(M.RayBundle(origins=torch.from_numpy(o).to(DEV), directions=torch.from_numpy(d).to(DEV)))
            loss = loss + m.get_loss_dict(out, {"image": target})["rgb_loss"]
            rgbs.append(out["rgb"].detach().clone())
        loss.backward()
        grads[mode] = (rgbs, {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None})
    for x, y in zip(grads["fused"][0], grads["unfused"][0]):
        assert (x - y).abs().max().item() < 1e-4
    assert set(grads["fused"][1]) == set(grads["unfused"][1]) and "tetrahedra_field" in grads["fused"][1]
    for n, g in grads["unfused"][1].items():
        a = grads["fused"][1][n]
        rel = ((a - g).abs().max() / g.abs().max().clamp_min(1e-30)).item()
        l2 = ((a - g).norm() / g.norm().clamp_min(1e-30)).item()
        print(f"  {n:34s} fused vs unfused: max {rel:.2e}  L2 {l2:.2e}")
        assert torch.isfinite(a).all()
        assert rel < 5e-3 and l2 < 1e-3, (n, rel, l2)
