"""CPU: the occupancy-sampling oracle (oracle/placement.py, DESIGN §4.13), for both samplers -- every coarse edge in a kept record,
equal shares per kept record (biased) and uniform spacing over the kept length (uniform), today's bins when nothing or everything is
skipped, and the straddling bound on hand-made records (gap records, skipped first / last records)."""
import numpy as np
import pytest
import torch

from oracle import occupancy as ocu
from oracle import oracle as orc
from oracle import placement as pl
from tetranerf.b200 import synthetic as syn

THR = 0.5


def _records(bounds, cells, S, biased, t_rand=None, occ=None):
    """one ray per entry of `bounds` (lists of (t_in, t_out)); cells as the trace gives them (-1: gap record); occ per cell"""
    R, M = len(bounds), max(len(b) for b in bounds)
    hd = np.zeros((R, M, 2), np.float32)
    vc = np.full((R, M), -1, np.int32)
    num = np.array([len(b) for b in bounds], np.int32)
    for r, (b, c) in enumerate(zip(bounds, cells)):
        hd[r, :len(b)] = b
        vc[r, :len(c)] = c
    occ = np.asarray(occ, np.float32)
    kept = pl.kept_records(num, vc, occ, THR)
    hdt = torch.from_numpy(hd)
    nears = hdt[:, 0, 0][:, None]
    fars = torch.gather(hdt[:, :, 1], 1, (torch.from_numpy(num)[:, None].long() - 1).clamp_min(0))
    cfg = orc.RenderConfig(num_samples=S, num_fine_samples=0, use_biased_sampler=biased)
    e, sb = pl.place_coarse_bins(cfg, nears, fars, torch.from_numpy(num), hdt, kept, t_rand)
    base = orc.coarse_bins(cfg, nears, fars, torch.from_numpy(num), hdt, t_rand)
    return e.numpy(), sb.numpy(), base, hd, kept, num, (nears, fars)


# ray 0: kept / skipped alternating; ray 1: skipped first and last records, a gap record (between two hull faces) in the middle;
# ray 2: a gap between records (no record) and a skipped run of three cells.  occ: cell c has occ[c]
BOUNDS = [[(0, 1), (1, 3), (3, 4), (4, 8), (8, 9)],
          [(1, 2), (2, 2.5), (2.5, 4), (4, 4.5), (4.5, 7)],
          [(0, 0.5), (0.5, 1), (2, 3), (3, 3.25), (3.25, 3.5), (3.5, 6), (6, 7)]]
CELLS = [[0, 1, 2, 3, 4], [1, 0, -1, 2, 3], [0, 2, 1, 3, 5, 1, 4]]
OCC = [1.0, 0.0, 1.0, 0.0, 1.0, 0.0]  # odd cells are empty


def _in_kept(e, hd, kept, n):
    k = np.nonzero(kept[:n])[0]
    return bool(np.all([np.any((hd[k, 0] <= x) & (x <= hd[k, 1])) for x in e]))


@pytest.mark.parametrize("biased", [True, False])
@pytest.mark.parametrize("jitter", [False, True])
def test_edges_in_kept_records(biased, jitter):
    S = 48
    t_rand = torch.rand((len(BOUNDS), S + 1), generator=torch.Generator().manual_seed(1)) if jitter else None
    e, sb, base, hd, kept, num, (nears, fars) = _records(BOUNDS, CELLS, S, biased, t_rand, OCC)
    for r in range(len(BOUNDS)):
        assert _in_kept(e[r], hd[r], kept[r], num[r]), r
        assert np.all(np.diff(e[r]) >= 0), r
        assert e[r, 0] == hd[r, np.nonzero(kept[r])[0][0], 0] or jitter
        np.testing.assert_array_equal(sb[r], (e[r] - nears[r].numpy()) / (fars[r].numpy() - nears[r].numpy()))


def test_biased_equal_shares():
    S = 30  # three kept records on ray 0: 10 of the 31 edges each, plus one at a boundary (floor(u n_kept) rounds there)
    e, *_ , hd, kept, num, _ = _records(BOUNDS[:1], CELLS[:1], S, True, None, OCC)
    k = np.nonzero(kept[0])[0]
    which = [int(k[np.nonzero((hd[0, k, 0] <= x) & (x <= hd[0, k, 1]))[0][0]]) for x in e[0]]
    counts = [which.count(int(c)) for c in k]
    assert sum(counts) == S + 1 and all(c in (10, 11) for c in counts), counts
    for c in k:  # equal steps of len / 10 inside each kept record
        x = np.array([v for v, w in zip(e[0], which) if w == c])
        np.testing.assert_allclose(np.diff(x), (hd[0, c, 1] - hd[0, c, 0]) / 10, atol=2e-6)


def test_uniform_over_kept_length():
    S = 64
    for r in range(len(BOUNDS)):
        e, _, _, hd, kept, num, _ = _records([BOUNDS[r]], [CELLS[r]], S, False, None, OCC)
        k = np.nonzero(kept[0])[0]
        lens = hd[0, k, 1] - hd[0, k, 0]
        P = np.concatenate([[0], np.cumsum(lens)])
        # the compressed coordinate (kept length before the edge) of each edge: uniform steps of L / S
        comp = []
        for x in e[0]:
            i = max(i for i in range(len(k)) if hd[0, k[i], 0] <= x)
            comp.append(P[i] + min(x - hd[0, k[i], 0], lens[i]))
        np.testing.assert_allclose(np.diff(comp), P[-1] / S, atol=2e-6)


@pytest.mark.parametrize("biased", [True, False])
def test_nothing_or_everything_skipped_is_today(biased):
    S = 40
    t_rand = torch.rand((len(BOUNDS), S + 1), generator=torch.Generator().manual_seed(2))
    for occ in ([1.0] * 6, [0.0] * 6):
        cells = [[c if c >= 0 else 0 for c in cs] for cs in CELLS]  # no gap record: all skipped really is all
        e, sb, (be, bsb), *_ = _records(BOUNDS, cells, S, biased, t_rand, occ)
        assert np.array_equal(e, be.numpy()) and np.array_equal(sb, bsb.numpy())


def _straddle(e, hd, kept, n):
    """per bin: (midpoint kept, kept length, skipped length, skipped cells on one side of the midpoint)"""
    out = []
    for a, b in zip(e[:-1], e[1:]):
        m = (a + b) / 2
        kl = sl = 0.0
        left = right = False
        for k in range(n):
            lo, hi = max(a, hd[k, 0]), min(b, hd[k, 1])
            if hi <= lo:
                continue
            if kept[k]:
                kl += hi - lo
            else:
                sl += hi - lo
                left |= lo < m
                right |= hi > m
        mk = any(kept[k] and hd[k, 0] <= m <= hd[k, 1] for k in range(n))
        out.append((mk, kl, sl, not (left and right)))
    return out


@pytest.mark.parametrize("biased", [True, False])
@pytest.mark.parametrize("S", [3, 7, 16, 64])
def test_straddling_bound(biased, S):
    """a bin whose midpoint is in a kept record, with its skipped length on one side of the midpoint, holds at most as much skipped
    as kept length (DESIGN §4.13); every bin's kept length is at most one compressed bin"""
    e, _, _, hd, kept, num, _ = _records(BOUNDS, CELLS, S, biased, None, OCC)
    for r in range(len(BOUNDS)):
        n = int(num[r])
        L = float(sum(hd[r, k, 1] - hd[r, k, 0] for k in range(n) if kept[r, k]))
        for mk, kl, sl, one_side in _straddle(e[r], hd[r], kept[r], n):
            if mk and one_side:
                assert sl <= kl + 1e-6, (r, kl, sl)
            if not biased:
                assert kl <= L / S + 1e-5
    # the condition matters: skipped runs on both sides of a kept midpoint can hold more than the kept length
    e2, _, _, hd2, kept2, num2, _ = _records([[(0, 0.1), (0.1, 5), (5, 5.1), (5.1, 9.9), (9.9, 10)]], [[0, 1, 2, 3, 4]], 1, False, None, OCC)
    st = _straddle(e2[0], hd2[0], kept2[0], int(num2[0]))
    assert any(mk and not one and sl > kl for mk, kl, sl, one in st)


def test_oracle_render_places_in_kept_cells():
    """on surface_scene: the oracle's placed render has every coarse edge in a kept record, and fewer culled coarse samples"""
    V, C = syn.delaunay_mesh(400, seed=0)
    field, params = syn.surface_scene(V, 100, orc.init_mlp_params(0))
    mesh = orc.OracleMesh(V, C)
    o, d = syn.camera_rays(60, seed=3)
    occ = ocu.occupancy(field, params, C).float()
    F = torch.from_numpy(field)
    for biased in (True, False):
        cfg = orc.RenderConfig(num_samples=32, num_fine_samples=32, use_biased_sampler=biased)
        cull = ocu.render(mesh, F, params, o, d, cfg, occupancy=(occ, 0.01))
        got = pl.render(mesh, F, params, o, d, cfg, occupancy=(occ, 0.01))
        tr = got["aux"]["trace"]
        m = tr["num_visited_cells"] > 0
        hd, num, kept = tr["hit_distances"][m], tr["num_visited_cells"][m], got["aux"]["kept"]
        ce = got["aux"]["coarse_euclid"].numpy()
        for r in range(len(ce)):
            if 0 < kept[r].sum() < num[r]:
                assert _in_kept(ce[r], hd[r], kept[r], int(num[r]))
        fc, fp = cull["aux"]["coarse_culled"].float().mean().item(), got["aux"]["coarse_culled"].float().mean().item()
        assert fp < 0.5 * fc, (biased, fc, fp)
