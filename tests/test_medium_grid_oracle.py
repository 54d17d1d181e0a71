"""The density grid's definition (EZRT_PARAM_MEDIUM_GRID, ezrt_math.h, DESIGN.md section 20) against exact references, on the CPU:
the lookup against float64 trilinear, the majorant bound over hostile rays, the free-flight law against the float64 CDF, ratio
tracking's mean against exp(-tau), and the restatement's agreement with the header's functions."""
import numpy as np
import pytest
from scipy import stats

from tests import oracle_medium_grid as og

BOX = ((-1.0, -0.5, 0.25), (2.0, 1.5, 1.0))


def _plume(n, seed=3):
    """a seeded smooth grid [n, n, n] with empty regions and a dense core"""
    rng = np.random.default_rng(seed)
    z, y, x = np.meshgrid(*[np.linspace(0, 1, n)] * 3, indexing="ij")
    g = np.exp(-((x - 0.5) ** 2 + (y - 0.4) ** 2 + (z - 0.5) ** 2) / 0.05) * (1.0 - y)
    g += 0.3 * rng.random((n, n, n)) * (g > 0.1)
    return np.clip(g, 0, None).astype(np.float32)


def _dirs(rng, n):
    d = rng.normal(size=(n, 3))
    return (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


@pytest.mark.parametrize("shape", [(1, 1, 1), (2, 2, 2), (1, 5, 9), (7, 1, 3), (17, 9, 33), (24, 24, 24)])
def test_lookup_matches_float64_trilinear(shape):
    rng = np.random.default_rng(sum(shape))
    rho = (10.0 ** rng.uniform(-15, 15, size=shape)).astype(np.float32)   # 30 orders of magnitude
    rho[rng.random(shape) < 0.2] = 0.0
    lo, hi = np.array(BOX[0]), np.array(BOX[1])
    P = lo + (hi - lo) * rng.random((20000, 3))
    # hostile points: lattice points, faces, corners, beyond the box (clamped)
    n = np.array([shape[2], shape[1], shape[0]])
    lat = np.stack([rng.integers(0, n[a], 4000) / max(n[a] - 1, 1) for a in range(3)], 1)
    P = np.concatenate([P, lo + (hi - lo) * lat, lo + (hi - lo) * rng.integers(0, 2, (64, 3)), lo - 1 + (hi - lo + 2) * rng.random((500, 3))])
    P = P.astype(np.float32)
    got = og.density(rho, 1.0, *BOX, P).astype(np.float64)
    ref = og.rho64(rho, *BOX, P)
    # no lerp exceeds its corners: every value lies within its cell's corners
    assert np.all(np.isfinite(got)) and np.all(got >= 0)
    def corners(P64, lo, hi):
        u = [np.clip((P64[:, a] - lo[a]) / (hi[a] - lo[a]) * P64.dtype.type(n[a] - 1), 0, n[a] - 1) if n[a] > 1 else np.zeros(len(P)) for a in range(3)]
        cmax, cmin = np.zeros(len(P)), np.full(len(P), np.inf)
        for dk in (0, 1):
            for dj in (0, 1):
                for di in (0, 1):
                    c = [np.minimum(np.minimum(np.floor(u[a]).astype(int), max(n[a] - 2, 0)) + (di, dj, dk)[a], n[a] - 1) for a in range(3)]
                    v = rho.astype(np.float64)[c[2], c[1], c[0]]
                    cmax, cmin = np.maximum(cmax, v), np.minimum(cmin, v)
        return cmax, cmin
    # the cell of the definition's fp32 lattice coordinate bounds the lookup
    cell_max, cell_min = corners(P, lo.astype(np.float32), hi.astype(np.float32))
    assert np.all(got <= cell_max) and np.all(got >= cell_min)
    # against float64 to fp32 rounding of the coordinates and the seven lerps, relative to the largest corner of the two cells (the
    # fp32 and the float64 coordinate may fall on either side of a lattice plane)
    err = np.abs(got - ref) / np.maximum(np.maximum(cell_max, corners(P.astype(np.float64), lo, hi)[0]), 1e-300)
    assert np.max(err) < 2e-5, np.max(err)


def test_constant_grids_are_exact():
    for v in (0.0, 1.0, 3.25e-30, 7.5e30):
        rho = np.full((5, 6, 7), v, np.float32)
        P = np.random.default_rng(1).uniform(-2, 3, (5000, 3)).astype(np.float32)
        assert np.all(og.density(rho, 1.0, *BOX, P) == np.float32(v))


def test_brick_maxima_are_dilated_cell_maxima():
    rng = np.random.default_rng(5)
    rho = rng.random((19, 26, 33)).astype(np.float32)
    b = og.bricks(rho)
    assert b.shape == (3, 4, 4)
    for k in range(b.shape[0]):
        for j in range(b.shape[1]):
            for i in range(b.shape[2]):
                sl = tuple(slice(max(0, 8 * c - 1), min(n - 1, 8 * c + 9) + 1) for c, n in zip((k, j, i), rho.shape))
                assert b[k, j, i] == rho[sl].max()
    assert og.bricks(np.ones((1, 1, 1), np.float32)).shape == (1, 1, 1)
    assert og.bricks(np.ones((9, 9, 9), np.float32)).shape == (1, 1, 1)
    assert og.bricks(np.ones((10, 9, 2), np.float32)).shape == (2, 1, 1)


def _hostile_rays(rng, n, lo, hi, nlat):
    """origins and directions that stress the walk: axis-parallel rays, origins on faces and on brick boundaries, rays grazing edges"""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    ext = hi - lo
    o = lo - 0.25 * ext + 1.5 * ext * rng.random((n, 3))
    d = _dirs(rng, n).astype(np.float64)
    k = n // 5
    ax = rng.integers(0, 3, k)   # axis-parallel
    d[:k] = 0.0
    d[np.arange(k), ax] = rng.choice([-1.0, 1.0], k)
    # origins on brick boundaries (lattice coordinate a multiple of 8) and on faces
    b = slice(k, 2 * k)
    a = rng.integers(0, 3, k)
    frac = np.array([(8 * rng.integers(0, max(1, (nlat[x] - 1) // 8) + 1)) / max(nlat[x] - 1, 1) for x in a])
    oo = o[b].copy()
    oo[np.arange(k), a] = lo[a] + np.minimum(frac, 1.0) * ext[a]
    o[b] = oo
    f = slice(2 * k, 3 * k)   # on faces
    oo = lo + ext * rng.random((k, 3))
    a2 = rng.integers(0, 3, k)
    oo[np.arange(k), a2] = np.where(rng.random(k) < 0.5, lo[a2], hi[a2])
    o[f] = oo
    g = slice(3 * k, 4 * k)   # grazing an edge: along an axis through a box edge
    oo = lo + ext * rng.random((k, 3))
    a3 = rng.integers(0, 3, k)
    for t in range(k):
        others = [x for x in range(3) if x != a3[t]]
        for x in others:
            oo[t, x] = lo[x] if rng.random() < 0.5 else hi[x]
        oo[t, a3[t]] = lo[a3[t]] - 0.1 * ext[a3[t]]
    dd = np.zeros((k, 3))
    dd[np.arange(k), a3] = 1.0
    dd += 1e-7 * rng.normal(size=(k, 3))
    o[g], d[g] = oo, dd / np.linalg.norm(dd, axis=1, keepdims=True)
    return o.astype(np.float32), d.astype(np.float32)


@pytest.mark.parametrize("box", [BOX, ((-1e-4, 0, 0), (1e-4, 2e-4, 1e-4)), ((-3e5, -1e5, -2e5), (3e5, 1e5, 4e5))], ids=["unit", "tiny", "huge"])
def test_majorant_bound_over_hostile_rays(box):
    rng = np.random.default_rng(11)
    rho = _plume(41)
    lo, hi = np.array(box[0]), np.array(box[1])
    sigma_t = float(4.0 / np.max(hi - lo))   # a few mean free paths across
    n = 500000
    o, d = _hostile_rays(rng, n, lo, hi, (41, 41, 41))
    L = np.full(n, np.float32(np.inf))
    seed = rng.integers(1, 2 ** 32 - 1, n, dtype=np.uint64).astype(np.uint32)
    tot = 0
    for which in (1, 2):
        r = og.track(rho, sigma_t, *box, which, o, d, L, seed)
        assert r["violations"] == 0
        assert np.array_equal(r["out"].view(np.uint32), r["out2"].view(np.uint32)) and np.array_equal(r["seed"], r["seed2"])
        if which == 1:
            assert np.array_equal(r["flag"], r["flag2"])
        else:
            assert np.all((r["out"] >= 0) & (r["out"] <= 1))
        tot += r["collisions"]
    assert tot > n // 10   # the rays do collide


def _tau64(rho, sigma_t, lo, hi, o, d, t):
    """float64 optical depth from 0 to each t (sorted grid of t) along one ray, by the trapezoid rule on a fine grid"""
    ts = np.linspace(0, t[-1], 200001)
    s = sigma_t * og.rho64(rho, lo, hi, o[None, :].astype(np.float64) + ts[:, None] * d[None, :].astype(np.float64))
    P = np.asarray(o, np.float64)[None, :] + ts[:, None] * np.asarray(d, np.float64)[None, :]
    inside = np.all((P >= np.asarray(lo)) & (P <= np.asarray(hi)), axis=1)
    s = s * inside
    cum = np.concatenate([[0], np.cumsum(0.5 * (s[1:] + s[:-1]) * np.diff(ts))])
    return np.interp(t, ts, cum)


def test_free_flight_law_matches_float64_cdf():
    rho = _plume(33)
    lo, hi = (0.0, 0.0, 0.0), (1.0, 1.0, 1.0)
    o = np.array([-0.2, 0.35, 0.45], np.float32)
    d = np.array([1.0, 0.1, 0.05], np.float32)
    d = (d / np.linalg.norm(d)).astype(np.float32)
    sigma_t = 3.0
    n = 1000000
    seed = np.random.default_rng(2).integers(1, 2 ** 32 - 1, n, dtype=np.uint64).astype(np.uint32)
    r = og.track(rho, sigma_t, lo, hi, 1, np.tile(o, (n, 1)), np.tile(d, (n, 1)), np.inf, seed, twin=False)
    t_s = r["out"][r["flag"] == 1].astype(np.float64)
    edges = np.linspace(0.2, 1.25, 41)
    cdf = 1.0 - np.exp(-_tau64(rho, sigma_t, lo, hi, o, d, edges))
    p = np.diff(cdf)
    p_escape = 1.0 - cdf[-1]
    obs = np.concatenate([np.histogram(t_s, edges)[0], [n - len(t_s)]])
    exp = n * np.concatenate([p, [p_escape]])
    keep = exp > 20
    chi2 = np.sum((obs[keep] - exp[keep]) ** 2 / exp[keep])
    pval = stats.chi2.sf(chi2, keep.sum() - 1)
    assert pval > 1e-4, (chi2, keep.sum(), pval)


@pytest.mark.parametrize("sigma_t", [0.5, 3.0, 40.0])
def test_ratio_tracking_mean_is_transmittance(sigma_t):
    rho = _plume(33)
    lo, hi = (0.0, 0.0, 0.0), (1.0, 1.0, 1.0)
    o = np.array([0.1, 0.2, 0.5], np.float32)
    d = np.array([0.8, 0.5, -0.1], np.float32)
    d = (d / np.linalg.norm(d)).astype(np.float32)
    L = np.float32(0.9)
    n = 1000000
    seed = np.random.default_rng(int(sigma_t * 10)).integers(1, 2 ** 32 - 1, n, dtype=np.uint64).astype(np.uint32)
    r = og.track(rho, sigma_t, lo, hi, 2, np.tile(o, (n, 1)), np.tile(d, (n, 1)), L, seed, twin=False)
    T = r["out"].astype(np.float64)
    assert np.all((T >= 0) & (T <= 1))
    ref = np.exp(-_tau64(rho, sigma_t, lo, hi, o, d, np.array([float(L)]))[0])
    z = (T.mean() - ref) / (T.std(ddof=1) / np.sqrt(n))
    assert abs(z) < 4.5, (T.mean(), ref, z)


def test_zero_grid_and_missed_box_draw_nothing():
    rng = np.random.default_rng(4)
    n = 20000
    o = rng.uniform(-2, 2, (n, 3)).astype(np.float32)
    d = _dirs(rng, n)
    seed = rng.integers(1, 2 ** 32 - 1, n, dtype=np.uint64).astype(np.uint32)
    r = og.track(np.zeros((9, 9, 9), np.float32), 5.0, *BOX, 1, o, d, np.inf, seed)
    assert np.all(r["flag"] == 0) and np.array_equal(r["seed"], seed) and r["collisions"] == 0
    r = og.track(np.zeros((9, 9, 9), np.float32), 5.0, *BOX, 2, o, d, np.inf, seed)
    assert np.all(r["out"] == 1.0) and r["collisions"] == 0


def test_shadow_streams_differ_by_pixel_frame_and_bounce():
    px, py, f, b = np.meshgrid(np.arange(16), np.arange(16), np.arange(8), np.arange(8), indexing="ij")
    s = og.shadow_seed(px, py, f, b)
    assert len(np.unique(s)) == s.size


def _stepped():
    """a grid whose density reaches its brick maximum over whole bricks: 1 in x-brick 0, 2 in x-brick 1 (17 points, 2 bricks)"""
    g = np.ones((3, 3, 17), np.float32)
    g[:, :, 9:] = 2.0
    return g


@pytest.mark.parametrize("scale", [1.0, 0.9])
def test_laws_catch_a_majorant_below_sigma(scale):
    """the flight-law and ratio-tracking tests hold the definition (scale 1) and reject brick maxima scaled by 0.9"""
    rho = _stepped()
    lo, hi = (0.0, 0.0, 0.0), (1.0, 1.0, 1.0)
    o = np.array([-0.1, 0.5, 0.5], np.float32)
    d = np.array([1.0, 0.0, 0.0], np.float32)
    sigma_t, n = 1.5, 400000
    seed = np.random.default_rng(9).integers(1, 2 ** 32 - 1, n, dtype=np.uint64).astype(np.uint32)
    r = og.track(rho, sigma_t, lo, hi, 1, np.tile(o, (n, 1)), np.tile(d, (n, 1)), np.inf, seed, twin=False, brick_scale=scale)
    edges = np.linspace(0.1, 1.1, 21)
    cdf = 1.0 - np.exp(-_tau64(rho, sigma_t, lo, hi, o, d, edges))
    t_s = r["out"][r["flag"] == 1].astype(np.float64)
    obs = np.concatenate([np.histogram(t_s, edges)[0], [n - len(t_s)]])
    exp = n * np.concatenate([np.diff(cdf), [1.0 - cdf[-1]]])
    pval = stats.chi2.sf(np.sum((obs - exp) ** 2 / exp), len(exp) - 1)
    r = og.track(rho, sigma_t, lo, hi, 2, np.tile(o, (n, 1)), np.tile(d, (n, 1)), np.float32(1.05), seed, twin=False, brick_scale=scale)
    T = r["out"].astype(np.float64)
    ref = np.exp(-_tau64(rho, sigma_t, lo, hi, o, d, np.array([1.05]))[0])
    z = (T.mean() - ref) / (T.std(ddof=1) / np.sqrt(n))
    print("scale %.1f: flight chi-square p %.3g, ratio tracking z %.1f, violations %d" % (scale, pval, z, r["violations"]))
    if scale == 1.0:
        assert pval > 1e-4 and abs(z) < 4.5 and r["violations"] == 0
    else:
        assert pval < 1e-6 and abs(z) > 6 and r["violations"] > 0
