"""The homogeneous medium's arithmetic (ezrt_math.h, DESIGN.md section 14) on the CPU: the Henyey-Greenstein sampler and density,
free flight, box clipping and transmittance against float64, and the restatement's renders -- a pure absorber, a white furnace,
unbiasedness against the phase-only estimator, equality with mode 4 where no segment meets the box, and hostile inputs."""
import numpy as np
import pytest
from scipy import stats

from ezrt_b200 import api, scenes
from tests import oracle_medium as om
from tests.test_light_sampling_laws import _block_z, _stats

G_VALUES = [-0.999, -0.9, -0.3, 0.0, 0.3, 0.9, 0.999]


def _peak_angles(g):
    """a grid of angles psi from the law's peak axis (d for g >= 0, -d for g < 0), dense at the peak"""
    return np.unique(np.concatenate([[0.0], np.geomspace(1e-9, 1e-3, 40000), np.linspace(1e-3, np.pi, 400000)]))


def _density_cdf_edges(g, K):
    """K + 1 bin edges in psi, equiprobable under the density ez_hg_pdf itself: its float64 cumulative integral
    2 pi int p(psi) sin(psi) dpsi over fp32 directions at angle psi from the peak axis, inverted by interpolation"""
    psi = _peak_angles(g)
    sgn = 1.0 if g >= 0 else -1.0
    L = np.stack([np.sin(psi), np.zeros_like(psi), sgn * np.cos(psi)], 1).astype(np.float32)
    d = np.tile(np.float32([0, 0, 1]), (psi.size, 1))
    f = 2 * np.pi * om.hg_pdf(d, L, g).astype(np.float64) * np.sin(psi)
    cdf = np.concatenate([[0.0], np.cumsum(0.5 * (f[1:] + f[:-1]) * np.diff(psi))])
    cdf /= cdf[-1]
    return np.interp(np.linspace(0, 1, K + 1), cdf, psi)


@pytest.mark.parametrize("g", G_VALUES)
def test_hg_sampler_chi_square(g):
    """the sampler's directions against the density function: cos bins equiprobable under ez_hg_pdf's own integral (independent of
    the sampler's closed-form inversion), phi bins uniform around d"""
    n, K, P = 1_000_000, 32, 16
    rng = np.random.default_rng(1234 + int(g * 1000))
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    h = rng.random((n, 2), dtype=np.float32)
    L, pdf = om.hg_sample(d.astype(np.float32), g, h)
    d32 = d.astype(np.float32).astype(np.float64)
    L64 = L.astype(np.float64)
    L64 /= np.linalg.norm(L64, axis=1, keepdims=True)
    # the angle from the peak axis, from the chord |d -+ L| (resolves the forward peak of g = 0.999 in float64)
    chord = np.linalg.norm(d32 - L64, axis=1) if g >= 0 else np.linalg.norm(d32 + L64, axis=1)
    psi = 2 * np.arcsin(np.clip(chord / 2, 0, 1))
    edges = _density_cdf_edges(g, K)
    cbin = np.clip(np.searchsorted(edges, psi, side="right") - 1, 0, K - 1)
    # phi around d in the frame of ez_to_normal_hemisphere
    helper = np.where(np.abs(d32[:, :1]) > 0.999, [[0, 0, 1.0]], [[1.0, 0, 0]])
    t = np.cross(d32, helper); t /= np.linalg.norm(t, axis=1, keepdims=True)
    b = np.cross(d32, t)
    phi = np.mod(np.arctan2(np.sum(L64 * b, 1), np.sum(L64 * t, 1)), 2 * np.pi)
    pbin = np.clip((phi / (2 * np.pi) * P).astype(int), 0, P - 1)
    counts = np.bincount(cbin * P + pbin, minlength=K * P)
    p = stats.chisquare(counts).pvalue
    print("g %g: chi-square p = %.3g" % (g, p))
    assert p > 1e-4
    # the pdf a medium vertex stores in its path record is the density function at the sampled direction, bit for bit
    assert np.array_equal(pdf, om.hg_pdf(d.astype(np.float32), L, g))


@pytest.mark.parametrize("g", G_VALUES)
def test_hg_pdf_integrates_to_one(g):
    # fp32 directions at angle theta from d = +z, theta on a grid dense at the peak; 2 pi int p sin(theta) dtheta
    peak = 0.0 if g >= 0 else np.pi
    u = np.concatenate([np.geomspace(1e-9, 1e-3, 40000), np.linspace(1e-3, np.pi, 200000)[1:]])
    th = np.sort(np.abs(peak - u))
    L = np.stack([np.sin(th), np.zeros_like(th), np.cos(th)], 1).astype(np.float32)
    d = np.tile(np.float32([0, 0, 1]), (th.size, 1))
    p = om.hg_pdf(d, L, g).astype(np.float64)
    total = 2 * np.pi * np.trapezoid(p * np.sin(th), th)
    assert abs(total - 1) < 1e-4, total


def test_free_flight_law():
    sigma = 0.7
    r = np.random.default_rng(5).random(1_000_000, dtype=np.float32)
    s = om.free_flight(r, sigma).astype(np.float64)
    edges = np.concatenate([-np.log(1 - np.linspace(0, 1, 65)[:-1]) / sigma, [np.inf]])
    counts = np.histogram(s, edges)[0]
    assert stats.chisquare(counts).pvalue > 1e-4


def _slab64(o, d, t_end, bmin, bmax):
    t0 = np.zeros(len(o)); t1 = np.array(t_end, np.float64)
    ok = np.ones(len(o), bool)
    for k in range(3):
        if not bmin[k] < bmax[k]:
            ok[:] = False
        par = d[:, k] == 0
        ok &= ~(par & ((o[:, k] < bmin[k]) | (o[:, k] > bmax[k])))
        with np.errstate(divide="ignore", invalid="ignore"):
            ta = (bmin[k] - o[:, k]) / d[:, k]; tb = (bmax[k] - o[:, k]) / d[:, k]
        lo, hi = np.where(par, -np.inf, np.minimum(ta, tb)), np.where(par, np.inf, np.maximum(ta, tb))
        t0 = np.maximum(t0, lo); t1 = np.minimum(t1, hi)
    return ok & (t0 < t1), t0, t1


@pytest.mark.parametrize("box", [((-1, -1, -1), (1, 1, 1)), ((0.2, -3, 0.5), (0.7, 3, 0.5001)), ((0, 0, 0), (1, 0, 1))])
def test_box_overlap_and_transmittance_against_float64(box):
    rng = np.random.default_rng(7)
    n = 20000
    o = rng.uniform(-2, 2, (n, 3)).astype(np.float32)
    o[: n // 4] = rng.uniform(-0.5, 0.5, (n // 4, 3))           # inside the box
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True); d = d.astype(np.float32)
    d[n // 4: n // 4 + 500, 0] = 0.0                                # parallel to the x faces
    d[n // 4 + 500: n // 4 + 1000, 1:] = 0.0; d[n // 4 + 500: n // 4 + 1000, 0] = 1.0
    t_end = rng.uniform(0.1, 6, n).astype(np.float32); t_end[:100] = np.inf
    bmin, bmax = np.float32(box[0]), np.float32(box[1])
    ok, t01 = om.box_overlap(o, d, t_end, bmin, bmax)
    ok64, t0, t1 = _slab64(o.astype(np.float64), d.astype(np.float64), t_end.astype(np.float64), bmin.astype(np.float64), bmax.astype(np.float64))
    clear = np.abs(t1 - t0) > 1e-4   # away from the grazing cases the two decide alike
    assert np.array_equal(ok[clear], ok64[clear])
    both = ok & ok64
    assert np.allclose(t01[both, 0], t0[both], atol=1e-5, rtol=1e-5) and np.allclose(t01[both, 1], t1[both], atol=1e-5, rtol=1e-5)
    sigma = 1.3
    T = om.transmittance(om.medium(sigma, box_min=bmin, box_max=bmax), o, d, t_end)
    T64 = np.where(ok64, np.exp(-sigma * np.clip(t1 - t0, 0, None)), 1.0)
    assert np.allclose(T[clear], T64[clear], rtol=2e-5, atol=1e-6)
    assert (T[~ok] == 1.0).all()


def _quad(z, half, mat):
    """two triangles of a square in the plane z facing +z (the camera at +z)"""
    p = [(-half, -half, z), (half, -half, z), (half, half, z), (-half, half, z)]
    tris = []
    for a, b, c in ((0, 1, 2), (0, 2, 3)):
        t = np.zeros(36, np.float32)
        t[0:3], t[3:6], t[6:9] = p[a], p[b], p[c]
        t[9:18] = [0, 0, 1] * 3
        t[18:21] = mat.emissive; t[21:24] = mat.baseColor
        t[24:36] = mat.as_array()[6:18]
        tris.append(t)
    return np.array(tris)


def _scene(tris):
    tl = api.TriangleList()
    tl.append_encoded(tris)
    return tl.build_bvh(8, api.BVH_SAH_FAST)


def test_pure_absorber():
    Le = 2.0
    emitter = api.Material(emissive=(Le, Le, Le), baseColor=(0, 0, 0))
    tris, nodes = _scene(_quad(0.0, 3.0, emitter))
    sigma, depth = 0.9, 1.5   # the box spans z in [0.5, 2.0]
    cfg = api.RenderConfig(width=16, height=16, spp=64, max_bounce=0, mode=api.MODE_DISNEY_LIGHTS, eye=(0, 0, 4), medium=True)
    m = om.medium(sigma, albedo=(0, 0, 0), box_min=(-5, -5, 0.5), box_max=(5, 5, 2.0))
    img = om.render(tris, nodes, cfg, m)[0]
    # every sample is Le (passed) or 0 (absorbed): the mean over pixels and frames against Le exp(-sigma * path length in the box)
    ys, xs = np.mgrid[0:16, 0:16]
    vx, vy = (xs + 0.5) / 16 * 2 - 1, (ys + 0.5) / 16 * 2 - 1
    cosz = 1.5 / np.sqrt(vx ** 2 + vy ** 2 + 1.5 ** 2)
    want = Le * np.exp(-sigma * depth / cosz)
    se = np.sqrt((want * (Le - want)).mean() / (cfg.spp * want.size))   # each sample is Le with probability want / Le, else 0
    print("absorber: mean %.5f, expected %.5f, SE %.5f" % (img[..., 0].mean(), want.mean(), se))
    assert abs(img[..., 0].mean() - want.mean()) < 3 * se


def test_white_furnace():
    # an empty scene but for a far invisible speck: env_color 1, a white non-absorbing medium around the camera
    speck = api.Material(baseColor=(0, 0, 0))
    tris, nodes = _scene(_quad(-1000.0, 1e-3, speck))
    cfg = api.RenderConfig(width=16, height=16, spp=8, max_bounce=64, mode=api.MODE_DISNEY_LIGHTS, eye=(0, 0, 0), env_color=(1, 1, 1), medium=True)
    m = om.medium(1.5, albedo=(1, 1, 1), g=0.3, box_min=(-2, -2, -2), box_max=(2, 2, 2))
    img = om.render(tris, nodes, cfg, m)[0]
    # a sample is 1 unless cut by the bounce cap (0); the mean per pixel is k / 8
    frac = np.round(img[..., 0] * 8) / 8
    assert np.array_equal(img[..., 0], frac.astype(np.float32)) or np.allclose(img[..., 0], frac, atol=1e-6)
    print("furnace: cut fraction %.4f" % (1 - float(img[..., 0].mean())))
    assert img.mean() > 0.9


def test_untouched_box_equals_mode4():
    tris, nodes, eye, cam = scenes.s_bunny()
    hdr = scenes.synth_hdr(64, 32)
    cache = api.hdr_cache(hdr)
    for kw in (dict(), dict(env_light=True), dict(lens_radius=0.1, focus_distance=3.5), dict(env_light=True, lens_radius=0.1, focus_distance=3.5)):
        cfg = api.RenderConfig(width=24, height=16, spp=2, max_bounce=3, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam), **kw)
        plain = om.render(tris, nodes, cfg, None, hdr=hdr, hdr_cache=cache)
        cfg.medium = True
        got = om.render(tris, nodes, cfg, om.medium(3.0, box_min=(40, 40, 40), box_max=(41, 41, 41)), hdr=hdr, hdr_cache=cache)
        assert got[0].tobytes() == plain[0].tobytes() and got[3] == plain[3]


def _unbiased_cases():
    hdr = scenes.synth_hdr(64, 32)
    bunny = scenes.s_p3_bunny()
    fog = dict(albedo=(0.9, 0.8, 0.7), g=0.5, box_min=(-1.2, -1.0, -1.2), box_max=(1.2, 1.4, 1.2))
    return [
        ("P3 bunny in a fog box", bunny, None, False, dict(sigma_t=0.8, **fog), {}),
        ("P3 bunny, dense fog, backward g", bunny, None, False, dict(sigma_t=3.0, albedo=(0.95, 0.95, 0.95), g=-0.6,
                                                                    box_min=(-2, -2, -2), box_max=(2, 2, 2)), {}),
        ("map sun through fog with ENV_LIGHT", bunny, hdr, True, dict(sigma_t=0.6, **fog), {}),
        ("lens render in fog", bunny, hdr, True, dict(sigma_t=0.8, **fog), dict(lens_radius=0.2, focus_distance=3.4)),
    ]


@pytest.mark.parametrize("k", range(4))
def test_unbiased_against_phase_only(k):
    name, (tris, nodes, eye, cam), hdr, env_light, fog, lens = _unbiased_cases()[k]
    cache = None if hdr is None else api.hdr_cache(hdr)
    W, H, spp = 32, 16, 64
    out = []
    for phase_only in (False, True):
        # the phase-only arm renders frames spp .. 2 spp - 1 (independent of the other arm's); from a zero framebuffer its running
        # means come out scaled by spp / (2 spp)
        first = spp if phase_only else 0
        cfg = api.RenderConfig(width=W, height=H, spp=spp, first_frame=first, max_bounce=6, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye),
                               camera_rotate=tuple(cam), env_color=(0.1, 0.1, 0.12), env_light=env_light, medium=True, **lens)
        img, luma2, _, _ = om.render(tris, nodes, cfg, om.medium(**fog), hdr=hdr, hdr_cache=cache, phase_only=phase_only)
        assert np.isfinite(img).all()
        scale = np.float64(first + spp) / spp
        y = _stats(img, luma2)[0] * scale
        out.append((y, np.maximum(luma2.astype(np.float64) * scale - y ** 2, 0.0)))
    z8 = _block_z(out[0], out[1], spp, W, H, 8, 8)
    zf = float(_block_z(out[0], out[1], spp, W, H, H, W).max())
    print("unbiased %-40s means %.5f / %.5f, frame z %.2f, largest 8x8 z %.2f" % (name, out[0][0].mean(), out[1][0].mean(), zf, z8.max()))
    assert zf <= 4, (name, zf)
    assert z8.max() <= 5, (name, z8.max())


def test_hostile_inputs():
    tris, nodes, eye, cam = scenes.s_bunny()
    cfg = api.RenderConfig(width=12, height=8, spp=1, max_bounce=4, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam), medium=True)
    for bad in (om.medium(-1), om.medium(np.inf), om.medium(np.nan), om.medium(1, albedo=(1.5, 0, 0)), om.medium(1, albedo=(np.nan, 0, 0)),
                om.medium(1, g=1.0), om.medium(1, g=-1.0), om.medium(1, g=np.nan), om.medium(1, box_min=(1, 0, 0), box_max=(0, 1, 1)),
                om.medium(1, box_max=(np.inf, 1, 1)), None):
        with pytest.raises(ValueError):
            om.render(tris, nodes, cfg, bad)
    good = om.medium(1.0, box_min=(-2, -2, -2), box_max=(2, 2, 2))
    for kw in (dict(mode=api.MODE_DISNEY_IS_MIS_P5), dict(pipeline=api.PIPELINE_MEGAKERNEL), dict(transmission=True)):
        c = api.RenderConfig(**{**cfg.__dict__, **kw})
        with pytest.raises(ValueError):
            om.render(tris, nodes, c, good)
    for m in (om.medium(2500.0, box_min=(-2, -2, -2), box_max=(2, 2, 2)), om.medium(1.0, g=0.999, box_min=(-2, -2, -2), box_max=(2, 2, 2)),
              om.medium(1.0, g=-0.999, box_min=(-2, -2, -2), box_max=(2, 2, 2))):
        assert np.isfinite(om.render(tris, nodes, cfg, m)[0]).all()
