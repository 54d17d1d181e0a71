"""The materials' transmission (EZRT_PARAM_TRANSMISSION, ezrt_math.h, DESIGN.md section 12) on the CPU restatement
(tests/oracle_transmission.cpp): the sampler's law against the pdf, Fresnel against float64, reciprocity, albedo, a white furnace,
a smooth slab against its closed form, the estimator against a BSDF-only one, and the flag's behaviour on scenes without glass
and on hostile materials."""
import numpy as np
import pytest
from scipy import stats

from ezrt_b200 import api, scenes
from tests import oracle_env_light as oe
from tests import oracle_transmission as ot
from tests import transmission_scenes as ts
from tests.test_light_sampling_laws import NC, NPHI, _bin_integrals, _block_z, _dirs, _frame, _stats

L4 = api.MODE_DISNEY_LIGHTS
N_DIRS = 1_000_000


def _mat(roughness, ior, t=1.0, metallic=0.0, color=(0.8, 0.6, 0.4)):
    return api.Material(baseColor=color, roughness=roughness, IOR=ior, transmission=t, metallic=metallic).as_array()


def law_inputs(n, seed):
    """random (V, N, L, xi, inside, material) tuples over the law tests' parameter ranges, L on the whole sphere"""
    rng = np.random.default_rng(seed)
    N = rng.normal(size=(n, 3)); N /= np.linalg.norm(N, axis=1, keepdims=True)
    V = rng.normal(size=(n, 3)); V /= np.linalg.norm(V, axis=1, keepdims=True)
    V = np.where((np.einsum("ij,ij->i", V, N) < 0)[:, None], -V, V)
    L = rng.normal(size=(n, 3)); L /= np.linalg.norm(L, axis=1, keepdims=True)
    xi = rng.random((n, 4), dtype=np.float32)
    inside = rng.integers(0, 2, n).astype(np.int32)
    rough = rng.choice([0.0, 0.1, 0.3, 0.8], n)
    ior = rng.choice([1.5, 1.33, 2.4, 0.67, 1.0, 1.0 + 2.0 ** -9], n)
    t = rng.choice([1.0, 0.5], n)
    met = rng.choice([0.0, 0.5], n)
    mats = np.stack([_mat(r, i, tt, m) for r, i, tt, m in zip(rough, ior, t, met)])
    f = lambda a: a.astype(np.float32)
    return f(V), f(N), f(L), xi, inside, mats


# ------------------------------------------------------------------ 1. the sampling law
# (roughness, IOR, inside, cos_v, transmission, metallic): every value of each parameter appears
LAW_CASES = [
    (0.3, 1.5, 0, 1.0, 1.0, 0.0), (0.3, 1.5, 1, 0.5, 1.0, 0.0), (0.3, 1.33, 0, 0.05, 1.0, 0.0), (0.1, 1.5, 0, 0.5, 1.0, 0.0),
    (0.1, 2.4, 1, 1.0, 1.0, 0.0), (0.8, 0.67, 0, 0.5, 1.0, 0.0), (0.8, 2.4, 0, 0.05, 0.5, 0.0), (0.3, 0.67, 1, 0.5, 0.5, 0.5),
    (0.3, 1.33, 1, 0.05, 1.0, 0.0), (0.1, 1.33, 0, 0.05, 0.5, 0.5), (0.8, 1.5, 1, 1.0, 0.5, 0.0),
]


def _law_case(case, seed):
    rough, ior, inside, cos_v, t, met = case
    n, tv, _ = _frame()
    V = (cos_v * n + np.sqrt(1 - cos_v * cos_v) * tv).astype(np.float32)
    N = n.astype(np.float32)
    mat = _mat(rough, ior, t, met)
    xi = np.random.default_rng(seed).random((N_DIRS, 4), dtype=np.float32)
    b = lambda a, k: np.broadcast_to(a, (k,) + a.shape)
    ins = np.full(N_DIRS, inside, np.int32)
    s = ot.eval_bsdf(2, b(V, N_DIRS), b(N, N_DIRS), None, xi, ins, b(mat, N_DIRS))
    L = s[:, :3].astype(np.float64)
    ended = (s[:, :3] == 0).all(1)
    # the sampler's pdf is the pdf function's, bit for bit
    ok = ~ended
    pdf_fn = ot.eval_bsdf(1, b(V, ok.sum()), b(N, ok.sum()), s[ok, :3], None, ins[ok], b(mat, ok.sum()))[:, 0]
    assert s[ok, 6].tobytes() == pdf_fn.tobytes(), case
    c = L @ n.astype(np.float32).astype(np.float64)
    phi = np.mod(np.arctan2(L @ np.cross(n, tv), L @ tv), 2 * np.pi)
    ic = np.minimum((np.abs(c) * NC).astype(int), NC - 1)
    ib = ic * NPHI + np.minimum((phi / (2 * np.pi) * NPHI).astype(int), NPHI - 1) + np.where(c < 0, NC * NPHI, 0)
    obs = np.append(np.bincount(ib[ok], minlength=2 * NC * NPHI), ended.sum()).astype(np.float64)

    def pdf(sign):
        def f(cc, pp):
            d = _dirs(sign * cc, pp).astype(np.float32)
            k = len(d)
            return ot.eval_bsdf(1, b(V, k), b(N, k), d, None, np.full(k, inside, np.int32), b(mat, k))[:, 0].astype(np.float64)
        return f

    p = np.concatenate([_bin_integrals(pdf(1.0)), _bin_integrals(pdf(-1.0))])
    exp = N_DIRS * np.append(p, max(0.0, 1.0 - p.sum()))
    if rough <= 0.1:
        # alpha 0.01: the bin quadrature misses about 5e-4 of the lobe's mass (as for the BRDF at roughness 0.05,
        # tests/test_light_sampling_laws.py), which would all land in "path ends": the directions are compared given that the
        # path goes on, and the path-ends fraction is printed
        exp = np.append(p / p.sum() * ok.sum(), 0.0)
        obs = obs.copy()
        obs[-1] = 0.0
    small = exp < 5
    e = np.append(exp[~small], exp[small].sum())
    o = np.append(obs[~small], obs[small].sum())
    keep = e > 0
    chi2 = float((((o - e) ** 2)[keep] / e[keep]).sum() + (o[~keep].sum() if (~keep).any() else 0.0) * 1e12)
    dof = int(keep.sum()) - 1
    return chi2, dof, float(stats.chi2.sf(chi2, dof)), float(obs[-1] / N_DIRS), float(1.0 - p.sum()), float((c[ok] < 0).mean())


@pytest.mark.parametrize("case", LAW_CASES, ids=lambda c: "r%g-ior%g-in%d-cos%g-t%g-m%g" % c)
def test_sampler_density_is_the_mixture_pdf(case):
    chi2, dof, pval, ends, ends_exp, below = _law_case(case, seed=int(sum(case) * 1000) % 100003)
    print("law %r: chi2 %.1f / %d dof (p %.3g), path ends %.4f (expected %.4f), below %.4f" % (case, chi2, dof, pval, ends, ends_exp, below))
    assert pval > 1e-4, (case, chi2, dof)


# ------------------------------------------------------------------ 2. the functions' laws
def test_fresnel_against_float64():
    rng = np.random.default_rng(1)
    c = rng.random(200000).astype(np.float32)
    eta = rng.choice(np.array([1.5, 1.33, 2.4, 0.67, 1 / 1.5, 1 / 2.4], np.float32), c.size)
    got = ot.fresnel(c, eta).astype(np.float64)
    c64, e64 = c.astype(np.float64), eta.astype(np.float64)
    s2 = (1 - c64 * c64) / (e64 * e64)
    ct = np.sqrt(np.maximum(0.0, 1 - s2))
    rs = (c64 - e64 * ct) / (c64 + e64 * ct)
    rp = (e64 * c64 - ct) / (e64 * c64 + ct)
    want = np.where(s2 >= 1, 1.0, 0.5 * (rs * rs + rp * rp))
    clear = np.abs(s2 - 1) > 1e-5   # away from the critical angle, where fp32 decides which side s2 lies on
    err = np.abs(got - want)
    # near the critical angle cos_t = sqrt(1 - s2) amplifies the rounding of s2: fp32 holds F to 1e-4 there, to 2e-6 elsewhere
    assert err[clear].max() <= 1e-4 and err[np.abs(s2 - 1) > 1e-2].max() <= 2e-6, (err[clear].max(), err[np.abs(s2 - 1) > 1e-2].max())
    assert (got[clear & (s2 > 1)] == 1.0).all()          # total internal reflection exactly beyond the critical angle
    assert (got[clear & (s2 < 1)] < 1.0).all()


def test_reciprocity_of_the_btdf():
    """f(V -> L) / eta_V^2 = f(L -> V) / eta_L^2 (radiance convention; Veach 1997, section 5.2), evaluated from both sides"""
    rng = np.random.default_rng(2)
    n = 50000
    N = np.tile(np.array([0.0, 0.0, 1.0], np.float32), (n, 1))
    th_v, th_l = np.arccos(rng.uniform(0.1, 1.0, n)), np.arccos(rng.uniform(0.1, 1.0, n))
    ph_v, ph_l = rng.uniform(0, 2 * np.pi, n), rng.uniform(0, 2 * np.pi, n)
    V = np.stack([np.sin(th_v) * np.cos(ph_v), np.sin(th_v) * np.sin(ph_v), np.cos(th_v)], 1).astype(np.float32)
    L = np.stack([np.sin(th_l) * np.cos(ph_l), np.sin(th_l) * np.sin(ph_l), -np.cos(th_l)], 1).astype(np.float32)
    for rough in (0.1, 0.3, 0.8):
        for ior in (1.5, 1.33, 2.4, 0.67):
            mats = np.tile(_mat(rough, ior, color=(1, 1, 1)), (n, 1))
            f_vl = ot.eval_bsdf(0, V, N, L, None, np.zeros(n, np.int32), mats)[:, 0].astype(np.float64)   # V outside (eta_V = 1)
            f_lv = ot.eval_bsdf(0, L, -N, V, None, np.ones(n, np.int32), mats)[:, 0].astype(np.float64)   # L inside (eta_L = IOR)
            # the pairs away from grazing microfacets (|V.h|, |L.h| > 0.1): at V.h -> 0 one side is at the critical angle, where
            # 1 - F and so f are ill-conditioned in fp32 (there the two sides differ by up to 12 % relative, on 4 % of the pairs)
            h = -(V.astype(np.float64) + ior * L.astype(np.float64))
            h /= np.linalg.norm(h, axis=1, keepdims=True)
            cond = (np.abs((V * h).sum(1)) > 0.1) & (np.abs((L * h).sum(1)) > 0.1)
            both = (f_vl > 0) & (f_lv > 0)
            assert both.sum() > 1000, (rough, ior, both.sum())   # random pairs: many have no microfacet normal that refracts V into L
            assert ((f_vl > 0) == (f_lv > 0)).mean() > 0.999, (rough, ior)
            rel = np.abs(f_vl * ior * ior - f_lv) / np.where(both, f_lv, 1.0)
            print("reciprocity roughness %g IOR %g: %d pairs, largest relative difference %.2e (%d conditioned pairs: %.2e)" %
                  (rough, ior, both.sum(), rel[both].max(), (both & cond).sum(), rel[both & cond].max()))
            # and D's slope: an fp32 rounding of h moves a narrow lobe's D by up to 1e-3 relative at a few pairs
            r = rel[both & cond]
            assert r.size > 1000 and np.quantile(r, 0.99) <= 1e-4 and r.max() <= 2e-3, (rough, ior, np.quantile(r, 0.99), r.max())


@pytest.mark.parametrize("rough", [0.0, 0.1, 0.3, 0.8])
def test_white_lobe_albedo(rough):
    """E[f |cos| / pdf] of a white dielectric lobe in flux: a refracted sample's weight times eta^2, since radiance scales by
    1 / eta^2 across the interface.  At most 1 (plus 3 standard errors); within 1e-3 of 1 for a smooth surface."""
    n, tv, _ = _frame()
    N = n.astype(np.float32)
    k = 400000
    for ior in (1.5, 1.33, 2.4, 0.67):
        for inside in (0, 1):
            for cos_v in (1.0, 0.5, 0.05):
                V = (cos_v * n + np.sqrt(1 - cos_v * cos_v) * tv).astype(np.float32)
                xi = np.random.default_rng(int(ior * 100) + inside * 7 + int(cos_v * 1000)).random((k, 4), dtype=np.float32)
                mat = _mat(rough, ior, color=(1, 1, 1))
                s = ot.eval_bsdf(2, np.broadcast_to(V, (k, 3)), np.broadcast_to(N, (k, 3)), None, xi, np.full(k, inside, np.int32),
                                 np.broadcast_to(mat, (k, 18))).astype(np.float64)
                w = np.where(s[:, 6] > 0, s[:, 3] * np.abs(s[:, 7]) / np.where(s[:, 6] > 0, s[:, 6], 1.0), 0.0)
                eta = ior if inside == 0 else 1.0 / ior
                w = np.where(s[:, 7] < 0, w * eta * eta, w)
                m, se = w.mean(), w.std() / np.sqrt(k)
                assert np.isfinite(w).all()
                assert m <= 1 + 3 * se + 1e-6, (rough, ior, inside, cos_v, m, se)
                if rough == 0.0:
                    assert abs(m - 1) <= 1e-3, (ior, inside, cos_v, m)


# ------------------------------------------------------------------ 3. furnace, 4. slab
def _furnace_scene():
    tl = api.TriangleList()
    tl.read_obj_text(scenes.sphere_obj(), ts.glass(0.0, 1.5), api.transform_matrix((0, 0, 0), (0, 0, 0), (1, 1, 1)), False)
    tris, nodes = tl.build_bvh(8)
    eye, cam = api.camera_orbit(0.0, 0.0, 3.0)
    return np.asarray(tris, np.float32).reshape(-1, 36), nodes, eye, cam


def test_white_furnace():
    tris, nodes, eye, cam = _furnace_scene()
    cfg = api.RenderConfig(width=160, height=160, spp=1, max_bounce=32, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam), env_color=(1, 1, 1),
                           transmission=True)
    img, _, _ = ot.oracle_render_transmission(tris, nodes, cfg)   # one sample per pixel: every pixel value is one sample
    y = (0.3 * img[..., 0] + 0.6 * img[..., 1] + 0.1 * img[..., 2]).ravel()
    cut = y < 0.5
    print("furnace: %d samples, %.3f %% cut, largest |L - 1| of the others %.2e" % (y.size, 100 * cut.mean(), np.abs(y[~cut] - 1).max()))
    assert cut.mean() < 0.01
    # alpha = 0.001, not a delta: a sample's weight G (V.h) / ((N.V) (N.h)) differs from 1 by about 1e-3 / (N.V), so grazing
    # samples (about 1 %) leave 1e-3; the escaping samples' mean is 1 within 1e-5
    d = np.abs(y[~cut] - 1)
    assert (d <= 1e-3).mean() >= 0.98 and abs(y[~cut].mean() - 1) <= 1e-4, ((d <= 1e-3).mean(), y[~cut].mean())


def _slab_scene(roughness=0.0, ior=1.5, emitter=(4.0, -1.5, 2.0)):
    """a glass slab (2.4 x 2.4 x 0.4, centred at z = 0.5) between the camera and a black, non-reflecting square emitter on a black
    environment; emitter = (half size, z, emission), default 8 x 8 at z = -1.5 with emission 2, None: no emitter"""
    tl = api.TriangleList()
    tl.read_obj_text(scenes.box_obj(), ts.glass(roughness, ior), api.transform_matrix((0, 0, 0), (0, 0, 0.5), (1.2, 1.2, 0.2)), False)
    if emitter is not None:
        size, z, e = emitter
        tl.read_obj_text(scenes.box_obj(), api.Material(emissive=(e, e, e), baseColor=(0, 0, 0), specular=0.0),
                         api.transform_matrix((0, 0, 0), (0, 0, z), (size, size, 0.01)), False)
    tris, nodes = tl.build_bvh(8)
    eye, cam = api.camera_orbit(0.0, 0.0, 4.0)
    return np.asarray(tris, np.float32).reshape(-1, 36), nodes, eye, cam


@pytest.mark.parametrize("max_bounce", [2, 4, 6])
def test_smooth_slab_closed_form(max_bounce):
    tris, nodes, eye, cam = _slab_scene()
    spp = 512
    cfg = api.RenderConfig(width=64, height=64, spp=spp, max_bounce=max_bounce, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam),
                           transmission=True)
    img, luma2, _ = ot.oracle_render_transmission(tris, nodes, cfg, window=(28, 28, 36, 36))
    y, var = _stats(img, luma2)
    F = ((1.5 - 1) / (1.5 + 1)) ** 2
    K = (max_bounce - 2) // 2 + 1   # a path with k internal round trips reaches the emitter at bounce 2 + 2 k
    want = 2.0 * (1 - F) ** 2 * sum(F ** (2 * k) for k in range(K))
    z = abs(y.mean() - want) / np.sqrt(var.sum() / spp / y.size ** 2)
    print("slab max_bounce %d: %.6f against %.6f, z %.2f" % (max_bounce, y.mean(), want, z))
    assert z <= 5


# ------------------------------------------------------------------ 5. the estimator against the BSDF-only one
def _sun_map():
    """synth_hdr(64, 32) dimmed, with a 2 x 2 texel sun of luminance 5000 straight behind the slab (direction -z: u = 0.25, v = 0.5)"""
    hdr = scenes.synth_hdr(64, 32) * np.float32(0.02)
    hdr[15:17, 15:17] = 5000.0
    return hdr


# (name, scene, map, env light, bounces, spp, image, block statistics asserted)
def _unbiased_cases():
    hdr = scenes.synth_hdr(64, 32)
    return [
        ("rough glass blob on the P3 floor", ts.p3_glass("blob", ts.glass(0.3)), None, False, 4, 256, (64, 48), True),
        ("the same under a map, env light", ts.p3_glass("blob", ts.glass(0.3)), hdr, True, 4, 256, (64, 48), True),
        # a small bright light seen only through rough glass: every light sample is shadowed by the glass, and a refracted BSDF
        # sample's light pdf is far above its own, so an MIS weight on that hit in place of 1 loses almost all of its light
        ("small light behind rough glass (0.8)", _slab_scene(0.8, emitter=(0.25, -0.5, 20.0)), None, False, 4, 256, (32, 32), True),
        ("smooth glass blob (frame only)", ts.p3_glass("blob", ts.glass(0.0)), None, False, 6, 256, (64, 48), False),
        # the same for the environment: refracted exits that reach a small sun of the map, with the map as a light
        ("map sun behind rough glass (0.8), env light", _slab_scene(0.8, emitter=None), _sun_map(), True, 4, 256, (32, 32), True),
    ]


@pytest.mark.parametrize("k", range(5))
def test_estimator_agrees_with_bsdf_samples_only(k):
    name, (tris, nodes, eye, cam), hdr, env_light, bounces, spp, (W, H), blocks = _unbiased_cases()[k]
    cache = None if hdr is None else api.hdr_cache(hdr)
    out = []
    for bsdf_only in (False, True):
        # the BSDF-only arm renders frames spp .. 2 spp - 1, so that its samples are independent of the flagged arm's; from a zero
        # framebuffer its running means come out scaled by spp / (2 spp)
        first = spp if bsdf_only else 0
        cfg = api.RenderConfig(width=W, height=H, spp=spp, first_frame=first, max_bounce=bounces, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam),
                               env_color=(0.1, 0.1, 0.12), transmission=True, env_light=env_light)
        img, luma2, _ = ot.oracle_render_transmission(tris, nodes, cfg, hdr=hdr, hdr_cache=cache, bsdf_only=bsdf_only)
        assert np.isfinite(img).all()
        scale = np.float64(first + spp) / spp
        y = _stats(img, luma2)[0] * scale
        out.append((y, np.maximum(luma2.astype(np.float64) * scale - y ** 2, 0.0)))
    z8, z16 = _block_z(out[0], out[1], spp, W, H, 8, 8), _block_z(out[0], out[1], spp, W, H, 16, 16)
    zf = float(_block_z(out[0], out[1], spp, W, H, H, W).max())
    print("unbiased %-44s means %.5f / %.5f, frame z %.2f, largest 16x16 z %.2f, largest 8x8 z %.2f, variance ratio %.1f" %
          (name, out[0][0].mean(), out[1][0].mean(), zf, z16.max(), z8.max(), out[1][1].mean() / max(out[0][1].mean(), 1e-30)))
    assert zf <= 4, (name, zf)
    if blocks:
        assert z16.max() <= 5 and z8.max() <= 5, (name, z16.max(), z8.max())


# ------------------------------------------------------------------ 6. unchanged behaviour and hostile materials
def test_flag_without_glass_is_mode_4():
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    hdr = scenes.synth_hdr(64, 32)
    cache = api.hdr_cache(hdr)
    for h, c, env_light in ((None, None, False), (hdr, cache, False), (hdr, cache, True)):
        cfg = api.RenderConfig(width=48, height=32, spp=2, max_bounce=4, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam),
                               env_color=(0.3, 0.4, 0.5), env_light=env_light)
        want, wl, wc = oe.oracle_render_env_light(tris, nodes, cfg, hdr=h, hdr_cache=c)
        cfg.transmission = True
        got, gl, gc = ot.oracle_render_transmission(tris, nodes, cfg, hdr=h, hdr_cache=c)
        assert got.tobytes() == want.tobytes() and gl.tobytes() == wl.tobytes(), (h is not None, env_light)
        assert gc["rays"] == wc["rays"]


HOSTILE = [("ior %s" % v, dict(ior=v)) for v in ("1", "1+2^-9", "1-2^-9", "1+2^-7", "1-2^-7", "0", "-1", "nan", "inf", "1e6")] + \
          [("transmission %s" % v, dict(t=v)) for v in ("nan", "-1", "2")] + [("metallic 1, transmission 1", dict(metallic=1.0))]
_IOR = {"1": 1.0, "1+2^-9": 1 + 2.0 ** -9, "1-2^-9": 1 - 2.0 ** -9, "1+2^-7": 1 + 2.0 ** -7, "1-2^-7": 1 - 2.0 ** -7, "0": 0.0, "-1": -1.0,
        "nan": float("nan"), "inf": float("inf"), "1e6": 1e6}


def hostile_scene(name):
    kw = dict(HOSTILE)[name]
    ior = _IOR[kw["ior"]] if "ior" in kw else 1.5
    t = {"nan": float("nan"), "-1": -1.0, "2": 2.0}[kw["t"]] if "t" in kw else 1.0
    return ts.p3_glass("blob", ts.glass(0.3, ior, color=(0.9, 0.8, 0.7), transmission=t, metallic=kw.get("metallic", 0.0)))


@pytest.mark.parametrize("name", [h[0] for h in HOSTILE])
def test_hostile_materials_are_finite_and_defined(name):
    tris, nodes, eye, cam = hostile_scene(name)
    cfg = api.RenderConfig(width=32, height=24, spp=2, max_bounce=4, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam), env_color=(1, 1, 1),
                           transmission=True)
    img, _, _ = ot.oracle_render_transmission(tris, nodes, cfg)
    assert np.isfinite(img).all(), name
    opaque = name in ("ior 0", "ior -1", "ior nan", "ior inf", "transmission nan", "transmission -1", "metallic 1, transmission 1")
    if opaque:   # t = 0: the plain mode-4 render, bit for bit
        cfg.transmission = False
        want, _, _ = ot.oracle_render_transmission(tris, nodes, cfg)
        assert img.tobytes() == want.tobytes(), name


def test_index_matched_pass_through():
    """|IOR - 1| <= 2^-8 with t = 1: every BSDF sample passes straight through with weight baseColor"""
    V, N, _, _, _, _ = law_inputs(1000, seed=9)
    for ior in (1.0, 1 + 2.0 ** -9, 1 - 2.0 ** -9):
        mats = np.tile(_mat(0.3, ior, color=(0.9, 0.8, 0.7)), (1000, 1))
        xi = np.random.default_rng(3).random((1000, 4), dtype=np.float32)
        s = ot.eval_bsdf(2, V, N, None, xi, np.zeros(1000, np.int32), mats)
        assert (s[:, :3] == -V).all() and (s[:, 3:6] == np.float32([0.9, 0.8, 0.7])).all()
        assert (s[:, 6] == 1).all() and (s[:, 7] == -1).all()
