"""The volumes inside transmissive meshes (EZRT_PARAM_VOLUMES, ezrt_math.h, DESIGN.md section 21) on the CPU restatement
(tests/oracle_volumes.cpp): sigma_a against float64, the identities with the renders without absorption (bit for bit, with ray counts)
under every option of the light sampling mode, an index-matched slab and a smooth slab against their closed forms, the estimator against
a BSDF-only one, glass inside the homogeneous medium and the density grid (identities, a clear box displacing an absorbing fog, the
estimator against a BSDF- and phase-only one), the rejections, and mutations the analytic checks catch."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_lens
from tests import oracle_light_tree as olt
from tests import oracle_medium
from tests import oracle_volumes as ov
from tests import volume_scenes as vs
from tests.test_gpu_emission_maps import FOG, _maps
from tests.test_light_sampling_laws import _block_z, _stats
from tests.texture_model import constant_textures

L4 = api.MODE_DISNEY_LIGHTS


# ------------------------------------------------------------------ 1. sigma_a
def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    return np.abs(ia - ib)


def test_sigma_a_against_float64():
    rng = np.random.default_rng(1)
    n = 1_000_000
    c = rng.uniform(0, 1, n).astype(np.float32)
    c[: n // 4] = np.exp(rng.uniform(-80, 0, n // 4)).astype(np.float32)   # deep colours, down to 1e-35
    d = np.exp(rng.uniform(np.log(1e-6), np.log(1e6), n)).astype(np.float32)
    c = c[c > 0]
    d = d[: c.size]
    got = ov.sigma_a(c, d)
    want = (-np.log(c.astype(np.float64)) / d.astype(np.float64)).astype(np.float32)
    u = _ulps(got, want)
    print("sigma_a: %d pairs, largest error %d ulp, %.3f %% off by 1" % (c.size, u.max(), 100 * (u == 1).mean()))
    assert u.max() <= 2


def test_sigma_a_edge_cases():
    inf = np.float32(np.inf)
    cases = [(1.0, 1.0, 0.0), (1.0, inf, 0.0), (0.0, 1.0, inf), (0.0, inf, 0.0), (0.5, inf, 0.0), (0.0, 1e-30, inf), (0.0, 1e30, inf),
             (0.5, 1e-30, np.log(2.0) / 1e-30), (0.5, 1e30, np.log(2.0) / 1e30), (0.5, 1e-38, np.log(2.0) / 1e-38), (1e-3, 1.2e-38, inf)]
    for c, d, want in cases:
        got = ov.sigma_a(np.float32([c]), np.float32([d]))[0]
        w = np.float32(want)
        assert (got == w and np.signbit(got) == np.signbit(w)) or _ulps(got, w) <= 2, (c, d, got, w)
    # T = exp(-sigma_a t) at the smallest hit distance: 0 for sigma_a = inf, 1 for sigma_a = 0, never NaN
    assert ov.sigma_a(np.float32([0.0]), np.float32([1.0]))[0] == inf


# ------------------------------------------------------------------ 2. identities with the renders without absorption
def blob_scene():
    """volume_scenes.p3_coloured_glass with seeded textures (constant ones, random UVs and ids) and the emissive sphere mapped by
    scenes.emission_bands: (tris, nodes, eye, cam, textures, texcoords, texture_id, emission_id)"""
    tris, nodes, eye, cam, _, _ = vs.p3_coloured_glass(0.3)
    rng = np.random.default_rng(7)
    tex, _ = constant_textures(rng, [(1, 1), (3, 2)])
    tex = tex + [scenes.emission_bands()]
    n = tris.shape[0]
    uv = rng.uniform(-2, 2, (n, 3, 2)).astype(np.float32)
    ids = rng.integers(-1, 2, n).astype(np.int32)
    eid = np.where((tris[:, 18:21] > 0).any(axis=1), len(tex) - 1, -1).astype(np.int32)
    return tris, nodes, eye, cam, tex, uv, ids, eid


@pytest.fixture(scope="module")
def p3():
    hdr = scenes.synth_hdr(64, 32)
    return blob_scene() + (hdr, api.hdr_cache(hdr))


OPTS = {
    "plain": dict(), "env": dict(env_light=True), "lens": dict(lens_radius=0.12, focus_distance=3.6, env_light=True),
    "textures": dict(textures=True), "maps": dict(textures=True, material_maps=True, env_light=True),
    "punct": dict(punctual_lights=True, env_light=True), "emap": dict(textures=True, emission_maps=True),
    "tree": dict(light_tree=True, env_light=True), "tree_emap_punct": dict(light_tree=True, textures=True, emission_maps=True, punctual_lights=True),
}


def _setup(p3, opt):
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache = p3
    kw = dict(OPTS[opt])
    rk = dict(hdr=hdr, hdr_cache=cache, emission_id=eid, textures=tex, texcoords=uv, texture_id=ids)
    if kw.get("material_maps"):
        rk["textures"], rk["metal_rough_id"], rk["normal_id"] = _maps(tex, ids)
    if kw.get("punctual_lights"):
        rk["lights"] = scenes.punctual_rig(tris, seed=1, power=0.5)
    cfg = api.RenderConfig(width=32, height=24, spp=2, max_bounce=5, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam), transmission=True, **kw)
    return tris, nodes, cfg, rk


def _bunny_ids(tris, v=0):
    return np.where(tris[:, 35] > 0, v, -1).astype(np.int32)


@pytest.mark.parametrize("opt", sorted(OPTS))
def test_clear_volumes_give_the_transmission_render(p3, opt):
    """the flag without volumes, with every id -1, with white colours and with infinite distances renders EZRT_PARAM_TRANSMISSION's bits"""
    tris, nodes, cfg, rk = _setup(p3, opt)
    want, wl, _, wc = olt.render(tris, nodes, cfg, **rk)
    cfg.volumes = True
    n = tris.shape[0]
    ids = _bunny_ids(tris)
    for vols, vid in ((None, None), ([vs.AMBER], np.full(n, -1, np.int32)), ([api.volume((1, 1, 1), 0.01)], ids),
                      ([api.volume((0.0, 0.3, 0.9), np.inf)], ids)):
        got, gl, _, gc = ov.render(tris, nodes, cfg, volumes=vols, volume_id=vid, **rk)
        assert got.tobytes() == want.tobytes() and gl.tobytes() == wl.tobytes(), (opt, vols is None)
        assert gc == wc


@pytest.mark.parametrize("opt", ["plain", "env", "tree_emap_punct"])
def test_absorbing_render_keeps_the_ray_counts(p3, opt):
    tris, nodes, cfg, rk = _setup(p3, opt)
    _, _, _, wc = olt.render(tris, nodes, cfg, **rk)
    cfg.volumes = True
    got, _, _, gc = ov.render(tris, nodes, cfg, volumes=[vs.AMBER], volume_id=_bunny_ids(tris), **rk)
    assert gc == wc
    cfg.volumes = False
    plain, _, _, _ = olt.render(tris, nodes, cfg, **rk)
    assert got.tobytes() != plain.tobytes() and np.isfinite(got).all()


def test_ids_on_opaque_triangles_are_ignored(p3):
    tris, nodes, cfg, rk = _setup(p3, "env")
    want, _, _, wc = olt.render(tris, nodes, cfg, **rk)
    cfg.volumes = True
    opaque = np.where(tris[:, 35] > 0, -1, 0).astype(np.int32)
    got, _, _, gc = ov.render(tris, nodes, cfg, volumes=[api.volume((0.0, 0.0, 0.0), 0.1)], volume_id=opaque, **rk)
    assert got.tobytes() == want.tobytes() and gc == wc


def test_feature_buffers_and_adaptive_forms(p3):
    """the feature buffers describe the first hit as without volumes; the adaptive form's tiles agree with plain renders' arithmetic"""
    tris, nodes, cfg, rk = _setup(p3, "env")
    cfg.volumes = True
    vk = dict(volumes=[vs.AMBER], volume_id=_bunny_ids(tris))
    img, _, feat, _ = ov.render(tris, nodes, cfg, aov=True, **vk, **rk)
    cfg.volumes = False
    _, _, feat0, _ = olt.render(tris, nodes, cfg, aov=True, **rk)
    assert feat.tobytes() == feat0.tobytes()
    cfg.volumes, cfg.spp = True, 6
    a, spp, _, _ = ov.render_adaptive(tris, nodes, cfg, 1e9, 2, 2, **vk, **rk)   # a threshold every tile meets at 2 spp
    assert (spp == 2).all()
    cfg.spp = 2
    b, _, _, _ = ov.render(tris, nodes, cfg, **vk, **rk)
    assert a.tobytes() == b.tobytes()


# ------------------------------------------------------------------ 3. analytic slabs
def _slab_T(sig, mutate=False, width=32, height=32):
    """the index-matched white slab (thickness 0.4) in front of the emitter (2): per pixel of the central window, the render's value
    and the camera ray's inside length 0.4 / |d_z|"""
    tris, nodes, eye, cam = vs.slab(ior=1.0)
    cfg = api.RenderConfig(width=width, height=height, spp=1, max_bounce=2, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam), transmission=True,
                           volumes=True)
    vid = np.zeros(tris.shape[0], np.int32)
    vid[tris[:, 35] == 0] = -1
    img, _, _, _ = ov.render(tris, nodes, cfg, volumes=[(np.exp(-np.float64(sig)), 1.0)], volume_id=vid, mutate=mutate)
    py, px = np.mgrid[0:height, 0:width]
    r = oracle_lens.camera_rays(cfg, px.ravel(), py.ravel(), np.zeros(px.size, np.uint32))
    o, d = r["o"].astype(np.float64), r["d"].astype(np.float64)
    length = 0.4 / np.abs(d[:, 2])
    # the pixels whose camera ray crosses both faces at least 0.05 inside the slab's edges
    hit = np.ones(px.size, bool)
    for z in (0.7, 0.3):
        q = o + d * ((z - o[:, 2]) / d[:, 2])[:, None]
        hit &= (np.abs(q[:, 0]) < 1.15) & (np.abs(q[:, 1]) < 1.15)
    return img.reshape(-1, 3), length, ov.table([(np.exp(-np.float64(sig)), 1.0)])[0], hit


def test_index_matched_slab_carries_le_exp_minus_sigma_l():
    sig = (0.3, 1.1, 2.7)
    img, length, s, hit = _slab_T(sig)
    T = img / np.float32(2.0)
    want = np.exp(-s.astype(np.float64)[None, :] * length[:, None])
    assert hit.sum() >= 100
    rel = np.abs(T[hit] / want[hit] - 1)
    print("index-matched slab: %d pixels, largest relative error %.2e" % (hit.sum(), rel.max()))
    assert rel.max() <= 2e-6 * (1 + s.max() * length.max())


def test_mutation_dropping_the_first_segments_absorption_fails_the_slab():
    sig = (0.3, 1.1, 2.7)
    img, length, s, hit = _slab_T(sig, mutate=True)
    T = img / np.float32(2.0)
    want = np.exp(-s.astype(np.float64)[None, :] * length[:, None])
    assert np.abs(T[hit] / want[hit] - 1).max() > 0.5


@pytest.mark.parametrize("max_bounce", [2, 4, 6])
def test_smooth_absorbing_slab_closed_form(max_bounce):
    """IOR 1.5, grey sigma_a: Le (1 - F)^2 sum_k F^(2k) exp(-(2k + 1) sigma_a L) over the paths of k internal round trips that reach
    the emitter within max_bounce (normal incidence; the central window's rays are within 1 degree of it)"""
    tris, nodes, eye, cam = vs.slab(ior=1.5)
    spp = 512
    cfg = api.RenderConfig(width=64, height=64, spp=spp, max_bounce=max_bounce, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam), transmission=True,
                           volumes=True)
    vid = np.where(tris[:, 35] > 0, 0, -1).astype(np.int32)
    sig = 1.5
    img, luma2, _, _ = ov.render(tris, nodes, cfg, volumes=[(np.full(3, np.exp(-sig)), 1.0)], volume_id=vid, window=(28, 28, 36, 36))
    y, var = _stats(img, luma2)
    F = ((1.5 - 1) / (1.5 + 1)) ** 2
    s = float(ov.table([(np.full(3, np.exp(-sig)), 1.0)])[0, 0])
    K = (max_bounce - 2) // 2 + 1
    want = 2.0 * (1 - F) ** 2 * sum(F ** (2 * k) * np.exp(-(2 * k + 1) * s * 0.4) for k in range(K))
    z = abs(y.mean() - want) / np.sqrt(var.sum() / spp / y.size ** 2)
    print("absorbing slab max_bounce %d: %.6f against %.6f, z %.2f" % (max_bounce, y.mean(), want, z))
    assert z <= 5
    # the mutation: the first BSDF sample's hit not absorbed
    img, luma2, _, _ = ov.render(tris, nodes, cfg, volumes=[(np.full(3, np.exp(-sig)), 1.0)], volume_id=vid, window=(28, 28, 36, 36), mutate=True)
    y, var = _stats(img, luma2)
    assert abs(y.mean() - want) / np.sqrt(var.sum() / spp / y.size ** 2) > 50


# ------------------------------------------------------------------ 4. the estimator against the BSDF-only one
def _unbiased_cases():
    hdr = scenes.synth_hdr(64, 32)
    return [
        ("rough amber glass blob on the P3 floor", vs.p3_coloured_glass(0.3), None, False),
        ("the same under a map, env light", vs.p3_coloured_glass(0.3), hdr, True),
    ]


@pytest.mark.parametrize("k", range(2))
def test_estimator_agrees_with_bsdf_samples_only(k):
    name, (tris, nodes, eye, cam, vols, vid), hdr, env_light = _unbiased_cases()[k]
    cache = None if hdr is None else api.hdr_cache(hdr)
    spp, W, H = 256, 64, 48
    out = []
    for bsdf_only in (False, True):
        first = spp if bsdf_only else 0
        cfg = api.RenderConfig(width=W, height=H, spp=spp, first_frame=first, max_bounce=4, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam),
                               env_color=(0.1, 0.1, 0.12), transmission=True, env_light=env_light, volumes=True)
        img, luma2, _, _ = ov.render(tris, nodes, cfg, volumes=vols, volume_id=vid, hdr=hdr, hdr_cache=cache, bsdf_only=bsdf_only)
        assert np.isfinite(img).all()
        scale = np.float64(first + spp) / spp
        y = _stats(img, luma2)[0] * scale
        out.append((y, np.maximum(luma2.astype(np.float64) * scale - y ** 2, 0.0)))
    z8, z16 = _block_z(out[0], out[1], spp, W, H, 8, 8), _block_z(out[0], out[1], spp, W, H, 16, 16)
    zf = float(_block_z(out[0], out[1], spp, W, H, H, W).max())
    print("unbiased %-40s means %.5f / %.5f, frame z %.2f, largest 16x16 z %.2f, largest 8x8 z %.2f" %
          (name, out[0][0].mean(), out[1][0].mean(), zf, z16.max(), z8.max()))
    assert zf <= 4, (name, zf)
    assert z16.max() <= 5 and z8.max() <= 5, (name, z16.max(), z8.max())


# ------------------------------------------------------------------ 5. glass inside the medium
def _fog_cfg(eye, cam, **kw):
    base = dict(width=32, height=24, spp=2, max_bounce=5, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam), medium=True)
    base.update(kw)
    return api.RenderConfig(**base)


@pytest.mark.parametrize("opt", ["plain", "env", "lens", "tree_emap_punct", "maps"])
@pytest.mark.parametrize("grid", [False, True])
def test_flag_beside_the_medium_without_glass_is_the_medium_render(p3, opt, grid):
    """VOLUMES | TRANSMISSION | MEDIUM (homogeneous and grid) on a scene without transmissive material renders the MEDIUM render's bits
    and rays; with sigma_t = 0 it renders VOLUMES | TRANSMISSION's"""
    from tests import oracle_medium_grid as og
    tris, nodes, cfg, rk = _setup(p3, opt)
    opaque = np.array(tris, np.float32, copy=True)
    opaque[:, 35] = 0.0
    cfg.transmission = False
    cfg.medium = True
    cfg.medium_grid = grid
    rho = scenes.smoke_grid(16, 1) if grid else None
    m = oracle_medium.medium(**vs.FOG)
    want = og.render(opaque, nodes, cfg, rho, m=m, **rk)
    cfg.transmission = cfg.volumes = True
    got = ov.render(opaque, nodes, cfg, volumes=[vs.AMBER], volume_id=_bunny_ids(tris), m=m, rho=rho, **rk)
    assert got[0].tobytes() == want[0].tobytes() and got[3] == want[3], (opt, grid)
    # sigma_t = 0: the medium draws nothing, the render is VOLUMES | TRANSMISSION's
    zero = oracle_medium.medium(**dict(vs.FOG, sigma_t=0.0))
    got = ov.render(tris, nodes, cfg, volumes=[vs.AMBER], volume_id=_bunny_ids(tris), m=zero, rho=rho, **rk)
    cfg.medium = cfg.medium_grid = False
    want = ov.render(tris, nodes, cfg, volumes=[vs.AMBER], volume_id=_bunny_ids(tris), **rk)
    assert got[0].tobytes() == want[0].tobytes() and got[3] == want[3], (opt, grid)


def _fog_window_means(mutate_flight):
    """the clear box in the pure absorber at 2 bounces: per pixel of a central window, the render's mean over spp samples (each sample is
    Le = 2 when the camera ray reaches the emitter, 0 when it is absorbed), and the exact mean 2 exp(-sigma_t (L_fog - L_glass)) from the
    restatement's camera rays of every sample"""
    tris, nodes, eye, cam, fog = vs.clear_box_in_absorber()
    spp, win = 256, (12, 12, 20, 20)
    cfg = api.RenderConfig(width=32, height=32, spp=spp, max_bounce=2, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam), transmission=True,
                           volumes=True, medium=True)
    img, _, _, _ = ov.render(tris, nodes, cfg, m=oracle_medium.medium(**fog), window=win, mutate_flight=mutate_flight)
    x0, y0, x1, y1 = win
    py, px, fr = np.meshgrid(np.arange(y0, y1), np.arange(x0, x1), np.arange(spp), indexing="ij")
    r = oracle_lens.camera_rays(cfg, px.ravel(), py.ravel(), fr.ravel())
    o, d = r["o"].astype(np.float64), r["d"].astype(np.float64)
    t_in = lambda z: (z - o[:, 2]) / d[:, 2]
    fog_len = t_in(-1.0) - t_in(1.5)            # the ray enters the fog at z = 1.5 and meets the emitter's front face inside it
    glass_len = t_in(0.3) - t_in(0.7)
    q = o + d * t_in(0.3)[:, None]
    assert (np.abs(q[:, :2]) < 1.15).all()      # every sample crosses both faces of the box
    want = (2.0 * np.exp(-fog["sigma_t"] * (fog_len - glass_len))).reshape(y1 - y0, x1 - x0, spp).mean(axis=2)
    got = img[..., 0].astype(np.float64)
    var = (want * (2.0 - want)).sum() / spp     # Bernoulli values 0 or 2
    return got.mean(), want.mean(), abs(got.sum() - want.sum()) / np.sqrt(var)


def test_clear_glass_displaces_absorbing_fog():
    got, want, z = _fog_window_means(False)
    print("clear box in absorbing fog: mean %.5f against exp(-sigma_t (L_fog - L_glass)) %.5f, z %.2f" % (got, want, z))
    assert z <= 4


def test_mutation_drawing_the_flight_inside_glass_fails_the_fog_check():
    got, want, z = _fog_window_means(True)
    print("mutated: mean %.5f against %.5f, z %.2f" % (got, want, z))
    assert z > 10


def _fog_cases():
    tris, nodes, eye, cam, vols, vid, fog = vs.p3_glass_in_fog()
    st, sn, se, sc_, sv, sid, smed, rho = vs.p3_glass_in_smoke()
    return [("amber glass in homogeneous fog", (tris, nodes, eye, cam, vols, vid), fog, None),
            ("amber glass in the smoke grid", (st, sn, se, sc_, sv, sid), smed, rho)]


@pytest.mark.parametrize("k", range(2))
def test_glass_in_fog_agrees_with_bsdf_and_phase_samples_only(k):
    name, (tris, nodes, eye, cam, vols, vid), fog, rho = _fog_cases()[k]
    spp, W, H = 256, 64, 48
    out = []
    for bsdf_only in (False, True):
        first = spp if bsdf_only else 0
        cfg = api.RenderConfig(width=W, height=H, spp=spp, first_frame=first, max_bounce=4, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam),
                               env_color=(0.1, 0.1, 0.12), transmission=True, volumes=True, medium=True, medium_grid=rho is not None)
        img, luma2, _, _ = ov.render(tris, nodes, cfg, volumes=vols, volume_id=vid, m=oracle_medium.medium(**fog), rho=rho, bsdf_only=bsdf_only)
        assert np.isfinite(img).all()
        scale = np.float64(first + spp) / spp
        y = _stats(img, luma2)[0] * scale
        out.append((y, np.maximum(luma2.astype(np.float64) * scale - y ** 2, 0.0)))
    z8, z16 = _block_z(out[0], out[1], spp, W, H, 8, 8), _block_z(out[0], out[1], spp, W, H, 16, 16)
    zf = float(_block_z(out[0], out[1], spp, W, H, H, W).max())
    print("unbiased %-40s means %.5f / %.5f, frame z %.2f, largest 16x16 z %.2f, largest 8x8 z %.2f" %
          (name, out[0][0].mean(), out[1][0].mean(), zf, z16.max(), z8.max()))
    assert zf <= 4, (name, zf)
    assert z16.max() <= 5 and z8.max() <= 5, (name, z16.max(), z8.max())


# ------------------------------------------------------------------ 6. rejections
def test_rejections(p3):
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache = p3
    vk = dict(volumes=[vs.AMBER], volume_id=_bunny_ids(tris))
    base = dict(width=16, height=16, spp=1, max_bounce=2, eye=tuple(eye), camera_rotate=tuple(cam))
    with pytest.raises(ValueError):   # without transmission
        ov.render(tris, nodes, api.RenderConfig(mode=L4, volumes=True, **base), **vk)
    for mode in (api.MODE_DIFFUSE_P3, api.MODE_DISNEY_ANISO_P4, api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5):
        with pytest.raises(ValueError):
            ov.render(tris, nodes, api.RenderConfig(mode=mode, transmission=True, volumes=True, **base), hdr=hdr, hdr_cache=cache, **vk)
    with pytest.raises(ValueError):
        ov.render(tris, nodes, api.RenderConfig(mode=L4, transmission=True, volumes=True, pipeline=api.PIPELINE_MEGAKERNEL, **base), **vk)
    with pytest.raises(ValueError):   # the medium beside transmission without the flag
        ov.render(tris, nodes, api.RenderConfig(mode=L4, transmission=True, medium=True, **base), m=oracle_medium.medium(**FOG))
    # ... and accepted with it
    img, _, _, _ = ov.render(tris, nodes, api.RenderConfig(mode=L4, transmission=True, medium=True, volumes=True, **base), m=oracle_medium.medium(**FOG),
                             **vk)
    assert np.isfinite(img).all()
    bad = np.full(tris.shape[0], 1, np.int32)   # an id out of range
    with pytest.raises(ValueError):
        ov.render(tris, nodes, api.RenderConfig(mode=L4, transmission=True, volumes=True, **base), volumes=[vs.AMBER], volume_id=bad)
