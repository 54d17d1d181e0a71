"""GPU renders with emission maps (EZRT_PARAM_EMISSION_MAPS, DESIGN.md section 18): emission textures on emissive triangles, and the
emission table weighted by each emitter's mapped emission.

Whole renders are held bit for bit, with equal primary, bounce and shadow ray counts, to the CPU restatement
(tests/oracle_emission_maps.cpp) under every option of the light sampling mode; the emission table and the sampled emission to the
restatement and to float64; the invariances (no maps, white maps) to the unflagged renders; and the rejections."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from ezrt_b200._lib import EzrtError
from tests import oracle_emission_maps as oe
from tests import oracle_medium
from tests.test_gpu_light_tables import _blob_geometry, _hostile
from tests.texture_model import bary64, sample64

pytestmark = pytest.mark.gpu

FOG = dict(sigma_t=0.6, albedo=(0.9, 0.8, 0.7), g=0.4, box_min=(-1.2, -1.0, -1.2), box_max=(1.2, 1.4, 1.2))


@pytest.fixture(scope="module")
def p3():
    tris, nodes, eye, cam, tex, uv, ids, eid = scenes.s_p3_bunny_emission_mapped()
    tris = np.asarray(tris, np.float32).reshape(-1, 36)
    hdr = scenes.synth_hdr(64, 32)
    return tris, nodes, eye, cam, tex, uv, ids, eid, hdr, api.hdr_cache(hdr)


def _cfg(eye, cam, **kw):
    base = dict(width=48, height=32, spp=2, max_bounce=4, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam), textures=True,
                emission_maps=True)
    base.update(kw)
    return api.RenderConfig(**base)


def _rays(c):
    return (c.primary_rays, c.bounce_rays, c.shadow_rays)


def _crays(c):
    return (c["rays_primary"], c["rays_bounce"], c["rays_shadow"])


def _glass(tris):
    """the bunny as rough glass: IOR 1.5, transmission 0.8"""
    t = np.array(tris, np.float32, copy=True)
    bunny = (t[:, 18:21] == 0).all(axis=1) & (t[:, 21:24] == 1).all(axis=1)
    t[bunny, 34] = 1.5
    t[bunny, 35] = 0.8
    return t


def _scene(tris, nodes, tex, uv, ids, eid, hdr=None, cache=None, medium=False, mr=None, nm=None, lights=None):
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    if medium:
        sc.set_medium(**FOG)
    sc.set_textures(tex, uv, ids)
    if mr is not None:
        sc.set_material_maps(mr, nm)
    if lights is not None:
        sc.set_punctual_lights(lights)
    sc.set_emission_maps(eid)
    return sc


def _maps(tex, ids):
    """the material maps of scenes._with_maps over these textures (appended after the emission texture)"""
    n = len(tex)
    k = np.arange(len(ids))
    on = ids >= 0
    mr = np.where(on & (k % 7 != 0), n, -1).astype(np.int32)
    nm = np.where(on & (k % 11 != 0), n + 1, -1).astype(np.int32)
    return tex + [scenes.noise_mr_map(), scenes.height_normal_map()], mr, nm


@pytest.mark.parametrize("bounces", [1, 4, 8])
@pytest.mark.parametrize("emit", ["none", "map", "light"])
def test_p3_equals_the_restatement(p3, bounces, emit):
    """no map (ids -1), a map on the emitter seen directly, and the map as a light (env map beside it)"""
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache = p3
    e = np.full_like(eid, -1) if emit == "none" else eid
    kw = dict(max_bounce=bounces, env_light=(emit == "light"))
    cfg = _cfg(eye, cam, **kw)
    sc = _scene(tris, nodes, tex, uv, ids, e, hdr, cache)
    try:
        got, gc = sc.render(cfg), sc.counters()
    finally:
        sc.close()
    ref, _, _, c = oe.render(tris, nodes, cfg, e, textures=tex, texcoords=uv, texture_id=ids, hdr=hdr, hdr_cache=cache)
    assert got.tobytes() == ref.tobytes(), "L-inf %.3g" % float(np.abs(got - ref).max())
    assert _rays(gc) == _crays(c)


OPTS = {
    "lens": dict(lens_radius=0.12, focus_distance=3.6, env_light=True), "glass": dict(transmission=True), "glass_env": dict(transmission=True, env_light=True),
    "medium": dict(medium=True, env_light=True), "maps": dict(material_maps=True, env_light=True), "maps_glass": dict(material_maps=True, transmission=True),
    "maps_medium": dict(material_maps=True, medium=True), "punct": dict(punctual_lights=True, env_light=True),
    "punct_medium": dict(punctual_lights=True, medium=True), "punct_glass": dict(punctual_lights=True, transmission=True),
    "reference": dict(traverse=api.TRAVERSE_REFERENCE), "pruned": dict(traverse=api.TRAVERSE_PRUNED), "batch1": dict(frames_per_batch=1, spp=3),
    "batch3": dict(frames_per_batch=3, spp=5), "resume": dict(first_frame=2), "parts": dict(part_count=2, part_rank=1), "profile2": dict(profile=2),
}


@pytest.mark.parametrize("opt", sorted(OPTS))
def test_p3_options_equal_the_restatement(p3, opt):
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache = p3
    kw = dict(OPTS[opt])
    mr = nm = None
    if kw.get("material_maps"):
        tex, mr, nm = _maps(tex, ids)
    if kw.get("transmission"):
        tris = _glass(tris)
    rig = scenes.punctual_rig(tris, seed=1, power=0.5) if kw.get("punctual_lights") else None
    cfg = _cfg(eye, cam, **kw)
    sc = _scene(tris, nodes, tex, uv, ids, eid, hdr, cache, medium=cfg.medium, mr=mr, nm=nm, lights=rig)
    try:
        if cfg.first_frame:   # a resumed frame: the first frames from the device, then the rest on top
            fb = sc.render(_cfg(eye, cam, spp=2, **{k: v for k, v in kw.items() if k != "first_frame"}))
            got = sc.render(cfg, framebuffer=fb)
        else:
            got = sc.render(cfg)
        gc = sc.counters()
    finally:
        sc.close()
    full = _cfg(eye, cam, **{k: v for k, v in kw.items() if k not in ("part_count", "part_rank", "first_frame")})
    if cfg.first_frame:
        full.spp = cfg.first_frame + cfg.spp
    ref, _, _, c = oe.render(tris, nodes, full, eid, lights=rig, m=oracle_medium.medium(**FOG) if cfg.medium else None, textures=tex, texcoords=uv,
                             texture_id=ids, metal_rough_id=mr, normal_id=nm, hdr=hdr, hdr_cache=cache)
    if cfg.part_count > 1:
        want = np.zeros_like(ref)
        api.partition_scatter_host(got, want, cfg.width, cfg.height, cfg.out_channels, cfg.part_rank, cfg.part_count)
        mask = np.zeros((cfg.height, cfg.width, 1), np.float32)
        api.partition_scatter_host(np.ones((got.shape[0], 1), np.float32), mask, cfg.width, cfg.height, 1, cfg.part_rank, cfg.part_count)
        m = mask[..., 0] > 0
        assert m.any() and want[m].tobytes() == ref[m].tobytes()
        return
    assert got.tobytes() == ref.tobytes(), "L-inf %.3g" % float(np.abs(got - ref).max())
    if not cfg.first_frame:
        assert _rays(gc) == _crays(c)


@pytest.mark.parametrize("opt", ["plain", "glass", "medium"])
def test_p3_aov_and_adaptive_equal_the_restatement(p3, opt):
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache = p3
    kw = dict(plain=dict(env_light=True), glass=dict(transmission=True, env_light=True), medium=dict(medium=True, env_light=True))[opt]
    if opt == "glass":
        tris = _glass(tris)
    m = oracle_medium.medium(**FOG) if opt == "medium" else None
    targs = dict(textures=tex, texcoords=uv, texture_id=ids)
    sc = _scene(tris, nodes, tex, uv, ids, eid, hdr, cache, medium=(opt == "medium"))
    try:
        cfg = _cfg(eye, cam, spp=3, **kw)
        got, gaov, _ = sc.render_aov(cfg)
        ref, _, raov, c = oe.render(tris, nodes, cfg, eid, m=m, hdr=hdr, hdr_cache=cache, aov=True, **targs)
        assert got.tobytes() == ref.tobytes() and gaov.tobytes() == raov.tobytes()
        assert sc.counters().rays == c["rays"]
        acfg = _cfg(eye, cam, spp=6, **kw)
        img, spp, luma2 = sc.render_adaptive(acfg, 0.3, 2, 2)
        ac = sc.counters()
        rimg, rspp, rluma2, rc = oe.render_adaptive(tris, nodes, acfg, eid, 0.3, 2, 2, m=m, hdr=hdr, hdr_cache=cache, **targs)
        assert img.tobytes() == rimg.tobytes() and luma2.tobytes() == rluma2.tobytes() and np.array_equal(spp, rspp)
        assert ac.rays == rc["rays"]
    finally:
        sc.close()


def test_s1m_mapped_windows_at_1920x1080():
    tris, nodes, eye, cam, tex, uv, ids, eid = scenes.s_1m_bunny_emission_mapped()
    sc = _scene(tris, nodes, tex, uv, ids, eid)
    try:
        cfg = _cfg(eye, cam, width=1920, height=1080, spp=1, max_bounce=3)
        img = sc.render(cfg)
    finally:
        sc.close()
    for win in ((0, 0, 48, 32), (928, 528, 976, 560), (1872, 1040, 1920, 1080)):
        ref, _, _, _ = oe.render(tris, nodes, cfg, eid, textures=tex, texcoords=uv, texture_id=ids, window=win)
        x0, y0, x1, y1 = win
        assert img[y0:y1, x0:x1].tobytes() == ref.tobytes(), "S-1M window %r" % (win,)


def test_w8_screen_equals_the_restatement(monkeypatch):
    """a small scene forced onto the 8-wide tree: deferred rays and the LIST pass carry E(Q) too"""
    monkeypatch.setenv("EZRT_ACCEL", "8")
    tris, nodes, eye, cam, tex, uv, ids, eid = scenes.s_screen()
    cfg = _cfg(eye, cam, spp=2, max_bounce=4)
    sc = _scene(tris, nodes, tex, uv, ids, eid)
    try:
        got, gc = sc.render(cfg), sc.counters()
    finally:
        sc.close()
    ref, _, _, c = oe.render(tris, nodes, cfg, eid, textures=tex, texcoords=uv, texture_id=ids)
    assert got.tobytes() == ref.tobytes() and _rays(gc) == _crays(c)


def _lum32(e):
    e = np.asarray(e, np.float32)
    return (np.float32(0.3) * e[:, 0] + np.float32(0.6) * e[:, 1]) + np.float32(0.1) * e[:, 2]


def test_emission_table_on_hostile_emitters():
    """the emission table against the restatement bit for bit and float64 numpy, on test_gpu_light_tables.py's hostile scene: mapped
    with white (the table is mode 4's, bit for bit) and with a banded texture"""
    tris, nodes, _, _ = _blob_geometry()
    tris = _hostile(tris)
    n = tris.shape[0]
    rng = np.random.default_rng(3)
    uv = rng.uniform(-2, 2, (n, 6)).astype(np.float32)
    white, bands = np.full((2, 2, 3), 255, np.uint8), scenes.emission_bands()
    eid = np.where(np.arange(n) % 3 == 0, 1, 0).astype(np.int32)
    sc = api.Scene(tris, nodes, device=0)
    try:
        sc.set_textures([white, bands], uv, np.full(n, -1, np.int32))
        mode4 = sc.lights()
        sc.set_emission_maps(np.zeros(n, np.int32))
        t, cdf, lum, W = sc.emission_light_table()
        assert t.tobytes() == mode4[0].tobytes() and cdf.tobytes() == mode4[1].tobytes() and W == mode4[2]
        assert lum.tobytes() == _lum32(tris[t, 18:21]).tobytes()
        sc.set_emission_maps(eid)
        t, cdf, lum, W = sc.emission_light_table()
    finally:
        sc.close()
    rt, rcdf, rlum, _, rW = oe.table(tris, [white, bands], uv, eid)
    assert t.tobytes() == rt.tobytes() and cdf.tobytes() == rcdf.tobytes() and lum.tobytes() == rlum.tobytes() and W == rW
    p = tris[t, 0:9].astype(np.float64).reshape(-1, 3, 3)
    area = 0.5 * np.linalg.norm(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]), axis=1)
    assert np.isclose(W, float((area * lum.astype(np.float64)).sum()), rtol=1e-5)


def test_sample_emission_matches_numpy(p3):
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache = p3
    rng = np.random.default_rng(9)
    tri = rng.choice(np.flatnonzero(eid >= 0), 300).astype(np.int32)
    tri = np.concatenate([tri, rng.choice(np.flatnonzero(eid < 0), 20).astype(np.int32)])
    p = tris[tri, 0:9].reshape(-1, 3, 3)
    b = rng.dirichlet((1, 1, 1), len(tri)).astype(np.float32)
    Q = (b[:, :, None] * p).sum(1).astype(np.float32)
    sc = _scene(tris, nodes, tex, uv, ids, eid)
    try:
        got = sc.sample_emission(tri, Q)
        sc.set_emission_maps(None)
        plain = sc.sample_emission(tri, Q)
    finally:
        sc.close()
    assert plain.tobytes() == tris[tri, 18:21].tobytes()
    w = bary64(Q, p)
    uv6 = np.asarray(uv, np.float32).reshape(-1, 6)[tri].astype(np.float64)
    want = []
    for i, t in enumerate(tri):
        E = tris[t, 18:21].astype(np.float64)
        if eid[t] < 0:
            want.append(E)
            continue
        u = w[i, 0] * uv6[i, 0] + w[i, 1] * uv6[i, 2] + w[i, 2] * uv6[i, 4]
        v = w[i, 0] * uv6[i, 1] + w[i, 1] * uv6[i, 3] + w[i, 2] * uv6[i, 5]
        want.append(E * sample64(tex[eid[t]], u, v))
    np.testing.assert_allclose(got.astype(np.float64), np.array(want), rtol=2e-3, atol=2e-3 * 30)


@pytest.mark.parametrize("opt", ["plain", "env_light", "medium", "glass"])
def test_invariances_on_the_device(p3, opt):
    """all ids -1 and white emission textures render the unflagged textured image, bit for bit and ray for ray"""
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache = p3
    kw = dict(plain={}, env_light=dict(env_light=True), medium=dict(medium=True, env_light=True), glass=dict(transmission=True, env_light=True))[opt]
    if opt == "glass":
        tris = _glass(tris)
    texw = tex[:-1] + [np.full((2, 2, 3), 255, np.uint8)]
    sc = _scene(tris, nodes, texw, uv, ids, np.full_like(eid, -1), hdr, cache, medium=(opt == "medium"))
    try:
        want, wc = sc.render(_cfg(eye, cam, emission_maps=False, **kw)), _rays(sc.counters())
        got, gc = sc.render(_cfg(eye, cam, **kw)), _rays(sc.counters())
        assert got.tobytes() == want.tobytes() and gc == wc
        sc.set_emission_maps(eid)
        got, gc = sc.render(_cfg(eye, cam, **kw)), _rays(sc.counters())
        assert got.tobytes() == want.tobytes() and gc == wc
    finally:
        sc.close()


def test_rejections(p3):
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache = p3
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        with pytest.raises(EzrtError):   # no textures: neither maps nor the flag
            sc.set_emission_maps(eid)
        sc.set_textures(tex, uv, ids)
        with pytest.raises(EzrtError):   # the flag without maps
            sc.render(_cfg(eye, cam))
        sc.set_emission_maps(eid)
        with pytest.raises(EzrtError):   # the flag without textures
            sc.render(_cfg(eye, cam, textures=False))
        for mode in (api.MODE_DIFFUSE_P3, api.MODE_DISNEY_IS_MIS_P5):
            with pytest.raises(EzrtError):
                sc.render(_cfg(eye, cam, mode=mode))
        with pytest.raises(EzrtError):
            sc.render(_cfg(eye, cam, pipeline=api.PIPELINE_MEGAKERNEL))
        before = sc.emission_light_table()
        ok = sc.render(_cfg(eye, cam))
        for bad in (len(tex), -2):   # out-of-range ids keep the previous maps
            e = eid.copy()
            e[5] = bad
            with pytest.raises(EzrtError):
                sc.set_emission_maps(e)
            after = sc.emission_light_table()
            assert all(np.array_equal(a, b) for a, b in zip(before[:3], after[:3])) and before[3] == after[3]
        assert sc.render(_cfg(eye, cam)).tobytes() == ok.tobytes()
        sc.set_textures(tex, uv, ids)   # set_textures clears the maps
        with pytest.raises(EzrtError):
            sc.render(_cfg(eye, cam))
        with pytest.raises(EzrtError):
            sc.emission_light_table()
        sc.set_emission_maps(eid)
        sc.set_textures(None)
        with pytest.raises(EzrtError):
            sc.emission_light_table()
    finally:
        sc.close()
