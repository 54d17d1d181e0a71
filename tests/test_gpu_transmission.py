"""The materials' transmission (RenderConfig.transmission / EZRT_PARAM_TRANSMISSION in the light sampling mode, DESIGN.md section 12)
on the GPU against its CPU restatement (tests/oracle_transmission.cpp): renders bit for bit with their ray counts, with and without
the map as a light, the same bits under every render option, hostile materials, the inputs it rejects, and ezrt_eval_bsdf against
the CPU functions."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_transmission as ot
from tests import transmission_scenes as ts
from tests.test_gpu_parity import assert_same_bits
from tests.test_transmission_oracle import HOSTILE, _slab_scene, _sun_map, hostile_scene, law_inputs

pytestmark = pytest.mark.gpu

ENV = (0.35, 0.45, 0.6)
L4 = api.MODE_DISNEY_LIGHTS


def _cfg(eye, cam, **kw):
    base = dict(width=64, height=48, spp=2, max_bounce=4, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam), env_color=ENV, transmission=True)
    base.update(kw)
    return api.RenderConfig(**base)


@pytest.fixture(scope="module")
def glass_scenes(small_hdr):
    hdr, cache = small_hdr
    out = {}
    for mesh in ("bunny", "blob"):
        tris, nodes, eye, cam = ts.p3_glass(mesh)
        out[mesh] = dict(tris=tris, nodes=nodes, eye=eye, cam=cam, sc=api.Scene(tris, nodes, hdr, cache), sc_none=api.Scene(tris, nodes))
    yield out, hdr, cache
    for d in out.values():
        d["sc"].close()
        d["sc_none"].close()


def _assert_matches_restatement(sc, tris, nodes, cfg, what, hdr=None, cache=None, window=None):
    img = sc.render(cfg)
    c = sc.counters()
    ref, _, rc = ot.oracle_render_transmission(tris, nodes, cfg, hdr=hdr, hdr_cache=cache, window=window)
    if window is not None:
        x0, y0, x1, y1 = window
        img = img[y0:y1, x0:x1]
    assert_same_bits(img, ref, what)
    if window is None:
        assert (c.primary_rays, c.bounce_rays, c.shadow_rays) == (rc["rays_primary"], rc["rays_bounce"], rc["rays_shadow"]), what
    return img


@pytest.mark.parametrize("env_light", [False, True])
@pytest.mark.parametrize("bounces", [1, 4, 8])
@pytest.mark.parametrize("mesh", ["bunny", "blob"])
def test_p3_glass_bit_identical(glass_scenes, mesh, bounces, env_light):
    d, hdr, cache = glass_scenes[0][mesh], glass_scenes[1], glass_scenes[2]
    cfg = _cfg(d["eye"], d["cam"], max_bounce=bounces, env_light=env_light)
    _assert_matches_restatement(d["sc"], d["tris"], d["nodes"], cfg, "P3 %s glass, map, env light %s, %d bounces" % (mesh, env_light, bounces),
                                hdr, cache)
    _assert_matches_restatement(d["sc_none"], d["tris"], d["nodes"], cfg, "P3 %s glass, no map, %d bounces" % (mesh, bounces))


def test_same_bits_under_every_render_option(glass_scenes, monkeypatch):
    (d, hdr, cache) = glass_scenes[0]["blob"], glass_scenes[1], glass_scenes[2]
    sc, eye, cam = d["sc"], d["eye"], d["cam"]
    for env_light in (False, True):
        want = sc.render(_cfg(eye, cam, spp=3, env_light=env_light))
        for trav in (api.TRAVERSE_REFERENCE, api.TRAVERSE_PRUNED):
            assert_same_bits(sc.render(_cfg(eye, cam, spp=3, traverse=trav, env_light=env_light)), want, "traverse %d" % trav)
        for fpb in (1, 3, 0):
            assert_same_bits(sc.render(_cfg(eye, cam, spp=3, frames_per_batch=fpb, env_light=env_light)), want, "frames_per_batch %d" % fpb)
        first = sc.render(_cfg(eye, cam, spp=1, env_light=env_light))
        assert_same_bits(sc.render(_cfg(eye, cam, spp=2, first_frame=1, env_light=env_light), framebuffer=first.reshape(-1, 3).copy()), want,
                         "1 then 2 frames")
        W, H = 64, 48
        full = np.zeros((H * W, 3), np.float32)
        for r in range(2):
            part = sc.render(_cfg(eye, cam, spp=3, part_rank=r, part_count=2, env_light=env_light))
            api.partition_scatter_host(part, full, W, H, 3, r, 2)
        assert_same_bits(full.reshape(H, W, 3), want, "two parts")
        assert_same_bits(sc.render(_cfg(eye, cam, spp=3, profile=2, env_light=env_light)), want, "profile 2")
        monkeypatch.setenv("EZRT_DEFERRED_LANE", "0")
        sc2 = api.Scene(d["tris"], d["nodes"], hdr, cache)
        try:
            assert_same_bits(sc2.render(_cfg(eye, cam, spp=3, env_light=env_light)), want, "deferred lane off")
        finally:
            sc2.close()
            monkeypatch.delenv("EZRT_DEFERRED_LANE")


def test_small_scene_forced_to_w8(small_hdr, monkeypatch):
    tris, nodes, eye, cam = ts.grid_glass(3, 2, 2)
    hdr, cache = small_hdr
    monkeypatch.setenv("EZRT_ACCEL", "8")
    sc = api.Scene(tris, nodes, hdr, cache)
    try:
        for env_light in (False, True):
            _assert_matches_restatement(sc, tris, nodes, _cfg(eye, cam, env_light=env_light), "glass grid, W8", hdr, cache)
    finally:
        sc.close()


def test_s1m_glass_windows_at_1920x1080():
    """S-1M's blob grid with every other blob glass (roughness 0.05 and 0.3), in tile-aligned windows of a 1920 x 1080 render."""
    tris, nodes, eye, cam = ts.grid_glass(15, 13, 4)
    sc = api.Scene(tris, nodes)
    try:
        cfg = _cfg(eye, cam, width=1920, height=1080, spp=1, max_bounce=4)
        img = sc.render(cfg)
        assert sc.counters().shadow_rays > 0
        for win in ((0, 0, 48, 32), (928, 528, 976, 560), (1872, 1040, 1920, 1080), (640, 400, 704, 448)):
            ref, _, _ = ot.oracle_render_transmission(tris, nodes, cfg, window=win)
            x0, y0, x1, y1 = win
            assert_same_bits(img[y0:y1, x0:x1], ref, "S-1M glass window %r" % (win,))
    finally:
        sc.close()


def test_refracted_hits_on_a_small_light_and_a_map_sun():
    """the scenes where a refracted BSDF sample's weight of 1 on a light or on the map is what keeps the estimate unbiased"""
    for tris, nodes, eye, cam, hdr in ((*_slab_scene(0.8, emitter=(0.25, -0.5, 20.0)), None), (*_slab_scene(0.8, emitter=None), _sun_map())):
        cache = None if hdr is None else api.hdr_cache(hdr)
        sc = api.Scene(tris, nodes, hdr, cache)
        try:
            _assert_matches_restatement(sc, tris, nodes, _cfg(eye, cam, width=32, height=32, spp=8, env_light=hdr is not None),
                                        "slab, %s" % ("map sun" if hdr is not None else "small light"), hdr, cache)
        finally:
            sc.close()


@pytest.mark.parametrize("name", [h[0] for h in HOSTILE])
def test_hostile_materials(name):
    tris, nodes, eye, cam = hostile_scene(name)
    sc = api.Scene(tris, nodes)
    try:
        img = _assert_matches_restatement(sc, tris, nodes, _cfg(eye, cam, env_color=(1.0, 1.0, 1.0)), "hostile material %s" % name)
        assert np.isfinite(img).all(), name
    finally:
        sc.close()


def test_adaptive_and_feature_buffers(glass_scenes):
    (d, hdr, cache) = glass_scenes[0]["blob"], glass_scenes[1], glass_scenes[2]
    sc, eye, cam = d["sc"], d["eye"], d["cam"]
    for env_light in (False, True):
        img, spp, _ = sc.render_adaptive(_cfg(eye, cam, spp=6, env_light=env_light), 0.5, 2, 2)
        for s in np.unique(spp):
            plain = sc.render(_cfg(eye, cam, spp=int(s), env_light=env_light))
            m = spp == s
            assert_same_bits(img[m], plain[m], "tiles at %d spp" % s)
        cfg = _cfg(eye, cam, spp=3, env_light=env_light)
        img, aov, luma2 = sc.render_aov(cfg)
        assert_same_bits(img, sc.render(cfg), "aov render framebuffer")
        _, rluma2, _ = ot.oracle_render_transmission(d["tris"], d["nodes"], cfg, hdr=hdr, hdr_cache=cache)
        assert luma2.tobytes() == rluma2.tobytes()


def test_flag_without_glass_is_mode_4(small_hdr):
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    hdr, cache = small_hdr
    for h, c in ((None, None), (hdr, cache)):
        sc = api.Scene(tris, nodes, h, c)
        try:
            for env_light in ((False, True) if h is not None else (False,)):
                cfg = _cfg(eye, cam, env_light=env_light)
                plain = sc.render(_cfg(eye, cam, env_light=env_light, transmission=False))
                pc = sc.counters()
                flagged = sc.render(cfg)
                fc = sc.counters()
                assert_same_bits(flagged, plain, "no glass: flagged vs plain, map %s, env light %s" % (h is not None, env_light))
                assert (fc.primary_rays, fc.bounce_rays, fc.shadow_rays) == (pc.primary_rays, pc.bounce_rays, pc.shadow_rays)
        finally:
            sc.close()


def test_rejected_inputs(glass_scenes):
    d = glass_scenes[0]["blob"]
    sc, eye, cam = d["sc"], d["eye"], d["cam"]
    bad = [_cfg(eye, cam, mode=m) for m in (api.MODE_DIFFUSE_P3, api.MODE_DISNEY_ANISO_P4, api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5)]
    bad.append(_cfg(eye, cam, pipeline=api.PIPELINE_MEGAKERNEL))
    for cfg in bad:
        with pytest.raises(api.EzrtError) as e:
            sc.render(cfg)
        assert e.value.code == -1, cfg.mode
    with pytest.raises(api.EzrtError):
        sc.render_adaptive(_cfg(eye, cam, mode=api.MODE_DISNEY_IS_MIS_P5, spp=4), 0.5, 2, 2)
    with pytest.raises(api.EzrtError):
        sc.render_aov(_cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5))


def test_eval_bsdf_equals_cpu_functions():
    V, N, L, xi, inside, mats = law_inputs(20000, seed=5)
    for which in (0, 1, 2):
        got = api.eval_bsdf(which, V, N, None if which == 2 else L, xi if which == 2 else None, inside, mats)
        want = ot.eval_bsdf(which, V, N, L, xi, inside, mats)
        assert got.tobytes() == want.tobytes(), which
