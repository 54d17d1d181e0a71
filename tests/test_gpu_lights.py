"""The light sampling mode (EZRT_MODE_DISNEY_LIGHTS, DESIGN.md section 10) on the GPU against its CPU restatement
(tests/oracle_lights.cpp): renders bit for bit with their ray counts, the same bits under every render option, and the bounded
occlusion query of its shadow rays ray by ray on the hostile scenes of tests/test_gpu_w8.py."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_lights as ol
from tests.test_gpu_parity import assert_same_bits

pytestmark = pytest.mark.gpu

ENV = (0.35, 0.45, 0.6)
L4 = api.MODE_DISNEY_LIGHTS


def _cfg(eye, cam, **kw):
    base = dict(width=64, height=48, spp=2, max_bounce=2, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam), env_color=ENV)
    base.update(kw)
    return api.RenderConfig(**base)


@pytest.fixture(scope="module")
def p3(small_hdr):
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    hdr, cache = small_hdr
    sc, sc_env = api.Scene(tris, nodes, hdr, cache), api.Scene(tris, nodes)
    yield dict(tris=tris, nodes=nodes, eye=eye, cam=cam, hdr=hdr, cache=cache, sc=sc, sc_env=sc_env)
    sc.close()
    sc_env.close()


def _assert_matches_restatement(sc, tris, nodes, cfg, what, hdr=None, cache=None, window=None):
    img = sc.render(cfg)
    c = sc.counters()
    ref, _, rc = ol.oracle_render_lights(tris, nodes, cfg, hdr=hdr, hdr_cache=cache, window=window)
    if window is not None:
        x0, y0, x1, y1 = window
        img = img[y0:y1, x0:x1]
    assert_same_bits(img, ref, what)
    if window is None:
        assert (c.primary_rays, c.bounce_rays, c.shadow_rays) == (rc["rays_primary"], rc["rays_bounce"], rc["rays_shadow"]), what
        assert c.shadow_rays > 0, what
    return img


@pytest.mark.parametrize("with_map", [False, True])
@pytest.mark.parametrize("bounces", [1, 2, 4])
def test_p3_bunny_bit_identical(p3, with_map, bounces):
    sc = p3["sc"] if with_map else p3["sc_env"]
    hdr = (p3["hdr"], p3["cache"]) if with_map else (None, None)
    _assert_matches_restatement(sc, p3["tris"], p3["nodes"], _cfg(p3["eye"], p3["cam"], max_bounce=bounces), "P3 bunny, map %s, %d bounces" %
                                (with_map, bounces), *hdr)


def test_light_table_matches_restatement(p3):
    tri, cdf, total = p3["sc"].lights()
    rtri, rcdf, rtotal = ol.oracle_light_table(p3["tris"])
    assert len(tri) == 320 and (tri == rtri).all() and cdf.tobytes() == rcdf.tobytes() and total == rtotal


def test_same_bits_under_every_render_option(p3, monkeypatch):
    sc, eye, cam = p3["sc"], p3["eye"], p3["cam"]
    want = sc.render(_cfg(eye, cam, spp=3))
    for trav in (api.TRAVERSE_REFERENCE, api.TRAVERSE_PRUNED):
        assert_same_bits(sc.render(_cfg(eye, cam, spp=3, traverse=trav)), want, "traverse %d" % trav)
    for fpb in (1, 3):
        assert_same_bits(sc.render(_cfg(eye, cam, spp=3, frames_per_batch=fpb)), want, "frames_per_batch %d" % fpb)
    first = sc.render(_cfg(eye, cam, spp=1))
    assert_same_bits(sc.render(_cfg(eye, cam, spp=2, first_frame=1), framebuffer=first.reshape(-1, 3).copy()), want, "1 then 2 frames")
    W, H = 64, 48
    full = np.zeros((H * W, 3), np.float32)
    for r in range(2):
        part = sc.render(_cfg(eye, cam, spp=3, part_rank=r, part_count=2))
        api.partition_scatter_host(part, full, W, H, 3, r, 2)
    assert_same_bits(full.reshape(H, W, 3), want, "two parts")
    monkeypatch.setenv("EZRT_DEFERRED_LANE", "0")
    sc2 = api.Scene(p3["tris"], p3["nodes"], p3["hdr"], p3["cache"])
    try:
        assert_same_bits(sc2.render(_cfg(eye, cam, spp=3)), want, "deferred lane off")
    finally:
        sc2.close()


def test_small_scene_forced_to_w8(grid_scene, monkeypatch):
    tris, nodes, eye, cam = grid_scene
    monkeypatch.setenv("EZRT_ACCEL", "8")
    sc = api.Scene(tris, nodes)
    try:
        _assert_matches_restatement(sc, tris, nodes, _cfg(eye, cam), "grid scene, W8")
        c = sc.render(_cfg(eye, cam, profile=2)) is not None and sc.counters()
        assert c.node_visits_96 > 0 and c.shadow_rays > 0
    finally:
        sc.close()


def test_s1m_windows_at_1920x1080():
    tris, nodes, eye, cam = scenes.s_1m_bunny()
    sc = api.Scene(tris, nodes)
    try:
        cfg = _cfg(eye, cam, width=1920, height=1080, spp=1, max_bounce=2)
        img = sc.render(cfg)
        assert sc.counters().shadow_rays > 0
        for win in ((0, 0, 48, 32), (936, 524, 984, 556), (1872, 1048, 1920, 1080)):
            ref, _, _ = ol.oracle_render_lights(tris, nodes, cfg, window=win)
            x0, y0, x1, y1 = win
            assert_same_bits(img[y0:y1, x0:x1], ref, "S-1M window %r" % (win,))
    finally:
        sc.close()


def test_adaptive_tiles_equal_plain_renders(p3):
    sc, eye, cam = p3["sc"], p3["eye"], p3["cam"]
    cfg = _cfg(eye, cam, spp=6)
    img, spp, _ = sc.render_adaptive(cfg, 0.5, 2, 2)
    assert len(np.unique(spp)) >= 1
    for s in np.unique(spp):
        plain = sc.render(_cfg(eye, cam, spp=int(s)))
        m = spp == s
        assert_same_bits(img[m], plain[m], "tiles at %d spp" % s)


def test_feature_buffer_render_and_denoise(p3):
    sc, eye, cam = p3["sc"], p3["eye"], p3["cam"]
    cfg = _cfg(eye, cam, spp=3)
    img, aov, luma2 = sc.render_aov(cfg)
    assert_same_bits(img, sc.render(cfg), "aov render framebuffer")
    den = sc.denoise(img, aov, luma2, cfg.spp)
    assert np.isfinite(den).all()


def test_counting_instantiation(p3):
    sc, eye, cam = p3["sc"], p3["eye"], p3["cam"]
    want = sc.render(_cfg(eye, cam))
    assert_same_bits(sc.render(_cfg(eye, cam, profile=2)), want, "profile 2")
    c = sc.counters()
    assert c.node_visits > 0 and c.tri_tests > 0 and c.shadow_rays > 0


def test_rejected_inputs(p3):
    sc, eye, cam = p3["sc"], p3["eye"], p3["cam"]
    for cfg in (_cfg(eye, cam, pipeline=api.PIPELINE_MEGAKERNEL), _cfg(eye, cam, mode=5)):
        with pytest.raises(api.EzrtError) as e:
            sc.render(cfg)
        assert e.value.code == -1


# ------------------------------------------------------------------ the bounded occlusion query, ray by ray
def _hostile_scenes():
    from tests import test_gpu_w8 as w8
    yield "twins", w8.twin_scene()[:2], lambda t: w8.grid_rays(4096, 5, 3.0)
    yield "coincident stacks", w8.stack_scene(0, 11)[:2], lambda t: w8.stack_rays(t, 48, 12)
    yield "ulp stacks", w8.stack_scene(3, 13)[:2], lambda t: w8.stack_rays(t, 48, 14)
    yield "1e8 wide", w8.far_scene(1.0e8, 4)[:2], lambda t: w8.far_rays(t, 2048, 15)


def test_occluded_rays_ray_by_ray(oracle):
    rng = np.random.default_rng(3)
    for name, (tris, nodes), rays in _hostile_scenes():
        o, d = rays(tris)
        hit = oracle.trace_rays(tris, nodes, o, d, traverse=api.TRAVERSE_REFERENCE)
        t = np.where(hit["hit"] != 0, hit["distance"], 10.0).astype(np.float32)
        n = len(o)
        # bounds below, at exactly, and above the closest hit; tiny bounds; and (far scene) origins beyond the decode bound
        tmax = np.choose(rng.integers(0, 4, n), [t * 0.5, t, np.nextafter(t, np.float32(np.inf)), rng.uniform(0, 5e-4, n).astype(np.float32)])
        tmax = tmax.astype(np.float32)
        sc = api.Scene(tris, nodes)
        try:
            for trav in (api.TRAVERSE_ACCEL, api.TRAVERSE_REFERENCE, api.TRAVERSE_PRUNED):
                got = sc.occluded_rays(o, d, tmax, traverse=trav)
                ref = ol.oracle_occluded(tris, nodes, o, d, tmax, traverse=trav)
                bad = np.flatnonzero(got != ref)
                assert bad.size == 0, "%s traverse %d: %d of %d rays differ (first %d)" % (name, trav, bad.size, n, bad[0])
                assert 0 < ref.sum() < n, name
                inf = np.full(n, np.inf, np.float32)
                got = sc.occluded_rays(o, d, inf, traverse=trav)
                assert (got == 1 - sc.trace_rays(o, d, traverse=trav, any_hit=True)["hit"]).all(), name
                assert (got == ol.oracle_occluded(tris, nodes, o, d, inf, traverse=trav)).all(), name
        finally:
            sc.close()
