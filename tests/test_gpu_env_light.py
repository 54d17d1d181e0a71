"""The environment map as a light (RenderConfig.env_light / EZRT_PARAM_ENV_LIGHT in the light sampling mode, DESIGN.md section 11)
on the GPU against its CPU restatement (tests/oracle_env_light.cpp): renders bit for bit with their ray counts, the table, the same
bits under every render option, the inputs it rejects, and the bounded shadow kernels at tmax = 114514 against mode 3's unbounded
ones ray by ray on the hostile scenes of tests/test_gpu_w8.py."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_env_light as oe
from tests import oracle_lights as ol
from tests.test_gpu_parity import assert_same_bits

pytestmark = pytest.mark.gpu

ENV = (0.35, 0.45, 0.6)
L4 = api.MODE_DISNEY_LIGHTS


def _cfg(eye, cam, **kw):
    base = dict(width=64, height=48, spp=2, max_bounce=2, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam), env_color=ENV, env_light=True)
    base.update(kw)
    return api.RenderConfig(**base)


@pytest.fixture(scope="module")
def p3(small_hdr):
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    hdr, cache = small_hdr
    sc = api.Scene(tris, nodes, hdr, cache)
    sc_near = api.Scene(tris, nodes, hdr, cache, hdr_filter_linear=False)
    sc_none = api.Scene(tris, nodes)
    yield dict(tris=tris, nodes=nodes, eye=eye, cam=cam, hdr=hdr, cache=cache, sc=sc, sc_near=sc_near, sc_none=sc_none)
    for s in (sc, sc_near, sc_none):
        s.close()


def _assert_matches_restatement(sc, tris, nodes, cfg, what, hdr=None, cache=None, linear=True, window=None):
    img = sc.render(cfg)
    c = sc.counters()
    ref, _, rc = oe.oracle_render_env_light(tris, nodes, cfg, hdr=hdr, hdr_cache=cache, hdr_linear=linear, window=window)
    if window is not None:
        x0, y0, x1, y1 = window
        img = img[y0:y1, x0:x1]
    assert_same_bits(img, ref, what)
    if window is None:
        assert (c.primary_rays, c.bounce_rays, c.shadow_rays) == (rc["rays_primary"], rc["rays_bounce"], rc["rays_shadow"]), what
        assert c.shadow_rays > 0, what
    return img


@pytest.mark.parametrize("filt", ["linear", "nearest"])
@pytest.mark.parametrize("bounces", [1, 2, 4])
def test_p3_bunny_bit_identical(p3, filt, bounces):
    linear = filt == "linear"
    sc = p3["sc"] if linear else p3["sc_near"]
    _assert_matches_restatement(sc, p3["tris"], p3["nodes"], _cfg(p3["eye"], p3["cam"], max_bounce=bounces), "P3 bunny, %s map, %d bounces" %
                                (filt, bounces), p3["hdr"], p3["cache"], linear)


def test_no_map_is_mode_4(p3):
    sc, eye, cam = p3["sc_none"], p3["eye"], p3["cam"]
    img = _assert_matches_restatement(sc, p3["tris"], p3["nodes"], _cfg(eye, cam), "P3 bunny, no map")
    assert_same_bits(img, sc.render(_cfg(eye, cam, env_light=False)), "no map: flagged vs plain mode 4")
    assert sc.env_light_table() is None


def test_env_table_matches_restatement(p3):
    got = p3["sc"].env_light_table()
    want = oe.env_table(p3["hdr"])
    for g, w, name in zip(got[:3], want[:3], ("row_cdf", "col_cdf", "texel_pdf")):
        assert g.tobytes() == w.tobytes(), name
    assert got[3] == want[3]


def test_same_bits_under_every_render_option(p3, monkeypatch):
    sc, eye, cam = p3["sc"], p3["eye"], p3["cam"]
    want = sc.render(_cfg(eye, cam, spp=3))
    for trav in (api.TRAVERSE_REFERENCE, api.TRAVERSE_PRUNED):
        assert_same_bits(sc.render(_cfg(eye, cam, spp=3, traverse=trav)), want, "traverse %d" % trav)
    for fpb in (1, 3, 0):
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


def test_small_scene_forced_to_w8(grid_scene, small_hdr, monkeypatch):
    tris, nodes, eye, cam = grid_scene
    hdr, cache = small_hdr
    monkeypatch.setenv("EZRT_ACCEL", "8")
    sc = api.Scene(tris, nodes, hdr, cache)
    try:
        _assert_matches_restatement(sc, tris, nodes, _cfg(eye, cam), "grid scene, W8", hdr, cache)
        sc.render(_cfg(eye, cam, profile=2))
        c = sc.counters()
        assert c.node_visits_96 > 0 and c.shadow_rays > 0
    finally:
        sc.close()


def test_c4_scene_windows_at_1920x1080():
    """bench.py's C4 scene: S-1M under the 2048 x 1024 map, in tile-aligned windows of a 1920 x 1080 render."""
    tris, nodes, eye, cam = scenes.s_1m_bunny()
    hdr = scenes.synth_hdr(2048, 1024)
    cache = api.hdr_cache(hdr)
    sc = api.Scene(tris, nodes, hdr, cache)
    try:
        cfg = _cfg(eye, cam, width=1920, height=1080, spp=1, max_bounce=2)
        img = sc.render(cfg)
        assert sc.counters().shadow_rays > 0
        for win in ((0, 0, 48, 32), (928, 528, 976, 560), (1872, 1040, 1920, 1080)):
            ref, _, _ = oe.oracle_render_env_light(tris, nodes, cfg, hdr=hdr, hdr_cache=cache, window=win)
            x0, y0, x1, y1 = win
            assert_same_bits(img[y0:y1, x0:x1], ref, "C4 window %r" % (win,))
    finally:
        sc.close()


def test_adaptive_tiles_equal_plain_renders(p3):
    sc, eye, cam = p3["sc"], p3["eye"], p3["cam"]
    img, spp, _ = sc.render_adaptive(_cfg(eye, cam, spp=6), 0.5, 2, 2)
    for s in np.unique(spp):
        plain = sc.render(_cfg(eye, cam, spp=int(s)))
        m = spp == s
        assert_same_bits(img[m], plain[m], "tiles at %d spp" % s)


def test_feature_buffer_render(p3):
    sc, eye, cam = p3["sc"], p3["eye"], p3["cam"]
    cfg = _cfg(eye, cam, spp=3)
    img, aov, luma2 = sc.render_aov(cfg)
    assert_same_bits(img, sc.render(cfg), "aov render framebuffer")
    _, rluma2, _ = oe.oracle_render_env_light(p3["tris"], p3["nodes"], cfg, hdr=p3["hdr"], hdr_cache=p3["cache"])
    assert luma2.tobytes() == rluma2.tobytes()


def test_counting_instantiation(p3):
    sc, eye, cam = p3["sc"], p3["eye"], p3["cam"]
    want = sc.render(_cfg(eye, cam))
    assert_same_bits(sc.render(_cfg(eye, cam, profile=2)), want, "profile 2")
    c = sc.counters()
    assert c.node_visits > 0 and c.tri_tests > 0 and c.shadow_rays > 0


def test_rejected_inputs(p3):
    sc, eye, cam = p3["sc"], p3["eye"], p3["cam"]
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


def test_occluded_rays_at_the_shaders_inf_equal_unbounded():
    """The environment samples' shadow rays run in the bounded kernels with tmax = 114514; mode 3's run in the unbounded ones."""
    from tests.test_gpu_lights import _hostile_scenes
    for name, (tris, nodes), rays in _hostile_scenes():
        o, d = rays(tris)
        n = len(o)
        sc = api.Scene(tris, nodes)
        try:
            for trav in (api.TRAVERSE_ACCEL, api.TRAVERSE_REFERENCE, api.TRAVERSE_PRUNED):
                bounded = sc.occluded_rays(o, d, np.full(n, 114514.0, np.float32), traverse=trav)
                unbounded = sc.occluded_rays(o, d, np.full(n, np.inf, np.float32), traverse=trav)
                bad = np.flatnonzero(bounded != unbounded)
                assert bad.size == 0, "%s traverse %d: %d of %d rays differ" % (name, trav, bad.size, n)
                assert (bounded == ol.oracle_occluded(tris, nodes, o, d, np.full(n, 114514.0, np.float32), traverse=trav)).all(), name
                assert 0 < bounded.sum() < n, name
        finally:
            sc.close()
