"""The thin-lens camera (RenderConfig.lens_radius / EZRT_PARAM_THIN_LENS, DESIGN.md section 13) on the GPU against its CPU
restatement (tests/oracle_lens.cpp): the camera rays bit for bit, renders of every mode bit for bit with their ray counts, the same
bits under every render option, adaptive and feature-buffer renders, the circle of confusion, and the parameters it rejects."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_lens as ol
from tests import transmission_scenes as ts
from tests.test_gpu_parity import assert_same_bits
from tests.test_lens_oracle import COC_CASES, EYE, CAM, _matrices, bad_lens_configs, check_coc, coc_case

pytestmark = pytest.mark.gpu

ENV = (0.35, 0.45, 0.6)


def _cfg(eye, cam, **kw):
    base = dict(width=64, height=48, spp=2, max_bounce=2, mode=api.MODE_DISNEY_SOBOL_P5, eye=tuple(eye), camera_rotate=tuple(cam),
                env_color=ENV, lens_radius=0.08, focus_distance=3.6)
    base.update(kw)
    return api.RenderConfig(**base)


def _check(sc, tris, nodes, cfg, what, hdr=None, cache=None):
    img = sc.render(cfg)
    c = sc.counters()
    ref, _, _, rc = ol.render(tris, nodes, cfg, hdr=hdr, hdr_cache=cache)
    assert_same_bits(img, ref, what)
    assert (c.primary_rays, c.bounce_rays, c.shadow_rays) == (rc["rays_primary"], rc["rays_bounce"], rc["rays_shadow"]), what
    return img


@pytest.fixture(scope="module")
def lens_scenes(small_hdr):
    hdr, cache = small_hdr
    out = {}
    for name, (tris, nodes, eye, cam) in (("bunny", scenes.s_p3_bunny()), ("glass", ts.p3_glass("blob"))):
        out[name] = dict(tris=tris, nodes=nodes, eye=eye, cam=cam, sc=api.Scene(tris, nodes, hdr, cache))
    yield out, hdr, cache
    for d in out.values():
        d["sc"].close()


def test_camera_rays_equal_the_restatement(lens_scenes):
    sc = lens_scenes[0]["bunny"]["sc"]
    rng = np.random.default_rng(1)
    n = 100000
    for name, eye, cam in _matrices():
        px, py, fr = rng.integers(0, 1920, n), rng.integers(0, 1080, n), rng.integers(0, 1 << 31, n)
        for R in (0.0, 0.02, 1.5):
            cfg = _cfg(eye, cam, width=1920, height=1080, lens_radius=R)
            o, d = sc.camera_rays(cfg, px, py, fr)
            want = ol.camera_rays(cfg, px, py, fr)
            assert o.tobytes() == want["o"].tobytes() and d.tobytes() == want["d"].tobytes(), (name, R)


MODES = [(m, False, False) for m in range(5)] + [(4, True, False), (4, False, True), (4, True, True)]


@pytest.mark.parametrize("bounces", [1, 2, 4])
@pytest.mark.parametrize("mode,env_light,trans", MODES)
@pytest.mark.parametrize("scene", ["bunny", "glass"])
def test_renders_bit_identical(lens_scenes, scene, mode, env_light, trans, bounces):
    d, hdr, cache = lens_scenes[0][scene], lens_scenes[1], lens_scenes[2]
    cfg = _cfg(d["eye"], d["cam"], mode=mode, max_bounce=bounces, env_light=env_light, transmission=trans)
    _check(d["sc"], d["tris"], d["nodes"], cfg, "%s mode %d env %s trans %s %d bounces" % (scene, mode, env_light, trans, bounces), hdr, cache)


def test_s1m_windows_at_1920x1080():
    tris, nodes, eye, cam = scenes.s_1m()
    sc = api.Scene(tris, nodes)
    try:
        cfg = _cfg(eye, cam, width=1920, height=1080, spp=1, mode=api.MODE_DISNEY_LIGHTS, max_bounce=2, lens_radius=0.3, focus_distance=12.0)
        img = sc.render(cfg)
        for win in ((0, 0, 48, 32), (928, 528, 976, 560), (1872, 1040, 1920, 1080)):
            ref, _, _, _ = ol.render(tris, nodes, cfg, window=win)
            x0, y0, x1, y1 = win
            assert_same_bits(img[y0:y1, x0:x1], ref, "S-1M lens window %r" % (win,))
    finally:
        sc.close()


def test_w8_gate_and_large_radii(small_hdr, monkeypatch):
    """a small scene forced onto the 8-wide tree; lens origins beyond its decode gate (deferred to the exact kernel); a lens larger
    than the scene"""
    tris, nodes, eye, cam = scenes.s_grid(3, 2, 2)
    hdr, cache = small_hdr
    monkeypatch.setenv("EZRT_ACCEL", "8")
    sc = api.Scene(tris, nodes, hdr, cache)
    try:
        extent = float(np.abs(tris[:, :9]).max())
        for R, what in ((0.05, "W8"), (40.0 * extent, "origins beyond the decode gate"), (3.0 * extent, "radius larger than the scene")):
            for mode in (api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_LIGHTS):
                cfg = _cfg(eye, cam, mode=mode, lens_radius=R, focus_distance=float(np.linalg.norm(eye)))
                _check(sc, tris, nodes, cfg, "%s, mode %d" % (what, mode), hdr, cache)
                if R > 10 * extent:
                    assert sc.counters().deferred_rays > 0
    finally:
        sc.close()


def test_same_bits_under_every_render_option(lens_scenes, monkeypatch):
    d, hdr, cache = lens_scenes[0]["bunny"], lens_scenes[1], lens_scenes[2]
    sc, eye, cam = d["sc"], d["eye"], d["cam"]
    for mode in (api.MODE_DISNEY_IS_MIS_P5, api.MODE_DISNEY_LIGHTS):
        want = sc.render(_cfg(eye, cam, spp=3, mode=mode))
        for trav in (api.TRAVERSE_REFERENCE, api.TRAVERSE_PRUNED):
            assert_same_bits(sc.render(_cfg(eye, cam, spp=3, mode=mode, traverse=trav)), want, "traverse %d" % trav)
            if mode != api.MODE_DISNEY_LIGHTS:
                assert_same_bits(sc.render(_cfg(eye, cam, spp=3, mode=mode, traverse=trav, pipeline=api.PIPELINE_MEGAKERNEL)), want,
                                 "megakernel, traverse %d" % trav)
        for fpb in (1, 3, 0):
            assert_same_bits(sc.render(_cfg(eye, cam, spp=3, mode=mode, frames_per_batch=fpb)), want, "frames_per_batch %d" % fpb)
        first = sc.render(_cfg(eye, cam, spp=1, mode=mode))
        assert_same_bits(sc.render(_cfg(eye, cam, spp=2, first_frame=1, mode=mode), framebuffer=first.reshape(-1, 3).copy()), want, "1 then 2")
        W, H = 64, 48
        full = np.zeros((H * W, 3), np.float32)
        for r in range(2):
            api.partition_scatter_host(sc.render(_cfg(eye, cam, spp=3, mode=mode, part_rank=r, part_count=2)), full, W, H, 3, r, 2)
        assert_same_bits(full.reshape(H, W, 3), want, "two parts")
        assert_same_bits(sc.render(_cfg(eye, cam, spp=3, mode=mode, profile=2)), want, "profile 2")
        monkeypatch.setenv("EZRT_DEFERRED_LANE", "0")
        sc2 = api.Scene(d["tris"], d["nodes"], hdr, cache)
        try:
            assert_same_bits(sc2.render(_cfg(eye, cam, spp=3, mode=mode)), want, "deferred lane off")
        finally:
            sc2.close()
            monkeypatch.delenv("EZRT_DEFERRED_LANE")
    for mode in (0, 1, 2):   # the megakernel in the other modes
        cfg = _cfg(eye, cam, spp=2, mode=mode, pipeline=api.PIPELINE_MEGAKERNEL)
        assert_same_bits(sc.render(cfg), ol.render(d["tris"], d["nodes"], cfg, hdr=hdr, hdr_cache=cache)[0], "megakernel mode %d" % mode)


def test_adaptive_and_feature_buffers(lens_scenes):
    d, hdr, cache = lens_scenes[0]["glass"], lens_scenes[1], lens_scenes[2]
    sc, eye, cam = d["sc"], d["eye"], d["cam"]
    for mode, trans in ((api.MODE_DISNEY_SOBOL_P5, False), (api.MODE_DISNEY_LIGHTS, True)):
        cfg = _cfg(eye, cam, spp=6, mode=mode, transmission=trans)
        img, spp, luma2 = sc.render_adaptive(cfg, 0.5, 2, 2)
        rimg, rspp, rluma2, _ = ol.render_adaptive(d["tris"], d["nodes"], cfg, 0.5, 2, 2, hdr=hdr, hdr_cache=cache)
        assert_same_bits(img, rimg, "adaptive")
        assert (spp == rspp).all() and luma2.tobytes() == rluma2.tobytes()
        for s in np.unique(spp):
            plain = sc.render(_cfg(eye, cam, spp=int(s), mode=mode, transmission=trans))
            assert_same_bits(img[spp == s], plain[spp == s], "tiles at %d spp" % s)
        cfg = _cfg(eye, cam, spp=3, mode=mode, transmission=trans)
        img, aov, luma2 = sc.render_aov(cfg)
        assert_same_bits(img, sc.render(cfg), "aov render framebuffer")
        _, rluma2, raov, _ = ol.render(d["tris"], d["nodes"], cfg, hdr=hdr, hdr_cache=cache, aov=True)
        assert aov.tobytes() == raov.tobytes() and luma2.tobytes() == rluma2.tobytes()


@pytest.mark.parametrize("z,R", COC_CASES)
def test_circle_of_confusion(z, R):
    def render(tris, nodes, cfg):
        sc = api.Scene(tris, nodes)
        try:
            return sc.render(cfg)
        finally:
            sc.close()
    check_coc(coc_case(render, z, R), z)


def test_rejected_parameters(lens_scenes):
    sc = lens_scenes[0]["bunny"]["sc"]
    for what, cfg in bad_lens_configs(EYE, CAM):
        for call in (lambda: sc.render(cfg), lambda: sc.camera_rays(cfg, [0], [0], [0]), lambda: sc.render_aov(cfg),
                     lambda: sc.render_adaptive(cfg, 0.5, 2, 2)):
            with pytest.raises(api.EzrtError) as e:
                call()
            assert e.value.code == -1, what
