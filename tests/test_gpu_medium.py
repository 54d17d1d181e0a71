"""GPU renders of the homogeneous medium (EZRT_PARAM_MEDIUM, DESIGN.md section 14) against the CPU restatement
(tests/oracle_medium.cpp), bit for bit and ray for ray, and the renders the library rejects."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_medium

pytestmark = pytest.mark.gpu

FOG = dict(sigma_t=0.8, albedo=(0.9, 0.8, 0.7), g=0.5, box_min=(-1.2, -1.0, -1.2), box_max=(1.2, 1.4, 1.2))


@pytest.fixture(scope="module")
def p3():
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    hdr = scenes.synth_hdr(64, 32)
    cache = api.hdr_cache(hdr)
    return tris, nodes, eye, cam, hdr, cache


def _render_both(sc, tris, nodes, cfg, fog, hdr, cache, aov=False):
    sc.set_medium(**fog)
    if aov:
        got, gaov, _ = sc.render_aov(cfg)
    else:
        got, gaov = sc.render(cfg), None
    gc = sc.counters()
    ref, _, raov, c = oracle_medium.render(tris, nodes, cfg, oracle_medium.medium(**fog), hdr=hdr, hdr_cache=cache, aov=aov)
    return got, gaov, gc, ref, raov, c


def _cfg(eye, cam, **kw):
    base = dict(width=48, height=32, spp=2, max_bounce=4, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam), medium=True)
    base.update(kw)
    return api.RenderConfig(**base)


@pytest.mark.parametrize("bounces", [1, 4, 8])
@pytest.mark.parametrize("env", ["none", "map", "env_light"])
@pytest.mark.parametrize("lens", [False, True])
def test_p3_fog_bits(p3, bounces, env, lens):
    tris, nodes, eye, cam, hdr, cache = p3
    h, c_ = (hdr, cache) if env != "none" else (None, None)
    sc = api.Scene(tris, nodes, h, c_, device=0)
    try:
        kw = dict(max_bounce=bounces, env_light=(env == "env_light"))
        if lens:
            kw.update(lens_radius=0.15, focus_distance=3.6)
        got, _, gc, ref, _, c = _render_both(sc, tris, nodes, _cfg(eye, cam, **kw), FOG, h, c_)
    finally:
        sc.close()
    assert got.tobytes() == ref.tobytes(), "L-inf %.3g" % float(np.abs(got - ref).max())
    assert (gc.primary_rays, gc.bounce_rays, gc.shadow_rays) == (c["rays_primary"], c["rays_bounce"], c["rays_shadow"])


@pytest.mark.parametrize("opt", ["reference", "pruned", "batch1", "batch3", "resume", "parts", "profile2", "dense", "g_back", "g_fwd"])
def test_fog_options_bits(p3, opt):
    tris, nodes, eye, cam, hdr, cache = p3
    fog = dict(FOG)
    kw = dict(env_light=True)
    if opt == "reference":
        kw["traverse"] = api.TRAVERSE_REFERENCE
    elif opt == "pruned":
        kw["traverse"] = api.TRAVERSE_PRUNED
    elif opt == "batch1":
        kw.update(frames_per_batch=1, spp=3)
    elif opt == "batch3":
        kw.update(frames_per_batch=3, spp=4)
    elif opt == "profile2":
        kw["profile"] = 2
    elif opt == "dense":
        fog.update(sigma_t=4000.0)
    elif opt == "g_back":
        fog.update(g=-0.999)
    elif opt == "g_fwd":
        fog.update(g=0.999)
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        if opt == "resume":
            cfg = _cfg(eye, cam, spp=2, **kw)
            sc.set_medium(**fog)
            first = sc.render(cfg)
            cfg2 = _cfg(eye, cam, spp=2, first_frame=2, **kw)
            got = sc.render(cfg2, framebuffer=first.copy())
            ref, _, _, _ = oracle_medium.render(tris, nodes, _cfg(eye, cam, spp=4, **kw), oracle_medium.medium(**fog), hdr=hdr, hdr_cache=cache)
            assert got.tobytes() == ref.tobytes()
            return
        if opt == "parts":
            sc.set_medium(**fog)
            cfg = _cfg(eye, cam, **kw)
            full = np.zeros((cfg.height, cfg.width, 3), np.float32)
            for r in range(2):
                full = api.partition_scatter_host(sc.render(_cfg(eye, cam, part_rank=r, part_count=2, **kw)), full, cfg.width, cfg.height, 3, r, 2)
            ref, _, _, _ = oracle_medium.render(tris, nodes, cfg, oracle_medium.medium(**fog), hdr=hdr, hdr_cache=cache)
            assert full.reshape(ref.shape).tobytes() == ref.tobytes()
            return
        got, _, gc, ref, _, c = _render_both(sc, tris, nodes, _cfg(eye, cam, **kw), fog, hdr, cache)
    finally:
        sc.close()
    assert np.isfinite(got).all()
    assert got.tobytes() == ref.tobytes(), "L-inf %.3g" % float(np.abs(got - ref).max())
    assert gc.rays == c["rays"]


def test_s1m_windows_at_1920x1080():
    tris, nodes, eye, cam = scenes.s_1m()
    p = tris[:, :9].reshape(-1, 3)
    lo, hi = p.min(0), p.max(0)
    fog = dict(sigma_t=2.0 / float(hi[1] - lo[1]), albedo=(0.8, 0.8, 0.8), g=0.3, box_min=tuple(lo), box_max=tuple(hi))
    sc = api.Scene(tris, nodes)
    try:
        sc.set_medium(**fog)
        cfg = _cfg(eye, cam, width=1920, height=1080, spp=1, max_bounce=3)
        img = sc.render(cfg)
        for win in ((0, 0, 48, 32), (928, 528, 976, 560), (1872, 1040, 1920, 1080)):
            ref, _, _, _ = oracle_medium.render(tris, nodes, cfg, oracle_medium.medium(**fog), window=win)
            x0, y0, x1, y1 = win
            assert img[y0:y1, x0:x1].tobytes() == ref.tobytes(), "S-1M fog window %r" % (win,)
    finally:
        sc.close()


def test_w8_and_a_fog_box_larger_than_the_scene(monkeypatch):
    """a small scene forced onto the 8-wide tree; then a fog box far larger than the scene, so that medium vertices lie beyond the
    8-wide tree's decode gate: their bounce and shadow rays are deferred to the exact kernel and shaded by the LIST pass"""
    tris, nodes, eye, cam = scenes.s_grid(3, 2, 2)
    hdr = scenes.synth_hdr(64, 32)
    cache = api.hdr_cache(hdr)
    monkeypatch.setenv("EZRT_ACCEL", "8")
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        extent = float(np.abs(tris[:, :9]).max())
        cases = (("W8, fog over the scene", dict(FOG, box_min=(-5.0, -1.5, -5.0), box_max=(5.0, 3.5, 5.0)), False),
                 ("fog box 100x the scene", dict(sigma_t=1.0 / (30.0 * extent), albedo=(0.9, 0.9, 0.9), g=0.2,
                                                 box_min=(-100 * extent,) * 3, box_max=(100 * extent,) * 3), True))
        for what, fog, far in cases:
            for env_light in (False, True):
                cfg = _cfg(eye, cam, spp=2, max_bounce=4, env_light=env_light)
                got, _, gc, ref, _, c = _render_both(sc, tris, nodes, cfg, fog, hdr, cache)
                assert got.tobytes() == ref.tobytes(), (what, env_light)
                assert (gc.primary_rays, gc.bounce_rays, gc.shadow_rays) == (c["rays_primary"], c["rays_bounce"], c["rays_shadow"]), what
                if far:
                    assert gc.deferred_rays > 0, what
    finally:
        sc.close()


def test_deferred_lane_off(p3, monkeypatch):
    tris, nodes, eye, cam, hdr, cache = p3
    cfg = _cfg(eye, cam, spp=3, env_light=True)
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        sc.set_medium(**FOG)
        want = sc.render(cfg)
    finally:
        sc.close()
    monkeypatch.setenv("EZRT_DEFERRED_LANE", "0")
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        sc.set_medium(**FOG)
        assert sc.render(cfg).tobytes() == want.tobytes()
    finally:
        sc.close()


def test_fog_aov_and_adaptive(p3):
    tris, nodes, eye, cam, hdr, cache = p3
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        cfg = _cfg(eye, cam, env_light=True, spp=3)
        got, gaov, gc, ref, raov, c = _render_both(sc, tris, nodes, cfg, FOG, hdr, cache, aov=True)
        assert got.tobytes() == ref.tobytes() and gaov.tobytes() == raov.tobytes()
        assert gc.rays == c["rays"]
        acfg = _cfg(eye, cam, env_light=True, spp=6)
        img, spp, luma2 = sc.render_adaptive(acfg, 0.3, 2, 2)
        ac = sc.counters()
        rimg, rspp, rluma2, rc = oracle_medium.render_adaptive(tris, nodes, acfg, oracle_medium.medium(**FOG), 0.3, 2, 2, hdr=hdr, hdr_cache=cache)
        assert img.tobytes() == rimg.tobytes() and luma2.tobytes() == rluma2.tobytes() and np.array_equal(spp, rspp)
        assert ac.rays == rc["rays"] and ac.samples == int(spp.sum())
        for n in sorted(set(spp.ravel().tolist())):
            plain = sc.render(_cfg(eye, cam, env_light=True, spp=int(n)))
            m = spp == n
            assert img[m].tobytes() == plain[m].tobytes()
    finally:
        sc.close()


@pytest.mark.parametrize("env_light", [False, True])
@pytest.mark.parametrize("lens", [False, True])
def test_untouched_box_equals_mode4(p3, env_light, lens):
    tris, nodes, eye, cam, hdr, cache = p3
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        kw = dict(env_light=env_light)
        if lens:
            kw.update(lens_radius=0.1, focus_distance=3.5)
        sc.set_medium(sigma_t=5.0, albedo=(0.5, 0.5, 0.5), g=0.2, box_min=(50.0, 50.0, 50.0), box_max=(51.0, 51.0, 51.0))
        got = sc.render(_cfg(eye, cam, **kw))
        gc = sc.counters()
        plain = sc.render(_cfg(eye, cam, medium=False, **kw))
        pc = sc.counters()
    finally:
        sc.close()
    assert got.tobytes() == plain.tobytes()
    assert (gc.primary_rays, gc.bounce_rays, gc.shadow_rays) == (pc.primary_rays, pc.bounce_rays, pc.shadow_rays)


def test_invalid_renders_rejected(p3):
    tris, nodes, eye, cam, hdr, cache = p3
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        with pytest.raises(api.EzrtError):   # no medium set
            sc.render(_cfg(eye, cam))
        sc.set_medium(**FOG)
        bad = [dict(mode=api.MODE_DISNEY_IS_MIS_P5), dict(mode=api.MODE_DISNEY_SOBOL_P5), dict(pipeline=api.PIPELINE_MEGAKERNEL),
               dict(transmission=True)]
        for kw in bad:
            for call in (lambda c: sc.render(c), lambda c: sc.render_aov(c), lambda c: sc.render_adaptive(c, 0.1, 2, 2)):
                with pytest.raises(api.EzrtError):
                    call(_cfg(eye, cam, **kw))
        box = dict(box_min=(-1.0, -1.0, -1.0), box_max=(1.0, 1.0, 1.0))
        for m in [dict(sigma_t=-1.0), dict(sigma_t=float("inf")), dict(sigma_t=float("nan")), dict(sigma_t=1.0, albedo=(1.5, 0, 0)),
                  dict(sigma_t=1.0, albedo=(float("nan"), 0, 0)), dict(sigma_t=1.0, g=1.0), dict(sigma_t=1.0, g=float("nan")),
                  dict(sigma_t=1.0, box_min=(1.0, 0, 0), box_max=(0.0, 1, 1)), dict(sigma_t=1.0, box_max=(float("inf"), 1, 1))]:
            with pytest.raises(api.EzrtError):   # rejected by the library
                sc.set_medium(**{**box, **m})
        with pytest.raises(ValueError):   # the box is required
            sc.set_medium(1.0)
    finally:
        sc.close()
