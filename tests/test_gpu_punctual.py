"""GPU renders with punctual lights (EZRT_PARAM_PUNCTUAL_LIGHTS, DESIGN.md section 17): point, spot and directional lights as a third
category of light samples.

Whole renders are held bit for bit, with equal primary, bounce and shadow ray counts, to the CPU restatement (tests/oracle_punctual.cpp)
under every option of the light sampling mode; the table to the restatement's; lights of weight 0 to mode 4; and the rejections."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from ezrt_b200._lib import EzrtError
from tests import oracle_medium
from tests import oracle_punctual as op

pytestmark = pytest.mark.gpu

FOG = dict(sigma_t=0.6, albedo=(0.9, 0.8, 0.7), g=0.4, box_min=(-1.2, -1.0, -1.2), box_max=(1.2, 1.4, 1.2))


@pytest.fixture(scope="module")
def p3():
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    tris = np.asarray(tris, np.float32).reshape(-1, 36)
    hdr = scenes.synth_hdr(64, 32)
    return tris, nodes, eye, cam, scenes.punctual_rig(tris, seed=1), hdr, api.hdr_cache(hdr)


def _cfg(eye, cam, **kw):
    base = dict(width=48, height=32, spp=2, max_bounce=4, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam),
                punctual_lights=True)
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


def _scene(tris, nodes, lights, hdr=None, cache=None, medium=False, textured=None):
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    if medium:
        sc.set_medium(**FOG)
    if textured is not None:
        tex, uv, ids, mr, nm = textured
        sc.set_textures(tex, uv, ids)
        if mr is not None:
            sc.set_material_maps(mr, nm)
    sc.set_punctual_lights(lights)
    return sc


@pytest.mark.parametrize("bounces", [1, 4, 8])
@pytest.mark.parametrize("env", ["none", "map", "env_light"])
@pytest.mark.parametrize("lens", [False, True])
def test_p3_rig_equals_the_restatement(p3, bounces, env, lens):
    tris, nodes, eye, cam, rig, hdr, cache = p3
    h, c_ = (hdr, cache) if env != "none" else (None, None)
    kw = dict(max_bounce=bounces, env_light=(env == "env_light"))
    if lens:
        kw.update(lens_radius=0.12, focus_distance=3.6)
    cfg = _cfg(eye, cam, **kw)
    sc = _scene(tris, nodes, rig, h, c_)
    try:
        got, gc = sc.render(cfg), sc.counters()
    finally:
        sc.close()
    ref, _, _, c = op.render(tris, nodes, cfg, rig, hdr=h, hdr_cache=c_)
    assert got.tobytes() == ref.tobytes(), "L-inf %.3g" % float(np.abs(got - ref).max())
    assert _rays(gc) == _crays(c)


OPTS = {
    "glass": dict(transmission=True), "glass_env": dict(transmission=True, env_light=True), "medium": dict(medium=True, env_light=True),
    "medium_plain": dict(medium=True), "textures": dict(textures=True, env_light=True), "maps": dict(textures=True, material_maps=True, env_light=True),
    "maps_glass": dict(textures=True, material_maps=True, transmission=True), "maps_medium": dict(textures=True, material_maps=True, medium=True),
    "reference": dict(traverse=api.TRAVERSE_REFERENCE), "pruned": dict(traverse=api.TRAVERSE_PRUNED), "batch1": dict(frames_per_batch=1, spp=3),
    "batch3": dict(frames_per_batch=3, spp=5), "resume": dict(first_frame=2), "parts": dict(part_count=2, part_rank=1), "profile2": dict(profile=2),
    "no_emitters": dict(), "no_emitters_medium": dict(medium=True),
}


@pytest.mark.parametrize("opt", sorted(OPTS))
def test_p3_rig_options_equal_the_restatement(p3, opt):
    tris, nodes, eye, cam, rig, hdr, cache = p3
    kw = dict(OPTS[opt])
    textured = None
    tex_args = {}
    if kw.get("textures"):
        mt, mnodes, meye, mcam, tex, uv, ids, mr, nm = scenes.s_p3_bunny_mapped()
        tris, nodes, eye, cam = np.asarray(mt, np.float32).reshape(-1, 36), mnodes, meye, mcam
        if not kw.get("material_maps"):
            mr = nm = None
        textured = (tex, uv, ids, mr, nm)
        tex_args = dict(textures=tex, texcoords=uv, texture_id=ids, metal_rough_id=mr, normal_id=nm)
    if kw.get("transmission"):
        tris = _glass(tris)
    if opt.startswith("no_emitters"):   # no triangle light and no map table: P_p = 1
        tris = np.array(tris, np.float32, copy=True)
        tris[:, 18:21] = 0.0
    cfg = _cfg(eye, cam, **kw)
    sc = _scene(tris, nodes, rig, hdr, cache, medium=cfg.medium, textured=textured)
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
    ref, _, _, c = op.render(tris, nodes, full, rig, m=oracle_medium.medium(**FOG) if cfg.medium else None, hdr=hdr, hdr_cache=cache, **tex_args)
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
def test_p3_rig_aov_and_adaptive_equal_the_restatement(p3, opt):
    tris, nodes, eye, cam, rig, hdr, cache = p3
    kw = dict(plain=dict(env_light=True), glass=dict(transmission=True, env_light=True), medium=dict(medium=True, env_light=True))[opt]
    if opt == "glass":
        tris = _glass(tris)
    m = oracle_medium.medium(**FOG) if opt == "medium" else None
    sc = _scene(tris, nodes, rig, hdr, cache, medium=(opt == "medium"))
    try:
        cfg = _cfg(eye, cam, spp=3, **kw)
        got, gaov, _ = sc.render_aov(cfg)
        ref, _, raov, c = op.render(tris, nodes, cfg, rig, m=m, hdr=hdr, hdr_cache=cache, aov=True)
        assert got.tobytes() == ref.tobytes() and gaov.tobytes() == raov.tobytes()
        assert sc.counters().rays == c["rays"]
        acfg = _cfg(eye, cam, spp=6, **kw)
        img, spp, luma2 = sc.render_adaptive(acfg, 0.3, 2, 2)
        ac = sc.counters()
        rimg, rspp, rluma2, rc = op.render_adaptive(tris, nodes, acfg, rig, 0.3, 2, 2, m=m, hdr=hdr, hdr_cache=cache)
        assert img.tobytes() == rimg.tobytes() and luma2.tobytes() == rluma2.tobytes() and np.array_equal(spp, rspp)
        assert ac.rays == rc["rays"]
        # each adaptive tile equals a plain render at its own spp
        n = int(spp[0, 0])
        plain = sc.render(_cfg(eye, cam, spp=n, **kw))
        assert img[:16, :16].tobytes() == plain[:16, :16].tobytes()
    finally:
        sc.close()


def test_s1m_rig_windows_at_1920x1080():
    tris, nodes, eye, cam = scenes.s_1m_bunny()
    rig = scenes.punctual_rig(tris, seed=2)
    sc = _scene(tris, nodes, rig)
    try:
        cfg = _cfg(eye, cam, width=1920, height=1080, spp=1, max_bounce=3)
        img = sc.render(cfg)
    finally:
        sc.close()
    for win in ((0, 0, 48, 32), (928, 528, 976, 560), (1872, 1040, 1920, 1080)):
        ref, _, _, _ = op.render(tris, nodes, cfg, rig, window=win)
        x0, y0, x1, y1 = win
        assert img[y0:y1, x0:x1].tobytes() == ref.tobytes(), "S-1M window %r" % (win,)


def test_w8_rig_equals_the_restatement(monkeypatch):
    """a small scene forced onto the 8-wide tree: deferred rays and the LIST pass carry punctual samples too"""
    monkeypatch.setenv("EZRT_ACCEL", "8")
    tris, nodes, eye, cam = scenes.s_grid(3, 2, 2)
    rig = scenes.punctual_rig(tris, seed=4)
    cfg = _cfg(eye, cam, spp=2, max_bounce=4)
    sc = _scene(tris, nodes, rig)
    try:
        got, gc = sc.render(cfg), sc.counters()
    finally:
        sc.close()
    ref, _, _, c = op.render(tris, nodes, cfg, rig)
    assert got.tobytes() == ref.tobytes() and _rays(gc) == _crays(c)


def test_table_equals_the_restatement(p3):
    tris, nodes, eye, cam, rig, hdr, cache = p3
    lights = rig + [api.point_light((0, 1, 0), (1, 1, 1), 0.0), api.spot_light((0, 2, 0), (0, -1, 0), (0.5, 0.2, 0.1), 1e-4, 0.3, 0.4)]
    sc = api.Scene(tris, nodes, device=0)
    try:
        assert sc.punctual_light_table()[0].size == 0
        sc.set_punctual_lights(lights)
        idx, cdf, q, W = sc.punctual_light_table()
    finally:
        sc.close()
    ridx, rcdf, rq, _, rW = op.table(tris, lights)
    assert idx.tobytes() == ridx.tobytes() and cdf.tobytes() == rcdf.tobytes() and q.tobytes() == rq.tobytes() and W == rW


@pytest.mark.parametrize("opt", ["plain", "env_light", "medium", "glass"])
def test_zero_lights_equal_mode4(p3, opt):
    tris, nodes, eye, cam, _, hdr, cache = p3
    kw = dict(plain={}, env_light=dict(env_light=True), medium=dict(medium=True, env_light=True), glass=dict(transmission=True, env_light=True))[opt]
    if opt == "glass":
        tris = _glass(tris)
    zero = [api.point_light((0, 1, 0), (1, 1, 1), 0.0), api.directional_light((0, -1, 0), (0, 0, 0), 3.0)]
    sc = _scene(tris, nodes, zero, hdr, cache, medium=(opt == "medium"))
    try:
        got, gc = sc.render(_cfg(eye, cam, **kw)), _rays(sc.counters())
        want, wc = sc.render(_cfg(eye, cam, punctual_lights=False, **kw)), _rays(sc.counters())
    finally:
        sc.close()
    assert got.tobytes() == want.tobytes() and gc == wc


def test_rejections(p3):
    tris, nodes, eye, cam, rig, hdr, cache = p3
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        with pytest.raises(EzrtError):   # the flag without lights
            sc.render(_cfg(eye, cam))
        sc.set_punctual_lights(rig)
        for mode in (api.MODE_DIFFUSE_P3, api.MODE_DISNEY_ANISO_P4, api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5):
            with pytest.raises(EzrtError):
                sc.render(_cfg(eye, cam, mode=mode))
        with pytest.raises(EzrtError):
            sc.render(_cfg(eye, cam, pipeline=api.PIPELINE_MEGAKERNEL))
        before = sc.punctual_light_table()
        for bad in (api.point_light((np.nan, 0, 0)), api.spot_light((0, 0, 0), (0, 0, 0)), api.point_light((0, 0, 0), intensity=-1.0),
                    api.spot_light((0, 0, 0), (0, -1, 0), inner_cone=0.6, outer_cone=0.5), api._punctual(7)):
            with pytest.raises(EzrtError):
                sc.set_punctual_lights(rig + [bad])
            after = sc.punctual_light_table()
            assert all(np.array_equal(a, b) for a, b in zip(before[:3], after[:3])) and before[3] == after[3]   # the previous lights are kept
        sc.set_punctual_lights(None)
        with pytest.raises(EzrtError):
            sc.render(_cfg(eye, cam))
    finally:
        sc.close()
