"""GPU renders with the light tree (EZRT_PARAM_LIGHT_TREE, DESIGN.md section 19): triangle light samples chosen by a tree over the
render's table from the shading point, and the emission hits' MIS pdf walked from the path's previous vertex.

The device's tree is held byte for byte to the host builder's, its descent and walk bit for bit to ezrt_math.h's on the CPU, and
whole renders bit for bit, with equal primary, bounce and shadow ray counts, to the CPU restatement (tests/oracle_light_tree.cpp)
under every option of the light sampling mode; a table without lights renders mode 4's bits; the rejections."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from ezrt_b200._lib import EzrtError
from tests import oracle_light_tree as ot
from tests import oracle_medium
from tests.test_gpu_emission_maps import FOG, _glass, _maps, _scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def p3():
    tris, nodes, eye, cam, tex, uv, ids, eid = scenes.s_p3_bunny_emission_mapped()
    tris = np.asarray(tris, np.float32).reshape(-1, 36)
    hdr = scenes.synth_hdr(64, 32)
    return tris, nodes, eye, cam, tex, uv, ids, eid, hdr, api.hdr_cache(hdr)


@pytest.fixture(scope="module")
def lamps():
    tris, nodes, eye, cam = scenes.s_lamps(3, 2, rough=True)
    return np.asarray(tris, np.float32).reshape(-1, 36), nodes, eye, cam


def _cfg(eye, cam, **kw):
    base = dict(width=48, height=32, spp=2, max_bounce=4, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam), light_tree=True)
    base.update(kw)
    return api.RenderConfig(**base)


def _rays(c):
    return (c.primary_rays, c.bounce_rays, c.shadow_rays)


def _crays(c):
    return (c["rays_primary"], c["rays_bounce"], c["rays_shadow"])


def _hostile_points(tree, n, seed):
    """n points: uniform over the root box and around it, on light vertices, at box centres, 1e30 away, and NaN"""
    rng = np.random.default_rng(seed)
    lo, hi = tree["lo"][0].astype(np.float64), tree["hi"][0].astype(np.float64)
    span = np.maximum(hi - lo, 1e-3)
    P = rng.uniform(lo - span, hi + span, (n, 3))
    m = n // 8
    P[:m] = 0.5 * (tree["lo"][rng.integers(0, len(tree["lo"]), m)] + tree["hi"][rng.integers(0, len(tree["hi"]), m)])
    P[m:2 * m] = tree["lo"][rng.integers(0, len(tree["lo"]), m)]
    P[2 * m:2 * m + 16] = 1e30 * rng.choice([-1.0, 1.0], (16, 3))
    P[2 * m + 16:2 * m + 32] = np.nan
    return P.astype(np.float32)


@pytest.mark.parametrize("emission", [False, True])
def test_device_tree_is_the_builders(p3, emission):
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache = p3
    sc = _scene(tris, nodes, tex, uv, ids, eid)
    try:
        dev = sc.light_tree(emission=emission)
    finally:
        sc.close()
    host = ot.tree_of(tris, eid if emission else None, tex, uv)
    assert dev["nodes"].tobytes() == host["nodes"].tobytes() and dev["paths"].tobytes() == host["paths"].tobytes()


@pytest.mark.parametrize("emission", [False, True])
def test_device_descent_and_walk_equal_the_restatement(p3, emission):
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache = p3
    sc = _scene(tris, nodes, tex, uv, ids, eid)
    try:
        tree = sc.light_tree(emission=emission)
        n = 1000000
        P = _hostile_points(tree, n, 3)
        r = np.random.default_rng(4).uniform(0, 1, n).astype(np.float32)
        r[:64] = np.float32(1.0)
        r[64:128] = np.float32(0.0)
        k, q = sc.sample_light_tree(P, r, emission=emission)
        kk, qq = ot.descend(tree, P, r)
        assert np.array_equal(k, kk) and q.tobytes() == qq.tobytes()
        K = (len(tree["phi"]) + 1) // 2
        light = np.random.default_rng(5).integers(0, K, n).astype(np.int32)
        assert sc.light_tree_prob(P, light, emission=emission).tobytes() == ot.prob(tree, P, light).tobytes()
        ok = k >= 0
        assert sc.light_tree_prob(P[ok], k[ok], emission=emission).tobytes() == q[ok].tobytes()
    finally:
        sc.close()


@pytest.mark.parametrize("traverse", [api.TRAVERSE_ACCEL, api.TRAVERSE_REFERENCE, api.TRAVERSE_PRUNED])
@pytest.mark.parametrize("bounces", [1, 4])
def test_lamps_equal_the_restatement(lamps, traverse, bounces):
    tris, nodes, eye, cam = lamps
    cfg = _cfg(eye, cam, max_bounce=bounces, traverse=traverse, spp=3)
    sc = api.Scene(tris, nodes, device=0)
    try:
        got, gc = sc.render(cfg), sc.counters()
    finally:
        sc.close()
    ref, _, _, c = ot.render(tris, nodes, cfg)
    assert got.tobytes() == ref.tobytes(), "L-inf %.3g" % float(np.abs(got - ref).max())
    assert _rays(gc) == _crays(c)


OPTS = {
    "plain": dict(), "env": dict(env_light=True), "emap": dict(textures=True, emission_maps=True),
    "emap_env": dict(textures=True, emission_maps=True, env_light=True),
    "lens": dict(lens_radius=0.12, focus_distance=3.6, env_light=True), "glass": dict(transmission=True), "glass_env": dict(transmission=True, env_light=True),
    "glass_emap": dict(transmission=True, textures=True, emission_maps=True), "medium": dict(medium=True, env_light=True),
    "medium_emap": dict(medium=True, textures=True, emission_maps=True), "maps": dict(textures=True, material_maps=True, emission_maps=True, env_light=True),
    "punct": dict(punctual_lights=True, env_light=True), "punct_medium": dict(punctual_lights=True, medium=True),
    "punct_glass_emap": dict(punctual_lights=True, transmission=True, textures=True, emission_maps=True),
    "reference": dict(traverse=api.TRAVERSE_REFERENCE, env_light=True), "pruned": dict(traverse=api.TRAVERSE_PRUNED, textures=True, emission_maps=True),
    "batch1": dict(frames_per_batch=1, spp=3), "batch3": dict(frames_per_batch=3, spp=5), "resume": dict(first_frame=2),
    "parts": dict(part_count=2, part_rank=1), "profile2": dict(profile=2),
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
    ref, _, _, c = ot.render(tris, nodes, full, eid, lights=rig, m=oracle_medium.medium(**FOG) if cfg.medium else None, textures=tex, texcoords=uv,
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


@pytest.mark.parametrize("opt", ["plain", "glass", "medium_emap"])
def test_p3_aov_and_adaptive_equal_the_restatement(p3, opt):
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache = p3
    kw = dict(plain=dict(env_light=True), glass=dict(transmission=True, env_light=True),
              medium_emap=dict(medium=True, env_light=True, textures=True, emission_maps=True))[opt]
    if opt == "glass":
        tris = _glass(tris)
    m = oracle_medium.medium(**FOG) if kw.get("medium") else None
    targs = dict(textures=tex, texcoords=uv, texture_id=ids)
    sc = _scene(tris, nodes, tex, uv, ids, eid, hdr, cache, medium=kw.get("medium", False))
    try:
        cfg = _cfg(eye, cam, spp=3, **kw)
        got, gaov, _ = sc.render_aov(cfg)
        ref, _, raov, c = ot.render(tris, nodes, cfg, eid, m=m, hdr=hdr, hdr_cache=cache, aov=True, **targs)
        assert got.tobytes() == ref.tobytes() and gaov.tobytes() == raov.tobytes()
        assert sc.counters().rays == c["rays"]
        acfg = _cfg(eye, cam, spp=6, **kw)
        img, spp, luma2 = sc.render_adaptive(acfg, 0.3, 2, 2)
        ac = sc.counters()
        rimg, rspp, rluma2, rc = ot.render_adaptive(tris, nodes, acfg, 0.3, 2, 2, emission_id=eid, m=m, hdr=hdr, hdr_cache=cache, **targs)
        assert img.tobytes() == rimg.tobytes() and luma2.tobytes() == rluma2.tobytes() and np.array_equal(spp, rspp)
        assert ac.rays == rc["rays"]
    finally:
        sc.close()


def test_w8_lamps_equal_the_restatement(lamps, monkeypatch):
    """a small scene forced onto the 8-wide tree: the deferred rays and the LIST pass walk the tree too"""
    monkeypatch.setenv("EZRT_ACCEL", "8")
    tris, nodes, eye, cam = lamps
    cfg = _cfg(eye, cam, spp=2, max_bounce=4)
    sc = api.Scene(tris, nodes, device=0)
    try:
        got, gc = sc.render(cfg), sc.counters()
    finally:
        sc.close()
    ref, _, _, c = ot.render(tris, nodes, cfg)
    assert got.tobytes() == ref.tobytes() and _rays(gc) == _crays(c)


def test_s1m_lamps_windows_at_1920x1080():
    tris, nodes, eye, cam = scenes.s_1m_lamps()
    sc = api.Scene(tris, nodes, device=0)
    try:
        cfg = _cfg(eye, cam, width=1920, height=1080, spp=1, max_bounce=2)
        img = sc.render(cfg)
    finally:
        sc.close()
    for win in ((0, 0, 48, 32), (928, 528, 976, 560), (1872, 1040, 1920, 1080)):
        ref, _, _, _ = ot.render(tris, nodes, cfg, window=win)
        x0, y0, x1, y1 = win
        assert img[y0:y1, x0:x1].tobytes() == ref.tobytes(), "S-1M lamps window %r" % (win,)


def test_no_lights_renders_mode_4(p3):
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache = p3
    dark = np.array(tris, np.float32, copy=True)
    dark[:, 18:21] = 0.0
    sc = api.Scene(dark, nodes, hdr, cache, device=0)
    try:
        for kw in (dict(), dict(env_light=True)):
            a = sc.render(_cfg(eye, cam, **kw))
            b = sc.render(_cfg(eye, cam, light_tree=False, **kw))
            assert a.tobytes() == b.tobytes()
    finally:
        sc.close()


def test_rejections(p3):
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache = p3
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        for mode in (api.MODE_DIFFUSE_P3, api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5):
            with pytest.raises(EzrtError):
                sc.render(_cfg(eye, cam, mode=mode))
        with pytest.raises(EzrtError):
            sc.render(_cfg(eye, cam, pipeline=api.PIPELINE_MEGAKERNEL))
        with pytest.raises(EzrtError):
            sc.light_tree(emission=True)   # no emission maps
        with pytest.raises(EzrtError):
            sc.light_tree_prob(np.zeros((1, 3)), [10 ** 6])
    finally:
        sc.close()
