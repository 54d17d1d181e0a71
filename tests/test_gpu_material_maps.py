"""GPU renders with material maps (EZRT_PARAM_MATERIAL_MAPS, DESIGN.md section 16): metallic-roughness and tangent-space normal maps.

Whole renders are held bit for bit, with equal ray counts, to the CPU restatement (tests/oracle_material_maps.cpp) under every option;
the per-hit lookup (Scene.sample_materials) to a float64 model; and the maps' exact invariances to the textured renders."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_material_maps as om
from tests import oracle_medium
from tests.material_maps_model import UNORM, normal_map64, unorm_sample64
from tests.texture_model import sample64

pytestmark = pytest.mark.gpu

FOG = dict(sigma_t=0.6, albedo=(0.9, 0.8, 0.7), g=0.4, box_min=(-1.2, -1.0, -1.2), box_max=(1.2, 1.4, 1.2))
ROUGH, METAL = 28, 25


@pytest.fixture(scope="module")
def p3():
    tris, nodes, eye, cam, tex, uv, ids, mr, nm = scenes.s_p3_bunny_mapped()
    hdr = scenes.synth_hdr(64, 32)
    return tris, nodes, eye, cam, tex, uv, ids, mr, nm, hdr, api.hdr_cache(hdr)


def _cfg(eye, cam, **kw):
    base = dict(width=48, height=32, spp=2, max_bounce=4, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam), textures=True,
                material_maps=True)
    base.update(kw)
    return api.RenderConfig(**base)


def _rays(c):
    return (c.primary_rays, c.bounce_rays, c.shadow_rays)


def _crays(c):
    return (c["rays_primary"], c["rays_bounce"], c["rays_shadow"])


def _glass(tris):
    """the bunny as normal-mapped glass: IOR 1.5, transmission 0.8"""
    t = np.array(tris, np.float32, copy=True)
    bunny = (t[:, 18:21] == 0).all(axis=1) & (t[:, 21:24] == 1).all(axis=1)
    t[bunny, 34] = 1.5
    t[bunny, 35] = 0.8
    return t


def _scene(tris, nodes, tex, uv, ids, mr, nm, hdr=None, cache=None, medium=False):
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    if medium:
        sc.set_medium(**FOG)
    sc.set_textures(tex, uv, ids)
    sc.set_material_maps(mr, nm)
    return sc


@pytest.mark.parametrize("bounces", [1, 4, 8])
@pytest.mark.parametrize("env", ["none", "map", "env_light"])
@pytest.mark.parametrize("lens", [False, True])
def test_p3_mapped_equals_the_restatement(p3, bounces, env, lens):
    tris, nodes, eye, cam, tex, uv, ids, mr, nm, hdr, cache = p3
    h, c_ = (hdr, cache) if env != "none" else (None, None)
    kw = dict(max_bounce=bounces, env_light=(env == "env_light"))
    if lens:
        kw.update(lens_radius=0.12, focus_distance=3.6)
    cfg = _cfg(eye, cam, **kw)
    sc = _scene(tris, nodes, tex, uv, ids, mr, nm, h, c_)
    try:
        got, gc = sc.render(cfg), sc.counters()
    finally:
        sc.close()
    ref, _, _, c = om.render(tris, nodes, cfg, tex, uv, ids, mr, nm, hdr=h, hdr_cache=c_)
    assert got.tobytes() == ref.tobytes(), "L-inf %.3g" % float(np.abs(got - ref).max())
    assert _rays(gc) == _crays(c)


OPTS = {
    "glass": dict(transmission=True), "glass_env": dict(transmission=True, env_light=True), "medium": dict(medium=True, env_light=True),
    "reference": dict(traverse=api.TRAVERSE_REFERENCE), "pruned": dict(traverse=api.TRAVERSE_PRUNED), "batch1": dict(frames_per_batch=1, spp=3),
    "batch3": dict(frames_per_batch=3, spp=5), "resume": dict(first_frame=2), "parts": dict(part_count=2, part_rank=1), "profile2": dict(profile=2),
}


@pytest.mark.parametrize("opt", sorted(OPTS))
def test_p3_mapped_options_equal_the_restatement(p3, opt):
    tris, nodes, eye, cam, tex, uv, ids, mr, nm, hdr, cache = p3
    kw = dict(OPTS[opt])
    if kw.get("transmission"):
        tris = _glass(tris)
    cfg = _cfg(eye, cam, **kw)
    sc = _scene(tris, nodes, tex, uv, ids, mr, nm, hdr, cache, medium=cfg.medium)
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
    ref, _, _, c = om.render(tris, nodes, full, tex, uv, ids, mr, nm, m=oracle_medium.medium(**FOG) if cfg.medium else None, hdr=hdr,
                             hdr_cache=cache)
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
def test_p3_mapped_aov_and_adaptive_equal_the_restatement(p3, opt):
    tris, nodes, eye, cam, tex, uv, ids, mr, nm, hdr, cache = p3
    kw = dict(plain=dict(env_light=True), glass=dict(transmission=True, env_light=True), medium=dict(medium=True, env_light=True))[opt]
    if opt == "glass":
        tris = _glass(tris)
    m = oracle_medium.medium(**FOG) if opt == "medium" else None
    sc = _scene(tris, nodes, tex, uv, ids, mr, nm, hdr, cache, medium=(opt == "medium"))
    try:
        cfg = _cfg(eye, cam, spp=3, **kw)
        got, gaov, _ = sc.render_aov(cfg)
        ref, _, raov, c = om.render(tris, nodes, cfg, tex, uv, ids, mr, nm, m=m, hdr=hdr, hdr_cache=cache, aov=True)
        assert got.tobytes() == ref.tobytes() and gaov.tobytes() == raov.tobytes()
        assert sc.counters().rays == c["rays"]
        none = np.full_like(nm, -1)
        _, _, uaov, _ = om.render(tris, nodes, cfg, tex, uv, ids, mr, none, m=m, hdr=hdr, hdr_cache=cache, aov=True)
        assert not np.array_equal(gaov[..., 4:7], uaov[..., 4:7])   # the feature normal is the mapped one
        acfg = _cfg(eye, cam, spp=6, **kw)
        img, spp, luma2 = sc.render_adaptive(acfg, 0.3, 2, 2)
        ac = sc.counters()
        rimg, rspp, rluma2, rc = om.render_adaptive(tris, nodes, acfg, tex, uv, ids, mr, nm, 0.3, 2, 2, m=m, hdr=hdr, hdr_cache=cache)
        assert img.tobytes() == rimg.tobytes() and luma2.tobytes() == rluma2.tobytes() and np.array_equal(spp, rspp)
        assert ac.rays == rc["rays"]
    finally:
        sc.close()


def test_s1m_mapped_windows_at_1920x1080():
    tris, nodes, eye, cam, tex, uv, ids, mr, nm = scenes.s_1m_bunny_mapped()
    sc = _scene(tris, nodes, tex, uv, ids, mr, nm)
    try:
        cfg = _cfg(eye, cam, width=1920, height=1080, spp=1, max_bounce=3)
        img = sc.render(cfg)
    finally:
        sc.close()
    for win in ((0, 0, 48, 32), (928, 528, 976, 560), (1872, 1040, 1920, 1080)):
        ref, _, _, _ = om.render(tris, nodes, cfg, tex, uv, ids, mr, nm, window=win)
        x0, y0, x1, y1 = win
        assert img[y0:y1, x0:x1].tobytes() == ref.tobytes(), "S-1M mapped window %r" % (win,)


def test_w8_mapped_equals_the_restatement(monkeypatch):
    """a small scene forced onto the 8-wide tree: the accel-order copy of the maps' ids, deferred rays and the LIST pass"""
    monkeypatch.setenv("EZRT_ACCEL", "8")
    tl = scenes._textured_list(scenes.grid_meshes(3, 2, 2), 2)
    tris, nodes = tl.build_bvh(8)
    uv, ids = tl.encode_texcoords()
    eye, cam = api.camera_orbit(30.0, 25.0, 0.62 * 3 * 1.2 + 3.0)
    tris, nodes, eye, cam, tex, uv, ids, mr, nm = scenes._with_maps((tris, nodes, eye, cam, scenes.procedural_textures(2), uv, ids))
    cfg = _cfg(eye, cam, spp=2, max_bounce=4)
    sc = _scene(tris, nodes, tex, uv, ids, mr, nm)
    try:
        got, gc = sc.render(cfg), sc.counters()
    finally:
        sc.close()
    ref, _, _, c = om.render(tris, nodes, cfg, tex, uv, ids, mr, nm)
    assert got.tobytes() == ref.tobytes() and gc.rays == c["rays"]


@pytest.mark.parametrize("opt", ["plain", "glass", "medium", "aov"])
def test_maps_invariances_on_the_device(p3, opt):
    """no maps and white metallic-roughness maps render the textured image bit for bit; constant metallic-roughness maps the textured
    image of the scene whose roughness and metallic carry the maps' values"""
    tris, nodes, eye, cam, tex, uv, ids, _, _, hdr, cache = p3
    kw = dict(plain=dict(env_light=True), glass=dict(transmission=True, env_light=True), medium=dict(medium=True, env_light=True), aov={})[opt]
    if opt == "glass":
        tris = _glass(tris)
    rng = np.random.default_rng(12)
    cols = rng.integers(0, 256, (2, 3))
    consts = [np.broadcast_to(np.append(c, 255).astype(np.uint8), (h, w, 4)).copy() for c, (h, w) in zip(cols, [(1, 1), (3, 2)])]
    white = np.full((2, 2, 4), 255, np.uint8)
    allt = tex + consts + [white]
    none = np.full(len(tris), -1, np.int32)
    mr = np.where(ids >= 0, rng.integers(0, 2, len(tris)) + len(tex), -1).astype(np.int32)
    pre = np.array(tris, np.float32, copy=True)
    on = mr >= 0
    c = cols[mr[on] - len(tex)]
    pre[on, ROUGH] = (pre[on, ROUGH] * UNORM[c[:, 1]]).astype(np.float32)
    pre[on, METAL] = (pre[on, METAL] * UNORM[c[:, 2]]).astype(np.float32)

    def run(t, maps):
        sc = api.Scene(t, nodes, hdr, cache, device=0)
        try:
            if kw.get("medium"):
                sc.set_medium(**FOG)
            sc.set_textures(allt, uv, ids)
            if maps is not None:
                sc.set_material_maps(*maps)
            cfg = _cfg(eye, cam, material_maps=maps is not None, **kw)
            out = sc.render_aov(cfg)[:2] if opt == "aov" else (sc.render(cfg),)
            return out, _rays(sc.counters())
        finally:
            sc.close()
    textured = run(tris, None)
    for maps in ((none, none), (np.where(ids >= 0, len(allt) - 1, -1), none)):
        got = run(tris, maps)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(got[0], textured[0])) and got[1] == textured[1]
    got, want = run(tris, (mr, none)), run(pre, None)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(got[0], want[0])) and got[1] == want[1]


def _hits(tris, rng, n):
    """rays toward random points of every triangle, from either side"""
    p = tris[:, :9].reshape(-1, 3, 3).astype(np.float64)
    b = rng.dirichlet((1, 1, 1), n)
    P = np.einsum("nk,nkj->nj", b, p)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    t = rng.uniform(0.5, 2.0, n)
    o = P - d * t[:, None]
    return o.astype(np.float32), d.astype(np.float32), t.astype(np.float32)


def test_sample_materials_matches_the_float64_model(p3):
    tris, nodes, eye, cam, tex, uv, ids, mr, nm, hdr, cache = p3
    n = len(tris)
    rng = np.random.default_rng(3)
    o, d, t = _hits(tris, rng, n)
    tri = np.arange(n, dtype=np.int32)
    sc = _scene(tris, nodes, tex, uv, ids, mr, nm, hdr, cache)
    try:
        got = sc.sample_materials(tri, o, d, t)
        sc.set_material_maps(None)
        plain = sc.sample_materials(tri, o, d, t)
    finally:
        sc.close()
    # without maps: the material's roughness and metallic, and surface_hit's normal
    assert np.array_equal(plain["roughness"], tris[:, ROUGH]) and np.array_equal(plain["metallic"], tris[:, METAL])
    assert np.array_equal(plain["uv"], got["uv"]) and np.array_equal(plain["base_color"], got["base_color"])
    p = tris[:, :9].reshape(-1, 3, 3)
    uv6 = np.asarray(uv, np.float32).reshape(n, 6)
    mapped = agree = total = 0
    for i in range(n):
        u, v = got["uv"][i]
        if mr[i] >= 0:
            f = unorm_sample64(tex[mr[i]], u, v)
            assert np.allclose(got["roughness"][i], tris[i, ROUGH] * f[1], rtol=1e-5, atol=3e-5)
            assert np.allclose(got["metallic"][i], tris[i, METAL] * f[2], rtol=1e-5, atol=3e-5)
        else:
            assert got["roughness"][i] == tris[i, ROUGH] and got["metallic"][i] == tris[i, METAL]
        if ids[i] >= 0:
            assert np.allclose(got["base_color"][i], tris[i, 21:24] * sample64(tex[ids[i]], u, v), rtol=1e-5, atol=3e-5)
        N = plain["normal"][i]
        if nm[i] < 0:
            assert got["normal"][i].tobytes() == N.tobytes()
            continue
        inside = np.dot(np.cross(p[i, 1].astype(np.float64) - p[i, 0], p[i, 2].astype(np.float64) - p[i, 0]), d[i]) > 0
        want = normal_map64(p[i], uv6[i], (u, v), unorm_sample64(tex[nm[i]], u, v), N, inside, -d[i])
        total += 1
        # the bunny's triangles are small: fp32 and float64 may take different sides of a fallback's border (dot(n, V) near 0)
        if want is None:
            agree += got["normal"][i].tobytes() == N.tobytes()
        elif np.allclose(got["normal"][i], want, atol=2e-3):
            agree += 1
            mapped += 1
    assert agree >= 0.99 * total and mapped > total // 2


def test_rejections_and_kept_maps(p3):
    tris, nodes, eye, cam, tex, uv, ids, mr, nm, hdr, cache = p3
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        with pytest.raises(api.EzrtError):
            sc.set_material_maps(mr, nm)   # no textures
        sc.set_textures(tex, uv, ids)
        for call in (lambda c: sc.render(c), lambda c: sc.render_aov(c), lambda c: sc.render_adaptive(c, 0.3, 2, 2)):
            with pytest.raises(api.EzrtError):
                call(_cfg(eye, cam, spp=4))   # no maps
        sc.set_material_maps(mr, nm)
        for call in (lambda c: sc.render(c), lambda c: sc.render_aov(c), lambda c: sc.render_adaptive(c, 0.3, 2, 2)):
            with pytest.raises(api.EzrtError):
                call(_cfg(eye, cam, spp=4, textures=False))   # the flag without EZRT_PARAM_TEXTURES
        cfg = _cfg(eye, cam)
        before = sc.render(cfg)
        for bad in (len(tex), -2, 70000):
            b = mr.copy()
            b[5] = bad
            with pytest.raises(api.EzrtError):
                sc.set_material_maps(b, nm)
            with pytest.raises(api.EzrtError):
                sc.set_material_maps(mr, b)
        assert sc.render(cfg).tobytes() == before.tobytes()   # the previous maps are kept
        sc.set_textures(tex, uv, ids)   # clears the maps
        with pytest.raises(api.EzrtError):
            sc.render(cfg)
        sc.set_material_maps(mr, nm)
        assert sc.render(cfg).tobytes() == before.tobytes()
        sc.set_material_maps(None)
        with pytest.raises(api.EzrtError):
            sc.render(cfg)
    finally:
        sc.close()
