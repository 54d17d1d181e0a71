"""GPU renders with base-colour textures (EZRT_PARAM_TEXTURES, DESIGN.md section 15).

The textured base colour is checked per hit against a float64 numpy model of the definition (Scene.sample_textures), and whole
renders by two exact invariances: 1x1 white textures render the unflagged image bit for bit, and constant textures render the image
of the untextured scene whose base colours are premultiplied by the textures' decoded colours, ray for ray, under every option."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_medium, oracle_textures
from tests.texture_model import LUT, bary64, constant_textures, sample64

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def p3():
    tris, nodes, eye, cam, tex, uv, ids = scenes.s_p3_bunny_textured()
    hdr = scenes.synth_hdr(64, 32)
    return tris, nodes, eye, cam, tex, uv, ids, hdr, api.hdr_cache(hdr)


def _cfg(eye, cam, **kw):
    base = dict(width=48, height=32, spp=2, max_bounce=4, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam), textures=True)
    base.update(kw)
    return api.RenderConfig(**base)


def _white(n):
    return [np.full((1, 1, 4), 255, np.uint8)], np.zeros((n, 3, 2), np.float32), np.zeros(n, np.int32)


def _premultiplied(tris, ids, colours):
    """the scene whose triangle k has base colour baseColor_k * LUT(colour of its texture), in fp32 as the kernels multiply"""
    t = np.array(tris, np.float32, copy=True)
    m = ids >= 0
    lin = LUT[np.asarray(colours)[ids[m]]]
    t[m, 21:24] = (t[m, 21:24].astype(np.float32) * lin.astype(np.float32)).astype(np.float32)
    return t


def _render(sc, cfg, kind):
    if kind == "aov":
        img, aov, _ = sc.render_aov(cfg)
        return (img, aov), sc.counters()
    if kind == "adaptive":
        img, spp, luma2 = sc.render_adaptive(cfg, 0.3, 2, 2)
        return (img, spp, luma2), sc.counters()
    return (sc.render(cfg),), sc.counters()


def _same(a, b):
    return all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def _rays(c):
    return (c.primary_rays, c.bounce_rays, c.shadow_rays)


OPTS = {
    "plain": {}, "env_light": dict(env_light=True), "lens": dict(lens_radius=0.12, focus_distance=3.6),
    "env_lens": dict(env_light=True, lens_radius=0.12, focus_distance=3.6), "b1": dict(max_bounce=1), "b8": dict(max_bounce=8),
    "transmission": dict(transmission=True), "medium": dict(medium=True, env_light=True), "reference": dict(traverse=api.TRAVERSE_REFERENCE),
    "pruned": dict(traverse=api.TRAVERSE_PRUNED), "batch1": dict(frames_per_batch=1, spp=3), "batch3": dict(frames_per_batch=3, spp=5),
    "resume": dict(first_frame=2), "profile2": dict(profile=2), "parts": dict(part_count=2, part_rank=1),
}
FOG = dict(sigma_t=0.6, albedo=(0.9, 0.8, 0.7), g=0.4, box_min=(-1.2, -1.0, -1.2), box_max=(1.2, 1.4, 1.2))


def _transmissive(tris):
    t = np.array(tris, np.float32, copy=True)
    bunny = (t[:, 18:21] == 0).all(axis=1) & (t[:, 21:24] == 1).all(axis=1)
    # Material.as_array: ... IOR and transmission are the last two of the 18 floats
    t[bunny, 34] = 1.5
    t[bunny, 35] = 0.8
    return t


CASES = [(o, "render") for o in sorted(OPTS)] + [(o, k) for k in ("aov", "adaptive") for o in ("plain", "env_lens", "transmission", "medium", "b8")]


@pytest.mark.parametrize("opt,kind", CASES)
def test_white_and_constant_textures_are_exact(p3, opt, kind):
    tris, nodes, eye, cam, _, _, _, hdr, cache = p3
    kw = dict(OPTS[opt])
    if kind == "adaptive":
        kw.update(spp=6, first_frame=0, frames_per_batch=0, profile=0)
    if opt == "transmission":
        tris = _transmissive(tris)
    rng = np.random.default_rng(5)
    ids = rng.integers(-1, 4, len(tris)).astype(np.int32)
    tex, colours = constant_textures(rng, [(1, 1), (3, 5), (7, 2), (4, 4)])
    uv = rng.uniform(-3, 3, (len(tris), 3, 2)).astype(np.float32)
    pre = _premultiplied(tris, ids, colours)
    out = {}
    for name, t in (("tex", tris), ("pre", pre)):
        sc = api.Scene(t, nodes, hdr, cache, device=0)
        try:
            if kw.get("medium"):
                sc.set_medium(**FOG)
            if name == "tex":
                sc.set_textures(*_white(len(t)))
                white = _render(sc, _cfg(eye, cam, **kw), kind)
                plain = _render(sc, _cfg(eye, cam, textures=False, **kw), kind)
                assert _same(white[0], plain[0]), "white textures differ from the unflagged render"
                assert _rays(white[1]) == _rays(plain[1])
                sc.set_textures(tex, uv, ids)
                out[name] = _render(sc, _cfg(eye, cam, **kw), kind)
            else:
                out[name] = _render(sc, _cfg(eye, cam, textures=False, **kw), kind)
        finally:
            sc.close()
    assert np.isfinite(out["tex"][0][0]).all()
    assert _same(out["tex"][0], out["pre"][0]), "L-inf %.3g" % float(np.abs(out["tex"][0][0] - out["pre"][0][0]).max())
    assert _rays(out["tex"][1]) == _rays(out["pre"][1])


@pytest.mark.parametrize("bounces", [1, 4, 8])
@pytest.mark.parametrize("env", ["none", "map", "env_light"])
@pytest.mark.parametrize("lens", [False, True])
def test_p3_textured_equals_the_restatement(p3, bounces, env, lens):
    tris, nodes, eye, cam, tex, uv, ids, hdr, cache = p3
    h, c_ = (hdr, cache) if env != "none" else (None, None)
    kw = dict(max_bounce=bounces, env_light=(env == "env_light"))
    if lens:
        kw.update(lens_radius=0.12, focus_distance=3.6)
    cfg = _cfg(eye, cam, **kw)
    sc = api.Scene(tris, nodes, h, c_, device=0)
    try:
        sc.set_textures(tex, uv, ids)
        got, gc = sc.render(cfg), sc.counters()
    finally:
        sc.close()
    ref, _, _, c = oracle_textures.render(tris, nodes, cfg, tex, uv, ids, hdr=h, hdr_cache=c_)
    assert got.tobytes() == ref.tobytes(), "L-inf %.3g" % float(np.abs(got - ref).max())
    assert _rays(gc) == (c["rays_primary"], c["rays_bounce"], c["rays_shadow"])


@pytest.mark.parametrize("opt", ["medium", "reference", "pruned", "batch1", "batch3", "parts", "profile2"])
def test_p3_textured_options_equal_the_restatement(p3, opt):
    tris, nodes, eye, cam, tex, uv, ids, hdr, cache = p3
    kw = dict(OPTS[opt])
    cfg = _cfg(eye, cam, **kw)
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        if cfg.medium:
            sc.set_medium(**FOG)
        sc.set_textures(tex, uv, ids)
        got, gc = sc.render(cfg), sc.counters()
    finally:
        sc.close()
    full = _cfg(eye, cam, **{k: v for k, v in kw.items() if k not in ("part_count", "part_rank")})
    ref, _, _, c = oracle_textures.render(tris, nodes, full, tex, uv, ids, m=oracle_medium.medium(**FOG) if cfg.medium else None, hdr=hdr,
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
    assert _rays(gc) == (c["rays_primary"], c["rays_bounce"], c["rays_shadow"])


def test_p3_textured_aov_and_adaptive_equal_the_restatement(p3):
    tris, nodes, eye, cam, tex, uv, ids, hdr, cache = p3
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        sc.set_textures(tex, uv, ids)
        cfg = _cfg(eye, cam, env_light=True, spp=3)
        got, gaov, _ = sc.render_aov(cfg)
        ref, _, raov, c = oracle_textures.render(tris, nodes, cfg, tex, uv, ids, hdr=hdr, hdr_cache=cache, aov=True)
        assert got.tobytes() == ref.tobytes() and gaov.tobytes() == raov.tobytes()
        assert sc.counters().rays == c["rays"]
        _, _, uaov, _ = oracle_textures.render(tris, nodes, cfg, tex, uv, np.full_like(ids, -1), hdr=hdr, hdr_cache=cache, aov=True)
        assert not np.array_equal(gaov[..., :3], uaov[..., :3])   # the albedo is textured
        acfg = _cfg(eye, cam, env_light=True, spp=6)
        img, spp, luma2 = sc.render_adaptive(acfg, 0.3, 2, 2)
        ac = sc.counters()
        rimg, rspp, rluma2, rc = oracle_textures.render_adaptive(tris, nodes, acfg, tex, uv, ids, 0.3, 2, 2, hdr=hdr, hdr_cache=cache)
        assert img.tobytes() == rimg.tobytes() and luma2.tobytes() == rluma2.tobytes() and np.array_equal(spp, rspp)
        assert ac.rays == rc["rays"]
    finally:
        sc.close()


def test_s1m_textured_windows_at_1920x1080():
    tris, nodes, eye, cam, tex, uv, ids = scenes.s_1m_bunny_textured()
    sc = api.Scene(tris, nodes)
    try:
        sc.set_textures(tex, uv, ids)
        cfg = _cfg(eye, cam, width=1920, height=1080, spp=1, max_bounce=3)
        img = sc.render(cfg)
    finally:
        sc.close()
    for win in ((0, 0, 48, 32), (928, 528, 976, 560), (1872, 1040, 1920, 1080)):
        ref, _, _, _ = oracle_textures.render(tris, nodes, cfg, tex, uv, ids, window=win)
        x0, y0, x1, y1 = win
        assert img[y0:y1, x0:x1].tobytes() == ref.tobytes(), "S-1M textured window %r" % (win,)


def test_w8_textured_equals_the_restatement(monkeypatch):
    """a small scene forced onto the 8-wide tree: accel-order texcoord records, deferred rays and the LIST pass"""
    monkeypatch.setenv("EZRT_ACCEL", "8")
    tl = scenes._textured_list(scenes.grid_meshes(3, 2, 2), 2)
    tris, nodes = tl.build_bvh(8)
    uv, ids = tl.encode_texcoords()
    tex = scenes.procedural_textures(2)
    eye, cam = api.camera_orbit(30.0, 25.0, 0.62 * 3 * 1.2 + 3.0)
    cfg = _cfg(eye, cam, spp=2, max_bounce=4)
    sc = api.Scene(tris, nodes)
    try:
        sc.set_textures(tex, uv, ids)
        got, gc = sc.render(cfg), sc.counters()
    finally:
        sc.close()
    ref, _, _, c = oracle_textures.render(tris, nodes, cfg, tex, uv, ids)
    assert got.tobytes() == ref.tobytes() and gc.rays == c["rays"]


def test_constant_textures_on_the_8wide_tree(monkeypatch):
    """a small scene forced onto the 8-wide tree (accel-order texcoord records, deferred rays) and the 1M-triangle scene"""
    monkeypatch.setenv("EZRT_ACCEL", "8")
    for fn, w, h in ((lambda: scenes.s_grid(3, 2, 2), 48, 32), (scenes.s_1m_bunny, 96, 54)):
        tris, nodes, eye, cam = fn()
        rng = np.random.default_rng(9)
        ids = rng.integers(-1, 3, len(tris)).astype(np.int32)
        tex, colours = constant_textures(rng, [(2, 3), (1, 1), (5, 5)])
        uv = rng.uniform(-2, 2, (len(tris), 3, 2)).astype(np.float32)
        imgs = []
        for t, on in ((tris, True), (_premultiplied(tris, ids, colours), False)):
            sc = api.Scene(t, nodes)
            try:
                if on:
                    sc.set_textures(tex, uv, ids)
                imgs.append((sc.render(_cfg(eye, cam, width=w, height=h, textures=on)), _rays(sc.counters())))
            finally:
                sc.close()
        assert imgs[0][0].tobytes() == imgs[1][0].tobytes() and imgs[0][1] == imgs[1][1]


def test_sample_textures_matches_the_float64_model(p3):
    tris, nodes, eye, cam, _, _, _, hdr, cache = p3
    rng = np.random.default_rng(3)
    n = len(tris)
    sizes = [(1, 1), (1, 7), (5, 1), (3, 5), (17, 9), (64, 64)]
    tex = [rng.integers(0, 256, (h, w, 4)).astype(np.uint8) for h, w in sizes]
    ids = rng.integers(0, len(tex), n).astype(np.int32)
    ids[::17] = -1
    uv = rng.uniform(-4, 4, (n, 3, 2)).astype(np.float32)
    special = np.array([0.0, 1.0, -1e-9, 1 - 1e-8, -0.5, 8388608.0, -8388609.0, 3e7, 0.999999, 1e-30], np.float32)
    uv[: len(special) * 3, 0, 0] = np.repeat(special, 3)
    uv[: len(special) * 3, 0, 1] = np.tile(special[::-1], 3)
    uv[200, 0] = (np.inf, 0.5)
    uv[201, 0] = (0.5, np.nan)
    p = tris[:, :9].reshape(-1, 3, 3)
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        sc.set_textures(tex, uv, ids)
        tri = np.arange(n, dtype=np.int32)
        # at vertex 1 (weights within rounding of (1, 0, 0)): the filter near the chosen UVs -- wrap edges, huge and negative ones
        got_uv, got = sc.sample_textures(tri, p[:, 0])
        # inside: random barycentric points, including the floor (degenerate xy projection)
        b = rng.dirichlet((1, 1, 1), n)
        pin = np.einsum("nk,nkj->nj", b, p.astype(np.float64)).astype(np.float32)
        got_uv2, got2 = sc.sample_textures(tri, pin)
    finally:
        sc.close()
    base = tris[:, 21:24].astype(np.float64)
    finite = np.isfinite(uv[:, 0]).all(axis=1)
    assert np.allclose(got_uv[finite], uv[finite, 0], rtol=1e-5, atol=1e-5)
    want = np.array([base[i] * (sample64(tex[ids[i]], *got_uv[i]) if ids[i] >= 0 else 1.0) for i in range(n)])
    # fp32 texel coordinates: the weights are off by up to ~W ulp(1) against float64, hence the absolute term
    assert np.allclose(got, want, rtol=1e-5, atol=3e-5)
    assert np.array_equal(got[~finite], tris[~finite, 21:24])   # a non-finite UV: white
    w = bary64(pin, p, tris)
    uv64 = np.einsum("nk,nkj->nj", w, uv.astype(np.float64))
    ok = np.isfinite(uv64).all(axis=1)
    # relative to the triangle's largest |uv| (the chosen UVs reach 3e7); points rounded to fp32 lie slightly off thin triangles' planes
    err = np.abs(got_uv2[ok] - uv64[ok]).max(axis=1) / (1.0 + np.abs(uv[ok]).max(axis=(1, 2)))
    assert np.quantile(err, 0.99) < 1e-5 and err.max() < 1e-3
    want2 = np.array([base[i] * (sample64(tex[ids[i]], *got_uv2[i]) if ids[i] >= 0 else 1.0) for i in range(n)])
    assert np.allclose(got2, want2, rtol=1e-5, atol=3e-5)
    floor = np.abs(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])[:, 1]) > 0
    floor &= (np.abs(p[:, :, 1] - p[:, :1, 1]) < 1e-6).all(axis=1)
    assert floor.sum() >= 2 and np.ptp(got_uv2[floor & ok], axis=0).min() > 0   # the floor's UVs do not collapse


def test_textured_render_is_deterministic_and_differs(p3):
    tris, nodes, eye, cam, tex, uv, ids, hdr, cache = p3
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        sc.set_textures(tex, uv, ids)
        a = sc.render(_cfg(eye, cam, env_light=True))
        b = sc.render(_cfg(eye, cam, env_light=True))
        plain = sc.render(_cfg(eye, cam, env_light=True, textures=False))
        sc.set_textures(None)
        with pytest.raises(api.EzrtError):
            sc.render(_cfg(eye, cam))
    finally:
        sc.close()
    assert a.tobytes() == b.tobytes() and np.isfinite(a).all()
    assert not np.array_equal(a, plain)


def test_invalid_textures_and_renders_rejected(p3):
    tris, nodes, eye, cam, tex, uv, ids, hdr, cache = p3
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        for call in (lambda c: sc.render(c), lambda c: sc.render_aov(c), lambda c: sc.render_adaptive(c, 0.3, 2, 2)):
            with pytest.raises(api.EzrtError):
                call(_cfg(eye, cam, spp=4))   # no textures set
        sc.set_textures(tex, uv, ids)
        for mode in (0, 1, 2, 3):
            for call in (lambda c: sc.render(c), lambda c: sc.render_aov(c), lambda c: sc.render_adaptive(c, 0.3, 2, 2)):
                with pytest.raises(api.EzrtError):
                    call(_cfg(eye, cam, spp=4, mode=mode))
        bad_ids = ids.copy()
        bad_ids[5] = len(tex)
        for args in ((tex, uv, bad_ids), (tex, uv, np.full(len(tris), -2, np.int32)), ([np.zeros((16385, 1, 4), np.uint8)], uv, ids * 0)):
            with pytest.raises(api.EzrtError):
                sc.set_textures(*args)
        sc.render(_cfg(eye, cam))   # the previous textures are kept
    finally:
        sc.close()
