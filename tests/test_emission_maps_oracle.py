"""CPU checks of the emission maps (EZRT_PARAM_EMISSION_MAPS, ezrt_math.h, DESIGN.md section 18) on their restatement
(tests/oracle_emission_maps.cpp): the C table weight against float64, the invariances against the punctual restatement bit for bit,
the light-sample pdf against the emission-hit pdf, direct light from a mapped screen against a float64 quadrature, and unbiasedness."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_binding as oracle
from tests import oracle_emission_maps as oe, oracle_lens, oracle_medium, oracle_punctual as op
from tests import transmission_scenes
from tests.test_light_sampling_laws import _block_z, _stats
from tests.texture_model import sample64

F = np.float32


def _points():
    """the 64 barycentrics (w1, w2, w3) of ez_emit_lum_eff, in its order, computed in fp32 as the C code"""
    out = []
    for i in range(8):
        for down in range(2):
            for j in range(8 - i - down):
                w1, w2 = F(3 * i + 1 + down) / F(24), F(3 * j + 1 + down) / F(24)
                out.append((w1, w2, (F(1) - w1) - w2))
    return np.array(out, np.float32)


def _lum_eff64(E, uv6, tex):
    """float64 model: the mean of lum(E * t(uv_j)) over the 64 points (uv_j in fp32 as ez_tex_uv, the filter in float64)"""
    E = np.asarray(E, np.float64)
    uv6 = np.asarray(uv6, np.float32)
    acc = 0.0
    for w1, w2, w3 in _points():
        u = (w1 * uv6[0] + w2 * uv6[2]) + w3 * uv6[4]
        v = (w1 * uv6[1] + w2 * uv6[3]) + w3 * uv6[5]
        c = E * sample64(tex, u, v)
        acc += 0.3 * c[0] + 0.6 * c[1] + 0.1 * c[2]
    return acc / 64.0


def test_point_set_is_the_subdivision_centroids():
    p = _points().astype(np.float64)
    assert p.shape == (64, 3) and len({tuple(np.round(x * 24).astype(int)) for x in p}) == 64
    np.testing.assert_allclose(p.sum(0), [64 / 3.0] * 3, rtol=1e-6)   # the centroids of an even subdivision average to the centroid


def test_table_weight_matches_float64():
    """random emitters, UVs (wrap edges, far and non-finite ones) and textures against the float64 model"""
    rng = np.random.default_rng(5)
    for k, (h, w) in enumerate([(1, 1), (3, 5), (16, 16), (7, 64)]):
        tex = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        n = 200
        E = rng.uniform(0, 20, (n, 3)).astype(np.float32)
        uv6 = rng.uniform(-3, 3, (n, 6)).astype(np.float32)
        uv6[:20] = np.round(uv6[:20])                            # on the wrap edges
        uv6[20:30] *= np.float32(1e7)                            # beyond 2^23: whole numbers
        uv6[30, 0], uv6[31, 3], uv6[32, 5] = np.nan, np.inf, -np.inf
        got = oe.lum_eff(E, uv6, tex)
        want = np.array([_lum_eff64(E[i], uv6[i], tex) for i in range(n)])
        np.testing.assert_allclose(got.astype(np.float64), want, rtol=2e-6, atol=1e-30, err_msg=str(k))


@pytest.mark.parametrize("scale", [1.0, 1e-42, 1e-38, 3e38, 1e30])
def test_white_and_constant_textures_are_exact(scale):
    """64 equal terms give that term: a white texture gives lum(E) bit for bit, a constant c gives lum(E * c), on hostile emitters
    (subnormal, near FLT_MAX) -- the pairwise midpoints keep both where 1/64 scaling or a final division would not"""
    rng = np.random.default_rng(7)
    E = (rng.uniform(0.1, 1.0, (64, 3)) * scale).astype(np.float32)
    uv6 = rng.uniform(-2, 2, (64, 6)).astype(np.float32)
    lum = lambda e: (F(0.3) * e[:, 0] + F(0.6) * e[:, 1]) + F(0.1) * e[:, 2]
    white = np.full((4, 4, 4), 255, np.uint8)
    assert oe.lum_eff(E, uv6, white).tobytes() == lum(E).tobytes()
    c = np.array([200, 31, 90], np.uint8)
    const = np.tile(np.append(c, 255).astype(np.uint8), (3, 5, 1))
    lin = oe.emit_eval(np.ones((1, 3)), np.zeros((1, 3)), np.array([[0, 0, 0, 1, 0, 0, 0, 1, 0]]), np.array([[0, 0, 1]]), np.zeros((1, 6)), const)[0]
    assert oe.lum_eff(E, uv6, const).tobytes() == lum(E * lin).tobytes()


def _scene(kind="bunny"):
    tris, nodes, eye, cam, tex, uv, ids, eid = scenes.s_p3_bunny_emission_mapped()
    return np.asarray(tris, np.float32).reshape(-1, 36), nodes, eye, cam, tex, uv, ids, eid


def _base(eye, cam, **kw):
    return dict(dict(width=32, height=24, spp=2, max_bounce=3, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam),
                     textures=True), **kw)


def test_scene_has_black_and_lit_mapped_triangles():
    tris, nodes, eye, cam, tex, uv, ids, eid = _scene()
    t, cdf, lum, hl, W = oe.table(tris, tex, uv, eid)
    mapped = np.flatnonzero(eid >= 0)
    assert len(mapped) == 320 and 0 < len(t) < 320   # some mapped triangles are black at all 64 points: not lights


@pytest.mark.parametrize("name", ["bands", "screen"])
def test_light_sample_and_hit_pdfs_agree(name):
    """for every light of the table, points on it seen from shading points around the scene: the pdf the light sample divides by and
    the pdf the emission-hit MIS assumes for the same point, through the restatement's two code paths, are equal bit for bit at equal
    distance and direction, and within the traced distance's rounding where the ray P -> Q hits that light"""
    if name == "bands":
        tris, nodes, eye, cam, tex, uv, ids, eid = _scene()
    else:
        tris, nodes, eye, cam, tex, uv, ids, eid = scenes.s_screen()
        tris = np.asarray(tris, np.float32).reshape(-1, 36)
    P = np.random.default_rng(1).uniform([-2.0, -1.3, -1.0], [2.0, 1.0, 2.0], (16, 3)).astype(np.float32)
    t, sp, hp, tp = oe.pdf_pairs(tris, nodes, tex, uv, eid, P)
    assert len(t) > 0 and (hp >= 0).all() and sp.tobytes() == hp.tobytes()
    ok = tp >= 0
    assert ok.sum() > 20 and np.abs(tp[ok].astype(np.float64) / sp[ok] - 1).max() < 1e-3


def test_screen_scene_lights_the_bunny():
    """s_screen: the camera sees the bunny, the screen and the floor, and the bunny stands between the screen and part of the floor"""
    tris, nodes, eye, cam, tex, uv, ids, eid = scenes.s_screen()
    tris = np.asarray(tris, np.float32).reshape(-1, 36)
    bunny = (tris[:, 18:21] == 0).all(1) & (tris[:, 21:24] == 1).all(1)
    floor = (eid < 0) & ~bunny
    cfg = api.RenderConfig(width=64, height=48, spp=1, max_bounce=1, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam))
    px, py = np.meshgrid(np.arange(64, dtype=np.uint32), np.arange(48, dtype=np.uint32))
    rays = oracle_lens.camera_rays(cfg, px.ravel(), py.ravel(), np.zeros(px.size, np.uint32))
    tr = oracle.trace_rays(tris, nodes, rays["o"], rays["d"])
    tri = np.where(tr["hit"] != 0, tr["triangle"], -1)
    n_bunny, n_screen, n_floor = bunny[tri[tri >= 0]].sum(), (eid[tri[tri >= 0]] >= 0).sum(), floor[tri[tri >= 0]].sum()
    # from the floor points the camera sees, toward the screen's centre
    P = tr["point"][(tri >= 0) & floor[np.maximum(tri, 0)]]
    q = tris[eid >= 0, 0:9].reshape(-1, 3)
    D = (q.min(0) + q.max(0)) / 2 - P
    sh = oracle.trace_rays(tris, nodes, (P + 1e-3 * np.array([0, 1, 0])).astype(np.float32), (D / np.linalg.norm(D, axis=1)[:, None]).astype(np.float32))
    blocked = (sh["hit"] != 0) & bunny[np.maximum(sh["triangle"], 0)]
    print("s_screen: %d bunny, %d screen, %d floor pixels; %d of %d floor points shadowed by the bunny" % (n_bunny, n_screen, n_floor, blocked.sum(), len(P)))
    assert n_bunny > 50 and n_screen > 100 and n_floor > 100 and blocked.sum() > 20


def _variants(tris, nodes, eye, cam):
    hdr = scenes.synth_hdr(128, 64)
    cache = api.hdr_cache(hdr)
    fog = oracle_medium.medium(sigma_t=0.5, albedo=(0.9, 0.8, 0.7), g=0.3, box_min=(-1.5, -1.5, -1.5), box_max=(1.5, 1.5, 1.5))
    rig = scenes.punctual_rig(tris, seed=2, power=0.5)
    return [("plain", {}, {}), ("env", dict(env_light=True), dict(hdr=hdr, hdr_cache=cache)),
            ("fog+punct", dict(env_light=True, medium=True, punctual_lights=True), dict(m=fog, lights=rig, hdr=hdr, hdr_cache=cache))]


def test_no_maps_and_white_maps_are_the_punctual_restatement():
    """all ids -1, and white emission textures, render the punctual restatement's images bit for bit and ray for ray; the white
    table is mode 4's bit for bit"""
    tris, nodes, eye, cam, tex, uv, ids, eid = _scene()
    white = np.full((2, 2, 3), 255, np.uint8)
    texw = tex[:-1] + [white]
    tw = oe.table(tris, texw, uv, eid)
    t1 = oe.table(tris, tex, uv, np.full_like(eid, -1))
    for a, b in zip(tw[:4], t1[:4]):
        assert a.tobytes() == b.tobytes()
    assert tw[4] == t1[4]
    for name, flags, kw in _variants(tris, nodes, eye, cam):
        cfg = api.RenderConfig(**_base(eye, cam, **flags))
        lights = kw.pop("lights", None)
        want, _, _, cw = op.render(tris, nodes, cfg, lights, textures=tex, texcoords=uv, texture_id=ids, **kw)
        cfg.emission_maps = True
        for e, tx in ((np.full_like(eid, -1), tex), (eid, texw)):
            got, _, _, cg = oe.render(tris, nodes, cfg, e, lights=lights, textures=tx, texcoords=uv, texture_id=ids, **kw)
            assert got.tobytes() == want.tobytes() and cg == cw, name


@pytest.mark.parametrize("variant", ["plain", "glass", "fog", "punct"])
def test_constant_maps_are_the_premultiplied_scene(variant):
    """a constant emission texture c renders the scene whose emission is E * c (premultiplied, no map), bit for bit"""
    if variant == "glass":
        tris, nodes, eye, cam = transmission_scenes.p3_glass("blob")
        tris = np.asarray(tris, np.float32).reshape(-1, 36)
        n = tris.shape[0]
        tex, uv, ids = [np.full((2, 2, 3), 128, np.uint8)], np.zeros((n, 6), np.float32), np.full(n, -1, np.int32)
        eid = np.where((tris[:, 18:21] > 0).any(1), 1, -1).astype(np.int32)
    else:
        tris, nodes, eye, cam, tex, uv, ids, eid = _scene()
        tex = tex[:-1]
    c = np.array([200, 90, 31], np.uint8)
    tex = tex + [np.tile(c, (3, 4, 1))]
    lin = sample64(np.tile(c, (3, 4, 1)), 0.3, 0.3).astype(np.float32)
    pre = tris.copy()
    on = eid >= 0
    pre[on, 18:21] = pre[on, 18:21] * lin
    flags, kw = dict(transmission=variant == "glass", env_light=True), dict(hdr=scenes.synth_hdr(64, 32))
    kw["hdr_cache"] = api.hdr_cache(kw["hdr"])
    if variant == "fog":
        flags["medium"] = True
        kw["m"] = oracle_medium.medium(sigma_t=0.5, albedo=(0.9, 0.8, 0.7), g=0.3, box_min=(-1.5, -1.5, -1.5), box_max=(1.5, 1.5, 1.5))
    lights = None
    if variant == "punct":
        flags["punctual_lights"] = True
        lights = scenes.punctual_rig(tris, seed=4, power=0.5)
    cfg = api.RenderConfig(**_base(eye, cam, **flags))
    want, _, _, cw = oe.render(pre, nodes, cfg, None, lights=lights, textures=tex, texcoords=uv, texture_id=ids, **kw)
    cfg.emission_maps = True
    got, _, _, cg = oe.render(tris, nodes, cfg, eid, lights=lights, textures=tex, texcoords=uv, texture_id=ids, **kw)
    assert got.tobytes() == want.tobytes() and cg == cw


def test_direct_light_from_a_screen_matches_float64():
    """max_bounce = 1 over a bare floor lit by the mapped screen, black environment: the mean of many pixels' direct light against a
    float64 midpoint quadrature of the mapped emission over the quad"""
    tris, nodes, eye, cam, tex, uv, ids, eid = scenes.s_screen(bunny=False)
    tris = np.asarray(tris, np.float32).reshape(-1, 36)
    W, H, n = 48, 32, 1024
    cfg = api.RenderConfig(width=W, height=H, spp=n, max_bounce=1, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam),
                           textures=True, emission_maps=True)
    img, luma2, _, c = oe.render(tris, nodes, cfg, eid, textures=tex, texcoords=uv, texture_id=ids)
    px, py = np.meshgrid(np.arange(W, dtype=np.uint32), np.arange(H, dtype=np.uint32))
    rays = oracle_lens.camera_rays(cfg, px.ravel(), py.ravel(), np.zeros(px.size, np.uint32))
    tr = oracle.trace_rays(tris, nodes, rays["o"], rays["d"])
    floor = (tr["hit"] != 0) & (eid[np.maximum(tr["triangle"], 0)] < 0)
    # the quad's emission on a 384 x 216 midpoint grid (3 points per texel) (its UVs are its local coordinates, v = 0 at the bottom)
    q = tris[eid >= 0]
    corners = q[:, 0:9].reshape(-1, 3).astype(np.float64)
    lo, hi = corners.min(0), corners.max(0)
    gu, gv = (np.arange(384) + 0.5) / 384, (np.arange(216) + 0.5) / 216
    E0 = q[0, 18:21].astype(np.float64)
    Le = np.array([[E0 * sample64(tex[0], u, v) for u in gu] for v in gv])        # [216, 384, 3]
    X, Y = np.meshgrid(lo[0] + gu * (hi[0] - lo[0]), lo[1] + gv * (hi[1] - lo[1]))
    dA = (hi[0] - lo[0]) * (hi[1] - lo[1]) / (384 * 216)
    m18 = np.asarray(tris[tr["triangle"][floor]][:, 18:36], np.float32)
    got, want = [], []
    far = tr["point"][:, 2] > lo[2] + 0.5   # away from the quad's base, where 1 / d^2 outruns the midpoint grid
    sel = np.flatnonzero(floor & far)[::5]
    for i in sel:
        P = tr["point"][i].astype(np.float64)
        D = np.stack([X - P[0], Y - P[1], np.full_like(X, lo[2]) - P[2]], -1)   # [216, 384, 3]
        d2 = (D * D).sum(-1)
        L = D / np.sqrt(d2)[..., None]
        cos_f, cos_l = L[..., 1], np.abs(L[..., 2])
        ok = cos_f > 0
        Lf = L.reshape(-1, 3).astype(np.float32)
        V = np.tile(-rays["d"][i], (Lf.shape[0], 1)).astype(np.float32)
        N = np.tile([0, 1, 0], (Lf.shape[0], 1)).astype(np.float32)
        f = oracle.eval_brdf(0, V, N, Lf, np.zeros_like(Lf), np.tile(m18[0], (Lf.shape[0], 1))).astype(np.float64).reshape(216, 384, 3)
        g = np.where(ok, cos_f * cos_l / d2, 0.0)[..., None]
        want.append((f * Le * g).sum((0, 1)) * dA)
        got.append(img.reshape(-1, 3)[i].astype(np.float64))
    got, want = np.array(got), np.array(want)
    y = lambda c: 0.3 * c[:, 0] + 0.6 * c[:, 1] + 0.1 * c[:, 2]
    var = np.maximum(luma2.reshape(-1)[sel].astype(np.float64) - y(got) ** 2, 0.0)
    se = np.sqrt(var.sum() / n) / len(sel)
    z = abs(y(got).mean() - y(want).mean()) / se
    print("screen direct light: %d pixels, mean luminance %.5g vs quadrature %.5g (z %.2f)" % (len(sel), y(got).mean(), y(want).mean(), z))
    assert len(sel) > 60 and c["rays_shadow"] > 0 and z < 4


def _z(a, b, n, W, H):
    """frame z, and the largest 16x16 and 8x8 block z over the blocks where both arms have a variance estimate: a BSDF-only arm can
    miss a small light in every sample of a block, whose variance estimate is then 0 (returned: the share of such 8x8 blocks)"""
    def blocks(bh, bw):
        z = _block_z(a, b, n, W, H, bh, bw)
        m = lambda x: x.reshape(H // bh, bh, W // bw, bw).sum((1, 3)) > 0
        ok = m(a[1]) == m(b[1])
        return float(z[ok].max()) if ok.any() else 0.0, 1.0 - ok.mean()
    z16, _ = blocks(16, 16)
    z8, skipped = blocks(8, 8)
    return float(_block_z(a, b, n, W, H, H, W).max()), z16, z8, skipped


def _mean_of(img, luma2, first, n):
    k = np.float32(first + n) / np.float32(n)
    return img.astype(np.float64) * float(k), luma2.astype(np.float64) * float(k)


def _unbiased_arms(tris, nodes, eye, cam, tex, uv, ids, eid, n=256, W=64, H=48, blind=False, mis_scale=1.0, bsdf_only=False):
    base = dict(width=W, height=H, spp=n, max_bounce=2, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam), textures=True,
                emission_maps=True)
    cfg = api.RenderConfig(**base)
    a = _stats(*oe.render(tris, nodes, cfg, eid, textures=tex, texcoords=uv, texture_id=ids, mis_scale=mis_scale)[:2])
    cfg = api.RenderConfig(**base, first_frame=n)
    lum = None
    if blind:   # texture-blind weights: lum_eff = lum(E) for every triangle
        E = tris[:, 18:21]
        lum = (F(0.3) * E[:, 0] + F(0.6) * E[:, 1]) + F(0.1) * E[:, 2]
    if bsdf_only:   # no triangle is a light (every lum_eff 0): BSDF hits only, weight 1
        lum = np.zeros(tris.shape[0], np.float32)
    img, l2, _, _ = oe.render(tris, nodes, cfg, eid, textures=tex, texcoords=uv, texture_id=ids, lum_eff=lum)
    b = _stats(*_mean_of(img, l2, n, n))
    return a, b


@pytest.mark.parametrize("scene,arm", [("screen", "blind"), ("screen", "bsdf_only"), ("bands", "blind")])
def test_mapped_table_is_unbiased(scene, arm):
    """the mapped table's render against the same render with texture-blind weights area * lum(E), and against a BSDF-only render;
    disjoint frame ranges, §10's frame / 16x16 / 8x8 z statistic.  screen: the bunny lit by the mapped quad, shadowing the floor;
    bands: the banded sphere, whose table drops the mapped triangles black at all 64 points"""
    if scene == "screen":
        tris, nodes, eye, cam, tex, uv, ids, eid = scenes.s_screen(bunny=True)
        tris = np.asarray(tris, np.float32).reshape(-1, 36)
    else:
        tris, nodes, eye, cam, tex, uv, ids, eid = _scene()
    n = 256 if arm == "blind" else 1024
    a, b = _unbiased_arms(tris, nodes, eye, cam, tex, uv, ids, eid, n=n, blind=arm == "blind", bsdf_only=arm == "bsdf_only")
    zf, z16, z8, skipped = _z(a, b, n, 64, 48)
    ratio = float(a[1].sum() / b[1].sum())   # the variance of the frame mean, mapped / other
    print("%s, emission maps vs %s: frame z %.2f, 16x16 z %.2f, 8x8 z %.2f (%.0f%% of 8x8 blocks without a variance in one arm), frame-mean "
          "variance ratio mapped / other %.3f" % (scene, arm, zf, z16, z8, 100 * skipped, ratio))
    assert zf <= 4 and z16 <= 5 and z8 <= 5.5 and skipped < 0.25, (zf, z16, z8, skipped)


def _stripe_quad():
    """a quad lit only on thin stripes that fall between the 64 points: lum_eff = 0, so it is no light, and BSDF hits render it"""
    tris, nodes, eye, cam, tex, uv, ids, eid = scenes.s_screen(bunny=False)
    img = np.zeros((64, 64, 3), np.uint8)
    img[:, 31:33] = 255      # u in [31/64, 33/64): between the subdivision's point columns on both triangles
    return np.asarray(tris, np.float32).reshape(-1, 36), nodes, eye, cam, [img], uv, ids, eid


def test_black_at_the_points_but_lit_between_is_unbiased():
    tris, nodes, eye, cam, tex, uv, ids, eid = _stripe_quad()
    t, cdf, lum, hl, W = oe.table(tris, tex, uv, eid)
    assert len(t) == 0   # both triangles are black at all 64 points
    n = 1024
    a, b = _unbiased_arms(tris, nodes, eye, cam, tex, uv, ids, eid, n=n, blind=True)
    zf, z16, z8, skipped = _z(a, b, n, 64, 48)
    print("stripes between the points: %d lights, frame z %.2f, 16x16 z %.2f, 8x8 z %.2f (%.0f%% of 8x8 blocks skipped), mean luminance %.4g" %
          (len(t), zf, z16, z8, 100 * skipped, a[0].mean()))
    assert a[0].mean() > 0 and zf <= 4 and z16 <= 5 and z8 <= 5.5 and skipped < 0.5


def test_mis_side_mutation_is_detected():
    """lum_eff scaled by 1.03 in the emission hits' MIS weights only (the restatement's test-only mis_scale) biases the estimator: a
    frame of the floor lit by the screen at 1 bounce, against the unmutated render on disjoint frames, fails the frame z test, while a
    third, unmutated range passes it"""
    tris, nodes, _, _, tex, uv, ids, eid = scenes.s_screen(bunny=False)
    tris = np.asarray(tris, np.float32).reshape(-1, 36)
    eye, cam = api.camera_look_at((0.0, 0.2, 2.2), (0.0, -1.4, -0.4), (0, 1, 0), 50.0, 4 / 3)
    W, H, n = 64, 48, 8192

    def arm(first, mis_scale):
        cfg = api.RenderConfig(width=W, height=H, spp=n, max_bounce=1, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam),
                               textures=True, emission_maps=True, first_frame=first)
        img, l2, _, _ = oe.render(tris, nodes, cfg, eid, textures=tex, texcoords=uv, texture_id=ids, mis_scale=mis_scale)
        return _stats(*_mean_of(img, l2, first, n)) if first else _stats(img, l2)

    mutated, plain, again = arm(0, 1.03), arm(n, 1.0), arm(2 * n, 1.0)
    z_mut = float(_block_z(mutated, plain, n, W, H, H, W).max())
    z_null = float(_block_z(again, plain, n, W, H, H, W).max())
    print("MIS-side mutation x1.03: frame z %.2f (unmutated: %.2f), frame mean moved by %.2e" % (z_mut, z_null, mutated[0].mean() / plain[0].mean() - 1))
    assert z_mut > 4 and z_null <= 4


def test_invalid_renders_are_rejected():
    tris, nodes, eye, cam, tex, uv, ids, eid = _scene()
    cfg = api.RenderConfig(**_base(eye, cam, textures=False, emission_maps=True))
    with pytest.raises(ValueError):
        oe.render(tris, nodes, cfg, eid, textures=tex, texcoords=uv, texture_id=ids)
    cfg = api.RenderConfig(**_base(eye, cam, emission_maps=True))
    with pytest.raises(ValueError):
        oe.render(tris, nodes, cfg, None, textures=tex, texcoords=uv, texture_id=ids)
    bad = eid.copy()
    bad[3] = len(tex)
    with pytest.raises(ValueError):
        oe.table(tris, tex, uv, bad)
