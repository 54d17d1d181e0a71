"""The punctual lights (EZRT_PARAM_PUNCTUAL_LIGHTS, DESIGN.md section 17) on the CPU: the table against float64 numpy, the category
split's exact law over all 2^32 rand01 hashes, the restatement's invariances against the restatements of mode 4 and its options,
direct light against a float64 evaluation, and the split's unbiasedness against two independent renders."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_binding as oracle
from tests import oracle_lens, oracle_material_maps, oracle_medium, oracle_punctual as op, oracle_transmission
from tests import transmission_scenes
from tests.test_light_sampling_laws import TWO32, _block_z, _count_below, _metrics, _stats


def _lum(c):
    c = np.asarray(c, np.float32)
    return float((np.float32(0.3) * c[0] + np.float32(0.6) * c[1]) + np.float32(0.1) * c[2])


def _box_r(tris):
    v = np.asarray(tris, np.float32).reshape(-1, 36)[:, :9].reshape(-1, 3).astype(np.float64)
    return 0.5 * float(np.linalg.norm(v.max(axis=0) - v.min(axis=0)))


def _weight64(l, r):
    I, lum = float(np.float32(l.intensity)), _lum(list(l.color))
    if l.type == api.PUNCTUAL_POINT:
        return 4 * np.pi * I * lum
    if l.type == api.PUNCTUAL_SPOT:
        ci, co = np.cos(float(np.float32(l.inner_cone))), np.cos(float(np.float32(l.outer_cone)))
        return 2 * np.pi * I * lum * (1 - ci + (ci - co) / 3)
    return np.pi * r * r * I * lum


def _rig_lights():
    return [api.point_light((1, 2, 3), (0.2, 0.5, 0.9), 3.0), api.spot_light((0, 3, 0), (0, -1, 0.2), (1, 1, 1), 5.0, 0.1, 0.7),
            api.directional_light((0.3, -1, 0.1), (1.0, 0.9, 0.8), 2.0), api.point_light((0, 0, 0), (1, 1, 1), 0.0),
            api.spot_light((1, 1, 1), (1, 0, 0), (0, 0, 0), 9.0, 0.0, 0.2), api.point_light((-1, 2, 0), (0.5, 0.5, 0.5), 1e-3)]


def test_table_matches_float64():
    tris = scenes.s_p3_bunny()[0]
    lights = _rig_lights()
    idx, cdf, q, rec, W = op.table(tris, lights)
    r = _box_r(tris)
    w = np.array([_weight64(l, r) for l in lights])
    keep = np.flatnonzero(w > 0)
    assert idx.tolist() == keep.tolist() == [0, 1, 2, 5]    # zero intensity and black lights are dropped
    assert W == pytest.approx(w[keep].sum(), rel=1e-15)
    S = np.cumsum(w[keep])
    np.testing.assert_array_equal(cdf[:-1], (S / W).astype(np.float32)[:-1])
    assert cdf[-1] == 1.0
    np.testing.assert_array_equal(q, (w[keep] / W).astype(np.float32))
    # the records: type, unit direction (float64-normalised), cos of the cones, intensity * color
    spot = lights[1]
    d = np.array(list(spot.direction), np.float64)
    np.testing.assert_array_equal(rec[1, 4:7], (d / np.linalg.norm(d)).astype(np.float32))
    assert rec[1, 3] == 1.0 and rec[2, 3] == 2.0 and rec[0, 3] == 0.0
    assert rec[1, 11] == np.float32(np.cos(np.float64(np.float32(0.1)))) and rec[1, 7] == np.float32(np.cos(np.float64(np.float32(0.7))))
    np.testing.assert_array_equal(rec[0, 8:11], np.float32(3.0) * np.array([0.2, 0.5, 0.9], np.float32))
    np.testing.assert_array_equal(rec[:, 12], q)


def test_spot_weight_is_the_falloffs_integral():
    """2 pi I lum (1 - cos_i + (cos_i - cos_o) / 3) is the solid-angle integral of glTF's falloff when it is linear in cos over
    [cos_o, cos_i] and squared: checked against a numerical integral of ez_spot_falloff's definition"""
    for inner, outer in ((0.0, 0.3), (0.2, 0.9), (0.5, 1.5707)):
        ci, co = np.cos(inner), np.cos(outer)
        c = np.linspace(-1, 1, 2_000_001)
        a = np.clip((c - co) / max(1e-3, ci - co), 0, 1) ** 2
        integral = 2 * np.pi * np.trapezoid(a, c)
        assert integral == pytest.approx(2 * np.pi * (1 - ci + (ci - co) / 3), rel=1e-6), (inner, outer)


def test_directional_weight_uses_the_vertex_box():
    tris = np.asarray(scenes.s_p3_bunny()[0], np.float32).reshape(-1, 36).copy()
    sun = [api.directional_light((0, -1, 0), (1, 1, 1), 1.0), api.point_light((0, 5, 0), (1, 1, 1), 1.0)]
    _, _, _, _, W = op.table(tris, sun)
    r = _box_r(tris)
    assert W == pytest.approx(np.pi * r * r * _lum((1, 1, 1)) + 4 * np.pi * _lum((1, 1, 1)), rel=1e-14)
    # the order of the triangles does not change r
    _, _, _, _, W2 = op.table(tris[::-1].copy(), sun)
    assert W2 == W


BAD_LIGHTS = [
    ("unknown type", lambda: api._punctual(3, color=(1, 1, 1))),
    ("non-finite position", lambda: api.point_light((np.nan, 0, 0))),
    ("non-finite intensity", lambda: api.point_light((0, 0, 0), intensity=np.inf)),
    ("zero spot direction", lambda: api.spot_light((0, 0, 0), (0, 0, 0))),
    ("zero sun direction", lambda: api.directional_light((0, 0, 0))),
    ("negative colour", lambda: api.point_light((0, 0, 0), color=(1, -0.1, 1))),
    ("negative intensity", lambda: api.point_light((0, 0, 0), intensity=-1.0)),
    ("inner == outer", lambda: api.spot_light((0, 0, 0), (0, -1, 0), inner_cone=0.5, outer_cone=0.5)),
    ("negative inner", lambda: api.spot_light((0, 0, 0), (0, -1, 0), inner_cone=-0.1, outer_cone=0.5)),
    ("outer beyond pi/2", lambda: api.spot_light((0, 0, 0), (0, -1, 0), inner_cone=0.1, outer_cone=1.571)),
    ("reserved", lambda: (lambda l: (setattr(l, "reserved", 1), l)[1])(api.point_light((0, 0, 0)))),
]


@pytest.mark.parametrize("name", [b[0] for b in BAD_LIGHTS])
def test_invalid_lights_are_rejected(name):
    tris = scenes.s_p3_bunny()[0]
    bad = dict(BAD_LIGHTS)[name]()
    with pytest.raises(ValueError) as e:
        op.table(tris, [api.point_light((0, 1, 0)), bad])
    assert e.value.args[1] == 1
    # pi/2 rounded to fp32 is accepted
    op.table(tris, [api.spot_light((0, 0, 0), (0, -1, 0), inner_cone=0.0, outer_cone=float(np.float32(np.pi / 2)))])


def test_category_split_law():
    """r_sel < 0.5 (r_p = 2 r_sel) holds (2^31 - 64) / 2^32 of the hashes at P_p = 1/2; inside it the selection law is within 1e-4 of
    q in total variation for weights spread over twelve orders of magnitude; the lights fp32's cdf cannot reach (equal entries behind
    far brighter ones) carry less than 1e-5 of q, as for the triangle lights (test_light_sampling_laws.py)"""
    half = int(_count_below(2.0 ** 31))
    assert half == (1 << 31) - 64
    rng = np.random.default_rng(5)
    lights = [api.point_light((0, 1, 0), (1, 1, 1), float(10.0 ** e)) for e in rng.uniform(-6, 6, 64)]
    _, cdf, q, _, _ = op.table(scenes.s_p3_bunny()[0], lights)
    for p_p, top in ((0.5, 2.0 ** 31), (1.0, 2.0 ** 32)):
        scale = 2.0 if p_p == 0.5 else 1.0
        base = int(_count_below(top))
        # light j iff r_p = r_sel * scale < cdf_j, exact as the scaling is exact; rand01 = 1.0 (P_p = 1) selects the last light
        n_below = _count_below(cdf[:-1].astype(np.float64) / scale * TWO32)
        edges = np.concatenate([[0], n_below, [base if p_p == 0.5 else TWO32]])
        P = np.diff(edges) / float(edges[-1])
        m = _metrics(P, q)
        print("punctual split P_p = %.1f: branch %d / 2^32 hashes, TV %.3g, max |P/q - 1| %.3g, unreachable %d" %
              (p_p, edges[-1], m["tv"], m["max_ratio"], m["zero_n"]))
        assert m["tv"] <= 1e-4 and m["zero_mass"] < 1e-5, m


def _zero_rig(tris):
    return [api.point_light((0, 1, 0), (1, 1, 1), 0.0), api.spot_light((0, 2, 0), (0, -1, 0), (0, 0, 0), 4.0, 0.1, 0.5)]


def test_zero_lights_are_mode4():
    """a flagged render whose lights all weigh 0 is the mode-4 restatements' render, bit for bit and ray for ray"""
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    hdr = scenes.synth_hdr(128, 64)
    cache = api.hdr_cache(hdr)
    zero = _zero_rig(tris)
    base = dict(width=32, height=24, spp=2, max_bounce=3, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam))
    for env in (False, True):
        cfg = api.RenderConfig(**base, env_light=env)
        want, _, _, cw = oracle_lens.render(tris, nodes, cfg, hdr=hdr, hdr_cache=cache)
        cfg.punctual_lights = True
        got, _, _, cg = op.render(tris, nodes, cfg, zero, hdr=hdr, hdr_cache=cache)
        assert got.tobytes() == want.tobytes() and cg == cw, env
    fog = oracle_medium.medium(sigma_t=0.6, albedo=(0.9, 0.8, 0.7), g=0.4, box_min=(-1.5, -1.5, -1.5), box_max=(1.5, 1.5, 1.5))
    cfg = api.RenderConfig(**base, env_light=True, medium=True)
    want, _, _, cw = oracle_medium.render(tris, nodes, cfg, fog, hdr=hdr, hdr_cache=cache)
    cfg.punctual_lights = True
    got, _, _, cg = op.render(tris, nodes, cfg, zero, m=fog, hdr=hdr, hdr_cache=cache)
    assert got.tobytes() == want.tobytes() and cg == cw
    gtris, gnodes, geye, gcam = transmission_scenes.p3_glass("blob")
    cfg = api.RenderConfig(**dict(base, eye=tuple(geye), camera_rotate=tuple(gcam)), env_light=True, transmission=True)
    want, _, cw = oracle_transmission.oracle_render_transmission(gtris, gnodes, cfg, hdr=hdr, hdr_cache=cache)
    cfg.punctual_lights = True
    got, _, _, cg = op.render(gtris, gnodes, cfg, _zero_rig(gtris), hdr=hdr, hdr_cache=cache)
    assert got.tobytes() == want.tobytes() and cg["rays"] == cw["rays"]
    mtris, mnodes, meye, mcam, tex, uv, ids, mr, nm = scenes.s_p3_bunny_mapped()
    cfg = api.RenderConfig(**dict(base, eye=tuple(meye), camera_rotate=tuple(mcam)), env_light=True, textures=True, material_maps=True)
    want, _, _, cw = oracle_material_maps.render(mtris, mnodes, cfg, tex, uv, ids, mr, nm, hdr=hdr, hdr_cache=cache)
    cfg.punctual_lights = True
    got, _, _, cg = op.render(mtris, mnodes, cfg, _zero_rig(mtris), textures=tex, texcoords=uv, texture_id=ids, metal_rough_id=mr, normal_id=nm,
                              hdr=hdr, hdr_cache=cache)
    assert got.tobytes() == want.tobytes() and cg == cw


def _floor_scene():
    """a 6 x 6 floor at y = 0, grey and rough, seen from above at a slant: no emitter"""
    tl = api.TriangleList()
    quad = "v -1 0 -1\nv 1 0 -1\nv 1 0 1\nv -1 0 1\nf 1 3 2\nf 1 4 3\n"
    mat = api.Material(baseColor=(0.6, 0.5, 0.4), roughness=0.7)
    tl.read_obj_text(quad, mat, api.transform_matrix((0, 0, 0), (0, 0, 0), (3, 1, 3)), False)
    tris, nodes = tl.build_bvh(8)
    eye, cam = api.camera_orbit(0.0, 40.0, 2.5)
    return np.asarray(tris, np.float32).reshape(-1, 36), nodes, eye, cam, mat


@pytest.mark.parametrize("kind", ["point", "spot"])
def test_direct_light_matches_float64(kind):
    """max_bounce = 1 over a floor, black environment, one light: every pixel that sees the floor is f cos I a / d^2 at its hit point
    (the BSDF sample reaches nothing), and the spot's pixels outside its outer cone are exactly 0"""
    tris, nodes, eye, cam, mat = _floor_scene()
    pos = np.array([0.3, 1.5, 0.2])
    light = api.point_light(pos, (1.0, 0.8, 0.6), 2.0) if kind == "point" else \
        api.spot_light(pos, (0.2, -1, 0.1), (1.0, 0.8, 0.6), 2.0, inner_cone=0.2, outer_cone=0.5)
    cfg = api.RenderConfig(width=48, height=32, spp=1, max_bounce=1, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam),
                           punctual_lights=True)
    img, _, _, c = op.render(tris, nodes, cfg, [light])
    px, py = np.meshgrid(np.arange(cfg.width, dtype=np.uint32), np.arange(cfg.height, dtype=np.uint32))
    rays = oracle_lens.camera_rays(cfg, px.ravel(), py.ravel(), np.zeros(px.size, np.uint32))
    tr = oracle.trace_rays(tris, nodes, rays["o"], rays["d"])
    d = rays["d"].astype(np.float64)
    P = tr["point"].astype(np.float64)
    on = tr["hit"] != 0
    D = pos[None] - P
    d2 = (D * D).sum(1)
    L = D / np.sqrt(d2)[:, None]
    cos = L[:, 1]
    a = np.ones(len(P))
    if kind == "spot":
        sd = np.array([0.2, -1, 0.1]) / np.linalg.norm([0.2, -1, 0.1])
        ci, co = np.cos(0.2), np.cos(0.5)
        a = np.clip(((-L) @ sd - co) / (ci - co), 0, 1) ** 2
    m18 = np.tile(np.asarray(mat.as_array(), np.float32)[:18], (len(P), 1))
    V = -d
    N = np.tile([0.0, 1.0, 0.0], (len(P), 1))
    f = oracle.eval_brdf(0, V.astype(np.float32), N.astype(np.float32), L.astype(np.float32), np.zeros((len(P), 3), np.float32), m18)
    want = f.astype(np.float64) * (cos * 2.0 * a / d2)[:, None] * np.array([1.0, 0.8, 0.6])
    got = img.reshape(-1, 3).astype(np.float64)
    sel = on & (cos > 1e-3)
    assert sel.sum() > 300
    np.testing.assert_allclose(got[sel], want[sel], rtol=2e-4, atol=1e-7)
    if kind == "spot":
        out = on & (a == 0) & (np.abs((-L) @ sd - co) > 1e-5)
        assert out.sum() > 100 and (got[out] == 0).all()
    assert c["rays_shadow"] > 0


def _split_scene():
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    hdr = scenes.synth_hdr(128, 64)
    return tris, nodes, eye, cam, hdr, api.hdr_cache(hdr)


def _mean_of(img, luma2, first, n):
    k = np.float32(first + n) / np.float32(n)   # a render from frame `first` onto a zero framebuffer blends its frames as (first + n)-ths
    return img.astype(np.float64) * float(k), luma2.astype(np.float64) * float(k)


@pytest.mark.parametrize("variant", ["plain", "fog", "glass"])
def test_split_is_unbiased(variant):
    """the flagged render of triangle lights + the map + a rig estimates the sum of mode 4 with the map (no punctual lights) and of the
    punctual-only render of the same scene with black emitters and a black map; disjoint frame ranges"""
    tris, nodes, eye, cam, hdr, cache = _split_scene()
    m = None
    if variant == "glass":
        tris, nodes, eye, cam = transmission_scenes.p3_glass("blob")
    tris = np.asarray(tris, np.float32).reshape(-1, 36)
    rig = scenes.punctual_rig(tris, seed=3, power=0.5)
    W, H, n = 64, 48, 256
    base = dict(width=W, height=H, spp=n, max_bounce=3, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam),
                transmission=variant == "glass", medium=variant == "fog")
    if variant == "fog":
        m = oracle_medium.medium(sigma_t=0.3, albedo=(0.9, 0.8, 0.7), g=0.4, box_min=(-1.5, -1.5, -1.5), box_max=(1.5, 1.5, 1.5))
    cfg = api.RenderConfig(**base, env_light=True, punctual_lights=True)
    a = _stats(*op.render(tris, nodes, cfg, rig, m=m, hdr=hdr, hdr_cache=cache, threads=0)[:2])
    cfg = api.RenderConfig(**base, env_light=True, first_frame=n)
    img1, l1, _, _ = op.render(tris, nodes, cfg, None, m=m, hdr=hdr, hdr_cache=cache)
    dark = tris.copy()
    dark[:, 18:21] = 0.0
    black = np.zeros_like(hdr)
    cfg = api.RenderConfig(**base, punctual_lights=True, first_frame=2 * n)
    img2, l2, _, _ = op.render(dark, nodes, cfg, rig, m=m, hdr=black, hdr_cache=api.hdr_cache(black))
    s1 = _stats(*_mean_of(img1, l1, n, n))
    s2 = _stats(*_mean_of(img2, l2, 2 * n, n))
    b = (s1[0] + s2[0], s1[1] + s2[1])
    z8, z16 = _block_z(a, b, n, W, H, 8, 8), _block_z(a, b, n, W, H, 16, 16)
    zf = float(_block_z(a, b, n, W, H, H, W).max())
    print("punctual split %-5s: frame z %.2f, largest 16x16 z %.2f, largest 8x8 z %.2f, mean luminance %.4g vs %.4g" %
          (variant, zf, z16.max(), z8.max(), a[0].mean(), b[0].mean()))
    assert np.isfinite(z8).all() and zf <= 4 and z16.max() <= 5 and z8.max() <= 5, (zf, z16.max(), z8.max())
