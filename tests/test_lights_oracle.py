"""The CPU restatement of the light sampling mode (tests/oracle_lights.cpp; DESIGN.md section 10) against independent
computations: the light table in float64 numpy, the triangle sampler's moments, the estimator against mode 2 on the same scene
(unbiased, lower variance), the shadow rays' tmax margin on an open scene, and a scene without lights."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_lights as ol


def _table_f64(tris):
    t = np.asarray(tris, np.float64).reshape(-1, 36)
    p1, p2, p3 = t[:, 0:3], t[:, 3:6], t[:, 6:9]
    area = 0.5 * np.linalg.norm(np.cross(p2 - p1, p3 - p1), axis=1)
    e = t[:, 18:21]
    with np.errstate(invalid="ignore", over="ignore"):
        w = area * (0.3 * e[:, 0] + 0.6 * e[:, 1] + 0.1 * e[:, 2])
        keep = np.isfinite(w) & (w > 0)
    idx = np.flatnonzero(keep)
    return idx, np.cumsum(w[idx]) / w[idx].sum(), w[idx].sum()


def _hostile_emitters():
    tris, nodes, _, _ = scenes.s_p3_bunny()
    t = np.array(tris, np.float32).reshape(-1, 36)
    extra = np.repeat(t[-1:], 5, 0)
    extra[0, 3:6] = extra[0, 0:3]; extra[0, 6:9] = extra[0, 0:3]    # zero area
    extra[1, 18:21] = [-5, -5, -5]                                   # negative emission
    extra[2, 18:21] = [np.nan, 1, 1]                                 # NaN emission
    extra[3, 18:21] = [0, 0, 0]                                      # black
    extra[4, 18:21] = [2, 0, 0]                                      # a plain light
    return np.concatenate([t, extra])


@pytest.mark.parametrize("which", ["p3", "hostile"])
def test_light_table_matches_float64(which):
    tris = scenes.s_p3_bunny()[0] if which == "p3" else _hostile_emitters()
    tri, cdf, total = ol.oracle_light_table(tris)
    idx, cdf64, total64 = _table_f64(tris)
    assert (tri == idx).all()
    assert abs(total - total64) <= 1e-6 * total64
    np.testing.assert_allclose(cdf, cdf64, rtol=1e-6)
    assert cdf[-1] == 1.0
    if which == "hostile":
        n = len(tris)
        assert list(tri[-1:]) == [n - 1] and not set(range(n - 5, n - 1)) & set(tri.tolist())


def test_triangle_sampler_is_uniform():
    p1, p2, p3 = np.array([0.0, 0, 0]), np.array([2.0, 0, 0]), np.array([0.5, 1.5, 0.3])
    r = np.random.default_rng(1).random((1_000_000, 2)).astype(np.float32)
    q = ol.triangle_points(p1, p2, p3, r).astype(np.float64)
    # inside: barycentric coordinates in [0, 1] (a few ulps of slack)
    e1, e2, v = p2 - p1, p3 - p1, q - p1
    g = np.array([[e1 @ e1, e1 @ e2], [e1 @ e2, e2 @ e2]])
    b = np.linalg.solve(g, np.stack([v @ e1, v @ e2]))
    assert (b > -1e-6).all() and (b.sum(0) < 1 + 1e-6).all()
    # uniform over the triangle: mean = centroid, covariance = (sum of outer products of the centred vertices) / 12
    verts = np.stack([p1, p2, p3])
    c = verts.mean(0)
    cov = sum(np.outer(x - c, x - c) for x in verts) / 12.0
    np.testing.assert_allclose(q.mean(0), c, atol=3e-3)
    np.testing.assert_allclose(np.cov(q.T), cov, atol=3e-3)


def test_unbiased_against_mode_2_with_lower_variance():
    """Mode 4 against mode 2 (the same Disney BRDF, uniform hemisphere sampling, emission hits at weight 1) under a constant
    environment.  Mode 3 cannot be the yardstick here: with a 1 x 1 map its hdrPdf is 0 (res * res / 2 = 0, P5/fsh:709) and
    its environment samples are NaN."""
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    out = {}
    for mode in (api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_LIGHTS):
        cfg = api.RenderConfig(width=64, height=48, spp=1024, max_bounce=2, mode=mode, eye=tuple(eye), camera_rotate=tuple(cam),
                               env_color=(0.5, 0.5, 0.5))
        img, luma2, _ = ol.oracle_render_lights(tris, nodes, cfg)
        y = (0.3 * img[..., 0] + 0.6 * img[..., 1] + 0.1 * img[..., 2]).astype(np.float64)
        out[mode] = (y, np.maximum(luma2.astype(np.float64) - y ** 2, 0.0), cfg.spp)
    (y2, v2, n), (y4, v4, _) = out[api.MODE_DISNEY_SOBOL_P5], out[api.MODE_DISNEY_LIGHTS]
    blk = lambda a: a.reshape(6, 8, 8, 8).swapaxes(1, 2).reshape(6, 8, 64)
    se = np.sqrt(blk(v2).sum(-1) / n / 64 ** 2 + blk(v4).sum(-1) / n / 64 ** 2)
    z = np.abs(blk(y2).mean(-1) - blk(y4).mean(-1)) / np.maximum(se, 1e-12)
    assert np.isfinite(z).all() and (z <= 5).all(), "block means differ by up to %.2f standard errors" % z.max()
    assert v4.mean() < v2.mean() / 4, (v4.mean(), v2.mean())   # 7.0x lower (DESIGN.md section 10)


def _quad_scene(with_light=True):
    """A 4 x 4 floor at y = 0 under an emissive 1 x 1 quad at y = 2 (facing down), nothing in between."""
    floor = api.Material(baseColor=(0.7, 0.7, 0.7), roughness=0.6)
    lamp = api.Material(baseColor=(1, 1, 1), emissive=(10, 10, 10) if with_light else (0, 0, 0))
    tl = api.TriangleList()
    quad = "v -1 0 -1\nv 1 0 -1\nv 1 0 1\nv -1 0 1\nf 1 3 2\nf 1 4 3\n"
    tl.read_obj_text(quad, floor, api.transform_matrix((0, 0, 0), (0, 0, 0), (2, 1, 2)), False)
    tl.read_obj_text(quad.replace("f 1 3 2\nf 1 4 3", "f 1 2 3\nf 1 3 4"), lamp, api.transform_matrix((0, 0, 0), (0, 2, 0), (0.5, 1, 0.5)), False)
    tris, nodes = tl.build_bvh(8)
    return np.asarray(tris, np.float32).reshape(-1, 36), nodes


def test_open_scene_no_light_sample_is_occluded():
    tris, nodes = _quad_scene()
    tri, _, _ = ol.oracle_light_table(tris)
    assert len(tri) == 2
    rng = np.random.default_rng(7)
    n = 20000
    P = np.column_stack([rng.uniform(-1.9, 1.9, n), np.zeros(n), rng.uniform(-1.9, 1.9, n)]).astype(np.float32)
    P[:, 1] = tris[0, 1]   # on the floor plane
    k = rng.integers(0, 2, n)
    v = tris[tri[k], :9].reshape(-1, 3, 3)
    r = rng.random((n, 2)).astype(np.float32)
    Q = np.stack([ol.triangle_points(v[i, 0], v[i, 1], v[i, 2], r[i:i + 1])[0] for i in range(n)])
    D = (Q - P).astype(np.float32)
    dist = np.sqrt((D * D).sum(1)).astype(np.float32)
    L = (D / dist[:, None]).astype(np.float32)
    tmax = (dist * np.float32(1 - 2 ** -10)).astype(np.float32)
    for trav in (api.TRAVERSE_REFERENCE, api.TRAVERSE_PRUNED):
        lit = ol.oracle_occluded(tris, nodes, P, L, tmax, traverse=trav)
        assert lit.all(), "%d of %d light samples occluded" % (n - lit.sum(), n)
    # without the margin the light's own triangle occludes some of them
    assert not ol.oracle_occluded(tris, nodes, P, L, dist * np.float32(1.01)).all()


def test_no_lights_no_shadow_rays():
    tris, nodes = _quad_scene(with_light=False)
    assert len(ol.oracle_light_table(tris)[0]) == 0
    eye, cam = api.camera_orbit(0.0, 30.0, 4.0)
    cfg = api.RenderConfig(width=16, height=16, spp=2, max_bounce=2, mode=api.MODE_DISNEY_LIGHTS, env_color=(0.5, 0.5, 0.5),
                           eye=tuple(eye), camera_rotate=tuple(cam))
    img, _, c = ol.oracle_render_lights(tris, nodes, cfg)
    assert c["rays_shadow"] == 0 and c["rays_bounce"] > 0 and np.isfinite(img).all()
