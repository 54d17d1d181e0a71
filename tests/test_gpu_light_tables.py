"""The light tables of the light sampling mode on the GPU against their CPU restatements, bit for bit, and against float64 numpy,
on the inputs where the device builders could go wrong (DESIGN.md sections 10 and 11):

- Scene.lights() (k_light_weights, then k_light_compact: one block, 1024-triangle chunks, ranks from block_append) with no light, one,
  1023 / 1024 / 1025 / 2049 lights contiguous from the first triangle and spread over several chunks, lights interleaved with
  non-lights across chunk boundaries, the first and last triangle lights, hostile emitters, a scene on the indexed vertex layout,
  and a scene whose every triangle is a light;
- Scene.env_light_table() (k_env_weights, then float64 sums on the host) on maps one texel wide or tall, odd shapes, shapes whose
  texel count is not a multiple of the 256-thread block, hostile texels, a black column, one live texel in a polar row or the last
  column, an all-black map and bench.py's 2048 x 1024 map;
- renders of those scenes and maps, bit for bit with their ray counts;
- hdr_cache_device against hdr_cache on shapes that are not multiples of k_lum_sum's 4096-texel chunk, and on maps whose cdf is NaN."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_env_light as oe
from tests import oracle_lights as ol
from tests.test_env_light_oracle import _table_f64 as _env_table_f64
from tests.test_gpu_parity import assert_same_bits
from tests.test_gpu_w8 import W8_MIN_TRIANGLES
from tests.test_lights_oracle import _table_f64 as _light_table_f64

pytestmark = pytest.mark.gpu

L4 = api.MODE_DISNEY_LIGHTS
ENV = (0.35, 0.45, 0.6)
CHUNK = 1024   # k_light_compact's block


# ------------------------------------------------------------------ scenes
def _blob_geometry():
    """the blob (5120 triangles) on a floor box (12): 5132 triangles, six compaction chunks; no emission"""
    tl = api.TriangleList()
    tl.read_obj_text(scenes.blob_obj(), api.Material(baseColor=(0.8, 0.8, 0.8), roughness=0.4), api.transform_matrix(), True)
    tl.read_obj_text(scenes.box_obj(), api.Material(baseColor=(0.725, 0.71, 0.68)), api.transform_matrix((0, 0, 0), (0, -1.4, 0), (8, 0.01, 8)), False)
    tris, nodes = tl.build_bvh(8)
    eye, cam = api.camera_orbit(20.0, 15.0, 3.5)
    return np.asarray(tris, np.float32).reshape(-1, 36), np.asarray(nodes, np.float32), eye, cam


def _with_lights(tris, idx, seed=1):
    """tris with emission only on the triangles idx (varied, positive)"""
    t = tris.copy()
    t[:, 18:21] = 0.0
    idx = np.asarray(idx, np.int64)
    t[idx, 18:21] = np.random.default_rng(seed).uniform(0.5, 20.0, (len(idx), 3)).astype(np.float32)
    return t


def _hostile(tris):
    """3000 lights spread over the scene, the first and last triangle among them, then hostile emitters in their place"""
    n = len(tris)
    rng = np.random.default_rng(5)
    idx = np.unique(np.concatenate([[0, n - 1], rng.choice(n, 3000, replace=False)]))
    t = _with_lights(tris, idx, seed=6)
    bad = rng.choice(idx[1:-1], 11 * 20, replace=False).reshape(11, 20)
    t[bad[0], 18:21] = [np.nan, 1, 1]                      # NaN
    t[bad[1], 18:21] = [np.inf, 1, 1]                      # inf weight
    t[bad[2], 18:21] = [-np.inf, 1, 1]
    t[bad[3], 18:21] = [-5, -5, -5]                        # negative
    t[bad[4], 18:21] = 0.0                                 # black
    t[bad[5], 18:21] = -0.0
    t[bad[6], 3:6] = t[bad[6], 0:3]                        # zero area
    t[bad[6], 6:9] = t[bad[6], 0:3]
    t[bad[7], 18:21] = [-1, 5, 0]                          # a negative channel, luminance 2.7 > 0: a light
    t[bad[8], 18:21] = [5, -3, 0]                          # a positive channel, luminance -0.3: not a light
    t[bad[9], 18:21] = [1e-38, 1e-38, 1e-38]               # a subnormal weight > 0: a light
    t[bad[10], 18:21] = [3e38, 3e38, 3e38]                 # huge, finite: one light outweighs all the others
    return t


def _light_scenes():
    """{name: (tris, nodes, eye, cam)} of the table tests"""
    tris, nodes, eye, cam = _blob_geometry()
    n = len(tris)
    rng = np.random.default_rng(3)
    out = {"K=0": _with_lights(tris, [])}
    out["K=1, first triangle"] = _with_lights(tris, [0])
    out["K=1, last triangle"] = _with_lights(tris, [n - 1])
    for k in (1023, 1024, 1025, 2049):
        out["K=%d, the first %d triangles" % (k, k)] = _with_lights(tris, np.arange(k))
        spread = np.unique(np.concatenate([[0, n - 1], rng.choice(np.arange(1, n - 1), k - 2, replace=False)]))
        assert len(spread) == k
        out["K=%d, spread" % k] = _with_lights(tris, spread)
    # every other triangle around each chunk boundary (both parities), plus the first and last triangle
    near = np.concatenate([np.arange(b - 37, min(b + 41, n)) for b in range(CHUNK, n, CHUNK)])
    inter = np.unique(np.concatenate([[0, n - 1], near[near % 2 == 0], np.arange(3 * CHUNK - 1, 3 * CHUNK + 2)]))
    out["interleaved across chunk boundaries"] = _with_lights(tris, inter)
    out["hostile emitters"] = _hostile(tris)
    return {k: (v, nodes, eye, cam) for k, v in out.items()}


@pytest.fixture(scope="module")
def light_scenes():
    return _light_scenes()


@pytest.fixture(scope="module")
def big_scenes():
    """s_grid(5, 4): 103,692 triangles, the indexed vertex layout; some lights, and every triangle a light"""
    tris, nodes, eye, cam = scenes.s_grid(5, 4, 4)
    tris = np.asarray(tris, np.float32).reshape(-1, 36)
    n = len(tris)
    assert n >= W8_MIN_TRIANGLES and n >= 100_000
    rng = np.random.default_rng(9)
    some = tris.copy()
    pick = rng.random(n) < 0.3
    some[pick, 18:21] = rng.uniform(0.1, 5.0, (int(pick.sum()), 3)).astype(np.float32)
    every = tris.copy()
    every[:, 18:21] = rng.uniform(0.01, 3.0, (n, 3)).astype(np.float32)
    return {"W8 indexed, 30% lights": (some, nodes, eye, cam), "W8 indexed, every triangle a light": (every, nodes, eye, cam)}


def _check_light_table(sc, tris, what):
    tri, cdf, total = sc.lights()
    rtri, rcdf, rtotal = ol.oracle_light_table(tris)
    assert tri.tobytes() == rtri.tobytes(), what
    assert cdf.tobytes() == rcdf.tobytes(), what
    assert total == rtotal, what
    idx, cdf64, total64 = _light_table_f64(tris)
    assert (tri == idx).all(), what
    if len(idx):
        assert abs(total - total64) <= 1e-6 * total64, what
        np.testing.assert_allclose(cdf, cdf64, rtol=1e-6, atol=1e-7, err_msg=what)
        assert cdf[-1] == 1.0 and (np.diff(cdf) >= 0).all(), what
    else:
        assert total == 0.0, what
    return len(tri)


# ------------------------------------------------------------------ (a) Scene.lights()
def test_light_tables_bit_identical(light_scenes):
    counts = {}
    for name, (tris, nodes, _, _) in light_scenes.items():
        sc = api.Scene(tris, nodes)
        try:
            counts[name] = _check_light_table(sc, tris, name)
        finally:
            sc.close()
    assert counts["K=0"] == 0 and counts["K=1, last triangle"] == 1
    for k in (1023, 1024, 1025, 2049):
        assert counts["K=%d, spread" % k] == k and counts["K=%d, the first %d triangles" % (k, k)] == k
    print("light tables: " + ", ".join("%s %d" % kv for kv in counts.items()))
    # the hostile scene keeps the emitters with a finite weight > 0: a negative channel with positive luminance, a subnormal
    # weight and a huge emission
    tris = light_scenes["hostile emitters"][0]
    tri = ol.oracle_light_table(tris)[0]
    e = tris[tri, 18]
    assert (e == -1).sum() == 20 and (e == np.float32(1e-38)).sum() == 20 and (e == np.float32(3e38)).sum() == 20


def test_light_tables_of_big_scenes(big_scenes):
    for name, (tris, nodes, _, _) in big_scenes.items():
        sc = api.Scene(tris, nodes)
        try:
            k = _check_light_table(sc, tris, name)
            print("%s: %d triangles, %d lights" % (name, len(tris), k))
            if "every" in name:
                assert k == len(tris)
        finally:
            sc.close()


# ------------------------------------------------------------------ (b) Scene.env_light_table()
def _hostile_texels(W=300, H=150):
    hdr = scenes.synth_hdr(W, H)
    hdr[3, 7] = -0.0
    hdr[4, 8] = (1e-40, 1e-40, 1e-40)                # subnormal texels: a subnormal weight > 0
    hdr[5, 9] = (2e-39, 0.0, 3e-39)
    hdr[6, 10] = (np.inf, 1.0, 1.0)
    hdr[7, 11] = (-np.inf, 1.0, 1.0)
    hdr[8, 12] = (np.nan, 1.0, 1.0)
    hdr[9, 13] = (-2.0, -2.0, -2.0)
    hdr[10, 14] = (-1.0, 5.0, 0.0)                   # a negative channel, positive luminance
    hdr[12] = 0.0                                    # a black row
    return hdr


def _one_live(W, H, i, j):
    hdr = np.zeros((H, W, 3), np.float32)
    hdr[i, j] = (40.0, 30.0, 20.0)
    return hdr


def _maps():
    """{name: W x H x 3 map}"""
    out = {"%dx%d" % (w, h): scenes.synth_hdr(w, h) for w, h in ((1, 1), (1, 7), (7, 1), (3, 5), (300, 150), (4100, 3))}
    out["hostile texels"] = _hostile_texels()
    col = scenes.synth_hdr(300, 150)
    col[:, 0] = 0.0
    col[:, 123] = 0.0
    out["black columns"] = col
    out["one live texel, top row"] = _one_live(300, 150, 0, 37)
    out["one live texel, bottom row"] = _one_live(300, 150, 149, 0)
    out["one live texel, last column"] = _one_live(300, 150, 75, 299)
    huge = scenes.synth_hdr(300, 150)
    huge[140, 200] = (3e38, 3e38, 3e38)              # finite, and all but this texel's pdf is subnormal or 0
    out["one huge texel"] = huge
    out["all black"] = np.zeros((150, 300, 3), np.float32)
    out["2048x1024"] = scenes.synth_hdr(2048, 1024)
    return out


@pytest.fixture(scope="module")
def maps():
    return _maps()


def test_env_tables_bit_identical(maps, light_scenes):
    tris, nodes, _, _ = light_scenes["K=1, first triangle"]
    for name, hdr in maps.items():
        sc = api.Scene(tris, nodes, hdr, api.hdr_cache(hdr))
        try:
            got, want, ref = sc.env_light_table(), oe.env_table(hdr), _env_table_f64(hdr)
            if name == "all black":
                assert got is None and want is None and ref is None, name
                continue
            for g, w, what in zip(got[:3], want[:3], ("row_cdf", "col_cdf", "texel_pdf")):
                assert g.tobytes() == w.tobytes(), "%s: %s" % (name, what)
            assert got[3] == want[3], name
            row, col, pdf, T = got
            row64, col64, pdf64, T64 = ref
            assert abs(T - T64) <= 1e-5 * T64, name
            np.testing.assert_allclose(row, row64, rtol=1e-5, atol=1e-7, err_msg=name)
            np.testing.assert_allclose(col, col64, rtol=1e-5, atol=1e-7, err_msg=name)
            np.testing.assert_allclose(pdf, pdf64, rtol=1e-5, atol=1e-12, err_msg=name)
            live = pdf.sum(1) > 0
            assert row[-1] == 1.0 and (col[live, -1] == 1.0).all() and (col[~live] == 0).all(), name
            if name.startswith("one live"):
                assert np.count_nonzero(pdf) == 1 and pdf.max() == 1.0, name
        finally:
            sc.close()
    hostile = oe.env_table(maps["hostile texels"])[2]
    # -0.0, inf, -inf, NaN and negative texels weigh 0; a negative channel with positive luminance is live; a subnormal texel's
    # weight is > 0, and its pdf rounds to 0 or to a subnormal
    assert hostile[10, 14] > 0 and hostile[3, 7] == 0 and (hostile[6:10, 10:14].diagonal() == 0).all()
    assert hostile[4, 8] == 0 and 0 < hostile[5, 9] < 1e-44
    assert (hostile[12] == 0).all()


# ------------------------------------------------------------------ (c) renders, bit for bit with ray counts
def _render_case(sc, tris, nodes, cfg, what, hdr=None, cache=None):
    img = sc.render(cfg)
    c = sc.counters()
    ref, _, rc = oe.oracle_render_env_light(tris, nodes, cfg, hdr=hdr, hdr_cache=cache)
    assert_same_bits(img, ref, what)
    assert (c.primary_rays, c.bounce_rays, c.shadow_rays) == (rc["rays_primary"], rc["rays_bounce"], rc["rays_shadow"]), what
    return c.shadow_rays


def _cfg(eye, cam, **kw):
    base = dict(width=32, height=24, spp=2, max_bounce=1, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam), env_color=ENV)
    base.update(kw)
    return api.RenderConfig(**base)


def test_renders_of_the_light_scenes(light_scenes, big_scenes):
    hdr = scenes.synth_hdr(300, 150)
    cache = api.hdr_cache(hdr)
    for name, (tris, nodes, eye, cam) in {**light_scenes, **big_scenes}.items():
        has_light = len(ol.oracle_light_table(tris)[0]) > 0
        for with_map in (False, True):
            if not (has_light or with_map):
                continue
            h, c = (hdr, cache) if with_map else (None, None)
            sc = api.Scene(tris, nodes, h, c)
            try:
                for bounces in (1, 3):
                    shadow = _render_case(sc, tris, nodes, _cfg(eye, cam, max_bounce=bounces, env_light=with_map),
                                          "%s, %s, %d bounces" % (name, "flagged, 300x150 map" if with_map else "mode 4", bounces), h, c)
                    assert shadow > 0, name
            finally:
                sc.close()


def test_renders_under_the_maps(maps, light_scenes):
    for scene_name in ("K=0", "K=1025, spread"):
        tris, nodes, eye, cam = light_scenes[scene_name]
        for name, hdr in maps.items():
            cache = api.hdr_cache(hdr)
            for linear in ((True, False) if name == "hostile texels" else (True,)):
                sc = api.Scene(tris, nodes, hdr, cache, hdr_filter_linear=linear)
                try:
                    for bounces in (1, 3):
                        cfg = _cfg(eye, cam, max_bounce=bounces, env_light=True)
                        what = "%s under the %s map (%s), %d bounces" % (scene_name, name, "linear" if linear else "nearest", bounces)
                        img = sc.render(cfg)
                        c = sc.counters()
                        ref, _, rc = oe.oracle_render_env_light(tris, nodes, cfg, hdr=hdr, hdr_cache=cache, hdr_linear=linear)
                        assert_same_bits(img, ref, what)
                        assert (c.primary_rays, c.bounce_rays, c.shadow_rays) == (rc["rays_primary"], rc["rays_bounce"], rc["rays_shadow"]), what
                        if name != "all black" or scene_name != "K=0":
                            assert c.shadow_rays > 0, what
                finally:
                    sc.close()


# ------------------------------------------------------------------ (d) hdr_cache_device
def _cache_maps():
    out = {"%dx%d" % (w, h): scenes.synth_hdr(w, h) for w, h in ((1, 1), (100, 37), (4097, 1), (1, 5000), (300, 150))}
    col = scenes.synth_hdr(300, 150)
    col[:, 17] = 0.0                                 # margin 0: that column's cdf_y is NaN (0 / 0), searched by k_samples
    out["black column"] = col
    bad = scenes.synth_hdr(100, 37)
    bad[3, 4] = (np.nan, 1.0, 1.0)
    bad[5, 6] = (np.inf, 1.0, 1.0)
    bad[7, 8] = (-np.inf, 0.0, 0.0)
    out["NaN and inf texels"] = bad
    inf = scenes.synth_hdr(100, 37)
    inf[20, 30] = (np.inf, np.inf, np.inf)
    out["one inf texel"] = inf
    return out


@pytest.mark.parametrize("name", list(_cache_maps().keys()))
def test_hdr_cache_device_equals_host(name):
    hdr = _cache_maps()[name]
    host = api.hdr_cache(hdr)
    dev, _ = api.hdr_cache_device(hdr)
    assert_same_bits(dev, host, name)
