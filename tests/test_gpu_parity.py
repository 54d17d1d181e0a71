"""GPU parity tests: the sm_90a path (through the C ABI) against the CPU oracle, bit for bit.

The north_star tolerance is 1e-4 per-channel L-infinity on the same Sobol seed; because host
and device evaluate the same fp32 operation sequence (include/ezrt_math.h) the tests assert
the stronger property: identical bits (NaNs in identical places)."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes

pytestmark = pytest.mark.gpu

TOL = 1e-4  # north_star: per-channel L-inf vs the reference CPU render


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def assert_same_bits(a, b, what=""):
    a = np.asarray(a, dtype=np.float32); b = np.asarray(b, dtype=np.float32)
    assert a.shape == b.shape, what
    same = (_bits(a) == _bits(b)) | (np.isnan(a) & np.isnan(b))
    if not same.all():
        bad = np.argwhere(~same)
        linf = np.nanmax(np.abs(a.astype(np.float64) - b.astype(np.float64)))
        raise AssertionError("%s: %d of %d values differ (first at %s: %r vs %r), L-inf %.3g" %
                             (what, len(bad), a.size, bad[0], a[tuple(bad[0])], b[tuple(bad[0])], linf))


@pytest.fixture(scope="module")
def gpu_bunny(bunny_scene):
    tris, nodes, eye, cam = bunny_scene
    sc = api.Scene(tris, nodes)
    yield sc
    sc.close()


@pytest.fixture(scope="module")
def gpu_grid(grid_scene):
    tris, nodes, eye, cam = grid_scene
    sc = api.Scene(tris, nodes)
    yield sc
    sc.close()


# ------------------------------------------------------------------ arithmetic definition
@pytest.mark.parametrize("which,name", [(0, "sin"), (1, "cos"), (2, "log"), (3, "exp"), (4, "pow"), (5, "atan2"), (6, "asin")])
def test_math_bit_exact(oracle, which, name):
    rng = np.random.default_rng(100 + which)
    n = 200000
    if name in ("sin", "cos"):
        a = np.concatenate([rng.uniform(-14, 14, n), rng.uniform(-1e-3, 1e-3, 1000), [0.0, 6.2831852, 3.1415926, 1e4, -1e4]])
        b = None
    elif name == "log":
        a = np.concatenate([rng.uniform(1e-7, 4, n), np.exp(rng.uniform(-80, 80, 5000)), [1.0, 1e-6, 0.01, 0.0, -1.0, 1e-42]])
        b = None
    elif name == "exp":
        a = np.concatenate([rng.uniform(-20, 20, n), rng.uniform(-110, 95, 5000), [0.0]])
        b = None
    elif name == "pow":
        a = rng.uniform(1e-6, 1.0, n); b = rng.uniform(0, 1, n)
    elif name == "atan2":
        a = np.concatenate([rng.uniform(-2, 2, n), [0, 0, 1, -1, 0.0]]); b = np.concatenate([rng.uniform(-2, 2, n), [0, 1, 0, 0, -1.0]])
    else:
        a = np.concatenate([rng.uniform(-1, 1, n), [1.0, -1.0, 1.0000001, 0.5, 1e-5, 0.0]]); b = None
    a = a.astype(np.float32); b = None if b is None else b.astype(np.float32)
    assert_same_bits(api.eval_math(which, a, b), oracle.eval_math(which, a, b), name)


def _random_brdf_inputs(n, seed):
    rng = np.random.default_rng(seed)

    def unit(v):
        return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)

    N = unit(rng.normal(size=(n, 3)))
    V = unit(N + 0.9 * rng.normal(size=(n, 3)))
    L = unit(N + 0.9 * rng.normal(size=(n, 3)))
    mats = np.zeros((n, 18), np.float32)
    mats[:, 0:3] = rng.uniform(0, 5, (n, 3)) * (rng.uniform(size=(n, 1)) < 0.1)
    mats[:, 3:6] = rng.uniform(0, 1, (n, 3))
    mats[:, 6:16] = rng.uniform(0, 1, (n, 10))
    mats[::7, 10] = 0.0  # roughness 0
    mats[::11, 15] = 1.0  # clearcoatGloss 1
    mats[::13, 3:6] = 0.0  # black base colour -> Cdlum == 0 branch
    mats[:, 16] = 1.0
    xi = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    return V, N, L, xi, mats


@pytest.mark.parametrize("which,name", [(0, "BRDF_Evaluate"), (1, "BRDF_Evaluate_aniso_P4"), (2, "BRDF_Pdf"), (3, "SampleBRDF")])
def test_brdf_bit_exact(oracle, which, name):
    V, N, L, xi, mats = _random_brdf_inputs(100000, 7 + which)
    assert_same_bits(api.eval_brdf(which, V, N, L, xi, mats), oracle.eval_brdf(which, V, N, L, xi, mats), name)


# ------------------------------------------------------------------ hitBVH / hitTriangle / hitAABB
def _random_rays(n, seed, extent=3.0):
    rng = np.random.default_rng(seed)
    o = rng.uniform(-extent, extent, (n, 3)).astype(np.float32)
    d = rng.normal(size=(n, 3))
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    # axis-aligned and zero-component directions exercise the inf/NaN slab arithmetic (P5/fsh:221-230)
    d[:64] = 0.0
    d[:64, 0] = 1.0
    d[64:128] = np.array([0.0, -1.0, 0.0], np.float32)
    d[128:160, 2] = 0.0
    d[128:160] /= np.linalg.norm(d[128:160], axis=1, keepdims=True)
    return o, d


@pytest.mark.parametrize("traverse", [api.TRAVERSE_ACCEL, api.TRAVERSE_PRUNED, api.TRAVERSE_REFERENCE])
@pytest.mark.parametrize("fudge", [False, True])
def test_trace_rays_match_oracle(oracle, bunny_scene, gpu_bunny, traverse, fudge):
    tris, nodes, eye, cam = bunny_scene
    o, d = _random_rays(20000, 11)
    got = gpu_bunny.trace_rays(o, d, traverse=traverse, p3_normal_fudge=fudge)
    ref = oracle.trace_rays(tris, nodes, o, d, traverse=api.TRAVERSE_REFERENCE, p3_fudge=fudge)
    assert ref["hit"].sum() > 1000
    np.testing.assert_array_equal(got["hit"], ref["hit"])
    np.testing.assert_array_equal(got["triangle"], ref["triangle"])
    np.testing.assert_array_equal(got["inside"], ref["inside"])
    assert_same_bits(got["distance"], ref["distance"], "distance")
    assert_same_bits(got["point"], ref["point"], "hitPoint")
    assert_same_bits(got["normal"], ref["normal"], "normal")


def test_any_hit_equals_closest_hit_flag(gpu_grid):
    o, d = _random_rays(20000, 13, extent=2.5)
    closest = gpu_grid.trace_rays(o, d)
    anyhit = gpu_grid.trace_rays(o, d, any_hit=True)
    np.testing.assert_array_equal(anyhit["hit"], closest["hit"])


def test_p2_demo_ray_bvh_equals_brute_force(oracle, bunny_scene, gpu_bunny):
    """The reference's only intersection fixture: P2/main.cpp:581-586, ray (0,0,1) -> normalize(0.1,-0.1,-0.7),
    hitBVH must equal the brute-force scan (commented cross-check at :585)."""
    tris, nodes, eye, cam = bunny_scene
    d = np.array([[0.1, -0.1, -0.7]], np.float64)
    d = (d / np.linalg.norm(d)).astype(np.float32)
    o = np.array([[0, 0, 1]], np.float32)
    brute = oracle.trace_rays(tris, nodes, o, d, brute=True)
    got = gpu_bunny.trace_rays(o, d)
    assert brute["hit"][0] == 1
    assert got["triangle"][0] == brute["triangle"][0]
    assert_same_bits(got["distance"], brute["distance"], "P2 demo ray")


# ------------------------------------------------------------------ whole-image parity
def _cfg(eye, cam, **kw):
    base = dict(width=96, height=64, spp=3, max_bounce=2, eye=tuple(eye), camera_rotate=tuple(cam), env_color=(0.35, 0.45, 0.6))
    base.update(kw)
    return api.RenderConfig(**base)


@pytest.mark.parametrize("pipeline", [api.PIPELINE_WAVEFRONT, api.PIPELINE_MEGAKERNEL])
@pytest.mark.parametrize("mode,bounces", [(api.MODE_DIFFUSE_P3, 3), (api.MODE_DISNEY_ANISO_P4, 4), (api.MODE_DISNEY_SOBOL_P5, 2)])
def test_render_matches_oracle_bunny(oracle, bunny_scene, gpu_bunny, mode, bounces, pipeline):
    tris, nodes, eye, cam = bunny_scene
    cfg = _cfg(eye, cam, mode=mode, max_bounce=bounces, pipeline=pipeline)
    ref, rc = oracle.render(tris, nodes, cfg)
    got = gpu_bunny.render(cfg)
    c = gpu_bunny.counters()
    assert np.abs(np.nan_to_num(got) - np.nan_to_num(ref)).max() <= TOL
    assert_same_bits(got, ref, "image mode %d" % mode)
    assert (c.primary_rays, c.bounce_rays, c.shadow_rays) == (rc["rays_primary"], rc["rays_bounce"], rc["rays_shadow"])


@pytest.mark.parametrize("pipeline", [api.PIPELINE_WAVEFRONT, api.PIPELINE_MEGAKERNEL])
@pytest.mark.parametrize("mode", [api.MODE_DISNEY_ANISO_P4, api.MODE_DISNEY_SOBOL_P5])
def test_render_matches_oracle_grid_materials(oracle, grid_scene, gpu_grid, mode, pipeline):
    tris, nodes, eye, cam = grid_scene
    cfg = _cfg(eye, cam, mode=mode, max_bounce=3, pipeline=pipeline, width=80, height=48, spp=2)
    ref, rc = oracle.render(tris, nodes, cfg)
    got = gpu_grid.render(cfg)
    assert_same_bits(got, ref, "grid image mode %d" % mode)
    assert gpu_grid.counters().rays == rc["rays"]


@pytest.mark.parametrize("pipeline", [api.PIPELINE_WAVEFRONT, api.PIPELINE_MEGAKERNEL])
@pytest.mark.parametrize("linear", [True, False])
def test_render_is_mis_matches_oracle(oracle, grid_scene, small_hdr, pipeline, linear):
    tris, nodes, eye, cam = grid_scene
    hdr, cache = small_hdr
    sc = api.Scene(tris, nodes, hdr, cache, hdr_filter_linear=linear)
    try:
        cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_IS_MIS_P5, max_bounce=2, pipeline=pipeline, width=80, height=48, spp=3)
        ref, rc = oracle.render(tris, nodes, cfg, hdr=hdr, hdr_cache=cache, hdr_linear=linear)
        got = sc.render(cfg)
        c = sc.counters()
        assert rc["rays_shadow"] > 0
        assert_same_bits(got, ref, "IS/MIS image")
        assert (c.primary_rays, c.bounce_rays, c.shadow_rays) == (rc["rays_primary"], rc["rays_bounce"], rc["rays_shadow"])
    finally:
        sc.close()


def test_hdr_environment_diffuse_clamp(oracle, bunny_scene, small_hdr):
    """P3's sampleHdr clamps the environment to 10 (P3/fsh:151-156); nearest filtering as P3/main.cpp:195-196."""
    tris, nodes, eye, cam = bunny_scene
    hdr, cache = small_hdr
    sc = api.Scene(tris, nodes, hdr, cache, hdr_filter_linear=False)
    try:
        cfg = _cfg(eye, cam, mode=api.MODE_DIFFUSE_P3, max_bounce=2)
        ref, _ = oracle.render(tris, nodes, cfg, hdr=hdr, hdr_cache=cache, hdr_linear=False)
        assert_same_bits(sc.render(cfg), ref, "P3 + HDR")
    finally:
        sc.close()


def test_c1_config_matches_oracle(oracle, bunny_scene, gpu_bunny):
    """BASELINE.json configs[0]: bunny-class scene, 256x256, 4 spp, 3 bounces (diffuse)."""
    tris, nodes, eye, cam = bunny_scene
    cfg = _cfg(eye, cam, width=256, height=256, spp=4, max_bounce=3, mode=api.MODE_DIFFUSE_P3)
    ref, rc = oracle.render(tris, nodes, cfg)
    got = gpu_bunny.render(cfg)
    assert np.abs(got - ref).max() <= TOL
    assert_same_bits(got, ref, "C1")
    assert gpu_bunny.counters().rays == rc["rays"]


def test_accumulation_continues_from_lastframe(oracle, bunny_scene, gpu_bunny):
    """spp frames in one call == the same frames in two calls with first_frame advanced (P5/fsh:942-944)."""
    tris, nodes, eye, cam = bunny_scene
    whole = gpu_bunny.render(_cfg(eye, cam, spp=5, mode=api.MODE_DISNEY_SOBOL_P5, frames_per_batch=2))
    part = gpu_bunny.render(_cfg(eye, cam, spp=2, mode=api.MODE_DISNEY_SOBOL_P5))
    part = gpu_bunny.render(_cfg(eye, cam, spp=3, first_frame=2, mode=api.MODE_DISNEY_SOBOL_P5), framebuffer=part.reshape(-1, 3).copy())
    assert_same_bits(whole, part, "split accumulation")
    ref, _ = oracle.render(tris, nodes, _cfg(eye, cam, spp=5, mode=api.MODE_DISNEY_SOBOL_P5))
    assert_same_bits(whole, ref, "5 spp vs oracle")


def test_rgba_output(bunny_scene, gpu_bunny):
    tris, nodes, eye, cam = bunny_scene
    rgb = gpu_bunny.render(_cfg(eye, cam))
    rgba = gpu_bunny.render(_cfg(eye, cam, out_channels=4))
    assert_same_bits(rgba[..., :3], rgb, "rgba")
    assert (rgba[..., 3] == 1.0).all()


# ------------------------------------------------------------------ size-independent properties at larger sizes
@pytest.mark.parametrize("policy", [api.TRAVERSE_ACCEL, api.TRAVERSE_PRUNED])
def test_fast_policies_equal_reference_traversal_large(gpu_grid, grid_scene, policy):
    """Neither pruning nor the acceleration tree may change a single bit: full-size property test (no oracle needed)."""
    tris, nodes, eye, cam = grid_scene
    cfg = _cfg(eye, cam, width=640, height=360, spp=4, max_bounce=3, mode=api.MODE_DISNEY_SOBOL_P5, traverse=policy)
    a = gpu_grid.render(cfg)
    ca = gpu_grid.counters()
    cfg.traverse = api.TRAVERSE_REFERENCE
    b = gpu_grid.render(cfg)
    cb = gpu_grid.counters()
    assert_same_bits(a, b, "policy %d vs reference traversal" % policy)
    assert ca.rays == cb.rays and ca.rays > 640 * 360 * 4


def test_accel_policy_defers_ties_to_the_exact_traversal(oracle, bunny_scene):
    """Every triangle twice (second copy with another material): every hit ties with its twin, the accel pass must
    defer all of them and the exact reference-order pass must pick the copy the shader picks."""
    tris, nodes, eye, cam = bunny_scene
    twin = tris.copy()
    twin[:, 21:24] = [0.9, 0.2, 0.1]  # baseColor of the copies
    tl = api.TriangleList()
    tl.append_encoded(np.concatenate([tris, twin]))
    tris2, nodes2 = tl.build_bvh(8)
    sc = api.Scene(tris2, nodes2)
    try:
        cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5, max_bounce=2, width=64, height=48, spp=2)
        ref, rc = oracle.render(tris2, nodes2, cfg)
        got = sc.render(cfg)
        c = sc.counters()
        assert_same_bits(got, ref, "twin triangles")
        assert c.rays == rc["rays"] and c.deferred_rays >= rc["hits"] > 1000
        o, d = _random_rays(4000, 21)
        a = sc.trace_rays(o, d, traverse=api.TRAVERSE_ACCEL)
        b = oracle.trace_rays(tris2, nodes2, o, d, traverse=api.TRAVERSE_REFERENCE)
        np.testing.assert_array_equal(a["triangle"], b["triangle"])
        assert_same_bits(a["distance"], b["distance"], "twin distance")
    finally:
        sc.close()


def test_accel_policy_rarely_defers(gpu_grid, grid_scene):
    tris, nodes, eye, cam = grid_scene
    gpu_grid.render(_cfg(eye, cam, width=320, height=180, spp=2, max_bounce=2))
    c = gpu_grid.counters()
    assert c.deferred_rays < c.rays // 1000


def test_wavefront_equals_megakernel_large(gpu_grid, grid_scene):
    tris, nodes, eye, cam = grid_scene
    cfg = _cfg(eye, cam, width=512, height=288, spp=3, max_bounce=4, mode=api.MODE_DISNEY_ANISO_P4)
    a = gpu_grid.render(cfg)
    cfg.pipeline = api.PIPELINE_MEGAKERNEL
    b = gpu_grid.render(cfg)
    assert_same_bits(a, b, "wavefront vs megakernel")


@pytest.mark.parametrize("count", [2, 3, 8])
def test_partitioned_render_equals_whole(gpu_bunny, bunny_scene, count):
    """Any image partition gives bit-identical pixels (SURVEY 8e): render each part, scatter, compare."""
    tris, nodes, eye, cam = bunny_scene
    W, H = 200, 120  # not a multiple of the 16-pixel tile
    whole = gpu_bunny.render(_cfg(eye, cam, width=W, height=H, spp=2))
    full = np.zeros((H, W, 3), np.float32)
    total = 0
    for rank in range(count):
        part = gpu_bunny.render(_cfg(eye, cam, width=W, height=H, spp=2, part_rank=rank, part_count=count))
        assert part.shape[0] == api.partition_pixels(W, H, rank, count)
        total += part.shape[0]
        api.partition_scatter_host(part, full, W, H, 3, rank, count)
    assert total == W * H
    assert_same_bits(full, whole, "partitioned image")


def test_errors_are_reported_not_fatal(bunny_scene):
    tris, nodes, eye, cam = bunny_scene
    bad = nodes.copy()
    bad[1, 0] = 0  # root loses its left child -> the shader would read the dummy node
    with pytest.raises(api.EzrtError) as e:
        api.Scene(tris, bad)
    assert e.value.code == -4
    sc = api.Scene(tris, nodes)
    try:
        with pytest.raises(api.EzrtError):
            sc.render(_cfg(eye, cam, mode=api.MODE_DISNEY_IS_MIS_P5))  # no HDR map
    finally:
        sc.close()


# ------------------------------------------------------------------ committed golden fixtures + edge cases
@pytest.mark.parametrize("name", ["p3", "bunny", "grid"])
def test_reference_shader_golden_frames(name):
    """tests/golden/refshader.npz holds frames rendered by THE REFERENCE'S OWN SHADER SOURCE (P3/P4/P5 fshader.fsh
    transpiled to C++, tests/golden/make_golden_refshader.py).  The CUDA path must reproduce them bit for bit
    through the C ABI, under every traversal policy and both pipelines."""
    from tests import refshader_cases as cases
    g = cases.load()
    hdr, cache = cases.environment()
    tris, nodes, eye, cam = cases.scene(name)
    built = {}
    try:
        for case in cases.CASES:
            key, mode, mb, lin, first, spp = case
            if lin not in built:
                built[lin] = api.Scene(tris, nodes, hdr, cache, hdr_filter_linear=lin)
            want = g["%s_%s" % (name, key)]
            for policy, pipeline in ((api.TRAVERSE_ACCEL, api.PIPELINE_WAVEFRONT), (api.TRAVERSE_REFERENCE, api.PIPELINE_WAVEFRONT),
                                     (api.TRAVERSE_PRUNED, api.PIPELINE_WAVEFRONT), (api.TRAVERSE_PRUNED, api.PIPELINE_MEGAKERNEL)):
                fb = g["%s_m3" % name].reshape(-1, 3).copy() if first else None
                got = built[lin].render(cases.config(case, eye, cam, traverse=policy, pipeline=pipeline), framebuffer=fb)
                assert_same_bits(got, want, "reference shader frame %s_%s policy %d pipeline %d" % (name, key, policy, pipeline))
    finally:
        for sc in built.values():
            sc.close()


def test_golden_p3_scene_images(small_hdr):
    """The reference's own P3 scene (real Stanford bunny, arrays committed in tests/golden/p3_scene.npz together
    with the oracle's images): the GPU must reproduce the committed images bit for bit, in all four modes."""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "p3_scene.npz"))
    hdr, cache = small_hdr
    sc = api.Scene(g["tris"], g["nodes"], hdr, cache)
    try:
        for mode, bounces in ((0, 3), (1, 4), (2, 2), (3, 2)):
            for policy in (api.TRAVERSE_ACCEL, api.TRAVERSE_REFERENCE):
                cfg = api.RenderConfig(width=48, height=32, spp=2, max_bounce=bounces, mode=mode, eye=tuple(g["eye"]),
                                       camera_rotate=tuple(g["cam"]), env_color=(0.35, 0.45, 0.6), traverse=policy)
                if mode != 3:  # the golden images of modes 0-2 were rendered without an environment map
                    sc2 = api.Scene(g["tris"], g["nodes"])
                    try:
                        got = sc2.render(cfg)
                        c = sc2.counters()
                    finally:
                        sc2.close()
                else:
                    got = sc.render(cfg)
                    c = sc.counters()
                assert_same_bits(got, g["img_mode%d" % mode], "golden P3 scene, mode %d policy %d" % (mode, policy))
                assert [c.primary_rays, c.bounce_rays, c.shadow_rays] == list(g["rays_mode%d" % mode][:3])
    finally:
        sc.close()


@pytest.mark.parametrize("policy", [api.TRAVERSE_ACCEL, api.TRAVERSE_PRUNED, api.TRAVERSE_REFERENCE])
def test_long_leaves_and_single_leaf_trees(oracle, bunny_scene, policy):
    """Caller-provided trees: leaves of up to 20 triangles (several octet passes) and a scene that is one leaf."""
    tris, nodes, eye, cam = bunny_scene
    tl = api.TriangleList()
    tl.append_encoded(tris)
    t20, n20 = tl.build_bvh(20)
    assert n20[:, 3].max() > 8
    sc = api.Scene(t20, n20)
    try:
        cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5, width=64, height=48, spp=2, traverse=policy)
        ref, rc = oracle.render(t20, n20, cfg)
        assert_same_bits(sc.render(cfg), ref, "20-triangle leaves")
        assert sc.counters().rays == rc["rays"]
    finally:
        sc.close()
    tl = api.TriangleList()
    tl.append_encoded(tris[-5:])  # five triangles of the emissive sphere: the root is a leaf
    t1, n1 = tl.build_bvh(8)
    assert n1.shape[0] == 2 and n1[1, 3] == 5
    sc = api.Scene(t1, n1)
    try:
        cfg = _cfg(eye, cam, mode=api.MODE_DIFFUSE_P3, width=48, height=32, spp=2, traverse=policy)
        ref, rc = oracle.render(t1, n1, cfg)
        assert_same_bits(sc.render(cfg), ref, "single-leaf tree")
        o, d = _random_rays(2000, 5, extent=1.5)
        a = sc.trace_rays(o, d, traverse=policy)
        b = oracle.trace_rays(t1, n1, o, d, traverse=api.TRAVERSE_REFERENCE)
        np.testing.assert_array_equal(a["triangle"], b["triangle"])
    finally:
        sc.close()


def test_zero_bounces_and_zero_spp(oracle, bunny_scene, gpu_bunny):
    tris, nodes, eye, cam = bunny_scene
    cfg = _cfg(eye, cam, max_bounce=0, spp=2)
    ref, rc = oracle.render(tris, nodes, cfg)
    assert_same_bits(gpu_bunny.render(cfg), ref, "max_bounce = 0")
    assert gpu_bunny.counters().rays == rc["rays"] == 96 * 64 * 2
    fb = np.full((64 * 96, 3), 7.0, np.float32)
    out = gpu_bunny.render(_cfg(eye, cam, spp=0, first_frame=3), framebuffer=fb)
    assert (out == 7.0).all()  # spp = 0 leaves lastFrame untouched


# ------------------------------------------------------------------ hostile geometry
def _soup(n, seed):
    """Random overlapping triangles incl. zero-area, sliver and duplicated-vertex ones, three materials."""
    rng = np.random.default_rng(seed)
    t = np.zeros((n, 36), np.float32)
    c = rng.uniform(-2, 2, (n, 1, 3))
    p = c + rng.normal(scale=0.35, size=(n, 3, 3))
    p[::17, 2] = p[::17, 1]                      # zero-area: p3 == p2  (N = NaN)
    p[5::23, 2] = p[5::23, 0] + 1e-6 * (p[5::23, 1] - p[5::23, 0])  # slivers
    p[7::29] = np.round(p[7::29], 1)             # axis-aligned-ish coordinates: exact plane hits
    t[:, :9] = p.reshape(n, 9)
    nrm = rng.normal(size=(n, 3, 3))
    nrm /= np.linalg.norm(nrm, axis=2, keepdims=True)
    t[:, 9:18] = nrm.reshape(n, 9)
    mats = [api.Material(baseColor=(0.8, 0.3, 0.2), roughness=0.4).as_array(),
            api.Material(baseColor=(0.2, 0.6, 0.9), metallic=0.8, roughness=0.2, clearcoat=1.0).as_array(),
            api.Material(emissive=(4, 3, 2)).as_array()]
    for k in range(3):
        t[k::3, 18:] = mats[k]
    return t


@pytest.mark.parametrize("policy", [api.TRAVERSE_ACCEL, api.TRAVERSE_PRUNED, api.TRAVERSE_REFERENCE])
def test_triangle_soup_with_degenerate_geometry(oracle, policy):
    tl = api.TriangleList()
    tl.append_encoded(_soup(3000, 4))
    tris, nodes = tl.build_bvh(8)
    sc = api.Scene(tris, nodes)
    try:
        o, d = _random_rays(30000, 17, extent=2.5)
        o[:200] = np.round(o[:200], 1)  # origins on the rounded coordinate planes
        got = sc.trace_rays(o, d, traverse=policy)
        ref = oracle.trace_rays(tris, nodes, o, d, traverse=api.TRAVERSE_REFERENCE)
        assert ref["hit"].sum() > 5000
        np.testing.assert_array_equal(got["triangle"], ref["triangle"])
        assert_same_bits(got["distance"], ref["distance"], "soup distance")
        assert_same_bits(got["normal"], ref["normal"], "soup normal")
        eye, cam = api.camera_orbit(30.0, 20.0, 6.0)
        cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_ANISO_P4, max_bounce=3, width=64, height=48, spp=2, traverse=policy)
        ref_img, rc = oracle.render(tris, nodes, cfg)
        assert_same_bits(sc.render(cfg), ref_img, "soup image")
        assert sc.counters().rays == rc["rays"]
    finally:
        sc.close()


def test_p5_style_scene_with_huge_floor(oracle, small_hdr):
    """P5's own set-up scales the floor by 13000 (P5/main.cpp:818-819): the INF = 114514 sentinel turns the upper
    tree levels into median splits and the scene extent (hence the pruning slack) is huge."""
    hdr, cache = small_hdr
    tl = api.TriangleList()
    m = api.Material(baseColor=(1, 0.73, 0.25), roughness=0.5, specular=1.0, metallic=1.0, clearcoat=1.0, clearcoatGloss=0.0)
    tl.read_obj_text(scenes.blob_obj(3), m, api.transform_matrix((0, 0, 0), (0, -0.1, 0), (0.75, 0.75, 0.75)), True)
    m = api.Material(baseColor=(1, 1, 1), roughness=0.01, metallic=0.1, specular=1.0)
    tl.read_obj_text(scenes.box_obj(), m, api.transform_matrix((0, 0, 0), (0, -0.5, 0), (13000.0, 0.01, 13000.0)), False)
    tris, nodes = tl.build_bvh(8)
    eye, cam = api.camera_orbit(90.0, 10.0, 2.0)  # P5/main.cpp:796-798
    sc = api.Scene(tris, nodes, hdr, cache)
    try:
        for policy in (api.TRAVERSE_ACCEL, api.TRAVERSE_PRUNED):
            cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_IS_MIS_P5, max_bounce=2, width=72, height=48, spp=2, traverse=policy)
            ref, rc = oracle.render(tris, nodes, cfg, hdr=hdr, hdr_cache=cache)
            assert_same_bits(sc.render(cfg), ref, "P5-style scene, policy %d" % policy)
            c = sc.counters()
            assert (c.primary_rays, c.bounce_rays, c.shadow_rays) == (rc["rays_primary"], rc["rays_bounce"], rc["rays_shadow"])
    finally:
        sc.close()


@pytest.mark.parametrize("policy", [api.TRAVERSE_ACCEL, api.TRAVERSE_PRUNED])
def test_irregular_caller_tree_is_walked_literally(oracle, bunny_scene, policy):
    """A caller-supplied tree whose leaf boxes do not bound their triangles (here: every leaf box shrunk) defeats
    the assumptions of the accel/pruned policies; the library must then reproduce the shader's literal walk."""
    tris, nodes, eye, cam = bunny_scene
    bad = nodes.copy()
    leaf = bad[:, 3] > 0
    leaf[0] = False
    centre = 0.5 * (bad[leaf, 6:9] + bad[leaf, 9:12])
    bad[leaf, 6:9] = centre + 0.6 * (bad[leaf, 6:9] - centre)
    bad[leaf, 9:12] = centre + 0.6 * (bad[leaf, 9:12] - centre)
    sc = api.Scene(tris, bad)
    try:
        cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5, width=64, height=48, spp=2, traverse=policy)
        ref, rc = oracle.render(tris, bad, _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5, width=64, height=48, spp=2, traverse=api.TRAVERSE_REFERENCE))
        good, _ = oracle.render(tris, nodes, cfg)
        assert ref.tobytes() != good.tobytes()  # the shrunk boxes really change what the shader sees
        assert_same_bits(sc.render(cfg), ref, "irregular tree")
        assert sc.counters().rays == rc["rays"]
    finally:
        sc.close()


# ------------------------------------------------------------------ BASELINE.json's full-size configuration
def test_c3_full_size_scene_matches_oracle_and_policies_agree(oracle):
    """The 999,692-triangle scene of configs[2] (C3) itself: (i) a small image of it against the CPU oracle, bit for
    bit, in the Sobol and the IS/MIS mode; (ii) the full 1920x1080 frame under the three traversal policies --
    identical bits (a checksum of checksums over rows) and identical ray counts; (iii) 2 x 1 spp == 1 x 2 spp."""
    import zlib
    tris, nodes, eye, cam = scenes.s_1m()
    hdr = scenes.synth_hdr(256, 128)
    cache = api.hdr_cache(hdr)
    sc = api.Scene(tris, nodes, hdr, cache)
    try:
        for mode in (api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5):
            cfg = _cfg(eye, cam, mode=mode, max_bounce=2, width=96, height=54, spp=2)
            ref, rc = oracle.render(tris, nodes, cfg, hdr=hdr, hdr_cache=cache)
            got = sc.render(cfg)
            assert_same_bits(got, ref, "1M-triangle scene, mode %d" % mode)
            assert sc.counters().rays == rc["rays"]
        sums, rays = [], []
        for policy in (api.TRAVERSE_ACCEL, api.TRAVERSE_PRUNED, api.TRAVERSE_REFERENCE):
            cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5, max_bounce=2, width=1920, height=1080, spp=1, traverse=policy)
            img = sc.render(cfg)
            assert np.isfinite(img).all()
            sums.append(zlib.crc32(np.array([zlib.crc32(np.ascontiguousarray(row).tobytes()) for row in img], np.uint32).tobytes()))
            rays.append(sc.counters().rays)
            if policy == api.TRAVERSE_ACCEL:
                first = img
                c = sc.counters()
                assert c.deferred_rays < 0.01 * c.rays, "the accel policy defers only ties / unreachable leaves"
        assert sums[0] == sums[1] == sums[2] and rays[0] == rays[1] == rays[2]
        # accumulation: frame 0 then frame 1 on top == two frames at once
        cfg2 = _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5, max_bounce=2, width=1920, height=1080, spp=2)
        both = sc.render(cfg2)
        cfg1 = _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5, max_bounce=2, width=1920, height=1080, spp=1, first_frame=1)
        step = sc.render(cfg1, framebuffer=first.reshape(-1, 3).copy())
        assert_same_bits(step, both, "frame-by-frame accumulation at full size")
    finally:
        sc.close()
