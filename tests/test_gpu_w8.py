"""The 8-wide quantised traversal ("W8": extend_w8 in ezrt_b200/csrc/device_functions.cuh, run by k_extend_w8,
k_extend_w8_camera and k_shadow_w8) against the CPU oracle, ray by ray and image by image.

Every scene has at least 2^16 triangles, so the size rule of ezrt_scene_create selects the W8 tree by itself.  The scenes are
built to load the warp-cooperative triangle step: twins and coincident stacks (ties), stacks of 1..63 triangles hit by
bundles of 32 nearly identical rays (more than 32 pending pairs per warp, owners split across steps, full 32-triangle
masks), parallel stacks a few ulps apart in shuffled order (the closest hit anywhere in an owner's run), a degenerate soup,
a huge floor under many small triangles (shadow rays through k_shadow_w8), and a scene 10^8 wide walked with directions
down to 2^-95 (the decode range of the quantised nodes).  tests/test_w8_tree.py runs the same scenes and rays through the
CPU model of the traversal and checks that they really produce those pile-ups."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes

pytestmark = pytest.mark.gpu

W8_MIN_TRIANGLES = 1 << 16     # capi.cu: scenes from this size on walk the W8 tree
DEPTHS = np.array([1, 2, 3, 5, 7, 13, 21, 29, 33, 35, 37, 39, 41, 45, 47, 63])   # no multiple of 4 or 32
STACK_Z = 0.25                  # plane of the stacks; parallel copies lie 2^-23 apart (one ulp of t for rays from z = 1.5)


def _bvh(tris):
    tl = api.TriangleList()
    tl.append_encoded(np.ascontiguousarray(tris, np.float32))
    return tl.build_bvh(8)


def _mesh_bvh(meshes):
    tl = api.TriangleList()
    for text, m, trans, smooth in meshes:
        tl.read_obj_text(text, m, trans, smooth)
    return tl.build_bvh(8)


def regular_tree(tris, nodes):
    """The checks ezrt_scene_create makes before it lets the accel policy walk a caller's tree (capi.cu): every triangle in
    exactly one leaf, leaf boxes bound their triangles, child boxes lie inside their parent's."""
    left, right, n, first = (nodes[:, k].astype(np.int64) for k in (0, 1, 3, 4))
    lo, hi = nodes[:, 6:9], nodes[:, 9:12]
    leaf = n > 0
    leaf[0] = False
    cover = np.zeros(len(tris), np.int64)
    v = tris[:, :9].reshape(-1, 3, 3)
    for i in np.flatnonzero(leaf):
        cover[first[i]:first[i] + n[i]] += 1
        p = v[first[i]:first[i] + n[i]]
        if not ((p >= lo[i]).all() and (p <= hi[i]).all()):
            return False
    inner = np.flatnonzero(~leaf)[1:]
    for c in (left[inner], right[inner]):
        if not ((lo[c] >= lo[inner]).all() and (hi[c] <= hi[inner]).all()):
            return False
    return bool((cover == 1).all())


# ------------------------------------------------------------------ scenes (plain numpy / host builders: no GPU needed)
def twin_scene():
    """Every triangle of a 4 x 2 blob grid twice, the copy with another base colour; half of the copies come before their
    originals in the input.  Every hit ties with its twin."""
    tris, _, eye, cam = scenes.s_grid(4, 2, 2)
    twin = tris.copy()
    twin[:, 21:24] = [0.9, 0.2, 0.1]
    t, nodes = _bvh(np.concatenate([twin[0::2], tris, twin[1::2]]))
    return t, nodes, eye, cam


def stack_scene(ulps, seed):
    """A 52 x 52 grid of stacks of DEPTHS triangles in the plane z = STACK_Z, facing +z, every layer with another material.
    ulps = 0: the layers of a stack coincide.  ulps > 0: layer k lies at STACK_Z + (pi(k) * s) * 2^-23 for a random
    permutation pi and a per-stack spacing s in 1..ulps.  All triangles in shuffled order."""
    rng = np.random.default_rng(seed)
    g, cell = 52, 0.1
    depth = rng.choice(DEPTHS, g * g)
    mats = np.stack([m.as_array() for m in scenes.MATERIAL_PRESETS])
    out = []
    for s in range(g * g):
        x0, y0 = (s % g - g / 2) * cell, (s // g - g / 2) * cell
        a, b = 0.05 + 0.03 * rng.random(2)
        base = np.array([x0, y0, 0, x0 + a, y0 + 0.01 * rng.random(), 0, x0 + 0.01 * rng.random(), y0 + b, 0], np.float64)
        d = int(depth[s])
        t = np.zeros((d, 36), np.float32)
        t[:, :9] = base
        z = np.full(d, STACK_Z)
        if ulps:
            z = STACK_Z + rng.permutation(d) * int(rng.integers(1, ulps + 1)) * 2.0 ** -23
        t[:, 2:9:3] = z[:, None]
        t[:, 9:18] = [0, 0, 1] * 3
        t[:, 18:] = mats[(s + np.arange(d)) % 8]
        out.append(t)
    tris = np.concatenate(out)
    tris = tris[rng.permutation(len(tris))]
    assert len(tris) >= W8_MIN_TRIANGLES
    t, nodes = _bvh(tris)
    eye, cam = api.camera_orbit(0.0, 0.0, 4.5)
    return t, nodes, eye, cam


def stack_rays(tris, n_bundles, seed):
    """Bundles of 32 consecutive rays (one warp's chunk of the ray queue) that leave z = 1.5 downwards, nearly parallel, aimed at
    one point of one stack (every other bundle at a stack deeper than 32), then random rays over the whole grid."""
    rng = np.random.default_rng(seed)
    _, stack, depth = np.unique(tris[:, 0:2], axis=0, return_inverse=True, return_counts=True)   # p1.xy identifies a stack
    deep = np.flatnonzero(depth[stack.ravel()] > 32)
    pick = np.where(np.arange(n_bundles) % 2 == 0, rng.choice(deep, n_bundles), rng.integers(0, len(tris), n_bundles))
    v = tris[pick, :9].reshape(-1, 3, 3).astype(np.float64)
    w = rng.dirichlet((4, 4, 4), n_bundles)
    aim = (v * w[:, :, None]).sum(1)
    tilt = rng.normal(scale=0.02, size=(n_bundles, 1, 2))
    o = np.repeat(aim[:, None, :], 32, 1)
    o[:, :, 2] = 1.5
    o[:, :, :2] += rng.normal(scale=2e-5, size=(n_bundles, 32, 2)) - 1.25 * tilt
    d = np.zeros((n_bundles, 32, 3))
    d[:, :, :2] = tilt + rng.normal(scale=1e-6, size=(n_bundles, 32, 2))
    d[:, :, 2] = -1.0
    o, d = o.reshape(-1, 3), d.reshape(-1, 3)
    m = 4096
    o2 = np.column_stack([rng.uniform(-2.7, 2.7, (m, 2)), np.full(m, 1.5)])
    d2 = np.column_stack([rng.normal(scale=0.3, size=(m, 2)), -np.ones(m)])
    o, d = np.concatenate([o, o2]), np.concatenate([d, d2])
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return o.astype(np.float32), d.astype(np.float32)


def soup_scene():
    from tests.test_gpu_parity import _soup
    t, nodes = _bvh(_soup(70000, 4))
    eye, cam = api.camera_orbit(30.0, 20.0, 6.0)
    return t, nodes, eye, cam


def huge_floor_scene():
    """P5's set-up (floor scaled by 13000, P5/main.cpp:818-819) with an 81,920-triangle blob."""
    m = api.Material(baseColor=(1, 0.73, 0.25), roughness=0.5, specular=1.0, metallic=1.0, clearcoat=1.0, clearcoatGloss=0.0)
    f = api.Material(baseColor=(1, 1, 1), roughness=0.01, metallic=0.1, specular=1.0)
    t, nodes = _mesh_bvh([(scenes.blob_obj(6), m, api.transform_matrix((0, 0, 0), (0, -0.1, 0), (0.75, 0.75, 0.75)), True),
                          (scenes.box_obj(), f, api.transform_matrix((0, 0, 0), (0, -0.5, 0), (13000.0, 0.01, 13000.0)), False)])
    eye, cam = api.camera_orbit(90.0, 10.0, 2.0)
    return t, nodes, eye, cam


def far_scene(shift, subdiv):
    """A blob at the origin and a copy `shift` away along x: the largest node scale grows with `shift`, and with it the
    decode's 2^15 * scale * |1/d| (W8; 2^23 for the Q16 nodes of the 4-wide form)."""
    m = api.Material(baseColor=(0.8, 0.8, 0.8), roughness=0.4)
    c = api.Material(baseColor=(0.2, 0.5, 0.9), roughness=0.4)
    t, nodes = _mesh_bvh([(scenes.blob_obj(subdiv), m, api.transform_matrix((0, 0, 0), (0, 0, 0), (1.5, 1.5, 1.5)), True),
                          (scenes.blob_obj(subdiv), c, api.transform_matrix((0, 0, 0), (shift, 0, 0), (1.5, 1.5, 1.5)), True)])
    eye, cam = api.camera_orbit(20.0, 10.0, 3.5)
    return t, nodes, eye, cam


FAR_COMPONENTS = np.array([2.0 ** -95, 2.0 ** -90, 2.0 ** -60, 0.0])


def far_rays(tris, n, seed):
    """Rays towards the blob at the origin from 3 units away (hits well within the reference's INF = 114514): the main axis
    component is about +-1, the other two are +-2^-95, +-2^-90, +-2^-60 or 0.  Then rays that start 3.9 and 4.1 times
    max|coordinate| out on the x axis (either side of W8_ORIGIN_LIMIT_REL) and look back at the scene."""
    rng = np.random.default_rng(seed)
    axis = rng.integers(0, 3, n)
    sign = rng.choice([-1.0, 1.0], n)
    d = rng.choice(FAR_COMPONENTS, (n, 3)) * rng.choice([-1.0, 1.0], (n, 3))
    d[np.arange(n), axis] = sign * (1.0 - rng.uniform(0, 1e-3, n))
    o = rng.uniform(-1.2, 1.2, (n, 3))
    o[np.arange(n), axis] = -3.0 * sign
    maxc = float(np.abs(tris[:, :9]).max())
    k = 256
    o2 = np.zeros((k, 3))
    o2[:, 0] = np.where(np.arange(k) % 2 == 0, 3.9, 4.1) * maxc * np.where(np.arange(k) % 4 < 2, 1.0, -1.0)
    o2[:, 1:] = rng.uniform(-1, 1, (k, 2))
    d2 = rng.choice(FAR_COMPONENTS[:3], (k, 3)) * rng.choice([-1.0, 1.0], (k, 3))
    d2[:, 0] = -np.sign(o2[:, 0])
    return np.concatenate([o, o2]).astype(np.float32), np.concatenate([d, d2]).astype(np.float32)


def grid_rays(n, seed, extent):
    from tests.test_gpu_parity import _random_rays
    return _random_rays(n, seed, extent=extent)


# ------------------------------------------------------------------ checks
def _assert_rays_match(oracle, sc, tris, nodes, o, d, what, min_hits):
    from tests.test_gpu_parity import assert_same_bits
    got = sc.trace_rays(o, d, traverse=api.TRAVERSE_ACCEL)
    ref = oracle.trace_rays(tris, nodes, o, d, traverse=api.TRAVERSE_REFERENCE)
    assert ref["hit"].sum() >= min_hits, what
    for k in ("hit", "triangle", "inside"):
        bad = np.flatnonzero(got[k] != ref[k])
        assert bad.size == 0, "%s: %s differs on %d of %d rays (first ray %d: %r vs %r)" % (what, k, bad.size, len(o), bad[0], got[k][bad[0]], ref[k][bad[0]])
    for k in ("distance", "point", "normal"):
        assert_same_bits(got[k], ref[k], "%s %s" % (what, k))
    return ref


def _assert_renders_match(oracle, sc, tris, nodes, cfg, what, hdr=None):
    from tests.test_gpu_parity import assert_same_bits
    h, cache = (None, None) if hdr is None else hdr
    ref, rc = oracle.render(tris, nodes, cfg, hdr=h, hdr_cache=cache)
    assert_same_bits(sc.render(cfg), ref, what)
    c = sc.counters()
    assert (c.primary_rays, c.bounce_rays, c.shadow_rays) == (rc["rays_primary"], rc["rays_bounce"], rc["rays_shadow"]), what
    return c


def _assert_w8_ran(sc, cfg, max_deferred):
    """The counting render (profile = 2) shows quantised node visits, and the accel kernels deferred at most the given share of
    the rays to the exact kernel."""
    p = api.RenderConfig(**{**cfg.__dict__, "profile": 2})
    sc.render(p)
    c = sc.counters()
    assert c.node_visits_96 > 0 and c.tri_tests > 0
    assert c.deferred_rays <= max_deferred * c.rays, (c.deferred_rays, c.rays)
    return c


def _cfg(eye, cam, **kw):
    base = dict(width=64, height=48, spp=2, max_bounce=2, eye=tuple(eye), camera_rotate=tuple(cam), env_color=(0.35, 0.45, 0.6))
    base.update(kw)
    return api.RenderConfig(**base)


def test_w8_twins_pick_the_reference_copy(oracle, small_hdr):
    tris, nodes, eye, cam = twin_scene()
    assert len(tris) >= W8_MIN_TRIANGLES
    sc = api.Scene(tris, nodes, *small_hdr)
    try:
        o, d = grid_rays(20000, 31, 2.5)
        _assert_rays_match(oracle, sc, tris, nodes, o, d, "twins", 3000)
        for mode in (api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5):
            cfg = _cfg(eye, cam, mode=mode)
            _assert_renders_match(oracle, sc, tris, nodes, cfg, "twins, mode %d" % mode, small_hdr)
        _assert_w8_ran(sc, cfg, 1.0)   # every hit ties: most rays go to the exact kernel by design
    finally:
        sc.close()


@pytest.mark.parametrize("ulps", [0, 3])
def test_w8_stacks_with_coherent_bundles(oracle, small_hdr, ulps):
    """ulps = 0: coincident stacks (ties inside a warp's step and across step boundaries); ulps = 3: parallel copies 1 to 3
    ulps of t apart in shuffled order (the closest hit first, last or inside an owner's run, in either part of a split)."""
    tris, nodes, eye, cam = stack_scene(ulps, 40 + ulps)
    sc = api.Scene(tris, nodes, *small_hdr)
    try:
        o, d = stack_rays(tris, 600, 7 + ulps)
        _assert_rays_match(oracle, sc, tris, nodes, o, d, "stacks (%d ulps)" % ulps, 18000)
        for mode in (api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5):
            cfg = _cfg(eye, cam, mode=mode, width=96, height=72)
            _assert_renders_match(oracle, sc, tris, nodes, cfg, "stacks (%d ulps), mode %d" % (ulps, mode), small_hdr)
        _assert_w8_ran(sc, cfg, 1.0 if ulps == 0 else 0.5)
    finally:
        sc.close()


def test_w8_degenerate_soup(oracle):
    tris, nodes, eye, cam = soup_scene()
    sc = api.Scene(tris, nodes)
    try:
        o, d = grid_rays(30000, 17, 2.5)
        o[:200] = np.round(o[:200], 1)
        _assert_rays_match(oracle, sc, tris, nodes, o, d, "soup", 5000)
        cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_ANISO_P4, max_bounce=3)
        _assert_renders_match(oracle, sc, tris, nodes, cfg, "soup")
        _assert_w8_ran(sc, cfg, 0.1)
    finally:
        sc.close()


def test_w8_huge_floor_with_shadow_rays(oracle, small_hdr):
    tris, nodes, eye, cam = huge_floor_scene()
    assert len(tris) >= W8_MIN_TRIANGLES
    sc = api.Scene(tris, nodes, *small_hdr)
    try:
        cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_IS_MIS_P5, width=72, height=48)
        c = _assert_renders_match(oracle, sc, tris, nodes, cfg, "P5-style scene with a fine blob", small_hdr)
        assert c.shadow_rays > 2000
        _assert_w8_ran(sc, cfg, 0.1)
        o, d = grid_rays(20000, 23, 1.2)
        _assert_rays_match(oracle, sc, tris, nodes, o, d, "huge floor", 3000)
    finally:
        sc.close()


@pytest.mark.parametrize("shift,subdiv", [(1e8, 6), (1e8, 4), (1e9, 6)])
def test_w8_and_q16_decode_range_on_wide_scenes(oracle, shift, subdiv):
    """subdiv 6: 163,840 triangles, the W8 tree; subdiv 4: 10,240 triangles, the Q16 nodes of the 4-wide form.  Before the
    decode range was derived per scene, rays with |1/d| up to 2^96 were walked on these trees and the decode overflowed:
    every hit of the 2^-95 rays was lost."""
    tris, nodes, eye, cam = far_scene(shift, subdiv)
    assert (len(tris) >= W8_MIN_TRIANGLES) == (subdiv == 6)
    assert regular_tree(tris, nodes)   # otherwise every policy walks the caller's tree and the test would prove nothing
    sc = api.Scene(tris, nodes)
    try:
        o, d = far_rays(tris, 6000, 3)
        ref = _assert_rays_match(oracle, sc, tris, nodes, o, d, "scene %g wide, subdiv %d" % (shift, subdiv), 800)
        tiny = (np.abs(d) == 2.0 ** -95).any(1) & (ref["hit"] == 1)
        assert tiny.sum() > 100
        cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5)
        _assert_renders_match(oracle, sc, tris, nodes, cfg, "scene %g wide" % shift)
        _assert_w8_ran(sc, cfg, 0.1)
    finally:
        sc.close()
