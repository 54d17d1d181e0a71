"""The refill and ray-end paths of the 8-wide bounce and shadow kernels (extend_w8: k_extend_w8 through trace_rays, k_shadow_w8
through occluded_rays) at queue lengths around their edges, ray by ray against the oracle.

A finished ray's leaf check runs at the next refill of its warp, and the kernel's last refill finishes every ray still waiting.  So
the queue lengths are 1, 31, 33 (a warp's first chunk partly used) and one warp chunk either side of the grid's thread count (the
last chunks claimed by some warps but not others); length 0 returns on the host without a launch.  The rays the kernel hands to the
exact kernel lie at the end of the queue, in its last chunk: at refill, the far scene's directions and origins beyond the decode
bound; at ray end, the twin scene's hits, which all tie with their twins.  The far scene's other rays are hits without a tie, which
take the deferred leaf-box check (reference_reaches_leaf_box on the leaf index loaded at the ray's end) in both kernels; the twin
scene's hits take it in the shadow kernel, where a tie does not defer.

The phase-cycle sums of the counting instantiation (ezrt_get_w8_phase_cycles) are checked on a render with shadow rays."""
import numpy as np
import pytest

from ezrt_b200 import api
from tests import oracle_lights as ol
from tests import test_gpu_w8 as w8
from tests.test_gpu_parity import assert_same_bits

pytestmark = pytest.mark.gpu

CHUNK = 32   # SceneDev::work_chunk: rays a warp claims at once


def _grid_threads():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 1024   # persistent_blocks: one 1024-thread block per SM


def _queue(o, d, hostile, n):
    """n rays: the plain rays cycled, then the hostile ones last (as many as fit)."""
    k = min(n, int(hostile.sum()))
    plain = np.flatnonzero(~hostile)
    idx = np.concatenate([np.resize(plain, n - k), np.flatnonzero(hostile)[:k]]).astype(np.int64)
    return o[idx], d[idx]


def _aimed_rays(n, seed):
    """Rays from 3 units out towards points within 0.8 of the origin, where the far scene's first blob lies."""
    rng = np.random.default_rng(seed)
    o = rng.normal(size=(n, 3))
    o *= 3.0 / np.linalg.norm(o, axis=1, keepdims=True)
    d = rng.uniform(-0.8, 0.8, (n, 3)) - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return o.astype(np.float32), d.astype(np.float32)


def _scenes():
    tris, nodes, _, _ = w8.twin_scene()
    o, d = w8.grid_rays(8192, 41, 2.5)
    yield "twins", tris, nodes, o, d, None          # hostile = hits (every hit ties with its twin: the bounce kernel defers it at ray end)
    tris, nodes, _, _ = w8.far_scene(1.0e8, 6)
    o, d = _aimed_rays(4096, 43)
    fo, fd = w8.far_rays(tris, 1024, 43)   # components down to 2^-95, origins far out: beyond the decode bound
    hostile = np.arange(len(o) + len(fo)) >= len(o)
    yield "1e8 wide", tris, nodes, np.concatenate([o, fo]), np.concatenate([d, fd]), hostile


@pytest.mark.parametrize("lengths", ["small", "grid"])
def test_w8_queue_edges_ray_by_ray(oracle, lengths):
    g = _grid_threads()
    ns = [0, 1, 31, 33] if lengths == "small" else [g - CHUNK, g + CHUNK]   # 0: the API's edge (no launch)
    for name, tris, nodes, o_all, d_all, hostile in _scenes():
        if hostile is None:
            hostile = oracle.trace_rays(tris, nodes, o_all, d_all, traverse=api.TRAVERSE_REFERENCE)["hit"] != 0
        assert hostile.sum() >= 64 and (~hostile).sum() >= 64, name
        if name == "1e8 wide":   # the plain rays are hits without a tie: the leaf-box check at the refill decides them
            plain = ~hostile
            assert (oracle.trace_rays(tris, nodes, o_all[plain], d_all[plain], traverse=api.TRAVERSE_REFERENCE)["hit"] != 0).sum() >= 1500
        sc = api.Scene(tris, nodes)
        try:
            for n in ns:
                o, d = _queue(o_all, d_all, hostile, n)
                what = "%s, %d rays" % (name, n)
                got = sc.trace_rays(o, d, traverse=api.TRAVERSE_ACCEL)
                ref = oracle.trace_rays(tris, nodes, o, d, traverse=api.TRAVERSE_REFERENCE)
                for k in ("hit", "triangle", "inside"):
                    bad = np.flatnonzero(got[k] != ref[k])
                    assert bad.size == 0, "%s: %s differs on %d rays (first %d)" % (what, k, bad.size, bad[0])
                for k in ("distance", "point", "normal"):
                    assert_same_bits(got[k], ref[k], "%s %s" % (what, k))
                if n == 0:
                    continue
                # shadow rays: bounded below, at and above the closest hit, and unbounded
                t = np.where(ref["hit"] != 0, ref["distance"], 10.0).astype(np.float32)
                rng = np.random.default_rng(n)
                tmax = np.choose(rng.integers(0, 3, n), [t * 0.5, t, np.nextafter(t, np.float32(np.inf))]).astype(np.float32)
                for bound in (tmax, np.full(n, np.inf, np.float32)):
                    lit = sc.occluded_rays(o, d, bound, traverse=api.TRAVERSE_ACCEL)
                    want = ol.oracle_occluded(tris, nodes, o, d, bound, traverse=api.TRAVERSE_ACCEL)
                    bad = np.flatnonzero(lit != want)
                    assert bad.size == 0, "%s, shadow: %d rays differ (first %d)" % (what, bad.size, bad[0])
        finally:
            sc.close()


def test_w8_phase_cycles(small_hdr):
    """profile = 2 fills the bounce and shadow kernels' four phase sums; a plain render leaves them all zero."""
    tris, nodes, eye, cam = w8.huge_floor_scene()
    sc = api.Scene(tris, nodes, *small_hdr)
    try:
        cfg = api.RenderConfig(width=72, height=48, spp=2, max_bounce=2, eye=tuple(eye), camera_rotate=tuple(cam), env_color=(0.35, 0.45, 0.6),
                               mode=api.MODE_DISNEY_IS_MIS_P5, profile=2)
        sc.render(cfg)
        c = sc.counters()
        assert c.bounce_rays > 0 and c.shadow_rays > 2000 and c.node_visits_96 > 0
        cyc = sc.w8_phase_cycles()
        for kernel in ("k_extend_w8", "k_shadow_w8"):
            assert all(v > 0 for v in cyc[kernel].values()), (kernel, cyc)
        sc.render(api.RenderConfig(**{**cfg.__dict__, "profile": 0}))
        cyc = sc.w8_phase_cycles()
        assert all(v == 0 for k in cyc for v in cyc[k].values()), cyc
    finally:
        sc.close()
