"""The indexed triangle records of the 8-wide (W8) traversal: 32 bytes per triangle, (N, d0) (i1, i2, i3, 0), plus a 16-byte array
of the distinct vertex positions, chosen by ezrt_scene_create for W8 scenes where 32 T + 16 V < 64 T (capi.cu), the flat 64-byte
record otherwise.  Every reader (the cooperative triangle step of extend_w8 for camera, bounce and shadow rays, surface_hit in
k_shade, the feature-buffer path and the deferred lane, and k_trace_finish) must give the oracle's bits in both layouts.

The layout a scene got is read from the EZRT_VERBOSE=1 report of ezrt_scene_create."""
import re

import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests.test_gpu_parity import assert_same_bits
from tests.test_gpu_w8 import (W8_MIN_TRIANGLES, _assert_rays_match, _assert_renders_match, _assert_w8_ran, _bvh, _cfg, far_rays, far_scene,
                               grid_rays, soup_scene, stack_rays, stack_scene, twin_scene)

pytestmark = pytest.mark.gpu

LAYOUT = re.compile(r"triangle records: (indexed|flat) \((\d+) triangles, (\d+) distinct vertices\)")


def _scene(tris, nodes, capfd, monkeypatch, hdr=(None, None)):
    """The scene and the layout ezrt_scene_create reported for it: (scene, layout, distinct vertices)."""
    monkeypatch.setenv("EZRT_VERBOSE", "1")
    capfd.readouterr()
    sc = api.Scene(tris, nodes, *hdr)
    monkeypatch.delenv("EZRT_VERBOSE")
    m = LAYOUT.findall(capfd.readouterr().err)
    assert len(m) == 1, "no layout report"
    layout, n, v = m[0][0], int(m[0][1]), int(m[0][2])
    assert n == len(tris)
    assert layout == ("indexed" if 32 * n + 16 * v < 64 * n else "flat")
    return sc, layout, v


def _distinct_positions(tris):
    """Distinct (x, y, z) bit patterns among all vertices (the order does not change the count)."""
    return len(np.unique(np.ascontiguousarray(tris[:, :9]).view(np.uint32).reshape(-1, 3), axis=0))


def signed_zero_scene():
    """A blob grid whose vertices lie on the coordinate planes (x, y or z exactly 0), copied with every 0 written as -0.0: the two
    copies have equal coordinates but different bits, so they keep separate vertices (and still index well)."""
    tris, _, eye, cam = scenes.s_grid(4, 2, 2)
    v = tris[:, :9].reshape(-1, 3, 3)
    v = np.where(np.abs(v) < 0.1, np.float32(0.0), v)          # put many vertices onto the planes
    neg = np.where(v == 0, np.float32(-0.0), v)
    a, b = tris.copy(), tris.copy()
    a[:, :9] = v.reshape(-1, 9)
    b[:, :9] = neg.reshape(-1, 9)
    b[:, 21:24] = [0.2, 0.7, 0.3]
    t, nodes = _bvh(np.concatenate([a, b]))
    return t, nodes, eye, cam


def test_indexed_twins_and_coincident_stacks(oracle, small_hdr, capfd, monkeypatch):
    for name, (tris, nodes, eye, cam), rays, min_hits in [
            ("twins", twin_scene(), lambda t: grid_rays(20000, 31, 2.5), 3000),
            ("coincident stacks", stack_scene(0, 40), lambda t: stack_rays(t, 600, 7), 18000)]:
        assert len(tris) >= W8_MIN_TRIANGLES
        sc, layout, v = _scene(tris, nodes, capfd, monkeypatch, small_hdr)
        try:
            assert layout == "indexed", name
            assert v == _distinct_positions(tris), name
            o, d = rays(tris)
            _assert_rays_match(oracle, sc, tris, nodes, o, d, name, min_hits)
            for mode in (api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5):
                cfg = _cfg(eye, cam, mode=mode)
                _assert_renders_match(oracle, sc, tris, nodes, cfg, "%s, mode %d" % (name, mode), small_hdr)
            _assert_w8_ran(sc, cfg, 1.0)
        finally:
            sc.close()


def test_flat_ulp_stacks_and_soup(oracle, small_hdr, capfd, monkeypatch):
    """Stacks whose layers lie 1 to 3 ulps apart share no vertex, and neither does the soup: both keep the flat record."""
    for name, (tris, nodes, eye, cam), rays, min_hits, hdr in [
            ("ulp-spaced stacks", stack_scene(3, 43), lambda t: stack_rays(t, 600, 10), 18000, small_hdr),
            ("soup", soup_scene(), lambda t: grid_rays(30000, 17, 2.5), 5000, (None, None))]:
        sc, layout, v = _scene(tris, nodes, capfd, monkeypatch, hdr)
        try:
            assert layout == "flat", name
            o, d = rays(tris)
            _assert_rays_match(oracle, sc, tris, nodes, o, d, name, min_hits)
            cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_IS_MIS_P5 if hdr[0] is not None else api.MODE_DISNEY_ANISO_P4)
            _assert_renders_match(oracle, sc, tris, nodes, cfg, name, hdr if hdr[0] is not None else None)
        finally:
            sc.close()


def test_indexed_signed_zeros(oracle, small_hdr, capfd, monkeypatch):
    tris, nodes, eye, cam = signed_zero_scene()
    bits = tris[:, :9].view(np.uint32)
    assert (bits == 0x80000000).sum() > 500 and (bits == 0).sum() > 500
    sc, layout, v = _scene(tris, nodes, capfd, monkeypatch, small_hdr)
    try:
        assert layout == "indexed"
        assert v == _distinct_positions(tris)
        vals = np.unique(tris[:, :9].astype(np.float64).reshape(-1, 3), axis=0)   # +0 == -0 as values
        assert v > len(vals)
        o, d = grid_rays(20000, 5, 2.5)
        _assert_rays_match(oracle, sc, tris, nodes, o, d, "signed zeros", 3000)
        for mode in (api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5):
            _assert_renders_match(oracle, sc, tris, nodes, _cfg(eye, cam, mode=mode), "signed zeros, mode %d" % mode, small_hdr)
    finally:
        sc.close()


def test_indexed_wide_scene(oracle, capfd, monkeypatch):
    tris, nodes, eye, cam = far_scene(1e8, 6)
    sc, layout, _ = _scene(tris, nodes, capfd, monkeypatch)
    try:
        assert layout == "indexed"
        o, d = far_rays(tris, 6000, 3)
        _assert_rays_match(oracle, sc, tris, nodes, o, d, "scene 1e8 wide", 800)
        _assert_renders_match(oracle, sc, tris, nodes, _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5), "scene 1e8 wide")
    finally:
        sc.close()


@pytest.fixture(scope="module")
def s1m_scene():
    tris, nodes, eye, cam = scenes.s_1m_bunny()
    hdr = scenes.synth_hdr(256, 128)
    cache = api.hdr_cache(hdr)
    return dict(tris=tris, nodes=nodes, eye=eye, cam=cam, hdr=hdr, cache=cache)


def test_s1m_indexed_all_modes_aov_and_deferred_lane(oracle, s1m_scene, capfd, monkeypatch):
    """bench.py's 1 M-triangle scene: indexed; windows of its 1920x1080 grid in all four modes, the feature-buffer render, and the
    deferred lane on and off, all with the oracle's bits."""
    from tests import oracle_aov
    s = s1m_scene
    tris, nodes = s["tris"], s["nodes"]
    for lane in ("1", "0"):
        monkeypatch.setenv("EZRT_DEFERRED_LANE", lane)
        sc, layout, v = _scene(tris, nodes, capfd, monkeypatch, (s["hdr"], s["cache"]))
        try:
            assert layout == "indexed" and v < 0.51 * len(tris)   # 503,759 distinct positions
            for mode in (api.MODE_DIFFUSE_P3, api.MODE_DISNEY_ANISO_P4, api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5):
                cfg = api.RenderConfig(width=1920, height=1080, spp=2, max_bounce=2, mode=mode, eye=tuple(s["eye"]), camera_rotate=tuple(s["cam"]))
                img = sc.render(cfg)
                for win in [(928, 528, 992, 576)] if lane == "0" else [(0, 0, 48, 32), (928, 528, 992, 576), (1872, 1048, 1920, 1080)]:
                    ref, _ = oracle.render(tris, nodes, cfg, hdr=s["hdr"], hdr_cache=s["cache"], window=win)
                    x0, y0, x1, y1 = win
                    assert_same_bits(img[y0:y1, x0:x1], ref, "S-1M mode %d window %s lane %s" % (mode, win, lane))
            cfg = api.RenderConfig(width=1920, height=1080, spp=2, max_bounce=2, mode=api.MODE_DISNEY_IS_MIS_P5, eye=tuple(s["eye"]),
                                   camera_rotate=tuple(s["cam"]))
            img, aov, luma2 = sc.render_aov(cfg)
            win = (928, 528, 992, 576)
            ref, raov, rl2, _ = oracle_aov.render_aov(tris, nodes, cfg, hdr=s["hdr"], hdr_cache=s["cache"], window=win)
            x0, y0, x1, y1 = win
            assert_same_bits(img[y0:y1, x0:x1], ref, "S-1M aov image")
            assert_same_bits(aov[y0:y1, x0:x1], raov, "S-1M aov features")
            assert_same_bits(luma2[y0:y1, x0:x1], rl2, "S-1M aov luma2")
        finally:
            sc.close()
