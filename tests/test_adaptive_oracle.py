"""Tile-adaptive sampling on the CPU: the oracle's restatement (tests/oracle_adaptive.cpp) against the plain oracle and
against a numpy float32 restatement of the criterion of include/ezrt_math.h.  The image (100x70) has clipped edge tiles."""
import numpy as np
import pytest

from ezrt_b200 import api
from tests import oracle_adaptive as oa

W, H, CAP, MIN_SPP, INTERVAL = 100, 70, 24, 4, 4
ENV = (0.35, 0.45, 0.6)
# thresholds at which the tiles of this view stop at several different test points
CASES = [(api.MODE_DIFFUSE_P3, 0.8), (api.MODE_DISNEY_IS_MIS_P5, 0.5)]


def _cfg(bunny_scene, mode, spp):
    _, _, eye, cam = bunny_scene
    return api.RenderConfig(width=W, height=H, spp=spp, max_bounce=2, mode=mode, eye=tuple(eye), camera_rotate=tuple(cam), env_color=ENV)


def _tiles(a):
    """the value at each tile's first pixel, [ty, tx]"""
    return a[::16, ::16]


@pytest.fixture(scope="module", params=CASES, ids=["mode%d" % m for m, _ in CASES])
def adaptive_case(request, bunny_scene, small_hdr):
    mode, thr = request.param
    tris, nodes, _, _ = bunny_scene
    hdr, cache = small_hdr
    img, spp, luma2, c = oa.render_adaptive(tris, nodes, _cfg(bunny_scene, mode, CAP), thr, MIN_SPP, INTERVAL, hdr=hdr, hdr_cache=cache)
    return dict(mode=mode, thr=thr, img=img, spp=spp, luma2=luma2, counters=c, tris=tris, nodes=nodes, hdr=hdr, cache=cache)


def test_spp_map_is_per_tile_and_on_the_test_grid(adaptive_case):
    spp = adaptive_case["spp"]
    grid = set(range(MIN_SPP, CAP, INTERVAL)) | {CAP}
    per_tile = _tiles(spp)
    assert set(np.unique(per_tile)) <= grid
    assert len(np.unique(per_tile)) >= 3, "the case should stop tiles at several test points"
    for ty in range(per_tile.shape[0]):
        for tx in range(per_tile.shape[1]):
            assert (spp[ty * 16:(ty + 1) * 16, tx * 16:(tx + 1) * 16] == per_tile[ty, tx]).all()
    assert adaptive_case["counters"]["samples"] == int(spp.sum())


def test_each_tile_equals_a_plain_render_at_its_spp(oracle, bunny_scene, adaptive_case):
    ac = adaptive_case
    per_tile = _tiles(ac["spp"])
    for n in np.unique(per_tile):
        ref, _ = oracle.render(ac["tris"], ac["nodes"], _cfg(bunny_scene, ac["mode"], int(n)), hdr=ac["hdr"], hdr_cache=ac["cache"])
        for ty, tx in zip(*np.nonzero(per_tile == n)):
            sl = (slice(ty * 16, (ty + 1) * 16), slice(tx * 16, (tx + 1) * 16))
            assert ac["img"][sl].tobytes() == ref[sl].tobytes(), "tile (%d, %d) at %d spp" % (tx, ty, n)


def test_numpy_criterion_reproduces_where_tiles_stopped(bunny_scene, adaptive_case):
    """At each test point t the state of every tile equals an adaptive render capped at t with min_spp = t (no test runs);
    the float32 criterion on that state says which tiles stop at t."""
    ac = adaptive_case
    expected = np.full(_tiles(ac["spp"]).shape, CAP, np.int32)
    for t in range(MIN_SPP, CAP, INTERVAL):
        img_t, spp_t, luma2_t, _ = oa.render_adaptive(ac["tris"], ac["nodes"], _cfg(bunny_scene, ac["mode"], t), ac["thr"], t, INTERVAL,
                                                       hdr=ac["hdr"], hdr_cache=ac["cache"])
        assert (spp_t == t).all()
        conv = oa.tile_converged(oa.adaptive_error(luma2_t, img_t, t), ac["thr"])
        expected = np.where((expected == CAP) & conv, t, expected)
        # the tiles that stopped at t hold exactly this state
        stopped = _tiles(ac["spp"]) == t
        for ty, tx in zip(*np.nonzero(stopped)):
            sl = (slice(ty * 16, (ty + 1) * 16), slice(tx * 16, (tx + 1) * 16))
            assert ac["luma2"][sl].tobytes() == luma2_t[sl].tobytes()
    np.testing.assert_array_equal(_tiles(ac["spp"]), expected)


def test_min_spp_equal_to_cap_is_the_plain_render(oracle, bunny_scene, small_hdr):
    tris, nodes, _, _ = bunny_scene
    hdr, cache = small_hdr
    cfg = _cfg(bunny_scene, api.MODE_DISNEY_SOBOL_P5, 6)
    img, spp, _, c = oa.render_adaptive(tris, nodes, cfg, 1e-9, 6, 1, hdr=hdr, hdr_cache=cache)
    ref, rc = oracle.render(tris, nodes, cfg, hdr=hdr, hdr_cache=cache)
    assert img.tobytes() == ref.tobytes() and (spp == 6).all() and c["rays"] == rc["rays"]


def test_criterion_edge_cases():
    """float32 restatement: black pixels with no variance converge, NaN fails, negative variance clamps to 0."""
    mean = np.zeros((1, 3, 3), np.float32)
    mean[0, 2] = 1.0
    luma2 = np.array([[0.0, np.nan, 0.999]], np.float32)
    err = oa.adaptive_error(luma2, mean, 8)
    assert err[0, 0] == 0.0 and np.isnan(err[0, 1]) and err[0, 2] == 0.0
    assert not oa.tile_converged(err, 1.0)[0, 0]
