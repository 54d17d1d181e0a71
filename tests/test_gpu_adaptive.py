"""Tile-adaptive sampling on the GPU (ezrt_render_adaptive): bit for bit against the CPU restatement
(tests/oracle_adaptive.cpp), and every tile equal to a plain GPU render at the frames it received."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_adaptive as oa
from tests.test_gpu_parity import assert_same_bits

pytestmark = pytest.mark.gpu

ENV = (0.35, 0.45, 0.6)
W, H, CAP, MIN_SPP, INTERVAL = 100, 70, 24, 4, 4
THRESHOLD = {api.MODE_DIFFUSE_P3: 0.8, api.MODE_DISNEY_ANISO_P4: 0.5, api.MODE_DISNEY_SOBOL_P5: 0.5, api.MODE_DISNEY_IS_MIS_P5: 0.5}


@pytest.fixture(scope="module")
def bunny(bunny_scene, small_hdr):
    tris, nodes, eye, cam = bunny_scene
    hdr, cache = small_hdr
    sc = api.Scene(tris, nodes, hdr, cache)
    yield dict(tris=tris, nodes=nodes, eye=eye, cam=cam, hdr=hdr, cache=cache, scene=sc)
    sc.close()


def _cfg(b, mode=api.MODE_DISNEY_IS_MIS_P5, spp=CAP, **kw):
    return api.RenderConfig(width=kw.pop("width", W), height=kw.pop("height", H), spp=spp, max_bounce=2, mode=mode, eye=tuple(b["eye"]),
                            camera_rotate=tuple(b["cam"]), env_color=ENV, **kw)


def _tiles(a):
    return a[::16, ::16]


@pytest.mark.parametrize("mode", sorted(THRESHOLD))
def test_bunny_matches_the_oracle(bunny, mode):
    thr = THRESHOLD[mode]
    cfg = _cfg(bunny, mode)
    img, spp, luma2 = bunny["scene"].render_adaptive(cfg, thr, MIN_SPP, INTERVAL)
    c = bunny["scene"].counters()
    ref, rspp, rluma2, rc = oa.render_adaptive(bunny["tris"], bunny["nodes"], cfg, thr, MIN_SPP, INTERVAL, hdr=bunny["hdr"], hdr_cache=bunny["cache"])
    np.testing.assert_array_equal(spp, rspp)
    assert_same_bits(img, ref, "mode %d framebuffer" % mode)
    assert_same_bits(luma2, rluma2, "mode %d luma2" % mode)
    assert c.rays == rc["rays"] and c.primary_rays == rc["rays_primary"]
    assert c.samples == int(spp.sum()) == rc["samples"]
    assert _tiles(spp).min() == MIN_SPP   # the sky tiles stop at the first test


def test_each_tile_equals_the_plain_gpu_render(bunny):
    cfg = _cfg(bunny)
    img, spp, _ = bunny["scene"].render_adaptive(cfg, THRESHOLD[cfg.mode], MIN_SPP, INTERVAL)
    per_tile = _tiles(spp)
    assert len(np.unique(per_tile)) >= 3
    for n in np.unique(per_tile):
        plain = bunny["scene"].render(_cfg(bunny, spp=int(n)))
        for ty, tx in zip(*np.nonzero(per_tile == n)):
            sl = (slice(ty * 16, (ty + 1) * 16), slice(tx * 16, (tx + 1) * 16))
            assert img[sl].tobytes() == plain[sl].tobytes(), "tile (%d, %d) at %d spp" % (tx, ty, n)


def test_min_spp_at_the_cap_and_a_huge_threshold(bunny):
    sc = bunny["scene"]
    plain = sc.render(_cfg(bunny, spp=6)).copy()
    rays = sc.counters().rays
    img, spp, _ = sc.render_adaptive(_cfg(bunny, spp=6), 1e-9, 6, 1)      # no test before the cap
    assert img.tobytes() == plain.tobytes() and (spp == 6).all() and sc.counters().rays == rays
    img, spp, _ = sc.render_adaptive(_cfg(bunny, spp=40), 3e38, 6, 5)      # every tile passes the first test
    assert img.tobytes() == plain.tobytes() and (spp == 6).all() and sc.counters().rays == rays


def _scatter(parts, channels):
    full = np.zeros((H, W, channels), np.float32)
    for rank, a in enumerate(parts):
        api.partition_scatter_host(np.ascontiguousarray(a, np.float32).reshape(-1, channels), full, W, H, channels, rank, len(parts))
    return full


def test_same_result_under_batch_sizes_policies_and_partitions(bunny):
    sc = bunny["scene"]
    thr = THRESHOLD[api.MODE_DISNEY_IS_MIS_P5]
    img, spp, luma2 = (a.copy() for a in sc.render_adaptive(_cfg(bunny), thr, MIN_SPP, INTERVAL))
    rays = sc.counters().rays
    variants = [dict(frames_per_batch=1), dict(frames_per_batch=3), dict(traverse=api.TRAVERSE_PRUNED), dict(traverse=api.TRAVERSE_REFERENCE),
                dict(out_channels=4)]
    for kw in variants:
        i2, s2, l2 = sc.render_adaptive(_cfg(bunny, **kw), thr, MIN_SPP, INTERVAL)
        assert i2[..., :3].tobytes() == img.tobytes() and s2.tobytes() == spp.tobytes() and l2.tobytes() == luma2.tobytes(), kw
        assert sc.counters().rays == rays, kw
    parts = [sc.render_adaptive(_cfg(bunny, part_rank=r, part_count=2), thr, MIN_SPP, INTERVAL) for r in range(2)]
    assert _scatter([p[0] for p in parts], 3).tobytes() == img.tobytes()
    assert _scatter([p[1].view(np.float32) for p in parts], 1)[..., 0].view(np.int32).tobytes() == spp.tobytes()
    assert _scatter([p[2] for p in parts], 1)[..., 0].tobytes() == luma2.tobytes()


def test_device_entry_point_and_profile_classes(bunny):
    import torch
    sc = bunny["scene"]
    thr = THRESHOLD[api.MODE_DISNEY_IS_MIS_P5]
    img, spp, luma2 = (a.copy() for a in sc.render_adaptive(_cfg(bunny), thr, MIN_SPP, INTERVAL))
    d_fb = torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")
    d_spp = torch.zeros(W * H, dtype=torch.int32, device="cuda")
    d_l2 = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    stream = torch.cuda.current_stream()
    sc.render_adaptive_device(_cfg(bunny, profile=1), thr, MIN_SPP, INTERVAL, d_fb, d_spp, d_l2, stream)
    torch.cuda.synchronize()
    assert d_fb.cpu().numpy().tobytes() == img.tobytes()
    assert d_spp.cpu().numpy().tobytes() == spp.tobytes() and d_l2.cpu().numpy().tobytes() == luma2.tobytes()
    kt = sc.kernel_times()
    n_tests = len(range(MIN_SPP, int(spp.max()), INTERVAL))
    assert kt["other"][1] >= n_tests and sc.counters().samples == int(spp.sum())


def test_invalid_inputs_are_rejected(bunny):
    sc = bunny["scene"]
    bad = [(_cfg(bunny), dict(threshold=float("nan"))), (_cfg(bunny), dict(threshold=float("inf"))), (_cfg(bunny), dict(threshold=0.0)),
           (_cfg(bunny), dict(threshold=-1.0)), (_cfg(bunny), dict(min_spp=1)), (_cfg(bunny), dict(check_interval=0)),
           (_cfg(bunny, first_frame=4), {}), (_cfg(bunny, pipeline=api.PIPELINE_MEGAKERNEL), {}), (_cfg(bunny), dict(reserved=1))]
    import ctypes as C
    import torch
    img = np.zeros(W * H * 4, np.float32); spp = np.zeros(W * H, np.int32); l2 = np.zeros(W * H, np.float32)
    d_fb = torch.zeros(W * H * 4, dtype=torch.float32, device="cuda")
    d_spp = torch.zeros(W * H, dtype=torch.int32, device="cuda")
    d_l2 = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    for cfg, over in bad:
        a = api.adaptive_params(0.5, MIN_SPP, INTERVAL)
        for k, v in over.items():
            setattr(a, k, v)
        p = cfg.to_struct()
        rc = api.lib.ezrt_render_adaptive(sc._h, C.byref(p), C.byref(a), api._fp(img), spp.ctypes.data_as(api._lib.c_int32_p), api._fp(l2))
        assert rc == -1, (over, cfg.first_frame, cfg.pipeline)
        assert api.lib.ezrt_last_error().decode().startswith("render_adaptive"), over
        rc = api.lib.ezrt_render_adaptive_device(sc._h, C.byref(p), C.byref(a), C.c_void_p(d_fb.data_ptr()), C.c_void_p(d_spp.data_ptr()),
                                                 C.c_void_p(d_l2.data_ptr()), None)
        assert rc == -1, over
    with pytest.raises(api.EzrtError):   # null output buffers
        sc.render_adaptive_device(_cfg(bunny), 0.5, MIN_SPP, INTERVAL, 0, 0, 0)


@pytest.fixture(scope="module")
def s1m():
    tris, nodes, eye, cam = scenes.s_1m_bunny()
    hdr = scenes.synth_hdr(2048, 1024)
    cache = api.hdr_cache_device(hdr)[0]
    sc = api.Scene(tris, nodes, hdr, cache)
    yield dict(tris=tris, nodes=nodes, eye=eye, cam=cam, hdr=hdr, cache=cache, scene=sc)
    sc.close()


def test_s1m_mode3_in_tile_aligned_windows(s1m):
    """C4's scene and integrator on its own 1920x1080 grid, checked against the oracle in windows aligned to the tiles
    (the last one includes the clipped bottom row of tiles)."""
    cfg = _cfg(s1m, api.MODE_DISNEY_IS_MIS_P5, spp=8, width=1920, height=1080)
    thr = 0.3
    img, spp, luma2 = s1m["scene"].render_adaptive(cfg, thr, 2, 2)
    c = s1m["scene"].counters()
    assert c.samples == int(spp.sum()) and 2 <= spp.min() and spp.max() <= 8
    for win in [(0, 0, 64, 48), (928, 528, 992, 576), (1856, 1024, 1920, 1080)]:
        ref, rspp, rl2, _ = oa.render_adaptive(s1m["tris"], s1m["nodes"], cfg, thr, 2, 2, hdr=s1m["hdr"], hdr_cache=s1m["cache"], window=win)
        x0, y0, x1, y1 = win
        np.testing.assert_array_equal(spp[y0:y1, x0:x1], rspp)
        assert_same_bits(img[y0:y1, x0:x1], ref, "window %s framebuffer" % (win,))
        assert_same_bits(luma2[y0:y1, x0:x1], rl2, "window %s luma2" % (win,))
