"""Feature buffers (ezrt_render_aov) and the a-trous denoiser (ezrt_denoise) on the GPU: bit for bit against the CPU
restatements (tests/oracle_aov.cpp), against the plain and adaptive renders, and the denoiser's quality on the P3 bunny."""
import ctypes as C

import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_aov as ov
from tests.test_gpu_parity import assert_same_bits

pytestmark = pytest.mark.gpu

ENV = (0.35, 0.45, 0.6)
W, H, SPP = 96, 72, 6
MODES = [api.MODE_DIFFUSE_P3, api.MODE_DISNEY_ANISO_P4, api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5]
# the denoised image of the P3 bunny at 16 spp has at most this fraction of the noisy image's luminance relMSE against 1024 spp
# (measured: 0.2484 -- noisy 0.1781, denoised 0.0443, default sigmas; seeded, so the ratio is the same on every run)
QUALITY_BOUND = 0.3


@pytest.fixture(scope="module")
def bunny(bunny_scene, small_hdr):
    tris, nodes, eye, cam = bunny_scene
    hdr, cache = small_hdr
    sc = api.Scene(tris, nodes, hdr, cache)
    yield dict(tris=tris, nodes=nodes, eye=eye, cam=cam, hdr=hdr, cache=cache, scene=sc)
    sc.close()


def _cfg(b, mode=api.MODE_DISNEY_IS_MIS_P5, spp=SPP, **kw):
    return api.RenderConfig(width=kw.pop("width", W), height=kw.pop("height", H), spp=spp, max_bounce=2, mode=mode, eye=tuple(b["eye"]),
                            camera_rotate=tuple(b["cam"]), env_color=ENV, **kw)


def _oracle(b, cfg, **kw):
    return ov.render_aov(b["tris"], b["nodes"], cfg, hdr=b["hdr"], hdr_cache=b["cache"], **kw)


@pytest.mark.parametrize("mode", MODES)
def test_bunny_matches_the_oracle(bunny, mode):
    cfg = _cfg(bunny, mode)
    img, aov, luma2 = bunny["scene"].render_aov(cfg)
    c = bunny["scene"].counters()
    ref, raov, rl2, rc = _oracle(bunny, cfg)
    assert_same_bits(img, ref, "mode %d framebuffer" % mode)
    assert_same_bits(aov, raov, "mode %d aov" % mode)
    assert_same_bits(luma2, rl2, "mode %d luma2" % mode)
    assert c.rays == rc["rays"] and c.primary_rays == rc["rays_primary"] and c.shadow_rays == rc["rays_shadow"]
    cov = aov[..., 3]
    assert (cov == 0).any() and (cov == 1).any(), "the view shows both the bunny and the sky"
    assert (aov[cov == 0] == 0).all()


def test_framebuffer_equals_the_plain_render_and_luma2_the_adaptive_one(bunny):
    sc = bunny["scene"]
    for mode in MODES:
        cfg = _cfg(bunny, mode, spp=8)
        img, _, luma2 = (a.copy() for a in sc.render_aov(cfg))
        assert sc.render(cfg).tobytes() == img.tobytes(), mode
        aimg, spp, al2 = sc.render_adaptive(cfg, 1e-9, 4, 4)   # no tile converges: every pixel gets all 8 frames
        assert (spp == 8).all() and aimg.tobytes() == img.tobytes() and al2.tobytes() == luma2.tobytes(), mode


def test_resuming_equals_one_call(bunny):
    sc = bunny["scene"]
    for mode in (api.MODE_DIFFUSE_P3, api.MODE_DISNEY_IS_MIS_P5):
        whole = [a.copy() for a in sc.render_aov(_cfg(bunny, mode, spp=7))]
        first = [a.copy() for a in sc.render_aov(_cfg(bunny, mode, spp=3))]
        rest = sc.render_aov(_cfg(bunny, mode, spp=4, first_frame=3), *[a.copy() for a in first])   # in/out
        for a, b, name in zip(rest, whole, ("image", "aov", "luma2")):
            assert a.tobytes() == b.tobytes(), (mode, name)
        ref = _oracle(bunny, _cfg(bunny, mode, spp=4, first_frame=3), prev=first)
        for a, b in zip(rest, ref[:3]):
            assert a.tobytes() == b.tobytes(), mode


def _scatter(parts, channels):
    full = np.zeros((H, W, channels), np.float32)
    for rank, a in enumerate(parts):
        api.partition_scatter_host(np.ascontiguousarray(a, np.float32).reshape(-1, channels), full, W, H, channels, rank, len(parts))
    return full


def test_same_bits_under_batch_sizes_policies_and_partitions(bunny):
    sc = bunny["scene"]
    cfg = _cfg(bunny)
    img, aov, luma2 = (a.copy() for a in sc.render_aov(cfg))
    rays = sc.counters().rays
    for kw in [dict(frames_per_batch=1), dict(frames_per_batch=3), dict(frames_per_batch=0), dict(traverse=api.TRAVERSE_PRUNED),
               dict(traverse=api.TRAVERSE_REFERENCE), dict(traverse=api.TRAVERSE_ACCEL), dict(out_channels=4)]:
        i2, a2, l2 = sc.render_aov(_cfg(bunny, **kw))
        assert i2[..., :3].tobytes() == img.tobytes() and a2.tobytes() == aov.tobytes() and l2.tobytes() == luma2.tobytes(), kw
        assert sc.counters().rays == rays, kw
    parts = [sc.render_aov(_cfg(bunny, part_rank=r, part_count=2)) for r in range(2)]
    assert _scatter([p[0] for p in parts], 3).tobytes() == img.tobytes()
    assert _scatter([p[1] for p in parts], 8).tobytes() == aov.tobytes()
    assert _scatter([p[2] for p in parts], 1)[..., 0].tobytes() == luma2.tobytes()


def test_device_entry_point_and_device_scatter(bunny):
    import torch
    sc = bunny["scene"]
    cfg = _cfg(bunny)
    img, aov, luma2 = (a.copy() for a in sc.render_aov(cfg))
    stream = torch.cuda.current_stream()
    d_fb = torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")
    d_aov = torch.zeros(W * H * 8, dtype=torch.float32, device="cuda")
    d_l2 = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    sc.render_aov_device(cfg, d_fb, d_aov, d_l2, stream)
    torch.cuda.synchronize()
    assert d_fb.cpu().numpy().tobytes() == img.tobytes() and d_aov.cpu().numpy().tobytes() == aov.tobytes()
    assert d_l2.cpu().numpy().tobytes() == luma2.tobytes()
    full = torch.zeros(W * H * 8, dtype=torch.float32, device="cuda")
    for r in range(2):
        n = api.partition_pixels(W, H, r, 2)
        part = torch.zeros(n * 8, dtype=torch.float32, device="cuda")
        sc.render_aov_device(_cfg(bunny, part_rank=r, part_count=2), torch.zeros(n * 3, dtype=torch.float32, device="cuda"), part,
                             torch.zeros(n, dtype=torch.float32, device="cuda"), stream)
        api.lib.ezrt_partition_scatter(C.c_void_p(part.data_ptr()), C.c_void_p(full.data_ptr()), W, H, 8, r, 2, C.c_void_p(stream.cuda_stream))
    torch.cuda.synchronize()
    assert full.cpu().numpy().tobytes() == aov.tobytes()


def test_invalid_inputs_are_rejected(bunny):
    import torch
    sc = bunny["scene"]
    with pytest.raises(api.EzrtError) as e:
        sc.render_aov(_cfg(bunny, pipeline=api.PIPELINE_MEGAKERNEL))
    assert e.value.code == -1 and api.lib.ezrt_last_error().decode().startswith("render_aov")
    with pytest.raises(api.EzrtError):   # null output buffers
        sc.render_aov_device(_cfg(bunny), 0, 0, 0)
    d_fb = torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")
    d_aov = torch.zeros(W * H * 8 + 4, dtype=torch.float32, device="cuda")
    d_l2 = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    with pytest.raises(api.EzrtError):   # aov not 16-byte aligned
        sc.render_aov_device(_cfg(bunny), d_fb, d_aov.data_ptr() + 4, d_l2)
    img, aov, luma2 = sc.render_aov(_cfg(bunny))
    bad = [dict(iterations=0), dict(iterations=11), dict(sigma_l=0.0), dict(sigma_n=-1.0), dict(sigma_z=float("nan")), dict(sigma_a=float("inf"))]
    for kw in bad:
        with pytest.raises(api.EzrtError):
            sc.denoise(img, aov, luma2, SPP, **kw)
    with pytest.raises(api.EzrtError):
        sc.denoise(img, aov, luma2, 0)
    d = api.denoise_params()
    d.reserved = 1
    rc = api.lib.ezrt_denoise(sc._h, C.byref(d), api._fp(img), 3, api._fp(aov), api._fp(luma2), W, H, SPP, api._fp(img))
    assert rc == -1
    rc = api.lib.ezrt_denoise(sc._h, C.byref(api.denoise_params()), api._fp(img), 5, api._fp(aov), api._fp(luma2), W, H, SPP, api._fp(img))
    assert rc == -1


def test_denoiser_matches_the_oracle(bunny):
    import torch
    sc = bunny["scene"]
    for (w, h, ch, mode) in [(W, H, 3, api.MODE_DISNEY_IS_MIS_P5), (77, 45, 4, api.MODE_DIFFUSE_P3), (33, 1, 3, api.MODE_DISNEY_SOBOL_P5),
                             (1, 1, 4, api.MODE_DISNEY_ANISO_P4)]:
        cfg = _cfg(bunny, mode, width=w, height=h, out_channels=ch)
        img, aov, luma2 = (a.copy() for a in sc.render_aov(cfg))
        for it in range(1, 11):
            got = sc.denoise(img, aov, luma2, SPP, iterations=it)
            want = ov.denoise(img, aov, luma2, SPP, iterations=it)
            assert_same_bits(got, want, "%dx%dx%d, %d iterations" % (w, h, ch, it))
        sig = dict(iterations=4, sigma_l=1.5, sigma_n=16.0, sigma_z=0.3, sigma_a=0.05)
        want = ov.denoise(img, aov, luma2, SPP, **sig)
        # the device entry point, output aliasing the input
        d_img = torch.from_numpy(img.copy()).cuda()
        d_aov, d_l2 = torch.from_numpy(aov).cuda(), torch.from_numpy(luma2).cuda()
        sc.denoise_device(d_img, ch, d_aov, d_l2, w, h, SPP, d_img, torch.cuda.current_stream(), **sig)
        torch.cuda.synchronize()
        assert_same_bits(d_img.cpu().numpy(), want, "%dx%d device, aliased" % (w, h))
        # the host entry point, aliased too
        same = img.copy()
        sc.denoise(same, aov, luma2, SPP, out=same, **sig)
        assert_same_bits(same, want, "%dx%d host, aliased" % (w, h))


def test_denoiser_injected_nan_stays_local(bunny):
    sc = bunny["scene"]
    img, aov, luma2 = (a.copy() for a in sc.render_aov(_cfg(bunny, api.MODE_DIFFUSE_P3, out_channels=4)))
    ys, xs = np.nonzero(aov[..., 3] == 1)
    y, x = ys[len(ys) // 2], xs[len(xs) // 2]
    img[y, x, 0] = np.nan
    got = sc.denoise(img, aov, luma2, SPP)
    assert_same_bits(got, ov.denoise(img, aov, luma2, SPP), "NaN injected")
    bad = ~np.isfinite(got[..., :3]).all(-1)
    assert bad[y, x] and bad.sum() == 1


@pytest.fixture(scope="module")
def s1m():
    tris, nodes, eye, cam = scenes.s_1m_bunny()
    hdr = scenes.synth_hdr(2048, 1024)
    cache = api.hdr_cache_device(hdr)[0]
    sc = api.Scene(tris, nodes, hdr, cache)
    yield dict(tris=tris, nodes=nodes, eye=eye, cam=cam, hdr=hdr, cache=cache, scene=sc)
    sc.close()


def test_s1m_mode3_in_tile_aligned_windows(s1m):
    """C4's scene and integrator on its own 1920x1080 grid, against the oracle in windows aligned to the tiles."""
    cfg = _cfg(s1m, api.MODE_DISNEY_IS_MIS_P5, spp=4, width=1920, height=1080)
    img, aov, luma2 = s1m["scene"].render_aov(cfg)
    for win in [(0, 0, 64, 48), (928, 528, 992, 576), (1856, 1024, 1920, 1080)]:
        ref, raov, rl2, _ = _oracle(s1m, cfg, window=win)
        x0, y0, x1, y1 = win
        assert_same_bits(img[y0:y1, x0:x1], ref, "window %s framebuffer" % (win,))
        assert_same_bits(aov[y0:y1, x0:x1], raov, "window %s aov" % (win,))
        assert_same_bits(luma2[y0:y1, x0:x1], rl2, "window %s luma2" % (win,))


def luminance_relmse(img, ref):
    lum = lambda a: 0.3 * a[..., 0].astype(np.float64) + 0.6 * a[..., 1].astype(np.float64) + 0.1 * a[..., 2].astype(np.float64)
    y, yr = lum(img), lum(ref)
    return float(np.mean((y - yr) ** 2 / (yr * yr + 1e-2)))


def test_denoised_p3_bunny_is_closer_to_the_converged_image(bunny):
    sc = bunny["scene"]
    cfg = lambda spp: _cfg(bunny, api.MODE_DIFFUSE_P3, spp=spp, width=128, height=96)
    ref = sc.render(cfg(1024)).copy()
    img, aov, luma2 = (a.copy() for a in sc.render_aov(cfg(16)))
    den = sc.denoise(img, aov, luma2, 16)
    noisy, denoised = luminance_relmse(img, ref), luminance_relmse(den, ref)
    print("P3 bunny 16 spp: relMSE noisy %.5f, denoised %.5f, ratio %.4f" % (noisy, denoised, denoised / noisy))
    assert denoised < QUALITY_BOUND * noisy
