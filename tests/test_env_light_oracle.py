"""The CPU restatement of the environment map as a light (tests/oracle_env_light.cpp; ezrt_math.h, DESIGN.md section 11) against
independent computations: the table in float64 numpy, the sampler's texel frequencies, its landing texels and its density
(an integral over the map's exact texel solid angles), the flagged estimator against plain mode 4 on the same scene (unbiased,
lower variance), and the cases without a table, which must render as mode 4 bit for bit."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_env_light as oe


def _lum64(hdr):
    h = np.asarray(hdr, np.float64)
    return 0.3 * h[..., 0] + 0.6 * h[..., 1] + 0.1 * h[..., 2]


def _table_f64(hdr):
    """(row_cdf, col_cdf, texel_pdf, T) in float64 from the definition, or None"""
    H, W = hdr.shape[:2]
    e = np.pi * (0.5 - (np.arange(H) + 0.5) / H)
    with np.errstate(invalid="ignore", over="ignore"):
        w = _lum64(hdr) * np.cos(e)[:, None]
        w = np.where(np.isfinite(w) & (w > 0), w, 0.0)
    R = np.cumsum(w, axis=1)[:, -1]
    T = np.cumsum(R)[-1]
    if not (np.isfinite(T) and T > 0):
        return None
    with np.errstate(invalid="ignore", divide="ignore"):
        col = np.where(R[:, None] > 0, np.cumsum(w, axis=1) / R[:, None], 0.0)
    return np.cumsum(R) / T, col, w / T, T


def _one_bright_texel(W=64, H=32):
    hdr = np.full((H, W, 3), 0.05, np.float32)
    hdr[H // 3, W // 5] = (400.0, 300.0, 200.0)
    return hdr


def _hostile_map():
    hdr = scenes.synth_hdr(64, 32).astype(np.float32)
    hdr[3, 7] = 0.0
    hdr[5, 9] = (-2.0, -2.0, -2.0)
    hdr[6, 10] = (np.nan, 1.0, 1.0)
    hdr[7, 11] = (np.inf, 1.0, 1.0)
    hdr[8] = 0.0   # a black row
    return hdr


@pytest.mark.parametrize("which", ["synth", "bright", "hostile"])
def test_table_matches_float64(which):
    hdr = {"synth": lambda: scenes.synth_hdr(64, 32), "bright": _one_bright_texel, "hostile": _hostile_map}[which]()
    row, col, pdf, T = oe.env_table(hdr)
    row64, col64, pdf64, T64 = _table_f64(hdr)
    assert abs(T - T64) <= 1e-5 * T64
    np.testing.assert_allclose(row, row64, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(col, col64, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(pdf, pdf64, rtol=1e-5, atol=1e-12)
    assert row[-1] == 1.0
    live = pdf.sum(1) > 0
    assert (col[live, -1] == 1.0).all()
    assert (np.diff(row) >= 0).all() and (np.diff(col, axis=1) >= 0).all()
    if which == "hostile":
        for i, j in ((3, 7), (5, 9), (6, 10), (7, 11)):
            assert pdf[i, j] == 0.0 and col[i, j] == (col[i, j - 1] if j else 0.0), (i, j)
        assert (pdf[8] == 0).all() and (col[8] == 0).all() and row[8] == row[7]


def test_black_map_has_no_table():
    assert oe.env_table(np.zeros((16, 32, 3), np.float32)) is None
    neg = np.full((16, 32, 3), -1.0, np.float32)
    assert oe.env_table(neg) is None


@pytest.mark.parametrize("which", ["synth", "bright"])
def test_sampler(which):
    hdr = (scenes.synth_hdr(64, 32) if which == "synth" else _one_bright_texel()).astype(np.float32)
    H, W = hdr.shape[:2]
    _, _, pdf_t, _ = oe.env_table(hdr)
    n = 1_000_000
    r = np.random.default_rng(11).random((n, 2)).astype(np.float32)
    d, texel, lookup, pdf = oe.env_samples(hdr, r)
    # texel frequencies match the table's probabilities
    p = pdf_t.ravel().astype(np.float64)
    cnt = np.bincount(texel, minlength=W * H).astype(np.float64)
    z = np.abs(cnt - n * p) / np.sqrt(np.maximum(n * p * (1 - p), 1.0))
    assert z.max() < 5.5, "texel frequency off by %.2f standard deviations" % z.max()
    assert (cnt[p == 0] == 0).all()
    # the direction lands back in the texel it was drawn from, but for rounding at texel borders
    miss = np.mean(lookup != texel)
    assert miss < 1e-3, miss
    # the sampler's pdf is ez_env_pdf of its direction, bit for bit
    assert pdf.tobytes() == oe.env_pdf(hdr, d).tobytes()
    assert (pdf > 0).all() and np.isfinite(pdf).all()
    # E[g / pdf] = the integral of g over the sphere, g = nearest-filtered luminance (exact texel solid angles)
    lum = _lum64(hdr).ravel()
    g = lum[lookup]
    est = g / pdf.astype(np.float64)
    e_top = np.pi * (0.5 - np.arange(H) / H)
    e_bot = np.pi * (0.5 - (np.arange(H) + 1) / H)
    omega = (2 * np.pi / W) * (np.sin(e_top) - np.sin(e_bot))
    integral = (_lum64(hdr) * omega[:, None]).sum()
    se = est.std() / np.sqrt(n)
    assert abs(est.mean() - integral) <= 4 * se + 1e-6 * integral, (est.mean(), integral, se)


def _p3_cfg(eye, cam, spp, **kw):
    base = dict(width=64, height=48, spp=spp, max_bounce=2, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam))
    base.update(kw)
    return api.RenderConfig(**base)


def _stats(img, luma2):
    y = (0.3 * img[..., 0] + 0.6 * img[..., 1] + 0.1 * img[..., 2]).astype(np.float64)
    return y, np.maximum(luma2.astype(np.float64) - y ** 2, 0.0)


def test_unbiased_against_mode_4_with_lower_variance(small_hdr):
    """The flagged estimator against plain mode 4 (an independent unbiased estimator of the same image) on the P3 bunny under
    the 128 x 64 map: every 8 x 8 block mean agrees, and the per-pixel luminance variance is lower."""
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    hdr, cache = small_hdr
    n = 1024
    out = {}
    for flag in (False, True):
        img, luma2, _ = oe.oracle_render_env_light(tris, nodes, _p3_cfg(eye, cam, n, env_light=flag), hdr=hdr, hdr_cache=cache)
        out[flag] = _stats(img, luma2)
    (y4, v4), (ye, ve) = out[False], out[True]
    blk = lambda a: a.reshape(6, 8, 8, 8).swapaxes(1, 2).reshape(6, 8, 64)
    se = np.sqrt(blk(v4).sum(-1) / n / 64 ** 2 + blk(ve).sum(-1) / n / 64 ** 2)
    z = np.abs(blk(y4).mean(-1) - blk(ye).mean(-1)) / np.maximum(se, 1e-12)
    assert np.isfinite(z).all() and (z <= 5).all(), "block means differ by up to %.2f standard errors" % z.max()
    assert ve.mean() < v4.mean() / 6, (ve.mean(), v4.mean())   # 12.6x lower (DESIGN.md section 11)


@pytest.mark.parametrize("case", ["no map", "black map"])
def test_without_a_table_the_render_is_mode_4(case):
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    hdr = None if case == "no map" else np.zeros((32, 64, 3), np.float32)
    cache = None if hdr is None else api.hdr_cache(hdr)
    kw = dict(width=32, height=24, max_bounce=2, env_color=(0.4, 0.5, 0.6))
    plain, pl2, pc = oe.oracle_render_env_light(tris, nodes, _p3_cfg(eye, cam, 4, **kw), hdr=hdr, hdr_cache=cache)
    flag, fl2, fc = oe.oracle_render_env_light(tris, nodes, _p3_cfg(eye, cam, 4, env_light=True, **kw), hdr=hdr, hdr_cache=cache)
    assert flag.tobytes() == plain.tobytes() and fl2.tobytes() == pl2.tobytes() and fc == pc
    assert fc["rays_shadow"] > 0
