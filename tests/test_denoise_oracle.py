"""The denoiser's definition (include/ezrt_math.h, DESIGN.md section 9) on the CPU: the scalar C++ restatement against an
independent numpy float64 one, edge cases, and the properties the filter promises.  No GPU."""
import numpy as np
import pytest

from tests import oracle_aov


def synthetic(h, w, seed=0, n=16, ch=3):
    """A noisy image with the feature buffers of a few flat regions (different normals, albedos, depths), a strip of
    background (coverage 0) and a few half-covered edge pixels; luma2 consistent with the noise after n frames."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    region = ((xx * 3) // max(w, 1) + 3 * ((yy * 2) // max(h, 1))).astype(int)
    normals = np.array([[0, 0, 1], [0, 1, 0], [1, 0, 0], [0.6, 0, 0.8], [0, 0.6, 0.8], [0.8, 0.6, 0]], np.float64)
    albedo = np.array([[0.8, 0.2, 0.2], [0.2, 0.8, 0.2], [0.7, 0.7, 0.7], [0.2, 0.2, 0.8], [0.5, 0.5, 0.1], [0.9, 0.9, 0.9]])
    aov = np.zeros((h, w, 8), np.float32)
    aov[..., 0:3] = albedo[region]
    aov[..., 3] = 1.0
    aov[..., 4:7] = normals[region]
    aov[..., 7] = 2.0 + region + 0.01 * xx
    if w > 4:
        aov[:, -2:, :] = 0.0                  # background: the primary rays left the scene
        aov[::3, -3, :] *= 0.5                # edge pixels hit in half the frames
    base = albedo[region] * (0.5 + 0.5 * yy[..., None] / max(h, 1))
    noise = rng.normal(0.0, 0.3, (h, w, 1)) * base
    img = np.clip(base + noise, 0, None).astype(np.float32)
    lum = 0.3 * img[..., 0] + 0.6 * img[..., 1] + 0.1 * img[..., 2]
    luma2 = (lum ** 2 * (1 + 0.5 * rng.random((h, w))) + 0.01).astype(np.float32)
    if ch == 4:
        img = np.concatenate([img, rng.random((h, w, 1)).astype(np.float32)], axis=-1)
    return img, aov, luma2, n


def test_scalar_restatement_matches_float64():
    img, aov, luma2, n = synthetic(37, 53)
    for sig in (dict(), dict(iterations=3, sigma_l=2.0, sigma_n=32.0, sigma_z=0.5, sigma_a=0.3)):
        got = oracle_aov.denoise(img, aov, luma2, n, **sig)
        want = oracle_aov.denoise_f64(img, aov, luma2, n, **sig)
        assert np.isfinite(got).all()
        scale = np.abs(want).max()
        np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5 * scale)
        assert not np.array_equal(got, img), "the filter changed nothing"


@pytest.mark.parametrize("shape", [(1, 1), (1, 7), (5, 1), (3, 3), (2, 9)])
def test_tiny_images_and_steps_wider_than_the_image(shape):
    img, aov, luma2, n = synthetic(*shape, seed=3)
    for it in (1, 4, 10):
        got = oracle_aov.denoise(img, aov, luma2, n, iterations=it)
        want = oracle_aov.denoise_f64(img, aov, luma2, n, iterations=it)
        np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-6)
    if shape == (1, 1):   # one pixel: only its own centre tap, h*c/h
        assert np.allclose(oracle_aov.denoise(img, aov, luma2, n), img, rtol=1e-6)


def test_nan_pixel_stays_local():
    img, aov, luma2, n = synthetic(24, 32, seed=5, ch=4)
    img[10, 7, 1] = np.nan
    got = oracle_aov.denoise(img, aov, luma2, n, iterations=5)
    bad = ~np.isfinite(got[..., :3]).all(-1)
    assert bad[10, 7] and bad.sum() == 1
    np.testing.assert_array_equal(got[..., 3], img[..., 3])   # alpha is copied
    want = oracle_aov.denoise_f64(img, aov, luma2, n, iterations=5)
    ok = ~bad
    np.testing.assert_allclose(got[ok], want[ok], rtol=1e-5, atol=1e-5 * np.abs(want[ok]).max())


def test_constant_image_stays_constant():
    h, w = 19, 23
    img = np.empty((h, w, 3), np.float32)
    img[:] = (0.25, 0.5, 0.75)
    aov = np.zeros((h, w, 8), np.float32)
    aov[..., 0:3] = 0.6
    aov[..., 3] = 1.0
    aov[..., 6] = 1.0
    aov[..., 7] = 3.0
    y = np.float32(0.3) * np.float32(0.25) + np.float32(0.6) * np.float32(0.5) + np.float32(0.1) * np.float32(0.75)
    luma2 = np.full((h, w), y * y, np.float32)
    got = oracle_aov.denoise(img, aov, luma2, 8, iterations=6)
    np.testing.assert_allclose(got, img, rtol=4e-7, atol=0)


def test_zero_coverage_pixels_pass_through_bit_for_bit():
    img, aov, luma2, n = synthetic(21, 40, seed=9)
    got = oracle_aov.denoise(img, aov, luma2, n, iterations=7)
    bg = aov[..., 3] == 0
    assert bg.sum() > 0
    assert got[bg].tobytes() == img[bg].tobytes()
