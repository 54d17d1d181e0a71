"""The feature-buffer and denoiser part of the C ABI: struct layout and bindings (no compute calls)."""
import ctypes


def test_denoise_params_layout_and_bindings():
    from ezrt_b200 import _lib, api
    assert ctypes.sizeof(_lib.DenoiseParams) == 24   # int32 iterations, float sigma_l, sigma_n, sigma_z, sigma_a, int32 reserved
    assert [f for f, _ in _lib.DenoiseParams._fields_] == ["iterations", "sigma_l", "sigma_n", "sigma_z", "sigma_a", "reserved"]
    assert [_lib.DenoiseParams.sigma_l.offset, _lib.DenoiseParams.reserved.offset] == [4, 20]
    d = api.denoise_params()
    assert (d.iterations, d.reserved) == (5, 0) and min(d.sigma_l, d.sigma_n, d.sigma_z, d.sigma_a) > 0
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for name in ("ezrt_render_aov", "ezrt_render_aov_device", "ezrt_denoise", "ezrt_denoise_device"):
        assert hasattr(raw, name) and name in _lib.SIGNATURES
    assert _lib.lib.ezrt_version() == 200
    for name in ("render_aov", "render_aov_device", "denoise", "denoise_device"):
        assert callable(getattr(api.Scene, name))
