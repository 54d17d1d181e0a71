"""The adaptive-sampling part of the C ABI: struct layout and bindings (no compute calls)."""
import ctypes


def test_adaptive_params_layout_and_bindings():
    from ezrt_b200 import _lib
    assert ctypes.sizeof(_lib.AdaptiveParams) == 16   # float threshold, int32 min_spp, check_interval, reserved
    assert [f for f, _ in _lib.AdaptiveParams._fields_] == ["threshold", "min_spp", "check_interval", "reserved"]
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for name in ("ezrt_render_adaptive", "ezrt_render_adaptive_device"):
        assert hasattr(raw, name) and name in _lib.SIGNATURES
