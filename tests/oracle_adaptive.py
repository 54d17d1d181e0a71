"""ctypes binding of the CPU restatement of tile-adaptive sampling (tests/oracle_adaptive.cpp ->
build/libezrt_oracle_adaptive.so).  TEST INFRASTRUCTURE, like tests/oracle_binding.py."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import build as _build
from ezrt_b200.api import adaptive_params
from ezrt_b200._lib import AdaptiveParams, RenderParams
from tests.oracle_binding import COUNTER_NAMES

if not os.path.exists(_build.ORACLE_ADAPTIVE_SO):
    _build.build_oracle_adaptive()
_o = C.CDLL(_build.ORACLE_ADAPTIVE_SO)

_fp = C.POINTER(C.c_float)
_o.oracle_render_adaptive.restype = C.c_int
_o.oracle_render_adaptive.argtypes = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams),
                                      C.POINTER(AdaptiveParams), C.c_int, C.c_int, C.c_int, C.c_int, _fp, C.POINTER(C.c_int32), _fp,
                                      C.POINTER(C.c_uint64), C.c_int]


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if shape is None else a.reshape(shape)


def render_adaptive(tris, nodes, cfg, threshold, min_spp, check_interval, hdr=None, hdr_cache=None, hdr_linear=True, window=None, threads=0):
    """oracle_render_adaptive: returns (image [h, w, C], spp_map [h, w], luma2 [h, w], counters dict) of the whole
    cfg.width x cfg.height grid, or of window = (x0, y0, x1, y1) aligned to the 16x16 tiles."""
    tris = _f32(tris, (-1, 36)); nodes = _f32(nodes, (-1, 12))
    hw = hh = 0
    if hdr is not None:
        hdr = _f32(hdr); hdr_cache = None if hdr_cache is None else _f32(hdr_cache)
        hh, hw = hdr.shape[0], hdr.shape[1]
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    img = np.zeros((y1 - y0, x1 - x0, cfg.out_channels), np.float32)
    spp = np.zeros((y1 - y0, x1 - x0), np.int32)
    luma2 = np.zeros((y1 - y0, x1 - x0), np.float32)
    cnt = np.zeros(9, np.uint64)
    p, a = cfg.to_struct(), adaptive_params(threshold, min_spp, check_interval)
    f = lambda arr: None if arr is None else arr.ctypes.data_as(_fp)
    rc = _o.oracle_render_adaptive(f(tris), tris.shape[0], f(nodes), nodes.shape[0], f(hdr), f(hdr_cache), hw, hh, int(bool(hdr_linear)),
                                   C.byref(p), C.byref(a), int(x0), int(y0), int(x1), int(y1), f(img),
                                   spp.ctypes.data_as(C.POINTER(C.c_int32)), f(luma2), cnt.ctypes.data_as(C.POINTER(C.c_uint64)), int(threads))
    if rc != 0:
        raise RuntimeError("oracle_render_adaptive failed (%d)" % rc)
    c = {k: int(v) for k, v in zip(COUNTER_NAMES, cnt)}
    c["rays"] = c["rays_primary"] + c["rays_bounce"] + c["rays_shadow"]
    return img, spp, luma2, c


def luminance(img):
    """ez_luminance (include/ezrt_math.h) in float32: (0.3 r + 0.6 g) + 0.1 b, each operation rounded."""
    img = np.asarray(img, np.float32)
    return (np.float32(0.3) * img[..., 0] + np.float32(0.6) * img[..., 1]) + np.float32(0.1) * img[..., 2]


def adaptive_error(luma2, mean_img, n):
    """ez_adaptive_error (include/ezrt_math.h) in float32."""
    with np.errstate(invalid="ignore", divide="ignore"):
        Y = luminance(mean_img)
        var = np.asarray(luma2, np.float32) - Y * Y
        var = np.where(var < 0, np.float32(0), var).astype(np.float32)
        return (np.sqrt(var / np.float32(n)) / (Y + np.float32(1e-3))).astype(np.float32)


def tile_converged(err, threshold, tile=16):
    """[ty, tx] bool: every pixel of the tile has err <= threshold (a NaN fails)."""
    h, w = err.shape
    ok = err <= np.float32(threshold)
    ty, tx = (h + tile - 1) // tile, (w + tile - 1) // tile
    out = np.ones((ty, tx), bool)
    for j in range(ty):
        for i in range(tx):
            out[j, i] = ok[j * tile:(j + 1) * tile, i * tile:(i + 1) * tile].all()
    return out
