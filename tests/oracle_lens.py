"""ctypes binding of the CPU restatement of the thin-lens camera (tests/oracle_lens.cpp -> build/libezrt_oracle_lens.so): the lens
set-up, the concentric map, the camera rays, and the render with RenderConfig.lens_radius in plain / window, feature-buffer and
adaptive forms.  TEST INFRASTRUCTURE, like tests/oracle_transmission.py."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import build as _build
from ezrt_b200._lib import AdaptiveParams, RenderParams
from tests.oracle_binding import COUNTER_NAMES

if not os.path.exists(_build.ORACLE_LENS_SO):
    _build.build_oracle_lens()
_o = C.CDLL(_build.ORACLE_LENS_SO)

_fp = C.POINTER(C.c_float)
_up = C.POINTER(C.c_uint32)
_ip = C.POINTER(C.c_int32)
_u64 = C.POINTER(C.c_uint64)
_o.oracle_lens_setup.restype = C.c_int
_o.oracle_lens_setup.argtypes = [_fp, _fp, C.c_float, C.c_float, _fp]
_o.oracle_concentric_disk.restype = None
_o.oracle_concentric_disk.argtypes = [C.c_int, _fp, _fp]
_o.oracle_camera_rays.restype = C.c_int
_o.oracle_camera_rays.argtypes = [C.POINTER(RenderParams), C.c_int, _up, _up, _up, _fp, _fp, _fp, _fp, _up]
_SCENE = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams)]
_o.oracle_render_lens.restype = C.c_int
_o.oracle_render_lens.argtypes = _SCENE + [C.c_int, C.c_int, C.c_int, C.c_int, _fp, _fp, _fp, _u64, C.c_int]
_o.oracle_render_lens_adaptive.restype = C.c_int
_o.oracle_render_lens_adaptive.argtypes = _SCENE + [C.POINTER(AdaptiveParams), C.c_int, C.c_int, C.c_int, C.c_int, _fp, _ip, _fp, _u64, C.c_int]


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if shape is None else a.reshape(shape)


def _u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32).reshape(-1)


def lens_setup(eye, cam, R, f):
    """ez_lens_setup: dict(eye, u0, u1, k, R) float32, or None when the parameters are invalid."""
    out = np.zeros(11, np.float32)
    if not _o.oracle_lens_setup(_f32(eye, (3,)).ctypes.data_as(_fp), _f32(cam, (16,)).ctypes.data_as(_fp), float(R), float(f),
                                out.ctypes.data_as(_fp)):
        return None
    return dict(eye=out[0:3], u0=out[3:6], u1=out[6:9], k=out[9], R=out[10])


def concentric_disk(u):
    """ez_concentric_disk of every row of u [n, 2] -> [n, 2] float32."""
    u = _f32(u, (-1, 2))
    xy = np.zeros_like(u)
    _o.oracle_concentric_disk(u.shape[0], u.ctypes.data_as(_fp), xy.ctypes.data_as(_fp))
    return xy


def camera_rays(cfg, px, py, frame):
    """The restatement's camera rays of the samples (px[i], py[i], frame[i]) -> dict(o, d, dir_pin [n, 3], draws [n, 2], seed [n]);
    raises ValueError when cfg's lens parameters are invalid."""
    px, py, frame = _u32(px), _u32(py), _u32(frame)
    n = px.size
    o, d, dp = (np.zeros((n, 3), np.float32) for _ in range(3))
    draws, seed = np.zeros((n, 2), np.float32), np.zeros(n, np.uint32)
    p = cfg.to_struct()
    f = lambda a: a.ctypes.data_as(_fp)
    u = lambda a: a.ctypes.data_as(_up)
    if _o.oracle_camera_rays(C.byref(p), n, u(px), u(py), u(frame), f(o), f(d), f(dp), f(draws), u(seed)) != 0:
        raise ValueError("invalid lens parameters")
    return dict(o=o, d=d, dir_pin=dp, draws=draws, seed=seed)


def _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear):
    tris = _f32(tris, (-1, 36)); nodes = _f32(nodes, (-1, 12))
    hw = hh = 0
    if hdr is not None:
        hdr = _f32(hdr); hdr_cache = None if hdr_cache is None else _f32(hdr_cache)
        hh, hw = hdr.shape[0], hdr.shape[1]
    f = lambda arr: None if arr is None else arr.ctypes.data_as(_fp)
    keep = (tris, nodes, hdr, hdr_cache)
    return keep, [f(tris), tris.shape[0], f(nodes), nodes.shape[0], f(hdr), f(hdr_cache), hw, hh, int(bool(hdr_linear))]


def _counters(cnt):
    c = {k: int(v) for k, v in zip(COUNTER_NAMES, cnt)}
    c["rays"] = c["rays_primary"] + c["rays_bounce"] + c["rays_shadow"]
    return c


def render(tris, nodes, cfg, hdr=None, hdr_cache=None, hdr_linear=True, window=None, aov=False, threads=0):
    """(image [h, w, C], luma2 [h, w], aov [h, w, 8] or None, counters) of the whole grid or of window = (x0, y0, x1, y1)."""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.float32)
    feat = np.zeros((h, w, 8), np.float32) if aov else None
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    rc = _o.oracle_render_lens(*args, C.byref(p), int(x0), int(y0), int(x1), int(y1), img.ctypes.data_as(_fp),
                               None if feat is None else feat.ctypes.data_as(_fp), luma2.ctypes.data_as(_fp), cnt.ctypes.data_as(_u64), int(threads))
    del keep
    if rc == -2:
        raise ValueError("invalid lens parameters")
    if rc != 0:
        raise RuntimeError("oracle_render_lens failed (%d)" % rc)
    return img, luma2, feat, _counters(cnt)


def render_adaptive(tris, nodes, cfg, threshold, min_spp, check_interval, hdr=None, hdr_cache=None, hdr_linear=True, window=None, threads=0):
    """(image, spp map, luma2, counters) of the adaptive render (ezrt_render_adaptive's tiles) of the grid or a tile-aligned window."""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, spp, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.int32), np.zeros((h, w), np.float32)
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    a = AdaptiveParams()
    a.threshold, a.min_spp, a.check_interval, a.reserved = float(threshold), int(min_spp), int(check_interval), 0
    rc = _o.oracle_render_lens_adaptive(*args, C.byref(p), C.byref(a), int(x0), int(y0), int(x1), int(y1), img.ctypes.data_as(_fp),
                                        spp.ctypes.data_as(_ip), luma2.ctypes.data_as(_fp), cnt.ctypes.data_as(_u64), int(threads))
    del keep
    if rc != 0:
        raise RuntimeError("oracle_render_lens_adaptive failed (%d)" % rc)
    return img, spp, luma2, _counters(cnt)
