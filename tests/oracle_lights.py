"""ctypes binding of the CPU restatement of the light sampling mode (tests/oracle_lights.cpp -> build/libezrt_oracle_lights.so):
the light table, the bounded occlusion query and the mode-4 render.  TEST INFRASTRUCTURE, like tests/oracle_binding.py."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import build as _build
from ezrt_b200._lib import RenderParams
from tests.oracle_binding import COUNTER_NAMES

if not os.path.exists(_build.ORACLE_LIGHTS_SO):
    _build.build_oracle_lights()
_o = C.CDLL(_build.ORACLE_LIGHTS_SO)

_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int32)
_o.oracle_light_table.restype = C.c_int
_o.oracle_light_table.argtypes = [_fp, C.c_int, C.c_int, _ip, _fp, C.POINTER(C.c_double)]
_o.oracle_occluded.restype = C.c_int
_o.oracle_occluded.argtypes = [_fp, C.c_int, _fp, C.c_int, C.c_int, _fp, _fp, _fp, C.c_int, _ip]
_o.oracle_triangle_points.restype = None
_o.oracle_triangle_points.argtypes = [_fp, C.c_int, _fp, _fp]
_o.oracle_render_lights.restype = C.c_int
_o.oracle_render_lights.argtypes = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams), C.c_int, C.c_int,
                                    C.c_int, C.c_int, _fp, _fp, C.POINTER(C.c_uint64), C.c_int]


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if shape is None else a.reshape(shape)


def oracle_light_table(tris):
    """(triangle indices int32 [K], cdf float32 [K], W float64) of the restatement."""
    tris = _f32(tris, (-1, 36))
    k = _o.oracle_light_table(tris.ctypes.data_as(_fp), tris.shape[0], 0, None, None, None)
    if k < 0:
        raise RuntimeError("oracle_light_table failed")
    tri, cdf, total = np.zeros(k, np.int32), np.zeros(k, np.float32), C.c_double(0.0)
    _o.oracle_light_table(tris.ctypes.data_as(_fp), tris.shape[0], k, tri.ctypes.data_as(_ip), cdf.ctypes.data_as(_fp), C.byref(total))
    return tri, cdf, total.value


def oracle_occluded(tris, nodes, origins, dirs, tmax, traverse=0):
    """1 where no triangle the shader's hitBVH tests is accepted strictly before tmax (all tmax = +inf: unbounded, mode 3's rays)."""
    tris = _f32(tris, (-1, 36)); nodes = _f32(nodes, (-1, 12))
    o = _f32(origins, (-1, 3)); d = _f32(dirs, (-1, 3))
    n = o.shape[0]
    t = _f32(np.broadcast_to(np.asarray(tmax, np.float32), (n,)))
    lit = np.zeros(n, np.int32)
    rc = _o.oracle_occluded(tris.ctypes.data_as(_fp), tris.shape[0], nodes.ctypes.data_as(_fp), nodes.shape[0], n, o.ctypes.data_as(_fp),
                            d.ctypes.data_as(_fp), t.ctypes.data_as(_fp), int(traverse), lit.ctypes.data_as(_ip))
    if rc != 0:
        raise RuntimeError("oracle_occluded failed")
    return lit


def triangle_points(p1, p2, p3, r):
    """ez_triangle_point for every (r_1, r_2) row of r."""
    p = _f32(np.concatenate([p1, p2, p3]))
    r = _f32(r, (-1, 2))
    out = np.zeros((r.shape[0], 3), np.float32)
    _o.oracle_triangle_points(p.ctypes.data_as(_fp), r.shape[0], r.ctypes.data_as(_fp), out.ctypes.data_as(_fp))
    return out


def oracle_render_lights(tris, nodes, cfg, hdr=None, hdr_cache=None, hdr_linear=True, window=None, threads=0):
    """(image [h, w, C], luma2 [h, w], counters dict) of the whole grid or of window = (x0, y0, x1, y1); cfg.mode 4 runs the
    light sampling integrator, the other modes the oracle's."""
    tris = _f32(tris, (-1, 36)); nodes = _f32(nodes, (-1, 12))
    hw = hh = 0
    if hdr is not None:
        hdr = _f32(hdr); hdr_cache = None if hdr_cache is None else _f32(hdr_cache)
        hh, hw = hdr.shape[0], hdr.shape[1]
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.float32)
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    f = lambda arr: None if arr is None else arr.ctypes.data_as(_fp)
    rc = _o.oracle_render_lights(f(tris), tris.shape[0], f(nodes), nodes.shape[0], f(hdr), f(hdr_cache), hw, hh, int(bool(hdr_linear)), C.byref(p),
                                 int(x0), int(y0), int(x1), int(y1), f(img), f(luma2), cnt.ctypes.data_as(C.POINTER(C.c_uint64)), int(threads))
    if rc != 0:
        raise RuntimeError("oracle_render_lights failed (%d)" % rc)
    c = {k: int(v) for k, v in zip(COUNTER_NAMES, cnt)}
    c["rays"] = c["rays_primary"] + c["rays_bounce"] + c["rays_shadow"]
    return img, luma2, c
