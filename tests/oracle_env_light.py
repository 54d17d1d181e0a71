"""ctypes binding of the CPU restatement of the environment map as a light (tests/oracle_env_light.cpp ->
build/libezrt_oracle_env_light.so): the environment table, its sampler and density, and the render with
RenderConfig.env_light.  TEST INFRASTRUCTURE, like tests/oracle_lights.py."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import build as _build
from ezrt_b200._lib import RenderParams
from tests.oracle_binding import COUNTER_NAMES

if not os.path.exists(_build.ORACLE_ENV_LIGHT_SO):
    _build.build_oracle_env_light()
_o = C.CDLL(_build.ORACLE_ENV_LIGHT_SO)

_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int32)
_o.oracle_env_table.restype = C.c_int
_o.oracle_env_table.argtypes = [_fp, C.c_int, C.c_int, _fp, _fp, _fp, C.POINTER(C.c_double)]
_o.oracle_env_samples.restype = C.c_int
_o.oracle_env_samples.argtypes = [_fp, C.c_int, C.c_int, C.c_int, _fp, _fp, _ip, _ip, _fp]
_o.oracle_env_pdf.restype = C.c_int
_o.oracle_env_pdf.argtypes = [_fp, C.c_int, C.c_int, C.c_int, _fp, _fp]
_o.oracle_render_env_light.restype = C.c_int
_o.oracle_render_env_light.argtypes = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams), C.c_int,
                                       C.c_int, C.c_int, C.c_int, _fp, _fp, C.POINTER(C.c_uint64), C.c_int]


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if shape is None else a.reshape(shape)


def env_table(hdr):
    """(row_cdf [H], col_cdf [H, W], texel_pdf [H, W], T) of the restatement, or None when the map has no table."""
    hdr = _f32(hdr)
    h, w = hdr.shape[0], hdr.shape[1]
    row, col, pdf, total = np.zeros(h, np.float32), np.zeros((h, w), np.float32), np.zeros((h, w), np.float32), C.c_double(0.0)
    ok = _o.oracle_env_table(hdr.ctypes.data_as(_fp), w, h, row.ctypes.data_as(_fp), col.ctypes.data_as(_fp), pdf.ctypes.data_as(_fp),
                             C.byref(total))
    return (row, col, pdf, total.value) if ok else None


def env_samples(hdr, r):
    """ez_env_sample for every (r_1, r_2) row of r: (directions [n, 3], texel drawn [n], texel found by toSphericalCoord [n],
    ez_env_pdf [n])."""
    hdr = _f32(hdr)
    h, w = hdr.shape[0], hdr.shape[1]
    r = _f32(r, (-1, 2))
    n = r.shape[0]
    d, t, lk, p = np.zeros((n, 3), np.float32), np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.float32)
    rc = _o.oracle_env_samples(hdr.ctypes.data_as(_fp), w, h, n, r.ctypes.data_as(_fp), d.ctypes.data_as(_fp), t.ctypes.data_as(_ip),
                               lk.ctypes.data_as(_ip), p.ctypes.data_as(_fp))
    if rc != 0:
        raise RuntimeError("oracle_env_samples: the map has no table")
    return d, t, lk, p


def env_pdf(hdr, dirs):
    """ez_env_pdf of every direction (0 without a table)."""
    hdr = _f32(hdr)
    d = _f32(dirs, (-1, 3))
    out = np.zeros(d.shape[0], np.float32)
    _o.oracle_env_pdf(hdr.ctypes.data_as(_fp), hdr.shape[1], hdr.shape[0], d.shape[0], d.ctypes.data_as(_fp), out.ctypes.data_as(_fp))
    return out


def oracle_render_env_light(tris, nodes, cfg, hdr=None, hdr_cache=None, hdr_linear=True, window=None, threads=0):
    """(image [h, w, C], luma2 [h, w], counters dict) of the whole grid or of window = (x0, y0, x1, y1): mode 4 with cfg.env_light
    runs the flagged integrator, everything else what tests/oracle_lights.py's render runs."""
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
    rc = _o.oracle_render_env_light(f(tris), tris.shape[0], f(nodes), nodes.shape[0], f(hdr), f(hdr_cache), hw, hh, int(bool(hdr_linear)),
                                    C.byref(p), int(x0), int(y0), int(x1), int(y1), f(img), f(luma2), cnt.ctypes.data_as(C.POINTER(C.c_uint64)),
                                    int(threads))
    if rc != 0:
        raise RuntimeError("oracle_render_env_light failed (%d)" % rc)
    c = {k: int(v) for k, v in zip(COUNTER_NAMES, cnt)}
    c["rays"] = c["rays_primary"] + c["rays_bounce"] + c["rays_shadow"]
    return img, luma2, c
