"""ctypes binding of the CPU restatement of the homogeneous medium (tests/oracle_medium.cpp -> build/libezrt_oracle_medium.so): the
Henyey-Greenstein sampler and density, the box overlap, free flight and transmittance, and the render with RenderConfig.medium in plain /
window, feature-buffer and adaptive forms, with the test-only phase-only switch.  TEST INFRASTRUCTURE, like tests/oracle_lens.py."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import build as _build
from ezrt_b200._lib import AdaptiveParams, Medium, RenderParams
from tests.oracle_lens import _counters, _scene_args

if not os.path.exists(_build.ORACLE_MEDIUM_SO):
    _build.build_oracle_medium()
_o = C.CDLL(_build.ORACLE_MEDIUM_SO)

_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int32)
_u64 = C.POINTER(C.c_uint64)
_o.oracle_hg_sample.restype = None
_o.oracle_hg_sample.argtypes = [C.c_int, _fp, _fp, _fp, _fp, _fp]
_o.oracle_hg_pdf.restype = None
_o.oracle_hg_pdf.argtypes = [C.c_int, _fp, _fp, _fp, _fp]
_o.oracle_box_overlap.restype = None
_o.oracle_box_overlap.argtypes = [C.c_int, _fp, _fp, _fp, _fp, _fp, _ip, _fp]
_o.oracle_transmittance.restype = C.c_int
_o.oracle_transmittance.argtypes = [C.POINTER(Medium), C.c_int, _fp, _fp, _fp, _fp]
_o.oracle_free_flight.restype = None
_o.oracle_free_flight.argtypes = [C.c_int, _fp, C.c_float, _fp]
_SCENE = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams)]
_o.oracle_render_medium.restype = C.c_int
_o.oracle_render_medium.argtypes = _SCENE + [C.POINTER(Medium), C.c_int, C.c_int, C.c_int, C.c_int, _fp, _fp, _fp, _u64, C.c_int, C.c_int]
_o.oracle_render_medium_adaptive.restype = C.c_int
_o.oracle_render_medium_adaptive.argtypes = _SCENE + [C.POINTER(Medium), C.POINTER(AdaptiveParams), C.c_int, C.c_int, C.c_int, C.c_int, _fp, _ip,
                                                      _fp, _u64, C.c_int]


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if shape is None else a.reshape(shape)


def _p(a):
    return a.ctypes.data_as(_fp)


def medium(sigma_t, albedo=(1.0, 1.0, 1.0), g=0.0, box_min=(0.0, 0.0, 0.0), box_max=(0.0, 0.0, 0.0), reserved=0):
    """struct ezrt_medium, as Scene.set_medium fills it."""
    m = Medium()
    m.sigma_t, m.g, m.reserved = float(sigma_t), float(g), int(reserved)
    m.albedo[:] = [float(x) for x in albedo]
    m.box_min[:] = [float(x) for x in box_min]
    m.box_max[:] = [float(x) for x in box_max]
    return m


def hg_sample(d, g, h):
    """ez_hg_sample of rows d [n, 3], g [n], h [n, 2] -> (L [n, 3], ez_hg_pdf(d, L, g) [n])."""
    d, h = _f32(d, (-1, 3)), _f32(h, (-1, 2))
    g = _f32(np.broadcast_to(np.asarray(g, np.float32), (d.shape[0],)).copy())
    L, pdf = np.zeros_like(d), np.zeros(d.shape[0], np.float32)
    _o.oracle_hg_sample(d.shape[0], _p(d), _p(g), _p(h), _p(L), _p(pdf))
    return L, pdf


def hg_pdf(d, L, g):
    d, L = _f32(d, (-1, 3)), _f32(L, (-1, 3))
    g = _f32(np.broadcast_to(np.asarray(g, np.float32), (d.shape[0],)).copy())
    out = np.zeros(d.shape[0], np.float32)
    _o.oracle_hg_pdf(d.shape[0], _p(d), _p(L), _p(g), _p(out))
    return out


def box_overlap(o, d, t_end, bmin, bmax):
    """ez_box_overlap of segments (o [n, 3], d [n, 3], t_end [n]) -> (ok [n] bool, t0t1 [n, 2])."""
    o, d, t_end = _f32(o, (-1, 3)), _f32(d, (-1, 3)), _f32(t_end, (-1,))
    ok, t01 = np.zeros(o.shape[0], np.int32), np.zeros((o.shape[0], 2), np.float32)
    _o.oracle_box_overlap(o.shape[0], _p(o), _p(d), _p(t_end), _p(_f32(bmin, (3,))), _p(_f32(bmax, (3,))), ok.ctypes.data_as(_ip), _p(t01))
    return ok.astype(bool), t01


def transmittance(m, o, d, L):
    o, d, L = _f32(o, (-1, 3)), _f32(d, (-1, 3)), _f32(L, (-1,))
    out = np.zeros(o.shape[0], np.float32)
    if _o.oracle_transmittance(C.byref(m), o.shape[0], _p(o), _p(d), _p(L), _p(out)) != 0:
        raise ValueError("invalid medium")
    return out


def free_flight(r, sigma_t):
    r = _f32(r, (-1,))
    out = np.zeros_like(r)
    _o.oracle_free_flight(r.size, _p(r), float(sigma_t), _p(out))
    return out


def render(tris, nodes, cfg, m, hdr=None, hdr_cache=None, hdr_linear=True, window=None, aov=False, phase_only=False, threads=0):
    """(image [h, w, C], luma2 [h, w], aov [h, w, 8] or None, counters) of the whole grid or of window = (x0, y0, x1, y1), with the
    medium m (None: no medium); raises ValueError where the library returns EZRT_ERR_INVALID."""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.float32)
    feat = np.zeros((h, w, 8), np.float32) if aov else None
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    rc = _o.oracle_render_medium(*args, C.byref(p), None if m is None else C.byref(m), int(x0), int(y0), int(x1), int(y1), _p(img),
                                 None if feat is None else _p(feat), _p(luma2), cnt.ctypes.data_as(_u64), int(threads), int(bool(phase_only)))
    del keep
    if rc == -2:
        raise ValueError("invalid medium render")
    if rc != 0:
        raise RuntimeError("oracle_render_medium failed (%d)" % rc)
    return img, luma2, feat, _counters(cnt)


def render_adaptive(tris, nodes, cfg, m, threshold, min_spp, check_interval, hdr=None, hdr_cache=None, hdr_linear=True, window=None, threads=0):
    """(image, spp map, luma2, counters) of the adaptive render (ezrt_render_adaptive's tiles) of the grid or a tile-aligned window, with
    the medium m; cfg must set medium."""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, spp, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.int32), np.zeros((h, w), np.float32)
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    a = AdaptiveParams()
    a.threshold, a.min_spp, a.check_interval, a.reserved = float(threshold), int(min_spp), int(check_interval), 0
    rc = _o.oracle_render_medium_adaptive(*args, C.byref(p), None if m is None else C.byref(m), C.byref(a), int(x0), int(y0), int(x1), int(y1),
                                          _p(img), spp.ctypes.data_as(_ip), _p(luma2), cnt.ctypes.data_as(_u64), int(threads))
    del keep
    if rc == -2:
        raise ValueError("invalid medium render")
    if rc != 0:
        raise RuntimeError("oracle_render_medium_adaptive failed (%d)" % rc)
    return img, spp, luma2, _counters(cnt)
