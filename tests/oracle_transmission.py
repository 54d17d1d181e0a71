"""ctypes binding of the CPU restatement of the materials' transmission (tests/oracle_transmission.cpp ->
build/libezrt_oracle_transmission.so): the mixture, its sampler, Fresnel, and the render with RenderConfig.transmission.
TEST INFRASTRUCTURE, like tests/oracle_env_light.py."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import build as _build
from ezrt_b200._lib import RenderParams
from tests.oracle_binding import COUNTER_NAMES

if not os.path.exists(_build.ORACLE_TRANSMISSION_SO):
    _build.build_oracle_transmission()
_o = C.CDLL(_build.ORACLE_TRANSMISSION_SO)

_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int32)
_o.oracle_eval_bsdf.restype = C.c_int
_o.oracle_eval_bsdf.argtypes = [C.c_int, C.c_int, _fp, _fp, _fp, _fp, _ip, _fp, _fp]
_o.oracle_fresnel.restype = None
_o.oracle_fresnel.argtypes = [C.c_int, _fp, _fp, _fp]
_o.oracle_render_transmission.restype = C.c_int
_o.oracle_render_transmission.argtypes = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams), C.c_int,
                                          C.c_int, C.c_int, C.c_int, _fp, _fp, C.POINTER(C.c_uint64), C.c_int, C.c_int]


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if shape is None else a.reshape(shape)


def eval_bsdf(which, V, N, L, xi, inside, materials):
    """oracle_eval_bsdf, as ezrt_b200.api.eval_bsdf: [n, 8] float32 (which 0: f, 1: pdf, 2: sample of xi [n, 4])."""
    V = _f32(V, (-1, 3)); N = _f32(N, (-1, 3))
    n = V.shape[0]
    L = _f32(np.zeros((n, 3)) if L is None else L, (-1, 3))
    xi = _f32(np.zeros((n, 4)) if xi is None else xi, (-1, 4))
    inside = np.ascontiguousarray(inside, dtype=np.int32).reshape(-1)
    materials = _f32(materials, (-1, 18))
    out = np.zeros((n, 8), np.float32)
    f = lambda a: a.ctypes.data_as(_fp)
    if _o.oracle_eval_bsdf(which, n, f(V), f(N), f(L), f(xi), inside.ctypes.data_as(_ip), f(materials), f(out)) != 0:
        raise ValueError("oracle_eval_bsdf: bad which")
    return out


def fresnel(cos_i, eta):
    """ez_fresnel_dielectric of every (cos_i, eta) pair."""
    c = _f32(cos_i).reshape(-1); e = _f32(eta).reshape(-1)
    out = np.zeros_like(c)
    _o.oracle_fresnel(c.size, c.ctypes.data_as(_fp), e.ctypes.data_as(_fp), out.ctypes.data_as(_fp))
    return out


def oracle_render_transmission(tris, nodes, cfg, hdr=None, hdr_cache=None, hdr_linear=True, window=None, threads=0, bsdf_only=False):
    """(image [h, w, C], luma2 [h, w], counters dict) of the whole grid or of window = (x0, y0, x1, y1): mode 4 with
    cfg.transmission runs the mixture (bsdf_only: BSDF samples only, every emission and environment hit at weight 1), everything
    else what tests/oracle_env_light.py's render runs."""
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
    rc = _o.oracle_render_transmission(f(tris), tris.shape[0], f(nodes), nodes.shape[0], f(hdr), f(hdr_cache), hw, hh, int(bool(hdr_linear)),
                                       C.byref(p), int(x0), int(y0), int(x1), int(y1), f(img), f(luma2),
                                       cnt.ctypes.data_as(C.POINTER(C.c_uint64)), int(threads), int(bool(bsdf_only)))
    if rc != 0:
        raise RuntimeError("oracle_render_transmission failed (%d)" % rc)
    c = {k: int(v) for k, v in zip(COUNTER_NAMES, cnt)}
    c["rays"] = c["rays_primary"] + c["rays_bounce"] + c["rays_shadow"]
    return img, luma2, c
