"""ctypes binding of the CPU restatement of the feature-buffer render and of the denoiser (tests/oracle_aov.cpp ->
build/libezrt_oracle_aov.so), plus an independent numpy float64 restatement of the denoiser.  TEST INFRASTRUCTURE, like
tests/oracle_binding.py."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import build as _build
from ezrt_b200.api import DENOISE_DEFAULTS, denoise_params
from ezrt_b200._lib import DenoiseParams, RenderParams
from tests.oracle_binding import COUNTER_NAMES

if not os.path.exists(_build.ORACLE_AOV_SO):
    _build.build_oracle_aov()
_o = C.CDLL(_build.ORACLE_AOV_SO)

_fp = C.POINTER(C.c_float)
_o.oracle_render_aov.restype = C.c_int
_o.oracle_render_aov.argtypes = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams), C.c_int, C.c_int,
                                 C.c_int, C.c_int, _fp, _fp, _fp, C.POINTER(C.c_uint64), C.c_int]
_o.oracle_denoise.restype = C.c_int
_o.oracle_denoise.argtypes = [C.POINTER(DenoiseParams), _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, _fp]


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if shape is None else a.reshape(shape)


def render_aov(tris, nodes, cfg, hdr=None, hdr_cache=None, hdr_linear=True, window=None, prev=None, threads=0):
    """oracle_render_aov: returns (image [h, w, C], aov [h, w, 8], luma2 [h, w], counters dict) of the whole grid or of
    window = (x0, y0, x1, y1).  prev = (image, aov, luma2) of the frames before cfg.first_frame (copied, not changed)."""
    tris = _f32(tris, (-1, 36)); nodes = _f32(nodes, (-1, 12))
    hw = hh = 0
    if hdr is not None:
        hdr = _f32(hdr); hdr_cache = None if hdr_cache is None else _f32(hdr_cache)
        hh, hw = hdr.shape[0], hdr.shape[1]
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    if prev is None:
        img, aov, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w, 8), np.float32), np.zeros((h, w), np.float32)
    else:
        img, aov, luma2 = (np.array(a, np.float32, copy=True).reshape(s) for a, s in zip(prev, ((h, w, cfg.out_channels), (h, w, 8), (h, w))))
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    f = lambda arr: None if arr is None else arr.ctypes.data_as(_fp)
    rc = _o.oracle_render_aov(f(tris), tris.shape[0], f(nodes), nodes.shape[0], f(hdr), f(hdr_cache), hw, hh, int(bool(hdr_linear)), C.byref(p),
                              int(x0), int(y0), int(x1), int(y1), f(img), f(aov), f(luma2), cnt.ctypes.data_as(C.POINTER(C.c_uint64)), int(threads))
    if rc != 0:
        raise RuntimeError("oracle_render_aov failed (%d)" % rc)
    c = {k: int(v) for k, v in zip(COUNTER_NAMES, cnt)}
    c["rays"] = c["rays_primary"] + c["rays_bounce"] + c["rays_shadow"]
    return img, aov, luma2, c


def denoise(image, aov, luma2, n, **sigmas):
    """oracle_denoise: the scalar C++ restatement of ezrt_denoise (float32, ezrt_math.h)."""
    img = _f32(image)
    h, w, ch = img.shape
    out = np.zeros_like(img)
    d = denoise_params(**{**DENOISE_DEFAULTS, **sigmas})
    rc = _o.oracle_denoise(C.byref(d), img.ctypes.data_as(_fp), ch, _f32(aov, (h, w, 8)).ctypes.data_as(_fp), _f32(luma2, (h, w)).ctypes.data_as(_fp),
                           w, h, int(n), out.ctypes.data_as(_fp))
    if rc != 0:
        raise RuntimeError("oracle_denoise failed (%d)" % rc)
    return out


_B3 = np.array([1 / 16, 1 / 4, 3 / 8, 1 / 4, 1 / 16])


def denoise_f64(image, aov, luma2, n, **sigmas):
    """The filter of DESIGN.md section 9 in numpy float64, written from the formulas, not from ezrt_math.h: exact exp / pow,
    whole-image shifts instead of a per-pixel loop."""
    s = {**DENOISE_DEFAULTS, **sigmas}
    img = np.asarray(image, np.float64)
    h, w, ch = img.shape
    f = np.asarray(aov, np.float64).reshape(h, w, 8)
    alb, cov, nrm, z = f[..., 0:3], f[..., 3], f[..., 4:7], f[..., 7]
    lum = lambda c: 0.3 * c[..., 0] + 0.6 * c[..., 1] + 0.1 * c[..., 2]
    c = img[..., :3].copy()
    v = np.maximum(np.asarray(luma2, np.float64).reshape(h, w) - lum(c) ** 2, 0.0) / n
    covered = cov != 0
    for k in range(s["iterations"]):
        step = 1 << k
        Yp, sdp = lum(c), np.sqrt(v)
        sw = np.zeros((h, w)); sc = np.zeros((h, w, 3)); sv = np.zeros((h, w))
        for j in range(-2, 3):
            for i in range(-2, 3):
                hw_ = _B3[i + 2] * _B3[j + 2]
                dy, dx = step * j, step * i
                # q = p + (dx, dy): the source window of the valid p
                ys, xs = slice(max(0, -dy), min(h, h - dy)), slice(max(0, -dx), min(w, w - dx))
                yq, xq = slice(ys.start + dy, ys.stop + dy), slice(xs.start + dx, xs.stop + dx)
                if ys.start >= ys.stop or xs.start >= xs.stop:
                    continue
                cq, vq = c[yq, xq], v[yq, xq]
                if i == 0 and j == 0:
                    wt = np.full(cq.shape[:2], hw_)
                else:
                    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
                        ok = covered[ys, xs] & covered[yq, xq] & np.isfinite(cq).all(-1) & np.isfinite(vq)
                        d = (nrm[ys, xs] * nrm[yq, xq]).sum(-1)
                        wn = np.where(d > 0, np.abs(d) ** s["sigma_n"], 0.0)
                        wz = np.exp(-np.abs(z[ys, xs] - z[yq, xq]) / (s["sigma_z"] * z[ys, xs] * step * max(abs(i), abs(j))))
                        wl = np.exp(-np.abs(Yp[ys, xs] - lum(cq)) / (s["sigma_l"] * sdp[ys, xs] + 1e-4))
                        wa = np.exp(-np.abs(alb[ys, xs] - alb[yq, xq]).sum(-1) / s["sigma_a"])
                        wt = np.where(ok, hw_ * wn * wz * wl * wa, 0.0)
                    cq = np.where(wt[..., None] > 0, cq, 0.0)
                    vq = np.where(wt > 0, vq, 0.0)
                sw[ys, xs] += wt
                sc[ys, xs] += wt[..., None] * cq
                sv[ys, xs] += wt * wt * vq
        with np.errstate(invalid="ignore", divide="ignore"):
            nc, nv = sc / sw[..., None], sv / (sw * sw)
        c = np.where(covered[..., None], nc, c)
        v = np.where(covered, nv, v)
    out = img.copy()
    out[..., :3] = c
    return out
