"""ctypes binding of the CPU restatement of base-colour textures (tests/oracle_textures.cpp -> build/libezrt_oracle_textures.so): the
definition's barycentrics and filter, and the render with RenderConfig.textures in plain / window, feature-buffer and adaptive forms.
TEST INFRASTRUCTURE, like tests/oracle_medium.py."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import build as _build
from ezrt_b200._lib import AdaptiveParams, Medium, RenderParams, Texture
from tests.oracle_lens import _counters, _scene_args

if not os.path.exists(_build.ORACLE_TEXTURES_SO):
    _build.build_oracle_textures()
_o = C.CDLL(_build.ORACLE_TEXTURES_SO)

_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int32)
_u64 = C.POINTER(C.c_uint64)
_o.oracle_tri_bary.restype = None
_o.oracle_tri_bary.argtypes = [C.c_int, _fp, _fp, _fp, _fp, _fp, _fp]
_o.oracle_tex_sample.restype = None
_o.oracle_tex_sample.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, _fp, _fp]
_o.oracle_srgb_table.restype = None
_o.oracle_srgb_table.argtypes = [_fp]
_SCENE = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams)]
_TEX = [C.POINTER(Medium), C.c_int, C.POINTER(Texture), _fp, _ip]
_o.oracle_render_textures.restype = C.c_int
_o.oracle_render_textures.argtypes = _SCENE + _TEX + [C.c_int, C.c_int, C.c_int, C.c_int, _fp, _fp, _fp, _u64, C.c_int]
_o.oracle_render_textures_adaptive.restype = C.c_int
_o.oracle_render_textures_adaptive.argtypes = _SCENE + _TEX + [C.POINTER(AdaptiveParams), C.c_int, C.c_int, C.c_int, C.c_int, _fp, _ip, _fp, _u64, C.c_int]


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if shape is None else a.reshape(shape)


def _p(a):
    return a.ctypes.data_as(_fp)


def srgb_table():
    out = np.zeros(256, np.float32)
    _o.oracle_srgb_table(_p(out))
    return out


def tri_bary(P, p1, p2, p3, Ng):
    """ez_tri_bary of rows [n, 3] -> w [n, 3]"""
    a = [_f32(x, (-1, 3)) for x in (P, p1, p2, p3, Ng)]
    w = np.zeros_like(a[0])
    _o.oracle_tri_bary(a[0].shape[0], *[_p(x) for x in a], _p(w))
    return w


def _rgba(t):
    t = np.asarray(t, np.uint8)
    if t.shape[2] == 3:
        t = np.concatenate([t, np.full(t.shape[:2] + (1,), 255, np.uint8)], axis=2)
    return np.ascontiguousarray(t)


def tex_sample(tex, uv):
    """ez_tex_sample of the uint8 texture [H, W, 3|4] at rows uv [n, 2] -> rgb [n, 3]"""
    t = _rgba(tex)
    uv = _f32(uv, (-1, 2))
    out = np.zeros((uv.shape[0], 3), np.float32)
    _o.oracle_tex_sample(t.ctypes.data, t.shape[1], t.shape[0], uv.shape[0], _p(uv), _p(out))
    return out


def _textures(textures, texcoords, texture_id, n):
    keep = [_rgba(t) for t in textures]
    arr = (Texture * len(keep))()
    for k, t in enumerate(keep):
        arr[k].width, arr[k].height, arr[k].rgba, arr[k].reserved = t.shape[1], t.shape[0], t.ctypes.data, 0
    uv = _f32(texcoords, (n, 6))
    ids = np.ascontiguousarray(np.asarray(texture_id, np.int32).reshape(n))
    return (keep, uv, ids), [len(keep), arr, _p(uv), ids.ctypes.data_as(_ip)]


def render(tris, nodes, cfg, textures, texcoords, texture_id, m=None, hdr=None, hdr_cache=None, hdr_linear=True, window=None, aov=False, threads=0):
    """(image [h, w, C], luma2 [h, w], aov [h, w, 8] or None, counters) of the grid or of window = (x0, y0, x1, y1) with the textures
    (as Scene.set_textures takes them) and the medium m (oracle_medium.medium, for cfg.medium); ValueError where the library returns
    EZRT_ERR_INVALID."""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    tkeep, targs = _textures(textures, texcoords, texture_id, np.asarray(tris).shape[0])
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.float32)
    feat = np.zeros((h, w, 8), np.float32) if aov else None
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    rc = _o.oracle_render_textures(*args, C.byref(p), None if m is None else C.byref(m), *targs, int(x0), int(y0), int(x1), int(y1), _p(img),
                                   None if feat is None else _p(feat), _p(luma2), cnt.ctypes.data_as(_u64), int(threads))
    del keep, tkeep
    if rc == -2:
        raise ValueError("invalid textured render")
    if rc != 0:
        raise RuntimeError("oracle_render_textures failed (%d)" % rc)
    return img, luma2, feat, _counters(cnt)


def render_adaptive(tris, nodes, cfg, textures, texcoords, texture_id, threshold, min_spp, check_interval, m=None, hdr=None, hdr_cache=None,
                    hdr_linear=True, window=None, threads=0):
    """(image, spp map, luma2, counters) of the adaptive render of the grid or a tile-aligned window with the textures."""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    tkeep, targs = _textures(textures, texcoords, texture_id, np.asarray(tris).shape[0])
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, spp, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.int32), np.zeros((h, w), np.float32)
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    a = AdaptiveParams()
    a.threshold, a.min_spp, a.check_interval, a.reserved = float(threshold), int(min_spp), int(check_interval), 0
    rc = _o.oracle_render_textures_adaptive(*args, C.byref(p), None if m is None else C.byref(m), *targs, C.byref(a), int(x0), int(y0), int(x1),
                                            int(y1), _p(img), spp.ctypes.data_as(_ip), _p(luma2), cnt.ctypes.data_as(_u64), int(threads))
    del keep, tkeep
    if rc == -2:
        raise ValueError("invalid textured render")
    if rc != 0:
        raise RuntimeError("oracle_render_textures_adaptive failed (%d)" % rc)
    return img, spp, luma2, _counters(cnt)
