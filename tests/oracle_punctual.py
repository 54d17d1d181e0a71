"""ctypes binding of the CPU restatement of the punctual lights (tests/oracle_punctual.cpp -> build/libezrt_oracle_punctual.so): the
table, the sample, and the render with RenderConfig.punctual_lights in plain / window, feature-buffer and adaptive forms, with every
other option of the light sampling mode.  TEST INFRASTRUCTURE, like tests/oracle_material_maps.py."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import api
from ezrt_b200 import build as _build
from ezrt_b200._lib import AdaptiveParams, Medium, PunctualLight, RenderParams, Texture
from tests.oracle_lens import _counters, _scene_args
from tests.oracle_material_maps import _maps

if not os.path.exists(_build.ORACLE_PUNCTUAL_SO):
    _build.build_oracle_punctual()
_o = C.CDLL(_build.ORACLE_PUNCTUAL_SO)

_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int32)
_u64 = C.POINTER(C.c_uint64)
_LP = C.POINTER(PunctualLight)
_o.oracle_punct_table.restype = C.c_int
_o.oracle_punct_table.argtypes = [_fp, C.c_int, C.c_int, _LP, C.c_int, _ip, _fp, _fp, _fp, C.POINTER(C.c_double)]
_o.oracle_punct_sample.restype = None
_o.oracle_punct_sample.argtypes = [C.c_int, _fp, _fp, _fp, _fp, _ip, _ip, _fp, _fp, _fp]
_SCENE = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams)]
_OPTS = [C.POINTER(Medium), C.c_int, C.POINTER(Texture), _fp, _ip, _ip, _ip, C.c_int, _LP]
_o.oracle_render_punctual.restype = C.c_int
_o.oracle_render_punctual.argtypes = _SCENE + _OPTS + [C.c_int, C.c_int, C.c_int, C.c_int, _fp, _fp, _fp, _u64, C.c_int]
_o.oracle_render_punctual_adaptive.restype = C.c_int
_o.oracle_render_punctual_adaptive.argtypes = _SCENE + _OPTS + [C.POINTER(AdaptiveParams), C.c_int, C.c_int, C.c_int, C.c_int, _fp, _ip, _fp,
                                                               _u64, C.c_int]


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if shape is None else a.reshape(shape)


def _p(a):
    return a.ctypes.data_as(_fp)


def table(tris, lights):
    """(index int32 [J], cdf [J], q [J], records float32 [J, 16], W) of the lights over the triangles' vertex box; ValueError (with the
    invalid light's index as .args[1]) where ezrt_scene_set_punctual_lights returns EZRT_ERR_INVALID"""
    tris = _f32(tris, (-1, 36))
    arr, n = api.punctual_array(lights)
    cap = max(1, n)
    idx, cdf, q, rec = np.zeros(cap, np.int32), np.zeros(cap, np.float32), np.zeros(cap, np.float32), np.zeros((cap, 16), np.float32)
    total = C.c_double(0.0)
    j = _o.oracle_punct_table(_p(tris), tris.shape[0], n, arr, cap, idx.ctypes.data_as(_ip), _p(cdf), _p(q), _p(rec), C.byref(total))
    if j < 0:
        raise ValueError("invalid punctual light", -1 - j)
    return idx[:j], cdf[:j], q[:j], rec[:j], total.value


def sample(rec, pq, P, N, medium):
    """ez_punct_sample of rows: records [n, 16], pq [n], P [n, 3], N [n, 3], medium [n] -> (ok bool [n], L [n, 3], tmax [n], s [n])"""
    rec, P, N = _f32(rec, (-1, 16)), _f32(P, (-1, 3)), _f32(N, (-1, 3))
    n = rec.shape[0]
    pq = _f32(np.broadcast_to(np.asarray(pq, np.float32), (n,)))
    med = np.ascontiguousarray(np.broadcast_to(np.asarray(medium, np.int32), (n,)))
    ok, L, tmax, s = np.zeros(n, np.int32), np.zeros((n, 3), np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)
    _o.oracle_punct_sample(n, _p(rec), _p(pq), _p(P), _p(N), med.ctypes.data_as(_ip), ok.ctypes.data_as(_ip), _p(L), _p(tmax), _p(s))
    return ok != 0, L, tmax, s


def _opts(tris, lights, m, textures, texcoords, texture_id, metal_rough_id, normal_id):
    n = np.asarray(tris).reshape(-1, 36).shape[0]
    keep, args = [], [None if m is None else C.byref(m)]
    if textures is None:
        args += [0, None, None, None, None, None]
    else:
        if metal_rough_id is None:
            metal_rough_id = normal_id = np.full(n, -1, np.int32)
        k, a = _maps(textures, texcoords, texture_id, metal_rough_id, normal_id, n)
        keep.append(k)
        args += a
    if lights is None:
        args += [0, None]
    else:
        arr, nl = api.punctual_array(lights)
        keep.append(arr)
        args += [nl, arr]
    return keep, args


def render(tris, nodes, cfg, lights, m=None, textures=None, texcoords=None, texture_id=None, metal_rough_id=None, normal_id=None, hdr=None,
           hdr_cache=None, hdr_linear=True, window=None, aov=False, threads=0):
    """(image [h, w, C], luma2 [h, w], aov [h, w, 8] or None, counters) of the grid or of window = (x0, y0, x1, y1) with the punctual
    lights (as Scene.set_punctual_lights takes them), the medium m (oracle_medium.medium, for cfg.medium) and the textures and maps (as
    Scene.set_textures / set_material_maps take them, for cfg.textures / cfg.material_maps); ValueError where the library returns
    EZRT_ERR_INVALID."""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    okeep, oargs = _opts(tris, lights, m, textures, texcoords, texture_id, metal_rough_id, normal_id)
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.float32)
    feat = np.zeros((h, w, 8), np.float32) if aov else None
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    rc = _o.oracle_render_punctual(*args, C.byref(p), *oargs, int(x0), int(y0), int(x1), int(y1), _p(img), None if feat is None else _p(feat),
                                   _p(luma2), cnt.ctypes.data_as(_u64), int(threads))
    del keep, okeep
    if rc == -2:
        raise ValueError("invalid punctual render")
    if rc != 0:
        raise RuntimeError("oracle_render_punctual failed (%d)" % rc)
    return img, luma2, feat, _counters(cnt)


def render_adaptive(tris, nodes, cfg, lights, threshold, min_spp, check_interval, m=None, textures=None, texcoords=None, texture_id=None,
                    metal_rough_id=None, normal_id=None, hdr=None, hdr_cache=None, hdr_linear=True, window=None, threads=0):
    """(image, spp map, luma2, counters) of the adaptive render of the grid or a tile-aligned window with the punctual lights."""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    okeep, oargs = _opts(tris, lights, m, textures, texcoords, texture_id, metal_rough_id, normal_id)
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, spp, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.int32), np.zeros((h, w), np.float32)
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    a = AdaptiveParams()
    a.threshold, a.min_spp, a.check_interval, a.reserved = float(threshold), int(min_spp), int(check_interval), 0
    rc = _o.oracle_render_punctual_adaptive(*args, C.byref(p), *oargs, C.byref(a), int(x0), int(y0), int(x1), int(y1), _p(img),
                                            spp.ctypes.data_as(_ip), _p(luma2), cnt.ctypes.data_as(_u64), int(threads))
    del keep, okeep
    if rc == -2:
        raise ValueError("invalid punctual render")
    if rc != 0:
        raise RuntimeError("oracle_render_punctual_adaptive failed (%d)" % rc)
    return img, spp, luma2, _counters(cnt)
