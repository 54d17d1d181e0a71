"""ctypes binding of the CPU restatement of the emission maps (tests/oracle_emission_maps.cpp -> build/libezrt_oracle_emission_maps.so):
the C table weight, E(Q), the emission table, and the render with RenderConfig.emission_maps in plain / window, feature-buffer and
adaptive forms, with every other option of the light sampling mode.  TEST INFRASTRUCTURE, like tests/oracle_punctual.py."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import build as _build
from ezrt_b200._lib import AdaptiveParams, Medium, PunctualLight, RenderParams, Texture
from tests.oracle_lens import _counters, _scene_args
from tests.oracle_material_maps import _maps
from tests.oracle_punctual import _opts

if not os.path.exists(_build.ORACLE_EMISSION_MAPS_SO):
    _build.build_oracle_emission_maps()
_o = C.CDLL(_build.ORACLE_EMISSION_MAPS_SO)

_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int32)
_up = C.POINTER(C.c_uint32)
_u64 = C.POINTER(C.c_uint64)
_LP = C.POINTER(PunctualLight)
_o.oracle_emit_lum_eff.restype = None
_o.oracle_emit_lum_eff.argtypes = [C.c_int, _fp, _fp, _up, C.c_int, C.c_int, _fp]
_o.oracle_emit_eval.restype = None
_o.oracle_emit_eval.argtypes = [C.c_int, _fp, _fp, _fp, _fp, _fp, _up, C.c_int, C.c_int, _fp]
_o.oracle_emission_table.restype = C.c_int
_o.oracle_emission_table.argtypes = [_fp, C.c_int, _fp, C.c_int, C.c_int, C.POINTER(Texture), _fp, _ip, C.c_int, _ip, _fp, _fp, _fp,
                                     C.POINTER(C.c_double)]
_o.oracle_emission_pdf_pairs.restype = C.c_int
_o.oracle_emission_pdf_pairs.argtypes = [_fp, C.c_int, _fp, C.c_int, C.c_int, C.POINTER(Texture), _fp, _ip, C.c_int, C.c_int, _fp, _fp, _fp, _fp, _fp]
_SCENE = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams)]
_OPTS = [C.POINTER(Medium), C.c_int, C.POINTER(Texture), _fp, _ip, _ip, _ip, C.c_int, _LP, _ip, _fp, C.c_float]
_o.oracle_render_emission_maps.restype = C.c_int
_o.oracle_render_emission_maps.argtypes = _SCENE + _OPTS + [C.c_int, C.c_int, C.c_int, C.c_int, _fp, _fp, _fp, _u64, C.c_int]
_o.oracle_render_emission_maps_adaptive.restype = C.c_int
_o.oracle_render_emission_maps_adaptive.argtypes = _SCENE + _OPTS + [C.POINTER(AdaptiveParams), C.c_int, C.c_int, C.c_int, C.c_int, _fp, _ip,
                                                                     _fp, _u64, C.c_int]


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if shape is None else a.reshape(shape)


def _p(a):
    return a.ctypes.data_as(_fp)


def _words(img):
    """RGBA8 words of a uint8 image [H, W, 3 or 4] (alpha 255 where absent), row 0 on top"""
    img = np.asarray(img, np.uint8)
    if img.shape[2] == 3:
        img = np.concatenate([img, np.full(img.shape[:2] + (1,), 255, np.uint8)], axis=2)
    return np.ascontiguousarray(img).view(np.uint32).reshape(img.shape[:2])


def lum_eff(E, uv6, img):
    """ez_emit_lum_eff of rows E [n, 3], uv6 [n, 6] over the texture img (uint8 [H, W, 3|4])"""
    E, uv6 = _f32(E, (-1, 3)), _f32(uv6, (-1, 6))
    w = _words(img)
    out = np.zeros(E.shape[0], np.float32)
    _o.oracle_emit_lum_eff(E.shape[0], _p(E), _p(uv6), w.ctypes.data_as(_up), w.shape[1], w.shape[0], _p(out))
    return out


def emit_eval(E, Q, P, Ng, uv6, img):
    """ez_emit_eval of rows E [n, 3], Q [n, 3], vertices P [n, 9], Ng [n, 3], uv6 [n, 6] over img -> [n, 3]"""
    E, Q, P, Ng, uv6 = _f32(E, (-1, 3)), _f32(Q, (-1, 3)), _f32(P, (-1, 9)), _f32(Ng, (-1, 3)), _f32(uv6, (-1, 6))
    w = _words(img)
    out = np.zeros((E.shape[0], 3), np.float32)
    _o.oracle_emit_eval(E.shape[0], _p(E), _p(Q), _p(P), _p(Ng), _p(uv6), w.ctypes.data_as(_up), w.shape[1], w.shape[0], _p(out))
    return out


def table(tris, textures, texcoords, emission_id):
    """(triangles int32 [K], cdf [K], record lum_eff [K], the lum an emission hit on each light uses [K], W) of the emission table;
    ValueError where ezrt_scene_set_emission_maps returns EZRT_ERR_INVALID"""
    tris = _f32(tris, (-1, 36))
    n = tris.shape[0]
    keep, a = _maps(textures, texcoords, np.full(n, -1, np.int32), np.full(n, -1, np.int32), np.full(n, -1, np.int32), n)
    nt, tex, uv = a[0], a[1], a[2]
    ids = np.ascontiguousarray(np.asarray(emission_id, np.int32).reshape(n))
    cap = max(1, n)
    tri, cdf, lum, hl = np.zeros(cap, np.int32), np.zeros(cap, np.float32), np.zeros(cap, np.float32), np.zeros(cap, np.float32)
    total = C.c_double(0.0)
    k = _o.oracle_emission_table(_p(tris), n, None, 0, nt, tex, uv, ids.ctypes.data_as(_ip), cap, tri.ctypes.data_as(_ip), _p(cdf), _p(lum),
                                 _p(hl), C.byref(total))
    del keep
    if k < 0:
        raise ValueError("invalid emission maps")
    return tri[:k], cdf[:k], lum[:k], hl[:k], total.value


def pdf_pairs(tris, nodes, textures, texcoords, emission_id, P, seed=0):
    """(light triangles [K], sample_pdf [K, m], hit_pdf [K, m], traced_pdf [K, m]) of a point on every light of the emission table seen
    from each shading point P [m, 3]: the light sample's pdf and the emission hit's pdf of that point through the restatement's two code
    paths, at the sample's distance and at the traced hit's (-1: no light, or another triangle hit first)"""
    tris = _f32(tris, (-1, 36))
    n = tris.shape[0]
    nodes = _f32(nodes, (-1, 12))
    keep, a = _maps(textures, texcoords, np.full(n, -1, np.int32), np.full(n, -1, np.int32), np.full(n, -1, np.int32), n)
    ids = np.ascontiguousarray(np.asarray(emission_id, np.int32).reshape(n))
    P = _f32(P, (-1, 3))
    t = table(tris, textures, texcoords, emission_id)[0]
    K, m = len(t), P.shape[0]
    r = _f32(np.random.default_rng(seed).uniform(0, 1, (max(K, 1), m, 2)))
    sp, hp, tp = (np.zeros((max(K, 1), m), np.float32) for _ in range(3))
    k = _o.oracle_emission_pdf_pairs(_p(tris), n, _p(nodes), nodes.shape[0], a[0], a[1], a[2], ids.ctypes.data_as(_ip), K, m, _p(P), _p(r), _p(sp),
                                     _p(hp), _p(tp))
    del keep
    assert k == K
    return t, sp[:K], hp[:K], tp[:K]


def _eopts(tris, emission_id, lum_eff, mis_scale):
    n = np.asarray(tris).reshape(-1, 36).shape[0]
    keep = []
    ids = None if emission_id is None else np.ascontiguousarray(np.asarray(emission_id, np.int32).reshape(n))
    le = None if lum_eff is None else _f32(lum_eff, (n,))
    keep += [ids, le]
    return keep, [None if ids is None else ids.ctypes.data_as(_ip), None if le is None else _p(le), float(mis_scale)]


def render(tris, nodes, cfg, emission_id, lights=None, m=None, textures=None, texcoords=None, texture_id=None, metal_rough_id=None,
           normal_id=None, hdr=None, hdr_cache=None, hdr_linear=True, window=None, aov=False, threads=0, lum_eff=None, mis_scale=1.0):
    """(image [h, w, C], luma2 [h, w], aov [h, w, 8] or None, counters) of the grid or of window = (x0, y0, x1, y1) with the emission
    maps emission_id (as Scene.set_emission_maps takes them, for cfg.emission_maps), the punctual lights, the medium m and the textures
    and maps; lum_eff [N] and mis_scale are the restatement's test-only inputs (tests/oracle_emission_maps.cpp); ValueError where the
    library returns EZRT_ERR_INVALID."""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    okeep, oargs = _opts(tris, lights, m, textures, texcoords, texture_id, metal_rough_id, normal_id)
    ekeep, eargs = _eopts(tris, emission_id, lum_eff, mis_scale)
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.float32)
    feat = np.zeros((h, w, 8), np.float32) if aov else None
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    rc = _o.oracle_render_emission_maps(*args, C.byref(p), *oargs, *eargs, int(x0), int(y0), int(x1), int(y1), _p(img),
                                        None if feat is None else _p(feat), _p(luma2), cnt.ctypes.data_as(_u64), int(threads))
    del keep, okeep, ekeep
    if rc == -2:
        raise ValueError("invalid emission-map render")
    if rc != 0:
        raise RuntimeError("oracle_render_emission_maps failed (%d)" % rc)
    return img, luma2, feat, _counters(cnt)


def render_adaptive(tris, nodes, cfg, emission_id, threshold, min_spp, check_interval, lights=None, m=None, textures=None, texcoords=None,
                    texture_id=None, metal_rough_id=None, normal_id=None, hdr=None, hdr_cache=None, hdr_linear=True, window=None, threads=0):
    """(image, spp map, luma2, counters) of the adaptive render of the grid or a tile-aligned window with the emission maps."""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    okeep, oargs = _opts(tris, lights, m, textures, texcoords, texture_id, metal_rough_id, normal_id)
    ekeep, eargs = _eopts(tris, emission_id, None, 1.0)
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, spp, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.int32), np.zeros((h, w), np.float32)
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    a = AdaptiveParams()
    a.threshold, a.min_spp, a.check_interval, a.reserved = float(threshold), int(min_spp), int(check_interval), 0
    rc = _o.oracle_render_emission_maps_adaptive(*args, C.byref(p), *oargs, *eargs, C.byref(a), int(x0), int(y0), int(x1), int(y1), _p(img),
                                                 spp.ctypes.data_as(_ip), _p(luma2), cnt.ctypes.data_as(_u64), int(threads))
    del keep, okeep, ekeep
    if rc == -2:
        raise ValueError("invalid emission-map render")
    if rc != 0:
        raise RuntimeError("oracle_render_emission_maps_adaptive failed (%d)" % rc)
    return img, spp, luma2, _counters(cnt)
