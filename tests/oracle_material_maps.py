"""ctypes binding of the CPU restatement of the material maps (tests/oracle_material_maps.cpp -> build/libezrt_oracle_material_maps.so):
the definition's table, tangent frame, mapped normal and maps filter, and the render with RenderConfig.material_maps in plain / window,
feature-buffer and adaptive forms.  TEST INFRASTRUCTURE, like tests/oracle_textures.py."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import build as _build
from ezrt_b200._lib import AdaptiveParams, Medium, RenderParams, Texture
from tests.oracle_lens import _counters, _scene_args
from tests.oracle_textures import _rgba, _textures

if not os.path.exists(_build.ORACLE_MATERIAL_MAPS_SO):
    _build.build_oracle_material_maps()
_o = C.CDLL(_build.ORACLE_MATERIAL_MAPS_SO)

_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int32)
_u64 = C.POINTER(C.c_uint64)
_o.oracle_unorm8_table.restype = None
_o.oracle_unorm8_table.argtypes = [_fp]
_o.oracle_unorm_sample.restype = None
_o.oracle_unorm_sample.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, _fp, _fp]
_o.oracle_mr_apply.restype = None
_o.oracle_mr_apply.argtypes = [C.c_int, _fp, _fp]
_o.oracle_tangent_frame.restype = None
_o.oracle_tangent_frame.argtypes = [C.c_int, _fp, _fp, _fp, _fp, _ip]
_o.oracle_normal_map.restype = None
_o.oracle_normal_map.argtypes = [C.c_int, _fp, _fp, _fp, _fp, _fp, _ip, _fp, _fp]
_SCENE = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams)]
_MAPS = [C.POINTER(Medium), C.c_int, C.POINTER(Texture), _fp, _ip, _ip, _ip]
_o.oracle_render_material_maps.restype = C.c_int
_o.oracle_render_material_maps.argtypes = _SCENE + _MAPS + [C.c_int, C.c_int, C.c_int, C.c_int, _fp, _fp, _fp, _u64, C.c_int]
_o.oracle_render_material_maps_adaptive.restype = C.c_int
_o.oracle_render_material_maps_adaptive.argtypes = _SCENE + _MAPS + [C.POINTER(AdaptiveParams), C.c_int, C.c_int, C.c_int, C.c_int, _fp, _ip, _fp,
                                                                       _u64, C.c_int]


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if shape is None else a.reshape(shape)


def _p(a):
    return a.ctypes.data_as(_fp)


def _i(a):
    return a.ctypes.data_as(_ip)


def unorm8_table():
    out = np.zeros(256, np.float32)
    _o.oracle_unorm8_table(_p(out))
    return out


def unorm_sample(tex, uv):
    """ez_tex_sample with ez_unorm8_table of the uint8 texture [H, W, 3|4] at rows uv [n, 2] -> [n, 3]"""
    t = _rgba(tex)
    uv = _f32(uv, (-1, 2))
    out = np.zeros((uv.shape[0], 3), np.float32)
    _o.oracle_unorm_sample(t.ctypes.data, t.shape[1], t.shape[0], uv.shape[0], _p(uv), _p(out))
    return out


def mr_apply(f, roughness, metallic):
    """ez_mr_apply of filtered colours f [n, 3] -> (roughness [n], metallic [n])"""
    f = _f32(f, (-1, 3))
    rm = np.ascontiguousarray(np.stack([_f32(roughness).reshape(-1), _f32(metallic).reshape(-1)], axis=1))
    _o.oracle_mr_apply(f.shape[0], _p(f), _p(rm))
    return rm[:, 0], rm[:, 1]


def tangent_frame(p, uv6, No):
    """ez_tangent_frame of triangles p [n, 3, 3], UVs uv6 [n, 6] about No [n, 3] -> (T' [n, 3], B [n, 3], ok [n] bool)"""
    p, uv6, No = _f32(p, (-1, 9)), _f32(uv6, (-1, 6)), _f32(No, (-1, 3))
    tb = np.zeros((p.shape[0], 6), np.float32)
    ok = np.zeros(p.shape[0], np.int32)
    _o.oracle_tangent_frame(p.shape[0], _p(p), _p(uv6), _p(No), _p(tb), _i(ok))
    return tb[:, :3], tb[:, 3:], ok != 0


def normal_map(p, uv6, uv, f, N, inside, V):
    """ez_normal_map of rows: triangles p [n, 3, 3], UVs uv6 [n, 6], the hit's uv [n, 2], the filtered colour f [n, 3], surface_hit's N
    [n, 3], inside [n], V [n, 3] -> the shading normal [n, 3]"""
    p, uv6, uv, f, N, V = _f32(p, (-1, 9)), _f32(uv6, (-1, 6)), _f32(uv, (-1, 2)), _f32(f, (-1, 3)), _f32(N, (-1, 3)), _f32(V, (-1, 3))
    ins = np.ascontiguousarray(np.asarray(inside, np.int32).reshape(-1))
    out = np.zeros((p.shape[0], 3), np.float32)
    _o.oracle_normal_map(p.shape[0], _p(p), _p(uv6), _p(uv), _p(f), _p(N), _i(ins), _p(V), _p(out))
    return out


def _maps(textures, texcoords, texture_id, metal_rough_id, normal_id, n):
    tkeep, targs = _textures(textures, texcoords, texture_id, n)
    mr = np.ascontiguousarray(np.asarray(metal_rough_id, np.int32).reshape(n))
    nm = np.ascontiguousarray(np.asarray(normal_id, np.int32).reshape(n))
    return (tkeep, mr, nm), targs + [_i(mr), _i(nm)]


def render(tris, nodes, cfg, textures, texcoords, texture_id, metal_rough_id, normal_id, m=None, hdr=None, hdr_cache=None, hdr_linear=True,
           window=None, aov=False, threads=0):
    """(image [h, w, C], luma2 [h, w], aov [h, w, 8] or None, counters) of the grid or of window = (x0, y0, x1, y1) with the textures
    (as Scene.set_textures takes them), the maps' ids (as Scene.set_material_maps takes them) and the medium m (oracle_medium.medium,
    for cfg.medium); ValueError where the library returns EZRT_ERR_INVALID."""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    mkeep, margs = _maps(textures, texcoords, texture_id, metal_rough_id, normal_id, np.asarray(tris).shape[0])
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.float32)
    feat = np.zeros((h, w, 8), np.float32) if aov else None
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    rc = _o.oracle_render_material_maps(*args, C.byref(p), None if m is None else C.byref(m), *margs, int(x0), int(y0), int(x1), int(y1), _p(img),
                                        None if feat is None else _p(feat), _p(luma2), cnt.ctypes.data_as(_u64), int(threads))
    del keep, mkeep
    if rc == -2:
        raise ValueError("invalid material-maps render")
    if rc != 0:
        raise RuntimeError("oracle_render_material_maps failed (%d)" % rc)
    return img, luma2, feat, _counters(cnt)


def render_adaptive(tris, nodes, cfg, textures, texcoords, texture_id, metal_rough_id, normal_id, threshold, min_spp, check_interval, m=None,
                    hdr=None, hdr_cache=None, hdr_linear=True, window=None, threads=0):
    """(image, spp map, luma2, counters) of the adaptive render of the grid or a tile-aligned window with the textures and maps."""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    mkeep, margs = _maps(textures, texcoords, texture_id, metal_rough_id, normal_id, np.asarray(tris).shape[0])
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, spp, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.int32), np.zeros((h, w), np.float32)
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    a = AdaptiveParams()
    a.threshold, a.min_spp, a.check_interval, a.reserved = float(threshold), int(min_spp), int(check_interval), 0
    rc = _o.oracle_render_material_maps_adaptive(*args, C.byref(p), None if m is None else C.byref(m), *margs, C.byref(a), int(x0), int(y0),
                                                 int(x1), int(y1), _p(img), spp.ctypes.data_as(_ip), _p(luma2), cnt.ctypes.data_as(_u64),
                                                 int(threads))
    del keep, mkeep
    if rc == -2:
        raise ValueError("invalid material-maps render")
    if rc != 0:
        raise RuntimeError("oracle_render_material_maps_adaptive failed (%d)" % rc)
    return img, spp, luma2, _counters(cnt)
