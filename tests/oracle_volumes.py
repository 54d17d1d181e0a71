"""ctypes binding of the CPU restatement of the volumes inside transmissive meshes (tests/oracle_volumes.cpp ->
build/libezrt_oracle_volumes.so): ez_volume_sigma_a, and the render with RenderConfig.volumes in plain / window, feature-buffer and adaptive
forms, with every other option of the light sampling mode, and its BSDF-only estimator.  TEST INFRASTRUCTURE, like
tests/oracle_light_tree.py."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import build as _build
from ezrt_b200._lib import AdaptiveParams, Medium, PunctualLight, RenderParams, Texture
from tests.oracle_lens import _counters, _scene_args
from tests.oracle_light_tree import _topts
from tests.oracle_punctual import _opts

if not os.path.exists(_build.ORACLE_VOLUMES_SO):
    _build.build_oracle_volumes()
_o = C.CDLL(_build.ORACLE_VOLUMES_SO)

_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int32)
_up = C.POINTER(C.c_uint32)
_u64 = C.POINTER(C.c_uint64)
_LP = C.POINTER(PunctualLight)
_o.oracle_volume_sigma_a.restype = None
_o.oracle_volume_sigma_a.argtypes = [C.c_int, _fp, _fp, _fp]
_SCENE = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams)]
_OPTS = [C.POINTER(Medium), C.c_int, C.POINTER(Texture), _fp, _ip, _ip, _ip, C.c_int, _LP, _ip, _fp, _up, C.c_float]
_VOLS = [C.c_int, _fp, _ip]
_o.oracle_grid_render_set.restype = None
_o.oracle_grid_render_set.argtypes = [C.c_int, C.c_int, C.c_int, _fp, C.c_float]
_o.oracle_render_volumes.restype = C.c_int
_o.oracle_render_volumes.argtypes = _SCENE + _OPTS + _VOLS + [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _fp, _fp, _fp, _u64, C.c_int]
_o.oracle_render_volumes_adaptive.restype = C.c_int
_o.oracle_render_volumes_adaptive.argtypes = _SCENE + _OPTS + _VOLS + [C.POINTER(AdaptiveParams), C.c_int, C.c_int, C.c_int, C.c_int, _fp, _ip, _fp,
                                                                      _u64, C.c_int]


def _p(a):
    return a.ctypes.data_as(_fp)


def sigma_a(color, distance):
    """ez_volume_sigma_a elementwise over broadcast (colour channel, distance) arrays: float32"""
    c, d = np.broadcast_arrays(np.asarray(color, np.float32), np.asarray(distance, np.float32))
    c, d = np.ascontiguousarray(c.reshape(-1)), np.ascontiguousarray(d.reshape(-1))
    out = np.zeros(c.shape[0], np.float32)
    _o.oracle_volume_sigma_a(c.shape[0], _p(c), _p(d), _p(out))
    return out.reshape(np.broadcast(np.asarray(color), np.asarray(distance)).shape)


def table(volumes):
    """sigma_a [V, 3] of a sequence of (attenuation_color (3), attenuation_distance) pairs or api.volume values, as the library's"""
    cs, ds = [], []
    for v in volumes:
        if hasattr(v, "attenuation_color"):
            cs.append(list(v.attenuation_color)); ds.append(v.attenuation_distance)
        else:
            cs.append(list(v[0])); ds.append(v[1])
    c = np.asarray(cs, np.float32).reshape(-1, 3)
    d = np.asarray(ds, np.float32).reshape(-1, 1)
    return sigma_a(c, d).reshape(-1, 3)


def _vargs(tris, volumes, volume_id):
    n = np.asarray(tris).reshape(-1, 36).shape[0]
    if volumes is None or len(volumes) == 0:
        return [], [0, None, None]
    sig = np.ascontiguousarray(table(volumes), np.float32)
    ids = np.ascontiguousarray(np.asarray(volume_id, np.int32).reshape(n))
    return [sig, ids], [sig.shape[0], _p(sig), ids.ctypes.data_as(_ip)]


def _grid(cfg, rho):
    """the density grid of the renders that follow: rho [nz, ny, nx] with cfg.medium_grid, else none (the homogeneous medium)"""
    if rho is None or not cfg.medium_grid:
        _o.oracle_grid_render_set(0, 0, 0, None, 1.0)
        return None
    g = np.ascontiguousarray(np.asarray(rho, np.float32))
    nz, ny, nx = g.shape
    _o.oracle_grid_render_set(nx, ny, nz, _p(g), 1.0)
    return g


def render(tris, nodes, cfg, volumes=None, volume_id=None, emission_id=None, lights=None, m=None, textures=None, texcoords=None, texture_id=None,
           metal_rough_id=None, normal_id=None, hdr=None, hdr_cache=None, hdr_linear=True, window=None, aov=False, threads=0, tree=None,
           bsdf_only=False, mutate=False, mutate_flight=False, rho=None):
    """(image [h, w, C], luma2 [h, w], aov [h, w, 8] or None, counters) of the grid or of window = (x0, y0, x1, y1) as
    tests/oracle_light_tree.render, with cfg.volumes rendered by `volumes` (api.volume values or (colour, distance) pairs; None: no
    volumes) and the triangles' volume_id, with the medium m (ezrt_medium, tests/oracle_medium.medium) and with cfg.medium_grid its
    density grid rho [nz, ny, nx]; bsdf_only: the independent estimator, mutate: the first BSDF sample's hit not absorbed,
    mutate_flight: interior segments draw the medium's flight (all three test-only)"""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    okeep, oargs = _opts(tris, lights, m, textures, texcoords, texture_id, metal_rough_id, normal_id)
    tkeep, targs = _topts(tris, cfg, emission_id, tree, 1.0, textures, texcoords)
    vkeep, vargs = _vargs(tris, volumes, volume_id)
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.float32)
    feat = np.zeros((h, w, 8), np.float32) if aov else None
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    flags = int(bool(bsdf_only)) | (2 if mutate else 0) | (4 if mutate_flight else 0)
    g = _grid(cfg, rho)
    try:
        rc = _o.oracle_render_volumes(*args, C.byref(p), *oargs, *targs, *vargs, flags, int(x0), int(y0), int(x1), int(y1), _p(img),
                                      None if feat is None else _p(feat), _p(luma2), cnt.ctypes.data_as(_u64), int(threads))
    finally:
        _o.oracle_grid_render_set(0, 0, 0, None, 1.0)
    del keep, okeep, tkeep, vkeep, g
    if rc == -2:
        raise ValueError("invalid volumes render")
    if rc != 0:
        raise RuntimeError("oracle_render_volumes failed (%d)" % rc)
    return img, luma2, feat, _counters(cnt)


def render_adaptive(tris, nodes, cfg, threshold, min_spp, check_interval, volumes=None, volume_id=None, emission_id=None, lights=None, m=None,
                    textures=None, texcoords=None, texture_id=None, metal_rough_id=None, normal_id=None, hdr=None, hdr_cache=None, hdr_linear=True,
                    window=None, threads=0, rho=None):
    """(image, spp map, luma2, counters) of the adaptive render of the grid or a tile-aligned window with the volumes (and the medium m
    with the grid rho, as render)."""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    okeep, oargs = _opts(tris, lights, m, textures, texcoords, texture_id, metal_rough_id, normal_id)
    tkeep, targs = _topts(tris, cfg, emission_id, None, 1.0, textures, texcoords)
    vkeep, vargs = _vargs(tris, volumes, volume_id)
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, spp, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.int32), np.zeros((h, w), np.float32)
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    a = AdaptiveParams()
    a.threshold, a.min_spp, a.check_interval, a.reserved = float(threshold), int(min_spp), int(check_interval), 0
    g = _grid(cfg, rho)
    try:
        rc = _o.oracle_render_volumes_adaptive(*args, C.byref(p), *oargs, *targs, *vargs, C.byref(a), int(x0), int(y0), int(x1), int(y1), _p(img),
                                               spp.ctypes.data_as(_ip), _p(luma2), cnt.ctypes.data_as(_u64), int(threads))
    finally:
        _o.oracle_grid_render_set(0, 0, 0, None, 1.0)
    del keep, okeep, tkeep, vkeep, g
    if rc == -2:
        raise ValueError("invalid volumes render")
    if rc != 0:
        raise RuntimeError("oracle_render_volumes_adaptive failed (%d)" % rc)
    return img, spp, luma2, _counters(cnt)
