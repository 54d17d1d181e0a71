"""ctypes binding of the CPU restatement of the light tree (tests/oracle_light_tree.cpp -> build/libezrt_oracle_light_tree.so): the
builder's inputs for a render's table, ezrt_math.h's descent and hit-side walk, and the render with RenderConfig.light_tree in plain /
window, feature-buffer and adaptive forms, with every other option of the light sampling mode.  The tree itself is the library's host
builder's (api.build_light_tree).  TEST INFRASTRUCTURE, like tests/oracle_emission_maps.py."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import api
from ezrt_b200 import build as _build
from ezrt_b200._lib import AdaptiveParams, Medium, PunctualLight, RenderParams, Texture
from tests.oracle_lens import _counters, _scene_args
from tests.oracle_material_maps import _maps
from tests.oracle_punctual import _opts

if not os.path.exists(_build.ORACLE_LIGHT_TREE_SO):
    _build.build_oracle_light_tree()
_o = C.CDLL(_build.ORACLE_LIGHT_TREE_SO)

_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int32)
_up = C.POINTER(C.c_uint32)
_u64 = C.POINTER(C.c_uint64)
_LP = C.POINTER(PunctualLight)
_o.oracle_light_tree_table.restype = C.c_int
_o.oracle_light_tree_table.argtypes = [_fp, C.c_int, _fp, C.c_int, C.c_int, C.POINTER(Texture), _fp, _ip, C.c_int, _fp, _fp]
_o.oracle_light_tree_eval.restype = None
_o.oracle_light_tree_eval.argtypes = [_fp, _up, C.c_int, C.c_int, _fp, _fp, _ip, _ip, _fp]
_SCENE = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams)]
_OPTS = [C.POINTER(Medium), C.c_int, C.POINTER(Texture), _fp, _ip, _ip, _ip, C.c_int, _LP, _ip, _fp, _up, C.c_float]
_o.oracle_render_light_tree.restype = C.c_int
_o.oracle_render_light_tree.argtypes = _SCENE + _OPTS + [C.c_int, C.c_int, C.c_int, C.c_int, _fp, _fp, _fp, _u64, C.c_int]
_o.oracle_render_light_tree_adaptive.restype = C.c_int
_o.oracle_render_light_tree_adaptive.argtypes = _SCENE + _OPTS + [C.POINTER(AdaptiveParams), C.c_int, C.c_int, C.c_int, C.c_int, _fp, _ip, _fp,
                                                                  _u64, C.c_int]


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if shape is None else a.reshape(shape)


def _p(a):
    return a.ctypes.data_as(_fp)


def table_inputs(tris, emission_id=None, textures=None, texcoords=None):
    """(verts [K, 9], weights [K]) of the render's table -- mode 4's, or the emission table of emission_id -- as ezrt_light_tree_build
    takes them"""
    tris = _f32(tris, (-1, 36))
    n = tris.shape[0]
    keep, a = [], [0, None, None]
    ids = None
    if emission_id is not None:
        keep, a = _maps(textures, texcoords, np.full(n, -1, np.int32), np.full(n, -1, np.int32), np.full(n, -1, np.int32), n)
        ids = np.ascontiguousarray(np.asarray(emission_id, np.int32).reshape(n))
    cap = max(1, n)
    verts, w = np.zeros((cap, 9), np.float32), np.zeros(cap, np.float32)
    k = _o.oracle_light_tree_table(_p(tris), n, None, 0, a[0], a[1], a[2], None if ids is None else ids.ctypes.data_as(_ip), cap, _p(verts), _p(w))
    del keep
    if k < 0:
        raise ValueError("invalid emission maps")
    return verts[:k], w[:k]


def tree_of(tris, emission_id=None, textures=None, texcoords=None):
    """api.build_light_tree over the render's table (the tree the library renders with)"""
    v, w = table_inputs(tris, emission_id, textures, texcoords)
    return api.build_light_tree(v, w)


def descend(tree, P, r):
    """ezrt_math.h's descent: (light int32 [n], -1 for no sample; P_sel float32 [n])"""
    P, r = _f32(P, (-1, 3)), _f32(r, (-1,))
    k, q = np.zeros(P.shape[0], np.int32), np.zeros(P.shape[0], np.float32)
    _o.oracle_light_tree_eval(_p(tree["nodes"]), tree["paths"].ctypes.data_as(_up), 0, P.shape[0], _p(P), _p(r), None, k.ctypes.data_as(_ip), _p(q))
    return k, q


def prob(tree, P, light):
    """ezrt_math.h's hit-side walk: P_sel float32 [n] of lights light [n] at P [n, 3]"""
    P = _f32(P, (-1, 3))
    light = np.ascontiguousarray(np.asarray(light, np.int32).reshape(-1))
    q = np.zeros(P.shape[0], np.float32)
    _o.oracle_light_tree_eval(_p(tree["nodes"]), tree["paths"].ctypes.data_as(_up), 1, P.shape[0], _p(P), None, light.ctypes.data_as(_ip), None, _p(q))
    return q


def _topts(tris, cfg, emission_id, tree, mis_scale, textures, texcoords):
    n = np.asarray(tris).reshape(-1, 36).shape[0]
    ids = None if emission_id is None else np.ascontiguousarray(np.asarray(emission_id, np.int32).reshape(n))
    if tree is None and cfg.light_tree:
        tree = tree_of(tris, emission_id if cfg.emission_maps else None, textures, texcoords)
    nodes = None if tree is None else np.ascontiguousarray(tree["nodes"], np.float32)
    paths = None if tree is None else np.ascontiguousarray(tree["paths"], np.uint32)
    keep = [ids, nodes, paths]
    return keep, [None if ids is None else ids.ctypes.data_as(_ip), None if nodes is None or nodes.size == 0 else _p(nodes),
                  None if paths is None or paths.size == 0 else paths.ctypes.data_as(_up), float(mis_scale)]


def render(tris, nodes, cfg, emission_id=None, lights=None, m=None, textures=None, texcoords=None, texture_id=None, metal_rough_id=None,
           normal_id=None, hdr=None, hdr_cache=None, hdr_linear=True, window=None, aov=False, threads=0, tree=None, mis_scale=1.0):
    """(image [h, w, C], luma2 [h, w], aov [h, w, 8] or None, counters) of the grid or of window = (x0, y0, x1, y1) as
    tests/oracle_emission_maps.render, with cfg.light_tree rendered by `tree` (default: the library's builder over the render's table);
    mis_scale scales the emission hits' P_sel (test-only)"""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    okeep, oargs = _opts(tris, lights, m, textures, texcoords, texture_id, metal_rough_id, normal_id)
    tkeep, targs = _topts(tris, cfg, emission_id, tree, mis_scale, textures, texcoords)
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.float32)
    feat = np.zeros((h, w, 8), np.float32) if aov else None
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    rc = _o.oracle_render_light_tree(*args, C.byref(p), *oargs, *targs, int(x0), int(y0), int(x1), int(y1), _p(img),
                                     None if feat is None else _p(feat), _p(luma2), cnt.ctypes.data_as(_u64), int(threads))
    del keep, okeep, tkeep
    if rc == -2:
        raise ValueError("invalid light-tree render")
    if rc != 0:
        raise RuntimeError("oracle_render_light_tree failed (%d)" % rc)
    return img, luma2, feat, _counters(cnt)


def render_adaptive(tris, nodes, cfg, threshold, min_spp, check_interval, emission_id=None, lights=None, m=None, textures=None, texcoords=None,
                    texture_id=None, metal_rough_id=None, normal_id=None, hdr=None, hdr_cache=None, hdr_linear=True, window=None, threads=0):
    """(image, spp map, luma2, counters) of the adaptive render of the grid or a tile-aligned window with the light tree."""
    keep, args = _scene_args(tris, nodes, hdr, hdr_cache, hdr_linear)
    okeep, oargs = _opts(tris, lights, m, textures, texcoords, texture_id, metal_rough_id, normal_id)
    tkeep, targs = _topts(tris, cfg, emission_id, None, 1.0, textures, texcoords)
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    h, w = y1 - y0, x1 - x0
    img, spp, luma2 = np.zeros((h, w, cfg.out_channels), np.float32), np.zeros((h, w), np.int32), np.zeros((h, w), np.float32)
    cnt = np.zeros(9, np.uint64)
    p = cfg.to_struct()
    a = AdaptiveParams()
    a.threshold, a.min_spp, a.check_interval, a.reserved = float(threshold), int(min_spp), int(check_interval), 0
    rc = _o.oracle_render_light_tree_adaptive(*args, C.byref(p), *oargs, *targs, C.byref(a), int(x0), int(y0), int(x1), int(y1), _p(img),
                                              spp.ctypes.data_as(_ip), _p(luma2), cnt.ctypes.data_as(_u64), int(threads))
    del keep, okeep, tkeep
    if rc == -2:
        raise ValueError("invalid light-tree render")
    if rc != 0:
        raise RuntimeError("oracle_render_light_tree_adaptive failed (%d)" % rc)
    return img, spp, luma2, _counters(cnt)
