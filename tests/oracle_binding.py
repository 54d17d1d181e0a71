"""ctypes binding of the CPU oracle (oracle/libezrt_oracle.so).  TEST INFRASTRUCTURE: only
tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs import this module."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import build as _build
from ezrt_b200._lib import RenderParams

if not os.path.exists(_build.ORACLE_SO):
    _build.build_oracle()
_o = C.CDLL(_build.ORACLE_SO)

_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int32)
_u64p = C.POINTER(C.c_uint64)
_o.oracle_render.restype = C.c_int
_o.oracle_render.argtypes = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams), _fp, _u64p, C.c_int]
_o.oracle_render_window.restype = C.c_int
_o.oracle_render_window.argtypes = [_fp, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(RenderParams), C.c_int, C.c_int, C.c_int, C.c_int,
                                    _fp, _u64p, C.c_int]
_o.oracle_trace_rays.restype = C.c_int
_o.oracle_trace_rays.argtypes = [_fp, C.c_int, _fp, C.c_int, C.c_int, _fp, _fp, C.c_int, C.c_int, C.c_int, _ip, _fp, _ip, _ip, _fp, _fp, _u64p]
_o.oracle_eval_brdf.restype = C.c_int
_o.oracle_eval_brdf.argtypes = [C.c_int, C.c_int, _fp, _fp, _fp, _fp, _fp, _fp]
_o.oracle_eval_math.restype = C.c_int
_o.oracle_eval_math.argtypes = [C.c_int, C.c_int, _fp, _fp, _fp]
_o.oracle_wang_chain.restype = None
_o.oracle_wang_chain.argtypes = [C.c_uint32, C.c_int, C.POINTER(C.c_uint32), _fp]
_o.oracle_sobol.restype = C.c_float
_o.oracle_sobol.argtypes = [C.c_uint32, C.c_uint32]
_o.oracle_cp_rotation.restype = None
_o.oracle_cp_rotation.argtypes = [_fp, C.c_uint32, C.c_uint32]
_o.oracle_pi.restype = C.c_float
_o.oracle_set_ray_dump.restype = C.c_uint64
_o.oracle_set_ray_dump.argtypes = [_fp, C.c_uint64]

COUNTER_NAMES = ["rays_primary", "rays_bounce", "rays_shadow", "n_node", "n_tri", "hits", "hdr_lookups", "samples", "max_stack"]


def _f(a):
    return None if a is None else a.ctypes.data_as(_fp)


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if shape is None else a.reshape(shape)


def render(tris, nodes, cfg, hdr=None, hdr_cache=None, hdr_linear=True, framebuffer=None, threads=0, window=None):
    """ezrt_ref_render: `cfg.spp` display() calls on the CPU.  Returns (image [H,W,C], counters dict).
    window = (x0, y0, x1, y1): only that pixel rectangle of the cfg.width x cfg.height grid, image [y1-y0, x1-x0, C]."""
    tris = _f32(tris, (-1, 36)); nodes = _f32(nodes, (-1, 12))
    hw = hh = 0
    if hdr is not None:
        hdr = _f32(hdr); hdr_cache = None if hdr_cache is None else _f32(hdr_cache)
        hh, hw = hdr.shape[0], hdr.shape[1]
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    fb = np.zeros((y1 - y0, x1 - x0, cfg.out_channels), dtype=np.float32) if framebuffer is None else framebuffer
    cnt = np.zeros(9, dtype=np.uint64)
    p = cfg.to_struct()
    rc = _o.oracle_render_window(_f(tris), tris.shape[0], _f(nodes), nodes.shape[0], _f(hdr), _f(hdr_cache), hw, hh, int(bool(hdr_linear)),
                                 C.byref(p), int(x0), int(y0), int(x1), int(y1), _f(fb), cnt.ctypes.data_as(_u64p), int(threads))
    if rc != 0:
        raise RuntimeError("oracle_render failed (%d)" % rc)
    c = {k: int(v) for k, v in zip(COUNTER_NAMES, cnt)}
    c["rays"] = c["rays_primary"] + c["rays_bounce"] + c["rays_shadow"]
    return fb, c


def render_rays(tris, nodes, cfg, hdr=None, hdr_cache=None, hdr_linear=True, window=None):
    """render() that also returns the rays the render traced: (image, counters, rays [n, 7] float32), every ray's origin,
    direction and kind (0 camera, 1 bounce, 2 shadow; oracle_set_ray_dump).  The oracle renders on many threads, so the
    rows come in no fixed order: compare sums over rays only."""
    x0, y0, x1, y1 = (0, 0, cfg.width, cfg.height) if window is None else window
    cap = (x1 - x0) * (y1 - y0) * cfg.spp * (2 * cfg.max_bounce + 3)   # a camera ray, then a bounce and a shadow ray per bounce
    buf = np.zeros((cap, 7), np.float32)
    _o.oracle_set_ray_dump(_f(buf), cap)
    try:
        img, c = render(tris, nodes, cfg, hdr=hdr, hdr_cache=hdr_cache, hdr_linear=hdr_linear, window=window)
    finally:
        seen = int(_o.oracle_set_ray_dump(None, 0))
    if seen > cap or seen != c["rays"]:
        raise RuntimeError("oracle ray dump: %d rays seen, %d counted, room for %d" % (seen, c["rays"], cap))
    return img, c, buf[:seen]


def trace_rays(tris, nodes, origins, dirs, traverse=0, p3_fudge=False, brute=False):
    tris = _f32(tris, (-1, 36)); nodes = _f32(nodes, (-1, 12))
    o = _f32(origins, (-1, 3)); d = _f32(dirs, (-1, 3))
    n = o.shape[0]
    hit = np.zeros(n, np.int32); tri = np.zeros(n, np.int32); inside = np.zeros(n, np.int32)
    dist = np.zeros(n, np.float32); point = np.zeros((n, 3), np.float32); normal = np.zeros((n, 3), np.float32)
    cnt = np.zeros(5, np.uint64)
    ip = lambda a: a.ctypes.data_as(_ip)
    rc = _o.oracle_trace_rays(_f(tris), tris.shape[0], _f(nodes), nodes.shape[0], n, _f(o), _f(d), int(traverse), int(bool(p3_fudge)),
                              int(bool(brute)), ip(hit), _f(dist), ip(tri), ip(inside), _f(point), _f(normal), cnt.ctypes.data_as(_u64p))
    assert rc == 0
    return dict(hit=hit, distance=dist, triangle=tri, inside=inside, point=point, normal=normal,
                counters=dict(rays=int(cnt[0]), n_node=int(cnt[1]), n_tri=int(cnt[2]), hits=int(cnt[3]), max_stack=int(cnt[4])))


def eval_brdf(which, V, N, L, xi, materials):
    V = _f32(V, (-1, 3)); N = _f32(N, (-1, 3))
    L = None if L is None else _f32(L, (-1, 3)); xi = None if xi is None else _f32(xi, (-1, 3))
    materials = _f32(materials, (-1, 18))
    out = np.zeros_like(V)
    assert _o.oracle_eval_brdf(which, V.shape[0], _f(V), _f(N), _f(L), _f(xi), _f(materials), _f(out)) == 0
    return out


def eval_math(which, a, b=None):
    a = _f32(a).reshape(-1); b = None if b is None else _f32(b).reshape(-1)
    out = np.zeros_like(a)
    assert _o.oracle_eval_math(which, a.size, _f(a), _f(b), _f(out)) == 0
    return out


def wang_chain(seed, n):
    h = np.zeros(n, np.uint32); r = np.zeros(n, np.float32)
    _o.oracle_wang_chain(seed, n, h.ctypes.data_as(C.POINTER(C.c_uint32)), _f(r))
    return h, r


def sobol(d, i):
    return float(_o.oracle_sobol(d, i))


def cp_rotation(x, y, px, py):
    xy = np.array([x, y], np.float32)
    _o.oracle_cp_rotation(_f(xy), px, py)
    return float(xy[0]), float(xy[1])


_o.oracle_tonemap.restype = None
_o.oracle_tonemap.argtypes = [_fp, C.c_int, _fp, C.c_longlong, C.c_float]


def tonemap(fb, limit=1.5):
    fb = _f32(fb)
    ch = fb.shape[-1]
    out = np.zeros(fb.shape[:-1] + (3,), np.float32)
    _o.oracle_tonemap(_f(fb), ch, _f(out), fb.size // ch, float(limit))
    return out


def pi():
    return float(_o.oracle_pi())
