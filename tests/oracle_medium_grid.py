"""ctypes binding of the CPU restatement of the density grid's definition (tests/oracle_medium_grid.cpp ->
build/libezrt_oracle_medium_grid.so): brick maxima, lookup, free flight and transmittance with their majorant counters, beside the
header's own functions.  TEST INFRASTRUCTURE."""
import ctypes as C
import os

import numpy as np

from ezrt_b200 import build as _build

if not os.path.exists(_build.ORACLE_MEDIUM_GRID_SO):
    _build.build_oracle_medium_grid()
_o = C.CDLL(_build.ORACLE_MEDIUM_GRID_SO)

_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int32)
_up = C.POINTER(C.c_uint32)
_o.oracle_grid_bricks.restype = C.c_int
_o.oracle_grid_bricks.argtypes = [C.c_int, C.c_int, C.c_int, _fp, C.c_int, _fp, _ip]
_o.oracle_grid_eval.restype = None
_o.oracle_grid_eval.argtypes = [_fp, C.c_int, C.c_int, C.c_int, _fp, C.c_int, C.c_int, _fp, _fp, _fp, _up, _ip, _fp, _up, _ip, _fp, _up,
                                C.POINTER(C.c_ulonglong), C.c_float]
_o.oracle_grid_shadow_seed.restype = None
_o.oracle_grid_shadow_seed.argtypes = [C.c_int, _up, _up, _up, _up, _up]


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def _grid(rho):
    rho = np.ascontiguousarray(np.asarray(rho, np.float32))
    assert rho.ndim == 3
    return rho, rho.shape[2], rho.shape[1], rho.shape[0]


def bricks(rho):
    """The brick maxima float32 [bz, by, bx] of the grid rho [nz, ny, nx]."""
    rho, nx, ny, nz = _grid(rho)
    dims = np.zeros(3, np.int32)
    b = _o.oracle_grid_bricks(nx, ny, nz, _p(rho, _fp), 0, None, _p(dims, _ip))
    out = np.zeros(b, np.float32)
    _o.oracle_grid_bricks(nx, ny, nz, _p(rho, _fp), b, _p(out, _fp), None)
    return out.reshape(int(dims[2]), int(dims[1]), int(dims[0]))


def _med7(sigma_t, box_min, box_max):
    return np.array([sigma_t] + list(box_min) + list(box_max), np.float32)


def density(rho, sigma_t, box_min, box_max, points):
    """sigma at points [n, 3] (ezrt_scene_medium_eval's which 0)."""
    rho, nx, ny, nz = _grid(rho)
    m = _med7(sigma_t, box_min, box_max)
    P = np.ascontiguousarray(np.asarray(points, np.float32).reshape(-1, 3))
    out = np.zeros(P.shape[0], np.float32)
    _o.oracle_grid_eval(_p(m, _fp), nx, ny, nz, _p(rho, _fp), 0, P.shape[0], _p(P, _fp), None, None, None, None, _p(out, _fp), None, None, None,
                        None, None, 1.0)
    return out


def track(rho, sigma_t, box_min, box_max, which, o, d, L, seed, twin=True, brick_scale=1.0):
    """which 1 (free flight) or 2 (transmittance) of the rays (o, d, L) from seed: a dict of flag, out (t_s / T), seed (advanced), the
    header's own results flag2, out2, seed2 (twin), and the counters collisions, violations, outside, clamped.  brick_scale != 1 scales
    the restatement's brick maxima (a mutation, test-only; twin then stays the definition's)."""
    rho, nx, ny, nz = _grid(rho)
    m = _med7(sigma_t, box_min, box_max)
    o = np.ascontiguousarray(np.asarray(o, np.float32).reshape(-1, 3))
    n = o.shape[0]
    d = np.ascontiguousarray(np.asarray(d, np.float32).reshape(-1, 3))
    L = np.ascontiguousarray(np.broadcast_to(np.asarray(L, np.float32), (n,)))
    seed = np.ascontiguousarray(np.asarray(seed, np.uint32).reshape(-1))
    r = {k: np.zeros(n, t) for k, t in (("flag", np.int32), ("out", np.float32), ("seed", np.uint32))}
    if twin:
        r.update({k: np.zeros(n, t) for k, t in (("flag2", np.int32), ("out2", np.float32), ("seed2", np.uint32))})
    st = (C.c_ulonglong * 4)()
    _o.oracle_grid_eval(_p(m, _fp), nx, ny, nz, _p(rho, _fp), which, n, _p(o, _fp), _p(d, _fp), _p(L, _fp), _p(seed, _up), _p(r["flag"], _ip),
                        _p(r["out"], _fp), _p(r["seed"], _up), _p(r.get("flag2"), _ip), _p(r.get("out2"), _fp), _p(r.get("seed2"), _up), st, float(brick_scale))
    r.update(collisions=st[0], violations=st[1], outside=st[2], clamped=st[3])
    return r


def shadow_seed(px, py, frame, bounce):
    a = [np.ascontiguousarray(np.asarray(x, np.uint32).reshape(-1)) for x in (px, py, frame, bounce)]
    out = np.zeros(a[0].shape[0], np.uint32)
    _o.oracle_grid_shadow_seed(a[0].shape[0], *[_p(x, _up) for x in a], _p(out, _up))
    return out


def rho64(rho, box_min, box_max, P):
    """float64 trilinear of the grid at points P [n, 3] (lattice coordinate clamped to the lattice)."""
    rho = np.asarray(rho, np.float64)
    P = np.asarray(P, np.float64).reshape(-1, 3)
    lo, hi = np.asarray(box_min, np.float64), np.asarray(box_max, np.float64)
    n = np.array([rho.shape[2], rho.shape[1], rho.shape[0]])
    c0 = np.zeros((P.shape[0], 3), np.int64)
    f = np.zeros((P.shape[0], 3))
    for a in range(3):
        if n[a] == 1:
            continue
        u = np.clip((P[:, a] - lo[a]) / (hi[a] - lo[a]) * (n[a] - 1), 0, n[a] - 1)
        c = np.minimum(np.floor(u).astype(np.int64), n[a] - 2)
        c0[:, a], f[:, a] = c, u - c
    c1 = np.minimum(c0 + 1, n - 1)
    out = np.zeros(P.shape[0])
    for dk in (0, 1):
        for dj in (0, 1):
            for di in (0, 1):
                w = (f[:, 0] if di else 1 - f[:, 0]) * (f[:, 1] if dj else 1 - f[:, 1]) * (f[:, 2] if dk else 1 - f[:, 2])
                idx = ((c1 if dk else c0)[:, 2], (c1 if dj else c0)[:, 1], (c1 if di else c0)[:, 0])
                out += w * rho[idx]
    return out


# ---------------------------------------------------------------- renders: the included restatements with the grid's flight and transmittance
_o.oracle_grid_render_set.restype = None
_o.oracle_grid_render_set.argtypes = [C.c_int, C.c_int, C.c_int, _fp, C.c_float]


def _as_grid_library(mod, names, rho, brick_scale, fn, *args, **kw):
    """mod.fn(*args, **kw) with this library's copies of mod's render functions (same signatures), the grid rho set (None: the
    homogeneous medium)"""
    for name in names:
        mine, theirs = getattr(_o, name), getattr(mod._o, name)
        mine.restype, mine.argtypes = theirs.restype, theirs.argtypes
    if rho is None:
        _o.oracle_grid_render_set(0, 0, 0, None, 1.0)
    else:
        g, nx, ny, nz = _grid(rho)
        _o.oracle_grid_render_set(nx, ny, nz, _p(g, _fp), float(brick_scale))
    saved, mod._o = mod._o, _o
    try:
        return fn(*args, **kw)
    finally:
        mod._o = saved
        _o.oracle_grid_render_set(0, 0, 0, None, 1.0)


def render(tris, nodes, cfg, rho, brick_scale=1.0, **kw):
    """tests/oracle_light_tree.render (every option of the light sampling mode, plain / window / feature-buffer) with cfg.medium_grid
    rendered through the grid rho [nz, ny, nx] of the medium kw["m"]"""
    from tests import oracle_light_tree
    return _as_grid_library(oracle_light_tree, ["oracle_render_light_tree"], rho if cfg.medium_grid else None, brick_scale,
                            oracle_light_tree.render, tris, nodes, cfg, **kw)


def render_adaptive(tris, nodes, cfg, rho, threshold, min_spp, check_interval, **kw):
    """tests/oracle_light_tree.render_adaptive with cfg.medium_grid rendered through the grid rho"""
    from tests import oracle_light_tree
    return _as_grid_library(oracle_light_tree, ["oracle_render_light_tree_adaptive"], rho if cfg.medium_grid else None, 1.0,
                            oracle_light_tree.render_adaptive, tris, nodes, cfg, threshold, min_spp, check_interval, **kw)


def render_medium(tris, nodes, cfg, m, rho, brick_scale=1.0, phase_only=False, **kw):
    """tests/oracle_medium.render (with its phase-only estimator) through the grid rho (None: the homogeneous medium)"""
    from tests import oracle_medium
    return _as_grid_library(oracle_medium, ["oracle_render_medium"], rho, brick_scale, oracle_medium.render, tris, nodes, cfg, m,
                            phase_only=phase_only, **kw)
