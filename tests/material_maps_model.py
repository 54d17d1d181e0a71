"""A float64 numpy model of the material maps (EZRT_PARAM_MATERIAL_MAPS; include/ezrt_math.h, DESIGN.md section 16), independent of the C
definition: the linear table, the per-triangle tangent frame and the mapped shading normal with its fallbacks."""
import numpy as np

UNORM = (np.arange(256, dtype=np.float64) / 255.0).astype(np.float32)


def unorm_sample64(tex, u, v):
    """the filtered linear (c / 255) colour of the uint8 texture [H, W, 3|4] at (u, v) in float64; white for a non-finite uv"""
    if not (np.isfinite(u) and np.isfinite(v)):
        return np.ones(3)
    H, W = tex.shape[:2]
    lin = UNORM[tex[:, :, :3]].astype(np.float64)
    s, t = float(u) - np.floor(float(u)), float(v) - np.floor(float(v))
    x, y = s * W - 0.5, (1.0 - t) * H - 0.5
    x0, y0 = int(np.floor(x)), int(np.floor(y))
    fx, fy = x - x0, y - y0
    c = lambda yy, xx: lin[yy % H, xx % W]
    top = c(y0, x0) * (1 - fx) + c(y0, x0 + 1) * fx
    bot = c(y0 + 1, x0) * (1 - fx) + c(y0 + 1, x0 + 1) * fx
    return top * (1 - fy) + bot * fy


def tangent_frame64(p, uv6, No):
    """(T' [3], B [3]) of triangle p [3, 3] with UVs uv6 [6] about No [3], or None where the definition falls back"""
    p, uv6, No = (np.asarray(x, np.float64) for x in (p, uv6, No))
    e1, e2 = p[1] - p[0], p[2] - p[0]
    du1, dv1, du2, dv2 = uv6[2] - uv6[0], uv6[3] - uv6[1], uv6[4] - uv6[0], uv6[5] - uv6[1]
    det = du1 * dv2 - du2 * dv1
    if det == 0 or not np.isfinite(det):
        return None
    T = (dv2 * e1 - dv1 * e2) / det
    Buv = (du1 * e2 - du2 * e1) / det
    Tp = T - np.dot(No, T) * No
    l2 = np.dot(Tp, Tp)
    if l2 == 0 or not np.isfinite(l2):
        return None
    Tn = Tp / np.sqrt(l2)
    B = np.cross(No, Tn)
    s = np.dot(B, Buv)
    if s == 0 or not np.isfinite(s):
        return None
    return Tn, (-B if s < 0 else B)


def normal_map64(p, uv6, uv, f, N, inside, V):
    """the mapped shading normal in float64, or None where the definition returns surface_hit's N"""
    if not np.all(np.isfinite(uv)):
        return None
    N = np.asarray(N, np.float64)
    No = -N if inside else N
    fr = tangent_frame64(p, uv6, No)
    if fr is None:
        return None
    T, B = fr
    nt = 2.0 * np.asarray(f, np.float64) - 1.0
    n = nt[0] * T + nt[1] * B + nt[2] * No
    n = n / np.linalg.norm(n)
    if not np.all(np.isfinite(n)):
        return None
    if inside:
        n = -n
    if not np.dot(n, np.asarray(V, np.float64)) > 0:
        return None
    return n

