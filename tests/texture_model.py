"""A float64 numpy model of the base-colour texture lookup (EZRT_PARAM_TEXTURES; include/ezrt_math.h, DESIGN.md section 15), independent
of the C definition: the sRGB table, the dominant-plane barycentrics and the wrapped bilinear filter."""
import numpy as np


def srgb_eotf64(c):
    c = np.asarray(c, np.float64)
    return np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)


LUT = srgb_eotf64(np.arange(256) / 255.0).astype(np.float32)


def sample64(tex, u, v):
    """the filtered linear colour of the uint8 texture [H, W, 3|4] at (u, v), in float64 from the fp32 table; white for non-finite uv"""
    if not (np.isfinite(u) and np.isfinite(v)):
        return np.ones(3)
    H, W = tex.shape[:2]
    lin = LUT[tex[:, :, :3]].astype(np.float64)
    s, t = float(u) - np.floor(float(u)), float(v) - np.floor(float(v))
    x, y = s * W - 0.5, (1.0 - t) * H - 0.5
    x0, y0 = int(np.floor(x)), int(np.floor(y))
    fx, fy = x - x0, y - y0
    c = lambda yy, xx: lin[yy % H, xx % W]
    top = c(y0, x0) * (1 - fx) + c(y0, x0 + 1) * fx
    bot = c(y0 + 1, x0) * (1 - fx) + c(y0 + 1, x0 + 1) * fx
    return top * (1 - fy) + bot * fy


def bary64(P, p, tris=None):
    """barycentric weights [n, 3] of points P [n, 3] on triangles p [n, 3, 3], on the plane of the dominant normal axis, in float64"""
    p = np.asarray(p, np.float64)
    P = np.asarray(P, np.float64)
    ng = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    k = np.argmax(np.abs(ng), axis=1)
    a, b = (k + 1) % 3, (k + 2) % 3
    r = np.arange(len(p))
    e = lambda q, s, x: (s[r, a] - q[r, a]) * (x[r, b] - q[r, b]) - (s[r, b] - q[r, b]) * (x[r, a] - q[r, a])
    A = e(p[:, 0], p[:, 1], p[:, 2])
    with np.errstate(divide="ignore", invalid="ignore"):
        w1, w2 = e(p[:, 1], p[:, 2], P) / A, e(p[:, 2], p[:, 0], P) / A
    w = np.stack([w1, w2, 1 - w1 - w2], axis=1)
    w[~(np.isfinite(A) & (A != 0))] = 1.0 / 3.0
    return w


def constant_textures(rng, sizes):
    """textures of one colour each (RGBA8, random alpha), and those colours [k, 3]"""
    colours = rng.integers(0, 256, (len(sizes), 3))
    tex = []
    for (h, w), c in zip(sizes, colours):
        t = np.empty((h, w, 4), np.uint8)
        t[:, :, :3] = c
        t[:, :, 3] = rng.integers(0, 256, (h, w))
        tex.append(t)
    return tex, colours
