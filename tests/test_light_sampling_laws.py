"""The light sampling mode's sampling laws and estimators against exact references (DESIGN.md sections 10 and 11), on the CPU:

(a) the exact law of the light selection and of the map's texel selection -- every one of the 2^32 hash values h of rand01 =
    fl32(h) * 2^-32 counted, in integer and float64 numpy -- against the probabilities the estimators divide by;
(b) SampleBRDF's density against BRDF_Pdf, the density mode 4's MIS weights assume, over a grid of materials and view angles;
(c) the estimators against independent ones on scenes the P3 bunny does not reach: two-sided emission, many material lobes,
    weights spread over eight orders of magnitude, a map with one bright texel, 1 and 4 bounces, many lights."""
import numpy as np
import pytest
from scipy import stats

from ezrt_b200 import api, scenes
from tests import oracle_env_light as oe
from tests import oracle_lights as ol

TWO32 = 1 << 32


# ------------------------------------------------------------------ (a) the exact selection laws
def _fl32(h):
    """fl32(h) for integers h in [0, 2^32): round to nearest even, as __uint2float_rn and the oracle's conversion"""
    return np.asarray(h, np.int64).astype(np.uint32).astype(np.float32).astype(np.float64)


def _count_below(C):
    """#{h in [0, 2^32) : fl32(h) < C} for every C (float64; fl32 is monotone, so a vectorised bisection on h)"""
    C = np.asarray(C, np.float64)
    lo, hi = np.zeros(C.shape, np.int64), np.full(C.shape, TWO32, np.int64)
    while (lo < hi).any():
        mid = (lo + hi) >> 1
        ge = _fl32(np.minimum(mid, TWO32 - 1)) >= C
        hi = np.where(ge, mid, hi)
        lo = np.where(ge, lo, mid + 1)
    return lo


def _selection_law(cdf, lo=0.0, scale=1.0):
    """Exact probabilities of ez_light_select(cdf, n, r) over the h whose r = lo + (rand01(h) - lo) / scale... restated as: entry
    k is selected iff lo + scale * cdf_{k-1} <= rand01(h) < lo + scale * cdf_k among the h with rand01(h) >= lo, and rand01 = 1.0
    (fl32(h) = 2^32) selects the last entry.  Returns (probabilities, number of h in the branch)."""
    cdf = np.asarray(cdf, np.float64)
    base = int(_count_below(lo * TWO32))
    n_below = _count_below((lo + scale * cdf[:-1]) * TWO32)
    edges = np.concatenate([[base], n_below, [TWO32]])
    return np.diff(edges) / float(TWO32 - base), TWO32 - base


def _metrics(P, q):
    P, q = np.asarray(P, np.float64).ravel(), np.asarray(q, np.float64).ravel()
    big = q >= 2.0 ** -20
    zero = (P == 0) & (q > 0)
    return dict(tv=0.5 * np.abs(P - q).sum(), max_ratio=float(np.abs(P[big] / q[big] - 1).max()) if big.any() else 0.0,
                zero_n=int(zero.sum()), zero_mass=float(q[zero].sum()))


def _lum_f32(e):
    e = np.asarray(e, np.float32)
    return (np.float32(0.3) * e[:, 0] + np.float32(0.6) * e[:, 1]) + np.float32(0.1) * e[:, 2]


def _assumed_light_probs(tris, tri, total):
    """q_k = lum_f(E_k) * area64_k / W_f: what pdf_l = lum / W_f * dist^2 / cos_l divides by, with the sampler uniform in area"""
    t = np.asarray(tris, np.float32).reshape(-1, 36)[tri]
    p = t[:, 0:9].astype(np.float64).reshape(-1, 3, 3)
    area = 0.5 * np.linalg.norm(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]), axis=1)
    return _lum_f32(t[:, 18:21]).astype(np.float64) * area / float(np.float32(total))


def _texel_law(row, col):
    """P_ij = P_row(i) * P_col(j | i), each counted exactly"""
    H, W = col.shape
    prow, _ = _selection_law(row)
    pcol = np.zeros((H, W))
    live = np.flatnonzero(col[:, -1] == 1.0)
    # every live row's conditional law in one bisection: rows are independent draws r_2
    n_below = _count_below(col[live, :-1].astype(np.float64) * TWO32)
    edges = np.concatenate([np.zeros((len(live), 1), np.int64), n_below, np.full((len(live), 1), TWO32, np.int64)], axis=1)
    pcol[live] = np.diff(edges, axis=1) / float(TWO32)
    return prow[:, None] * pcol


def _many_light_scene():
    """s_grid(5, 4) with every triangle emissive: 103,692 lights whose weights follow the triangles' areas (tris, nodes, eye, cam)"""
    tris, nodes, eye, cam = scenes.s_grid(5, 4, 4)
    tris = np.asarray(tris, np.float32).reshape(-1, 36).copy()
    tris[:, 18:21] = np.random.default_rng(9).uniform(0.01, 3.0, (len(tris), 3)).astype(np.float32)
    return tris, nodes, eye, cam


def _many_light_tris():
    return _many_light_scene()[0]


def _spread_tris():
    """the P3 bunny with its first light (in triangle order) 10^8 times brighter than the other 319, which are dimmed"""
    tris = np.asarray(scenes.s_p3_bunny()[0], np.float32).reshape(-1, 36).copy()
    tri = ol.oracle_light_table(tris)[0]
    tris[tri[1:], 18:21] *= np.float32(1e-8)
    return tris


def _bright_texel_map(W, H):
    hdr = np.full((H, W, 3), 0.05, np.float32)
    hdr[H // 3, W // 5] = (4e5, 3e5, 2e5)
    return hdr


def test_rand01_counting():
    """fl32 rounds to nearest even; 128 hash values give rand01 = 1.0; the map branch r_sel < 0.5 holds 2^31 - 64 of 2^32"""
    assert _fl32(TWO32 - 128) == 2.0 ** 32 and _fl32(TWO32 - 129) == 2.0 ** 32 - 256
    assert _fl32((1 << 31) - 64) == 2.0 ** 31 and _fl32((1 << 31) - 65) == 2.0 ** 31 - 128
    assert _count_below(2.0 ** 32) == TWO32 - 128
    # P_env = 1/2 is really (2^31 - 64) / 2^32 = 0.5 - 2^-26: the map branch is 1.5e-8 short of a half, the triangles' branch over
    assert _count_below(2.0 ** 31) == (1 << 31) - 64
    assert _selection_law(np.array([0.5, 1.0], np.float32))[0][0] == ((1 << 31) - 64) / 2.0 ** 32
    # exact brute-force counts over all h < 2^20, where every conversion is exact and so every C counts itself
    h = np.arange(0, 1 << 20, dtype=np.int64)
    for C in (0.0, 1.0, 3.0e5 + 0.5, 2.0 ** 20 - 1.0):
        assert _count_below(C) == (_fl32(h) < C).sum(), C
    # around the rounding steps above 2^24, where one float stands for 2^k hashes, counted hash by hash
    for top in (1 << 25, 1 << 31, TWO32):
        h = np.arange(top - 4096, top, dtype=np.int64)
        for C in np.unique(_fl32(h))[1:]:     # the lowest value's rounding group may start below the window
            assert _count_below(C) == top - 4096 + (_fl32(h) < C).sum(), (top, C)


def _light_law_rows():
    rows = []
    p3 = scenes.s_p3_bunny()[0]
    s1m = scenes.s_1m_bunny()[0]
    for name, tris, bench in (("P3 (C1, C2)", p3, True), ("S-1M (C3, C4, C5)", s1m, True), ("many lights", _many_light_tris(), False),
                              ("spread weights", _spread_tris(), False)):
        tri, cdf, total = ol.oracle_light_table(tris)
        assert cdf[-1] == 1.0, name    # else the rand01 in [cdf_{K-1}, 1] would select the last light by the search's fall-through
        q = _assumed_light_probs(tris, tri, total)
        P, _ = _selection_law(cdf)
        rows.append((name, len(tri), "r_sel", _metrics(P, q), bench))
        P2, n2 = _selection_law(cdf, lo=0.5, scale=0.5)     # with the map as a light: r_tri = (r_sel - 0.5) * 2
        assert n2 == (1 << 31) + 64
        rows.append((name, len(tri), "r_tri", _metrics(P2, q), bench))
    return rows


def test_light_selection_law():
    rows = _light_law_rows()
    for name, k, which, m, _ in rows:
        print("light law %-18s K=%7d %s: TV %.3g, max |P/q - 1| %.3g, P = 0 < q: %d lights, q-mass %.3g" %
              (name, k, which, m["tv"], m["max_ratio"], m["zero_n"], m["zero_mass"]))
    for name, k, which, m, bench in rows:
        if bench:
            assert m["tv"] <= 1e-4 and m["zero_n"] == 0, (name, which, m)
    # the adversarial tables: the spread set has lights that are never selected (equal cdf entries behind the dominant one)
    spread = [m for name, _, _, m, _ in rows if name == "spread weights"]
    assert all(m["zero_n"] > 0 and m["zero_mass"] < 1e-5 for m in spread), spread


@pytest.mark.parametrize("which", ["synth 128x64", "synth 2048x1024 (C4)", "one bright texel 2048x1024"])
def test_texel_selection_law(which):
    hdr = {"synth 128x64": lambda: scenes.synth_hdr(128, 64), "synth 2048x1024 (C4)": lambda: scenes.synth_hdr(2048, 1024),
           "one bright texel 2048x1024": lambda: _bright_texel_map(2048, 1024)}[which]()
    row, col, pdf, _ = oe.env_table(hdr)
    assert row[-1] == 1.0 and (col[:, -1] == 1.0).all()
    P = _texel_law(row, col)
    m = _metrics(P, pdf)
    H = hdr.shape[0]
    polar = _metrics(P[[0, H - 1]], pdf[[0, H - 1]])
    print("texel law %-26s TV %.3g, max |P/q - 1| %.3g, P = 0 < q: %d texels, q-mass %.3g; polar rows: TV %.3g" %
          (which, m["tv"], m["max_ratio"], m["zero_n"], m["zero_mass"], polar["tv"]))
    assert abs(P.sum() - 1.0) < 1e-12
    if which.startswith("synth"):
        assert m["tv"] <= 1e-4 and m["zero_n"] == 0, m


# ------------------------------------------------------------------ (b) SampleBRDF's density against BRDF_Pdf
N_DIRS = 1_000_000
NC, NPHI = 20, 36


def _frame():
    n = np.array([0.3, 0.8, 0.52])
    n /= np.linalg.norm(n)
    t = np.cross(n, [0.0, 0.0, 1.0])
    t /= np.linalg.norm(t)
    return n, t, np.cross(n, t)


def _dirs(c, phi):
    n, t, b = _frame()
    s = np.sqrt(np.maximum(0.0, 1.0 - c * c))
    return c[:, None] * n + (s * np.cos(phi))[:, None] * t + (s * np.sin(phi))[:, None] * b


_GL = np.polynomial.legendre.leggauss(5)


def _gl_cells(pdf, c0, c1, p0, p1):
    """m x m Gauss-Legendre integral of pdf(c, phi) dc dphi over every cell"""
    x, w = _GL
    m = len(x)
    cc = (c0[:, None] + (c1 - c0)[:, None] * (x + 1) / 2)[:, :, None]
    pp = (p0[:, None] + (p1 - p0)[:, None] * (x + 1) / 2)[:, None, :]
    cc, pp = np.broadcast_arrays(cc, pp)
    f = pdf(cc.ravel(), pp.ravel()).reshape(-1, m, m)
    return (f * w[None, :, None] * w[None, None, :]).sum((1, 2)) * (c1 - c0) * (p1 - p0) / 4


def _bin_integrals(pdf, tol=2e-8, max_depth=30):
    """the integral of pdf over every (cos theta, phi) bin, adaptively: a cell is halved along the dimension whose halving changes
    the estimate most, until halving changes it by at most tol (probability)"""
    ce, pe = np.linspace(0, 1, NC + 1), np.linspace(0, 2 * np.pi, NPHI + 1)
    ic, ip = np.meshgrid(np.arange(NC), np.arange(NPHI), indexing="ij")
    b = (ic * NPHI + ip).ravel()
    c0, c1, p0, p1 = ce[ic].ravel(), ce[ic + 1].ravel(), pe[ip].ravel(), pe[ip + 1].ravel()
    est = _gl_cells(pdf, c0, c1, p0, p1)
    out = np.zeros(NC * NPHI)
    for depth in range(max_depth + 1):
        cm, pm = (c0 + c1) / 2, (p0 + p1) / 2
        ha = _gl_cells(pdf, np.concatenate([c0, cm, c0, c0]), np.concatenate([cm, c1, c1, c1]),
                       np.concatenate([p0, p0, p0, pm]), np.concatenate([p1, p1, pm, p1]))
        n = len(c0)
        lc, uc, lp, up = ha[:n], ha[n:2 * n], ha[2 * n:3 * n], ha[3 * n:]
        ec, ep = np.abs(lc + uc - est), np.abs(lp + up - est)
        done = (np.maximum(ec, ep) <= tol) | (depth == max_depth)
        np.add.at(out, b[done], np.where(ec >= ep, lc + uc, lp + up)[done])
        split_c = (ec >= ep) & ~done
        split_p = (ec < ep) & ~done
        if not (split_c.any() or split_p.any()):
            break
        sc, sp = split_c, split_p
        c0, c1, p0, p1, b, est = (np.concatenate(a) for a in (
            [c0[sc], cm[sc], c0[sp], c0[sp]], [cm[sc], c1[sc], c1[sp], c1[sp]], [p0[sc], p0[sc], p0[sp], pm[sp]],
            [p1[sc], p1[sc], pm[sp], p1[sp]], [b[sc], b[sc], b[sp], b[sp]], [lc[sc], uc[sc], lp[sp], up[sp]]))
    return out


def _material(roughness, metallic, clearcoat, gloss, aniso=0.0, black=False):
    return api.Material(baseColor=(0, 0, 0) if black else (0.8, 0.6, 0.4), roughness=roughness, metallic=metallic, clearcoat=clearcoat,
                        clearcoatGloss=gloss, anisotropic=aniso).as_array()


def _brdf_case(oracle, mat, cos_v, seed):
    n, t, _ = _frame()
    sin_v = np.sqrt(1 - cos_v * cos_v)
    V = (cos_v * n + sin_v * t).astype(np.float32)
    N = n.astype(np.float32)
    xi = np.random.default_rng(seed).random((N_DIRS, 3), dtype=np.float32)
    L = oracle.eval_brdf(3, np.broadcast_to(V, (N_DIRS, 3)), np.broadcast_to(N, (N_DIRS, 3)), None, xi,
                         np.broadcast_to(mat, (N_DIRS, 18))).astype(np.float64)
    c = L @ n.astype(np.float32).astype(np.float64)
    below = c <= 0          # NdotL <= 0: the integrator stops there
    phi = np.mod(np.arctan2(L @ np.cross(n, t), L @ t), 2 * np.pi)
    ib = np.minimum((c[~below] * NC).astype(int), NC - 1) * NPHI + np.minimum((phi[~below] / (2 * np.pi) * NPHI).astype(int), NPHI - 1)
    obs = np.append(np.bincount(ib, minlength=NC * NPHI), below.sum()).astype(np.float64)

    def pdf(cc, pp):
        d = _dirs(cc, pp).astype(np.float32)
        k = len(d)
        return oracle.eval_brdf(2, np.broadcast_to(V, (k, 3)), np.broadcast_to(N, (k, 3)), d, None,
                                np.broadcast_to(mat, (k, 18)))[:, 0].astype(np.float64)

    p = _bin_integrals(pdf)
    exp = N_DIRS * np.append(p, max(0.0, 1.0 - p.sum()))
    # chi-square over the bins expecting >= 5, the rest pooled into one
    small = exp < 5
    e = np.append(exp[~small], exp[small].sum())
    o = np.append(obs[~small], obs[small].sum())
    keep = e > 0
    chi2 = float((((o - e) ** 2)[keep] / e[keep]).sum() + (o[~keep].sum() if (~keep).any() else 0.0) * 1e12)
    dof = int(keep.sum()) - 1
    z = np.abs(obs - exp) / np.sqrt(np.maximum(exp, 1.0))
    return chi2, dof, float(stats.chi2.sf(chi2, dof)), float(z.max()), float(obs[-1] / N_DIRS), float(1.0 - p.sum())


BRDF_MATERIALS = [(m, cc, g) for m in (0.0, 1.0) for cc, g in ((0.0, 1.0), (1.0, 0.0), (1.0, 1.0))]


@pytest.mark.parametrize("roughness", [0.3, 0.8])
def test_sample_brdf_density_is_brdf_pdf(oracle, roughness):
    """Roughness 0.05 (GGX alpha 0.0025) is out of this check's reach: the bin quadrature misses up to 0.5 % of so narrow a lobe's
    mass, with BRDF_Pdf and with a float64 restatement of it alike, so its chi-square measures the quadrature.  The narrowest lobe
    checked is the clearcoat's at gloss 1 (GTR1 alpha 0.001): its peak bin is the largest z (up to 8.5 at normal view), and the
    chi-square over all bins passes."""
    mats = [("metallic %g clearcoat %g gloss %g" % k, _material(roughness, *k)) for k in BRDF_MATERIALS]
    mats.append(("anisotropic 0.8, black base", _material(roughness, 0.0, 1.0, 1.0, aniso=0.8, black=True)))
    worst = 1.0
    for i, (name, mat) in enumerate(mats):
        for j, cos_v in enumerate((1.0, 0.5, 0.05)):
            chi2, dof, pval, zmax, below, below_exp = _brdf_case(oracle, mat, cos_v, seed=1000 * i + 10 * j + int(roughness * 100))
            print("BRDF roughness %.2f %-36s cos_v %.2f: chi2 %.1f / %d dof (p %.3g), max z %.2f, below the horizon %.4f (expected %.4f)" %
                  (roughness, name, cos_v, chi2, dof, pval, zmax, below, below_exp))
            assert pval > 1e-4, (roughness, name, cos_v, chi2, dof, zmax)
            worst = min(worst, pval)
    print("BRDF roughness %.2f: smallest p %.3g" % (roughness, worst))


# ------------------------------------------------------------------ (c) the estimators against independent ones
def _block_z(a, b, n, W, H, bh, bw):
    """|difference of the bh x bw block means| / combined standard error per block; a, b = (luminance, per-pixel variance).
    Pixels are independent (each has its own seed), so the variance of a block mean is the sum of its pixels' variances / n / m^2."""
    m = bh * bw
    blk = lambda x: x.reshape(H // bh, bh, W // bw, bw).swapaxes(1, 2).reshape(H // bh, W // bw, m)
    se = np.sqrt(blk(a[1]).sum(-1) / n / m ** 2 + blk(b[1]).sum(-1) / n / m ** 2)
    return np.abs(blk(a[0]).mean(-1) - blk(b[0]).mean(-1)) / np.maximum(se, 1e-12)


def _stats(img, luma2):
    y = (0.3 * img[..., 0] + 0.6 * img[..., 1] + 0.1 * img[..., 2]).astype(np.float64)
    return y, np.maximum(luma2.astype(np.float64) - y ** 2, 0.0)


def _two_sided_scene():
    """an open, one-sided quad light at y = 1.5 (triangles facing down) between a floor at y = 0 and a ceiling at y = 3: the
    ceiling sees its back"""
    tl = api.TriangleList()
    quad = "v -1 0 -1\nv 1 0 -1\nv 1 0 1\nv -1 0 1\nf 1 3 2\nf 1 4 3\n"
    down = quad.replace("f 1 3 2\nf 1 4 3", "f 1 2 3\nf 1 3 4")
    tl.read_obj_text(quad, api.Material(baseColor=(0.7, 0.7, 0.7), roughness=0.6), api.transform_matrix((0, 0, 0), (0, 0, 0), (3, 1, 3)), False)
    tl.read_obj_text(down, api.Material(baseColor=(0.6, 0.7, 0.8), roughness=0.3, metallic=0.5),
                     api.transform_matrix((0, 0, 0), (0, 3, 0), (3, 1, 3)), False)
    tl.read_obj_text(down, api.Material(emissive=(8, 8, 8)), api.transform_matrix((0, 0, 0), (0, 1.5, 0), (0.6, 1, 0.6)), False)
    tris, nodes = tl.build_bvh(8)
    eye, cam = api.camera_orbit(0.0, 0.0, 5.0)
    eye = (eye[0], eye[1] + 1.5, eye[2])
    return np.asarray(tris, np.float32).reshape(-1, 36), nodes, eye, cam


def _rough(scene):
    """the scene with every roughness raised to at least 0.5: mode 2's uniform hemisphere samples are a heavy-tailed estimator of a
    glossy lobe that reflects a bright emitter, and its per-pixel variance estimate then misses the tail"""
    tris = np.array(scene[0], np.float32).reshape(-1, 36)
    tris[:, 28] = np.maximum(tris[:, 28], 0.5)   # Material.roughness (api.Material.as_array, after the 18 geometry floats)
    return (tris,) + tuple(scene[1:])


def _estimator_cases(grid_scene):
    p3 = scenes.s_p3_bunny()
    spread = (_spread_tris(),) + tuple(p3[1:])
    g = grid_scene
    bright = scenes.synth_hdr(128, 64) * np.float32(0.02)
    bright[20, 30] = (4e3, 3e3, 2e3)
    L4, M2 = api.MODE_DISNEY_LIGHTS, api.MODE_DISNEY_SOBOL_P5
    env = (0.1, 0.1, 0.12)
    return [
        ("two-sided open quad light", _two_sided_scene(), None, True, 2, (M2, L4), 1024),
        ("grid scene materials, 1 bounce", g, None, True, 1, (M2, L4), 16384),
        ("grid scene, 4 bounces, rough", _rough(g), None, True, 4, (M2, L4), 512),
        ("spread weights (10^8), one lit triangle", spread, None, True, 1, (M2, L4), 4096),
        ("the 103,692-light table of (a), rough", _rough(_many_light_scene()), None, True, 2, (M2, L4), 512),
        ("bright texel beside the sphere, linear", p3, bright, True, 2, (L4, "flag"), 1024),
        ("bright texel beside the sphere, nearest", p3, bright, False, 2, (L4, "flag"), 1024),
    ], env


def test_estimators_agree_on_hard_scenes(grid_scene):
    cases, env = _estimator_cases(grid_scene)
    W, H = 64, 48
    worst = []
    for name, (tris, nodes, eye, cam), hdr, linear, bounces, (a, b), spp in cases:
        cache = None if hdr is None else api.hdr_cache(hdr)
        out = []
        for mode in (a, b):
            flag = mode == "flag"
            cfg = api.RenderConfig(width=W, height=H, spp=spp, max_bounce=bounces, mode=api.MODE_DISNEY_LIGHTS if flag else mode,
                                   eye=tuple(eye), camera_rotate=tuple(cam), env_color=env, env_light=flag)
            img, luma2, c = oe.oracle_render_env_light(tris, nodes, cfg, hdr=hdr, hdr_cache=cache, hdr_linear=linear)
            out.append(_stats(img, luma2))
        z8, z16 = _block_z(out[0], out[1], spp, W, H, 8, 8), _block_z(out[0], out[1], spp, W, H, 16, 16)
        zf = float(_block_z(out[0], out[1], spp, W, H, H, W).max())
        rel = (out[1][0].mean() - out[0][0].mean()) / out[0][0].mean()
        ratio = out[0][1].mean() / max(out[1][1].mean(), 1e-30)
        print("estimators %-42s %d bounces, %d spp: frame z %.2f (relative difference %+.2e), largest 16x16 z %.2f, largest 8x8 z %.2f "
              "(mean %.2f), variance ratio %.1f" % (name, bounces, spp, zf, rel, z16.max(), z8.max(), z8.mean(), ratio))
        worst.append((name, zf, float(z16.max()), float(z8.max())))
        # the whole frame is where a bias of the light or map pdf shows: its standard error is about 1/7 of an 8x8 block's
        assert np.isfinite(z8).all() and zf <= 4 and z16.max() <= 5 and z8.max() <= 5, (name, zf, z16.max(), z8.max())
    print("frame / 16x16 / 8x8 z per case: " + ", ".join("%s %.2f / %.2f / %.2f" % w for w in worst))
