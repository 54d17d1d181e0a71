"""The light tree (EZRT_PARAM_LIGHT_TREE, DESIGN.md section 19) on the CPU: the host builder's invariants, the selection law of the
descent (nominal and exact over every rand01 hash), the descent against the hit-side walk, and the flagged render's estimator against
mode 4's (tests/oracle_light_tree.cpp), including a tree with wrong cones and a mutated MIS pdf that must be caught."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from ezrt_b200._lib import EzrtError
from tests import oracle_light_tree as ot
from tests.test_emission_maps_oracle import _mean_of
from tests.test_light_sampling_laws import TWO32, _block_z, _fl32, _many_light_scene, _rough, _stats

pytest.importorskip("scipy")


# ------------------------------------------------------------------ the builder
def _quad_tris(n, coplanar=False, seed=0):
    """n small triangles: coplanar ones on y = 0, else randomly oriented in a unit box (verts [n, 9])"""
    rng = np.random.default_rng(seed)
    c = rng.uniform(-1, 1, (n, 1, 3))
    d = rng.uniform(-0.05, 0.05, (n, 3, 3))
    if coplanar:
        c[..., 1] = 0.0
        d[..., 1] = 0.0
    return (c + d).reshape(n, 9).astype(np.float32)


def _light_sets():
    p3 = np.asarray(scenes.s_p3_bunny()[0], np.float32).reshape(-1, 36)
    grid = np.asarray(scenes.s_grid(3, 2, 4)[0], np.float32).reshape(-1, 36)   # S-1M's four spheres: 1,280 lights
    lamps = np.asarray(scenes.s_lamps(3, 3)[0], np.float32).reshape(-1, 36)
    one = _quad_tris(1)
    dup = np.repeat(_quad_tris(1, seed=3), 1000, axis=0)
    rng = np.random.default_rng(7)
    return {
        "p3_bunny": ot.table_inputs(p3), "s1m_lights": ot.table_inputs(grid), "s_lamps": ot.table_inputs(lamps),
        "103692_lights": ot.table_inputs(_many_light_scene()[0]),
        "one": (one, np.ones(1, np.float32)), "two": (_quad_tris(2, seed=1), np.array([1.0, 3.0], np.float32)),
        "1000_duplicates": (dup, np.ones(1000, np.float32)), "coplanar": (_quad_tris(500, True, 2), np.ones(500, np.float32)),
        "weights_1e8": (_quad_tris(700, seed=4), (10.0 ** rng.uniform(-4, 4, 700)).astype(np.float32)),
    }


@pytest.fixture(scope="module")
def light_sets():
    return _light_sets()


def _normals64(v):
    v = np.asarray(v, np.float64).reshape(-1, 3, 3)
    n = np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])
    return n / np.linalg.norm(n, axis=1, keepdims=True)


def _leaves_under(t):
    """per node the list of its lights, its depth and its path from the root (bit j: step j goes right)"""
    child = t["child"]
    M = len(child)
    under, depth, bits = [None] * M, np.zeros(M, np.int64), [0] * M
    order = [0]
    for i in order:   # breadth first: children after parents
        if child[i] >= 0:
            depth[child[i]] = depth[child[i] + 1] = depth[i] + 1
            bits[child[i]], bits[child[i] + 1] = bits[i], bits[i] | (1 << int(depth[i]))
            order += [child[i], child[i] + 1]
    for i in reversed(order):
        under[i] = [~child[i]] if child[i] < 0 else under[child[i]] + under[child[i] + 1]
    return under, depth, bits


@pytest.mark.parametrize("name", ["p3_bunny", "s1m_lights", "s_lamps", "103692_lights", "one", "two", "1000_duplicates", "coplanar", "weights_1e8"])
def test_tree_invariants(light_sets, name):
    verts, w = light_sets[name]
    K = len(w)
    t = api.build_light_tree(verts, w)
    assert len(t["phi"]) == 2 * K - 1 and len(t["path"]) == K
    under, depth, bits = _leaves_under(t)
    leaves = sorted(~c for c in t["child"] if c < 0)
    assert leaves == list(range(K)), "every light in exactly one leaf"
    v = np.asarray(verts, np.float64).reshape(-1, 3, 3)
    N = _normals64(verts)
    w64 = np.asarray(w, np.float64)
    for i, ks in enumerate(under):
        ks = np.array(ks)
        pts = v[ks].reshape(-1, 3)
        assert (t["lo"][i] <= pts.min(0)).all() and (t["hi"][i] >= pts.max(0)).all()
        c = t["child"][i]
        if c >= 0:
            assert (t["lo"][i] <= np.minimum(t["lo"][c], t["lo"][c + 1])).all() and (t["hi"][i] >= np.maximum(t["hi"][c], t["hi"][c + 1])).all()
        assert (np.abs(N[ks] @ t["axis"][i].astype(np.float64)) >= float(t["cos_o"][i])).all(), "cone of node %d" % i
        assert t["phi"][i] == np.float32(np.sum(w64[ks])), "phi of node %d" % i
    leaf = np.empty(K, np.int64)
    leaf[~t["child"][t["child"] < 0]] = np.nonzero(t["child"] < 0)[0]
    assert depth.max() <= 64 and (t["depth"] == depth[leaf]).all()
    assert (t["path"] == np.array([bits[i] for i in leaf], np.uint64)).all(), "each light's path leads to its leaf"
    again = api.build_light_tree(verts, w)
    assert again["nodes"].tobytes() == t["nodes"].tobytes() and again["paths"].tobytes() == t["paths"].tobytes()
    print("light tree %-16s K %7d  depth %2d" % (name, K, depth.max()))


def test_builder_rejects_bad_input():
    v = _quad_tris(3)
    for w in ([1, 0, 1], [1, -1, 1], [1, np.nan, 1], [1, np.inf, 1]):
        with pytest.raises(EzrtError):
            api.build_light_tree(v, np.array(w, np.float32))
    bad = v.copy()
    bad[1, 4] = np.inf
    with pytest.raises(EzrtError):
        api.build_light_tree(bad, np.ones(3, np.float32))
    assert len(api.build_light_tree(np.zeros((0, 9), np.float32), np.zeros(0, np.float32))["phi"]) == 0


# ------------------------------------------------------------------ the selection law
def _points(t, n, seed):
    rng = np.random.default_rng(seed)
    lo, hi = t["lo"][0].astype(np.float64), t["hi"][0].astype(np.float64)
    span = np.maximum(hi - lo, 1e-3)
    P = [rng.uniform(lo - span, hi + span, (n, 3)), t["lo"][rng.integers(0, len(t["lo"]), 4)],
         0.5 * (t["lo"][1:5] + t["hi"][1:5]) if len(t["lo"]) > 4 else t["lo"][:1], np.full((1, 3), 1e30), np.full((1, 3), np.nan)]
    return np.concatenate(P).astype(np.float32)


@pytest.mark.parametrize("name", ["p3_bunny", "s_lamps", "103692_lights", "two", "1000_duplicates", "weights_1e8"])
def test_selection_probabilities_sum_to_one(light_sets, name):
    verts, w = light_sets[name]
    t = api.build_light_tree(verts, w)
    K = len(w)
    D = int(t["depth"].max())
    worst = 0.0
    for P in _points(t, 6, 11):
        q = ot.prob(t, np.repeat(P[None], K, 0), np.arange(K)).astype(np.float64)
        assert (q >= 0).all()
        worst = max(worst, abs(q.sum() - 1.0))
    print("sum of P_sel %-16s depth %2d: largest |sum - 1| %.3g" % (name, D, worst))
    assert worst <= 3 * (D + 1) * 2.0 ** -24


def test_descent_equals_the_walk_bit_for_bit(light_sets):
    verts, w = light_sets["s_lamps"]
    t = api.build_light_tree(verts, w)
    n = 1000000
    rng = np.random.default_rng(2)
    P = np.concatenate([_points(t, n - 64, 3), np.repeat(_points(t, 0, 5), 8, 0)])[:n]
    r = rng.uniform(0, 1, len(P)).astype(np.float32)
    r[:32] = 1.0
    k, q = ot.descend(t, P, r)
    ok = k >= 0
    assert ok.mean() > 0.999
    assert ot.prob(t, P[ok], k[ok]).tobytes() == q[ok].tobytes()


def _inorder(t):
    out, stack = [], [0]
    while stack:   # right pushed first: left subtrees come first
        i = stack.pop()
        c = t["child"][i]
        if c < 0:
            out.append(~c)
        else:
            stack += [c + 1, c]
    return np.array(out)


def _exact_law(t, P):
    """The exact law of the descent at P over every 32-bit hash h (r = rand01(h) = fl32(h) 2^-32): the leaf is a non-decreasing
    function of r in in-order (each step's rescaling is monotone), so the h at which it passes each in-order position are found by
    bisection.  Returns (probabilities per light, probability of no sample)."""
    order = _inorder(t)
    K = len(order)
    pos = np.empty(K, np.int64)
    pos[order] = np.arange(K)

    def leaf_pos(h):
        r = (_fl32(h) * 2.0 ** -32).astype(np.float32)
        k, _ = ot.descend(t, np.repeat(P[None], len(h), 0), r)
        return np.where(k >= 0, pos[np.maximum(k, 0)], K)

    # first h with leaf position > j, for j = 0..K-1
    lo, hi = np.zeros(K, np.int64), np.full(K, TWO32, np.int64)
    j = np.arange(K)
    while (lo < hi).any():
        mid = (lo + hi) >> 1
        gt = leaf_pos(np.minimum(mid, TWO32 - 1)) > j
        hi = np.where(gt, mid, hi)
        lo = np.where(gt, lo, mid + 1)
    edges = np.concatenate([[0], lo])
    cnt = np.diff(edges)
    law = np.zeros(K)
    law[order] = cnt / float(TWO32)
    return law, (TWO32 - edges[-1]) / float(TWO32)


@pytest.mark.parametrize("name", ["s1m_lights", "s_lamps", "p3_bunny"])
def test_exact_descent_law(light_sets, name):
    verts, w = light_sets[name]
    t = api.build_light_tree(verts, w)
    K = len(w)
    worst = 0.0
    for P in _points(t, 3, 21)[:4]:
        law, none = _exact_law(t, P)
        nominal = ot.prob(t, np.repeat(P[None], K, 0), np.arange(K)).astype(np.float64)
        tv = 0.5 * (np.abs(law - nominal).sum() + none)
        worst = max(worst, tv)
    print("exact law of the descent %-12s K %5d depth %2d: largest total variation %.3g" % (name, K, int(t["depth"].max()), worst))
    assert worst <= 1e-4


# ------------------------------------------------------------------ the estimator
W, H = 32, 32


def _z(a, b, spp):
    z8, z16 = _block_z(a, b, spp, W, H, 8, 8), _block_z(a, b, spp, W, H, 16, 16)
    zf = float(_block_z(a, b, spp, W, H, H, W).max())
    return zf, float(z16.max()), float(z8.max())


def _pair(tris, nodes, eye, cam, spp, bounces, tree=None, mis_scale=1.0, **kw):
    out = []
    for flag in (False, True):
        cfg = api.RenderConfig(width=W, height=H, spp=spp, max_bounce=bounces, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam),
                               env_color=(0.05, 0.05, 0.06), light_tree=flag, **{k: v for k, v in kw.items() if k in ("env_light", "transmission",
                                                                                                                     "medium", "punctual_lights",
                                                                                                                     "textures", "emission_maps")})
        o = {k: v for k, v in kw.items() if k in ("emission_id", "lights", "m", "textures_", "hdr", "hdr_cache")}
        if "textures_" in o:
            o["textures"], o["texcoords"], o["texture_id"] = o.pop("textures_")
        img, luma2, _, _ = ot.render(tris, nodes, cfg, tree=tree if flag else None, mis_scale=mis_scale, **o)
        out.append(_stats(img, luma2))
    return out


def _cases():
    lamps = scenes.s_lamps(3, 3, rough=True)
    grid = _rough(scenes.s_grid(3, 2, 4))
    p3 = scenes.s_p3_bunny()
    t3 = np.asarray(p3[0], np.float32).reshape(-1, 36).copy()
    glass = t3.copy()
    bunny = (glass[:, 18:21] == 0).all(axis=1) & (glass[:, 21:24] == 1).all(axis=1)
    glass[bunny, 34], glass[bunny, 35] = 1.5, 0.8
    hdr = scenes.synth_hdr(64, 32)
    from tests import oracle_medium
    fog = oracle_medium.medium(sigma_t=0.4, albedo=(0.9, 0.8, 0.7), g=0.3, box_min=(-1.2, -1.0, -1.2), box_max=(1.2, 1.4, 1.2))
    st, sn, se, sc, stex, suv, sids, seid = scenes.s_screen()
    bt, bn, be, bc, btex, buv, bids, beid = scenes.s_p3_bunny_emission_mapped()
    return [
        ("s_lamps, 1 bounce", lamps, 1, 1024, {}),
        ("s_lamps, 4 bounces", lamps, 4, 256, {}),
        ("S-1M-like grid, rough", grid, 2, 512, {}),
        ("P3 bunny, env light", p3, 2, 512, dict(env_light=True, hdr=hdr, hdr_cache=api.hdr_cache(hdr))),
        ("P3 bunny, punctual lights", p3, 2, 512, dict(punctual_lights=True, lights=scenes.punctual_rig(t3, seed=1, power=0.5))),
        ("P3 bunny, fog", p3, 2, 512, dict(medium=True, m=fog)),
        ("P3 bunny, glass", (glass,) + tuple(p3[1:]), 2, 512, dict(transmission=True)),
        ("screen, emission maps", (st, sn, se, sc), 2, 512, dict(textures=True, emission_maps=True, emission_id=seid, textures_=(stex, suv, sids))),
        ("banded spheres, emission maps", (bt, bn, be, bc), 2, 512,
         dict(textures=True, emission_maps=True, emission_id=beid, textures_=(btex, buv, bids))),
    ]


@pytest.mark.parametrize("case", range(9))
def test_flagged_render_is_unbiased(case):
    name, (tris, nodes, eye, cam), bounces, spp, kw = _cases()[case]
    a, b = _pair(tris, nodes, eye, cam, spp, bounces, **kw)
    zf, z16, z8 = _z(a, b, spp)
    ratio = a[1].mean() / max(b[1].mean(), 1e-30)
    print("light tree vs mode 4, %-30s %d bounces, %d spp: frame z %.2f, 16x16 z %.2f, 8x8 z %.2f, variance ratio %.2f" %
          (name, bounces, spp, zf, z16, z8, ratio))
    assert zf <= 4 and z16 <= 5 and z8 <= 5, (name, zf, z16, z8)


def test_direct_light_from_a_screen_matches_float64(monkeypatch):
    """the emission maps' float64 quadrature check (tests/test_emission_maps_oracle.py: a floor at 1 bounce, lit by the mapped screen,
    pixels at distances from about 0.5 to 4 screen heights) with the light tree choosing the screen's triangles"""
    import tests.test_emission_maps_oracle as tem

    class Flagged:
        @staticmethod
        def render(tris, nodes, cfg, eid, **kw):
            cfg.light_tree = True
            return ot.render(tris, nodes, cfg, eid, **kw)

    monkeypatch.setattr(tem, "oe", Flagged)
    tem.test_direct_light_from_a_screen_matches_float64()


def test_too_tight_cones_stay_unbiased():
    """cos_o = 1 at every node: the importance wrongly culls or dims lights, yet BSDF samples reach them at MIS weight 1"""
    tris, nodes, eye, cam = scenes.s_lamps(3, 3, rough=True)
    t = ot.tree_of(tris)
    nodes_t = t["nodes"].copy()
    nodes_t[:, 7] = 1.0
    tight = api.light_tree_arrays(nodes_t, t["paths"])
    a, b = _pair(tris, nodes, eye, cam, 1024, 1, tree=tight)
    zf, z16, z8 = _z(a, b, 1024)
    print("too-tight cones: frame z %.2f, 16x16 z %.2f, 8x8 z %.2f" % (zf, z16, z8))
    assert zf <= 4 and z16 <= 5 and z8 <= 5


def test_mutated_mis_pdf_is_caught():
    """the emission hits' P_sel scaled by 1.03 (the restatement's test-only mis_scale) biases the estimator: the floor lit by the screen
    at 1 bounce, against the unmutated flagged render on disjoint frames, fails the frame z test, while a third, unmutated range passes"""
    tris, nodes, _, _, tex, uv, ids, eid = scenes.s_screen(bunny=False)
    tris = np.asarray(tris, np.float32).reshape(-1, 36)
    eye, cam = api.camera_look_at((0.0, 0.2, 2.2), (0.0, -1.4, -0.4), (0, 1, 0), 50.0, 4 / 3)
    Wm, Hm, n = 64, 48, 8192

    def arm(first, mis_scale):
        cfg = api.RenderConfig(width=Wm, height=Hm, spp=n, max_bounce=1, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam),
                               textures=True, emission_maps=True, light_tree=True, first_frame=first)
        img, l2, _, _ = ot.render(tris, nodes, cfg, eid, textures=tex, texcoords=uv, texture_id=ids, mis_scale=mis_scale)
        return _stats(*_mean_of(img, l2, first, n)) if first else _stats(img, l2)

    mutated, plain, again = arm(0, 1.03), arm(n, 1.0), arm(2 * n, 1.0)
    z_mut = float(_block_z(mutated, plain, n, Wm, Hm, Hm, Wm).max())
    z_null = float(_block_z(again, plain, n, Wm, Hm, Hm, Wm).max())
    print("hit-side P_sel x 1.03: frame z %.2f (unmutated: %.2f), frame mean moved by %.2e" % (z_mut, z_null, mutated[0].mean() / plain[0].mean() - 1))
    assert z_mut > 4 and z_null <= 4


def test_variance_at_equal_spp():
    """per-pixel luminance variance at 256 spp, 2 bounces, mode 4 against the flagged render: the mean over the frame, and the mean of
    each pixel's variance over its squared mean (the relative variance, which the bright pixels next to the lamps do not dominate)"""
    rows = []
    for name, sc in (("s_lamps(5, 5)", scenes.s_lamps(5, 5, rough=True)), ("S-1M-like grid", _rough(scenes.s_grid(3, 2, 4))),
                     ("P3 bunny", scenes.s_p3_bunny())):
        a, b = _pair(*sc, 256, 2)
        rel = lambda x: float(np.mean(x[1] / np.maximum(x[0] ** 2, 1e-6)))
        rows.append((name, float(a[1].mean()), float(b[1].mean()), rel(a), rel(b)))
    for name, va, vb, ra, rb in rows:
        print("per-pixel luminance variance at 256 spp, %-16s mode 4 %.4g, light tree %.4g (ratio %.2f); relative variance ratio %.2f" %
              (name, va, vb, va / vb, ra / rb))
    assert rows[0][2] < rows[0][1] and rows[0][4] * 1.3 < rows[0][3]
