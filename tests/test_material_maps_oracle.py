"""CPU tests of the material maps' definition (EZRT_PARAM_MATERIAL_MAPS; include/ezrt_math.h, DESIGN.md section 16) and of its render
restatement (tests/oracle_material_maps.cpp).

The C tangent frame and mapped normal are checked against an independent float64 model on random and hostile triangles; the restatement
by exact invariances against the textures' restatement and against scenes whose materials carry the maps' constant values."""
import sys
import os

import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_material_maps as om
from tests import oracle_textures
from tests.material_maps_model import UNORM, normal_map64, tangent_frame64, unorm_sample64

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import gen_srgb_table  # noqa: E402

ROUGH, METAL = 28, 25   # the roughness and metallic floats of a triangle record (Material.as_array at offset 18)


def test_unorm8_table_is_c_over_255_rounded():
    want = (np.arange(256, dtype=np.float64) / 255.0).astype(np.float32)
    assert om.unorm8_table().tobytes() == want.tobytes()
    assert gen_srgb_table.unorm8_table().tobytes() == want.tobytes() and UNORM.tobytes() == want.tobytes()


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _cases(rng, n):
    p = rng.uniform(-2, 2, (n, 3, 3)).astype(np.float32)
    uv6 = rng.uniform(-3, 3, (n, 6)).astype(np.float32)
    ng = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    N = _unit(ng + rng.normal(0, 0.3, (n, 3)) * np.linalg.norm(ng, axis=1, keepdims=True)).astype(np.float32)
    inside = rng.integers(0, 2, n).astype(np.int32)
    V = _unit(N.astype(np.float64) + rng.normal(0, 0.5, (n, 3))).astype(np.float32)
    f = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    uv = rng.uniform(-4, 4, (n, 2)).astype(np.float32)
    return p, uv6, uv, f, N, inside, V


def _check(p, uv6, uv, f, N, inside, V, atol=2e-4):
    got = om.normal_map(p, uv6, uv, f, N, inside, V)
    fell = mapped = 0
    for i in range(len(p)):
        want = normal_map64(p[i], uv6[i], uv[i], f[i], N[i], inside[i], V[i])
        if want is None:
            assert got[i].tobytes() == N[i].tobytes(), "row %d: the fallback is surface_hit's N bit for bit" % i
            fell += 1
        else:
            assert np.allclose(got[i], want, atol=atol), (i, got[i], want)
            mapped += 1
    return fell, mapped


def test_normal_map_matches_the_float64_model_on_random_triangles():
    rng = np.random.default_rng(1)
    p, uv6, uv, f, N, inside, V = _cases(rng, 4000)
    # keep the random set away from the borders of the fallbacks, where fp32 and float64 may decide differently
    keep = []
    for i in range(len(p)):
        No = -N[i] if inside[i] else N[i]
        fr = tangent_frame64(p[i], uv6[i], No)
        det = (uv6[i, 2] - uv6[i, 0]) * (uv6[i, 5] - uv6[i, 1]) - (uv6[i, 4] - uv6[i, 0]) * (uv6[i, 3] - uv6[i, 1])
        if abs(det) < 1e-2:
            continue
        if fr is not None:
            T, B = fr
            nt = 2.0 * f[i].astype(np.float64) - 1.0
            raw = nt[0] * T + nt[1] * B + nt[2] * No
            m = raw / np.linalg.norm(raw) * (-1 if inside[i] else 1)
            if np.linalg.norm(raw) < 1e-2 or abs(np.dot(m, V[i])) < 1e-3:
                continue
        keep.append(i)
    keep = np.array(keep)
    fell, mapped = _check(*(a[keep] for a in (p, uv6, uv, f, N, inside, V)))
    assert fell > 200 and mapped > 1000


def test_tangent_frame_matches_the_model_and_is_orthonormal():
    rng = np.random.default_rng(2)
    p, uv6, _, _, N, _, _ = _cases(rng, 2000)
    T, B, ok = om.tangent_frame(p, uv6, N)
    assert ok.sum() > 1900
    for i in np.nonzero(ok)[0]:
        want = tangent_frame64(p[i], uv6[i], N[i])
        assert want is not None
        assert np.allclose(T[i], want[0], atol=1e-4) and np.allclose(B[i], want[1], atol=1e-4)
    assert np.allclose(np.einsum("ij,ij->i", T[ok], N[ok]), 0, atol=1e-5)
    assert np.allclose(np.linalg.norm(T[ok], axis=1), 1, atol=1e-6) and np.allclose(np.linalg.norm(B[ok], axis=1), 1, atol=1e-5)


def _one(p, uv6, uv, f, N, inside, V):
    a = [np.asarray(x, np.float32)[None] for x in (p, uv6, uv, f, N)]
    return om.normal_map(a[0], a[1], a[2], a[3], a[4], [int(inside)], np.asarray(V, np.float32)[None])[0]


FLAT = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)   # in the z = 0 plane, normal +z; u along x, v along y
UV = np.array([0, 0, 1, 0, 0, 1], np.float32)
Z = np.array([0, 0, 1], np.float32)


def test_handedness_follows_the_uv_layout():
    f = np.array([0.5, 0.8, 0.8], np.float32)   # n_t = (0, 0.6, 0.6): halfway toward +B
    n = _one(FLAT, UV, (0.2, 0.2), f, Z, 0, Z)
    assert n[1] > 0.4   # +v runs along +y
    mirrored = np.array([0, 1, 1, 1, 0, 0], np.float32)   # v flipped: det < 0, B_uv along -y
    m = _one(FLAT, mirrored, (0.2, 0.2), f, Z, 0, Z)
    assert m[1] < -0.4 and np.allclose(_one(FLAT, mirrored, (0.2, 0.2), f, Z, 0, Z), normal_map64(FLAT, mirrored, (0.2, 0.2), f, Z, 0, Z), atol=1e-6)
    # vertex normals disagreeing with the winding: the handedness still comes from the UVs
    flipped = np.array([[0, 0, 0], [0, 1, 0], [1, 0, 0]], np.float32)
    fl = _one(flipped, np.array([0, 0, 0, 1, 1, 0], np.float32), (0.2, 0.2), f, Z, 0, Z)
    assert fl[1] > 0.4


def test_fallbacks_return_the_shading_normal_bit_for_bit():
    f = np.array([0.8, 0.3, 0.9], np.float32)
    N = _unit(np.array([0.1, -0.05, 1.0])).astype(np.float32)
    cases = {
        "zero-area uv": (FLAT, np.array([0, 0, 1, 1, 2, 2], np.float32), (0.1, 0.1), f, N, 0, Z),
        "T parallel to N_o": (FLAT, UV, (0.1, 0.1), f, np.array([1, 0, 0], np.float32), 0, np.array([1, 0, 0], np.float32)),
        "non-finite u": (FLAT, UV, (np.inf, 0.1), f, N, 0, Z),
        "non-finite v": (FLAT, UV, (0.1, np.nan), f, N, 0, Z),
        "non-finite vertex uv": (FLAT, np.array([np.inf, 0, 1, 0, 0, 1], np.float32), (0.1, 0.1), f, N, 0, Z),
        "view below the mapped normal": (FLAT, UV, (0.1, 0.1), np.array([1.0, 0.5, 0.55], np.float32), Z, 0, _unit(np.array([-1.0, 0, 0.05]))),
        "zero n": (FLAT, UV, (0.1, 0.1), np.array([0.5, 0.5, 0.5], np.float32), Z, 0, Z),
    }
    for name, c in cases.items():
        got = _one(*c)
        assert got.tobytes() == np.asarray(c[4], np.float32).tobytes(), name
        assert normal_map64(*c) is None, name


def test_inside_hits_flip_the_mapped_normal():
    f = np.array([0.7, 0.4, 0.9], np.float32)
    out = _one(FLAT, UV, (0.3, 0.3), f, Z, 0, Z)
    ins = _one(FLAT, UV, (0.3, 0.3), f, -Z, 1, -Z)   # the same surface seen from behind: N = -N_o
    assert ins.tobytes() == (-out).tobytes()
    assert np.allclose(ins, normal_map64(FLAT, UV, (0.3, 0.3), f, -Z, 1, -Z), atol=1e-6)


def test_huge_uvs():
    rng = np.random.default_rng(4)
    n = 300
    p, uv6, uv, f, N, inside, V = _cases(rng, n)
    uv6 = uv6 + np.float32(2.0 ** 23) * np.sign(rng.normal(size=(n, 1))).astype(np.float32)   # |u| >= 2^23: UV deltas are whole numbers
    uv6 = uv6.astype(np.float32)
    uv = (uv + np.float32(2.0 ** 23)).astype(np.float32)
    got = om.normal_map(p, uv6, uv, f, N, inside, V)
    for i in range(n):
        want = normal_map64(p[i], uv6[i], uv[i], f[i], N[i], inside[i], V[i])
        if want is None:
            assert got[i].tobytes() == N[i].tobytes()
        else:
            assert np.allclose(got[i], want, atol=2e-4)


def test_mr_decode_at_channel_edges():
    vals = np.array([0, 1, 127, 128, 254, 255], np.uint8)
    tex = np.zeros((1, len(vals), 4), np.uint8)
    tex[0, :, 1] = vals
    tex[0, :, 2] = vals[::-1]
    tex[0, :, 0] = 77
    u = (np.arange(len(vals)) + 0.5) / len(vals)   # texel centres
    uv = np.stack([u, np.full_like(u, 0.5)], axis=1).astype(np.float32)
    f = om.unorm_sample(tex, uv)
    assert f[:, 1].tobytes() == UNORM[vals].tobytes() and f[:, 2].tobytes() == UNORM[vals[::-1]].tobytes()
    r, m = om.mr_apply(f, np.full(len(vals), 0.7, np.float32), np.full(len(vals), 0.9, np.float32))
    assert r.tobytes() == (np.float32(0.7) * UNORM[vals]).astype(np.float32).tobytes()
    assert m.tobytes() == (np.float32(0.9) * UNORM[vals[::-1]]).astype(np.float32).tobytes()
    # between texels: the bilinear filter against the float64 model
    rng = np.random.default_rng(6)
    t = rng.integers(0, 256, (5, 7, 4)).astype(np.uint8)
    uvr = rng.uniform(-3, 3, (200, 2)).astype(np.float32)
    got = om.unorm_sample(t, uvr)
    want = np.array([unorm_sample64(t, *x) for x in uvr])
    assert np.allclose(got, want, rtol=1e-5, atol=3e-6)


@pytest.fixture(scope="module")
def p3():
    tris, nodes, eye, cam, tex, uv, ids, mr, nm = scenes.s_p3_bunny_mapped()
    hdr = scenes.synth_hdr(64, 32)
    return tris, nodes, eye, cam, tex, uv, ids, mr, nm, hdr, api.hdr_cache(hdr)


def _cfg(eye, cam, **kw):
    base = dict(width=24, height=16, spp=2, max_bounce=4, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam), textures=True,
                material_maps=True)
    base.update(kw)
    return api.RenderConfig(**base)


def test_mapped_scene_geometry_is_the_textured_scenes():
    a = scenes.s_p3_bunny_mapped()
    b = scenes.s_p3_bunny_textured()
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes() and a[5].tobytes() == b[5].tobytes()
    assert (a[7] >= 0).sum() > 0 and (a[8] >= 0).sum() > 0 and ((a[7] < 0) & (a[6] >= 0)).any() and ((a[8] < 0) & (a[6] >= 0)).any()


@pytest.mark.parametrize("opt", ["plain", "env_lens", "medium"])
def test_no_maps_and_white_mr_equal_the_textures_restatement(p3, opt):
    from tests import oracle_medium
    tris, nodes, eye, cam, tex, uv, ids, mr, nm, hdr, cache = p3
    kw = dict(plain={}, env_lens=dict(env_light=True, lens_radius=0.12, focus_distance=3.6), medium=dict(medium=True, env_light=True))[opt]
    m = oracle_medium.medium(sigma_t=0.6, albedo=(0.9, 0.8, 0.7), g=0.4, box_min=(-1.2, -1.0, -1.2), box_max=(1.2, 1.4, 1.2)) if opt == "medium" else None
    cfg = _cfg(eye, cam, **kw)
    ref = oracle_textures.render(tris, nodes, _cfg(eye, cam, material_maps=False, **kw), tex, uv, ids, m=m, hdr=hdr, hdr_cache=cache, aov=True)
    none = np.full(len(tris), -1, np.int32)
    got = om.render(tris, nodes, cfg, tex, uv, ids, none, none, m=m, hdr=hdr, hdr_cache=cache, aov=True)
    white = tex + [np.full((2, 3, 4), 255, np.uint8)]
    got2 = om.render(tris, nodes, cfg, white, uv, ids, np.where(ids >= 0, len(tex), -1), none, m=m, hdr=hdr, hdr_cache=cache, aov=True)
    for g in (got, got2):
        assert g[0].tobytes() == ref[0].tobytes() and g[2].tobytes() == ref[2].tobytes() and g[3] == ref[3]


def _transmissive(tris):
    t = np.array(tris, np.float32, copy=True)
    bunny = (t[:, 18:21] == 0).all(axis=1) & (t[:, 21:24] == 1).all(axis=1)
    t[bunny, 34] = 1.5
    t[bunny, 35] = 0.8
    return t


@pytest.mark.parametrize("trans", [False, True])
def test_constant_mr_maps_equal_premultiplied_materials(p3, trans):
    tris, nodes, eye, cam, tex, uv, ids, _, _, hdr, cache = p3
    if trans:
        tris = _transmissive(tris)
    rng = np.random.default_rng(8)
    cols = rng.integers(0, 256, (3, 3))
    consts = [np.broadcast_to(np.append(c, 255).astype(np.uint8), (h, w, 4)).copy() for c, (h, w) in zip(cols, [(1, 1), (2, 5), (4, 3)])]
    mr = np.where(ids >= 0, rng.integers(-1, 3, len(tris)) + len(tex), -1).astype(np.int32)
    mr[mr == len(tex) - 1] = -1
    none = np.full(len(tris), -1, np.int32)
    pre = np.array(tris, np.float32, copy=True)
    on = mr >= 0
    c = cols[mr[on] - len(tex)]
    pre[on, ROUGH] = (pre[on, ROUGH] * UNORM[c[:, 1]]).astype(np.float32)
    pre[on, METAL] = (pre[on, METAL] * UNORM[c[:, 2]]).astype(np.float32)
    cfg = _cfg(eye, cam, env_light=True, transmission=trans, max_bounce=5)
    got = om.render(tris, nodes, cfg, tex + consts, uv, ids, mr, none, hdr=hdr, hdr_cache=cache, aov=True)
    ref = om.render(pre, nodes, cfg, tex + consts, uv, ids, none, none, hdr=hdr, hdr_cache=cache, aov=True)
    assert got[0].tobytes() == ref[0].tobytes() and got[2].tobytes() == ref[2].tobytes() and got[3] == ref[3]
    plain = om.render(tris, nodes, cfg, tex + consts, uv, ids, none, none, hdr=hdr, hdr_cache=cache)
    assert not np.array_equal(plain[0], got[0])


def test_invalid_maps_renders_are_rejected(p3):
    tris, nodes, eye, cam, tex, uv, ids, mr, nm, hdr, cache = p3
    with pytest.raises(ValueError):
        om.render(tris, nodes, _cfg(eye, cam, textures=False), tex, uv, ids, mr, nm)
    bad = mr.copy()
    bad[3] = len(tex)
    with pytest.raises(ValueError):
        om.render(tris, nodes, _cfg(eye, cam), tex, uv, ids, bad, nm)
    with pytest.raises(ValueError):
        om.render(tris, nodes, _cfg(eye, cam, medium=True, transmission=True), tex, uv, ids, mr, nm)
