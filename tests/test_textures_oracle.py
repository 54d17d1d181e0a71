"""CPU checks of the base-colour textures (EZRT_PARAM_TEXTURES, DESIGN.md section 15): the committed sRGB table, the ABI struct, the C
definitions against a float64 model, the OBJ vt reader and the triangle list, and the restatement's invariances."""
import ctypes
import os
import re

import numpy as np
import pytest

from tests.texture_model import LUT, bary64, sample64

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_srgb_table_is_the_float64_eotf_rounded():
    text = open(os.path.join(ROOT, "include", "ezrt_srgb_table.inc")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    vals = np.array([float(x.rstrip("f")) for x in re.findall(r"[-+0-9.e]+f", text)], np.float32)
    assert vals.shape == (256,)
    assert vals.tobytes() == LUT.tobytes()
    assert vals[0] == 0.0 and vals[255] == 1.0 and (np.diff(vals) > 0).all()


def test_texture_struct_and_flag():
    from ezrt_b200 import _lib, api
    assert ctypes.sizeof(_lib.Texture) == 24   # int32 width, height; pointer; int32 reserved (+ padding)
    assert [f[0] for f in _lib.Texture._fields_] == ["width", "height", "rgba", "reserved"]
    assert api.PARAM_TEXTURES == 32
    header = open(os.path.join(ROOT, "include", "ezrt.h")).read()
    assert "#define EZRT_PARAM_TEXTURES 32" in header
    cfg = api.RenderConfig(textures=True, medium=True)
    assert cfg.to_struct().reserved[0] == 32 | 16


def test_model_filter_constants_and_wrap():
    rng = np.random.default_rng(1)
    t = np.zeros((3, 5, 4), np.uint8)
    t[:, :, :3] = (10, 128, 250)
    for u, v in rng.uniform(-50, 50, (50, 2)):
        assert np.array_equal(sample64(t, u, v), LUT[[10, 128, 250]].astype(np.float64))
    g = rng.integers(0, 256, (4, 6, 3)).astype(np.uint8)
    assert np.allclose(sample64(g, 0.3, 0.7), sample64(g, 5.3, -2.3))
    assert np.array_equal(sample64(g, np.inf, 0.0), np.ones(3))
    # texel centres: row 0 is the top (v near 1)
    assert np.allclose(sample64(g, 0.5 / 6, 1 - 0.5 / 4), LUT[g[0, 0]])


def test_model_barycentrics_on_a_floor_triangle():
    p = np.array([[[0.0, -1.4, 0.0], [2.0, -1.4, 0.0], [0.0, -1.4, 3.0]]])
    w = bary64(np.array([[0.5, -1.4, 0.75]]), p)
    assert np.allclose(w, [[0.5, 0.25, 0.25]])
    assert np.allclose(bary64(np.zeros((1, 3)), np.zeros((1, 3, 3))), 1.0 / 3.0)


# ---- the C definitions (include/ezrt_math.h, compiled in the restatement) against the float64 model ----

def test_c_table_equals_the_committed_one():
    from tests import oracle_textures as ot
    assert ot.srgb_table().tobytes() == LUT.tobytes()


def test_c_filter_matches_the_float64_model():
    from tests import oracle_textures as ot
    rng = np.random.default_rng(4)
    # beyond 2^23 every float is a whole number: s = t = 0 up to FLT_MAX, past 2^31 and int's range included
    huge = np.array([2.0 ** 31 - 128, 2.0 ** 31, -2.0 ** 31, 3e9, -3e9, 2.0 ** 40, -2.0 ** 40, 3.4028235e38, -3.4028235e38, 0.25], np.float32)
    for h, w in ((1, 1), (1, 9), (7, 1), (3, 5), (17, 13), (64, 64), (1, 16384)):
        t = rng.integers(0, 256, (h, w, 4)).astype(np.uint8)
        uv = np.concatenate([rng.uniform(-5, 5, (300, 2)),
                             np.array([[0, 0], [1, 1], [-1e-9, 1 - 1e-8], [-0.5, 2.5], [8388608, -8388609], [3e7, -3e7], [0.9999999, 1e-30],
                                       [-1e-30, -0.9999999]]),
                             np.stack(np.meshgrid(huge, huge), axis=-1).reshape(-1, 2)]).astype(np.float32)
        got = ot.tex_sample(t, uv)
        want = np.array([sample64(t, u, v) for u, v in uv])
        assert np.allclose(got, want, rtol=1e-5, atol=max(w, h) * 1e-6), (h, w)
    c = np.zeros((3, 4, 4), np.uint8)
    c[:, :, :3] = (7, 99, 201)
    assert (ot.tex_sample(c, rng.uniform(-9, 9, (50, 2))) == LUT[[7, 99, 201]]).all()   # four equal texels: that texel exactly
    nf = ot.tex_sample(c, np.array([[np.inf, 0], [0, np.nan], [-np.inf, np.inf]], np.float32))
    assert (nf == 1.0).all()


def test_c_barycentrics_match_float64():
    from tests import oracle_textures as ot
    rng = np.random.default_rng(6)
    p = rng.uniform(-3, 3, (400, 3, 3)).astype(np.float32)
    p[:100, :, 1] = np.float32(-1.4)   # the floor case: the reference's xy-projected weights collapse there
    p[100:150, :, 0] = np.float32(0.25)
    b = rng.dirichlet((1, 1, 1), 400)
    P = np.einsum("nk,nkj->nj", b, p.astype(np.float64)).astype(np.float32)
    ng = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]).astype(np.float32)
    got = ot.tri_bary(P, p[:, 0], p[:, 1], p[:, 2], ng)
    want = bary64(P, p)
    ok = np.abs(np.linalg.norm(ng, axis=1)) > 1e-2
    assert np.allclose(got[ok], want[ok], atol=2e-4)
    assert (np.ptp(got[:100], axis=0) > 0.1).all()
    deg = np.zeros((2, 3), np.float32)
    w = ot.tri_bary(np.ones((2, 3)), deg, deg, deg, deg)
    assert (w == np.float32(1.0 / 3.0)).all()


# ---- the OBJ vt reader and the triangle list ----

OBJ = """v 0 0 0
v 1 0 0
v 1 1 0
v 0 1 0
v 0.5 0.5 1
vt 0 0
vt 1 0 0.7
vt 1 1
vt 0 1
vt 0.5 0.5
vn 0 0 1
f 1/1 2/2 3/3
f 1/1/1 3/3/1 4/4/1
f 1//1 2//1 5//1
f 2 3 5
f -5/-5 -4/-4 -1/-1
f 1/1 2/2 3/3 4/4
"""


def _read(text, tid=None, hardened=True):
    from ezrt_b200 import api
    tl = api.TriangleList()
    flags = 1 | (2 if hardened else 0)
    tl.read_obj_text(text, api.Material(baseColor=(0.5, 0.6, 0.7)), api.transform_matrix(), flags, texture_id=tid)
    return tl


def test_obj_vt_faces_fans_and_relative_indices():
    tl = _read(OBJ, 3)
    uv, ids = tl.encode_texcoords()
    assert len(tl) == 7
    assert ids.tolist() == [3, 3, -1, -1, 3, 3, 3]
    assert uv[0].tolist() == [[0, 0], [1, 0], [1, 1]]
    assert uv[1].tolist() == [[0, 0], [1, 1], [0, 1]]
    assert uv[4].tolist() == [[0, 0], [1, 0], [0.5, 0.5]]
    assert uv[5].tolist() == [[0, 0], [1, 0], [1, 1]] and uv[6].tolist() == [[0, 0], [1, 1], [0, 1]]   # the fan
    assert (uv[2:4] == 0).all()
    plain = _read(OBJ.replace("f -5/-5 -4/-4 -1/-1\n", "f 1 2 5\n"), None)
    assert len(plain) == 7 and (plain.encode_texcoords()[1] == -1).all()


def test_obj_vt_geometry_equals_read_obj():
    from ezrt_b200 import api, scenes
    for text in (scenes.bunny_obj(), scenes.box_obj()):
        for proj in ("spherical", "planar"):
            a, b = _read(text, None, False), _read(scenes.obj_with_vt(text, proj), 0, False)
            assert a.encode_triangles().tobytes() == b.encode_triangles().tobytes()
            assert (b.encode_texcoords()[1] == 0).all()


def test_obj_vt_out_of_range_rejected():
    from ezrt_b200 import api
    for bad in ("f 1/6 2/2 3/3\n", "f 1/0 2/2 3/3\n", "f 1/-9 2/2 3/3\n"):
        with pytest.raises(api.EzrtError):
            _read(OBJ + bad, 0)
    with pytest.raises(api.EzrtError):
        _read(OBJ, -2)


@pytest.mark.parametrize("builder", [0, 1, 2])
def test_texcoords_follow_their_triangles_through_build_bvh(builder):
    from ezrt_b200 import api, scenes
    text = scenes.obj_with_vt(scenes.bunny_obj(), "spherical")
    tex = api.TriangleList()
    tex.read_obj_text(text, api.Material(), api.transform_matrix(), 1, texture_id=1)
    tex.read_obj_text(scenes.box_obj(), api.Material(baseColor=(0.2, 0.3, 0.4)), api.transform_matrix((0, 0, 0), (0, -1, 0), (4, 0.01, 4)), 0)
    plain = api.TriangleList()
    plain.read_obj_text(scenes.bunny_obj(), api.Material(), api.transform_matrix(), 1)
    plain.read_obj_text(scenes.box_obj(), api.Material(baseColor=(0.2, 0.3, 0.4)), api.transform_matrix((0, 0, 0), (0, -1, 0), (4, 0.01, 4)), 0)
    before = dict(zip(map(bytes, tex.encode_triangles()), zip(*tex.encode_texcoords())))
    t1, n1 = tex.build_bvh(4, builder)
    t2, n2 = plain.build_bvh(4, builder)
    assert t1.tobytes() == t2.tobytes() and n1.tobytes() == n2.tobytes()
    uv, ids = tex.encode_texcoords()
    for k in range(len(t1)):
        u0, i0 = before[bytes(t1[k])]
        assert i0 == ids[k] and u0.tobytes() == uv[k].tobytes()
    assert (ids == -1).sum() == 12


def test_textured_scene_is_the_plain_scene():
    from ezrt_b200 import scenes
    t, n, e, c = scenes.s_p3_bunny()
    t2, n2, e2, c2, tex, uv, ids = scenes.s_p3_bunny_textured()
    assert t.tobytes() == t2.tobytes() and n.tobytes() == n2.tobytes()
    assert np.bincount(ids + 1).tolist() == [320, 4968, 12]


# ---- restatement invariances ----

def _p3():
    from ezrt_b200 import api, scenes
    tris, nodes, eye, cam, tex, uv, ids = scenes.s_p3_bunny_textured()
    cfg = api.RenderConfig(width=24, height=16, spp=2, max_bounce=3, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam),
                           textures=True)
    return tris, nodes, cfg, tex, uv, ids


def test_restatement_white_and_no_ids_equal_mode4():
    from tests import oracle_lights, oracle_textures as ot
    tris, nodes, cfg, tex, uv, ids = _p3()
    ref, _, c = oracle_lights.oracle_render_lights(tris, nodes, cfg)
    for t, i in (([np.full((1, 1, 3), 255, np.uint8)], np.zeros_like(ids)), (tex, np.full_like(ids, -1))):
        img, _, _, c2 = ot.render(tris, nodes, cfg, t, uv, i)
        assert img.tobytes() == ref.tobytes() and c2["rays"] == c["rays"]


def test_restatement_constant_texture_is_premultiplied_base():
    from tests import oracle_lights, oracle_textures as ot
    tris, nodes, cfg, tex, uv, ids = _p3()
    col = np.array([[30, 140, 250], [200, 90, 10]])
    const = [np.broadcast_to(col[0].astype(np.uint8), (5, 3, 3)).copy(), np.broadcast_to(col[1].astype(np.uint8), (2, 2, 3)).copy()]
    img, _, _, _ = ot.render(tris, nodes, cfg, const, uv, ids)
    pre = np.array(tris, np.float32, copy=True)
    m = ids >= 0
    pre[m, 21:24] = pre[m, 21:24] * LUT[col[ids[m]]]
    ref, _, _ = oracle_lights.oracle_render_lights(pre, nodes, cfg)
    assert img.tobytes() == ref.tobytes()
    varying, _, _, _ = ot.render(tris, nodes, cfg, tex, uv, ids)
    assert not np.array_equal(varying, ref)
