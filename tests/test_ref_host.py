"""The product's host pipeline against THE REFERENCE'S OWN HOST CODE.

oracle/ref_host_shim.cpp compiles P5/main.cpp and lib/hdrloader.cpp from where they lie in the reference's source
tree (GL/GLUT: no-op stand-ins that capture uploads; glm: the subset main.cpp uses, oracle/ref_stubs/) and exposes
readObj / buildBVH / buildBVHwithSAH / calculateHdrCache.  The product (ezrt_b200/csrc/host_scene.cpp, SURVEY.md 8f rows)
must produce the same BYTES.  What the reference computed for the inputs below is committed (tests/golden/refhost.npz,
make_golden_refhost.py; tests/golden/refcompare.npz, make_golden_refcompare.py): the sampling cache of the synthetic
environment and crc32s of reference-built scenes, transforms, caches, OBJ face forms, and of what the reference's main() of
tutorial parts 4 and 5 uploads when run on generated stand-ins for the model and map it ships (main_dir)."""
import os
import zlib

import numpy as np
import pytest

from ezrt_b200 import api, scenes

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refhost.npz")
REFCOMPARE = os.path.join(os.path.dirname(GOLDEN), "refcompare.npz")


def same_bytes(a, b):
    a = np.ascontiguousarray(a, np.float32); b = np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def crc(a):
    return zlib.crc32(np.ascontiguousarray(a).tobytes())


def _write(tmp_path, name, text):
    p = tmp_path / name
    p.write_text(text)
    return str(p)


QUAD_OBJ = "v -1 0 -1\nv 1 0 -1\nv 1 0 1\nv -1 0 1\nf 1 2 3\nf 1 3 4\n"
MAIN_HDR = {4: "peppermint_powerplant_4k.hdr", 5: "chinese_garden_2k.hdr"}


def main_dir(tmp_path, part):
    """A directory laid out as the reference's main() of tutorial part `part` (4 or 5) expects it (models/, HDR/, shaders/), with
    generated stand-ins for the model and the environment map it ships: the blob mesh as teapot.obj, a unit quad, a 128x64
    run-length encoded RGBE map.  tests/golden/make_golden_refcompare.py runs that main() there and stores crc32s of its uploads."""
    from tests.test_host_scene import _write_hdr
    d = tmp_path / ("main%d" % part)
    for sub in ("models", "HDR", "shaders"):
        os.makedirs(d / sub, exist_ok=True)
    (d / "models" / "teapot.obj").write_text(scenes.blob_obj(3, 11))
    (d / "models" / "quad.obj").write_text(QUAD_OBJ)
    for f in ("fshader.fsh", "vshader.vsh", "pass2.fsh", "pass3.fsh"):
        (d / "shaders" / f).write_text("")
    rng = np.random.default_rng(part)
    rgbe = rng.integers(0, 256, (64, 128, 4), dtype=np.uint8)
    rgbe[:, :, 3] = rng.integers(120, 136, (64, 128))
    rgbe[10:20, 5:90, :] = rgbe[10, 5, :]  # long runs
    _write_hdr(str(d / "HDR" / MAIN_HDR[part]), rgbe, True)
    return str(d)


def p5_scene(src, builder):
    """P5/main.cpp:773-788 with the product: teapot + 13000-unit floor quad"""
    tl = api.TriangleList()
    m = api.Material(roughness=0.5, specular=1.0, metallic=1.0, clearcoat=1.0, clearcoatGloss=0.0, baseColor=(1, 0.73, 0.25))
    tl.read_obj(src + "/models/teapot.obj", m, api.transform_matrix((0, 0, 0), (0, -0.5, 0), (0.75, 0.75, 0.75)), True)
    m = api.Material(roughness=0.01, metallic=0.1, specular=1.0, clearcoat=1.0, clearcoatGloss=0.0, baseColor=(1, 1, 1))
    tl.read_obj(src + "/models/quad.obj", m, api.transform_matrix((0, 0, 0), (0, -0.5, 0), (13000.0, 0.01, 13000.0)), False)
    return tl.build_bvh(8, builder)


def test_reference_main_uploads_are_reproduced_byte_for_byte(tmp_path):
    """the reference's P5 main(), run on main_dir(5), uploaded a triangle buffer, a BVH buffer, the HDR map and its sampling cache
    (shapes and crc32s in tests/golden/refcompare.npz); the product's pipeline must produce the same bytes"""
    g = np.load(REFCOMPARE)
    want, shapes = [int(c) for c in g["main5_crc"]], [tuple(int(x) for x in s if x) for s in g["main5_shape"]]
    src = main_dir(tmp_path, 5)
    for builder in (api.BVH_SAH_LITERAL, api.BVH_SAH_FAST):
        tris, nodes = p5_scene(src, builder)
        assert [tris.shape, nodes.shape] == shapes[:2]
        assert crc(tris) == want[0], "triangle texture buffer, builder %d" % builder
        assert crc(nodes) == want[1], "BVH texture buffer, builder %d" % builder
    hdr = api.hdr_load(src + "/HDR/" + MAIN_HDR[5])
    assert hdr.shape == shapes[2] and crc(hdr) == want[2]
    assert crc(api.hdr_cache(hdr)) == want[3], "calculateHdrCache"


def test_reference_p4_main_uploads_are_reproduced_byte_for_byte(tmp_path):
    """P4/main.cpp:689-743 on main_dir(4): one golden teapot, SAH tree, the map"""
    g = np.load(REFCOMPARE)
    want = [int(c) for c in g["main4_crc"]]
    src = main_dir(tmp_path, 4)
    tl = api.TriangleList()
    m = api.Material(baseColor=(0.75, 0.7, 0.15), roughness=0.15, metallic=1.0, clearcoat=1.0, subsurface=1.0)
    tl.read_obj(src + "/models/teapot.obj", m, api.transform_matrix((0, 0, 0), (0, -0.4, 0), (1.75, 1.75, 1.75)), True)
    tris, nodes = tl.build_bvh(8, api.BVH_SAH_FAST)
    assert [crc(tris), crc(nodes)] == want[:2]
    assert crc(api.hdr_load(src + "/HDR/" + MAIN_HDR[4])) == want[2]


def synthetic_meshes(tmp_path, leaf_n):
    """[(obj path, material, trans16, smooth)]: three synthetic meshes under random transforms and materials"""
    blob = _write(tmp_path, "blob.obj", scenes.blob_obj(3, 11))
    sphere = _write(tmp_path, "sphere.obj", scenes.sphere_obj(2))
    box = _write(tmp_path, "box.obj", scenes.box_obj())
    rng = np.random.default_rng(leaf_n)
    meshes = []
    for path, smooth in ((blob, True), (sphere, False), (box, False), (blob, False), (sphere, True)):
        rot, tr, sc = rng.uniform(-180, 180, 3), rng.uniform(-2, 2, 3), rng.uniform(0.2, 3, 3)
        mat = api.Material(baseColor=tuple(rng.uniform(0, 1, 3)), emissive=tuple(rng.uniform(0, 5, 3)), roughness=float(rng.uniform()),
                           metallic=float(rng.uniform()), sheen=float(rng.uniform()), clearcoat=float(rng.uniform()))
        meshes.append((path, mat, (rot, tr, sc), smooth))
    return meshes


@pytest.mark.parametrize("leaf_n", [1, 4, 8, 13])
def test_builders_equal_reference_functions_on_synthetic_meshes(tmp_path, leaf_n):
    """the reference's transform, readObj and buildBVH / buildBVHwithSAH results for these meshes are stored (crc32 of its
    texture buffers, the transform matrices) in tests/golden/refcompare.npz"""
    g = np.load(REFCOMPARE)
    meshes = synthetic_meshes(tmp_path, leaf_n)
    trans = [api.transform_matrix(*map(tuple, rts)) for _, _, rts, _ in meshes]
    assert same_bytes(np.stack(trans), g["host_trans_%d" % leaf_n])  # same restatement of glm on both sides (see glm.hpp)
    for sah, builders in ((True, (api.BVH_SAH_LITERAL, api.BVH_SAH_FAST)), (False, (api.BVH_MEDIAN,))):
        want = [int(c) for c in g["host_build_%d_%d" % (leaf_n, sah)]]
        for b in builders:
            tl = api.TriangleList()
            for (p, m, _, s), t in zip(meshes, trans):
                tl.read_obj(p, m, t, s)
            tris, nodes = tl.build_bvh(leaf_n, b)
            assert [crc(tris), crc(nodes)] == want, (sah, b)


CACHE_SIZES = [(128, 64), (64, 32), (96, 40), (16, 8)]


@pytest.mark.parametrize("w,h", CACHE_SIZES)
def test_hdr_cache_equals_reference_function(w, h):
    """crc32 of the reference's calculateHdrCache of the same map, stored in tests/golden/refcompare.npz"""
    hdr = scenes.synth_hdr(w, h)
    assert crc(api.hdr_cache(hdr)) == int(np.load(REFCOMPARE)["host_cache_%dx%d" % (w, h)])


def test_golden_is_current():
    """refhost.npz's cache is what the reference's calculateHdrCache computes (crc32 of a separate run of it, refcompare.npz)"""
    assert crc(np.load(GOLDEN)["cache_128x64"]) == int(np.load(REFCOMPARE)["host_cache_128x64"])


def test_hdr_cache_equals_reference_computed_golden():
    """runs everywhere: the cache the REFERENCE's calculateHdrCache computed for the synthetic environment"""
    g = np.load(GOLDEN)
    hdr = scenes.synth_hdr(128, 64)
    assert crc(hdr) == int(g["hdr_crc_128x64"])
    assert same_bytes(api.hdr_cache(hdr), g["cache_128x64"])


def test_synthetic_scenes_equal_reference_built_golden(bunny_scene, grid_scene):
    """runs everywhere: crc32 of the arrays the REFERENCE's readObj + buildBVHwithSAH built from the same OBJ text"""
    g = np.load(GOLDEN)
    for name, sc in (("bunny", bunny_scene), ("grid", grid_scene)):
        tris, nodes = sc[0], sc[1]
        assert (crc(tris), crc(nodes)) == (int(g[name + "_crc_tris"]), int(g[name + "_crc_nodes"])), name


FORMS = ["v", "v/vt", "v/vt/vn"]
FORMS_MAT = dict(baseColor=(0.3, 0.5, 0.7))
FORMS_TRANS = ((10, 20, 30), (0.1, -0.2, 0.3), (1.5, 0.5, 1.0))


def forms_obj(form):
    """OBJ text whose faces use `form`, among vt / vn / comment / blank lines and trailing spaces"""
    base = scenes.blob_obj(2, 5).splitlines()
    rng = np.random.default_rng(len(form))
    out = ["# a comment", "", "vt 0.5 0.5", "vn 0 1 0"]
    for ln in base:
        if ln.startswith("f "):
            ids = ln.split()[1:]
            if form == "v":
                tok = ids
            elif form == "v/vt":
                tok = ["%s/1" % i for i in ids]
            elif form == "v/vt/vn":
                tok = ["%s/1/1" % i for i in ids]
            else:
                tok = ["%s//1" % i for i in ids]
            out.append("f " + " ".join(tok) + ("  " if rng.uniform() < 0.2 else ""))
        else:
            out.append(ln)
    return "\n".join(out) + "\n"


@pytest.mark.parametrize("form", FORMS)
def test_read_obj_face_forms_equal_reference(tmp_path, form):
    """the three `f` forms the reference's parser distinguishes by counting slashes (P5/main.cpp:306-333): same triangles and
    tree as the reference's own parser (crc32 of its texture buffers stored in tests/golden/refcompare.npz).  (`v//vn` makes
    the reference read uninitialised indices; the product reads the leading integer of every token, see
    test_read_obj_tolerates_the_form_the_reference_cannot_parse.)"""
    path = _write(tmp_path, "forms.obj", forms_obj(form))
    g = np.load(REFCOMPARE)
    for smooth in (False, True):
        tl = api.TriangleList()
        tl.read_obj(path, api.Material(**FORMS_MAT), api.transform_matrix(*FORMS_TRANS), smooth)
        tris, nodes = tl.build_bvh(8, api.BVH_SAH_FAST)
        assert [crc(tris), crc(nodes)] == [int(c) for c in g["host_forms_%s_%d" % (form.replace("/", "_"), smooth)]], (form, smooth)


def test_read_obj_tolerates_the_form_the_reference_cannot_parse():
    plain = "v 0 0 0\nv 1 0 0\nv 0 1 0\nv 0 0 1\nf 1 2 3\nf 1 3 4\n"
    vn = "v 0 0 0\nv 1 0 0\nv 0 1 0\nv 0 0 1\nvn 0 0 1\nf 1//1 2//1 3//1\nf 1//1 3//1 4//1\n"
    out = []
    for text in (plain, vn):
        tl = api.TriangleList()
        tl.read_obj_text(text, api.Material(), api.transform_matrix(), False)
        out.append(tl.build_bvh(8, api.BVH_SAH_LITERAL))
    assert same_bytes(out[0][0], out[1][0]) and same_bytes(out[0][1], out[1][1])
