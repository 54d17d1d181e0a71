"""The oracle against THE REFERENCE'S OWN SHADER SOURCE.

oracle/ref_shader/ transpiles P3/P4/P5 shaders/fshader.fsh (read where they lie in the
reference's source tree, never copied) to C++ and runs them per fragment on the CPU; GLSL's built-ins -- which the GLSL
specification leaves bit-unspecified -- are bound to include/ezrt_math.h.  Everything else (statements,
expression order, control flow, constants, the Sobol table, the RNG seeding) is the reference's text.

  * frames rendered that way are committed in tests/golden/refshader.npz and the hand-written oracle
    must reproduce them bit for bit (the GPU tests replay them too);
  * more inputs (other shapes, cameras, filters, bounce counts, a closed box, a degenerate triangle soup, the
    tone-mapping pass), with fingerprints of the transpiled shaders' outputs committed in tests/golden/refcompare.npz
    (tests/golden/make_golden_refcompare.py, which needs the reference's sources)."""
import zlib

import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import refshader_cases as cases


def same_bits(a, b):
    a = np.ascontiguousarray(a, np.float32); b = np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and bool(((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all())


@pytest.mark.parametrize("name", cases.SCENES)
def test_oracle_reproduces_reference_shader_frames(oracle, name):
    g = cases.load()
    hdr, cache = cases.environment()
    tris, nodes, eye, cam = cases.scene(name)
    for case in cases.CASES:
        key, mode, mb, lin, first, spp = case
        want = g["%s_%s" % (name, key)]
        assert np.isfinite(want).all() and float(want.mean()) > 0.05, "golden frame is not a trivial image"
        for traverse in (api.TRAVERSE_REFERENCE, api.TRAVERSE_PRUNED):
            fb = g["%s_m3" % name].copy() if first else None
            got, _ = oracle.render(tris, nodes, cases.config(case, eye, cam, traverse=traverse), hdr=hdr, hdr_cache=cache, hdr_linear=lin,
                                   framebuffer=fb)
            assert same_bits(got, want), "%s %s traverse %d" % (name, key, traverse)


def test_golden_inputs_are_the_committed_ones():
    """refshader.npz was rendered from exactly these arrays (synth.npz pins their crc32)."""
    import os
    import zlib
    s = np.load(os.path.join(cases.GOLDEN, "synth.npz"))
    hdr, cache = cases.environment()
    crc = lambda a: zlib.crc32(np.ascontiguousarray(a).tobytes())
    assert crc(hdr) == int(s["hdr_crc"]) and crc(cache) == int(s["cache_crc"])
    tris, nodes, _, _ = cases.scene("bunny")
    assert crc(tris) == int(s["bunny_crc_tris"]) and crc(nodes) == int(s["bunny_crc_nodes"])
    tris, nodes, _, _ = cases.scene("grid")
    assert crc(tris) == int(s["grid_crc_tris"]) and crc(nodes) == int(s["grid_crc_nodes"])


def test_golden_frames_are_current():
    """the committed frames are what the transpiled shaders produce (fingerprints of a separate run of them, refcompare.npz)"""
    g = cases.load()
    want = cases.load_refcompare()
    for case in cases.CASES[:4]:
        key = case[0]
        assert fingerprint(g["bunny_" + key])[0] == want["current_bunny_" + key][0], key


LIVE = [(0, 2), (0, 3), (1, 4), (1, 1), (2, 2), (2, 4), (3, 2), (3, 3)]


def live_run(grid_scene, mode, bounces, linear):
    """(key, tris, nodes, cfg, hdr, cache, linear): another image shape, camera, environment size, filter and bounce count than
    the committed frames"""
    tris, nodes, _, _ = grid_scene
    hdr = scenes.synth_hdr(64, 32)
    cache = api.hdr_cache(hdr)
    eye, cam = api.camera_orbit(37.0, 12.0, 5.5)
    cfg = api.RenderConfig(width=37, height=23, spp=4, max_bounce=bounces, mode=mode, eye=tuple(eye), camera_rotate=tuple(cam),
                           traverse=api.TRAVERSE_REFERENCE)
    return "live_%d_%d_%d" % (mode, bounces, linear), tris, nodes, cfg, hdr, cache, linear


def box_runs():
    """camera inside closed geometry (isInside hits, every path terminates on geometry or an emitter)"""
    tl = api.TriangleList()
    tl.read_obj_text(scenes.box_obj(), api.Material(baseColor=(0.7, 0.6, 0.5), roughness=0.4, metallic=0.3), api.transform_matrix((0, 0, 0), (0, 0, 0), (3, 3, 3)), False)
    tl.read_obj_text(scenes.sphere_obj(2), api.Material(baseColor=(1, 1, 1), emissive=(9, 8, 7)), api.transform_matrix((0, 0, 0), (0, 0.6, 0), (0.5, 0.5, 0.5)), True)
    tris, nodes = tl.build_bvh(4, api.BVH_SAH_LITERAL)
    hdr, cache = cases.environment()
    eye, cam = api.camera_orbit(20.0, -10.0, 1.2)
    out = []
    for mode, mb, lin in ((0, 3, False), (1, 4, False), (2, 3, True), (3, 3, True)):
        cfg = api.RenderConfig(width=32, height=24, spp=3, max_bounce=mb, mode=mode, eye=tuple(eye), camera_rotate=tuple(cam),
                               traverse=api.TRAVERSE_REFERENCE)
        out.append(("box_%d" % mode, tris, nodes, cfg, hdr, cache, lin))
    return out


def soup_runs():
    """zero-area triangles (NaN normals), slivers, duplicated vertices, axis-aligned coordinates"""
    from tests.test_gpu_parity import _soup
    tl = api.TriangleList()
    tl.append_encoded(_soup(3000, 4))
    tris, nodes = tl.build_bvh(8)
    hdr, cache = cases.environment()
    eye, cam = api.camera_orbit(30.0, 20.0, 6.0)
    out = []
    for mode, mb, lin in ((0, 3, False), (1, 3, False), (2, 2, True), (3, 2, True)):
        cfg = api.RenderConfig(width=64, height=48, spp=2, max_bounce=mb, mode=mode, eye=tuple(eye), camera_rotate=tuple(cam),
                               traverse=api.TRAVERSE_REFERENCE)
        out.append(("soup_%d" % mode, tris, nodes, cfg, hdr, cache, lin))
    return out


def fingerprint(img):
    """(crc32 of the float32 bits with every NaN made the same NaN, mean): what same_bits compares, in 16 bytes"""
    a = np.ascontiguousarray(img, np.float32)
    a = np.where(np.isnan(a), np.float32(np.nan), a)
    return np.array([zlib.crc32(a.tobytes()), float(np.nanmean(a))], np.float64)


def check_runs(oracle, runs):
    want_all = cases.load_refcompare()
    for key, tris, nodes, cfg, hdr, cache, lin in runs:
        want = want_all["shader_" + key]
        got, _ = oracle.render(tris, nodes, cfg, hdr=hdr, hdr_cache=cache, hdr_linear=lin)
        assert want[1] > 0.01, key
        assert fingerprint(got)[0] == want[0], key


@pytest.mark.parametrize("mode,bounces", LIVE)
@pytest.mark.parametrize("linear", [False, True])
def test_oracle_equals_transpiled_shader_live(oracle, grid_scene, mode, bounces, linear):
    """the fingerprint of the transpiled shader's frame of these inputs is stored in tests/golden/refcompare.npz"""
    check_runs(oracle, [live_run(grid_scene, mode, bounces, linear)])


def test_oracle_equals_transpiled_shader_inside_a_box(oracle):
    check_runs(oracle, box_runs())


def _hdr_frame(seed=5, h=24, w=40, c=3):
    rng = np.random.default_rng(seed)
    fb = (rng.uniform(0, 1, (h, w, c)) ** 4 * 40.0).astype(np.float32)  # HDR range, many dark texels
    fb[0, 0, :3] = 0.0
    fb[0, 1, :3] = (1e-30, 1.0, 3e4)
    return fb


@pytest.mark.parametrize("channels", [3, 4])
def test_tonemap_equals_transpiled_pass3_shader(oracle, channels):
    """shaders/pass3.fsh (identical in parts 3, 4, 5): toneMapping(c, 1.5) then pow(c, 1/2.2); the fingerprint of
    its output is stored in tests/golden/refcompare.npz"""
    fb = _hdr_frame(c=channels)
    want = cases.load_refcompare()["pass3_c%d" % channels]
    assert fingerprint(oracle.tonemap(fb))[0] == want[0]


def test_tonemap_reproduces_reference_pass3_golden(oracle):
    """runs everywhere: pass3 output of the reference shader for a fixed frame, committed in refshader.npz"""
    g = cases.load()
    assert same_bits(oracle.tonemap(_hdr_frame()), g["pass3_out"])


def test_oracle_equals_transpiled_shader_on_degenerate_soup(oracle):
    """the NaN / tie behaviour of the oracle is the shader's, statement by statement"""
    check_runs(oracle, soup_runs())


def p5_main_run(tmp_path):
    """the reference's P5 set-up end to end: what its main() uploads for main_dir(5) (tests/test_ref_host.py checks that the product
    produces those bytes), rendered with its own camera (P5/main.cpp:796-798) at a reduced size"""
    from tests import test_ref_host
    src = test_ref_host.main_dir(tmp_path, 5)
    tris, nodes = test_ref_host.p5_scene(src, api.BVH_SAH_LITERAL)
    hdr = api.hdr_load(src + "/HDR/" + test_ref_host.MAIN_HDR[5])
    eye, cam = api.camera_orbit(90.0, 10.0, 2.0)
    cfg = api.RenderConfig(width=64, height=64, spp=2, max_bounce=2, mode=api.MODE_DISNEY_IS_MIS_P5, eye=tuple(eye), camera_rotate=tuple(cam),
                           traverse=api.TRAVERSE_REFERENCE)
    return "p5_main", tris, nodes, cfg, hdr, api.hdr_cache(hdr), True


def test_oracle_equals_transpiled_shader_on_the_reference_p5_scene(oracle, tmp_path):
    """the transpiled P5 shader rendered the reference main()'s own uploads (fingerprint in refcompare.npz); the oracle must agree"""
    key, tris, nodes, cfg, hdr, cache, lin = p5_main_run(tmp_path)
    _, c = oracle.render(tris, nodes, cfg, hdr=hdr, hdr_cache=cache, hdr_linear=lin)
    assert c["rays_shadow"] > 0
    check_runs(oracle, [(key, tris, nodes, cfg, hdr, cache, lin)])
