#!/usr/bin/env python
"""Generate tests/golden/refcompare.npz where the reference's sources are present (oracle/build_ref.py compiles them).

It holds what THE REFERENCE'S OWN CODE computes for the inputs of the comparison tests, so that those tests run
anywhere and keep comparing with the reference:
  shader_<key>            crc32 and mean of the frames of the transpiled fragment shaders (tests/test_ref_shader.py: live_run,
                          box_runs, soup_runs; crc32 of test_ref_shader.bits_crc, NaNs canonical)
  pass3_c3 / pass3_c4     the same of shaders/pass3.fsh on the fixed HDR frame, 3 and 4 channels
  host_trans_<leaf_n>     the reference's transform matrices of the synthetic meshes (tests/test_ref_host.py)
  host_build_<leaf_n>_<sah>   crc32 of the triangle / BVH texture buffers readObj + buildBVH(withSAH) produce for them
  host_cache_<w>x<h>      crc32 of calculateHdrCache of scenes.synth_hdr(w, h)
  host_forms_<form>_<smooth>  crc32 of the texture buffers of the OBJ face-form file
  hdrload_rle<0|1>        crc32 of the reference's hdrloader decoding the RGBE test file (tests/test_host_scene.py)
  main<4|5>_crc / _shape  crc32s and shapes of what the reference's main() of tutorial part 4 / 5 uploads when run in
                          tests/test_ref_host.main_dir (generated model and map in place of the shipped ones)
  shader_p5_main          the transpiled P5 shader's frame of those part-5 uploads (tests/test_ref_shader.p5_main_run)
  hdrload_main5           crc32 of the reference's hdrloader decoding that part-5 map
  current_bunny_<key>     a second run of the transpiled shaders on the first four refshader.npz cases
It also checks that include/ezrt_sobol_table.inc is the reference shader's V[] literal, which tests/test_kat.py pins by crc32."""
import ctypes as C
import os
import pathlib
import re
import sys
import tempfile
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from ezrt_b200 import api, build, scenes  # noqa: E402
from tests import refhost_binding as refhost  # noqa: E402
from tests import refshader_binding as refshader  # noqa: E402
from tests import refshader_cases as cases  # noqa: E402
from tests import test_host_scene, test_kat, test_ref_host, test_ref_shader  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def crc(a):
    return zlib.crc32(np.ascontiguousarray(a).tobytes())


def main():
    assert refshader.available() and refhost.available() and build.build_reference_hdrloader(), "needs the reference's sources"
    src = open(os.path.join(build.REFERENCE_P5, "shaders", "fshader.fsh")).read()
    m = re.search(r"const uint V\[8\*32\] = \{\s*([0-9u,\s]+)\};", src)
    assert [int(x.strip().rstrip("u")) for x in m.group(1).split(",") if x.strip()] == test_kat._table()
    d = {}
    grid = scenes.s_grid(3, 2, 2)
    runs = [test_ref_shader.live_run(grid, m, b, lin) for m, b in test_ref_shader.LIVE for lin in (False, True)]
    runs += test_ref_shader.box_runs() + test_ref_shader.soup_runs()
    for key, tris, nodes, cfg, hdr, cache, lin in runs:
        d["shader_" + key] = test_ref_shader.fingerprint(refshader.render(tris, nodes, cfg, hdr, cache, hdr_linear=lin))
    tris, nodes, eye, cam = cases.scene("bunny")
    hdr, cache = cases.environment()
    for case in cases.CASES[:4]:
        d["current_bunny_" + case[0]] = test_ref_shader.fingerprint(refshader.render(tris, nodes, cases.config(case, eye, cam), hdr, cache, hdr_linear=case[3]))
    for ch in (3, 4):
        d["pass3_c%d" % ch] = test_ref_shader.fingerprint(refshader.pass3(test_ref_shader._hdr_frame(c=ch)))
    with tempfile.TemporaryDirectory() as tmp:
        tmp = pathlib.Path(tmp)
        for leaf_n in (1, 4, 8, 13):
            meshes = test_ref_host.synthetic_meshes(tmp, leaf_n)
            trans = [refhost.transform_matrix(*rts) for _, _, rts, _ in meshes]
            d["host_trans_%d" % leaf_n] = np.stack(trans)
            for sah in (True, False):
                tris, nodes = refhost.build_scene([(p, m.as_array(), t, s) for (p, m, _, s), t in zip(meshes, trans)], leaf_n, sah)
                d["host_build_%d_%d" % (leaf_n, sah)] = np.array([crc(tris), crc(nodes)], np.uint32)
        for form in test_ref_host.FORMS:
            path = str(tmp / "forms.obj")
            pathlib.Path(path).write_text(test_ref_host.forms_obj(form))
            mat = api.Material(**test_ref_host.FORMS_MAT)
            trans = api.transform_matrix(*test_ref_host.FORMS_TRANS)
            for smooth in (False, True):
                tris, nodes = refhost.build_scene([(path, mat.as_array(), trans, smooth)], 8, True)
                d["host_forms_%s_%d" % (form.replace("/", "_"), smooth)] = np.array([crc(tris), crc(nodes)], np.uint32)
        ref = C.CDLL(build.REF_HDR_SO)
        for part in (4, 5):
            src = test_ref_host.main_dir(tmp, part)
            up = refhost.run_main(part, src)
            d["main%d_crc" % part] = np.array([crc(a) for a in up], np.uint32)
            d["main%d_shape" % part] = np.array([list(a.shape) + [0] * (3 - a.ndim) for a in up])
        key, _, _, cfg, _, _, lin = test_ref_shader.p5_main_run(tmp)
        img = refshader.render(up[0], up[1], cfg, up[2], up[3], hdr_linear=lin)
        d["shader_" + key] = test_ref_shader.fingerprint(img)
        print("p5 main():", [a.shape for a in up], "frame mean", d["shader_" + key][1])
        W, H, ptr = C.c_int(), C.c_int(), C.POINTER(C.c_float)()
        assert ref.ref_hdr_load((src + "/HDR/" + test_ref_host.MAIN_HDR[5]).encode(), C.byref(W), C.byref(H), C.byref(ptr)) == 0
        d["hdrload_main5"] = np.uint32(crc(np.ctypeslib.as_array(ptr, shape=(H.value, W.value, 3)).copy()))
        ref.ref_hdr_free(ptr)
        for rle in (False, True):
            path = str(tmp / "t.hdr")
            h, w = test_host_scene.write_rgbe_test_file(path, rle).shape[:2]
            W, H, ptr = C.c_int(), C.c_int(), C.POINTER(C.c_float)()
            assert ref.ref_hdr_load(path.encode(), C.byref(W), C.byref(H), C.byref(ptr)) == 0 and (W.value, H.value) == (w, h)
            d["hdrload_rle%d" % rle] = np.uint32(crc(np.ctypeslib.as_array(ptr, shape=(h, w, 3)).copy()))
            ref.ref_hdr_free(ptr)
    for w, h in test_ref_host.CACHE_SIZES:
        d["host_cache_%dx%d" % (w, h)] = np.uint32(crc(refhost.hdr_cache(scenes.synth_hdr(w, h))))
    np.savez_compressed(os.path.join(HERE, "refcompare.npz"), **d)
    print("wrote %d arrays" % len(d))


if __name__ == "__main__":
    main()
