"""The render path's lookups over every fp32 input, on the CPU (DESIGN.md section 2's deviations, section 15's filter).

Host C++ and the device disagree where a float is converted to an int out of int's range or from NaN: the host leaves it undefined
(x86 returns INT_MIN), the device saturates and turns NaN into 0.  ez_floor therefore converts nothing but |x| < 2^23, and every
texel index is clamped in float before its conversion.  These tests check

  - ez_floor against numpy.floor on all 2^32 bit patterns;
  - every texture, HDR-map and environment-table lookup at hostile coordinates under AddressSanitizer and UndefinedBehaviorSanitizer
    (tests/lookup_domains.cpp), which must report nothing;
  - whole renders of the CPU restatement built under the same sanitizers, with UVs past 2^31, hostile materials and NaN directions.
"""
import os
import subprocess
import sys
import textwrap
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from ezrt_b200 import build as _build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVER = os.path.join(ROOT, "tests", "lookup_domains.cpp")
SANITIZE = ["-fsanitize=address,undefined,float-cast-overflow", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer"]
HOST = [f for f in _build.HOST_FLAGS if f != "-fPIC"] + ["-Wno-misleading-indentation", "-Wno-unknown-pragmas", "-pthread"]


def _sanitizers_link(tmp):
    src = os.path.join(tmp, "probe.cpp")
    with open(src, "w") as f:
        f.write("int main() { return 0; }\n")
    r = subprocess.run(["g++"] + SANITIZE + [src, "-o", os.path.join(tmp, "probe")], capture_output=True, text=True)
    return r.returncode == 0


@pytest.fixture(scope="module")
def sanitized_dir(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("sanitized"))
    if not _sanitizers_link(d):
        pytest.skip("the address and undefined-behaviour sanitizer runtimes do not link here")
    return d


def _compile(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


def _assert_clean(r, what):
    report = r.stdout + r.stderr
    assert r.returncode == 0 and "runtime error" not in report and "AddressSanitizer" not in report, "%s:\n%s" % (what, report[-6000:])


# ------------------------------------------------------------------ ez_floor on every input
def _floor_chunk(k, chunk):
    from tests import oracle_binding as oracle
    x = (np.arange(k * chunk, (k + 1) * chunk, dtype=np.uint64).astype(np.uint32)).view(np.float32)
    got = oracle.eval_math(7, x)
    with np.errstate(invalid="ignore"):
        want = np.floor(x)
    want[want == 0] = 0.0           # floor(-0) = +0
    nan = np.isnan(x)
    same = (got.view(np.uint32) == want.view(np.uint32)) | (nan & np.isnan(got))
    bad = np.flatnonzero(~same)
    return None if bad.size == 0 else (x[bad[0]], got[bad[0]], want[bad[0]], bad.size)


def test_floor_is_exact_on_every_input():
    chunk = 1 << 24
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as pool:
        bad = [b for b in pool.map(lambda k: _floor_chunk(k, chunk), range((1 << 32) // chunk)) if b is not None]
    assert not bad, "ez_floor differs from floor on %d inputs, e.g. floor(%r) = %r, want %r" % (sum(b[3] for b in bad), *bad[0][:3])


# ------------------------------------------------------------------ the lookups under the sanitizers
def test_lookups_are_defined_on_hostile_coordinates(sanitized_dir):
    """ez_tex_sample and ez_normal_map at UVs from 0 to +-FLT_MAX, +-inf and NaN on textures from 1x1 to 16384x1, the oracle's tex2D in
    both filters, ez_env_texel and ez_env_pdf, NaN and zero-length directions included: no out-of-bounds read, no conversion out of
    int's range, and each result what the definition promises (tests/lookup_domains.cpp)."""
    exe = os.path.join(sanitized_dir, "lookup_domains")
    _compile(["g++"] + HOST + SANITIZE + ["-I", _build.INCLUDE, DRIVER, "-o", exe])
    r = subprocess.run([exe, "lookups"], capture_output=True, text=True, timeout=600)
    _assert_clean(r, "lookup_domains")
    assert "failures 0" in r.stdout


_RENDERS = textwrap.dedent("""
    import sys
    import numpy as np
    from ezrt_b200 import build as b
    for name in ("ORACLE_SO", "ORACLE_LIGHTS_SO", "ORACLE_ENV_LIGHT_SO", "ORACLE_TRANSMISSION_SO", "ORACLE_LENS_SO", "ORACLE_MEDIUM_SO",
                 "ORACLE_TEXTURES_SO", "ORACLE_MATERIAL_MAPS_SO"):
        setattr(b, name, sys.argv[1])   # the whole restatement chain, built under the sanitizers
    from ezrt_b200 import api, scenes
    from tests import oracle_env_light as oe, oracle_material_maps as om, oracle_transmission as ot
    from tests.test_transmission_oracle import HOSTILE, hostile_scene

    hdr = scenes.synth_hdr(64, 32)
    cache = api.hdr_cache(hdr)
    L4 = api.MODE_DISNEY_LIGHTS
    # the mapped P3 scene with every UV moved past 2^31, under the environment light and the thin lens
    tris, nodes, eye, cam, tex, uv, ids, mr, nm = scenes.s_p3_bunny_mapped()
    for shift in (np.float32(3e9), np.float32(-2.0 ** 31), np.float32(2.0 ** 40)):
        cfg = api.RenderConfig(width=16, height=16, spp=2, max_bounce=4, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam), textures=True,
                               material_maps=True, env_light=True, lens_radius=0.05, focus_distance=4.0)
        img = om.render(tris, nodes, cfg, tex, (uv + shift).astype(np.float32), ids, mr, nm, hdr=hdr, hdr_cache=cache, aov=True)[0]
        assert np.isfinite(img).all()
        print("mapped, UVs %+g: mean %.6f" % (shift, img.mean()))
    # the transmission lobe's hostile materials
    for name, _ in HOSTILE:
        t, n, e, c = hostile_scene(name)
        cfg = api.RenderConfig(width=16, height=16, spp=2, max_bounce=4, mode=L4, eye=tuple(e), camera_rotate=tuple(c), env_color=(1, 1, 1),
                               transmission=True, env_light=True)
        img = ot.oracle_render_transmission(t, n, cfg, hdr=hdr, hdr_cache=cache)[0]
        print("hostile %s: mean %.6f" % (name, img.mean()))
    # NaN directions into the map's lookups: NaN shading normals (every BRDF sample and its environment pdf), and a NaN camera
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    bad = np.array(tris, np.float32, copy=True)
    bad[:, 9:18] = np.nan
    for linear in (True, False):
        cfg = api.RenderConfig(width=16, height=16, spp=2, max_bounce=3, mode=L4, eye=tuple(eye), camera_rotate=tuple(cam), env_light=True)
        oe.oracle_render_env_light(bad, nodes, cfg, hdr=hdr, hdr_cache=cache, hdr_linear=linear)
        cfg = api.RenderConfig(width=16, height=16, spp=2, max_bounce=3, mode=L4, eye=tuple(eye), camera_rotate=(np.nan,) * 16, env_light=True)
        img = oe.oracle_render_env_light(tris, nodes, cfg, hdr=hdr, hdr_cache=cache, hdr_linear=linear)[0]
        print("NaN camera, %s: %d NaN values" % ("bilinear" if linear else "nearest", int(np.isnan(img).sum())))
    print("renders done")
""")


def test_renders_are_defined_under_the_sanitizers(sanitized_dir):
    """The restatement chain (tests/oracle_material_maps.cpp includes every restatement and the oracle) built with the sanitizers and
    loaded into a fresh interpreter: tiny renders of the mapped scene with UVs past 2^31, the hostile transmission materials and NaN
    directions into the environment lookups report nothing."""
    so = os.path.join(sanitized_dir, "libezrt_oracle_sanitized.so")
    _compile(["g++"] + _build.HOST_FLAGS + SANITIZE + ["-Wno-misleading-indentation", "-fopenmp", "-shared", "-I", _build.INCLUDE,
                                                         os.path.join(ROOT, "tests", "oracle_material_maps.cpp"), "-o", so])
    asan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0", OMP_NUM_THREADS="4")
    r = subprocess.run([sys.executable, "-c", _RENDERS, so], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    _assert_clean(r, "sanitized renders")
    assert "renders done" in r.stdout
