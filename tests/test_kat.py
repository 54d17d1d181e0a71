"""Known-answer tests that pin the oracle (and the shared tables) to values derivable directly
from the reference's constants (SURVEY.md section 4) -- the only reference-provided pins there are."""
import os
import re
import struct
import subprocess
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _table():
    text = open(os.path.join(ROOT, "include", "ezrt_sobol_table.inc")).read()
    return [int(x[:-1]) for x in re.findall(r"\d+u", text)]


def test_pi_literal_is_one_ulp_below_float_pi(oracle):
    # "#define PI 3.1415926", P5/fsh:27
    assert struct.pack("<f", oracle.pi()) == struct.pack("<I", 0x40490FDA)


def test_wang_hash_chain_from_seed_1(oracle):
    # P5/fsh:320-331
    h, r = oracle.wang_chain(1, 3)
    assert list(h) == [663891101, 1738326990, 801461103]
    np.testing.assert_allclose(r, [0.15457419, 0.40473580, 0.18660471], rtol=0, atol=1e-8)


def test_sobol_first_points_match_joe_kuo(oracle):
    # sobol(d, grayCode(i)), i = 0..7, dims 0..3 (P5/fsh:356-369; T5/tutorial.md:241-247)
    expect = {
        0: [0, .5, .75, .25, .375, .875, .625, .125],
        1: [0, .5, .25, .75, .375, .875, .125, .625],
        2: [0, .5, .25, .75, .625, .125, .875, .375],
        3: [0, .5, .25, .75, .875, .375, .625, .125],
    }
    for d, vals in expect.items():
        assert [oracle.sobol(d, i) for i in range(8)] == vals


def test_sobol_table_checksum_and_reference_literal():
    # 0xAB08B2B2: crc32 of the V[8*32] literal of P5/fsh, which tests/golden/make_golden_refcompare.py compares with the table
    t = _table()
    assert len(t) == 256
    assert zlib.crc32(struct.pack("<256I", *t)) == 0xAB08B2B2


def test_cranley_patterson_seed_and_wrap(oracle):
    # pseed = (px*1973 + py*9277 + 59*26699) | 1, two wang_hash draws, wrap into [0,1] (P5/fsh:378-396)
    assert 114514 // 1919 == 59
    px, py = 17, 5
    h, r = oracle.wang_chain((px * 1973 + py * 9277 + 59 * 26699) | 1, 2)
    x, y = oracle.cp_rotation(0.75, 0.5, px, py)
    ex = np.float32(0.75) + r[0]
    ey = np.float32(0.5) + r[1]
    ex = ex - np.float32(1) if ex > 1 else ex
    ey = ey - np.float32(1) if ey > 1 else ey
    assert (np.float32(x), np.float32(y)) == (ex, ey)
    assert 0.0 <= x <= 1.0 and 0.0 <= y <= 1.0


# the largest error of each function over every fp32 input of its domain against float64 libm, in ulps of the exact result (rounded
# up from the measured 13.79, 0.829, 0.99999, 2.404 and 2.831); sin and cos also in absolute error over |x| < 8192 (measured 7.82e-8)
WHOLE_DOMAIN_ULP = {"sin": 14.0, "cos": 14.0, "log": 0.85, "exp": 1.0, "asin": 2.45, "atan": 2.85}   # sin, cos: |x| <= 4 pi
WHOLE_DOMAIN_ABS = {"sin": 8e-8, "cos": 8e-8}


def test_math_functions_are_accurate(oracle, tmp_path):
    """ezrt_math.h defines sin/cos/log/exp/atan2/asin itself; they must still be those functions: whole-domain bounds for the one-argument
    functions (tests/lookup_domains.cpp's scan, on every hardware thread), and random inputs for pow and atan2."""
    from ezrt_b200 import build as _build
    exe = str(tmp_path / "scan")
    src = os.path.join(ROOT, "tests", "lookup_domains.cpp")
    r = subprocess.run(["g++"] + [f for f in _build.HOST_FLAGS if f != "-fPIC"] + ["-Wno-misleading-indentation", "-Wno-unknown-pragmas", "-pthread",
                        "-I", _build.INCLUDE, src, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for fn, bound in WHOLE_DOMAIN_ULP.items():
        out = subprocess.run([exe, "scan", fn], capture_output=True, text=True, timeout=900).stdout
        m = re.search(r"inputs (\d+) max_ulp (\S+) at (\S+) max_abs (\S+)", out)
        assert m, out
        assert int(m.group(1)) > 2 ** 30 and float(m.group(2)) <= bound, out
        assert float(m.group(4)) <= WHOLE_DOMAIN_ABS.get(fn, 0.0), out
    rng = np.random.default_rng(0)
    a = rng.uniform(1e-6, 1, 20000).astype(np.float32); b = rng.uniform(0, 1, 20000).astype(np.float32)
    np.testing.assert_allclose(oracle.eval_math(4, a, b), np.power(a.astype(np.float64), b.astype(np.float64)), rtol=4e-6)
    y = rng.uniform(-2, 2, 20000).astype(np.float32); z = rng.uniform(-2, 2, 20000).astype(np.float32)
    np.testing.assert_allclose(oracle.eval_math(5, y, z), np.arctan2(y.astype(np.float64), z.astype(np.float64)), atol=5e-7)
