"""The device against the host over whole input domains (DESIGN.md section 2): ezrt_math.h's one-argument functions on all 2^32 inputs, pow
and atan2 on a grid of every exponent pair, the per-hit lookups at UVs up to +-FLT_MAX, +-inf and NaN, and textured and mapped renders of
the P3 scene with UVs beyond 2^31, bit for bit and ray for ray against the CPU restatement."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_binding as oracle
from tests import oracle_material_maps as om
from tests import oracle_textures as ot
from tests.texture_model import sample64

pytestmark = pytest.mark.gpu

ROUGH, METAL = 28, 25
CHUNK = 1 << 25
SPECIAL = np.array([0.0, 8388608.0, -8388608.0, 2.0 ** 31 - 128, 2.0 ** 31, -2.0 ** 31, 3e9, -3e9, 2.0 ** 40, -2.0 ** 40, 3.4028235e38,
                    -3.4028235e38, np.inf, -np.inf, np.nan], np.float32)


def _same_bits(a, b):
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _check_chunk(which, k):
    x = np.arange(k * CHUNK, (k + 1) * CHUNK, dtype=np.uint64).astype(np.uint32).view(np.float32)
    dev = api.eval_math(which, x)
    host = oracle.eval_math(which, x)
    bad = np.flatnonzero(~_same_bits(dev, host))
    return None if bad.size == 0 else (bad.size, x[bad[0]], dev[bad[0]], host[bad[0]])


@pytest.mark.parametrize("which,name", [(0, "sin"), (1, "cos"), (2, "log"), (3, "exp"), (6, "asin"), (7, "floor")])
def test_math_bit_exact_on_every_input(which, name):
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as pool:
        bad = [b for b in pool.map(lambda k: _check_chunk(which, k), range((1 << 32) // CHUNK)) if b is not None]
    assert not bad, "%s: device and host differ on %d inputs, e.g. at %r: %r vs %r" % (name, sum(b[0] for b in bad), *bad[0][1:])


def _grid():
    """every pair of exponent bytes under both signs with a few mantissas, and every pair of special values"""
    e = np.arange(256, dtype=np.uint32) << 23
    m = np.array([0, 1, 0x400000, 0x7FFFFF], np.uint32)
    one = (e[:, None] | m[None, :]).reshape(-1)
    one = np.concatenate([one, one | 0x80000000]).view(np.float32)
    a, b = np.meshgrid(one, one, indexing="ij")
    s = np.concatenate([SPECIAL, np.array([1.0, -1.0, -0.0, 1e-45, 0.5, 2.0, 1.17549435e-38], np.float32)])
    sa, sb = np.meshgrid(s, s, indexing="ij")
    return np.concatenate([a.reshape(-1), sa.reshape(-1)]), np.concatenate([b.reshape(-1), sb.reshape(-1)])


@pytest.mark.parametrize("which,name", [(4, "pow"), (5, "atan2")])
def test_two_argument_math_bit_exact_on_an_exponent_grid(which, name):
    a, b = _grid()
    dev, host = api.eval_math(which, a, b), oracle.eval_math(which, a, b)
    bad = np.flatnonzero(~_same_bits(dev, host))
    assert bad.size == 0, "%s: %d of %d differ, e.g. (%r, %r): %r vs %r" % (name, bad.size, a.size, a[bad[0]], b[bad[0]], dev[bad[0]], host[bad[0]])


@pytest.fixture(scope="module")
def p3():
    tris, nodes, eye, cam, tex, uv, ids, mr, nm = scenes.s_p3_bunny_mapped()
    hdr = scenes.synth_hdr(64, 32)
    return tris, nodes, eye, cam, tex, np.asarray(uv, np.float32), ids, mr, nm, hdr, api.hdr_cache(hdr)


def _scene(tris, nodes, tex, uv, ids, mr, nm, hdr, cache):
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    sc.set_textures(tex, uv, ids)
    if mr is not None:
        sc.set_material_maps(mr, nm)
    return sc


def _hostile_uvs(n):
    """each triangle's UVs from the special values: equal at its three vertices on two triangles in three, one apart on the third"""
    k = len(SPECIAL)
    uv = np.empty((n, 3, 2), np.float32)
    uv[:, :, 0] = SPECIAL[np.arange(n) % k][:, None]
    uv[:, :, 1] = SPECIAL[(np.arange(n) // k) % k][:, None]
    step = np.arange(n) % 3 == 2
    uv[step, 1, 0] += np.float32(1)
    uv[step, 2, 1] += np.float32(1)
    return uv


def test_lookups_at_hostile_uvs_equal_the_restatement(p3):
    tris, nodes, eye, cam, tex, _, ids, mr, nm, hdr, cache = p3
    n = len(tris)
    uv = _hostile_uvs(n)
    rng = np.random.default_rng(5)
    p = tris[:, :9].reshape(-1, 3, 3).astype(np.float64)
    b = rng.dirichlet((1, 1, 1), n)
    P = np.einsum("nk,nkj->nj", b, p)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    t = rng.uniform(0.5, 2.0, n)
    o, d, t = (P - d * t[:, None]).astype(np.float32), d.astype(np.float32), t.astype(np.float32)
    tri = np.arange(n, dtype=np.int32)
    sc = _scene(tris, nodes, tex, uv, ids, mr, nm, hdr, cache)
    try:
        tuv, tcol = sc.sample_textures(tri, P.astype(np.float32))
        got = sc.sample_materials(tri, o, d, t)
        sc.set_material_maps(None)
        plain = sc.sample_materials(tri, o, d, t)
    finally:
        sc.close()
    assert (~np.isfinite(got["uv"])).any() and (np.abs(got["uv"][np.isfinite(got["uv"])]) > 2.0 ** 31).any()
    base = tris[:, 21:24]
    uv6 = uv.reshape(n, 6)
    for i in range(n):
        for u, col in ((tuv[i], tcol[i]), (got["uv"][i], got["base_color"][i])):
            want = base[i] if ids[i] < 0 else base[i] * ot.tex_sample(tex[ids[i]], u[None])[0]
            assert col.tobytes() == want.astype(np.float32).tobytes(), (i, u)
            if ids[i] >= 0:
                assert np.allclose(col, base[i] * sample64(tex[ids[i]], *u), rtol=1e-5, atol=3e-5), (i, u)
        u = got["uv"][i]
        if mr[i] >= 0:
            f = om.unorm_sample(tex[mr[i]], u[None])[0]
            assert got["roughness"][i] == np.float32(tris[i, ROUGH] * f[1]) and got["metallic"][i] == np.float32(tris[i, METAL] * f[2]), i
        if nm[i] >= 0:
            ng = np.cross(p[i, 1] - p[i, 0], p[i, 2] - p[i, 0])
            c = np.dot(ng, d[i]) / np.linalg.norm(ng)
            if abs(c) > 1e-3:   # the side of the hit is the device's fp32 test; away from grazing float64 agrees with it
                f = om.unorm_sample(tex[nm[i]], u[None])
                want = om.normal_map(tris[i, :9].reshape(1, 3, 3), uv6[i:i + 1], u[None], f, plain["normal"][i:i + 1], [int(c > 0)], -d[i:i + 1])
                assert got["normal"][i].tobytes() == want[0].tobytes(), i
        else:
            assert got["normal"][i].tobytes() == plain["normal"][i].tobytes(), i


def _cfg(eye, cam, maps, **kw):
    base = dict(width=48, height=32, spp=2, max_bounce=4, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam), textures=True,
                material_maps=maps, env_light=True)
    base.update(kw)
    return api.RenderConfig(**base)


def _render(tris, nodes, cfg, tex, uv, ids, mr, nm, hdr, cache):
    sc = _scene(tris, nodes, tex, uv, ids, mr if cfg.material_maps else None, nm, hdr, cache)
    try:
        return sc.render(cfg), sc.counters()
    finally:
        sc.close()


@pytest.mark.parametrize("maps", [False, True])
@pytest.mark.parametrize("shift", [3e9, -2.0 ** 31, 2.0 ** 40])
def test_renders_with_uvs_beyond_2_31_equal_the_restatement(p3, maps, shift):
    tris, nodes, eye, cam, tex, uv, ids, mr, nm, hdr, cache = p3
    uv = (uv + np.float32(shift)).astype(np.float32)
    cfg = _cfg(eye, cam, maps)
    got, gc = _render(tris, nodes, cfg, tex, uv, ids, mr, nm, hdr, cache)
    if maps:
        ref, _, _, c = om.render(tris, nodes, cfg, tex, uv, ids, mr, nm, hdr=hdr, hdr_cache=cache)
    else:
        ref, _, _, c = ot.render(tris, nodes, cfg, tex, uv, ids, hdr=hdr, hdr_cache=cache)
    assert got.tobytes() == ref.tobytes(), "L-inf %.3g" % float(np.nanmax(np.abs(got - ref)))
    assert (gc.primary_rays, gc.bounce_rays, gc.shadow_rays) == (c["rays_primary"], c["rays_bounce"], c["rays_shadow"])


@pytest.mark.parametrize("maps", [False, True])
def test_equal_huge_uvs_render_as_uv_zero(p3, maps):
    """each triangle's three UVs equal and beyond 2^31: s = t = 0 as at UV (0, 0), so the same texels, and a normal map with a zero UV
    determinant falls back -- the render of all-zero UVs, bit for bit"""
    tris, nodes, eye, cam, tex, uv, ids, mr, nm, hdr, cache = p3
    n = len(tris)
    rng = np.random.default_rng(11)
    huge = SPECIAL[[3, 4, 5, 6, 7, 8, 9]]   # 2^31 - 128 ... -2^40
    same = np.empty((n, 3, 2), np.float32)
    same[:, :, 0] = rng.choice(huge, n)[:, None]
    same[:, :, 1] = rng.choice(huge, n)[:, None]
    cfg = _cfg(eye, cam, maps)
    a, ac = _render(tris, nodes, cfg, tex, same, ids, mr, nm, hdr, cache)
    b, bc = _render(tris, nodes, cfg, tex, np.zeros_like(same), ids, mr, nm, hdr, cache)
    assert a.tobytes() == b.tobytes() and (ac.primary_rays, ac.bounce_rays, ac.shadow_rays) == (bc.primary_rays, bc.bounce_rays, bc.shadow_rays)
