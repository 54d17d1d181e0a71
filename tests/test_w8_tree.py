"""The 8-wide quantised acceleration tree (ezrt_b200/csrc/accel_w8.cpp, w8_node.h) is conservative: walking it with the
device's decode arithmetic and visit rule (CPU model tools/w8_model.cpp, built over the PRODUCT builders) finds, for every
ray, exactly the closest-hit distance brute force over all triangles finds.  No GPU needed."""
import os
import re
import subprocess

import numpy as np
import pytest

from ezrt_b200 import build, scenes


def _run_model(tmp_path, tris, rays, brute, *flags):
    exe = build.build_w8_model()
    tf, rf = os.path.join(tmp_path, "tris.f32"), os.path.join(tmp_path, "rays.f32")
    np.ascontiguousarray(tris, np.float32).tofile(tf)
    np.ascontiguousarray(rays, np.float32).tofile(rf)
    r = subprocess.run([exe, tf, str(tris.shape[0]), rf] + (["brute"] if brute else []) + list(flags), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout
    assert "differing from" in r.stdout and ": 0 of" in r.stdout, r.stdout
    assert "violations 0" in r.stdout, r.stdout        # the 4-wide collapse covers every triangle exactly once, leaves <= 4
    return r.stdout


def _rays(tris, n, seed):
    """Half start on surfaces (bounce-like, random directions incl. grazing and axis-parallel ones), half outside looking in."""
    rng = np.random.default_rng(seed)
    v = tris[:, :9].reshape(-1, 3, 3)
    pick = rng.integers(0, v.shape[0], n)
    w = rng.dirichlet((1, 1, 1), n).astype(np.float32)
    o = (v[pick] * w[:, :, None]).sum(1)
    d = rng.normal(size=(n, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    lo, hi = v.reshape(-1, 3).min(0), v.reshape(-1, 3).max(0)
    far = rng.uniform(lo - 3, hi + 3, (n // 2, 3)).astype(np.float32)
    o[: n // 2] = far
    d[: n // 2] = (v[pick[: n // 2]].mean(1) - far)
    d[: n // 2] /= np.linalg.norm(d[: n // 2], axis=1, keepdims=True)
    d[::101, 0] = 0.0            # exactly axis-parallel components: left to the exact kernel, must not miscount
    d[::103, 1] = 1e-30
    rays = np.zeros((n, 7), np.float32)
    rays[:, :3], rays[:, 3:6], rays[:, 6] = o, d, 1
    return rays


def test_w8_traversal_equals_brute_force_on_the_bunny_scene(tmp_path):
    tris, _, _, _ = scenes.s_p3_bunny()
    out = _run_model(str(tmp_path), tris, _rays(tris, 20000, 1), brute=True)
    assert "8-wide nodes" in out


def test_w8_traversal_on_a_degenerate_soup(tmp_path):
    """Coincident, needle and zero-area triangles: the builder must neither fail nor lose a hit."""
    rng = np.random.default_rng(5)
    n = 3000
    tris = np.zeros((n, 36), np.float32)
    p = rng.uniform(-1, 1, (n, 3, 3)).astype(np.float32) * rng.choice([1e-3, 0.1, 1.0], (n, 1, 1)).astype(np.float32)
    p += rng.uniform(-2, 2, (n, 1, 3)).astype(np.float32)
    p[:200] = p[0]                      # 200 coincident triangles
    p[200:260, 2] = p[200:260, 1]       # zero-area
    tris[:, :9] = p.reshape(n, 9)
    tris[:, 21:24] = 1.0
    _run_model(str(tmp_path), tris, _rays(tris, 6000, 2), brute=True)


def test_w8_traversal_large_grid_against_exact_boxes(tmp_path):
    tris, _, _, _ = scenes.s_grid(4, 3, 2, mesh="bunny")
    out = _run_model(str(tmp_path), tris, _rays(tris, 40000, 3), brute=False)
    print(out)


def _far_copy_rays(n, comp, seed):
    """Rays from below the floor of the P3 scene, under the bunny, along +z with x and y components `comp`."""
    rng = np.random.default_rng(seed)
    rays = np.zeros((n, 7), np.float32)
    rays[:, 0], rays[:, 1], rays[:, 2] = rng.uniform(-0.4, 1.0, n), rng.uniform(-2.5, -1.45, n), -3.0
    rays[:, 3:6] = (comp, comp, 1.0)
    rays[:, 6] = 1
    return rays


def _model_stat(out, pattern):
    m = re.search(pattern, out)
    assert m, (pattern, out)
    return m


def test_w8_decode_range_on_a_scene_10e8_wide(tmp_path):
    """The P3 scene and a copy 10^8 along x: the root's scale is 2^19, so 2^15 * scale * |1/d| overflows float for |1/d| =
    2^95, A = fma(-2^15, B, ...) becomes -inf and a ray with d_a > 0 misses every child.  The gate on |1/d| is derived from
    the tree (here 2^90): such rays go to the exact kernel, the others keep every hit."""
    tris, _, _, _ = scenes.s_p3_bunny()
    far = tris.copy()
    far[:, 0:9:3] += 1e8
    both = np.concatenate([tris, far])
    rays = np.concatenate([_far_copy_rays(256, 2.0 ** -95, 0), _far_copy_rays(256, 2.0 ** -80, 0)])
    out = _run_model(str(tmp_path), both, rays, brute=True)
    assert _model_stat(out, r"decode range \|1/d\| <= (\S+)").group(1) == "%g" % 2.0 ** 90
    assert _model_stat(out, r"rays left to the exact kernel (\d+)").group(1) == "256"
    assert int(_model_stat(out, r"\((\d+) of them hit\)").group(1)) > 100


def _pending_hist(out, kind="bounce"):
    """{pending triangles: share of the node visits that pend any} of the model's distribution line"""
    line = _model_stat(out, kind + r" rays: \S+ of the node visits pend triangles.*distribution(.*)").group(1)
    return {int(k): float(v) for k, v in (p.split(":") for p in line.split())}


def _model_rays(o, d):
    rays = np.zeros((len(o), 7), np.float32)
    rays[:, :3], rays[:, 3:6], rays[:, 6] = o, d, 1
    return rays


def _ties(out):
    return int(_model_stat(out, r"rays with a tie (\d+)").group(1))


def test_w8_gpu_scenes_load_the_cooperative_step(tmp_path):
    """The scenes and rays of tests/test_gpu_w8.py through the CPU model: node visits that leave all 32 triangle bits pending,
    and many rays with a tie, so that the GPU tests run the cooperative step's split owners and tie rules."""
    from tests import test_gpu_w8 as g
    tris = g.twin_scene()[0]
    o, d = g.grid_rays(20000, 31, 2.5)
    out = _run_model(str(tmp_path), tris, _model_rays(o, d), brute=False)
    assert _ties(out) > 0.2 * len(o)
    for ulps in (0, 3):
        tris = g.stack_scene(ulps, 40 + ulps)[0]
        o, d = g.stack_rays(tris, 600, 7 + ulps)
        out = _run_model(str(tmp_path), tris, _model_rays(o, d), brute=False)
        hist = _pending_hist(out)
        assert hist.get(32, 0.0) > 0.0, hist
        if ulps == 0:
            assert _ties(out) > 0.5 * len(o)
    tris = g.huge_floor_scene()[0]
    o, d = g.grid_rays(20000, 23, 1.2)
    out = _run_model(str(tmp_path), tris, _model_rays(o, d), brute=False)
    assert max(_pending_hist(out)) >= 24


def test_w8_decode_range_of_the_wide_gpu_scenes(tmp_path):
    """The 10^8 and 10^9 wide scenes of tests/test_gpu_w8.py: the model walks them with the same gate and finds every hit."""
    from tests import test_gpu_w8 as g
    for shift in (1e8, 1e9):
        tris, nodes, _, _ = g.far_scene(shift, 6)
        assert g.regular_tree(tris, nodes)
        o, d = g.far_rays(tris, 6000, 3)
        out = _run_model(str(tmp_path), tris, _model_rays(o, d), brute=False)
        limit = float(_model_stat(out, r"decode range \|1/d\| <= (\S+)").group(1))
        assert limit < 2.0 ** 96
        tiny = (np.abs(d) == 2.0 ** -95).any(1)
        assert int(_model_stat(out, r"rays left to the exact kernel (\d+)").group(1)) >= tiny.sum() > 1000


def _run_w4_check(tmp_path, tris):
    exe = build.build_w4_check()
    tf = os.path.join(tmp_path, "tris_w4.f32")
    np.ascontiguousarray(tris, np.float32).tofile(tf)
    r = subprocess.run([exe, tf, str(tris.shape[0])], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout
    return r.stdout


def test_w4_builder_is_thread_count_independent_and_well_formed(tmp_path):
    """ezrt_build_w4 (the default 4-wide form + its 96-byte Q16 twin): the same arrays for 1, 2, 5 and 16 threads and both collapse
    rules; every triangle in exactly one leaf, child boxes (exact and quantised) contain their triangles."""
    tris, _, _, _ = scenes.s_p3_bunny()
    out = _run_w4_check(str(tmp_path), tris)
    assert "violations 0" in out
    rng = np.random.default_rng(11)
    soup = np.zeros((70000, 36), np.float32)     # > 65536 binary nodes: the threaded path without the override, too
    c = rng.uniform(-5, 5, (70000, 1, 3))
    soup[:, :9] = (c + rng.uniform(-0.05, 0.05, (70000, 3, 3))).reshape(-1, 9).astype(np.float32)
    soup[:300, :9] = soup[0, :9]                 # coincident triangles
    _run_w4_check(str(tmp_path), soup)


_TOTALS = r"^totals %s rays (\d+) gate (\d+) ties (\d+) visits (\d+) tests (\d+) tests_max (\d+)$"


def _totals(out, kind):
    return dict(zip(("rays", "gate", "ties", "visits", "tests", "tests_max"), map(int, _model_stat(out, re.compile(_TOTALS % kind, re.M)).groups())))


def _as_kind(rays, kind):
    r = rays.copy()
    r[:, 6] = kind
    return r


def _any_hit_against_brute_force(tmp_path, tris, rays):
    """Shadow rays (kind 2) walked any-hit: hit exactly where brute force finds a hit (the model's own check, brute), min <=
    max, and on rays that miss everything both equal the closest-hit walk's count, and so do the node visits."""
    out = _run_model(tmp_path, tris, _as_kind(rays, 2), brute=True)
    s = _totals(out, "shadow")
    assert s["rays"] > 0 and s["tests"] <= s["tests_max"]
    assert s["tests"] < s["tests_max"]          # some first hits leave triangles of their node untested in the serial order
    hits = int(_model_stat(out, r"\((\d+) of them hit\)").group(1))
    assert 0 < hits < s["rays"]
    b = _totals(_run_model(tmp_path, tris, _as_kind(rays, 1), brute=True), "bounce")
    assert s["visits"] < b["visits"] and s["tests"] < b["tests"]   # the first hit ends a shadow ray early
    # per ray: a ray that misses walks the same nodes and tests the same triangles either way
    both = np.concatenate([_as_kind(rays, 1), _as_kind(rays, 2)])
    per = {}
    for r, kind, v, t, tm, hit in (map(int, m.groups()) for m in re.finditer(r"^ray (\d+) (\d) (\d+) (\d+) (\d+) (\d)$", _run_model(tmp_path, tris, both, True, "per_ray"), re.M)):
        per[(kind, r % len(rays))] = (v, t, tm, hit)
    misses = [r for (kind, r), x in per.items() if kind == 2 and not x[3]]
    assert len(misses) > 100
    for r in misses:
        v, t, tm, _ = per[(2, r)]
        assert t == tm and (v, t, t) == per[(1, r)][:3], (r, per[(1, r)], per[(2, r)])
    assert all(per[(1, r)][3] == per[(2, r)][3] for kind, r in per if kind == 2)


def test_w8_any_hit_walk_on_the_bunny_scene(tmp_path):
    tris, _, _, _ = scenes.s_p3_bunny()
    _any_hit_against_brute_force(str(tmp_path), tris, _rays(tris, 20000, 4))


def test_w8_any_hit_walk_on_a_degenerate_soup(tmp_path):
    rng = np.random.default_rng(6)
    n = 3000
    tris = np.zeros((n, 36), np.float32)
    p = rng.uniform(-1, 1, (n, 3, 3)).astype(np.float32) * rng.choice([1e-3, 0.1, 1.0], (n, 1, 1)).astype(np.float32)
    p += rng.uniform(-2, 2, (n, 1, 3)).astype(np.float32)
    p[:200] = p[0]                      # 200 coincident triangles
    p[200:260, 2] = p[200:260, 1]       # zero-area
    tris[:, :9] = p.reshape(n, 9)
    tris[:, 21:24] = 1.0
    _any_hit_against_brute_force(str(tmp_path), tris, _rays(tris, 6000, 7))


def test_w8_totals_agree_with_the_per_ray_averages(tmp_path):
    """The integer totals line and the per-ray summary line describe the same walk."""
    tris, _, _, _ = scenes.s_p3_bunny()
    rays = _rays(tris, 20000, 1)
    rays[1::3, 6] = 2
    out = _run_model(str(tmp_path), tris, rays, brute=True)
    gate = 0
    for kind in ("bounce", "shadow"):
        t = _totals(out, kind)
        m = _model_stat(out, r"%s rays (\d+): (\S+) node visits, (\S+) triangle tests" % kind)
        assert int(m.group(1)) == t["rays"]
        assert float(m.group(2)) == pytest.approx(t["visits"] / t["rays"], abs=0.005)
        assert float(m.group(3)) == pytest.approx(t["tests"] / t["rays"], abs=0.005)
        gate += t["gate"]
        assert t["rays"] + t["gate"] == (rays[:, 6] == (1 if kind == "bounce" else 2)).sum()
    assert gate == int(_model_stat(out, r"rays left to the exact kernel (\d+)").group(1)) > 0
    assert _totals(out, "bounce")["ties"] + _totals(out, "shadow")["ties"] == _ties(out)


def _run_threads(tmp_path, tris, threads="1,2,5,16"):
    exe = build.build_w8_model()
    tf, rf = os.path.join(tmp_path, "tris_t.f32"), os.path.join(tmp_path, "rays_t.f32")
    np.ascontiguousarray(tris, np.float32).tofile(tf)
    _rays(tris, 64, 9).tofile(rf)
    r = subprocess.run([exe, tf, str(tris.shape[0]), rf, "threads=" + threads], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout
    for t in threads.split(","):
        assert "threads %s: identical" % t in r.stdout, r.stdout


def test_w8_builder_is_thread_count_independent(tmp_path):
    """ezrt_build_w8's collapse runs on ezrt_host_threads() threads: the same node words, tri_order and leaf_first for 1, 2, 5
    and 16 threads, on the bunny and on 70,000 triangles with coincident ones (> 65,536 binary nodes)."""
    tris, _, _, _ = scenes.s_p3_bunny()
    _run_threads(str(tmp_path), tris)
    rng = np.random.default_rng(11)
    soup = np.zeros((70000, 36), np.float32)
    c = rng.uniform(-5, 5, (70000, 1, 3))
    soup[:, :9] = (c + rng.uniform(-0.05, 0.05, (70000, 3, 3))).reshape(-1, 9).astype(np.float32)
    soup[:300, :9] = soup[0, :9]
    _run_threads(str(tmp_path), soup)
