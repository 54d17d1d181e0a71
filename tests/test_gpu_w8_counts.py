"""The counting kernels of the 8-wide traversal (params.profile = 2) against an exact CPU walk of the same rays.

A bounce ray's node visits and triangle tests in extend_w8 do not depend on the warp schedule: a lane with pending triangles
takes no node step, and the cooperative triangle step gives the serial order's results.  So every render's per-pass sums
are exact integers, and the CPU model of the traversal (tools/w8_model.cpp) must reproduce them from the rays the oracle
traces in the same render (the renders match bit for bit, so those are the GPU's rays):
  - bounce pass (k_extend_w8): node visits and triangle tests equal the model's closest-hit walk;
  - shadow pass (k_shadow_w8, any-hit): node visits equal; triangle tests lie between the serial order's count and every
    triangle pending at the node of the first hit (how the cooperative step splits an owner's run depends on the warp);
  - camera pass (k_extend_w8_camera, warp bundles): the model's bundle walk over the slots in the kernel's work order.
These counts are what DESIGN.md section 6 and bench.py's roofline are built on, and they prove that the model walks the
tree the GPU walks -- which tests/test_w8_tree.py relies on for its conservativeness proofs.  When a sum differs, the test
re-renders single pixels to name the first ray whose counts differ."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from ezrt_b200 import api, build, scenes

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE = 16
KINDS = ("camera", "bounce", "shadow")
DIAGNOSE_PIXELS = 24


# ------------------------------------------------------------------ scenes
def _scene(name):
    """(tris, nodes, eye, cam, env): the scene and the environment it needs at scene creation"""
    from tests import test_gpu_w8 as g
    if name == "bunny":   # 5,300 triangles: forced onto the 8-wide tree
        return scenes.s_p3_bunny() + ({"EZRT_ACCEL": "8"},)
    if name == "s1m":     # the tree DESIGN.md section 6's numbers are about
        return scenes.s_1m() + ({},)
    if name in ("stack0", "stack3"):
        ulps = int(name[-1])
        return g.stack_scene(ulps, 40 + ulps) + ({},)
    if name == "twins":
        return g.twin_scene() + ({},)
    if name == "floor":
        return g.huge_floor_scene() + ({},)
    raise KeyError(name)


_SCENES = {}


def _cached_scene(name):
    if name not in _SCENES:
        _SCENES[name] = _scene(name)
    return _SCENES[name]


def _cfg(eye, cam, **kw):
    base = dict(width=48, height=32, spp=2, max_bounce=2, eye=tuple(eye), camera_rotate=tuple(cam), env_color=(0.35, 0.45, 0.6))
    base.update(kw)
    return api.RenderConfig(**base)


def _with(cfg, **kw):
    return api.RenderConfig(**{**cfg.__dict__, **kw})


# ------------------------------------------------------------------ the GPU side
def gpu_counts(sc, cfg):
    """Render with the counting kernels -> (image, {pass: {visits, tests}}, step counts, phase cycles).  The camera pass's
    counts are the render's quantised node visits and triangle tests less those of the two other passes."""
    img = sc.render(_with(cfg, profile=2))
    c, st, cyc = sc.counters(), sc.w8_step_counts(), sc.w8_phase_cycles()
    b, s = st["k_extend_w8"], st["k_shadow_w8"]
    counts = dict(bounce=dict(visits=b["node_visits"], tests=b["triangle_tests"]), shadow=dict(visits=s["node_visits"], tests=s["triangle_tests"]),
                  camera=dict(visits=c.node_visits_96 - b["node_visits"] - s["node_visits"], tests=c.tri_tests - b["triangle_tests"] - s["triangle_tests"]))
    return img, counts, st, cyc


def camera_slot_rays(sc, cfg, pixel_major=True):
    """The camera pass's rays in its work order, as 7-float model records (kind 0): one batch of cfg.spp frames, one part.
    Work item i is sample slot (i mod spp) * per_frame + i / spp in pixel-major order, slot i in frame-major order
    (kernels.cu: AccelCameraIO::slot_of); a slot is (frame, 16x16 tile, position in the tile as eight 8x4 blocks)
    (slot_pixel, in_tile_xy).  Slots of clipped tiles outside the image hold a NaN ray: no bundle takes it."""
    tx_n, ty_n = -(-cfg.width // TILE), -(-cfg.height // TILE)
    per_frame = tx_n * ty_n * TILE * TILE
    nf = cfg.spp
    i = np.arange(per_frame * nf, dtype=np.int64)
    slot = (i % nf) * per_frame + i // nf if pixel_major else i
    frame, r = slot // per_frame, slot % per_frame
    tile, t = r >> 8, r & 255
    sub, lane = t >> 5, t & 31
    px = (tile % tx_n) * TILE + (sub & 1) * 8 + (lane & 7)
    py = (tile // tx_n) * TILE + (sub >> 1) * 4 + (lane >> 3)
    valid = (px < cfg.width) & (py < cfg.height)
    o, d = sc.camera_rays(cfg, px[valid], py[valid], cfg.first_frame + frame[valid])
    rays = np.full((len(i), 7), np.nan, np.float32)
    rays[:, 6] = 0
    rays[valid, :3], rays[valid, 3:6] = o, d
    return rays


# ------------------------------------------------------------------ the model side
_TOTALS = re.compile(r"^totals (\w+) rays (\d+) gate (\d+) ties (\d+) visits (\d+) tests (\d+) tests_max (\d+)$", re.M)
_BUNDLE = re.compile(r"^bundle totals bundles (\d+) members (\d+) visits (\d+) tests (\d+)$", re.M)


def run_model(tmp_path, tris, rays, *flags):
    """tools/w8_model over `rays` -> (stdout, {kind: {rays, gate, ties, visits, tests, tests_max}}, bundle totals or None)"""
    exe = build.build_w8_model()
    tf, rf = os.path.join(tmp_path, "tris.f32"), os.path.join(tmp_path, "rays.f32")
    np.ascontiguousarray(tris, np.float32).tofile(tf)
    np.ascontiguousarray(rays, np.float32).tofile(rf)
    r = subprocess.run([exe, tf, str(len(tris)), rf] + list(flags), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:]
    totals = {m.group(1): dict(zip(("rays", "gate", "ties", "visits", "tests", "tests_max"), map(int, m.groups()[1:]))) for m in _TOTALS.finditer(r.stdout)}
    assert set(totals) == set(KINDS), r.stdout[-4000:]
    m = _BUNDLE.search(r.stdout)
    bundle = dict(zip(("bundles", "members", "visits", "tests"), map(int, m.groups()))) if m else None
    return r.stdout, totals, bundle


def model_counts(tmp_path, tris, dump, camera):
    """The model's counts of a render: the dumped bounce and shadow rays walked per ray, the camera slots walked as bundles."""
    _, t, _ = run_model(tmp_path, tris, dump[dump[:, 6] > 0])
    _, _, b = run_model(tmp_path, tris, camera, "bundle")
    return dict(bounce=dict(visits=t["bounce"]["visits"], tests=t["bounce"]["tests"]),
                shadow=dict(visits=t["shadow"]["visits"], tests=t["shadow"]["tests"], tests_max=t["shadow"]["tests_max"]),
                camera=dict(visits=b["visits"], tests=b["tests"]), walked=t, bundle=b)


def mismatches(gpu, model):
    """The passes whose counts differ from the model's: exact except the shadow pass's triangle tests, which lie in
    [serial order, all pending at the node of the first hit]"""
    bad = []
    for k in KINDS:
        g, m = gpu[k], model[k]
        ok = g["visits"] == m["visits"] and (m["tests"] <= g["tests"] <= m["tests_max"] if k == "shadow" else g["tests"] == m["tests"])
        if not ok:
            bad.append("%s: GPU %d visits, %d tests; model %d visits, %s tests" %
                       (k, g["visits"], g["tests"], m["visits"], "%d..%d" % (m["tests"], m["tests_max"]) if k == "shadow" else m["tests"]))
    return bad


def _bits(v):
    return "(%s)" % ", ".join("0x%08x" % x for x in np.asarray(v, np.float32).view(np.uint32))


def first_differing_ray(oracle, sc, tris, nodes, cfg, hdr, tmp_path, pixel_major=True):
    """Re-render single pixels -- a 1x1 image at 1 spp and 1 bounce, frame k for k < DIAGNOSE_PIXELS, whose jitter spreads
    the camera ray over the whole view -- each one a per-ray count on the GPU, and walk the same rays in the model
    (per_ray).  Returns a description of the first pixel whose counts differ, with its rays as float bits, or None."""
    h, cache = hdr
    gpu, dumps, cams = [], [], []
    for k in range(DIAGNOSE_PIXELS):
        c1 = _with(cfg, width=1, height=1, spp=1, max_bounce=1, first_frame=cfg.first_frame + k, profile=0)
        _, counts, _, _ = gpu_counts(sc, c1)
        _, _, rays = oracle.render_rays(tris, nodes, c1, hdr=h, hdr_cache=cache)
        gpu.append(counts)
        dumps.append(rays[rays[:, 6] > 0])
        cams.append(camera_slot_rays(sc, c1, pixel_major))
    owner = np.concatenate([np.full(len(d), k) for k, d in enumerate(dumps)])
    out, _, _ = run_model(tmp_path, tris, np.concatenate(dumps), "per_ray")
    model = [dict(bounce=dict(visits=0, tests=0), shadow=dict(visits=0, tests=0, tests_max=0), camera=dict(visits=0, tests=0)) for _ in gpu]
    for r, kind, v, t, tm in (map(int, m.groups()) for m in re.finditer(r"^ray (\d+) (\d) (\d+) (\d+) (\d+) \d$", out, re.M)):
        e = model[owner[r]][KINDS[kind]]
        e["visits"] += v
        e["tests"] += t
        e.setdefault("tests_max", 0)
        e["tests_max"] += tm
    per = len(cams[0])
    out, _, _ = run_model(tmp_path, tris, np.concatenate(cams), "bundle", "per_ray")
    for at, v, t in (map(int, m.groups()) for m in re.finditer(r"^bundle_at (\d+) (\d+) (\d+)$", out, re.M)):
        model[at // per]["camera"] = dict(visits=v, tests=t)
    for k in range(DIAGNOSE_PIXELS):
        bad = mismatches(gpu[k], model[k])
        if bad:
            rays = np.concatenate([cams[k][~np.isnan(cams[k][:, 0])], dumps[k]])
            desc = ["kind %d o=%s d=%s" % (int(r[6]), _bits(r[:3]), _bits(r[3:6])) for r in rays]
            return "1x1 render at frame %d: %s; its rays: %s" % (cfg.first_frame + k, "; ".join(bad), "; ".join(desc))
    return None


# ------------------------------------------------------------------ checks
def check_render(oracle, sc, tris, nodes, cfg, hdr, tmp_path, pixel_major=True):
    """Counting render on the GPU == oracle render bit for bit, and its counts == the model's.  Returns (gpu counts, model counts)."""
    from tests.test_gpu_parity import assert_same_bits
    h, cache = hdr
    img, gpu, st, cyc = gpu_counts(sc, cfg)
    ref, rc, dump = oracle.render_rays(tris, nodes, cfg, hdr=h, hdr_cache=cache)
    assert_same_bits(img, ref, "counting render")
    c = sc.counters()
    assert (c.primary_rays, c.bounce_rays, c.shadow_rays) == (rc["rays_primary"], rc["rays_bounce"], rc["rays_shadow"])
    model = model_counts(tmp_path, tris, dump, camera_slot_rays(sc, cfg, pixel_major))
    bad = mismatches(gpu, model)
    if bad:
        where = first_differing_ray(oracle, sc, tris, nodes, cfg, hdr, tmp_path, pixel_major)
        pytest.fail("counts differ from the model: %s.  %s" % ("; ".join(bad), where or "No single-pixel render of %d differs." % DIAGNOSE_PIXELS))
    # warp steps: between one visit (test) per step and 32
    for p in ("k_extend_w8", "k_shadow_w8"):
        s = st[p]
        assert s["node_visits"] / 32 <= s["node_steps"] <= s["node_visits"], (p, s)
        assert s["triangle_tests"] / 32 <= s["triangle_steps"] <= s["triangle_tests"], (p, s)
    # the phase cycles are non-zero exactly when the pass ran
    ran = {"k_extend_w8": model["walked"]["bounce"]["rays"] > 0, "k_shadow_w8": model["walked"]["shadow"]["rays"] > 0}
    for p in ran:
        assert (sum(cyc[p].values()) > 0) == ran[p], (p, cyc[p], model["walked"])
    assert model["walked"]["bounce"]["rays"] > 0 and model["bundle"]["members"] > 0
    assert (model["walked"]["shadow"]["rays"] > 0) == (cfg.mode == api.MODE_DISNEY_IS_MIS_P5)
    return gpu, model


SCENES = ["bunny", "s1m", "stack0", "stack3", "twins", "floor"]
SIZES = {"s1m": dict(width=64, height=36), "stack0": dict(width=64, height=48), "stack3": dict(width=64, height=48)}


@pytest.mark.parametrize("name", SCENES)
@pytest.mark.parametrize("mode", [api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5])
def test_w8_counts_equal_the_model(oracle, small_hdr, tmp_path, monkeypatch, name, mode):
    tris, nodes, eye, cam, env = _cached_scene(name)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    sc = api.Scene(tris, nodes, *small_hdr)
    try:
        gpu, model = check_render(oracle, sc, tris, nodes, _cfg(eye, cam, mode=mode, **SIZES.get(name, {})), small_hdr, tmp_path)
        print("%s mode %d: GPU %s, model %s" % (name, mode, gpu, {k: model[k] for k in KINDS}))
    finally:
        sc.close()


@pytest.mark.parametrize("name", ["bunny", "stack3"])
def test_w8_camera_counts_in_frame_major_order(oracle, small_hdr, tmp_path, monkeypatch, name):
    """EZRT_CAMERA_ORDER=frame: a warp's bundle is an 8x4 pixel block of one frame."""
    tris, nodes, eye, cam, env = _cached_scene(name)
    for k, v in {**env, "EZRT_CAMERA_ORDER": "frame"}.items():
        monkeypatch.setenv(k, v)
    sc = api.Scene(tris, nodes, *small_hdr)
    try:
        check_render(oracle, sc, tris, nodes, _cfg(eye, cam, mode=api.MODE_DISNEY_IS_MIS_P5, **SIZES.get(name, {})), small_hdr, tmp_path, pixel_major=False)
    finally:
        sc.close()


# the schedule knobs at non-default values; EZRT_EXTEND_THREADS is read once per process, so these renders run in a child
SCHEDULE_ENV = {"EZRT_TRI_W": "3", "EZRT_REFILL_T": "7", "EZRT_CHUNK": "96", "EZRT_EXTEND_THREADS": "96"}


def _child_counts(name, mode):
    """(run in a child process) the counting render's exact totals as JSON on stdout"""
    from ezrt_b200 import api as a
    tris, nodes, eye, cam, env = _scene(name)
    hdr = scenes.synth_hdr(128, 64)
    sc = a.Scene(tris, nodes, hdr, a.hdr_cache(hdr))
    _, counts, _, _ = gpu_counts(sc, _cfg(eye, cam, mode=mode, **SIZES.get(name, {})))
    sc.close()
    print("COUNTS " + json.dumps(counts))


@pytest.mark.parametrize("name", ["bunny", "stack3"])
def test_w8_counts_do_not_depend_on_the_schedule(oracle, small_hdr, tmp_path, monkeypatch, name):
    """The bounce pass's totals and the shadow pass's node visits are the same under other triangle-step weights, refill
    thresholds, work chunks and block sizes -- and equal the model's."""
    tris, nodes, eye, cam, env = _cached_scene(name)
    mode = api.MODE_DISNEY_IS_MIS_P5
    envs = {**os.environ, **env, **SCHEDULE_ENV, "PYTHONPATH": ROOT}
    code = "from tests.test_gpu_w8_counts import _child_counts; _child_counts(%r, %d)" % (name, mode)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=envs, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:]
    other = json.loads(r.stdout.split("COUNTS ", 1)[1].splitlines()[0])
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    sc = api.Scene(tris, nodes, *small_hdr)
    try:
        gpu, model = check_render(oracle, sc, tris, nodes, _cfg(eye, cam, mode=mode, **SIZES.get(name, {})), small_hdr, tmp_path)
    finally:
        sc.close()
    assert other["bounce"] == gpu["bounce"], (other, gpu)
    assert other["shadow"]["visits"] == gpu["shadow"]["visits"]
    assert model["shadow"]["tests"] <= other["shadow"]["tests"] <= model["shadow"]["tests_max"]
    assert other["camera"] == gpu["camera"]   # one bundle per warp whatever the block size


def test_w8_counts_reset_and_accumulate(small_hdr, monkeypatch):
    """Repeating a counting render repeats its exact totals; accumulate=True over two renders gives their sum; a profile=0
    render after them reads all zeros; counting does not change the image."""
    tris, nodes, eye, cam, env = _cached_scene("bunny")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    sc = api.Scene(tris, nodes, *small_hdr)
    exact = lambda c: (c["bounce"], c["shadow"]["visits"], c["camera"])
    try:
        cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_IS_MIS_P5)
        plain = sc.render(cfg).copy()
        img, a, st_a, _ = gpu_counts(sc, cfg)
        assert img.tobytes() == plain.tobytes()
        _, a2, _, _ = gpu_counts(sc, cfg)
        assert exact(a2) == exact(a)
        later = _with(cfg, first_frame=cfg.spp)
        _, b, st_b, _ = gpu_counts(sc, later)
        assert exact(b) != exact(a)
        gpu_counts(sc, cfg)
        _, ab, st_ab, _ = gpu_counts(sc, _with(later, accumulate=True))
        for k in KINDS:
            want = a[k]["visits"] + b[k]["visits"]
            assert ab[k]["visits"] == want, (k, ab, a, b)
            if k != "shadow":
                assert ab[k]["tests"] == a[k]["tests"] + b[k]["tests"], (k, ab, a, b)
        for p in st_ab:
            assert st_ab[p]["node_visits"] == st_a[p]["node_visits"] + st_b[p]["node_visits"]
        assert sc.render(cfg).tobytes() == plain.tobytes()
        c = sc.counters()
        assert (c.node_visits, c.node_visits_96, c.tri_tests) == (0, 0, 0)
        assert all(v == 0 for p in sc.w8_step_counts().values() for v in p.values())
        assert all(v == 0 for p in sc.w8_phase_cycles().values() for v in p.values())
    finally:
        sc.close()
