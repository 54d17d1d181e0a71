"""Every kernel variant of the light sampling mode (mode 4) on the device, bit for bit against its restatement (tests/oracle_volumes).

The scene (tests/light_mode_space.space_scene) holds every option's data at once: an HDR map, textures with material and emission
maps, punctual lights, fog and a density grid over the glass blob and the floor, and volumes in the glass.  One triangle in eight of
the floor and the blob is duplicated bit for bit, so that the accel policy defers the rays that hit them (a tie) in the camera and the
bounce passes, and the deferred lane's LIST = true kernels shade rays in every render.

- Instantiation rows: each of the 560 mode-4 k_shade keys (A, family, option bools) gets one render on the accel policy with the
  deferred lane on (A = true: the feature-buffer render).  Each asserts the framebuffer's bits (and the feature buffer's and the
  squared luminance's for A = true) equal to the restatement's, equal primary, bounce and shadow ray counts, 0 < deferred rays < 65536,
  and that the k_shade and k_nee kernels torch.profiler sees launched are the ones light_mode_space.predict names.  The render-path
  factors (tree form, lens, bounces, batch, resumed frame, part, channels, map filter, camera order) are spread over the rows by a
  deterministic greedy all-pairs assignment, which also pairs each with every family and A.
- Path rows: the families against the traversal policies, the deferred lane on and off and the four entry points (render, device,
  feature buffers, adaptive), all pairs; and one render per family with more than 65536 deferred rays in its camera pass, which then
  traces them in line.
- Reductions: each option light_options switches off when the scene gives it nothing to do renders the bits and rays of the render
  without it, and the restatement's; P_env = 1 and P_p = 1 on the emitter-free scene."""
import contextlib
import functools
import os

import numpy as np
import pytest

from ezrt_b200 import api
from tests import light_mode_space as lms
from tests import oracle_volumes as ov

pytestmark = pytest.mark.gpu

# ------------------------------------------------------------------ the factors
# tree form: (environment at scene creation, scene with the far soup -- the 8-wide tree's flat triangle records)
FORMS = {"w4q16": ({"EZRT_ACCEL": "4"}, False), "w4exact": ({"EZRT_ACCEL": "4", "EZRT_ACCEL_Q16": "0"}, False),
         "w8idx": ({"EZRT_ACCEL": "8"}, False), "w8flat": ({"EZRT_ACCEL": "8"}, True)}
FACTORS = [("form", ["w4q16", "w4exact", "w8idx", "w8flat"]), ("lens", [False, True]), ("bounces", [0, 1, 3, 6]), ("batch", [0, 1, 3]),
           ("resume", [False, True]), ("part", ["whole", "1of3"]), ("channels", [3, 4]), ("map", ["linear", "nearest"]),
           ("order", ["pixel", "frame"])]
FIXED = ("family", "aov")   # the row's own, paired with every factor too
LENS = dict(lens_radius=0.12, focus_distance=3.6)
PARTS = {"whole": (0, 1), "1of3": (1, 3)}
SIDE_CAP = 65536            # device_scene.h EZRT_SIDE_CAP: more deferred rays in one pass are traced in line
TILE = 16
ADAPT = (0.3, 2, 2)


def _pairs(row):
    names = list(FIXED) + [n for n, _ in FACTORS]
    return {(a, row[a], b, row[b]) for i, a in enumerate(names) for b in names[i + 1:]}


def _all_pairs():
    dom = dict(FACTORS, family=list(lms.FAMILIES), aov=[False, True])
    names = list(FIXED) + [n for n, _ in FACTORS]
    return {(a, va, b, vb) for i, a in enumerate(names) for b in names[i + 1:] for va in dom[a] for vb in dom[b]}


def uncovered_pairs(rows):
    got = set()
    for r in rows:
        got |= _pairs(r)
    return _all_pairs() - got


def instantiation_rows():
    """one row per k_shade key: its flags, and path factors chosen greedily -- each factor in turn takes the value that covers the
    most pairs not yet covered with the values the row already has, ties going to the value used least so far, then the first.  Of the
    two rows of a flag set (A = false, true) at least one bounces, so that its k_nee runs."""
    todo = _all_pairs()
    used = {(n, v): 0 for n, dom in FACTORS for v in dom}
    rows, no_nee = [], set()
    for key in lms.row_keys():
        row = dict(key=key, flags=lms.flags_of(key), family=lms.family_of(key), aov=key[2])
        for n, dom in FACTORS:
            if n == "bounces" and row["flags"] in no_nee:   # the flags' other row (A) launched no k_nee: this one bounces
                dom = [v for v in dom if v > 0]
            def gain(v):
                return sum(((m, row[m], n, v) in todo) for m in row if m in FIXED or m in dict(FACTORS))
            best = max(dom, key=lambda v: (gain(v), -used[(n, v)], -dom.index(v)))
            row[n] = best
            used[(n, best)] += 1
        todo -= _pairs(row)
        if row["bounces"] == 0:
            no_nee.add(row["flags"])
        rows.append(row)
    return rows


ROWS = instantiation_rows()


SHORT = {"env_light": "env", "transmission": "trans", "medium": "med", "textures": "tex", "material_maps": "maps", "punctual_lights": "punct",
         "emission_maps": "emap", "light_tree": "tree", "medium_grid": "grid", "volumes": "vol"}


def _row_id(r):
    f = "+".join(sorted(SHORT[x] for x in r["flags"])) or "none"
    return "%s-%s-a%d-%s-lens%d-b%d-fpb%d-res%d-%s-c%d-%s-%s" % (r["family"], f, r["aov"], r["form"], r["lens"], r["bounces"], r["batch"],
                                                                r["resume"], r["part"], r["channels"], r["map"], r["order"])


# ------------------------------------------------------------------ scenes on the device
@contextlib.contextmanager
def _environ(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


_SCENES = {}


def device_scene(form="w4q16", order="pixel", lane=True, linear=True, emitters=True, env=True):
    """the space scene on the device with every option's data set, cached (the tree form, camera order and deferred lane are read from
    the environment when a scene is created)"""
    key = (form, order, lane, linear, emitters, env)
    if key not in _SCENES:
        fenv, soup = FORMS[form]
        sd = lms.space_scene(emitters=emitters, soup=soup)
        e = dict(fenv, EZRT_DEFERRED_LANE="1" if lane else "0", EZRT_CAMERA_ORDER=order)
        with _environ(e):
            sc = api.Scene(sd["tris"], sd["nodes"], sd["hdr"] if env else None, sd["hdr_cache"] if env else None, device=0,
                           hdr_filter_linear=linear)
        sc.set_textures(sd["textures"], sd["texcoords"], sd["texture_id"])
        sc.set_material_maps(sd["metal_rough_id"], sd["normal_id"])
        sc.set_emission_maps(sd["emission_id"])
        sc.set_punctual_lights(sd["lights"])
        sc.set_volumes(sd["volumes"], sd["volume_id"])
        sc.set_medium(**lms.medium_for(()))
        sc.set_medium_grid(sd["rho"])
        _SCENES[key] = (sc, sd)
    return _SCENES[key]


@pytest.fixture(scope="module", autouse=True)
def _close_scenes():
    yield
    for sc, _ in _SCENES.values():
        sc.close()
    _SCENES.clear()


# ------------------------------------------------------------------ launched kernels
@functools.lru_cache(maxsize=None)
def _profiler():
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    return torch, profile, ProfilerActivity


def launched(fn, attempts=6):
    """(fn's result, [names of the kernels launched while fn ran]), from torch.profiler's CUDA activity.  The capture is complete when
    it holds one kernel record per cudaLaunchKernel call it recorded.  Now and then a session delivers the launch calls but only some
    of the kernel records, or none: a few sessions in a run of this file on an H100, at different rows from run to run, in renders whose
    bits and ray counts matched the restatement, so their kernels ran.  Such a session is repeated, with fn called again (a render's
    kernels do not depend on its state); a capture that never completes fails."""
    torch, profile, act = _profiler()
    cuda = torch.autograd.DeviceType.CUDA
    for _ in range(attempts):
        with profile(activities=[act.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        ev = prof.events()
        names = [e.name for e in ev if e.device_type == cuda and not e.name.startswith(("Memcpy", "Memset"))]
        calls = sum(e.device_type != cuda and e.name.startswith("cudaLaunchKernel") for e in ev)
        if calls and len(names) == calls:
            return out, names
    raise AssertionError("torch.profiler recorded %d kernels for %d cudaLaunchKernel calls in each of %d sessions" % (len(names), calls, attempts))


def _assert_kernels(names, flags, state, aov, bounces, lane, what):
    want = lms.predict(flags, state, aov=aov, max_bounce=bounces, lane=lane)
    got = lms.kernel_keys(names)
    assert got == want, "%s: launched k_shade %s / k_nee %s, predicted %s / %s (%d kernel records: %s)" % (
        what, sorted(got[0] - want[0])[:3], sorted(got[1] - want[1])[:3], sorted(want[0] - got[0])[:3], sorted(want[1] - got[1])[:3], len(names),
        [n[:40] for n in names[:8]])


# ------------------------------------------------------------------ the restatement over the whole image or a part's tiles
def _part_windows(cfg):
    """the 16 x 16 tiles (x0, y0, x1, y1) the part owns, and its pixel mask [H, W]"""
    mask = np.zeros((cfg.height, cfg.width, 1), np.float32)
    n = api.partition_pixels(cfg.width, cfg.height, cfg.part_rank, cfg.part_count)
    api.partition_scatter_host(np.ones((n, 1), np.float32), mask, cfg.width, cfg.height, 1, cfg.part_rank, cfg.part_count)
    m = mask[..., 0] > 0
    wins = []
    for y0 in range(0, cfg.height, TILE):
        for x0 in range(0, cfg.width, TILE):
            x1, y1 = min(x0 + TILE, cfg.width), min(y0 + TILE, cfg.height)
            if m[y0:y1, x0:x1].any():
                assert m[y0:y1, x0:x1].all()
                wins.append((x0, y0, x1, y1))
    return wins, m


def _oracle(sd, flags, cfg, aov=False, **okw):
    """(image, luma2, aov or None, (primary, bounce, shadow) rays) of the restatement over the image, or over the tiles of cfg's part
    (zeros elsewhere)"""
    full = api.RenderConfig(**{**cfg.__dict__, "part_rank": 0, "part_count": 1})
    kw = lms.oracle_kwargs(sd, flags, **okw)
    if cfg.part_count == 1:
        img, luma2, feat, c = ov.render(sd["tris"], sd["nodes"], full, aov=aov, **kw)
        return img, luma2, feat, np.array([c["rays_primary"], c["rays_bounce"], c["rays_shadow"]], np.int64)
    img = np.zeros((cfg.height, cfg.width, cfg.out_channels), np.float32)
    luma2 = np.zeros((cfg.height, cfg.width), np.float32)
    feat = np.zeros((cfg.height, cfg.width, 8), np.float32) if aov else None
    rays = np.zeros(3, np.int64)
    for x0, y0, x1, y1 in _part_windows(cfg)[0]:
        i, l2, f, c = ov.render(sd["tris"], sd["nodes"], full, aov=aov, window=(x0, y0, x1, y1), **kw)
        img[y0:y1, x0:x1], luma2[y0:y1, x0:x1] = i, l2
        if aov:
            feat[y0:y1, x0:x1] = f
        rays += np.array([c["rays_primary"], c["rays_bounce"], c["rays_shadow"]], np.int64)
    return img, luma2, feat, rays


def _scatter(cfg, a, ch):
    if cfg.part_count == 1:
        return a.reshape(cfg.height, cfg.width, ch) if ch > 1 else a.reshape(cfg.height, cfg.width)
    out = np.zeros((cfg.height, cfg.width, ch), np.float32)
    api.partition_scatter_host(np.ascontiguousarray(a.reshape(-1, ch)), out, cfg.width, cfg.height, ch, cfg.part_rank, cfg.part_count)
    return out if ch > 1 else out[..., 0]


def _rays(c):
    return np.array([c.primary_rays, c.bounce_rays, c.shadow_rays], np.int64)


def _device_render(sc, cfg, entry, prev=None):
    """(image, aov or None, luma2 or None) of one render through an entry point: render, device (a torch tensor), aov; prev: the
    arrays a resumed render continues"""
    if entry == "render":
        return sc.render(cfg, framebuffer=None if prev is None else prev[0]), None, None
    if entry == "device":
        import torch
        n = api.partition_pixels(cfg.width, cfg.height, cfg.part_rank, cfg.part_count)
        fb = torch.zeros(n * cfg.out_channels, dtype=torch.float32, device="cuda") if prev is None else \
            torch.from_numpy(np.ascontiguousarray(prev[0]).reshape(-1)).cuda()
        sc.render_device(cfg, fb)
        torch.cuda.synchronize()
        img = fb.cpu().numpy()
        return (img.reshape(cfg.height, cfg.width, cfg.out_channels) if cfg.part_count == 1 else img.reshape(n, cfg.out_channels)), None, None
    assert entry == "aov"
    if prev is None:
        return sc.render_aov(cfg)
    return sc.render_aov(cfg, framebuffer=prev[0], aov=prev[1], luma2=prev[2])


def check_render(row_flags, cfg, entry, form="w4q16", order="pixel", lane=True, linear=True, resume=False, policy_lane=None, what=""):
    """one render against the restatement: bits (feature buffer and squared luminance too for aov), ray counts, deferred rays on the
    accel policy with the lane, and the launched kernels.  Returns the device's counters."""
    sc, sd = device_scene(form, order, lane, linear)
    flags = frozenset(row_flags)
    sc.set_medium(**lms.medium_for(flags))
    aov = entry == "aov"
    first = 2 if resume else 0
    okw = dict(hdr_linear=linear)
    prev = None
    if first:
        c0 = api.RenderConfig(**{**cfg.__dict__, "spp": first, "first_frame": 0, "frames_per_batch": 0})
        prev = _device_render(sc, c0, entry)
        cfg = api.RenderConfig(**{**cfg.__dict__, "first_frame": first})

    def run():   # a resumed render continues copies of the first frames' arrays, so that a repeated session starts from the same state
        return _device_render(sc, cfg, entry, None if prev is None else tuple(None if a is None else np.array(a, copy=True) for a in prev))
    (img, feat, luma2), names = launched(run)
    gc = sc.counters()
    full = api.RenderConfig(**{**cfg.__dict__, "spp": cfg.spp + first, "first_frame": 0})
    rimg, rluma2, rfeat, rrays = _oracle(sd, flags, full, aov=aov, **okw)
    if first:
        rrays = rrays - _oracle(sd, flags, api.RenderConfig(**{**cfg.__dict__, "spp": first, "first_frame": 0}), **okw)[3]
    m = _part_windows(cfg)[1]
    got = _scatter(cfg, img, cfg.out_channels)
    assert m.any() and got[m].tobytes() == rimg[m].tobytes(), "%s: image differs, L-inf %.3g" % (what, float(np.nanmax(np.abs(got[m] - rimg[m]))))
    if aov:
        assert _scatter(cfg, feat, 8)[m].tobytes() == rfeat[m].tobytes(), "%s: feature buffer differs" % what
        assert _scatter(cfg, luma2, 1)[m].tobytes() == rluma2[m].tobytes(), "%s: squared luminance differs" % what
    assert np.array_equal(_rays(gc), rrays), "%s: rays %s, restatement %s" % (what, _rays(gc), rrays)
    on_lane = lane if policy_lane is None else policy_lane
    if on_lane:
        assert 0 < gc.deferred_rays < SIDE_CAP, "%s: %d deferred rays" % (what, gc.deferred_rays)
    _assert_kernels(names, flags, lms.FULL, aov, cfg.max_bounce, on_lane and cfg.traverse == api.TRAVERSE_ACCEL, what)
    return gc


def test_profiler_sees_the_library_kernels():
    sc, sd = device_scene()
    _, names = launched(lambda: sc.render(lms.config(sd, ())))
    assert any("k_shade<" in n for n in names) and any("k_nee<" in n for n in names), names[:10]


@pytest.mark.parametrize("row", ROWS, ids=[_row_id(r) for r in ROWS])
def test_instantiation_row(row):
    rank, count = PARTS[row["part"]]
    kw = dict(max_bounce=row["bounces"], spp=4 if row["batch"] == 3 else 2, frames_per_batch=row["batch"], out_channels=row["channels"],
              part_rank=rank, part_count=count)
    if row["lens"]:
        kw.update(LENS)
    sd = lms.space_scene(soup=FORMS[row["form"]][1])
    cfg = lms.config(sd, row["flags"], **kw)
    check_render(row["flags"], cfg, "aov" if row["aov"] else "render", form=row["form"], order=row["order"], linear=row["map"] == "linear",
                 resume=row["resume"], what=_row_id(row))


# ------------------------------------------------------------------ path rows
POLICIES = {"accel": api.TRAVERSE_ACCEL, "pruned": api.TRAVERSE_PRUNED, "reference": api.TRAVERSE_REFERENCE}
PATH_FACTORS = [("family", list(lms.FAMILIES)), ("policy", list(POLICIES)), ("lane", [True, False]), ("entry", ["render", "device", "aov", "adaptive"])]


def path_rows():
    """all pairs of (family, policy, lane, entry), greedily; each row renders the family's keys in turn (the richest first)"""
    names = [n for n, _ in PATH_FACTORS]
    dom = dict(PATH_FACTORS)
    todo = {(a, va, b, vb) for i, a in enumerate(names) for b in names[i + 1:] for va in dom[a] for vb in dom[b]}
    by_fam = {f: sorted({lms.flags_of(k) for k in lms.row_keys() if lms.family_of(k) == f}, key=lambda s: (-len(s), sorted(s)))
              for f in lms.FAMILIES}
    rows, n_fam = [], {f: 0 for f in lms.FAMILIES}
    while todo:
        a, va, b, vb = min(todo, key=lambda p: (names.index(p[0]), dom[p[0]].index(p[1]), names.index(p[2]), dom[p[2]].index(p[3])))
        row = {a: va, b: vb}
        for n in names:
            if n not in row:
                row[n] = max(dom[n], key=lambda v: (sum(((m, row[m], n, v) in todo) or ((n, v, m, row[m]) in todo) for m in row), -dom[n].index(v)))
        todo -= {(x, row[x], y, row[y]) for i, x in enumerate(names) for y in names[i + 1:]}
        f = row["family"]
        row["flags"] = by_fam[f][(7 * n_fam[f]) % len(by_fam[f])]
        n_fam[f] += 1
        rows.append(row)
    return rows


PATH_ROWS = path_rows()


@pytest.mark.parametrize("row", PATH_ROWS, ids=["%s-%s-lane%d-%s" % (r["family"], r["policy"], r["lane"], r["entry"]) for r in PATH_ROWS])
def test_path_row(row):
    what = "path row %r" % (row,)
    sd = lms.space_scene()
    pol = POLICIES[row["policy"]]
    if row["entry"] != "adaptive":
        cfg = lms.config(sd, row["flags"], traverse=pol)
        check_render(row["flags"], cfg, row["entry"], lane=row["lane"], policy_lane=row["lane"] and pol == api.TRAVERSE_ACCEL, what=what)
        return
    sc, _ = device_scene(lane=row["lane"])
    flags = row["flags"]
    sc.set_medium(**lms.medium_for(flags))
    cfg = lms.config(sd, flags, traverse=pol, spp=6)
    (img, spp, luma2), names = launched(lambda: sc.render_adaptive(cfg, *ADAPT))
    gc = sc.counters()
    rimg, rspp, rluma2, rc = ov.render_adaptive(sd["tris"], sd["nodes"], cfg, *ADAPT, **lms.oracle_kwargs(sd, flags))
    assert img.tobytes() == rimg.tobytes() and luma2.tobytes() == rluma2.tobytes() and np.array_equal(spp, rspp), what
    assert np.array_equal(_rays(gc), [rc["rays_primary"], rc["rays_bounce"], rc["rays_shadow"]]), what
    lane = row["lane"] and pol == api.TRAVERSE_ACCEL
    if lane:
        assert 0 < gc.deferred_rays < SIDE_CAP, what
    _assert_kernels(names, flags, lms.FULL, False, cfg.max_bounce, lane, what)


@pytest.mark.parametrize("family", lms.FAMILIES)
def test_more_deferred_rays_than_the_lane_takes(family):
    """a camera pass with more than EZRT_SIDE_CAP deferred rays traces them in line: 512 x 512 at 64 spp, no bounce (about 0.6 % of the
    camera rays hit a duplicated triangle); three windows against the restatement"""
    sc, sd = device_scene()
    flags = max((lms.flags_of(k) for k in lms.row_keys() if lms.family_of(k) == family), key=lambda s: (len(s), sorted(s)))
    sc.set_medium(**lms.medium_for(flags))
    cfg = lms.config(sd, flags, width=512, height=512, spp=64, max_bounce=0)
    img, names = launched(lambda: sc.render(cfg))
    gc = sc.counters()
    assert gc.deferred_rays > SIDE_CAP, gc.deferred_rays
    _assert_kernels(names, flags, lms.FULL, False, 0, True, family)
    for win in ((0, 0, 16, 16), (248, 240, 264, 256), (496, 496, 512, 512)):
        ref = ov.render(sd["tris"], sd["nodes"], cfg, window=win, **lms.oracle_kwargs(sd, flags))[0]
        x0, y0, x1, y1 = win
        assert img[y0:y1, x0:x1].tobytes() == ref.tobytes(), (family, win)


# ------------------------------------------------------------------ reductions on the device
RED_BASES = [frozenset(), frozenset({"light_tree", "textures", "emission_maps"}), frozenset({"transmission", "punctual_lights", "env_light"}),
             frozenset({"textures", "material_maps"})]


def _reduction_cases():
    out = []
    for i, base in enumerate(RED_BASES):
        out.append(("env_light", base))
        out.append(("medium", base))
        out.append(("medium_grid", base))
        out.append(("punctual_lights", base))
        out.append(("light_tree", base))
        out.append(("volumes", base))
    return out


@pytest.mark.parametrize("flag,base", _reduction_cases(), ids=["%s-%s" % (f, "+".join(sorted(b)) or "none") for f, b in _reduction_cases()])
def test_reduction_on_the_device(flag, base):
    """the degenerate option renders the bits and rays of the render without it, and the restatement's; its kernels are those of the
    render without it"""
    env = flag != "env_light"
    emitters = flag != "light_tree"
    sc, sd = device_scene(emitters=emitters, env=env)
    med = dict(lms.medium_for(()))
    okw = dict(env=env)
    state = lms.SceneState(env_table=env, K=1 if emitters else 0)
    if flag in ("medium", "medium_grid"):
        on = base | {"medium"} | ({"medium_grid"} if flag == "medium_grid" else set())
        on = on | ({"volumes"} if "transmission" in on else set())
        off = on - {"medium", "medium_grid"}
        med["sigma_t"] = 0.0
        state = lms.SceneState(sigma_t=False)
    elif flag == "volumes":
        on = base | {"transmission", "volumes"}
        off = on - {"volumes"}
        state = lms.SceneState(volumes=False)
    else:
        on = base | {flag}
        off = on - {flag}
        if flag == "punctual_lights":
            state = lms.SceneState(J=0)
    on, off = frozenset(on), frozenset(off)
    assert lms.valid(on) and lms.valid(off)
    assert lms.predict(on, state) == lms.predict(off, state)
    try:
        sc.set_medium(**med)
        if flag == "punctual_lights":
            sc.set_punctual_lights([])
        if flag == "volumes":
            sc.set_volumes(None)
        out = []
        for fl in (on, off):
            cfg = lms.config(sd, fl)
            img, names = launched(lambda: sc.render(cfg))
            out.append((img.tobytes(), tuple(_rays(sc.counters()))))
            _assert_kernels(names, off, state, False, cfg.max_bounce, True, "%s on %s" % (flag, sorted(base)))
        assert out[0] == out[1], (flag, sorted(base))
        kw = lms.oracle_kwargs(sd, off, **okw)
        ref, _, _, c = ov.render(sd["tris"], sd["nodes"], lms.config(sd, off), **kw)
        assert out[1][0] == ref.tobytes() and out[1][1] == (c["rays_primary"], c["rays_bounce"], c["rays_shadow"]), (flag, sorted(base))
    finally:
        sc.set_medium(**lms.medium_for(()))
        sc.set_punctual_lights(sd["lights"])
        sc.set_volumes(sd["volumes"], sd["volume_id"])


@pytest.mark.parametrize("flags", [frozenset({"env_light"}), frozenset({"punctual_lights"}), frozenset({"env_light", "punctual_lights", "light_tree"}),
                                   frozenset({"punctual_lights", "transmission", "volumes", "medium", "medium_grid"})],
                         ids=["p_env1", "p_p1", "p_env1_p_p_half_tree_off", "p_p1_vol_grid"])
def test_emitter_free_scene(flags):
    """K = 0: the map alone is the light (P_env = 1), the punctual lights alone (P_p = 1), and the light tree switched off"""
    sd = lms.space_scene(emitters=False)
    cfg = lms.config(sd, flags)
    sc, _ = device_scene(emitters=False)
    sc.set_medium(**lms.medium_for(flags))
    img, names = launched(lambda: sc.render(cfg))
    gc = sc.counters()
    ref, _, _, c = ov.render(sd["tris"], sd["nodes"], cfg, **lms.oracle_kwargs(sd, flags))
    assert img.tobytes() == ref.tobytes() and np.array_equal(_rays(gc), [c["rays_primary"], c["rays_bounce"], c["rays_shadow"]])
    state = lms.SceneState(K=0)
    o = lms.light_options(flags, state)
    assert o["p_env"] in (None, 1.0) and (o["p_p"] is None or o["p_p"] == (0.5 if o["env"] else 1.0))
    _assert_kernels(names, flags, state, False, cfg.max_bounce, True, "emitter-free %s" % sorted(flags))
