"""Render options and combinations that the rest of the GPU suite never reaches, each checked bit for bit, ray counts included,
against the CPU restatement that covers it: oracle.render (modes 0-3), tests/oracle_lights (mode 4, and luma2 in every mode),
tests/oracle_aov (first-hit features) and tests/oracle_adaptive (adaptive renders).

Targeted cases, one per path no other test runs on the GPU: the W8 camera pass in frame order and the W8 bounce pass over
sorted rays; k_shade's per-path Sobol pairs in batches of more than 256 frames; Sobol dimensions 8 and up; the uint32 frame
counter's wrap; parts that own no pixel; mode 4 beside the feature-buffer and adaptive renders, a nearest-filtered map and
no bounce; every tuning knob read from the environment at a non-default value.  Then a pairwise covering array over the
options that combine (scene form, mode, policy, pipeline, entry point, batch size, first frame, bounces, channels,
partition, map, camera order, deferred lane): 40 rows.  30 of them compare finite pixels and cover all 726 pairs of values
that such a row can hold; 10 rows render an empty part or across the frame counter's wrap (no pixel, or all NaN) and count
only for the 74 pairs that contain those values.  Every row also checks, with a counting render, which tree the accel
kernels walked."""
import functools
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_adaptive as oa
from tests import oracle_aov as ov
from tests import oracle_binding as ob
from tests import oracle_lights as ol
from tests.test_gpu_parity import assert_same_bits
from tests.test_gpu_w8 import W8_MIN_TRIANGLES, _assert_w8_ran, far_scene, soup_scene

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENV = (0.35, 0.45, 0.6)
L4 = api.MODE_DISNEY_LIGHTS
WAVE, MEGA = api.PIPELINE_WAVEFRONT, api.PIPELINE_MEGAKERNEL
WRAP = 2 ** 32 - 3          # a first_frame three frames before the uint32 frame counter wraps
SOBOL_TABLE = 256           # kernels.cu EZRT_SOBOL_TABLE: k_shade computes the Sobol pair per path in larger batches
BATCH_SLOTS = 32 << 20      # capi.cu: an automatic batch holds about this many sample slots (then capped by spp)
TILE = 16
ADAPT = (0.5, 2, 2)         # threshold, min_spp, check_interval of every adaptive render here


# ------------------------------------------------------------------ scenes
def room_scene():
    """A closed room: an 81,920-triangle blob (the W8 tree; a mesh, so its triangle records are indexed) and a small emissive
    sphere inside a box, the camera inside too.  Every bounce ray hits a wall, so paths live until max_bounce."""
    tl = api.TriangleList()
    tl.read_obj_text(scenes.blob_obj(6), scenes.MATERIAL_PRESETS[4], api.transform_matrix((0, 0, 0), (0, -0.4, 0), (1.2, 1.2, 1.2)), True)
    tl.read_obj_text(scenes.sphere_obj(), api.Material(emissive=(15, 12, 9)), api.transform_matrix((0, 0, 0), (1.1, 1.4, -0.9), (0.4, 0.4, 0.4)), False)
    tl.read_obj_text(scenes.box_obj(), api.Material(baseColor=(0.7, 0.65, 0.6), roughness=0.6), api.transform_matrix((0, 0, 0), (0, 0, 0), (6, 6, 6)), False)
    tris, nodes = tl.build_bvh(8)
    eye, cam = api.camera_orbit(25.0, 15.0, 2.6)
    return tris, nodes, eye, cam


GEOMETRY = {"grid": lambda: scenes.s_grid(3, 2, 2),   # 31,052 triangles with four emissive spheres: the 4-wide tree by size
            "far": lambda: far_scene(3.0, 6),         # 163,840 triangles, no emitter: the W8 tree, indexed records
            "soup": soup_scene,                       # 70,000 triangles, a third of them emissive: the W8 tree, flat records
            "room": room_scene}
AXIS_RADIUS = {"far": 4.0, "soup": 6.0, "room": 2.6}


@functools.lru_cache(maxsize=None)
def _geometry(name):
    return GEOMETRY[name]()


@functools.lru_cache(maxsize=None)
def _hdr():
    h = scenes.synth_hdr(128, 64)
    return h, api.hdr_cache(h)


def _indexed(tris):
    """capi.cu's rule for the W8 triangle records: indexed when 32 B per triangle + 16 B per distinct vertex beat 64 B per triangle."""
    n_vert = len(np.unique(np.ascontiguousarray(tris[:, :9]).view(np.uint32).reshape(-1, 3), axis=0))
    return 32 * len(tris) + 16 * n_vert < 64 * len(tris)


class Sd:
    """A scene's arrays and the map it is rendered with (map "none" | "linear" | "nearest"), for the GPU and the restatements alike."""

    def __init__(self, name, env="linear"):
        self.name, self.env = name, env
        self.tris, self.nodes, self.eye, self.cam = _geometry(name)
        self.hdr, self.cache = (None, None) if env == "none" else _hdr()
        self.linear = env != "nearest"

    def scene(self):
        return api.Scene(self.tris, self.nodes, self.hdr, self.cache, hdr_filter_linear=self.linear)

    def kw(self):
        return dict(hdr=self.hdr, hdr_cache=self.cache, hdr_linear=self.linear)

    def cfg(self, eye=None, cam=None, **kw):
        base = dict(width=64, height=48, spp=3, max_bounce=2, eye=tuple(self.eye if eye is None else eye),
                    camera_rotate=tuple(self.cam if cam is None else cam), env_color=ENV)
        base.update(kw)
        return api.RenderConfig(**base)


def _with(cfg, **kw):
    return api.RenderConfig(**{**cfg.__dict__, **kw})


# ------------------------------------------------------------------ one render against its restatement
def _rays(rc):
    return np.array([rc["rays_primary"], rc["rays_bounce"], rc["rays_shadow"]], np.int64)


def _adaptive_lights(sd, cfg, win):
    """Mode 4's adaptive render restated: each tile of the window stops at the first test (min_spp, then every check_interval
    frames, below the cap) at which oracle_render_lights' state at that frame count passes the float32 criterion of
    tests/oracle_adaptive.py, and is then that plain render."""
    thr, min_spp, interval = ADAPT
    x0, y0, x1, y1 = win
    out = dict(image=np.zeros((y1 - y0, x1 - x0, cfg.out_channels), np.float32), spp=np.zeros((y1 - y0, x1 - x0), np.int32),
               luma2=np.zeros((y1 - y0, x1 - x0), np.float32))
    rays = np.zeros(3, np.int64)
    for ty in range(y0, y1, TILE):
        for tx in range(x0, x1, TILE):
            t = (tx, ty, min(tx + TILE, x1), min(ty + TILE, y1))
            n = min_spp
            while n < cfg.spp:
                img, m2, _ = ol.oracle_render_lights(sd.tris, sd.nodes, _with(cfg, spp=n), window=t, **sd.kw())
                if oa.tile_converged(oa.adaptive_error(m2, img, n), thr).all():
                    break
                n += interval
            n = min(n, cfg.spp)
            img, m2, rc = ol.oracle_render_lights(sd.tris, sd.nodes, _with(cfg, spp=n), window=t, **sd.kw())
            sl = (slice(t[1] - y0, t[3] - y0), slice(t[0] - x0, t[2] - x0))
            out["image"][sl], out["spp"][sl], out["luma2"][sl] = img, n, m2
            rays += _rays(rc)
    return out, rays


def _restate_window(sd, cfg, entry, win):
    """{output: [h, w, ...]} and (primary, bounce, shadow) rays of the restatement of one window."""
    kw = sd.kw()
    if entry == "adaptive":
        if cfg.mode == L4:
            return _adaptive_lights(sd, cfg, win)
        img, spp, m2, rc = oa.render_adaptive(sd.tris, sd.nodes, cfg, *ADAPT, window=win, **kw)
        return dict(image=img, spp=spp, luma2=m2), _rays(rc)
    if entry == "aov":
        if cfg.mode == L4:
            img, m2, rc = ol.oracle_render_lights(sd.tris, sd.nodes, cfg, window=win, **kw)
            # The features are running means over the camera ray's first hit.  shadePixel draws that ray (seed, jitter,
            # direction) the same way in every mode and firstHit of tests/oracle_aov.cpp restates it, so mode 2's
            # restatement gives mode 4's features.
            feat = ov.render_aov(sd.tris, sd.nodes, _with(cfg, mode=api.MODE_DISNEY_SOBOL_P5), window=win, **kw)[1]
            return dict(image=img, aov=feat, luma2=m2), _rays(rc)
        img, feat, m2, rc = ov.render_aov(sd.tris, sd.nodes, cfg, window=win, **kw)
        return dict(image=img, aov=feat, luma2=m2), _rays(rc)
    if cfg.mode == L4:
        img, _, rc = ol.oracle_render_lights(sd.tris, sd.nodes, cfg, window=win, **kw)
    else:
        img, rc = ob.render(sd.tris, sd.nodes, cfg, window=win, **kw)
    return dict(image=img), _rays(rc)


def _part_tiles(cfg):
    """(pixel mask of the part, its 16x16 tile windows; the whole image for one part)."""
    W, H = cfg.width, cfg.height
    if cfg.part_count == 1:
        return np.ones((H, W), bool), [(0, 0, W, H)]
    n = api.partition_pixels(W, H, cfg.part_rank, cfg.part_count)
    full = np.zeros((H, W, 1), np.float32)
    if n:
        api.partition_scatter_host(np.ones((n, 1), np.float32), full, W, H, 1, cfg.part_rank, cfg.part_count)
    mask = full[..., 0] > 0
    wins = [(x, y, min(x + TILE, W), min(y + TILE, H)) for y in range(0, H, TILE) for x in range(0, W, TILE) if mask[y, x]]
    return mask, wins


def _restate(sd, cfg, entry):
    """The restatement of a render in whole-image layout: {output: [H, W, k]} and its rays."""
    W, H = cfg.width, cfg.height
    _, wins = _part_tiles(cfg)
    full, rays = {}, np.zeros(3, np.int64)
    for win in wins:
        x0, y0, x1, y1 = win
        got, r = _restate_window(sd, cfg, entry, win)
        for k, a in got.items():
            a = a.reshape(y1 - y0, x1 - x0, -1)
            full.setdefault(k, np.zeros((H, W, a.shape[2]), a.dtype))[y0:y1, x0:x1] = a
        rays += r
    return full, tuple(int(x) for x in rays)


def _run(sc, cfg, entry, stream=None):
    """One GPU render through `entry` ("render", "device" on a non-default stream, "aov", "adaptive"): {output: compact [n, k]}."""
    n = api.partition_pixels(cfg.width, cfg.height, cfg.part_rank, cfg.part_count)
    ch = cfg.out_channels
    if entry == "render":
        return dict(image=sc.render(cfg).reshape(n, ch))
    if entry == "device":
        import torch
        d_fb = torch.zeros(max(n, 1) * ch, dtype=torch.float32, device="cuda")
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        sc.render_device(cfg, d_fb, st)
        st.synchronize()
        return dict(image=d_fb[:n * ch].cpu().numpy().reshape(n, ch))
    if entry == "aov":
        img, feat, m2 = sc.render_aov(cfg)
        return dict(image=img.reshape(n, ch), aov=feat.reshape(n, 8), luma2=m2.reshape(n, 1))
    img, spp, m2 = sc.render_adaptive(cfg, *ADAPT)
    return dict(image=img.reshape(n, ch), spp=spp.reshape(n, 1), luma2=m2.reshape(n, 1))


def _scatter(a, cfg):
    """A part's compact [n, k] output in whole-image layout [H, W, k] (zeros elsewhere)."""
    W, H = cfg.width, cfg.height
    k = a.shape[1]
    if cfg.part_count == 1:
        return a.reshape(H, W, k)
    ints = a.dtype == np.int32
    full = np.zeros((H, W, k), np.float32)
    if a.size:
        api.partition_scatter_host(np.ascontiguousarray(a.view(np.float32) if ints else a), full, W, H, k, cfg.part_rank, cfg.part_count)
    return full.view(np.int32) if ints else full


def _check(sd, sc, cfg, entry, what, ref=None):
    """Render through `entry` and compare every output and the ray counts with the restatement (or with `ref`, a
    restatement of the same render computed before).  Returns ({output: [H, W, k] GPU}, ref)."""
    got = _run(sc, cfg, entry)
    c = sc.counters()
    if ref is None:
        ref = _restate(sd, cfg, entry)
    want, rays = ref
    mask, _ = _part_tiles(cfg)
    full = {}
    for k, a in got.items():
        full[k] = _scatter(a, cfg)
        if not mask.any():
            assert a.size == 0, "%s: %s of a part without pixels" % (what, k)
        elif k == "spp":
            np.testing.assert_array_equal(full[k][mask], want[k][mask], "%s: spp map" % what)
        else:
            assert_same_bits(full[k][mask], want[k][mask], "%s: %s" % (what, k))
    assert (c.primary_rays, c.bounce_rays, c.shadow_rays) == rays, "%s: ray counts %r vs %r" % (
        what, (c.primary_rays, c.bounce_rays, c.shadow_rays), rays)
    return full, ref


def _classify(node_visits, node_visits_96):
    """The tree form a counting render (profile = 2, accel policy, at least one bounce) walked, from its node visits: the W8
    kernels count only quantised records; the 4-wide camera pass reads exact records and, with the 16-bit planes, the
    incoherent passes read quantised ones; a scene without an accel tree (have_accel = false) counts none."""
    if node_visits == 0:
        return "none"
    if node_visits_96 == node_visits:
        return "W8"
    return "4-wide Q16" if node_visits_96 else "4-wide exact"


def _tree_form(sc, cfg):
    sc.render(_with(cfg, profile=2, spp=1, first_frame=0, frames_per_batch=0, part_rank=0, part_count=1, max_bounce=max(1, cfg.max_bounce),
                    traverse=api.TRAVERSE_ACCEL, pipeline=WAVE))
    c = sc.counters()
    return _classify(c.node_visits, c.node_visits_96)


# ------------------------------------------------------------------ the W8 camera pass in frame order, the W8 pass over sorted rays
@pytest.mark.parametrize("form", ["far", "soup", "room"])
@pytest.mark.parametrize("knob", [("EZRT_CAMERA_ORDER", "frame"), ("EZRT_SORT_RAYS", "1")])
def test_w8_in_frame_order_and_over_sorted_rays(monkeypatch, form, knob):
    """EZRT_CAMERA_ORDER=frame: a warp of k_extend_w8_camera takes an 8 x 4 pixel block of one frame, where the bundles' sub-bundle
    rule really splits (and, with the axis camera, where a component of d changes sign inside a bundle).  EZRT_SORT_RAYS=1:
    k_extend_w8 reads its rays through the sort's permutation.  Indexed (far, room) and flat (soup) triangle records."""
    sd = Sd(form)
    assert len(sd.tris) >= W8_MIN_TRIANGLES and _indexed(sd.tris) == (form != "soup")
    monkeypatch.setenv(*knob)
    sc = sd.scene()
    try:
        for view, (eye, cam) in (("orbit", (sd.eye, sd.cam)), ("axis", api.camera_orbit(0.0, 0.0, AXIS_RADIUS[form]))):
            for mode in (api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5, L4):
                cfg = sd.cfg(eye, cam, spp=4, mode=mode)
                _check(sd, sc, cfg, "render", "%s %s, %s camera, mode %d" % (form, knob[0], view, mode))
            _assert_w8_ran(sc, cfg, 0.25)
        assert _tree_form(sc, cfg) == "W8"
    finally:
        sc.close()


# ------------------------------------------------------------------ more frames per batch than k_shade's Sobol table holds
@pytest.mark.parametrize("mode", [api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5, L4])
def test_batches_of_more_than_256_frames(mode):
    sd = Sd("grid")
    cfg = sd.cfg(width=16, height=16, spp=300, mode=mode)
    per_frame = TILE * TILE                                    # one tile
    assert min(max(1, BATCH_SLOTS // per_frame), cfg.spp) == 300 > SOBOL_TABLE   # the automatic batch: all 300 frames at once
    sc = sd.scene()
    try:
        for _ in range(2):   # the first render of mode 4 also builds the light table
            sc.render(_with(cfg, spp=1))
        per_batch = sc.counters().kernel_launches   # every batch makes the same launches, and a render is nothing but batches
        ref, launches = None, {}
        for fpb in (0, 300, 17):
            _, ref = _check(sd, sc, _with(cfg, frames_per_batch=fpb), "render", "mode %d, 300 frames, frames_per_batch %d" % (mode, fpb), ref)
            launches[fpb] = sc.counters().kernel_launches
        # the device really ran the 300 frames as one batch (and as 18 batches of at most 17)
        assert launches == {0: per_batch, 300: per_batch, 17: 18 * per_batch}, (per_batch, launches)
    finally:
        sc.close()


# ------------------------------------------------------------------ Sobol dimensions 8 and up
@pytest.fixture(scope="module")
def room():
    sd = Sd("room")
    sc = sd.scene()
    yield sd, sc
    sc.close()


@pytest.mark.parametrize("bounces", [5, 7])
@pytest.mark.parametrize("mode,pipeline", [(api.MODE_DISNEY_SOBOL_P5, WAVE), (api.MODE_DISNEY_IS_MIS_P5, WAVE), (L4, WAVE),
                                           (api.MODE_DISNEY_SOBOL_P5, MEGA), (api.MODE_DISNEY_IS_MIS_P5, MEGA)])
def test_sobol_dimensions_past_eight(room, bounces, mode, pipeline):
    """Bounce b draws Sobol dimensions 2b and 2b + 1; from bounce 4 on they are 8 and up, where the device masks the table
    offset and the oracle the index.  In the closed room nearly every path reaches them."""
    sd, sc = room
    cfg = sd.cfg(width=48, height=32, spp=2, max_bounce=bounces, mode=mode, pipeline=pipeline)
    _check(sd, sc, cfg, "render", "room, mode %d, pipeline %d, %d bounces" % (mode, pipeline, bounces))
    assert sc.counters().bounce_rays > 0.5 * 48 * 32 * 2 * bounces


# ------------------------------------------------------------------ the frame counter's wrap
@pytest.mark.parametrize("entry,mode,pipeline", [("render", api.MODE_DISNEY_SOBOL_P5, WAVE), ("render", L4, WAVE), ("aov", api.MODE_DISNEY_SOBOL_P5, WAVE),
                                                 ("aov", L4, WAVE), ("render", api.MODE_DISNEY_SOBOL_P5, MEGA)])
def test_frame_counter_wrap(entry, mode, pipeline):
    """first_frame = 2^32 - 3: frames 0xFFFFFFFD, 0xFFFFFFFE, then 0xFFFFFFFF, whose blend weight is 1/float(0u) = +inf, then
    frame 0 (the reference's uint arithmetic, include/ezrt.h).  Two frames stay finite; from the third on every blended
    value is NaN, and alpha stays 1."""
    sd = Sd("grid")
    sc = sd.scene()
    try:
        for spp in (2, 4):
            for fpb in (0, 1):
                cfg = sd.cfg(width=40, height=24, spp=spp, first_frame=WRAP, frames_per_batch=fpb, out_channels=4, mode=mode, pipeline=pipeline)
                got, _ = _check(sd, sc, cfg, entry, "%s mode %d pipeline %d, %d frames from 2^32 - 3, frames_per_batch %d" % (entry, mode, pipeline, spp, fpb))
                blended = [got["image"][..., :3]] + [got[k] for k in ("aov", "luma2") if k in got]
                if spp == 2:
                    assert all(np.isfinite(a).all() for a in blended)
                else:
                    assert all(np.isnan(a).all() for a in blended)
                assert (got["image"][..., 3] == 1.0).all()
    finally:
        sc.close()


# ------------------------------------------------------------------ parts that own no pixel
@pytest.mark.parametrize("channels", [3, 4])
@pytest.mark.parametrize("entry", ["render", "aov", "adaptive"])
def test_parts_that_own_no_pixel(entry, channels):
    """A 20 x 20 image has 4 tiles; tile (tx, ty) goes to part (tx + ty) % 8, so of 8 parts only 0-2 own pixels.  Ranks 3-7
    return 0 pixels and 0 rays, the scatter of all ranks is the whole render, and a render that continues (first_frame > 0)
    leaves an empty part's buffers untouched."""
    import torch
    sd = Sd("grid")
    sc = sd.scene()
    try:
        for mode in (api.MODE_DISNEY_IS_MIS_P5, L4):
            cfg = sd.cfg(width=20, height=20, spp=4, mode=mode, out_channels=channels)
            whole, _ = _check(sd, sc, cfg, entry, "%s mode %d, one part" % (entry, mode))
            parts = {k: np.zeros_like(a) for k, a in whole.items()}
            for rank in range(8):
                p = _with(cfg, part_rank=rank, part_count=8)
                n = api.partition_pixels(20, 20, rank, 8)
                assert (n == 0) == (rank >= 3)
                got, _ = _check(sd, sc, p, entry, "%s mode %d, part %d of 8" % (entry, mode, rank))
                mask = _part_tiles(p)[0]
                for k, a in got.items():
                    parts[k][mask] = a[mask]
            for k in whole:
                assert parts[k].tobytes() == whole[k].tobytes(), "%s mode %d: scatter of the 8 parts, %s" % (entry, mode, k)
            # device buffers of an empty part, filled with a sentinel, after a render that continues (adaptive: from frame 0)
            p = _with(cfg, part_rank=6, part_count=8, first_frame=0 if entry == "adaptive" else 5)
            bufs = [torch.full((64,), 7.0, dtype=torch.float32, device="cuda") for _ in range(3)]
            if entry == "render":
                assert sc.render(p).shape == (0, channels)     # the host entry point: nothing to copy either way
                sc.render_device(p, bufs[0])
            elif entry == "aov":
                assert sc.render_aov(p)[0].shape == (0, channels)
                sc.render_aov_device(p, *bufs)
            else:
                sc.render_adaptive_device(p, *ADAPT, bufs[0], bufs[1], bufs[2])
            torch.cuda.synchronize()
            assert all((b.cpu().numpy() == 7.0).all() for b in bufs), "%s mode %d: an empty part wrote to its buffers" % (entry, mode)
            assert sc.counters().rays == 0
    finally:
        sc.close()


# ------------------------------------------------------------------ mode 4 beside the other entry points
@pytest.fixture(scope="module")
def grid():
    sd = Sd("grid")
    sc = sd.scene()
    yield sd, sc
    sc.close()


def test_mode4_feature_buffers(grid):
    sd, sc = grid
    got, _ = _check(sd, sc, sd.cfg(spp=3, mode=L4), "aov", "mode 4 feature buffers")
    cov = got["aov"][..., 3]
    assert (cov == 0).any() and (cov == 1).any()


def test_mode4_adaptive_tiles_and_spp_map(grid):
    sd, sc = grid
    got, _ = _check(sd, sc, sd.cfg(spp=8, mode=L4), "adaptive", "mode 4 adaptive")
    spp = got["spp"][..., 0]
    assert spp.min() < spp.max(), "every tile stopped at the same test: the criterion is not exercised"


def test_mode4_nearest_map_and_no_bounce(grid):
    sd, sc = grid
    _check(sd, sc, sd.cfg(mode=L4, max_bounce=0), "render", "mode 4, max_bounce 0")
    _check(sd, sc, sd.cfg(mode=L4, max_bounce=0), "aov", "mode 4 feature buffers, max_bounce 0")
    near = Sd("grid", "nearest")
    sc2 = near.scene()
    try:
        for bounces in (0, 2):
            _check(near, sc2, near.cfg(mode=L4, max_bounce=bounces), "render", "mode 4, nearest map, %d bounces" % bounces)
    finally:
        sc2.close()


# ------------------------------------------------------------------ the tuning knobs
# Read by ezrt_scene_create (capi.cu): set before api.Scene.  Values: those of tools/sweep_*.sh and the ends of each clamp.
# EZRT_VERBOSE only prints.  EZRT_L2_PERSIST is not tested: it changes a device-wide limit (cudaLimitPersistingL2CacheSize),
# which must not be touched on a GPU other work shares.
KNOBS = [("EZRT_TRI_W", "2"), ("EZRT_TRI_W", "64"), ("EZRT_TRI_L1_BYPASS", "0"), ("EZRT_TRI_L1_BYPASS", "1"),
         ("EZRT_TOP_NODES", "0"), ("EZRT_TOP_NODES", "1"),
         ("EZRT_REFILL_CAM", "1"), ("EZRT_REFILL_CAM", "8"), ("EZRT_REFILL_CAM", "28"), ("EZRT_REFILL_CAM", "32"),
         ("EZRT_REFILL_T", "1"), ("EZRT_REFILL_T", "20"), ("EZRT_REFILL_T", "32"),
         ("EZRT_CHUNK", "64"), ("EZRT_CHUNK", "128"), ("EZRT_CHUNK", "65536"),
         ("EZRT_CHUNK_CAM", "32"), ("EZRT_CHUNK_CAM", "128"), ("EZRT_CHUNK_CAM", "65536"),
         ("EZRT_LEAF_T", "1"), ("EZRT_LEAF_T", "6"), ("EZRT_LEAF_T", "33"),
         ("EZRT_INNER_T", "1"), ("EZRT_INNER_T", "12"), ("EZRT_INNER_T", "32"),
         ("EZRT_BUILD", "host"), ("EZRT_W4_COLLAPSE", "greedy")]
# Read once per process into function-level statics (kernels.cu extend_threads / extend_blocks_per_sm, capi.cu ezrt_render):
# tested in a child process.
STATIC_KNOBS = [("EZRT_EXTEND_THREADS", "32"), ("EZRT_EXTEND_THREADS", "256"), ("EZRT_EXTEND_BPS", "2"), ("EZRT_EXTEND_BPS", "16"),
                ("EZRT_RENDER_OVERLAP", "0")]
KNOB_FORMS = {"W8": ({"EZRT_ACCEL": "8"}, "W8"), "4-wide": ({"EZRT_ACCEL": "4"}, "4-wide Q16")}   # environment, the form it must walk
KNOB_MODES = (api.MODE_DISNEY_IS_MIS_P5, L4)


@functools.lru_cache(maxsize=None)
def _knob_reference(mode):
    sd = Sd("grid")
    return _restate(sd, sd.cfg(mode=mode), "render")


@pytest.mark.parametrize("var,value", KNOBS, ids=["%s=%s" % k for k in KNOBS])
def test_scene_knob_keeps_the_oracle_bits(monkeypatch, var, value):
    sd = Sd("grid")
    monkeypatch.setenv(var, value)
    for form, (env, _) in KNOB_FORMS.items():
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, v)
            sc = sd.scene()
        try:
            for mode in KNOB_MODES:
                _check(sd, sc, sd.cfg(mode=mode), "render", "%s=%s, %s tree, mode %d" % (var, value, form, mode), _knob_reference(mode))
            if form == "W8":
                _assert_w8_ran(sc, sd.cfg(mode=L4), 0.25)
            assert _tree_form(sc, sd.cfg(mode=L4)) == KNOB_FORMS[form][1], (var, value, form)
        finally:
            sc.close()


_CHILD = textwrap.dedent("""
    import os, sys
    import numpy as np
    sys.path.insert(0, {root!r})
    from ezrt_b200 import api, scenes
    tris, nodes, eye, cam = scenes.s_grid(3, 2, 2)
    hdr = scenes.synth_hdr(128, 64)
    cache = api.hdr_cache(hdr)
    out = {{}}
    for form, accel in (("W8", "8"), ("4-wide", "4")):
        os.environ["EZRT_ACCEL"] = accel
        sc = api.Scene(tris, nodes, hdr, cache)
        for mode in {modes!r}:
            cfg = dict(width=64, height=48, max_bounce=2, mode=mode, eye=tuple(eye), camera_rotate=tuple(cam), env_color={env!r})
            fb = sc.render(api.RenderConfig(spp=1, **cfg)).reshape(-1, 3).copy()
            # two more frames continue from the first: ezrt_render uploads the framebuffer (EZRT_RENDER_OVERLAP)
            out["%s_%d" % (form, mode)] = sc.render(api.RenderConfig(spp=2, first_frame=1, **cfg), framebuffer=fb)
            c = sc.counters()
            out["%s_%d_rays" % (form, mode)] = np.array([c.primary_rays, c.bounce_rays, c.shadow_rays])
        sc.render(api.RenderConfig(spp=1, profile=2, **cfg))   # a counting render: which tree the accel kernels walked
        c = sc.counters()
        out["%s_visits" % form] = np.array([c.node_visits, c.node_visits_96])
        sc.close()
    np.savez({path!r}, **out)
""")


@pytest.mark.parametrize("var,value", STATIC_KNOBS, ids=["%s=%s" % k for k in STATIC_KNOBS])
def test_process_knob_keeps_the_oracle_bits(tmp_path, var, value):
    sd = Sd("grid")
    path = str(tmp_path / "renders.npz")
    env = {**os.environ, var: value, "EZRT_AUTO_BUILD": "0"}
    code = _CHILD.format(root=ROOT, modes=KNOB_MODES, env=ENV, path=path)
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    got = np.load(path)
    for form in KNOB_FORMS:
        assert _classify(*(int(x) for x in got["%s_visits" % form])) == KNOB_FORMS[form][1], (var, value, form)
        for mode in KNOB_MODES:
            want, rays = _knob_reference(mode)
            assert_same_bits(got["%s_%d" % (form, mode)], want["image"], "%s=%s, %s tree, mode %d" % (var, value, form, mode))
            # the continued render's rays are those of its last two frames: the whole restatement's minus frame 0's
            first = _restate(sd, sd.cfg(mode=mode, spp=1), "render")[1]
            assert tuple(got["%s_%d_rays" % (form, mode)]) == tuple(a - b for a, b in zip(rays, first)), (var, value, form, mode)


# ------------------------------------------------------------------ a pairwise sweep
FACTORS = (
    ("form", ("w4q16", "w4exact", "w8flat", "w8idx")),
    ("mode", (0, 1, 2, 3, 4)),
    ("traverse", (api.TRAVERSE_ACCEL, api.TRAVERSE_REFERENCE, api.TRAVERSE_PRUNED)),
    ("pipeline", (WAVE, MEGA)),
    ("entry", ("render", "device", "aov", "adaptive")),
    ("fpb", (0, 1, 3, 300)),
    ("first", (0, 7, "end", "past")),   # end: the last frame is 0xFFFFFFFE (Sobol index 2^32 - 1); past: from 2^32 - 3 across the wrap
    ("bounces", (0, 1, 2, 5)),
    ("channels", (3, 4)),
    ("part", ("whole", "1of3", "empty")),
    ("map", ("none", "linear", "nearest")),
    ("order", ("pixel", "frame")),
    ("lane", ("on", "off")),
)
# Values whose rows compare no finite pixel: an empty part renders nothing, and past the wrap every blended value is NaN.  A
# row holds at most one of them and counts as covering only the pairs that contain it, so every other pair is covered by a row
# that compares finite pixels.
DEGENERATE = {("part", "empty"), ("first", "past")}
FORMS = {"w4q16": ("grid", {"EZRT_ACCEL": "4"}, "4-wide Q16"), "w4exact": ("grid", {"EZRT_ACCEL": "4", "EZRT_ACCEL_Q16": "0"}, "4-wide exact"),
         "w8flat": ("soup", {}, "W8"), "w8idx": ("grid", {"EZRT_ACCEL": "8"}, "W8")}
PARTS = {"whole": (0, 1), "1of3": (1, 3), "empty": (7, 8)}   # 40 x 24: 6 tiles, so part 7 of 8 owns none


def _allowed(row):
    """The constraints the API enforces, on a partial row: mode 3 needs a map; mode 4, feature buffers and adaptive renders
    need the wavefront pipeline; an adaptive render starts at frame 0.  And at most one degenerate value per row."""
    g = row.get
    if g("mode") == 3 and g("map") == "none":
        return False
    if g("pipeline") == MEGA and (g("mode") == 4 or g("entry") in ("aov", "adaptive")):
        return False
    if sum(item in DEGENERATE for item in row.items()) > 1:
        return False
    return not (g("entry") == "adaptive" and g("first") not in (None, 0))


def _completable(row):
    if not _allowed(row):
        return False
    for name, values in FACTORS:
        if name not in row:
            return any(_completable({**row, name: v}) for v in values)
    return True


def covering_array():
    """A fixed all-pairs covering array: every pair of values of two factors that some allowed row holds is in some row that
    checks it.  A row without a degenerate value checks all its pairs; a row with one checks only the pairs that contain it.
    Greedy and deterministic: each row starts from the smallest uncovered pair, and every other factor takes the first
    non-degenerate value that covers the most uncovered pairs and still leaves the row completable.
    Returns (rows, number of pairs, number of pairs without a degenerate value)."""
    names = [n for n, _ in FACTORS]
    dom = dict(FACTORS)
    key = lambda a, va, b, vb: (a, va, b, vb) if names.index(a) < names.index(b) else (b, vb, a, va)
    todo = {(a, va, b, vb) for i, a in enumerate(names) for b in names[i + 1:] for va in dom[a] for vb in dom[b] if _completable({a: va, b: vb})}
    pairs = len(todo)
    plain = sum((p[0], p[1]) not in DEGENERATE and (p[2], p[3]) not in DEGENERATE for p in todo)
    rows = []
    while todo:
        a, va, b, vb = min(todo, key=lambda p: (names.index(p[0]), dom[p[0]].index(p[1]), names.index(p[2]), dom[p[2]].index(p[3])))
        row = {a: va, b: vb}
        deg = [n for n in row if (n, row[n]) in DEGENERATE]
        for n in names:
            if n in row:
                continue
            best, gain = None, -1
            for v in dom[n]:
                cand = {**row, n: v}
                if (n, v) not in DEGENERATE and _completable(cand):
                    g = sum(key(n, v, m, row[m]) in todo for m in row if not deg or m in deg)
                    if g > gain:
                        best, gain = v, g
            row[n] = best
        assert _allowed(row)
        covered = {key(names[i], row[names[i]], m, row[m]) for i in range(len(names)) for m in names[i + 1:]
                   if not deg or deg[0] in (names[i], m)}
        assert covered & todo
        todo -= covered
        rows.append(row)
    return rows, pairs, plain


ROWS, N_PAIRS, N_PLAIN_PAIRS = covering_array()


def _row_id(i, r):
    return "r%02d-%s-m%d-t%d-%s-%s-fpb%d-ff%s-b%d-c%d-%s-%s-%s-lane%s" % (
        i, r["form"], r["mode"], r["traverse"], "mega" if r["pipeline"] == MEGA else "wave", r["entry"], r["fpb"],
        r["first"], r["bounces"], r["channels"], r["part"], r["map"], r["order"], r["lane"])


@pytest.mark.parametrize("row", ROWS, ids=[_row_id(i, r) for i, r in enumerate(ROWS)])
def test_pairwise_option_space(monkeypatch, row):
    geo, env, tree = FORMS[row["form"]]
    env = dict(env)
    if row["order"] == "frame":
        env["EZRT_CAMERA_ORDER"] = "frame"
    env["EZRT_DEFERRED_LANE"] = "1" if row["lane"] == "on" else "0"
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    sd = Sd(geo, row["map"])
    assert (len(sd.tris) >= W8_MIN_TRIANGLES) == (geo == "soup") and _indexed(sd.tris) == (geo == "grid")
    rank, count = PARTS[row["part"]]
    assert (api.partition_pixels(40, 24, rank, count) == 0) == (row["part"] == "empty")
    spp = 8 if row["entry"] == "adaptive" else (260 if row["fpb"] == 300 else 5)
    first = {"end": 2 ** 32 - 1 - spp, "past": WRAP}.get(row["first"], row["first"])
    cfg = sd.cfg(width=40, height=24, spp=spp, first_frame=first, max_bounce=row["bounces"], mode=row["mode"], traverse=row["traverse"],
                 pipeline=row["pipeline"], out_channels=row["channels"], part_rank=rank, part_count=count, frames_per_batch=row["fpb"])
    sc = sd.scene()
    try:
        got, _ = _check(sd, sc, cfg, row["entry"], "pairwise row %r" % (row,))
        img = got["image"][_part_tiles(cfg)[0]][:, :3]
        if row["part"] == "empty":
            assert img.size == 0
        elif row["first"] == "past":
            assert np.isnan(img).all(), "pairwise row %r: frame 0xFFFFFFFF must make every blended value NaN" % (row,)
        else:   # the row compares shading, not only ray counts
            assert img.size > 0 and np.isfinite(img).all(), "pairwise row %r: %d of %d values not finite" % (row, (~np.isfinite(img)).sum(), img.size)
        assert _tree_form(sc, cfg) == tree, "pairwise row %r: the accel kernels did not walk the %s tree" % (row, tree)
    finally:
        sc.close()
