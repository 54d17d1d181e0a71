#!/usr/bin/env python
"""Randomised comparison of the CUDA path (through the C ABI) with the CPU oracle, bit for bit: scenes incl. a degenerate
triangle soup and a W8 scene (flat and indexed triangle records), five modes (mode 4 against tests/oracle_lights), 0-7
bounces, three traversal policies, both pipelines, batches of up to 300 frames, random image shapes / cameras / frame offsets
(some next to the uint32 wrap of the frame counter).  A mode-4 case with first_frame > 0 continues from a black framebuffer,
because its restatement starts from one: continuing mode 4 from earlier frames is checked by tests/test_gpu_lights.py, not here.
usage (GPU box): python tools/fuzz_gpu_vs_oracle.py [seconds]"""
import os
import sys
import time
from collections import Counter

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ezrt_b200 import api, scenes  # noqa: E402
from tests import oracle_binding as oracle  # noqa: E402
from tests import oracle_lights  # noqa: E402
from tests.test_gpu_parity import _soup  # noqa: E402

# scene name -> the form of the acceleration tree its size selects (capi.cu: W8 from 2^16 triangles)
FORMS = {"bunny": "4-wide", "grid": "4-wide", "soup": "4-wide", "w8 soup": "W8 flat", "w8 grid": "W8 indexed"}


def main():
    budget = float(sys.argv[1]) if len(sys.argv) > 1 else 60.0
    rng = np.random.default_rng(7)
    geo = {"bunny": scenes.s_bunny()[:2], "grid": scenes.s_grid(2, 2, 1)[:2], "w8 grid": scenes.s_grid(4, 4, 2)[:2]}
    for name, n, seed, leaf in (("soup", 1500, 9, 5), ("w8 soup", 70000, 4, 8)):
        tl = api.TriangleList()
        tl.append_encoded(_soup(n, seed))
        geo[name] = tl.build_bvh(leaf)
    assert all((len(geo[k][0]) >= 1 << 16) == FORMS[k].startswith("W8") for k in geo)
    hdr = scenes.synth_hdr(64, 32)
    cache = api.hdr_cache(hdr)
    dev = {(k, lin): api.Scene(t, n, hdr, cache, hdr_filter_linear=lin) for k, (t, n) in geo.items() for lin in (False, True)}
    t0 = time.time()
    n = bad = 0
    tally = Counter()
    while time.time() - t0 < budget:
        name = str(rng.choice(list(geo)))
        tris, nodes = geo[name]
        lin = bool(rng.integers(0, 2))
        mode, mb = int(rng.integers(0, 5)), int(rng.integers(0, 8))
        w, h = int(rng.integers(1, 70)), int(rng.integers(1, 50))
        big = rng.uniform() < 0.05   # a batch of more than 256 frames (k_shade's per-path Sobol pairs) on a small image
        if big:
            w, h = int(rng.integers(1, 17)), int(rng.integers(1, 17))
        spp = int(rng.integers(257, 301)) if big else int(rng.integers(1, 4))
        fpb = 0 if big or rng.uniform() < 0.5 else int(rng.integers(1, 301))
        u = rng.uniform()
        ff = int(rng.integers(0, 2000)) if u < 0.4 else (int(rng.integers(2 ** 32 - 6, 2 ** 32)) if u < 0.5 else 0)
        eye, cam = api.camera_orbit(float(rng.uniform(-180, 180)), float(rng.uniform(-89, 89)), float(rng.uniform(0.3, 9)))
        policy = 0 if rng.uniform() < 0.6 else int(rng.integers(1, 3))   # mostly the accel policy (whose tree form EZRT_ACCEL / EZRT_ACCEL_Q16 select)
        pipeline = int(rng.integers(0, 2)) if policy != 0 and mode != api.MODE_DISNEY_LIGHTS else 0
        cfg = api.RenderConfig(width=w, height=h, spp=spp, max_bounce=mb, mode=mode, eye=tuple(eye), camera_rotate=tuple(cam), first_frame=ff,
                               traverse=policy, pipeline=pipeline, frames_per_batch=fpb)
        fb0 = rng.uniform(0, 3, (h, w, 3)).astype(np.float32) if ff else None
        if mode == api.MODE_DISNEY_LIGHTS:   # its restatement starts from a black framebuffer
            fb0 = np.zeros((h, w, 3), np.float32) if ff else None
            a, _, c = oracle_lights.oracle_render_lights(tris, nodes, cfg, hdr=hdr, hdr_cache=cache, hdr_linear=lin)
        else:
            a, c = oracle.render(tris, nodes, cfg, hdr=hdr, hdr_cache=cache, hdr_linear=lin, framebuffer=None if fb0 is None else fb0.copy())
        sc = dev[(name, lin)]
        b = sc.render(cfg, framebuffer=None if fb0 is None else fb0.reshape(-1, 3).copy())
        same = bool(((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all()) and sc.counters().rays == c["rays"]
        n += 1
        tally["mode %d" % mode] += 1
        tally[FORMS[name]] += 1
        if not same:
            bad += 1
            print("MISMATCH", name, "(%s tree)" % FORMS[name], "mode", mode, "bounces", mb, "linear", lin, w, h, spp, "first_frame", ff,
                  "frames_per_batch", fpb, "policy", policy, "pipeline", pipeline)
    print("cases", n, "mismatches", bad, "|", dict(sorted(tally.items())), "| env", {k: v for k, v in os.environ.items() if k.startswith("EZRT_")})
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
