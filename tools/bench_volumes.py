"""Measure the volumes inside transmissive meshes (RenderConfig.volumes with RenderConfig.transmission, DESIGN.md section 21).

It reports, alternating the arms rep by rep in one process:
  - S-1M's glass grid (tests/volume_scenes.grid_coloured_glass: every other blob glass, three volumes) at 1920 x 1080, max_bounce 2 and
    8, 16 and 64 spp: the render with the volumes against the same scene under transmission alone (the VOL kernels and the interior test)
  - the flag with every id -1 (the VOL kernels, nothing absorbed) against transmission alone, 16 spp, max_bounce 8
  - kernel times of one render of each arm at max_bounce 8, 16 spp, from a separate torch.profiler run
  - glass in fog against fog alone: the same scene in a homogeneous medium over the grid (vertical optical depth 0.5), rendered with
    the medium only (the glass rendered as its opaque BRDF) and with medium, transmission and volumes, 16 spp, max_bounce 2 and 8
and the card's name and power limit before and after.  Prints one JSON line.  bench.py itself is unchanged.

    python tools/bench_volumes.py [--spps 16,64] [--bounces 2,8] [--reps 3]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (quiet_stdout, emit)
from bench_adaptive import gpu_card  # noqa: E402

W, H = 1920, 1080


def timed(torch, sc, cfg, fb, stream, warm=True):
    if warm:   # the first call at a new batch shape sizes the scratch; the first light sampling call builds the light table
        sc.render_device(cfg, fb, stream)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    sc.render_device(cfg, fb, stream)
    ev1.record(stream)
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1)


def kernel_ms(torch, sc, cfg, fb, stream):
    """device time per kernel name (ms) of one render under torch.profiler, the render warmed first"""
    from torch.profiler import ProfilerActivity, profile
    sc.render_device(cfg, fb, stream)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        sc.render_device(cfg, fb, stream)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            name = e.key.split("<")[0].split("(")[0]
            out[name] = out.get(name, 0.0) + t / 1e3
    return dict(sorted(out.items(), key=lambda kv: -kv[1])[:8])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spps", default="16,64")
    ap.add_argument("--bounces", default="2,8")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    bench.quiet_stdout()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_volumes.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    from ezrt_b200 import api
    from tests import volume_scenes as vs
    stream = torch.cuda.current_stream()
    fb = torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")
    out = {"metric": "volumes: S-1M glass grid with volumes against transmission alone", "gpu": gpu_card(0), "image": [W, H]}

    tris, nodes, eye, cam, vols, vid = vs.grid_coloured_glass(15, 13, 4)
    sc = api.Scene(tris, nodes)
    try:
        sc.set_volumes(vols, vid)

        def cfg(mb, spp, volumes):
            return api.RenderConfig(width=W, height=H, spp=spp, max_bounce=mb, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam),
                                    env_color=(0.2, 0.25, 0.3), transmission=True, volumes=volumes)
        rows = {}
        for mb in [int(x) for x in args.bounces.split(",") if x]:
            for spp in [int(x) for x in args.spps.split(",") if x]:
                arms = {"transmission": cfg(mb, spp, False), "volumes": cfg(mb, spp, True)}
                times = {k: [] for k in arms}
                rays = {}
                for _ in range(args.reps):
                    for k, c in arms.items():
                        times[k].append(timed(torch, sc, c, fb, stream))
                        rays[k] = int(sc.counters().rays)
                rows["bounces %d, %d spp" % (mb, spp)] = {"ms": times, "rays": rays,
                                                          "ratio_of_medians": float(np.median(times["volumes"]) / np.median(times["transmission"]))}
        out["s1m_glass_volumes"] = rows
        out["kernel_ms_profiled"] = {k: kernel_ms(torch, sc, cfg(8, 16, v), fb, stream) for k, v in (("transmission", False), ("volumes", True))}
        # the flag with every id -1: the VOL kernels run and absorb nothing
        sc.set_volumes(vols, np.full(tris.shape[0], -1, np.int32))
        arms = {"transmission": cfg(8, 16, False), "volumes_ids_-1": cfg(8, 16, True)}
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, c in arms.items():
                times[k].append(timed(torch, sc, c, fb, stream))
        out["ids_minus_1"] = {"bounces": 8, "spp": 16, "ms": times,
                              "ratio_of_medians": float(np.median(times["volumes_ids_-1"]) / np.median(times["transmission"]))}
        # glass in fog against fog alone
        sc.set_volumes(vols, vid)
        lo, hi = tris[:, 0:9].reshape(-1, 3).min(axis=0), tris[:, 0:9].reshape(-1, 3).max(axis=0)
        fog = dict(sigma_t=0.5 / float(2.0 - lo[1]), albedo=(0.9, 0.9, 0.9), g=0.3, box_min=(float(lo[0]), float(lo[1]), float(lo[2])),
                   box_max=(float(hi[0]), 2.0, float(hi[2])))
        sc.set_medium(**fog)
        rows = {}
        for mb in (2, 8):
            fog_only = cfg(mb, 16, False)
            fog_only.transmission, fog_only.medium = False, True
            glass = cfg(mb, 16, True)
            glass.medium = True
            arms = {"fog": fog_only, "glass_in_fog": glass}
            times = {k: [] for k in arms}
            rays = {}
            for _ in range(args.reps):
                for k, c in arms.items():
                    times[k].append(timed(torch, sc, c, fb, stream))
                    rays[k] = int(sc.counters().rays)
            rows["bounces %d, 16 spp" % mb] = {"ms": times, "rays": rays,
                                               "ratio_of_medians": float(np.median(times["glass_in_fog"]) / np.median(times["fog"]))}
        out["glass_in_fog"] = {"medium": fog, "rows": rows}
    finally:
        sc.close()
    out["gpu_after"] = gpu_card(0)
    bench.emit(out)


if __name__ == "__main__":
    main()
