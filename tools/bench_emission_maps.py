"""Measure the emission maps (RenderConfig.emission_maps / EZRT_PARAM_EMISSION_MAPS, DESIGN.md section 18).

For bench.py's C3 and C4 views at 1920x1080, 16 spp, 2 and 8 bounces, in the light sampling mode: S-1M emission-mapped
(scenes.s_1m_bunny_emission_mapped: the textured S-1M with its emissive spheres mapped by banded emission textures) with the flag on,
alternated with the same scene and textures with the flag off, --reps times in this one process.  Also the emission table's build
(ezrt_scene_set_emission_maps, host clock around the call, which ends in a device synchronise), --reps times.  Per case: ms of each render (CUDA events), the median, Mrays/s, and
the per-kernel time of two profiled renders (torch.profiler), alternated.  Prints one JSON line with the card's name and power limit, read before and after.

    python tools/bench_emission_maps.py [--workloads c3,c4] [--reps 3] [--bounces 2,8]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (the workloads and the per-workload runner of the benchmark)
from bench_adaptive import gpu_card  # noqa: E402
from bench_lens import kernels, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c3,c4")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--bounces", default="2,8")
    args = ap.parse_args()
    bench.quiet_stdout()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_emission_maps.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    from ezrt_b200 import api, scenes
    run_args = argparse.Namespace(traverse="accel", pipeline="wavefront", frames_per_batch=0, spp_per_step=16, image="1920x1080", scaling="auto")
    import time
    out = {"metric": "emission maps: 16 spp renders of bench.py's views at 1920x1080, S-1M emission-mapped, the flag on alternated with off",
           "gpu": gpu_card(0), "workloads": {}}
    tris, _, _, _, tex, uv, ids, eid = scenes.s_1m_bunny_emission_mapped()
    for name in [x for x in args.workloads.split(",") if x]:
        wl = bench.build_workload(name, device_cache=True)
        W, H = 1920, 1080
        runner = bench.Runner(run_args, wl, 0, 1, 0, W, H)
        try:
            assert tris.tobytes() == runner.scene.tris.tobytes(), "the emission-mapped S-1M is not bench.py's scene"
            runner.scene.set_textures(tex, uv, ids)
            build_ms = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                runner.scene.set_emission_maps(eid)
                build_ms.append(round((time.perf_counter() - t0) * 1e3, 3))
            k = runner.scene.emission_light_table()[0].size
            rows = {"table": {"triangles": int(len(eid)), "mapped_emitters": int((eid >= 0).sum()), "lights": int(k), "build_ms": build_ms}}
            for nb in [int(x) for x in args.bounces.split(",") if x]:
                base = {**runner.cfg(0, 16).__dict__, "mode": api.MODE_DISNEY_LIGHTS, "max_bounce": nb, "textures": True}
                cases = (("flag_off", api.RenderConfig(**base)), ("flag_on", api.RenderConfig(**{**base, "emission_maps": True})))
                for _, cfg in cases:
                    timed(torch, runner, cfg)
                alt = {k: [] for k, _ in cases}
                rays = {}
                for _ in range(args.reps):
                    for k, cfg in cases:
                        alt[k].append(round(timed(torch, runner, cfg), 3))
                        c = runner.scene.counters()
                        rays[k] = (int(c.rays), int(c.primary_rays), int(c.bounce_rays), int(c.shadow_rays))
                prof = {k: [] for k, _ in cases}   # two profiled renders per case, alternated
                for _ in range(2):
                    for k, cfg in cases:
                        prof[k].append(kernels(torch, runner, cfg))
                row = {}
                for k, cfg in cases:
                    ms = sorted(alt[k])
                    cls = lambda kt, pre: round(sum(v for n, v in kt.items() if n.startswith(pre)), 3)
                    row[k] = {"ms": alt[k], "median_ms": ms[len(ms) // 2], "mrays_per_s": round(rays[k][0] / (ms[len(ms) // 2] * 1e3), 1),
                              "primary_bounce_shadow_rays": rays[k][1:],
                              "k_shade_ms": [cls(kt, "k_shade") for kt in prof[k]], "k_nee_ms": [cls(kt, "k_nee") for kt in prof[k]],
                              "all_kernels_ms": [round(sum(kt.values()), 3) for kt in prof[k]], "kernel_ms": prof[k][-1]}
                row["on_over_off"] = round(row["flag_on"]["median_ms"] / row["flag_off"]["median_ms"], 4)
                rows["bounces=%d" % nb] = row
            runner.scene.set_textures(None)
            out["workloads"][name] = {"image": [W, H], "cases": rows}
        finally:
            runner.close()
    out["gpu_after"] = gpu_card(0)
    bench.emit(out)


if __name__ == "__main__":
    main()
