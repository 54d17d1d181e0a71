"""Measure the punctual lights (RenderConfig.punctual_lights / EZRT_PARAM_PUNCTUAL_LIGHTS, DESIGN.md section 17).

For bench.py's C3 and C4 views at 1920x1080, 16 spp, 2 and 8 bounces, in the light sampling mode: plain mode 4 against mode 4 with 1,
8 and 64 punctual lights (scenes.punctual_rig: a sun, a key spot and points, seeded), the four alternated --reps times in this one
process.  Per case: the ms of each rep, Mrays/s at the median, primary / bounce / shadow rays and the per-kernel time of one render
(torch.profiler).  Prints one JSON line with the card's name and power limit, read before and after.

    python tools/bench_punctual.py [--workloads c3,c4] [--reps 3] [--lights 1,8,64] [--bounces 2,8]
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
    ap.add_argument("--lights", default="1,8,64")
    ap.add_argument("--bounces", default="2,8")
    args = ap.parse_args()
    bench.quiet_stdout()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_punctual.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    from ezrt_b200 import api, scenes
    run_args = argparse.Namespace(traverse="accel", pipeline="wavefront", frames_per_batch=0, spp_per_step=16, image="1920x1080", scaling="auto")
    out = {"metric": "punctual lights: 16 spp renders of bench.py's views at 1920x1080", "gpu": gpu_card(0), "workloads": {}}
    counts = [int(x) for x in args.lights.split(",") if x]
    for name in [x for x in args.workloads.split(",") if x]:
        wl = bench.build_workload(name, device_cache=True)
        W, H = 1920, 1080
        runner = bench.Runner(run_args, wl, 0, 1, 0, W, H)
        try:
            rigs = {n: scenes.punctual_rig(runner.scene.tris, seed=n, n_points=max(0, n - 2))[:n] for n in counts}
            rows = {}
            for nb in [int(x) for x in args.bounces.split(",") if x]:
                base = {**runner.cfg(0, 16).__dict__, "mode": api.MODE_DISNEY_LIGHTS, "max_bounce": nb}
                plain, flagged = api.RenderConfig(**base), api.RenderConfig(**{**base, "punctual_lights": True})
                cases = ["mode4"] + ["lights=%d" % n for n in counts]

                def setup(k):
                    if k == "mode4":
                        return plain
                    runner.scene.set_punctual_lights(rigs[int(k.split("=")[1])])
                    return flagged

                ms = {k: [] for k in cases}
                for k in cases:   # warm every instantiation once
                    timed(torch, runner, setup(k))
                for _ in range(args.reps):
                    for k in cases:
                        ms[k].append(round(timed(torch, runner, setup(k)), 3))
                for k in cases:
                    cfg = setup(k)
                    timed(torch, runner, cfg)
                    c = runner.scene.counters()
                    med = sorted(ms[k])[len(ms[k]) // 2]
                    rows["bounces=%d %s" % (nb, k)] = {"ms": ms[k], "mrays_per_s": round(c.rays / (med * 1e3), 1), "primary_rays": int(c.primary_rays),
                                                       "bounce_rays": int(c.bounce_rays), "shadow_rays": int(c.shadow_rays),
                                                       "kernel_ms": kernels(torch, runner, cfg)}
            runner.scene.set_punctual_lights(None)
            out["workloads"][name] = {"image": [W, H], "cases": rows}
        finally:
            runner.close()
    out["gpu_after"] = gpu_card(0)
    bench.emit(out)


if __name__ == "__main__":
    main()
