"""Per-kernel CUDA time of bench.py's workloads through torch.profiler: how much of a step the camera pass takes.

For each workload (default C3 and C4, bench.py's configurations and views) it runs `--warmup` steps, then profiles `--steps`
steps of `--spp-per-step` samples (the same render calls bench.py times) and reports the CUDA time of every kernel, summed over
the profiled steps and grouped by kernel name without template arguments (k_extend_w8_camera, k_extend_w8, k_shadow_w8,
k_shade, the exact passes, ...), with its share of the summed kernel time and of the CUDA-event time of the same steps taken
in a separate, unprofiled run.  Prints one JSON line with the card's name and power limit.  bench.py itself is unchanged.

    python tools/bench_camera.py [--workloads c3,c4] [--steps 16] [--warmup 3]
"""
import argparse
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (the workloads and the per-workload runner of the benchmark)
from bench_adaptive import gpu_card  # noqa: E402


def kernel_base(name):
    """'void k_shade<2, false, false>(SceneDev, ...)' -> 'k_shade'"""
    name = re.sub(r"^void\s+", "", name)
    return re.split(r"[<(]", name, 1)[0].strip()


def measure(runner, steps, warmup):
    from torch.profiler import ProfilerActivity, profile
    torch = runner.torch
    for s in range(warmup):
        runner.step(s)
    torch.cuda.synchronize()
    # CUDA-event time of the steps, profiler off
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(runner.stream)
    for s in range(steps):
        runner.step(warmup + s, accumulate=(s > 0))
    ev1.record(runner.stream)
    torch.cuda.synchronize()
    step_ms = ev0.elapsed_time(ev1)
    # the same steps again under the profiler
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(steps):
            runner.step(warmup + s, accumulate=(s > 0))
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.events():
        if e.device_type.name != "CUDA" or not e.name:
            continue
        us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        k = kernels.setdefault(kernel_base(e.name), [0.0, 0])
        k[0] += us / 1e3
        k[1] += 1
    total = sum(v[0] for v in kernels.values())
    rows = {k: {"ms": round(v[0], 3), "launches": v[1], "share_of_kernel_time": round(v[0] / total, 4), "share_of_step_time": round(v[0] / step_ms, 4)}
            for k, v in sorted(kernels.items(), key=lambda kv: -kv[1][0])}
    return {"image": [runner.W, runner.H], "steps": steps, "spp_per_step": runner.args.spp_per_step, "step_time_ms": round(step_ms, 3),
            "kernel_time_ms": round(total, 3), "kernels": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c3,c4")
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--spp-per-step", type=int, default=16)
    ap.add_argument("--frames-per-batch", type=int, default=0)
    args = ap.parse_args()
    bench.quiet_stdout()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_camera.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    run_args = argparse.Namespace(traverse="accel", pipeline="wavefront", frames_per_batch=args.frames_per_batch, spp_per_step=args.spp_per_step,
                                  image=None, scaling="auto")
    out = {"metric": "per-kernel CUDA time (torch.profiler) per --steps steps", "gpu": gpu_card(0), "workloads": {}}
    for name in [x for x in args.workloads.split(",") if x]:
        wl = bench.build_workload(name, device_cache=True)
        W, H, _ = bench.image_for(run_args, wl, 1)
        runner = bench.Runner(run_args, wl, 0, 1, 0, W, H)
        try:
            out["workloads"][name] = measure(runner, args.steps, args.warmup)
        finally:
            runner.close()
    bench.emit(out)


if __name__ == "__main__":
    main()
