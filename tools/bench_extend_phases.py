"""Where the 8-wide bounce and shadow kernels' warps spend their cycles, on bench.py's workloads.

For each workload (default C3 and C4, bench.py's configurations and views) it runs `--warmup` steps, then `--steps` steps with the
counting instantiation (params.profile = 2, the same render calls bench.py times) and reads the SM cycles each warp of k_extend_w8 and
k_shadow_w8 spent per phase (ezrt_get_w8_phase_cycles): refill (claiming a chunk, loading and setting up new rays), node steps,
triangle steps, and ray ends (the reference-leaf check, store or defer of a finished ray).  Each phase's share of the summed warp cycles
is printed as one JSON line with the card's name and power limit.  The counting instantiation is slower than the plain one and its
clock reads perturb the schedule a little; the shares are of its own cycles.

From the same run's step counts (ezrt_get_w8_step_counts) it also prints the price of each kind of step, the warp cycles of a node step
and of a triangle step, and the work per ray: node visits and triangle tests per ray (bounce rays for k_extend_w8, shadow rays for
k_shadow_w8, from the render's counters), and warp node and triangle steps per 32 rays.  These are the constants the collapse of the
8-wide tree weighs (accel_w8.cpp) and tools/w8_model.cpp predicts cycles with.

    python tools/bench_extend_phases.py [--workloads c3,c4] [--steps 2] [--warmup 3]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (the workloads and the per-workload runner of the benchmark)
from bench_adaptive import gpu_card  # noqa: E402


def measure(runner, steps, warmup):
    torch = runner.torch
    for s in range(warmup):
        runner.step(s)
    torch.cuda.synchronize()
    for s in range(steps):
        runner.step(warmup + s, profile=2, accumulate=(s > 0))
    torch.cuda.synchronize()
    out = {}
    steps_all = runner.scene.w8_step_counts()
    cnt = runner.scene.counters()
    rays = {"k_extend_w8": cnt.bounce_rays, "k_shadow_w8": cnt.shadow_rays}
    for kernel, phases in runner.scene.w8_phase_cycles().items():
        total = sum(phases.values())
        if total == 0:
            continue
        st, n = steps_all[kernel], rays[kernel]
        out[kernel] = {"warp_cycles": total, "share": {k: round(v / total, 4) for k, v in phases.items()},
                       "cycles_per_node_step": round(phases["node"] / max(st["node_steps"], 1), 1),
                       "cycles_per_triangle_step": round(phases["triangle"] / max(st["triangle_steps"], 1), 1),
                       "rays": n,
                       "node_visits_per_ray": round(st["node_visits"] / max(n, 1), 3),
                       "triangle_tests_per_ray": round(st["triangle_tests"] / max(n, 1), 3),
                       "node_steps_per_32_rays": round(32 * st["node_steps"] / max(n, 1), 3),
                       "triangle_steps_per_32_rays": round(32 * st["triangle_steps"] / max(n, 1), 3)}
    return {"image": [runner.W, runner.H], "steps": steps, "spp_per_step": runner.args.spp_per_step, "kernels": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c3,c4")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--spp-per-step", type=int, default=16)
    ap.add_argument("--frames-per-batch", type=int, default=0)
    args = ap.parse_args()
    bench.quiet_stdout()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_extend_phases.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    run_args = argparse.Namespace(traverse="accel", pipeline="wavefront", frames_per_batch=args.frames_per_batch, spp_per_step=args.spp_per_step,
                                  image=None, scaling="auto")
    out = {"metric": "share of k_extend_w8 / k_shadow_w8 warp cycles per phase, cycles per step, work per ray (counting instantiation)", "gpu": gpu_card(0), "workloads": {}}
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
