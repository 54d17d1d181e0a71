"""Measure the light sampling mode (EZRT_MODE_DISNEY_LIGHTS, DESIGN.md section 10) on bench.py's workloads and views (C3, C2, C4).

For each workload it reports:
  - luminance relMSE against a REF_SPP render in mode 4, of the workload's own mode and of mode 4 at equal time (mode 4's spp is
    the own mode's spp scaled by their measured per-spp times, then measured)
  - the relMSE of a REF_SPP render in the workload's own mode against the same reference: the two estimators agree on real scenes
    when it is small
  - mode 4's Mrays/s and its per-class kernel times (profile = 1)
and the card's name and power limit.  Prints one JSON line.  bench.py itself is unchanged.

    python tools/bench_lights.py [--workloads c3,c2,c4] [--spps 16,64]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (the workloads and the per-workload runner of the benchmark)
from bench_adaptive import gpu_card, luminance_relmse  # noqa: E402

REF_SPP = 2048


def measure(runner, spps):
    from ezrt_b200 import api
    torch, sc, W, H, C = runner.torch, runner.scene, runner.W, runner.H, runner.C
    stream = runner.stream
    fb = torch.zeros(W * H * C, dtype=torch.float32, device="cuda")
    own = runner.wl["mode"]

    def cfg(mode, spp, **kw):
        return api.RenderConfig(**{**runner.cfg(0, spp).__dict__, "mode": mode, **kw})

    def timed(mode, spp, warm=True, **kw):
        if warm:   # the first call at a new batch shape sizes the scratch (cudaMalloc), the first mode-4 call builds the light table
            sc.render_device(cfg(mode, spp, **kw), fb, stream)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream)
        sc.render_device(cfg(mode, spp, **kw), fb, stream)
        ev1.record(stream)
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1)

    img = lambda: fb.reshape(H, W, C).cpu().numpy()
    timed(api.MODE_DISNEY_LIGHTS, REF_SPP, warm=False)
    ref = img()
    timed(own, REF_SPP, warm=False)
    agree = luminance_relmse(img(), ref)
    rows = {}
    for spp in spps:
        t_own = timed(own, spp)
        e_own = luminance_relmse(img(), ref)
        t4 = timed(api.MODE_DISNEY_LIGHTS, spp)
        e4 = luminance_relmse(img(), ref)
        eq = max(1, int(round(spp * t_own / t4)))
        t_eq = timed(api.MODE_DISNEY_LIGHTS, eq)
        rows[str(spp)] = {"own_ms": t_own, "own_relmse": e_own, "mode4_same_spp_ms": t4, "mode4_same_spp_relmse": e4,
                          "mode4_equal_time": {"spp": eq, "ms": t_eq, "relmse": luminance_relmse(img(), ref)}}
    # throughput and kernel classes of mode 4 (profile = 1)
    spp = spps[-1]
    t = timed(api.MODE_DISNEY_LIGHTS, spp, profile=1)
    c = sc.counters()
    kt = sc.kernel_times()
    return {"image": [W, H], "own_mode": own, "reference_spp": REF_SPP, "own_mode_at_reference_spp_relmse": agree, "equal_time": rows,
            "mode4": {"spp": spp, "ms": t, "rays": int(c.rays), "shadow_rays": int(c.shadow_rays), "mrays_per_s": c.rays / (t * 1e3),
                      "kernel_ms": {k: v[0] for k, v in kt.items()}}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c3,c2,c4")
    ap.add_argument("--spps", default="16,64")
    args = ap.parse_args()
    bench.quiet_stdout()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_lights.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    run_args = argparse.Namespace(traverse="accel", pipeline="wavefront", frames_per_batch=0, spp_per_step=16, image=None, scaling="auto")
    out = {"metric": "light sampling mode: luminance relMSE at equal time against the workload's own mode", "gpu": gpu_card(0), "workloads": {}}
    spps = [int(x) for x in args.spps.split(",") if x]
    for name in [x for x in args.workloads.split(",") if x]:
        wl = bench.build_workload(name, device_cache=True)
        W, H, _ = bench.image_for(run_args, wl, 1)
        runner = bench.Runner(run_args, wl, 0, 1, 0, W, H)
        try:
            out["workloads"][name] = measure(runner, spps)
        finally:
            runner.close()
    bench.emit(out)


if __name__ == "__main__":
    main()
