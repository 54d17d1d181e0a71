#!/usr/bin/env python
"""tools/bench_adaptive.py -- work and image quality of tile-adaptive sampling on bench.py's workloads (one GPU).

  python tools/bench_adaptive.py --threshold 0.05 [--workloads c3,c2,c4] [--frames-per-batch 0]

For each workload's view (the scenes, image sizes and integrators of bench.py): a tile-adaptive render
(ezrt_render_adaptive_device, min_spp 16, interval 16, cap 256 spp), a 1024-spp plain render of the same view as the
reference, and a plain render at the adaptive render's rounded mean spp.  Prints one JSON line: per workload the rays and
CUDA-event ms of the adaptive render, its mean / max spp, the fraction of tiles stopped before the cap and the luminance
relMSE = mean((Y - Yref)^2 / (Yref^2 + 1e-2)) of both renders against the reference; plus the card's name and power limit.
Writes nothing to the tree.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the workloads and the per-workload runner of the benchmark)

MIN_SPP, INTERVAL, CAP, REF_SPP = 16, 16, 256, 1024


def gpu_card(index):
    """name and power limit of the card the numbers were measured on"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1])}
    except Exception:
        import torch
        return {"name": torch.cuda.get_device_name(index), "power_limit_w": None}


def luminance_relmse(img, ref):
    """mean((Y - Yref)^2 / (Yref^2 + 1e-2)) of the pass-3 luminance 0.3 r + 0.6 g + 0.1 b, in float64"""
    lum = lambda a: 0.3 * a[..., 0].astype(np.float64) + 0.6 * a[..., 1].astype(np.float64) + 0.1 * a[..., 2].astype(np.float64)
    y, yr = lum(img), lum(ref)
    return float(np.mean((y - yr) ** 2 / (yr * yr + 1e-2)))


def measure(runner, threshold):
    torch, sc, W, H, C = runner.torch, runner.scene, runner.W, runner.H, runner.C
    stream = runner.stream

    def timed(fn):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream)
        fn()
        ev1.record(stream)
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1), int(sc.counters().rays)

    fb = torch.zeros(W * H * C, dtype=torch.float32, device="cuda")

    def plain(spp):
        ms, rays = timed(lambda: sc.render_device(runner.cfg(0, spp), fb, stream))
        return fb.reshape(H, W, C).cpu().numpy(), rays, ms

    ref, _, _ = plain(REF_SPP)
    d_spp = torch.zeros(W * H, dtype=torch.int32, device="cuda")
    d_l2 = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    run = lambda: sc.render_adaptive_device(runner.cfg(0, CAP), threshold, MIN_SPP, INTERVAL, fb, d_spp, d_l2, stream)
    timed(run)   # warm-up: the first call sizes the tile lists
    ms, rays = timed(run)
    img = fb.reshape(H, W, C).cpu().numpy()
    spp = d_spp.reshape(H, W).cpu().numpy()
    eq_spp = max(1, int(round(float(spp.mean()))))
    eq_img, eq_rays, eq_ms = plain(eq_spp)
    return {"threshold": threshold, "min_spp": MIN_SPP, "interval": INTERVAL, "cap_spp": CAP, "image": [W, H],
            "rays": rays, "ms": ms, "mean_spp": float(spp.mean()), "max_spp": int(spp.max()),
            "tiles_stopped_before_cap": float((spp[::16, ::16] < CAP).mean()),
            "relmse": luminance_relmse(img, ref),
            "equal_spp_plain": {"spp": eq_spp, "rays": eq_rays, "ms": eq_ms, "relmse": luminance_relmse(eq_img, ref)},
            "reference_spp": REF_SPP}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--threshold", type=float, required=True)
    ap.add_argument("--workloads", default="c3,c2,c4")
    ap.add_argument("--frames-per-batch", type=int, default=0)
    args = ap.parse_args()
    bench.quiet_stdout()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_adaptive.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    # the runner's render settings, as bench.py's defaults give them at N = 1
    run_args = argparse.Namespace(traverse="accel", pipeline="wavefront", frames_per_batch=args.frames_per_batch, spp_per_step=16,
                                  image=None, scaling="auto")
    out = {"metric": "tile-adaptive sampling: work and luminance relMSE", "gpu": gpu_card(0), "workloads": {}}
    for name in [x for x in args.workloads.split(",") if x]:
        wl = bench.build_workload(name, device_cache=True)
        W, H, _ = bench.image_for(run_args, wl, 1)
        runner = bench.Runner(run_args, wl, 0, 1, 0, W, H)
        try:
            out["workloads"][name] = measure(runner, args.threshold)
        finally:
            runner.close()
    bench.emit(out)


if __name__ == "__main__":
    main()
