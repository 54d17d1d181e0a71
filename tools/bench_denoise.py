"""Measure the feature-buffer render and the a-trous denoiser on bench.py's workloads and views (C3, C2, C4).

For each workload it reports:
  - the time of the feature-buffer render against the plain render at the same spp (alternated, three runs each): the overhead
  - the denoise kernels' CUDA-event time at 1920x1080 and 1024x1024 (median of 20 after warm-up)
  - luminance relMSE against a 1024-spp render, noisy and denoised, at 4, 16 and 64 spp
  - the equal-time comparison: the denoised n-spp image against a plain render given the same time (render + denoise)
and the card's name and power limit.  Prints one JSON line.  bench.py itself is unchanged.

    python tools/bench_denoise.py [--workloads c3,c2,c4]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (the workloads and the per-workload runner of the benchmark)
from bench_adaptive import REF_SPP, gpu_card, luminance_relmse  # noqa: E402

SPPS = (4, 16, 64)
OVERHEAD_SPP = 16


def measure(runner):
    from ezrt_b200 import api
    torch, sc, W, H, C = runner.torch, runner.scene, runner.W, runner.H, runner.C
    stream = runner.stream

    def timed(fn, warm=True):
        if warm:   # the first call at a new batch shape sizes the scratch (cudaMalloc): not part of the render's time
            fn()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream)
        fn()
        ev1.record(stream)
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1)

    fb = torch.zeros(W * H * C, dtype=torch.float32, device="cuda")
    aov = torch.zeros(W * H * 8, dtype=torch.float32, device="cuda")
    l2 = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    den = torch.zeros(W * H * C, dtype=torch.float32, device="cuda")
    plain = lambda spp: timed(lambda: sc.render_device(runner.cfg(0, spp), fb, stream))
    with_aov = lambda spp: timed(lambda: sc.render_aov_device(runner.cfg(0, spp), fb, aov, l2, stream))
    denoise = lambda spp: timed(lambda: sc.denoise_device(fb, C, aov, l2, W, H, spp, den, stream))
    img = lambda t: t.reshape(H, W, C).cpu().numpy()

    t_plain, t_aov = [], []
    for _ in range(3):
        t_plain.append(plain(OVERHEAD_SPP))
        t_aov.append(with_aov(OVERHEAD_SPP))
    out = {"image": [W, H], "reference_spp": REF_SPP,
           "overhead": {"spp": OVERHEAD_SPP, "plain_ms": t_plain, "aov_ms": t_aov,
                        "ratio_median": float(np.median(t_aov) / np.median(t_plain))}}

    timed(lambda: sc.render_device(runner.cfg(0, REF_SPP), fb, stream), warm=False)
    ref = img(fb)
    rows = {}
    for spp in SPPS:
        t_r = with_aov(spp)
        noisy = img(fb)
        t_d = float(np.median([denoise(spp) for _ in range(5)]))
        d = img(den)
        # equal time: the plain render given the time of render + denoise, found by scaling spp (the render's time grows
        # about linearly in spp), then measured
        t_p1 = plain(spp)
        eq_spp = max(spp, int(round(spp * (t_r + t_d) / t_p1)))
        t_eq = plain(eq_spp)
        rows[str(spp)] = {"render_aov_ms": t_r, "denoise_ms": t_d, "relmse_noisy": luminance_relmse(noisy, ref),
                          "relmse_denoised": luminance_relmse(d, ref),
                          "equal_time_plain": {"spp": eq_spp, "ms": t_eq, "relmse": luminance_relmse(img(fb), ref)}}
    out["quality"] = rows
    return out


def denoise_kernel_times(sc, torch, stream):
    """CUDA-event time of the denoiser alone (5 iterations, 3 channels) on synthetic inputs at two sizes"""
    res = {}
    for (w, h) in ((1920, 1080), (1024, 1024)):
        g = torch.Generator(device="cuda").manual_seed(1)
        col = torch.rand(w * h * 3, device="cuda", generator=g)
        aov = torch.rand(w * h * 8, device="cuda", generator=g)
        aov.view(-1, 8)[:, 3] = 1.0
        l2 = torch.rand(w * h, device="cuda", generator=g)
        out = torch.zeros_like(col)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(3):
            sc.denoise_device(col, 3, aov, l2, w, h, 16, out, stream)
        ts = []
        for _ in range(20):
            ev0.record(stream)
            sc.denoise_device(col, 3, aov, l2, w, h, 16, out, stream)
            ev1.record(stream)
            torch.cuda.synchronize()
            ts.append(ev0.elapsed_time(ev1))
        res["%dx%d" % (w, h)] = {"median_ms": float(np.median(ts)), "min_ms": float(np.min(ts))}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c3,c2,c4")
    ap.add_argument("--frames-per-batch", type=int, default=0)
    args = ap.parse_args()
    bench.quiet_stdout()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_denoise.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    run_args = argparse.Namespace(traverse="accel", pipeline="wavefront", frames_per_batch=args.frames_per_batch, spp_per_step=16,
                                  image=None, scaling="auto")
    out = {"metric": "feature buffers and a-trous denoiser: overhead, kernel time, luminance relMSE", "gpu": gpu_card(0), "workloads": {}}
    for i, name in enumerate([x for x in args.workloads.split(",") if x]):
        wl = bench.build_workload(name, device_cache=True)
        W, H, _ = bench.image_for(run_args, wl, 1)
        runner = bench.Runner(run_args, wl, 0, 1, 0, W, H)
        try:
            out["workloads"][name] = measure(runner)
            if i == 0:
                out["denoise_kernel"] = denoise_kernel_times(runner.scene, torch, runner.stream)
        finally:
            runner.close()
    bench.emit(out)


if __name__ == "__main__":
    main()
