"""Measure the environment map as a light (RenderConfig.env_light in the light sampling mode, DESIGN.md section 11) on bench.py's
C4 workload (S-1M under the 2048 x 1024 map) at its own 1920 x 1080 view and 2 bounces.

It reports:
  - luminance relMSE against a REF_SPP flagged render, of mode 3, mode 4 and mode 4 with the flag at each of --spps, and of
    mode 4 and the flagged mode at mode 3's time for that spp (their spp scaled by the measured per-spp times, then measured)
  - the relMSE of REF_SPP renders of mode 4 and of mode 3 against the same reference: small for an estimator that agrees,
    a floor that does not fall with more samples for a biased one
  - the flagged mode's Mrays/s and per-class kernel times (profile = 1)
and the card's name and power limit.  Prints one JSON line.  bench.py itself is unchanged.

    python tools/bench_env_light.py [--workload c4] [--spps 16,64]
"""
import argparse
import os
import sys

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
    arms = {"mode3": (api.MODE_DISNEY_IS_MIS_P5, False), "mode4": (api.MODE_DISNEY_LIGHTS, False), "mode4_env": (api.MODE_DISNEY_LIGHTS, True)}

    def cfg(arm, spp, **kw):
        mode, flag = arms[arm]
        return api.RenderConfig(**{**runner.cfg(0, spp).__dict__, "mode": mode, "max_bounce": 2, "env_light": flag, **kw})

    def timed(arm, spp, warm=True, **kw):
        if warm:   # the first call at a new batch shape sizes the scratch; the first flagged call builds the tables
            sc.render_device(cfg(arm, spp, **kw), fb, stream)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream)
        sc.render_device(cfg(arm, spp, **kw), fb, stream)
        ev1.record(stream)
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1)

    img = lambda: fb.reshape(H, W, C).cpu().numpy()
    timed("mode4_env", REF_SPP)
    ref = img()
    at_ref = {}
    for arm in ("mode4", "mode3"):
        timed(arm, REF_SPP, warm=False)
        at_ref[arm] = luminance_relmse(img(), ref)
    rows = {}
    for spp in spps:
        row = {}
        for arm in arms:
            t = timed(arm, spp)
            row[arm] = {"spp": spp, "ms": t, "relmse": luminance_relmse(img(), ref)}
        for arm in ("mode4", "mode4_env"):   # at mode 3's time for this spp
            eq = max(1, int(round(spp * row["mode3"]["ms"] / row[arm]["ms"])))
            t = timed(arm, eq)
            row[arm + "_at_mode3_time"] = {"spp": eq, "ms": t, "relmse": luminance_relmse(img(), ref)}
        rows[str(spp)] = row
    spp = spps[-1]
    t = timed("mode4_env", spp, profile=1)
    c = sc.counters()
    kt = sc.kernel_times()
    return {"image": [W, H], "max_bounce": 2, "reference": "mode4_env at %d spp" % REF_SPP, "relmse_at_reference_spp": at_ref, "by_spp": rows,
            "mode4_env": {"spp": spp, "ms": t, "rays": int(c.rays), "shadow_rays": int(c.shadow_rays), "mrays_per_s": c.rays / (t * 1e3),
                          "kernel_ms": {k: v[0] for k, v in kt.items()}}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c4")
    ap.add_argument("--spps", default="16,64")
    args = ap.parse_args()
    bench.quiet_stdout()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_env_light.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    run_args = argparse.Namespace(traverse="accel", pipeline="wavefront", frames_per_batch=0, spp_per_step=16, image=None, scaling="auto")
    out = {"metric": "environment map as a light: luminance relMSE against a %d-spp flagged render" % REF_SPP, "gpu": gpu_card(0)}
    wl = bench.build_workload(args.workload, device_cache=True)
    W, H, _ = bench.image_for(run_args, wl, 1)
    runner = bench.Runner(run_args, wl, 0, 1, 0, W, H)
    try:
        out[args.workload] = measure(runner, [int(x) for x in args.spps.split(",") if x])
    finally:
        runner.close()
    out["gpu_after"] = gpu_card(0)
    bench.emit(out)


if __name__ == "__main__":
    main()
