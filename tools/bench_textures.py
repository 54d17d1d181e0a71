"""Measure base-colour textures (RenderConfig.textures / EZRT_PARAM_TEXTURES, DESIGN.md section 15).

For bench.py's C3 and C4 views at 1920x1080, 16 spp, 2 and 8 bounces, in the light sampling mode, on the textured S-1M
(scenes.s_1m_bunny_textured: vt read from OBJ text, the bunnies spherical, the floor planar, the lights untextured), three texture sets, each alternated with
plain mode 4 --reps times in this one process:
  l2     one 512 x 512 texture (1 MiB: fits in L2)
  big    eight 2048 x 2048 textures (128 MiB: far beyond L2)
  white  1x1 white textures (the image is mode 4's bit for bit): what the TEX kernels cost by themselves
Per case: ms of each render (CUDA events), Mrays/s, and k_shade / k_nee time of one render (torch.profiler).  Prints one JSON
line with the card's name and power limit, read before and after.

    python tools/bench_textures.py [--workloads c3,c4] [--reps 3] [--bounces 2,8] [--cases l2,big,white]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (the workloads and the per-workload runner of the benchmark)
from bench_adaptive import gpu_card  # noqa: E402
from bench_lens import kernels, timed  # noqa: E402


def texture_set(case):
    rng = np.random.default_rng(17)
    if case == "white":
        return [np.full((1, 1, 3), 255, np.uint8)] * 2
    if case == "l2":
        return [rng.integers(0, 256, (512, 512, 3), dtype=np.uint8)] * 2
    return [rng.integers(0, 256, (2048, 2048, 3), dtype=np.uint8) for _ in range(8)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c3,c4")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--bounces", default="2,8")
    ap.add_argument("--cases", default="l2,big,white")
    args = ap.parse_args()
    bench.quiet_stdout()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_textures.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    from ezrt_b200 import api, scenes
    run_args = argparse.Namespace(traverse="accel", pipeline="wavefront", frames_per_batch=0, spp_per_step=16, image="1920x1080", scaling="auto")
    out = {"metric": "base-colour textures: 16 spp renders of bench.py's views at 1920x1080, alternated with plain mode 4", "gpu": gpu_card(0),
           "workloads": {}}
    for name in [x for x in args.workloads.split(",") if x]:
        wl = bench.build_workload(name, device_cache=True)
        W, H = 1920, 1080
        runner = bench.Runner(run_args, wl, 0, 1, 0, W, H)
        try:
            rows = {}
            for case in [x for x in args.cases.split(",") if x]:
                tex = texture_set(case)
                tris, _, _, _, _, uv, ids = scenes.s_1m_bunny_textured(len(tex))
                assert tris.tobytes() == runner.scene.tris.tobytes(), "the textured S-1M is not bench.py's scene"
                runner.scene.set_textures(tex, uv, ids)
                for nb in [int(x) for x in args.bounces.split(",") if x]:
                    base = {**runner.cfg(0, 16).__dict__, "mode": api.MODE_DISNEY_LIGHTS, "max_bounce": nb}
                    plain, flagged = api.RenderConfig(**base), api.RenderConfig(**{**base, "textures": True})
                    timed(torch, runner, plain)
                    timed(torch, runner, flagged)
                    alt = {"mode4": [], case: []}
                    rays = {}
                    for _ in range(args.reps):
                        for k, cfg in (("mode4", plain), (case, flagged)):
                            alt[k].append(round(timed(torch, runner, cfg), 3))
                            rays[k] = int(runner.scene.counters().rays)
                    row = {}
                    for k, cfg in (("mode4", plain), (case, flagged)):
                        ms = sorted(alt[k])
                        kt = kernels(torch, runner, cfg)
                        row[k] = {"ms": alt[k], "mrays_per_s": round(rays[k] / (ms[len(ms) // 2] * 1e3), 1),
                                  "k_shade_ms": round(sum(v for n, v in kt.items() if n.startswith("k_shade")), 3),
                                  "k_nee_ms": round(sum(v for n, v in kt.items() if n.startswith("k_nee")), 3)}
                    rows["bounces=%d %s" % (nb, case)] = row
            runner.scene.set_textures(None)
            out["workloads"][name] = {"image": [W, H], "cases": rows}
        finally:
            runner.close()
    out["gpu_after"] = gpu_card(0)
    bench.emit(out)


if __name__ == "__main__":
    main()
