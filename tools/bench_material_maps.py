"""Measure the material maps (RenderConfig.material_maps / EZRT_PARAM_MATERIAL_MAPS, DESIGN.md section 16).

For bench.py's C3 and C4 views at 1920x1080, 16 spp, 2 and 8 bounces, in the light sampling mode: S-1M mapped
(scenes.s_1m_bunny_mapped: the textured S-1M plus a metallic-roughness and a normal map) alternated with S-1M textured (the same scene
and textures, the maps off) --reps times in this one process.  Per case: ms of each render (CUDA events), the median, Mrays/s, and
k_shade / k_nee time of one render (torch.profiler).  Prints one JSON line with the card's name and power limit, read before and after.

    python tools/bench_material_maps.py [--workloads c3,c4] [--reps 3] [--bounces 2,8]
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
        raise SystemExit("bench_material_maps.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    from ezrt_b200 import api, scenes
    run_args = argparse.Namespace(traverse="accel", pipeline="wavefront", frames_per_batch=0, spp_per_step=16, image="1920x1080", scaling="auto")
    out = {"metric": "material maps: 16 spp renders of bench.py's views at 1920x1080, S-1M mapped alternated with S-1M textured",
           "gpu": gpu_card(0), "workloads": {}}
    tris, _, _, _, tex, uv, ids, mr, nm = scenes.s_1m_bunny_mapped()
    for name in [x for x in args.workloads.split(",") if x]:
        wl = bench.build_workload(name, device_cache=True)
        W, H = 1920, 1080
        runner = bench.Runner(run_args, wl, 0, 1, 0, W, H)
        try:
            assert tris.tobytes() == runner.scene.tris.tobytes(), "the mapped S-1M is not bench.py's scene"
            runner.scene.set_textures(tex, uv, ids)
            runner.scene.set_material_maps(mr, nm)
            rows = {}
            for nb in [int(x) for x in args.bounces.split(",") if x]:
                base = {**runner.cfg(0, 16).__dict__, "mode": api.MODE_DISNEY_LIGHTS, "max_bounce": nb, "textures": True}
                cases = (("textured", api.RenderConfig(**base)), ("mapped", api.RenderConfig(**{**base, "material_maps": True})))
                for _, cfg in cases:
                    timed(torch, runner, cfg)
                alt = {k: [] for k, _ in cases}
                rays = {}
                for _ in range(args.reps):
                    for k, cfg in cases:
                        alt[k].append(round(timed(torch, runner, cfg), 3))
                        rays[k] = int(runner.scene.counters().rays)
                row = {}
                for k, cfg in cases:
                    ms = sorted(alt[k])
                    kt = kernels(torch, runner, cfg)
                    row[k] = {"ms": alt[k], "median_ms": ms[len(ms) // 2], "mrays_per_s": round(rays[k] / (ms[len(ms) // 2] * 1e3), 1),
                              "k_shade_ms": round(sum(v for n, v in kt.items() if n.startswith("k_shade")), 3),
                              "k_nee_ms": round(sum(v for n, v in kt.items() if n.startswith("k_nee")), 3)}
                row["mapped_over_textured"] = round(row["mapped"]["median_ms"] / row["textured"]["median_ms"], 4)
                rows["bounces=%d" % nb] = row
            runner.scene.set_textures(None)
            out["workloads"][name] = {"image": [W, H], "cases": rows}
        finally:
            runner.close()
    out["gpu_after"] = gpu_card(0)
    bench.emit(out)


if __name__ == "__main__":
    main()
