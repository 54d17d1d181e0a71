"""Measure the light tree (RenderConfig.light_tree / EZRT_PARAM_LIGHT_TREE, DESIGN.md section 19) against power-only selection.

Scenes at 1920x1080, 2 bounces, in the light sampling mode: S-1M (scenes.s_1m_bunny: four lamps), S-1M emission-mapped
(scenes.s_1m_bunny_emission_mapped, the emission table) and scenes.s_1m_lamps (a lamp over each of the 201 bunnies, 64,320 light
triangles).  Per scene and spp (16, 64): the flag on alternated with off --reps times in this one process, ms per render (CUDA events)
and their median, k_shade's time in two profiled renders (torch.profiler), and the luminance relMSE against a 2048-spp render of mode 4
(the flag off), at equal spp and at equal time (relMSE times the ratio of the medians: the variance of either estimator falls as 1/spp).
Prints one JSON line with the card's name and power limit, read before and after.

    python tools/bench_light_tree.py [--scenes s1m,s1m_emap,s1m_lamps] [--reps 3] [--spp 16,64] [--ref-spp 2048]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (quiet_stdout, emit)
from bench_adaptive import gpu_card, luminance_relmse  # noqa: E402
from bench_lens import kernel_base  # noqa: E402

W, H = 1920, 1080


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="s1m,s1m_emap,s1m_lamps")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--spp", default="16,64")
    ap.add_argument("--ref-spp", type=int, default=2048)
    ap.add_argument("--bounces", type=int, default=2)
    args = ap.parse_args()
    bench.quiet_stdout()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_light_tree.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    from torch.profiler import ProfilerActivity, profile

    from ezrt_b200 import api, scenes
    out = {"metric": "light tree: 1920x1080 renders, %d bounces, the flag on alternated with off; relMSE against a %d-spp mode-4 render"
                     % (args.bounces, args.ref_spp), "gpu": gpu_card(0), "scenes": {}}
    stream = torch.cuda.current_stream()
    d_fb = torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")

    def timed(sc, cfg):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream)
        sc.render_device(cfg, d_fb, stream)
        ev1.record(stream)
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1)

    def k_shade_ms(sc, cfg):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            sc.render_device(cfg, d_fb, stream)
            torch.cuda.synchronize()
        tot = 0.0
        for e in prof.events():
            if e.device_type.name == "CUDA" and e.name and kernel_base(e.name).startswith("k_shade"):
                tot += (e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total) / 1e3
        return round(tot, 3)

    def image(sc, cfg):
        sc.render_device(cfg, d_fb, stream)
        torch.cuda.synchronize()
        return d_fb.reshape(H, W, 3).cpu().numpy().copy()

    for name in [x for x in args.scenes.split(",") if x]:
        if name == "s1m_emap":
            tris, nodes, eye, cam, tex, uv, ids, eid = scenes.s_1m_bunny_emission_mapped()
        else:
            tris, nodes, eye, cam = scenes.s_1m_lamps() if name == "s1m_lamps" else scenes.s_1m_bunny()
        sc = api.Scene(tris, nodes, device=0)
        try:
            extra = {}
            if name == "s1m_emap":
                sc.set_textures(tex, uv, ids)
                sc.set_emission_maps(eid)
                extra = dict(textures=True, emission_maps=True)
            base = dict(width=W, height=H, max_bounce=args.bounces, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam), **extra)
            ref = image(sc, api.RenderConfig(spp=args.ref_spp, **base))
            K = int(len(sc.light_tree(emission=(name == "s1m_emap"))["phi"]) + 1) // 2
            rows = {"lights": K}
            for spp in [int(x) for x in args.spp.split(",") if x]:
                cases = (("flag_off", api.RenderConfig(spp=spp, **base)), ("flag_on", api.RenderConfig(spp=spp, light_tree=True, **base)))
                for _, cfg in cases:
                    timed(sc, cfg)
                alt = {k: [] for k, _ in cases}
                for _ in range(args.reps):
                    for k, cfg in cases:
                        alt[k].append(round(timed(sc, cfg), 3))
                row = {}
                for k, cfg in cases:
                    ms = sorted(alt[k])
                    row[k] = {"ms": alt[k], "median_ms": ms[len(ms) // 2], "k_shade_ms": [k_shade_ms(sc, cfg) for _ in range(2)],
                              "relmse": float(luminance_relmse(image(sc, cfg), ref))}
                ratio = row["flag_on"]["median_ms"] / row["flag_off"]["median_ms"]
                row["on_over_off_ms"] = round(ratio, 4)
                row["relmse_on_over_off_equal_spp"] = round(row["flag_on"]["relmse"] / row["flag_off"]["relmse"], 4)
                row["relmse_on_over_off_equal_time"] = round(row["flag_on"]["relmse"] * ratio / row["flag_off"]["relmse"], 4)
                rows["spp=%d" % spp] = row
            out["scenes"][name] = rows
        finally:
            sc.close()
        del ref
    out["gpu_after"] = gpu_card(0)
    bench.emit(out)


if __name__ == "__main__":
    main()
