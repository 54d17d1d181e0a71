"""world_size-2 gloo test (CPU) of the N>1 path: tile partition -> ONE gather -> de-interleave on rank 0.

No GPU here, so each rank fills its compact part buffer with a function of the pixel coordinates it owns
(through the same partition helpers the render uses) and rank 0 must reassemble the exact image."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _pixel_value(W, H, C):
    yy, xx = np.mgrid[0:H, 0:W]
    img = np.stack([(xx * 3 + yy * 7 + c * 1000).astype(np.float32) for c in range(C)], axis=-1)
    return img


def _worker(rank, world, port, W, H, C, out_path):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ezrt_b200 import api
    from ezrt_b200 import dist as ezdist
    full = _pixel_value(W, H, C)
    # this rank's compact part: gather its own pixels in partition order = scatter's inverse
    n = api.partition_pixels(W, H, rank, world)
    idx_img = np.arange(W * H, dtype=np.float32).reshape(H, W, 1)
    # recover the partition order by scattering pixel ids of a ramp through the host scatter
    probe = np.full((H, W, 1), -1, np.float32)
    api.partition_scatter_host(np.arange(n, dtype=np.float32).reshape(n, 1), probe, W, H, 1, rank, world)
    owned = probe[..., 0] >= 0
    order = np.argsort(probe[..., 0][owned])
    local = full[owned][order].reshape(-1)
    assert local.size == n * C
    img = ezdist.gather_framebuffer(torch.from_numpy(np.ascontiguousarray(local)), W, H, C, rank, world)
    if rank == 0:
        np.save(out_path, img.numpy())
    else:
        assert img is None
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world,W,H", [(2, 100, 52), (3, 64, 64)])
def test_gather_framebuffer_gloo(tmp_path, world, W, H):
    C = 3
    out = str(tmp_path / "img.npy")
    mp.spawn(_worker, args=(world, _free_port(), W, H, C, out), nprocs=world, join=True)
    got = np.load(out)
    np.testing.assert_array_equal(got, _pixel_value(W, H, C))


def test_bench_image_per_gpu_count():
    """bench.py: N = 1 renders the C3 image, N > 1 one fixed 3840x2160 image (BASELINE configs[4], strong scaling);
    --scaling weak keeps the pixels per GPU fixed."""
    sys.path.insert(0, ROOT)
    import argparse
    import bench
    wl = dict(width=1920, height=1080)
    strong = argparse.Namespace(image=None, scaling="auto")
    weak = argparse.Namespace(image=None, scaling="weak")
    assert bench.image_for(strong, wl, 1) == (1920, 1080, "strong")
    for n in (2, 4, 8):
        assert bench.image_for(strong, wl, n) == (3840, 2160, "strong")
        w, h, label = bench.image_for(weak, wl, n)
        assert w * h == 1920 * 1080 * n and label == "weak"
    assert bench.image_for(argparse.Namespace(image="640x360", scaling="auto"), wl, 4)[:2] == (640, 360)


def test_cpu_thread_count_is_explicit_and_bounded():
    sys.path.insert(0, ROOT)
    import bench
    n, info = bench.cpu_threads()
    assert 1 <= n <= (os.cpu_count() or 1) and info["affinity"] >= n


def test_bench_roofline_accounting():
    """roofline_of: own-layout bytes / HBM peak, with mixed node record sizes (no GPU: synthetic counters)."""
    sys.path.insert(0, ROOT)
    import bench
    res = {"kernel_ms": {"extend": 100.0, "shadow": 0.0, "shade": 10.0, "other": 1.0}, "kernel_launches": {"extend": 30, "shadow": 0, "shade": 30, "other": 10},
           "steps": 10, "ms": 120.0, "rank0_rays": 6.0e8, "workload": "c3"}
    counts = {"node_visits": 6.0e8, "node_visits_96": 4.0e8, "tri_tests": 4.0e8, "node_bytes": 2.0e8 * 128 + 4.0e8 * 96, "tri_bytes": 4.0e8 * 64,
              "rays": 6.0e7, "primary": 3.0e7, "bounce": 3.0e7, "shadow": 0}
    r = bench.roofline_of(res, counts, {"bytes_per_ray_reference": 11000.0}, 6574.8, "measured", "k_extend_accel")
    assert r["bound"] in ("hbm", "tensor") and r["unit"] == "GB/s"
    bytes_step = counts["node_bytes"] + counts["tri_bytes"] + 3.0e7 * 32 + 6.0e7 * 8
    assert abs(r["achieved"] - bytes_step / 0.010 / 1e9) < 1e-6 * r["achieved"]
    assert r["peak"] == 6574.8 and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-12
    assert r["demand"]["frac_of_hbm_peak"] > 1.0    # the reference-layout demand figure exceeds the HBM peak by design
    assert bench.roofline_of(res, None, None, 6574.8, "measured", "k") is None
