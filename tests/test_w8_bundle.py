"""A bundle traversal of the W8 tree for the camera pass: a warp's 32 rays walked as one bundle, one conservative interval test
per child slot for all of them (the bound is stated in tools/w8_model.cpp).  The CPU model (mode `bundle`) walks every 32
consecutive rays as one bundle and checks, for every ray, against its own per-ray walk: the same closest t, triangle and tie flag, every node of the per-ray walk visited
by the bundle and every triangle it tests tested by the bundle.  The scenes are the hostile ones of tests/test_gpu_w8.py, walked
by their own coherent bundles and by camera rays in the pass's pixel-major order (16 jittered samples per pixel).  No GPU."""
import os
import subprocess

import numpy as np

from ezrt_b200 import build, scenes
from tests import test_gpu_w8 as g
from tests.test_w8_tree import _model_rays, _model_stat


def camera_rays(eye, cam, width, height, x0, y0, w, h, spp, seed):
    """primary_ray (device_functions.cuh) in numpy for the pixels [x0, x0 + w) x [y0, y0 + h), pixel-major: the spp samples of a
    pixel are consecutive, as AccelCameraIO::slot_of orders a batch of spp frames"""
    rng = np.random.default_rng(seed)
    m = np.asarray(cam, np.float64).reshape(4, 4)
    py, px = np.mgrid[y0:y0 + h, x0:x0 + w]
    px, py = np.repeat(px.ravel(), spp), np.repeat(py.ravel(), spp)
    vx = (px + 0.5) / width * 2 - 1 + (rng.random(px.size) - 0.5) / width
    vy = (py + 0.5) / height * 2 - 1 + (rng.random(px.size) - 0.5) / height
    d = vx[:, None] * m[0, :3] + vy[:, None] * m[1, :3] - 1.5 * m[2, :3]
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    o = np.repeat(np.asarray(eye, np.float64)[None], px.size, 0)
    return o.astype(np.float32), d.astype(np.float32)


def _run_bundle(tmp_path, tris, o, d, supersets=True):
    """supersets=False: only the results must be equal.  The node and triangle supersets hold for equal limits; a bundle tests
    more triangles early, so its limit can fall below the per-ray walk's and skip a node that walk visited beyond its final
    best.  Incoherent bundles (random rays) show that; it changes no result."""
    exe = build.build_w8_model()
    tf, rf = os.path.join(str(tmp_path), "tris.f32"), os.path.join(str(tmp_path), "rays.f32")
    np.ascontiguousarray(tris, np.float32).tofile(tf)
    _model_rays(o, d).tofile(rf)
    r = subprocess.run([exe, tf, str(tris.shape[0]), rf, "bundle"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    out = r.stdout
    assert r.returncode in ((0, 5) if not supersets else (0,)), out
    m = _model_stat(out, r"bundle checks: results differing (\d+), rays with a node missing (\d+), rays with a triangle missing (\d+)")
    assert m.groups() == ("0", "0", "0") if supersets else m.group(1) == "0", out
    assert int(_model_stat(out, r"bundle: \d+ \(sub-\)bundles, (\d+) member rays").group(1)) > 0, out
    return out


def test_bundle_on_twins_and_stacks(tmp_path):
    tris, _, eye, cam = g.twin_scene()
    _run_bundle(tmp_path, tris, *camera_rays(eye, cam, 64, 48, 0, 0, 64, 48, 16, 1))
    for ulps in (0, 3):
        tris, _, eye, cam = g.stack_scene(ulps, 40 + ulps)
        _run_bundle(tmp_path, tris, *g.stack_rays(tris, 300, 7 + ulps))
        _run_bundle(tmp_path, tris, *camera_rays(eye, cam, 96, 72, 0, 0, 96, 72, 16, 2))


def test_bundle_on_the_soup_and_wide_scenes(tmp_path):
    tris, _, eye, cam = g.soup_scene()
    _run_bundle(tmp_path, tris, *camera_rays(eye, cam, 64, 48, 0, 0, 64, 48, 16, 3))
    tris, _, eye, cam = g.far_scene(1e8, 6)
    _run_bundle(tmp_path, tris, *g.far_rays(tris, 6000, 3), supersets=False)
    _run_bundle(tmp_path, tris, *camera_rays(eye, cam, 64, 48, 0, 0, 64, 48, 16, 4))


def test_bundle_on_c3_camera_rays(tmp_path):
    """A 128 x 64 window of C3 (bench.py: S-1M, 1920x1080) around the image centre, 16 samples per pixel; prints the prediction
    of the bundle's work against the per-ray walk's"""
    tris, _, eye, cam = scenes.s_1m_bunny()
    out = _run_bundle(tmp_path, tris, *camera_rays(eye, cam, 1920, 1080, 896, 508, 128, 64, 16, 5))
    print(out)
