"""The W8 camera pass (k_extend_w8_camera: extend_w8_bundle in ezrt_b200/csrc/device_functions.cuh), which traces a warp's 32
camera rays as bundles, against oracle.render bit for bit, on the layouts of work that make a bundle unusual: a camera looking
along an axis (directions whose components change sign inside a bundle), batch sizes that make a bundle span pixels, a clipped
image, an adaptive render whose converged tiles leave slots empty, camera rays that tie on coincident triangles, and an eye
beyond the decode gate (every camera ray deferred at load)."""
import numpy as np
import pytest

from ezrt_b200 import api
from tests.test_gpu_w8 import W8_MIN_TRIANGLES, _assert_renders_match, _assert_w8_ran, _cfg, far_scene, stack_scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def blob():
    tris, nodes, eye, cam = far_scene(3.0, 6)   # two 81,920-triangle blobs side by side: the W8 tree
    assert len(tris) >= W8_MIN_TRIANGLES
    sc = api.Scene(tris, nodes)
    yield tris, nodes, eye, cam, sc
    sc.close()


def test_camera_along_an_axis(oracle, blob):
    tris, nodes, _, _, sc = blob
    for rot, up in ((0.0, 0.0), (90.0, 0.0), (0.0, 89.999)):
        eye, cam = api.camera_orbit(rot, up, 4.0)
        cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5, width=64, height=48, spp=16)
        _assert_renders_match(oracle, sc, tris, nodes, cfg, "axis camera (%g, %g)" % (rot, up))
    _assert_w8_ran(sc, cfg, 0.1)


@pytest.mark.parametrize("fpb", [1, 3, 17])
def test_camera_bundles_span_pixels(oracle, blob, fpb):
    tris, nodes, eye, cam, sc = blob
    cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5, width=48, height=40, spp=17, frames_per_batch=fpb)
    _assert_renders_match(oracle, sc, tris, nodes, cfg, "frames_per_batch %d" % fpb)


def test_camera_clipped_image(oracle, blob):
    tris, nodes, eye, cam, sc = blob
    cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5, width=1000, height=37, spp=2)
    _assert_renders_match(oracle, sc, tris, nodes, cfg, "1000x37")


def test_camera_adaptive_with_converged_tiles(blob):
    from tests import oracle_adaptive
    tris, nodes, eye, cam, sc = blob
    cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5, width=80, height=48, spp=8)
    got, spp, luma2 = sc.render_adaptive(cfg, 0.5, 2, 2)
    ref, rspp, rluma2, _ = oracle_adaptive.render_adaptive(tris, nodes, cfg, 0.5, 2, 2)
    assert (spp == rspp).all() and got.tobytes() == ref.tobytes() and luma2.tobytes() == rluma2.tobytes()
    assert spp.min() < spp.max(), "no tile converged early: the case is not exercised"


def test_camera_rays_tie_on_coincident_triangles(oracle):
    tris, nodes, eye, cam = stack_scene(0, 40)   # coincident stacks in z = 0.25, facing the camera above them
    sc = api.Scene(tris, nodes)
    try:
        cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5, width=64, height=48, spp=16)
        _assert_renders_match(oracle, sc, tris, nodes, cfg, "coincident stacks")
        _assert_w8_ran(sc, cfg, 1.0)
    finally:
        sc.close()


def test_camera_eye_beyond_the_decode_gate(oracle, blob):
    tris, nodes, _, _, sc = blob
    maxc = float(np.abs(tris[:, :9]).max())
    eye, cam = api.camera_orbit(20.0, 10.0, 4.5 * maxc)   # |eye| > W8_ORIGIN_LIMIT_REL * max|coordinate|
    cfg = _cfg(eye, cam, mode=api.MODE_DISNEY_SOBOL_P5, width=48, height=32, spp=4)
    _assert_renders_match(oracle, sc, tris, nodes, cfg, "eye beyond the gate")
    sc.render(api.RenderConfig(**{**cfg.__dict__, "profile": 2}))
    c = sc.counters()
    assert c.deferred_rays >= c.primary_rays
