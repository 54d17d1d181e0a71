"""Renders of the density grid (EZRT_PARAM_MEDIUM_GRID, DESIGN.md section 20) in the CPU restatement (tests/oracle_medium_grid.cpp): a
pure absorber against Le exp(-tau), the white furnace, unbiasedness of the plume against the phase-only estimator and of a constant
grid against the homogeneous medium, a mutation of the majorants that the unbiasedness test must catch, and the renders that must
equal mode 4 or the homogeneous medium bit for bit."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_medium as om
from tests import oracle_medium_grid as og
from tests.test_light_sampling_laws import _block_z, _stats
from tests.test_medium_oracle import _quad, _scene


def _plume():
    return scenes.smoke_grid(24, 1)


@pytest.mark.parametrize("scale", [1.0, 0.9])
def test_pure_absorber(scale):
    """an emitter seen through an absorbing slab whose density steps along the view (1 then 2, one brick each): each sample is Le or 0,
    the mean Le exp(-tau); brick maxima scaled by 0.9 (a mutation, test-only) must fail the same check"""
    Le = 2.0
    emitter = api.Material(emissive=(Le, Le, Le), baseColor=(0, 0, 0))
    tris, nodes = _scene(_quad(0.0, 3.0, emitter))
    sigma = 0.9
    rho = np.ones((17, 2, 2), np.float32)
    rho[:8] = 2.0   # z-points 0..7 (the far half, toward the emitter) 2, the near half 1
    cfg = api.RenderConfig(width=16, height=16, spp=256, max_bounce=0, mode=api.MODE_DISNEY_LIGHTS, eye=(0, 0, 4), medium=True,
                           medium_grid=True)
    m = om.medium(sigma, albedo=(0, 0, 0), box_min=(-5.0, -5.0, 0.5), box_max=(5.0, 5.0, 2.0))
    img = og.render(tris, nodes, cfg, rho, brick_scale=scale, m=m)[0]
    ys, xs = np.mgrid[0:16, 0:16]
    vx, vy = (xs + 0.5) / 16 * 2 - 1, (ys + 0.5) / 16 * 2 - 1
    cosz = 1.5 / np.sqrt(vx ** 2 + vy ** 2 + 1.5 ** 2)
    mean_rho = (7 * 2.0 + 1.5 + 8 * 1.0) / 16   # the lattice's 16 cells along z: 7 of 2, one lerp from 2 to 1, 8 of 1
    want = Le * np.exp(-sigma * 1.5 * mean_rho / cosz)
    se = np.sqrt((want * (Le - want)).mean() / (cfg.spp * want.size))
    z = (img[..., 0].mean() - want.mean()) / se
    print("absorber, scale %.1f: mean %.5f, expected %.5f, z %.1f" % (scale, img[..., 0].mean(), want.mean(), z))
    assert (abs(z) < 4) if scale == 1.0 else (abs(z) > 4), z


def test_white_furnace():
    speck = api.Material(baseColor=(0, 0, 0))
    tris, nodes = _scene(_quad(-1000.0, 1e-3, speck))
    cfg = api.RenderConfig(width=16, height=16, spp=8, max_bounce=64, mode=api.MODE_DISNEY_LIGHTS, eye=(0, 0, 0), env_color=(1, 1, 1), medium=True,
                           medium_grid=True)
    m = om.medium(3.0, albedo=(1, 1, 1), g=0.3, box_min=(-2, -2, -2), box_max=(2, 2, 2))
    img = og.render(tris, nodes, cfg, _plume(), m=m)[0]
    frac = np.round(img[..., 0] * 8) / 8   # every sample is 1 unless cut by the bounce cap
    assert np.allclose(img[..., 0], frac, atol=1e-6) and img.mean() > 0.9


def _arms(tris, nodes, eye, cam, fog, rho, hdr, env_light, lens, lights=None, brick_scale=1.0, grid_ref=True, spp=64):
    """(estimator, phase-only reference) as running means of independent frame ranges, and the block z of their difference"""
    cache = None if hdr is None else api.hdr_cache(hdr)
    W, H = 32, 16
    out = []
    for ref in (False, True):
        first = spp if ref else 0
        cfg = api.RenderConfig(width=W, height=H, spp=spp, first_frame=first, max_bounce=6, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye),
                               camera_rotate=tuple(cam), env_color=(0.1, 0.1, 0.12), env_light=env_light, medium=True, medium_grid=True, **lens)
        m = om.medium(**fog)
        cfg.punctual_lights = lights is not None
        if ref and grid_ref:
            img, luma2, _, _ = og.render_medium(tris, nodes, cfg, m, rho, phase_only=True, hdr=hdr, hdr_cache=cache)
        elif ref:
            cfg.medium_grid = False
            img, luma2, _, _ = og.render(tris, nodes, cfg, None, m=m, lights=lights, hdr=hdr, hdr_cache=cache)
        else:
            img, luma2, _, _ = og.render(tris, nodes, cfg, rho, brick_scale=brick_scale, m=m, lights=lights, hdr=hdr, hdr_cache=cache)
        assert np.isfinite(img).all()
        scale = np.float64(first + spp) / spp
        y = _stats(img, luma2)[0] * scale
        out.append((y, np.maximum(luma2.astype(np.float64) * scale - y ** 2, 0.0)))
    zf = float(_block_z(out[0], out[1], spp, W, H, H, W).max())
    z8 = float(_block_z(out[0], out[1], spp, W, H, 8, 8).max())
    return zf, z8


FOG = dict(sigma_t=3.0, albedo=(0.9, 0.8, 0.7), g=0.5, box_min=(-1.2, -1.0, -1.2), box_max=(1.2, 1.4, 1.2))


@pytest.mark.parametrize("case", ["plain", "env_light", "lens"])
def test_plume_unbiased_against_phase_only(case):
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    hdr = scenes.synth_hdr(64, 32) if case != "plain" else None
    lens = dict(lens_radius=0.2, focus_distance=3.4) if case == "lens" else {}
    zf, z8 = _arms(tris, nodes, eye, cam, FOG, _plume(), hdr, case != "plain", lens)
    print("plume %s: frame z %.2f, largest 8x8 z %.2f" % (case, zf, z8))
    assert zf <= 4 and z8 <= 5, (case, zf, z8)


def test_constant_grid_unbiased_against_homogeneous():
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    fog = dict(FOG, sigma_t=1.5)
    zf, z8 = _arms(tris, nodes, eye, cam, fog, np.ones((9, 17, 10), np.float32), None, False, {}, grid_ref=False)
    print("constant grid: frame z %.2f, largest 8x8 z %.2f" % (zf, z8))
    assert zf <= 4 and z8 <= 5, (zf, z8)


def test_punctual_lights_through_a_constant_grid_unbiased_against_homogeneous():
    """punctual lights through the grid's ratio tracking: the phase-only estimator cannot reach delta lights, so a constant grid lit by
    them is held to the homogeneous medium lit by them"""
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    fog = dict(FOG, sigma_t=1.5)
    lights = scenes.punctual_rig(tris)
    zf, z8 = _arms(tris, nodes, eye, cam, fog, np.ones((3, 9, 17), np.float32), None, False, {}, lights=lights, grid_ref=False)
    print("constant grid, punctual: frame z %.2f, largest 8x8 z %.2f" % (zf, z8))
    assert zf <= 4 and z8 <= 5, (zf, z8)


def test_zero_grid_untouched_box_and_unflagged_equal_existing_renders():
    tris, nodes, eye, cam = scenes.s_p3_bunny()
    hdr = scenes.synth_hdr(64, 32)
    cache = api.hdr_cache(hdr)
    for kw in (dict(), dict(env_light=True, lens_radius=0.1, focus_distance=3.5)):
        cfg = api.RenderConfig(width=24, height=16, spp=2, max_bounce=4, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam), **kw)
        plain = og.render(tris, nodes, cfg, None, hdr=hdr, hdr_cache=cache)
        cfg.medium, cfg.medium_grid = True, True
        zero = og.render(tris, nodes, cfg, np.zeros((5, 5, 5), np.float32), m=om.medium(**FOG), hdr=hdr, hdr_cache=cache)
        assert zero[0].tobytes() == plain[0].tobytes() and zero[3] == plain[3]
        far = og.render(tris, nodes, cfg, _plume(), m=om.medium(**dict(FOG, box_min=(40, 40, 40), box_max=(41, 41, 41))), hdr=hdr, hdr_cache=cache)
        assert far[0].tobytes() == plain[0].tobytes() and far[3] == plain[3]
        cfg.medium_grid = False
        homo = og.render(tris, nodes, cfg, None, m=om.medium(**FOG), hdr=hdr, hdr_cache=cache)
        ref = om.render(tris, nodes, cfg, om.medium(**FOG), hdr=hdr, hdr_cache=cache)
        assert homo[0].tobytes() == ref[0].tobytes() and homo[3] == ref[3]
