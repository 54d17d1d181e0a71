"""The thin-lens camera's definition (EZRT_PARAM_THIN_LENS, ezrt_math.h, DESIGN.md section 13) on the CPU, through its restatement
(tests/oracle_lens.cpp): the ray's geometry against float64, the concentric map's law, the lens stream's independence from the path's
draws, the circle of confusion of a point, camera_look_at, and the parameters the flag rejects."""
import math

import numpy as np
import pytest
from scipy import stats

from ezrt_b200 import api, scenes
from tests import oracle_binding, oracle_lens as ol
from tests import oracle_transmission as ot

EYE, CAM = api.camera_orbit(30.0, 20.0, 4.0)


def _matrices():
    """unit (camera_orbit), scaled (field of view and aspect as a scaled matrix) and look-at cameras: (eye, cam)"""
    scaled = CAM.copy()
    scaled[0:3] *= 1.9
    scaled[4:8] *= 0.7
    scaled[8:11] *= 2.5
    return [("orbit", EYE, CAM), ("scaled", EYE, scaled),
            ("look_at", *api.camera_look_at((1.0, 2.0, 5.0), (0.3, -0.2, 0.0), (0.0, 1.0, 0.0), 40.0, 16.0 / 9.0))]


def _cfg(eye, cam, **kw):
    base = dict(width=640, height=360, spp=1, max_bounce=2, mode=api.MODE_DIFFUSE_P3, eye=tuple(eye), camera_rotate=tuple(cam))
    base.update(kw)
    return api.RenderConfig(**base)


def _concentric64(u):
    a, b = 2.0 * u[:, 0].astype(np.float64) - 1.0, 2.0 * u[:, 1].astype(np.float64) - 1.0
    first = np.abs(a) > np.abs(b)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(first, a, b)
        phi = np.where(first, (math.pi / 4) * (b / a), math.pi / 2 - (math.pi / 4) * (a / b))
    phi = np.where((a == 0) & (b == 0), 0.0, phi)
    return np.stack([r * np.cos(phi), r * np.sin(phi)], 1)


@pytest.mark.parametrize("which", [0, 1, 2])
def test_ray_geometry_against_float64(which):
    name, eye, cam = _matrices()[which]
    rng = np.random.default_rng(11 + which)
    n = 100000
    W, H = 640, 360
    px, py, fr = rng.integers(0, W, n), rng.integers(0, H, n), rng.integers(0, 1 << 20, n)
    R, f = 0.15, 3.7
    r = ol.camera_rays(_cfg(eye, cam, lens_radius=R, focus_distance=f), px, py, fr)
    pin = ol.camera_rays(_cfg(eye, cam), px, py, fr)
    # the pinhole part is the pinhole's, bit for bit
    assert r["dir_pin"].tobytes() == pin["dir_pin"].tobytes() and r["seed"].tobytes() == pin["seed"].tobytes()
    M = cam.astype(np.float64).reshape(4, 4)   # rows = columns of camera_rotate
    c0, c1, c2 = M[0, :3], M[1, :3], M[2, :3]
    e = eye.astype(np.float64)
    dp = r["dir_pin"].astype(np.float64)
    F = e + dp * (f / (1.5 * np.linalg.norm(c2)))
    lxy = _concentric64(r["draws"])
    o = e + R * (lxy[:, :1] * c0 / np.linalg.norm(c0) + lxy[:, 1:] * c1 / np.linalg.norm(c1))
    d = (F - o) / np.linalg.norm(F - o, axis=1, keepdims=True)
    scale = np.abs(e).max() + R
    assert np.abs(r["o"] - o).max() <= 1e-5 * scale, name
    assert np.abs(r["d"] - d).max() <= 1e-5, name
    # the focus point lies at depth f along -c2
    np.testing.assert_allclose((F - e) @ (-c2 / np.linalg.norm(c2)), f, rtol=1e-5)   # the columns are orthogonal
    # every ray passes within 1e-5 (relative) of its pixel jitter's F
    ro, rd = r["o"].astype(np.float64), r["d"].astype(np.float64)
    v = F - ro
    miss = np.linalg.norm(v - (v * rd).sum(1, keepdims=True) * rd, axis=1)
    assert (miss <= 1e-5 * np.linalg.norm(v, axis=1)).all(), name
    # and starts on the lens disk
    assert (np.linalg.norm(ro - e, axis=1) <= R * (1 + 1e-5)).all()


def test_concentric_map_is_uniform_in_area():
    rng = np.random.default_rng(5)
    u = rng.random((1000000, 2), dtype=np.float32)
    xy = ol.concentric_disk(u).astype(np.float64)
    np.testing.assert_allclose(xy, _concentric64(u), atol=2e-6)
    r2 = (xy ** 2).sum(1)
    assert r2.max() <= 1.0 + 1e-6
    n_r, n_s = 10, 16   # equal-area rings (in r^2) x equal sectors
    ring = np.minimum((r2 * n_r).astype(int), n_r - 1)
    sector = np.minimum(((np.arctan2(xy[:, 1], xy[:, 0]) + math.pi) / (2 * math.pi) * n_s).astype(int), n_s - 1)
    counts = np.bincount(ring * n_s + sector, minlength=n_r * n_s)
    p = stats.chisquare(counts).pvalue
    assert p > 1e-4, p


def test_lens_stream_leaves_the_path_draws_alone(bunny_scene):
    tris, nodes, eye, cam = bunny_scene
    rng = np.random.default_rng(3)
    px, py, fr = rng.integers(0, 96, 5000), rng.integers(0, 64, 5000), rng.integers(0, 1000, 5000)
    pin = ol.camera_rays(_cfg(eye, cam, width=96, height=64), px, py, fr)
    lens = ol.camera_rays(_cfg(eye, cam, width=96, height=64, lens_radius=0.05, focus_distance=3.0), px, py, fr)
    # the seed the path starts with is the pinhole's: every draw after the jitter is the same
    assert lens["seed"].tobytes() == pin["seed"].tobytes()
    assert lens["dir_pin"].tobytes() == pin["dir_pin"].tobytes()
    # with the flag off the restatement is the oracle, bit for bit, in every mode
    hdr = scenes.synth_hdr(64, 32)
    cache = api.hdr_cache(hdr)
    for mode in (0, 1, 2, 3):
        cfg = _cfg(eye, cam, width=48, height=32, spp=2, mode=mode)
        got, _, _, c = ol.render(tris, nodes, cfg, hdr=hdr, hdr_cache=cache)
        want, wc = oracle_binding.render(tris, nodes, cfg, hdr=hdr, hdr_cache=cache)
        assert got.tobytes() == want.tobytes() and c["rays"] == wc["rays"], mode
    for env_light, trans in ((False, False), (True, False), (True, True)):
        cfg = _cfg(eye, cam, width=48, height=32, spp=2, mode=api.MODE_DISNEY_LIGHTS, env_light=env_light, transmission=trans)
        got, luma2, _, c = ol.render(tris, nodes, cfg, hdr=hdr, hdr_cache=cache)
        want, wluma2, wc = ot.oracle_render_transmission(tris, nodes, cfg, hdr=hdr, hdr_cache=cache)
        assert got.tobytes() == want.tobytes() and luma2.tobytes() == wluma2.tobytes() and c["rays"] == wc["rays"]


def test_lens_stream_is_the_pixel_seed_with_the_salt():
    """ez_lens_draws = the first two rand() (wang_hash, P5/fsh:320-331; the oracle's chain) of pixel_seed(px, py, frame) ^
    EZRT_LENS_SALT: pins the lens stream to the path stream's seed and hash definitions"""
    rng = np.random.default_rng(9)
    n = 500
    px, py, fr = rng.integers(0, 4096, n), rng.integers(0, 4096, n), rng.integers(0, 1 << 32, n, dtype=np.uint64)
    got = ol.camera_rays(_cfg(EYE, CAM, width=4096, height=4096, lens_radius=0.1, focus_distance=3.0), px, py, fr)["draws"]
    for i in range(n):
        seed = ((int(px[i]) * 1973 + int(py[i]) * 9277 + int(fr[i]) * 26699) & 0xFFFFFFFF) | 1
        _, rands = oracle_binding.wang_chain(seed ^ 0x4C454E53, 2)
        assert got[i].tobytes() == np.asarray(rands, np.float32).tobytes(), i


def _point_scene(z, r_eye):
    """one small emissive triangle centred on the view axis of camera_orbit(0, 0, r_eye), at depth z, NDC radius 0.12"""
    a = 0.12 * z / 1.5
    cz = r_eye - z
    p = [(0.0, a, cz), (-0.8660254 * a, -0.5 * a, cz), (0.8660254 * a, -0.5 * a, cz)]
    t = np.zeros(36, np.float32)
    t[0:9] = np.array(p, np.float32).reshape(-1)
    for k in range(3):
        t[9 + 3 * k:12 + 3 * k] = (0.0, 0.0, 1.0)
    t[18:21] = (10.0, 10.0, 10.0)   # emissive
    t[21:24] = (1.0, 1.0, 1.0)
    tl = api.TriangleList()
    tl.append_encoded(t.reshape(1, 36))
    return tl.build_bvh(8)


def _moment(img):
    L = img[..., 0].astype(np.float64)
    H, W = L.shape
    y, x = np.mgrid[0:H, 0:W]
    nx, ny = (x + 0.5) / W * 2 - 1, (y + 0.5) / H * 2 - 1
    flux = L.sum()
    return ((nx ** 2 + ny ** 2) * L).sum() / flux, flux


COC_CASES = [(z, R) for R in (1.2, 2.4) for z in (2.0, 3.0, 4.5)]


def coc_case(render, z, R, f=3.0, r_eye=4.0, spp=2048):
    """(measured lens moment - pinhole moment, c^2 / 2, lens flux / pinhole flux) of the point at depth z; render(tris, nodes, cfg)"""
    tris, nodes = _point_scene(z, r_eye)
    eye, cam = api.camera_orbit(0.0, 0.0, r_eye)
    base = dict(width=64, height=64, spp=spp, max_bounce=0, mode=api.MODE_DIFFUSE_P3, eye=tuple(eye), camera_rotate=tuple(cam))
    m_pin, flux_pin = _moment(render(tris, nodes, api.RenderConfig(**base)))
    m_lens, flux_lens = _moment(render(tris, nodes, api.RenderConfig(lens_radius=R, focus_distance=f, **base)))
    c = 1.5 * R * abs(z - f) / (z * f)
    return m_lens - m_pin, c * c / 2, flux_lens / flux_pin, m_pin


def check_coc(got, z, f=3.0):
    dm, want, flux_ratio, m_pin = got
    if z == f:
        assert abs(dm) <= 0.05 * m_pin, (z, dm, m_pin)
    else:
        assert abs(dm - want) <= 0.05 * want, (z, dm, want)
    assert abs(flux_ratio - 1.0) <= 0.02, (z, flux_ratio)


@pytest.mark.parametrize("z,R", COC_CASES)
def test_circle_of_confusion(z, R):
    check_coc(coc_case(lambda t, n, cfg: ol.render(t, n, cfg)[0], z, R), z)


def test_camera_look_at():
    rng = np.random.default_rng(2)
    for _ in range(200):
        eye = rng.normal(size=3) * 5
        target = rng.normal(size=3)
        up = rng.normal(size=3)
        vfov, aspect = rng.uniform(5, 170), rng.uniform(0.2, 4)
        e, cam = api.camera_look_at(eye, target, up, vfov, aspect)
        f = (target - eye) / np.linalg.norm(target - eye)
        s = np.cross(f, up); s /= np.linalg.norm(s)
        u = np.cross(s, f)
        t = math.tan(math.radians(vfov) / 2) * 1.5
        want = np.concatenate([s * aspect * t, [0], u * t, [0], -f, [0], eye, [1]])
        np.testing.assert_allclose(cam, want, rtol=2e-5, atol=2e-5 * (1 + np.abs(want).max()))
    # the orbit's own view: vfov = 2 atan(2/3), aspect 1 -> camera_orbit's matrix within 2 ulp
    for ra, ua, r in ((0, 0, 4), (30, 20, 4), (-75, 60, 9.5), (140, -35, 0.7)):
        eye, cam = api.camera_orbit(ra, ua, r)
        _, la = api.camera_look_at(eye, (0, 0, 0), (0, 1, 0), math.degrees(2 * math.atan(2 / 3)), 1.0)
        # 2 ulp of each column's largest entry (the unit axes, and the eye in column 3)
        ulp = np.repeat([np.spacing(np.abs(cam[4 * k:4 * k + 4]).max()) for k in range(4)], 4)
        assert (np.abs(la - cam) <= 2 * ulp).all(), (ra, ua, r, (la - cam) / ulp)
    with pytest.raises(api.EzrtError):
        api.camera_look_at((0, 0, 1), (0, 0, 1))
    with pytest.raises(api.EzrtError):
        api.camera_look_at((0, 0, 1), (0, 0, 0), (0, 0, 1))
    with pytest.raises(api.EzrtError):
        api.camera_look_at((0, 0, 1), (0, 0, 0), vfov=180.0)


BAD_SCALARS = [float("nan"), float("inf"), float("-inf"), 0.0, -0.5]


class FlaggedConfig(api.RenderConfig):
    """a RenderConfig whose struct carries EZRT_PARAM_THIN_LENS even at lens_radius 0 (RenderConfig leaves the flag off there)"""

    def to_struct(self):
        p = super().to_struct()
        p.reserved[0] |= api.PARAM_THIN_LENS
        p.reserved[1], p.reserved[2] = (int(x) for x in np.array([self.lens_radius, self.focus_distance], np.float32).view(np.int32))
        return p


def bad_lens_configs(eye, cam, **kw):
    """every invalid EZRT_PARAM_THIN_LENS parameter set: R or f NaN, +-inf, 0, negative; a zero or non-finite column 0, 1 or 2"""
    base = dict(width=64, height=48, spp=1, max_bounce=2, mode=api.MODE_DIFFUSE_P3, eye=tuple(eye))
    base.update(kw)
    mk = lambda m, R, f: FlaggedConfig(camera_rotate=tuple(m), lens_radius=R, focus_distance=f, **base)
    out = [("R=%r" % v, mk(cam, v, 3.0)) for v in BAD_SCALARS] + [("f=%r" % v, mk(cam, 0.1, v)) for v in BAD_SCALARS]
    for col in (0, 1, 2):
        for v in (0.0, float("nan"), float("inf")):
            m = np.array(cam, np.float32).copy()
            m[4 * col:4 * col + 3] = v
            out.append(("column %d = %r" % (col, v), mk(m, 0.1, 3.0)))
    return out


def test_invalid_parameters():
    for what, cfg in bad_lens_configs(EYE, CAM):
        p = cfg.to_struct()
        R, f = np.array([p.reserved[1], p.reserved[2]], np.int32).view(np.float32)
        assert ol.lens_setup(cfg.eye, cfg.camera_rotate, R, f) is None, what
        with pytest.raises(ValueError):
            ol.camera_rays(cfg, [0], [0], [0])
    assert ol.lens_setup(EYE, CAM, 0.1, 3.0) is not None
    # RenderConfig sets the flag for any radius but 0, so that a negative or NaN one reaches the library's validation ...
    for R in (-0.5, float("nan"), float("inf")):
        assert api.RenderConfig(lens_radius=R, focus_distance=3.0).to_struct().reserved[0] & api.PARAM_THIN_LENS
    # ... and a lens without a focus distance is an error, not a default
    with pytest.raises(ValueError):
        api.RenderConfig(lens_radius=0.1).to_struct()
    assert api.RenderConfig(focus_distance=float("nan")).to_struct().reserved[0] & api.PARAM_THIN_LENS == 0
