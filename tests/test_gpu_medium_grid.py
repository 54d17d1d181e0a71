"""GPU side of the density grid (EZRT_PARAM_MEDIUM_GRID, DESIGN.md section 20): the device's brick maxima and grid code against the CPU
restatement (tests/oracle_medium_grid.cpp) bit for bit, the renders that must equal existing renders bit for bit and ray for ray, a
constant grid against the homogeneous medium, and the renders and grids the library rejects."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from tests import oracle_medium_grid as og
from tests.test_medium_grid_oracle import _hostile_rays, _plume

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def smoke():
    tris, nodes, eye, cam, med, grid = scenes.s_p3_bunny_smoke(n=48)
    hdr = scenes.synth_hdr(64, 32)
    return tris, nodes, eye, cam, med, grid, hdr, api.hdr_cache(hdr)


def _cfg(eye, cam, **kw):
    base = dict(width=48, height=32, spp=2, max_bounce=4, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam), medium=True,
                medium_grid=True)
    base.update(kw)
    return api.RenderConfig(**base)


def _rays(sc):
    c = sc.counters()
    return c.primary_rays, c.bounce_rays, c.shadow_rays


def test_brick_maxima_and_eval_bits():
    rho = _plume(41)
    box = ((-1.0, -0.5, 0.25), (2.0, 1.5, 1.0))
    sigma_t = 3.0
    tris, nodes, _, _ = scenes.s_p3_bunny()
    sc = api.Scene(tris, nodes, device=0)
    try:
        sc.set_medium(sigma_t, box_min=box[0], box_max=box[1])
        sc.set_medium_grid(rho)
        assert sc.medium_grid().tobytes() == og.bricks(rho).tobytes()
        rng = np.random.default_rng(7)
        n = 1000000
        o, d = _hostile_rays(rng, n, np.array(box[0]), np.array(box[1]), (41, 41, 41))
        L = np.where(rng.random(n) < 0.5, np.float32(np.inf), rng.uniform(0, 4, n)).astype(np.float32)
        seed = rng.integers(1, 2 ** 32 - 1, n, dtype=np.uint64).astype(np.uint32)
        assert sc.medium_density(o).tobytes() == og.density(rho, sigma_t, *box, o).tobytes()
        flag, t_s, s_out = sc.medium_flight(o, d, L, seed)
        r = og.track(rho, sigma_t, *box, 1, o, d, L, seed, twin=False)
        assert np.array_equal(flag, r["flag"]) and np.array_equal(s_out, r["seed"])
        assert t_s[flag == 1].tobytes() == r["out"][flag == 1].tobytes()
        assert flag.sum() > 1000
        T = sc.medium_transmittance(o, d, L, seed)
        r = og.track(rho, sigma_t, *box, 2, o, d, L, seed, twin=False)
        assert T.tobytes() == r["out"].tobytes() and r["violations"] == 0
    finally:
        sc.close()


@pytest.mark.parametrize("env", ["none", "env_light"])
@pytest.mark.parametrize("lens", [False, True])
def test_zero_grid_equals_mode4(smoke, env, lens):
    tris, nodes, eye, cam, med, grid, hdr, cache = smoke
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        kw = dict(env_light=(env == "env_light"))
        if lens:
            kw.update(lens_radius=0.15, focus_distance=3.6)
        sc.set_medium(**med)
        sc.set_medium_grid(np.zeros_like(grid))
        got = sc.render(_cfg(eye, cam, **kw))
        rg = _rays(sc)
        ref = sc.render(_cfg(eye, cam, medium=False, medium_grid=False, **kw))
        assert got.tobytes() == ref.tobytes() and rg == _rays(sc)
    finally:
        sc.close()


def test_unflagged_grid_and_missed_box(smoke):
    tris, nodes, eye, cam, med, grid, hdr, cache = smoke
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        sc.set_medium(**med)
        homo = sc.render(_cfg(eye, cam, medium_grid=False))
        rh = _rays(sc)
        sc.set_medium_grid(grid)
        assert sc.render(_cfg(eye, cam, medium_grid=False)).tobytes() == homo.tobytes() and _rays(sc) == rh
        far = dict(med, box_min=(50.0, 50.0, 50.0), box_max=(51.0, 51.0, 51.0))
        sc.set_medium(**far)   # keeps the grid
        got = sc.render(_cfg(eye, cam))
        rg = _rays(sc)
        ref = sc.render(_cfg(eye, cam, medium=False, medium_grid=False))
        assert got.tobytes() == ref.tobytes() and rg == _rays(sc)
    finally:
        sc.close()


@pytest.mark.parametrize("bounces", [1, 4, 8])
def test_policies_batches_and_forms_agree(smoke, bounces):
    """the grid render is one image whatever the traversal policy, the batch size, the deferred lane and the render form"""
    tris, nodes, eye, cam, med, grid, hdr, cache = smoke
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        sc.set_medium(**med)
        sc.set_medium_grid(grid)
        base = sc.render(_cfg(eye, cam, max_bounce=bounces, env_light=True))
        assert np.all(np.isfinite(base)) and base.max() > 0
        for kw in (dict(traverse=api.TRAVERSE_REFERENCE), dict(traverse=api.TRAVERSE_PRUNED), dict(frames_per_batch=1), dict(profile=2)):
            assert sc.render(_cfg(eye, cam, max_bounce=bounces, env_light=True, **kw)).tobytes() == base.tobytes(), kw
        # the two frames as a render of frame 0 resumed by a render of frame 1 over its framebuffer
        f0 = sc.render(_cfg(eye, cam, max_bounce=bounces, env_light=True, spp=1))
        f1 = sc.render(_cfg(eye, cam, max_bounce=bounces, env_light=True, spp=1, first_frame=1), framebuffer=f0.copy())
        assert f1.tobytes() == base.tobytes()
        got, _, _ = sc.render_aov(_cfg(eye, cam, max_bounce=bounces, env_light=True))
        assert got.tobytes() == base.tobytes()
    finally:
        sc.close()


@pytest.mark.parametrize("opts", ["tree", "punctual", "dense", "g_back", "g_fwd"])
def test_grid_with_other_options_renders(smoke, opts):
    tris, nodes, eye, cam, med, grid, hdr, cache = smoke
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        m = dict(med)
        kw = {}
        if opts == "tree":
            kw.update(light_tree=True)
        elif opts == "punctual":
            sc.set_punctual_lights(scenes.punctual_rig(tris))
            kw.update(punctual_lights=True)
        elif opts == "dense":
            m.update(sigma_t=400.0)
        else:
            m.update(g=-0.999 if opts == "g_back" else 0.999)
        sc.set_medium(**m)
        sc.set_medium_grid(grid)
        a = sc.render(_cfg(eye, cam, **kw))
        b = sc.render(_cfg(eye, cam, traverse=api.TRAVERSE_REFERENCE, **kw))
        assert np.all(np.isfinite(a)) and np.all(a >= 0) and a.tobytes() == b.tobytes()
    finally:
        sc.close()


def test_constant_grid_matches_homogeneous_medium(smoke):
    """a grid of ones is the homogeneous medium in law: block means of independent frame ranges agree within a z of 4.5"""
    tris, nodes, eye, cam, med, grid, hdr, cache = smoke
    m = dict(med, sigma_t=1.5)
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        sc.set_medium(**m)
        sc.set_medium_grid(np.ones((5, 4, 3), np.float32))
        blocks, spp = 24, 16

        def block(first, **kw):   # frames first .. first + spp - 1 alone: the render blends them over a zero framebuffer of `first` frames
            return sc.render(_cfg(eye, cam, spp=spp, first_frame=first, env_light=True, **kw))[..., :3].mean() * (first + spp) / spp
        a = [block(k * spp) for k in range(blocks)]
        b = [block((blocks + k) * spp, medium_grid=False) for k in range(blocks)]
        a, b = np.array(a), np.array(b)
        z = (a.mean() - b.mean()) / np.sqrt(a.var(ddof=1) / blocks + b.var(ddof=1) / blocks)
        assert abs(z) < 4.5, z
    finally:
        sc.close()


def test_invalid_renders_and_grids_rejected(smoke):
    tris, nodes, eye, cam, med, grid, hdr, cache = smoke
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        sc.set_medium(**med)
        with pytest.raises(Exception):
            sc.render(_cfg(eye, cam))   # no grid set
        sc.set_medium_grid(grid)
        with pytest.raises(Exception):
            sc.render(_cfg(eye, cam, medium=False))   # the grid needs the medium
        before = sc.medium_grid().copy()
        for bad in (np.full((2, 2, 2), -1.0, np.float32), np.full((2, 2, 2), np.nan, np.float32), np.full((2, 2, 2), np.inf, np.float32),
                    np.zeros((1, 1, 1025), np.float32), np.full((2, 2, 2), 3e38, np.float32)):
            with pytest.raises(Exception):
                sc.set_medium_grid(bad)
            assert sc.medium_grid().tobytes() == before.tobytes()
        # a grid set before the medium: sigma_t times its largest density overflows, and both the render and the eval refuse it
        sc.set_medium(None)
        sc.set_medium_grid(np.full((2, 2, 2), 3e38, np.float32))
        sc.set_medium(**med)
        with pytest.raises(Exception):
            sc.render(_cfg(eye, cam))
        with pytest.raises(Exception):
            sc.medium_flight(np.zeros((1, 3)), np.array([[1.0, 0.0, 0.0]]), np.array([np.inf]), np.array([1], np.uint32))
        sc.set_medium_grid(None)
        with pytest.raises(Exception):
            sc.medium_grid()
    finally:
        sc.close()


# ---------------------------------------------------------------- renders against the CPU restatement, bit for bit and ray for ray
from tests import oracle_medium  # noqa: E402
from tests.test_gpu_emission_maps import _maps, _scene  # noqa: E402

SMOKE = dict(sigma_t=6.0, albedo=(0.9, 0.9, 0.9), g=0.3, box_min=(-1.0, -1.0, -1.0), box_max=(1.0, 1.2, 1.0))


@pytest.fixture(scope="module")
def mapped():
    tris, nodes, eye, cam, tex, uv, ids, eid = scenes.s_p3_bunny_emission_mapped()
    tris = np.asarray(tris, np.float32).reshape(-1, 36)
    hdr = scenes.synth_hdr(64, 32)
    return tris, nodes, eye, cam, tex, uv, ids, eid, hdr, api.hdr_cache(hdr), scenes.smoke_grid(32, 0)


def _crays(c):
    return c["rays_primary"], c["rays_bounce"], c["rays_shadow"]


@pytest.mark.parametrize("bounces", [1, 4, 8])
@pytest.mark.parametrize("env", ["none", "map", "env_light"])
@pytest.mark.parametrize("lens", [False, True])
def test_p3_smoke_equals_the_restatement(smoke, bounces, env, lens):
    tris, nodes, eye, cam, med, grid, hdr, cache = smoke
    h, c_ = (hdr, cache) if env != "none" else (None, None)
    kw = dict(max_bounce=bounces, env_light=(env == "env_light"))
    if lens:
        kw.update(lens_radius=0.15, focus_distance=3.6)
    cfg = _cfg(eye, cam, **kw)
    sc = api.Scene(tris, nodes, h, c_, device=0)
    try:
        sc.set_medium(**med)
        sc.set_medium_grid(grid)
        got = sc.render(cfg)
        gc = _rays(sc)
    finally:
        sc.close()
    ref, _, _, c = og.render(tris, nodes, cfg, grid, m=oracle_medium.medium(**med), hdr=h, hdr_cache=c_)
    assert got.tobytes() == ref.tobytes(), "L-inf %.3g" % float(np.abs(got - ref).max())
    assert gc == _crays(c)


OPTS = {
    "textures": dict(textures=True), "maps": dict(textures=True, material_maps=True, env_light=True), "emap": dict(textures=True, emission_maps=True),
    "punct": dict(punctual_lights=True), "punct_emap_tree": dict(punctual_lights=True, textures=True, emission_maps=True, light_tree=True),
    "tree": dict(light_tree=True, env_light=True), "lens_emap": dict(textures=True, emission_maps=True, lens_radius=0.15, focus_distance=3.6),
    "reference": dict(traverse=api.TRAVERSE_REFERENCE, env_light=True), "pruned": dict(traverse=api.TRAVERSE_PRUNED, textures=True, emission_maps=True),
    "batch1": dict(frames_per_batch=1, spp=3), "batch3": dict(frames_per_batch=3, spp=5), "resume": dict(first_frame=2),
    "parts": dict(part_count=2, part_rank=1), "profile2": dict(profile=2), "dense": dict(), "g_back": dict(), "g_fwd": dict(),
}


@pytest.mark.parametrize("opt", sorted(OPTS))
def test_p3_options_equal_the_restatement(mapped, opt):
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache, grid = mapped
    kw = dict(OPTS[opt])
    med = dict(SMOKE, sigma_t=400.0) if opt == "dense" else dict(SMOKE, g=-0.999) if opt == "g_back" else dict(SMOKE, g=0.999) if opt == "g_fwd" else SMOKE
    mr = nm = None
    if kw.get("material_maps"):
        tex, mr, nm = _maps(tex, ids)
    rig = scenes.punctual_rig(tris, seed=1, power=0.5) if kw.get("punctual_lights") else None
    cfg = _cfg(eye, cam, **kw)
    sc = _scene(tris, nodes, tex, uv, ids, eid, hdr, cache, mr=mr, nm=nm, lights=rig)
    try:
        sc.set_medium(**med)
        sc.set_medium_grid(grid)
        if cfg.first_frame:   # a resumed frame: the first frames from the device, then the rest on top
            fb = sc.render(_cfg(eye, cam, spp=2, **{k: v for k, v in kw.items() if k != "first_frame"}))
            got = sc.render(cfg, framebuffer=fb)
        else:
            got = sc.render(cfg)
        gc = _rays(sc)
    finally:
        sc.close()
    full = _cfg(eye, cam, **{k: v for k, v in kw.items() if k not in ("part_count", "part_rank", "first_frame")})
    if cfg.first_frame:
        full.spp = cfg.first_frame + cfg.spp
    ref, _, _, c = og.render(tris, nodes, full, grid, emission_id=eid, lights=rig, m=oracle_medium.medium(**med), textures=tex, texcoords=uv,
                             texture_id=ids, metal_rough_id=mr, normal_id=nm, hdr=hdr, hdr_cache=cache)
    if cfg.part_count > 1:
        want = np.zeros_like(ref)
        api.partition_scatter_host(got, want, cfg.width, cfg.height, cfg.out_channels, cfg.part_rank, cfg.part_count)
        mask = np.zeros((cfg.height, cfg.width, 1), np.float32)
        api.partition_scatter_host(np.ones((got.shape[0], 1), np.float32), mask, cfg.width, cfg.height, 1, cfg.part_rank, cfg.part_count)
        m = mask[..., 0] > 0
        assert m.any() and want[m].tobytes() == ref[m].tobytes()
        return
    assert got.tobytes() == ref.tobytes(), "L-inf %.3g" % float(np.abs(got - ref).max())
    if not cfg.first_frame:
        assert gc == _crays(c)


@pytest.mark.parametrize("opt", ["plain", "emap_tree"])
def test_p3_aov_and_adaptive_equal_the_restatement(mapped, opt):
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache, grid = mapped
    kw = dict(plain=dict(env_light=True), emap_tree=dict(env_light=True, textures=True, emission_maps=True, light_tree=True))[opt]
    m = oracle_medium.medium(**SMOKE)
    targs = dict(textures=tex, texcoords=uv, texture_id=ids)
    sc = _scene(tris, nodes, tex, uv, ids, eid, hdr, cache)
    try:
        sc.set_medium(**SMOKE)
        sc.set_medium_grid(grid)
        cfg = _cfg(eye, cam, spp=3, **kw)
        got, gaov, _ = sc.render_aov(cfg)
        ref, _, raov, c = og.render(tris, nodes, cfg, grid, emission_id=eid, m=m, hdr=hdr, hdr_cache=cache, aov=True, **targs)
        assert got.tobytes() == ref.tobytes() and gaov.tobytes() == raov.tobytes()
        assert sc.counters().rays == c["rays"]
        acfg = _cfg(eye, cam, spp=6, **kw)
        img, spp, luma2 = sc.render_adaptive(acfg, 0.3, 2, 2)
        ac = sc.counters()
        rimg, rspp, rluma2, rc = og.render_adaptive(tris, nodes, acfg, grid, 0.3, 2, 2, emission_id=eid, m=m, hdr=hdr, hdr_cache=cache, **targs)
        assert img.tobytes() == rimg.tobytes() and luma2.tobytes() == rluma2.tobytes() and np.array_equal(spp, rspp)
        assert ac.rays == rc["rays"]
    finally:
        sc.close()


def test_w8_scene_with_a_large_box_equals_the_restatement(monkeypatch):
    """a small scene forced onto the 8-wide tree, a box larger than the scene: deferred rays and the LIST pass carry the grid too"""
    monkeypatch.setenv("EZRT_ACCEL", "8")
    tris, nodes, eye, cam = scenes.s_lamps(3, 2, rough=True)
    tris = np.asarray(tris, np.float32).reshape(-1, 36)
    med = dict(sigma_t=1.5, albedo=(0.8, 0.8, 0.8), g=0.2, box_min=(-20.0, -5.0, -20.0), box_max=(20.0, 15.0, 20.0))
    grid = scenes.smoke_grid(40, 2)
    cfg = _cfg(eye, cam, spp=2, max_bounce=4)
    sc = api.Scene(tris, nodes, device=0)
    try:
        sc.set_medium(**med)
        sc.set_medium_grid(grid)
        got, gc = sc.render(cfg), _rays(sc)
    finally:
        sc.close()
    ref, _, _, c = og.render(tris, nodes, cfg, grid, m=oracle_medium.medium(**med))
    assert got.tobytes() == ref.tobytes() and gc == _crays(c)


def test_s1m_smoke_windows_at_1920x1080():
    tris, nodes, eye, cam, med, grid = scenes.s_1m_smoke(n=64)
    cfg = api.RenderConfig(width=1920, height=1080, spp=1, max_bounce=3, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam),
                           medium=True, medium_grid=True)
    sc = api.Scene(tris, nodes, device=0)
    try:
        sc.set_medium(**med)
        sc.set_medium_grid(grid)
        img = sc.render(cfg)
    finally:
        sc.close()
    for x0, y0 in ((896, 512), (320, 208)):   # tile-aligned 32x32 windows
        ref = og.render(tris, nodes, cfg, grid, m=oracle_medium.medium(**med), window=(x0, y0, x0 + 32, y0 + 32))[0]
        assert img[y0:y0 + 32, x0:x0 + 32].tobytes() == ref.tobytes()
