"""GPU renders with volumes inside transmissive meshes (EZRT_PARAM_VOLUMES, DESIGN.md section 21): glTF's attenuation colour and
distance absorbing along every interior segment, and glass inside the homogeneous medium and the density grid, displacing it.

Whole renders are held bit for bit, with equal primary, bounce and shadow ray counts, to the CPU restatement (tests/oracle_volumes.cpp)
under every option of the light sampling mode, policy, batch size and form; the identities with the renders without absorption; the
device's sigma_a table against the host conversion; set_volumes' validation; the rejections."""
import numpy as np
import pytest

from ezrt_b200 import api, scenes
from ezrt_b200._lib import EzrtError
from tests import oracle_medium
from tests import oracle_volumes as ov
from tests import volume_scenes as vs
from tests.test_gpu_emission_maps import FOG, _maps
from tests.test_volumes_oracle import blob_scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def p3():
    hdr = scenes.synth_hdr(64, 32)
    return blob_scene() + (hdr, api.hdr_cache(hdr))


def _cfg(eye, cam, **kw):
    base = dict(width=48, height=32, spp=2, max_bounce=4, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye), camera_rotate=tuple(cam), transmission=True,
                volumes=True)
    base.update(kw)
    return api.RenderConfig(**base)


def _rays(c):
    return (c.primary_rays, c.bounce_rays, c.shadow_rays)


def _crays(c):
    return (c["rays_primary"], c["rays_bounce"], c["rays_shadow"])


def _ids(tris):
    return np.where(tris[:, 35] > 0, 0, -1).astype(np.int32)


@pytest.mark.parametrize("lens", [False, True])
@pytest.mark.parametrize("light", ["none", "map", "env"])
@pytest.mark.parametrize("bounces", [1, 4, 8])
def test_coloured_blob_equals_the_restatement(bounces, light, lens):
    tris, nodes, eye, cam, vols, vid = vs.p3_coloured_glass(0.3)
    hdr = None if light == "none" else scenes.synth_hdr(64, 32)
    cache = None if hdr is None else api.hdr_cache(hdr)
    kw = dict(max_bounce=bounces, env_light=(light == "env"))
    if lens:
        kw.update(lens_radius=0.1, focus_distance=3.5)
    cfg = _cfg(eye, cam, **kw)
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        sc.set_volumes(vols, vid)
        got, gc = sc.render(cfg), sc.counters()
    finally:
        sc.close()
    ref, _, _, c = ov.render(tris, nodes, cfg, volumes=vols, volume_id=vid, hdr=hdr, hdr_cache=cache)
    assert got.tobytes() == ref.tobytes(), "L-inf %.3g" % float(np.abs(got - ref).max())
    assert _rays(gc) == _crays(c)


OPTS = {
    "plain": dict(), "env": dict(env_light=True), "textures": dict(textures=True), "maps": dict(textures=True, material_maps=True, env_light=True),
    "emap": dict(textures=True, emission_maps=True), "punct": dict(punctual_lights=True, env_light=True), "tree": dict(light_tree=True, env_light=True),
    "tree_emap_punct": dict(light_tree=True, textures=True, emission_maps=True, punctual_lights=True),
    "lens": dict(lens_radius=0.12, focus_distance=3.6, env_light=True),
    "reference": dict(traverse=api.TRAVERSE_REFERENCE, env_light=True), "pruned": dict(traverse=api.TRAVERSE_PRUNED, textures=True, emission_maps=True),
    "batch1": dict(frames_per_batch=1, spp=3), "batch3": dict(frames_per_batch=3, spp=5), "resume": dict(first_frame=2),
    "parts": dict(part_count=2, part_rank=1), "profile2": dict(profile=2),
}


def _scene(p3, kw):
    tris, nodes, eye, cam, tex, uv, ids, eid, hdr, cache = p3
    rk = dict(hdr=hdr, hdr_cache=cache, emission_id=eid, textures=tex, texcoords=uv, texture_id=ids)
    if kw.get("material_maps"):
        rk["textures"], rk["metal_rough_id"], rk["normal_id"] = _maps(tex, ids)
    if kw.get("punctual_lights"):
        rk["lights"] = scenes.punctual_rig(tris, seed=1, power=0.5)
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    sc.set_textures(rk["textures"], uv, ids)
    if "metal_rough_id" in rk:
        sc.set_material_maps(rk["metal_rough_id"], rk["normal_id"])
    if "lights" in rk:
        sc.set_punctual_lights(rk["lights"])
    sc.set_emission_maps(eid)
    return sc, rk


@pytest.mark.parametrize("opt", sorted(OPTS))
def test_options_equal_the_restatement(p3, opt):
    tris, nodes, eye, cam = p3[:4]
    kw = dict(OPTS[opt])
    vk = dict(volumes=[vs.AMBER], volume_id=_ids(tris))
    cfg = _cfg(eye, cam, **kw)
    sc, rk = _scene(p3, kw)
    try:
        sc.set_volumes(**vk)
        if cfg.first_frame:   # a resumed frame: the first frames from the device, then the rest on top
            fb = sc.render(_cfg(eye, cam, spp=2, **{k: v for k, v in kw.items() if k != "first_frame"}))
            got = sc.render(cfg, framebuffer=fb)
        else:
            got = sc.render(cfg)
        gc = sc.counters()
    finally:
        sc.close()
    full = _cfg(eye, cam, **{k: v for k, v in kw.items() if k not in ("part_count", "part_rank", "first_frame")})
    if cfg.first_frame:
        full.spp = cfg.first_frame + cfg.spp
    ref, _, _, c = ov.render(tris, nodes, full, **vk, **rk)
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
        assert _rays(gc) == _crays(c)


@pytest.mark.parametrize("opt", ["env", "tree_emap_punct"])
def test_aov_and_adaptive_equal_the_restatement(p3, opt):
    tris, nodes, eye, cam = p3[:4]
    kw = dict(OPTS[opt])
    vk = dict(volumes=[vs.AMBER], volume_id=_ids(tris))
    sc, rk = _scene(p3, kw)
    try:
        sc.set_volumes(**vk)
        cfg = _cfg(eye, cam, spp=3, **kw)
        got, gaov, _ = sc.render_aov(cfg)
        ref, _, raov, c = ov.render(tris, nodes, cfg, aov=True, **vk, **rk)
        assert got.tobytes() == ref.tobytes() and gaov.tobytes() == raov.tobytes()
        assert sc.counters().rays == c["rays"]
        acfg = _cfg(eye, cam, spp=6, **kw)
        img, spp, luma2 = sc.render_adaptive(acfg, 0.3, 2, 2)
        ac = sc.counters()
        rimg, rspp, rluma2, rc = ov.render_adaptive(tris, nodes, acfg, 0.3, 2, 2, **vk, **rk)
        assert img.tobytes() == rimg.tobytes() and luma2.tobytes() == rluma2.tobytes() and np.array_equal(spp, rspp)
        assert ac.rays == rc["rays"]
        # every tile of an adaptive render is the plain render at its own sample count
        for n in np.unique(spp):
            plain = sc.render(_cfg(eye, cam, spp=int(n), **kw))
            m = spp == n
            assert img[m].tobytes() == plain[m].tobytes()
    finally:
        sc.close()


@pytest.mark.parametrize("opt", ["plain", "env", "tree_emap_punct", "lens"])
def test_clear_volumes_give_the_transmission_render(p3, opt):
    """on the device: the flag without volumes, with every id -1, with white colours and with infinite distances"""
    tris, nodes, eye, cam = p3[:4]
    kw = dict(OPTS[opt])
    n = tris.shape[0]
    sc, rk = _scene(p3, kw)
    try:
        want = sc.render(_cfg(eye, cam, volumes=False, **kw))
        wc = _rays(sc.counters())
        assert sc.render(_cfg(eye, cam, **kw)).tobytes() == want.tobytes()
        for vols, vid in (([vs.AMBER], np.full(n, -1, np.int32)), ([api.volume((1, 1, 1), 0.01)], _ids(tris)),
                          ([api.volume((0.0, 0.3, 0.9), np.inf)], _ids(tris))):
            sc.set_volumes(vols, vid)
            got = sc.render(_cfg(eye, cam, **kw))
            assert got.tobytes() == want.tobytes() and _rays(sc.counters()) == wc
        sc.set_volumes([vs.AMBER], _ids(tris))
        absorbed = sc.render(_cfg(eye, cam, **kw))
        assert _rays(sc.counters()) == wc and absorbed.tobytes() != want.tobytes()
    finally:
        sc.close()


def test_s1m_glass_grid_windows_at_1920x1080():
    tris, nodes, eye, cam, vols, vid = vs.grid_coloured_glass(15, 13)
    sc = api.Scene(tris, nodes, device=0)
    try:
        sc.set_volumes(vols, vid)
        out = {}
        for b in (1, 4, 8):
            cfg = _cfg(eye, cam, width=1920, height=1080, spp=1, max_bounce=b)
            out[b] = (cfg, sc.render(cfg))
    finally:
        sc.close()
    for b, (cfg, img) in out.items():
        for win in ((0, 0, 48, 32), (928, 528, 976, 560), (1872, 1040, 1920, 1080)):
            ref, _, _, _ = ov.render(tris, nodes, cfg, volumes=vols, volume_id=vid, window=win)
            x0, y0, x1, y1 = win
            assert img[y0:y1, x0:x1].tobytes() == ref.tobytes(), "S-1M glass grid, %d bounces, window %r" % (b, win)


def test_volume_table_and_validation(p3):
    tris, nodes, eye, cam = p3[:4]
    n = tris.shape[0]
    rng = np.random.default_rng(3)
    vols = [api.volume(tuple(rng.uniform(0, 1, 3)), float(d)) for d in np.exp(rng.uniform(-5, 5, 40))]
    vols += [api.volume((1, 0, 0.5), np.inf), api.volume((0, 0, 0), 1e-30), api.volume((1, 1, 1), 1e30)]
    sc = api.Scene(tris, nodes, device=0)
    try:
        assert sc.volume_table().shape == (0, 3)
        ids = rng.integers(-1, len(vols), n).astype(np.int32)
        sc.set_volumes(vols, ids)
        table = sc.volume_table()
        assert table.tobytes() == ov.table(vols).tobytes()
        cfg = _cfg(eye, cam)
        before = sc.render(cfg)
        bad = [
            ([api.volume((1.5, 0, 0), 1)], np.zeros(n, np.int32)), ([api.volume((-0.1, 0, 0), 1)], np.zeros(n, np.int32)),
            ([api.volume((np.nan, 0, 0), 1)], np.zeros(n, np.int32)), ([api.volume((0.5, 0.5, 0.5), 0)], np.zeros(n, np.int32)),
            ([api.volume((0.5, 0.5, 0.5), -1)], np.zeros(n, np.int32)), ([api.volume((0.5, 0.5, 0.5), np.nan)], np.zeros(n, np.int32)),
            ([api.volume((0.5, 0.5, 0.5), 1)], np.full(n, 1, np.int32)), ([api.volume((0.5, 0.5, 0.5), 1)], np.full(n, -2, np.int32)),
            ([], np.zeros(n, np.int32)),
        ]
        for v, i in bad:
            with pytest.raises(EzrtError):
                sc.set_volumes(v, i)
        r = api.volume((0.5, 0.5, 0.5), 1)
        r.reserved = 1
        with pytest.raises(EzrtError):
            sc.set_volumes([r], np.zeros(n, np.int32))
        with pytest.raises(EzrtError):
            sc.set_volumes([vs.AMBER], None)
        with pytest.raises(ValueError):
            sc.set_volumes([vs.AMBER], np.zeros(n + 1, np.int32))
        # the previous volumes are kept on every error
        assert sc.volume_table().tobytes() == table.tobytes()
        assert sc.render(cfg).tobytes() == before.tobytes()
        sc.set_volumes(None)
        assert sc.volume_table().shape == (0, 3)
        cfg.volumes = False
        assert sc.render(_cfg(eye, cam)).tobytes() == sc.render(cfg).tobytes()
    finally:
        sc.close()


def test_rejections(p3):
    tris, nodes, eye, cam = p3[:4]
    hdr, cache = p3[8], p3[9]
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        sc.set_volumes([vs.AMBER], _ids(tris))
        with pytest.raises(EzrtError):   # without transmission
            sc.render(_cfg(eye, cam, transmission=False))
        for mode in (api.MODE_DIFFUSE_P3, api.MODE_DISNEY_ANISO_P4, api.MODE_DISNEY_SOBOL_P5, api.MODE_DISNEY_IS_MIS_P5):
            with pytest.raises(EzrtError):
                sc.render(_cfg(eye, cam, mode=mode))
        with pytest.raises(EzrtError):
            sc.render(_cfg(eye, cam, pipeline=api.PIPELINE_MEGAKERNEL))
        sc.set_medium(**FOG)
        with pytest.raises(EzrtError):   # the medium beside transmission without the flag
            sc.render(_cfg(eye, cam, medium=True, volumes=False))
        assert np.isfinite(sc.render(_cfg(eye, cam, medium=True))).all()   # ... and with it
        with pytest.raises(EzrtError):   # the grid flag without a grid
            sc.render(_cfg(eye, cam, medium=True, medium_grid=True))
    finally:
        sc.close()


# ------------------------------------------------------------------ glass inside the medium
FOG_OPTS = {
    "plain": dict(), "env": dict(env_light=True), "lens": dict(lens_radius=0.12, focus_distance=3.6, env_light=True),
    "maps": dict(textures=True, material_maps=True, env_light=True), "emap": dict(textures=True, emission_maps=True),
    "punct": dict(punctual_lights=True, env_light=True), "tree_emap_punct": dict(light_tree=True, textures=True, emission_maps=True, punctual_lights=True),
    "reference": dict(traverse=api.TRAVERSE_REFERENCE, env_light=True), "pruned": dict(traverse=api.TRAVERSE_PRUNED),
    "batch1": dict(frames_per_batch=1, spp=3), "batch3": dict(frames_per_batch=3, spp=5), "profile2": dict(profile=2),
}


@pytest.mark.parametrize("grid", [False, True])
@pytest.mark.parametrize("opt", sorted(FOG_OPTS))
def test_glass_in_fog_equals_the_restatement(p3, opt, grid):
    tris, nodes, eye, cam = p3[:4]
    kw = dict(FOG_OPTS[opt])
    rho = scenes.smoke_grid(16, 1) if grid else None
    fog = dict(vs.FOG, sigma_t=4.0) if grid else vs.FOG
    vk = dict(volumes=[vs.AMBER], volume_id=_ids(tris))
    cfg = _cfg(eye, cam, medium=True, medium_grid=grid, **kw)
    sc, rk = _scene(p3, kw)
    try:
        sc.set_volumes(**vk)
        sc.set_medium(**fog)
        if grid:
            sc.set_medium_grid(rho)
        got, gc = sc.render(cfg), sc.counters()
    finally:
        sc.close()
    ref, _, _, c = ov.render(tris, nodes, cfg, m=oracle_medium.medium(**fog), rho=rho, **vk, **rk)
    assert got.tobytes() == ref.tobytes(), "L-inf %.3g" % float(np.abs(got - ref).max())
    assert _rays(gc) == _crays(c)


@pytest.mark.parametrize("bounces", [1, 4, 8])
@pytest.mark.parametrize("which", ["fog", "smoke"])
def test_coloured_blob_in_fog_equals_the_restatement(which, bounces):
    if which == "fog":
        tris, nodes, eye, cam, vols, vid, fog = vs.p3_glass_in_fog()
        rho = None
    else:
        tris, nodes, eye, cam, vols, vid, fog, rho = vs.p3_glass_in_smoke()
    hdr = scenes.synth_hdr(64, 32)
    cache = api.hdr_cache(hdr)
    cfg = _cfg(eye, cam, max_bounce=bounces, env_light=True, medium=True, medium_grid=rho is not None)
    sc = api.Scene(tris, nodes, hdr, cache, device=0)
    try:
        sc.set_volumes(vols, vid)
        sc.set_medium(**fog)
        if rho is not None:
            sc.set_medium_grid(rho)
        got, gc = sc.render(cfg), sc.counters()
        # the flag without volumes: clear glass displacing the fog, still the VOL kernels
        sc.set_volumes(None)
        clear = sc.render(cfg)
    finally:
        sc.close()
    kw = dict(m=oracle_medium.medium(**fog), rho=rho, hdr=hdr, hdr_cache=cache)
    ref, _, _, c = ov.render(tris, nodes, cfg, volumes=vols, volume_id=vid, **kw)
    assert got.tobytes() == ref.tobytes() and _rays(gc) == _crays(c)
    assert clear.tobytes() == ov.render(tris, nodes, cfg, **kw)[0].tobytes()


def test_glass_in_fog_aov_and_adaptive_equal_the_restatement(p3):
    tris, nodes, eye, cam = p3[:4]
    kw = dict(env_light=True, textures=True, emission_maps=True)
    vk = dict(volumes=[vs.AMBER], volume_id=_ids(tris))
    m = oracle_medium.medium(**vs.FOG)
    sc, rk = _scene(p3, kw)
    try:
        sc.set_volumes(**vk)
        sc.set_medium(**vs.FOG)
        cfg = _cfg(eye, cam, spp=3, medium=True, **kw)
        got, gaov, _ = sc.render_aov(cfg)
        ref, _, raov, c = ov.render(tris, nodes, cfg, aov=True, m=m, **vk, **rk)
        assert got.tobytes() == ref.tobytes() and gaov.tobytes() == raov.tobytes() and sc.counters().rays == c["rays"]
        acfg = _cfg(eye, cam, spp=6, medium=True, **kw)
        img, spp, luma2 = sc.render_adaptive(acfg, 0.3, 2, 2)
        rimg, rspp, rluma2, _ = ov.render_adaptive(tris, nodes, acfg, 0.3, 2, 2, m=m, **vk, **rk)
        assert img.tobytes() == rimg.tobytes() and luma2.tobytes() == rluma2.tobytes() and np.array_equal(spp, rspp)
    finally:
        sc.close()


@pytest.mark.parametrize("grid", [False, True])
def test_flag_beside_the_medium_without_glass_is_the_medium_render(p3, grid):
    """on the device: VOLUMES | TRANSMISSION | MEDIUM on a scene without transmissive material renders the MEDIUM render's bits and rays"""
    tris, nodes, eye, cam = p3[:4]
    opaque = np.array(tris, np.float32, copy=True)
    opaque[:, 35] = 0.0
    sc = api.Scene(opaque, nodes, p3[8], p3[9], device=0)
    try:
        sc.set_volumes([vs.AMBER], _ids(tris))
        sc.set_medium(**vs.FOG)
        if grid:
            sc.set_medium_grid(scenes.smoke_grid(16, 1))
        base = dict(env_light=True, medium=True, medium_grid=grid)
        want = sc.render(_cfg(eye, cam, transmission=False, volumes=False, **base))
        wc = _rays(sc.counters())
        got = sc.render(_cfg(eye, cam, **base))
        assert got.tobytes() == want.tobytes() and _rays(sc.counters()) == wc
    finally:
        sc.close()
