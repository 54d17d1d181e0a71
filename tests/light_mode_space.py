"""A model of how a render of the light sampling mode (mode 4, EZRT_MODE_DISNEY_LIGHTS) picks its kernels, in plain Python, and the
scene that exercises every kernel it can pick.  TEST INFRASTRUCTURE for tests/test_light_mode_space.py (the model against the library's
binary, coverage, power) and tests/test_gpu_light_mode_space.py (every instantiation against the restatement on the device).

The model restates, from the sources:
  - validate_params' constraints on mode 4's flags (capi.cu);
  - light_options (capi.cu), which turns the render's flags and the scene's state into the options the kernels are chosen by, and
    switches an option off where the scene gives it nothing to do;
  - launch_shade_t (kernels.cu) and the launchers of its families (kernels_ltree.cu, kernels_grid[_ltree].cu, kernels_vol[_ltree].cu,
    kernels_vol_medium[_ltree].cu), and launch_nee (kernels.cu, kernels_grid.cu, kernels_vol.cu);
  - the wavefront loop (render_device_impl): k_shade at every bounce (LIST = true too on the deferred lane, A = true at bounce 0 of a
    feature-buffer render), k_nee after every bounce but the last.

A k_shade key is its template arguments (MODE, LIST, A, E, T, X, TX, MP, P, EM, LTREE, GRID, VOL), a k_nee key its (MODE, E, T, X, TX,
MP, P, EM, GRID), as the demangled kernel names spell them."""
import functools
import itertools

import numpy as np

L4 = 4   # EZRT_MODE_DISNEY_LIGHTS

# the render flags of mode 4 that choose kernels (RenderConfig's names); the thin lens chooses none
FLAGS = ("env_light", "transmission", "medium", "textures", "material_maps", "punctual_lights", "emission_maps", "light_tree",
         "medium_grid", "volumes")
# flag -> the flags it needs (validate_params)
NEEDS = {"volumes": ("transmission",), "medium_grid": ("medium",), "material_maps": ("textures",), "emission_maps": ("textures",)}

FAMILIES = ("kernels", "ltree", "grid", "grid_ltree", "vol", "vol_ltree", "vol_medium", "vol_medium_ltree")

# the counts of mode-4 instantiations the library compiles (instantiations() and the binary must agree)
N_SHADE = 1120            # 560 without LIST, each with LIST = false and true
N_SHADE_BY_FAMILY = {"kernels": 240, "ltree": 240, "grid": 80, "grid_ltree": 80, "vol": 80, "vol_ltree": 80, "vol_medium": 160,
                     "vol_medium_ltree": 160}
N_NEE = 120               # 60 in kernels.cu, 20 in kernels_grid.cu, 40 in kernels_vol_medium.cu


def valid(flags):
    """validate_params on a set of mode-4 flags (the scene holds everything a flag needs): a medium with transmission needs the volumes"""
    f = set(flags)
    if not f <= set(FLAGS):
        return False
    if any(n in f and not set(need) <= f for n, need in NEEDS.items()):
        return False
    return not ("medium" in f and "transmission" in f and "volumes" not in f)


def closure_off(flags, flag):
    """flags with `flag` switched off, together with every flag that needs it (and the volumes when the medium would otherwise stand
    beside transmission without them: switching the volumes off switches the medium off with them)"""
    f = set(flags) - {flag}
    changed = True
    while changed:
        changed = False
        for n, need in NEEDS.items():
            if n in f and not set(need) <= f:
                f.discard(n)
                changed = True
        if "medium" in f and "transmission" in f and "volumes" not in f:
            f -= {"medium", "medium_grid"}
            changed = True
    assert valid(f), (flags, flag, f)
    return frozenset(f)


class SceneState:
    """What light_options reads of the scene: a map (hence an environment table), the medium's sigma_t > 0, J punctual lights, the
    light table's K (and the emission table's K_emit), and whether volumes are set"""

    def __init__(self, env_table=True, sigma_t=True, J=1, K=1, K_emit=None, volumes=True):
        self.env_table, self.sigma_t, self.J, self.K = bool(env_table), bool(sigma_t), int(J), int(K)
        self.K_emit = self.K if K_emit is None else int(K_emit)
        self.volumes = bool(volumes)


FULL = SceneState()


def light_options(flags, s=FULL):
    """capi.cu light_options: the option bools the kernels are chosen by, and P_env, P_p (None where the option is off)"""
    f = set(flags)
    assert valid(f), f
    o = dict(env=False, trans=False, medium=False, grid=False, vol=False, tex=False, maps=False, punct=False, emap=False, tree=False,
             p_env=None, p_p=None)
    n_lights = s.K
    if "emission_maps" in f:
        n_lights = s.K_emit
        o["emap"] = True
    if "env_light" in f and s.env_table:
        o["env"] = True
        o["p_env"] = 0.5 if n_lights > 0 else 1.0
    o["trans"] = "transmission" in f
    if "medium" in f and s.sigma_t:
        o["medium"] = True
        o["grid"] = "medium_grid" in f
    if "volumes" in f and (s.volumes or o["medium"]):
        o["vol"] = True
    if "textures" in f:
        o["tex"] = True
        o["maps"] = "material_maps" in f
    if "punctual_lights" in f and s.J > 0:
        o["punct"] = True
        o["p_p"] = 0.5 if (n_lights > 0 or o["env"]) else 1.0
    if "light_tree" in f and n_lights > 0:
        o["tree"] = True
    return o


def shade_key(o, LIST, A):
    """launch_shade_t's k_shade for the options o: (family, key)"""
    b = lambda k: bool(o[k])
    if o["vol"]:   # kernels_vol[_medium][_ltree].cu: T = true; X = the medium; GRID = the grid with the medium
        fam = ("vol_medium" if o["medium"] else "vol") + ("_ltree" if o["tree"] else "")
        key = (L4, LIST, A, b("env"), True, b("medium"), b("tex"), b("maps"), b("punct"), b("emap"), b("tree"), b("grid") and b("medium"), True)
    elif o["grid"]:   # kernels_grid[_ltree].cu: T = false, X = true
        fam = "grid_ltree" if o["tree"] else "grid"
        key = (L4, LIST, A, b("env"), False, True, b("tex"), b("maps"), b("punct"), b("emap"), b("tree"), True, False)
    else:   # kernels_ltree.cu or kernels.cu
        fam = "ltree" if o["tree"] else "kernels"
        key = (L4, LIST, A, b("env"), b("trans"), b("medium"), b("tex"), b("maps"), b("punct"), b("emap"), b("tree"), False, False)
    return fam, key


def nee_key(o):
    """launch_nee's k_nee for the options o: (family, key)"""
    b = lambda k: bool(o[k])
    if o["trans"] and o["medium"]:   # kernels_vol_medium.cu
        return "vol_medium", (L4, b("env"), True, True, b("tex"), b("maps"), b("punct"), b("emap"), b("grid"))
    if o["grid"]:   # kernels_grid.cu
        return "grid", (L4, b("env"), False, True, b("tex"), b("maps"), b("punct"), b("emap"), True)
    return "kernels", (L4, b("env"), b("trans"), b("medium"), b("tex"), b("maps"), b("punct"), b("emap"), False)


def predict(flags, scene_state=FULL, aov=False, max_bounce=1, lane=True):
    """({k_shade keys}, {k_nee keys}) that one wavefront render of mode 4 launches: k_shade at bounces 0..max_bounce (A only at bounce 0
    of a feature-buffer render; LIST = true beside it when the accel policy's deferred lane is on), k_nee after bounces 0..max_bounce-1"""
    o = light_options(flags, scene_state)
    shade, nee = set(), set()
    for b in range(max_bounce + 1):
        for LIST in ((False, True) if lane else (False,)):
            shade.add(shade_key(o, LIST, bool(aov) and b == 0)[1])
        if b < max_bounce:
            nee.add(nee_key(o)[1])
    return shade, nee


def _bools(n):
    return itertools.product((False, True), repeat=n)


def _maps_ok(TX, MP, EM):   # the maps with the textures
    return (TX or not MP) and (TX or not EM)


def instantiations():
    """({family: {k_shade keys}}, {family: {k_nee keys}}) of mode 4 as the launchers' with_bools and if-constexpr masks are written"""
    shade = {f: set() for f in FAMILIES}
    nee = {"kernels": set(), "grid": set(), "vol_medium": set()}
    for LIST in (False, True):
        for A, E, T, X, TX, MP, P, EM in _bools(8):   # kernels.cu / kernels_ltree.cu: !(T && X)
            if not (T and X) and _maps_ok(TX, MP, EM):
                shade["kernels"].add((L4, LIST, A, E, T, X, TX, MP, P, EM, False, False, False))
                shade["ltree"].add((L4, LIST, A, E, T, X, TX, MP, P, EM, True, False, False))
        for A, E, TX, MP, P, EM in _bools(6):
            if _maps_ok(TX, MP, EM):
                for LT in (False, True):
                    shade["grid_ltree" if LT else "grid"].add((L4, LIST, A, E, False, True, TX, MP, P, EM, LT, True, False))
                    shade["vol_ltree" if LT else "vol"].add((L4, LIST, A, E, True, False, TX, MP, P, EM, LT, False, True))
                    for G in (False, True):
                        shade["vol_medium_ltree" if LT else "vol_medium"].add((L4, LIST, A, E, True, True, TX, MP, P, EM, LT, G, True))
    for E, T, X, TX, MP, P, EM in _bools(7):
        if not (T and X) and _maps_ok(TX, MP, EM):
            nee["kernels"].add((L4, E, T, X, TX, MP, P, EM, False))
    for E, TX, MP, P, EM in _bools(5):
        if _maps_ok(TX, MP, EM):
            nee["grid"].add((L4, E, False, True, TX, MP, P, EM, True))
            for G in (False, True):
                nee["vol_medium"].add((L4, E, True, True, TX, MP, P, EM, G))
    return shade, nee


def all_shade():
    return set().union(*instantiations()[0].values())


def all_nee():
    return set().union(*instantiations()[1].values())


def flags_of(key):
    """the flags whose render (FULL scene state) launches the k_shade key (LIST aside): the inverse of shade_key"""
    _, _, _, E, T, X, TX, MP, P, EM, LT, G, V = key
    f = {n for n, on in (("env_light", E), ("transmission", T), ("medium", X), ("textures", TX), ("material_maps", MP),
                         ("punctual_lights", P), ("emission_maps", EM), ("light_tree", LT), ("medium_grid", G), ("volumes", V)) if on}
    return frozenset(f)


def family_of(key):
    o = light_options(flags_of(key))
    return shade_key(o, key[1], key[2])[0]


@functools.lru_cache(maxsize=None)
def row_keys():
    """the 560 (A, family, bools) keys: every mode-4 k_shade instantiation without LIST, in a fixed order"""
    keys = sorted({k[:1] + (False,) + k[2:] for k in all_shade()}, key=lambda k: (FAMILIES.index(family_of(k)), k))
    return tuple(keys)


# ------------------------------------------------------------------ the binary
def parse_template_args(s):
    """'(int)4, true, false' -> (4, True, False)"""
    import re
    out = []
    for a in s.split(","):
        a = re.sub(r"^\(\w+\)", "", a.strip())
        out.append(True if a == "true" else False if a == "false" else int(a.rstrip("uU")))
    return tuple(out)


def kernel_keys(names):
    """({k_shade keys of mode 4}, {k_nee keys of mode 4}) among demangled kernel names ('void k_shade<4, true, ...>(...)')"""
    import re
    shade, nee = set(), set()
    for n in names:
        m = re.search(r"\bk_(shade|nee)<([^<>]*)>", n)
        if not m:
            continue
        k = parse_template_args(m.group(2))
        if k[0] != L4:
            continue
        (shade if m.group(1) == "shade" else nee).add(k)
    return shade, nee


# ------------------------------------------------------------------ the scene
# fog over the blob and the floor under it (volume_scenes.FOG), and the same box with a denser sigma_t for the density grid
def _fog():
    from tests import volume_scenes as vs
    return dict(vs.FOG), dict(vs.FOG, sigma_t=4.0)


def medium_for(flags):
    """the medium (Scene.set_medium's keywords) a render with these flags is given: the denser one beside the grid"""
    fog, smoke = _fog()
    return smoke if "medium_grid" in flags else fog


DUP_EVERY = 8   # one non-emissive triangle in DUP_EVERY is duplicated exactly


@functools.lru_cache(maxsize=None)
def space_scene(emitters=True, soup=False):
    """The scene of the light mode space: tests/test_volumes_oracle.blob_scene (the P3 floor, an amber glass blob, the mapped emissive
    sphere, seeded textures) with the material maps of tests/test_gpu_emission_maps._maps, scenes.punctual_rig, the fog box over the
    blob and the floor, scenes.smoke_grid and an HDR map.  One non-emissive triangle in DUP_EVERY (floor and blob) is appended again,
    bit for bit: the two tie at every hit, which the accel policy defers to the exact pass in the camera and the bounce passes.
    emitters=False: the sphere's emission set to 0 (K = 0).  soup=True: 2 N tiny unconnected triangles far outside the scene, so that
    the 8-wide tree keeps flat (not indexed) triangle records.  The tree is rebuilt; every per-triangle array follows the new order.
    Returns a dict of the arrays both the library and the restatement take."""
    from ezrt_b200 import api, scenes
    from tests.test_gpu_emission_maps import _maps
    from tests import volume_scenes as vs
    from tests.test_volumes_oracle import blob_scene
    tris, _, eye, cam, tex, uv, ids, eid = blob_scene()
    tris = np.array(tris, np.float32, copy=True)
    n = tris.shape[0]
    vid = np.where(tris[:, 35] > 0, 0, -1).astype(np.int32)
    emissive = (tris[:, 18:21] > 0).any(axis=1)
    cand = np.flatnonzero(~emissive)
    dup = cand[3::DUP_EVERY]
    src = np.concatenate([np.arange(n), dup])
    all_tris = tris[src]
    if not emitters:
        all_tris[:, 18:21] = 0.0
    if soup:
        rng = np.random.default_rng(11)
        m = 2 * len(src)
        c = rng.normal(size=(m, 3))
        c = c / np.linalg.norm(c, axis=1, keepdims=True) * rng.uniform(40.0, 60.0, (m, 1))
        v = c[:, None, :] + rng.uniform(-0.02, 0.02, (m, 3, 3))
        st = np.zeros((m, 36), np.float32)
        st[:] = all_tris[cand[0]]   # a floor triangle's material, moved
        st[:, 0:9] = v.reshape(m, 9)
        e1, e2 = v[:, 1] - v[:, 0], v[:, 2] - v[:, 0]
        nrm = np.cross(e1, e2)
        nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        st[:, 9:18] = np.repeat(nrm, 3, axis=0).reshape(m, 9)
        all_tris = np.concatenate([all_tris, st.astype(np.float32)])
        src = np.concatenate([src, np.full(m, -1)])
    tl = api.TriangleList()
    tl.append_encoded(all_tris)
    out, nodes = tl.build_bvh(8)
    out = np.asarray(out, np.float32).reshape(-1, 36)
    # the new order: each output record is an input record, bit for bit (a duplicate and its original carry the same attributes)
    where = {all_tris[i].tobytes(): src[i] for i in range(len(src))}
    perm = np.array([where[r.tobytes()] for r in out])
    soup_rows = perm < 0
    take = np.where(soup_rows, 0, perm)

    def follow(a, fill):
        a = np.asarray(a)[take].copy()
        a[soup_rows] = fill
        return a
    tex_all, mr, nm = _maps(list(tex), ids)
    hdr = scenes.synth_hdr(64, 32)
    return dict(tris=out, nodes=nodes, eye=eye, cam=cam, textures=tex_all, texcoords=follow(uv, 0.0), texture_id=follow(ids, -1),
                metal_rough_id=follow(mr, -1), normal_id=follow(nm, -1), emission_id=follow(eid, -1), volume_id=follow(vid, -1),
                volumes=[vs.AMBER], lights=scenes.punctual_rig(out[~soup_rows], seed=1, power=0.5), rho=scenes.smoke_grid(16, 1),
                hdr=hdr, hdr_cache=api.hdr_cache(hdr), n_dup=len(dup), n_soup=int(soup_rows.sum()))


def oracle_kwargs(sd, flags, env=True, punct=True, volumes=True, sigma_t=None, hdr_linear=True):
    """the keyword arguments of tests/oracle_volumes.render for the scene dict sd rendered with these flags: each option's data is
    passed where the flag asks for it, as the library's scene holds it (env=False: no map; punct=False: J = 0; volumes=False: none;
    sigma_t: the medium's extinction instead of medium_for's)"""
    from tests import oracle_medium
    kw = dict(emission_id=sd["emission_id"], textures=sd["textures"], texcoords=sd["texcoords"], texture_id=sd["texture_id"])
    if env:
        kw.update(hdr=sd["hdr"], hdr_cache=sd["hdr_cache"], hdr_linear=hdr_linear)
    if "material_maps" in flags:
        kw.update(metal_rough_id=sd["metal_rough_id"], normal_id=sd["normal_id"])
    if "punctual_lights" in flags:
        kw["lights"] = sd["lights"] if punct else []
    if "medium" in flags:
        med = dict(medium_for(flags))
        if sigma_t is not None:
            med["sigma_t"] = sigma_t
        kw["m"] = oracle_medium.medium(**med)
        if "medium_grid" in flags:
            kw["rho"] = sd["rho"]
    if "volumes" in flags and volumes:
        kw.update(volumes=sd["volumes"], volume_id=sd["volume_id"])
    return kw


def config(sd, flags, **kw):
    """a RenderConfig of mode 4 with these flags over the scene dict sd: 32 x 24, 2 spp, 3 bounces unless kw says otherwise"""
    from ezrt_b200 import api
    base = dict(width=32, height=24, spp=2, max_bounce=3, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(sd["eye"]), camera_rotate=tuple(sd["cam"]),
                env_color=(0.3, 0.35, 0.4))
    base.update({f: True for f in flags})
    base.update(kw)
    return api.RenderConfig(**base)
