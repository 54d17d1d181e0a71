"""The light sampling mode's kernel dispatch (tests/light_mode_space.py) checked without a GPU.

- The model's mode-4 k_shade and k_nee instantiations equal the ones the library's binary holds, read with cuobjdump and cu++filt,
  and their counts are the ones stated here.
- The rows of tests/test_gpu_light_mode_space.py launch every instantiation, with LIST = false and true.
- Power: in every row, a kernel that dropped any option the row has on would render another image of the restatement, so no row can
  pass with a kernel that silently ignores one of its options.
- Each reduction of light_options (an option switched off where the scene gives it nothing to do) gives the restatement's bits
  of the render without that option."""
import os
import shutil
import subprocess

import pytest

from ezrt_b200 import build as _build
from tests import light_mode_space as lms
from tests import oracle_volumes as ov


# ------------------------------------------------------------------ the model alone
def test_instantiation_counts():
    shade, nee = lms.instantiations()
    assert {f: len(k) for f, k in shade.items()} == lms.N_SHADE_BY_FAMILY
    assert len(lms.all_shade()) == lms.N_SHADE == 1120
    assert len(lms.row_keys()) == 560
    assert {f: len(k) for f, k in nee.items()} == {"kernels": 60, "grid": 20, "vol_medium": 40}
    assert len(lms.all_nee()) == lms.N_NEE == 120
    # the families do not share an instantiation
    assert sum(len(k) for k in shade.values()) == len(lms.all_shade())


def test_every_key_is_launched_by_its_own_flags():
    """flags_of inverts the dispatch: a render with a key's flags (every option's data present) launches that key, from its family"""
    shade, _ = lms.instantiations()
    fam_of = {k: f for f, ks in shade.items() for k in ks}
    for key in lms.row_keys():
        flags = lms.flags_of(key)
        assert lms.valid(flags), key
        got, _ = lms.predict(flags, aov=key[2], max_bounce=1)
        assert key in got and key[:1] + (True,) + key[2:] in got
        assert fam_of[key] == lms.family_of(key)


def test_predicted_launches_are_instantiated():
    """every render of every valid flag set, scene state and form launches only kernels that exist"""
    shade, nee = lms.all_shade(), lms.all_nee()
    states = [lms.SceneState(env_table=e, sigma_t=s, J=j, K=k, volumes=v) for e in (0, 1) for s in (0, 1) for j in (0, 2) for k in (0, 5)
              for v in (0, 1)]
    n = 0
    for bits in range(1 << len(lms.FLAGS)):
        flags = frozenset(f for i, f in enumerate(lms.FLAGS) if bits >> i & 1)
        if not lms.valid(flags):
            continue
        for st in states:
            for aov in (False, True):
                s, k = lms.predict(flags, st, aov=aov, max_bounce=2)
                assert s <= shade and k <= nee, (flags, vars(st))
                n += 1
    assert n > 1000


def test_reductions_in_the_model():
    """light_options' reductions pick the kernels of the render without the option, and P_env, P_p are 1 or 1/2"""
    full = lms.FULL
    cases = [("env_light", lms.SceneState(env_table=False)), ("medium", lms.SceneState(sigma_t=False)),
             ("punctual_lights", lms.SceneState(J=0)), ("light_tree", lms.SceneState(K=0)), ("volumes", lms.SceneState(volumes=False))]
    for flag, st in cases:
        for bits in range(1 << len(lms.FLAGS)):
            flags = frozenset(f for i, f in enumerate(lms.FLAGS) if bits >> i & 1)
            if flag not in flags or not lms.valid(flags):
                continue
            if flag == "volumes" and "medium" in flags:   # glass displaces the medium: the VOL kernels run without volumes
                assert lms.predict(flags, st) == lms.predict(flags, full)
                continue
            off = flags - {flag} - ({"medium_grid"} if flag == "medium" else set())
            assert lms.predict(flags, st) == lms.predict(off, st), (flag, sorted(flags))
    assert lms.light_options({"env_light"})["p_env"] == 0.5
    assert lms.light_options({"env_light"}, lms.SceneState(K=0))["p_env"] == 1.0
    assert lms.light_options({"punctual_lights"}, lms.SceneState(K=0))["p_p"] == 1.0
    assert lms.light_options({"punctual_lights", "env_light"}, lms.SceneState(K=0))["p_p"] == 0.5
    assert lms.light_options({"punctual_lights", "emission_maps", "textures"}, lms.SceneState(K=3, K_emit=0))["p_p"] == 1.0


# ------------------------------------------------------------------ the model against the binary
def _binary_kernels():
    tool, filt = shutil.which("cuobjdump"), shutil.which("cu++filt")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    tool = tool or (os.path.join(cuda, "bin", "cuobjdump") if os.path.exists(os.path.join(cuda, "bin", "cuobjdump")) else None)
    filt = filt or (os.path.join(cuda, "bin", "cu++filt") if os.path.exists(os.path.join(cuda, "bin", "cu++filt")) else None)
    if tool is None or filt is None:
        pytest.skip("cuobjdump / cu++filt not found")
    if not os.path.exists(_build.PRODUCT_SO):
        _build.build()
    out = subprocess.run([tool, "-res-usage", _build.PRODUCT_SO], capture_output=True, text=True, check=True).stdout
    names = sorted({ln.split("Function ", 1)[1].split(":")[0].strip() for ln in out.splitlines() if ln.strip().startswith("Function ")})
    dem = subprocess.run([filt], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(dem) == len(names)
    return dem


def test_model_equals_the_binary():
    shade, nee = lms.kernel_keys(_binary_kernels())
    assert len(shade) == lms.N_SHADE and len(nee) == lms.N_NEE, (len(shade), len(nee))
    assert shade == lms.all_shade(), (sorted(shade - lms.all_shade())[:5], sorted(lms.all_shade() - shade)[:5])
    assert nee == lms.all_nee(), (sorted(nee - lms.all_nee())[:5], sorted(lms.all_nee() - nee)[:5])


# ------------------------------------------------------------------ the GPU file's rows
def test_rows_cover_every_instantiation():
    from tests import test_gpu_light_mode_space as g
    shade, nee = set(), set()
    for r in g.ROWS:
        s, k = lms.predict(r["flags"], lms.FULL, aov=r["aov"], max_bounce=r["bounces"], lane=True)
        shade |= s
        nee |= k
    assert shade == lms.all_shade(), sorted(lms.all_shade() - shade)[:5]
    assert nee == lms.all_nee(), sorted(lms.all_nee() - nee)[:5]
    # each of the 560 keys has a row of its own, with the deferred lane on, and every pair of path factors is in some row
    assert sorted(r["key"] for r in g.ROWS) == sorted(lms.row_keys())
    assert g.uncovered_pairs(g.ROWS) == set()


# ------------------------------------------------------------------ power, on the restatement
@pytest.fixture(scope="module")
def sd():
    return lms.space_scene()


def _image(sd, flags, med_flags, cache):
    """the restatement's image of flags, with the medium of med_flags (so that switching the grid off keeps the row's sigma_t)"""
    sigma = lms.medium_for(med_flags)["sigma_t"]
    key = (flags, sigma)
    if key not in cache:
        cfg = lms.config(sd, flags)
        kw = lms.oracle_kwargs(sd, flags, sigma_t=sigma)
        cache[key] = ov.render(sd["tris"], sd["nodes"], cfg, **kw)[0].tobytes()
    return cache[key]


def test_every_option_of_every_row_changes_the_image(sd):
    cache = {}
    seen = set()
    weak = []
    for key in lms.row_keys():
        flags = lms.flags_of(key)
        if flags in seen:   # A does not change the flags
            continue
        seen.add(flags)
        img = _image(sd, flags, flags, cache)
        for f in sorted(flags):
            off = lms.closure_off(flags, f)
            if _image(sd, off, flags, cache) == img:
                weak.append((sorted(flags), f))
    assert len(seen) == 280
    assert not weak, weak[:10]


# ------------------------------------------------------------------ reductions, on the restatement
REDUCTION_BASES = [frozenset(), frozenset({"light_tree", "textures"}), frozenset({"punctual_lights", "env_light"}),
                   frozenset({"transmission", "textures", "material_maps"}), frozenset({"textures", "emission_maps", "punctual_lights"})]


def _render(sd, flags, **kw):
    cfg = lms.config(sd, flags)
    img, luma2, _, c = ov.render(sd["tris"], sd["nodes"], cfg, **lms.oracle_kwargs(sd, flags, **kw))
    return img.tobytes() + luma2.tobytes(), (c["rays_primary"], c["rays_bounce"], c["rays_shadow"])


@pytest.mark.parametrize("flag", ["env_light", "medium", "medium_grid", "punctual_lights", "light_tree", "volumes"])
def test_reductions_give_the_bits_without_the_option(flag):
    """ENV_LIGHT with no map; MEDIUM (and MEDIUM_GRID with it) at sigma_t = 0; PUNCTUAL_LIGHTS with J = 0; LIGHT_TREE with K = 0 (the
    emitter-free scene); VOLUMES with no volumes and no medium"""
    sd = lms.space_scene(emitters=(flag != "light_tree"))
    for base in REDUCTION_BASES:
        kw_on = kw_off = {}
        if flag in ("medium", "medium_grid"):
            on = base | {"medium"} | ({"medium_grid"} if flag == "medium_grid" else set())
            on = on | ({"volumes"} if "transmission" in on else set())
            off, kw_on = on - {"medium", "medium_grid"}, dict(sigma_t=0.0)
        elif flag == "volumes":
            on = base | {"transmission", "volumes"}
            off, kw_on, kw_off = on - {"volumes"}, dict(volumes=False), dict(volumes=False)
        else:
            on = base | {flag}
            off = on - {flag}
            if flag == "env_light":
                kw_on = kw_off = dict(env=False)
            elif flag == "punctual_lights":
                kw_on = dict(punct=False)
        assert lms.valid(on) and lms.valid(off)
        assert _render(sd, on, **kw_on) == _render(sd, off, **kw_off), (flag, sorted(base))
