"""Build recipes for the in-tree native libraries.

  ezrt_b200/libezrt_b200.so   the product: C ABI (include/ezrt.h) + host scene pipeline + sm_90a (H100) kernels
  oracle/libezrt_oracle.so    the CPU oracle (test infrastructure, see oracle/README.md)
  oracle/_ref/libhdrloader_ref.so   the one reference translation unit that compiles stand-alone
                                     (P5/lib/hdrloader.cpp), built only where /root/reference exists
  oracle/_ref/libezrt_refhost.so    the reference's own host code (P5 main.cpp + hdrloader.cpp) compiled from where
                                     it lies against stand-in GL/GLUT/glm headers (oracle/ref_stubs/), same condition
  oracle/_ref/libezrt_refshader.so  the reference's own fragment shaders (P3/P4/P5 fshader.fsh) transpiled
                                     to C++ from where they lie (oracle/ref_shader/), same condition

Parity needs bit-identical fp32 arithmetic on host and device, hence
  host  : -ffp-contract=off -mfma      (FMA only where ezrt_math.h spells it)
  device: -fmad=false, IEEE div/sqrt, no FTZ (nvcc defaults), never -use_fast_math
"""
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ezrt_b200", "csrc")
INCLUDE = os.path.join(ROOT, "include")
PRODUCT_SO = os.path.join(ROOT, "ezrt_b200", "libezrt_b200.so")
ORACLE_SO = os.path.join(ROOT, "oracle", "libezrt_oracle.so")
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
REF_HDR_SO = os.path.join(REF_DIR, "libhdrloader_ref.so")
REF_SHADER_SO = os.path.join(REF_DIR, "libezrt_refshader.so")
REF_HOST_SO = os.path.join(REF_DIR, "libezrt_refhost.so")
REFERENCE_ROOT = "/root/reference"
REFERENCE_PARTS = ("part 3 -- OpenGL Raytracing", "part 4 -- Disney Principle BRDF",
                   "part 5 -- Importance Sampling & Low Discrepancy Sequence")
REFERENCE_P5 = os.path.join(REFERENCE_ROOT, REFERENCE_PARTS[2], "source code")

HOST_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-mfma", "-Wall"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-fmad=false",
    "-Xcompiler", "-fPIC,-ffp-contract=off,-mfma", "-Xptxas", "-v",
]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _run(cmd, log=None):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if log:
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + r.stdout)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("build failed: " + " ".join(cmd))
    return r.stdout


def _headers():
    hs = [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    hs += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh", ".inc"))]
    return hs


def build_product(force=False, verbose=False, variant=None, defines=()):
    """nvcc + g++ -> ezrt_b200/libezrt_b200.so (cross-compiles for sm_90a without a GPU).
    variant/defines build an experiment copy libezrt_b200_<variant>.so with extra -D macros
    (selected at import time by env EZRT_LIB_VARIANT; used for A/B runs on the GPU box)."""
    nvcc = _nvcc()
    if nvcc is None:
        raise RuntimeError("nvcc not found: cannot build libezrt_b200.so")
    target = PRODUCT_SO if not variant else PRODUCT_SO.replace(".so", "_%s.so" % variant)
    cu = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))
    cpp = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cpp"))
    if not force and not _newer(target, cu + cpp + _headers()):
        return target
    objdir = os.path.join(ROOT, "build", "obj" + ("_" + variant if variant else ""))
    os.makedirs(objdir, exist_ok=True)
    # one builder at a time (several ranks / pytest workers may import the package at once)
    import fcntl
    lock = open(os.path.join(ROOT, "build", ".lock"), "w")
    fcntl.flock(lock, fcntl.LOCK_EX)
    try:
        if not force and not _newer(target, cu + cpp + _headers()):
            return target
        return _build_product_locked(nvcc, target, cu, cpp, objdir, defines, verbose)
    finally:
        fcntl.flock(lock, fcntl.LOCK_UN)
        lock.close()


def _build_product_locked(nvcc, target, cu, cpp, objdir, defines, verbose):
    dflags = ["-D" + d for d in defines]
    jobs = []   # (command, object, ptxas log); compiled concurrently: the translation units are independent
    for src in cu:
        obj = os.path.join(objdir, os.path.basename(src) + ".o")
        jobs.append(([nvcc] + NVCC_FLAGS + dflags + ["-I", INCLUDE, "-I", CSRC, "-c", src, "-o", obj], obj,
                     os.path.join(objdir, os.path.basename(src) + ".ptxas.log")))
    for src in cpp:
        obj = os.path.join(objdir, os.path.basename(src) + ".o")
        jobs.append((["g++"] + HOST_FLAGS + dflags + ["-pthread", "-I", INCLUDE, "-I", CSRC, "-c", src, "-o", obj], obj, None))
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as pool:
        outs = list(pool.map(lambda j: _run(j[0], log=j[2]), jobs))
    if verbose:
        for (cmd, _, log), out in zip(jobs, outs):
            if log:
                print(out)
    objs = [obj for _, obj, _ in jobs]
    tmp = target + ".tmp%d" % os.getpid()
    _run([nvcc, "-shared", "-o", tmp] + objs + ["-Xcompiler", "-pthread", "-cudart", "static"])
    os.replace(tmp, target)  # atomic: a concurrent import never sees a half-written library
    return target


def _oracle_recipes():
    """oracle/build_ref.py -- the recipes of the checker libraries live under oracle/ (test infrastructure)"""
    import importlib.util
    spec = importlib.util.spec_from_file_location("ezrt_oracle_build_ref", os.path.join(ROOT, "oracle", "build_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def build_oracle(force=False):
    return _oracle_recipes().build_oracle(force)


ORACLE_ADAPTIVE_SO = os.path.join(ROOT, "build", "libezrt_oracle_adaptive.so")


def build_oracle_adaptive(force=False):
    """build/libezrt_oracle_adaptive.so: tests/oracle_adaptive.cpp, the CPU restatement of adaptive sampling over the
    oracle's sample function (test infrastructure, loaded only by tests/oracle_adaptive.py)."""
    src = os.path.join(ROOT, "tests", "oracle_adaptive.cpp")
    deps = [src, os.path.join(ROOT, "oracle", "ezrt_oracle.cpp")] + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if force or _newer(ORACLE_ADAPTIVE_SO, deps):
        os.makedirs(os.path.dirname(ORACLE_ADAPTIVE_SO), exist_ok=True)
        tmp = ORACLE_ADAPTIVE_SO + ".tmp%d" % os.getpid()
        _run(["g++"] + HOST_FLAGS + ["-fopenmp", "-Wno-misleading-indentation", "-shared", "-I", INCLUDE, src, "-o", tmp])
        os.replace(tmp, ORACLE_ADAPTIVE_SO)
    return ORACLE_ADAPTIVE_SO


ORACLE_AOV_SO = os.path.join(ROOT, "build", "libezrt_oracle_aov.so")


def build_oracle_aov(force=False):
    """build/libezrt_oracle_aov.so: tests/oracle_aov.cpp, the CPU restatement of the feature-buffer render over the oracle's
    sample function and of the denoiser (test infrastructure, loaded only by tests/oracle_aov.py)."""
    src = os.path.join(ROOT, "tests", "oracle_aov.cpp")
    deps = [src, os.path.join(ROOT, "oracle", "ezrt_oracle.cpp")] + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if force or _newer(ORACLE_AOV_SO, deps):
        os.makedirs(os.path.dirname(ORACLE_AOV_SO), exist_ok=True)
        tmp = ORACLE_AOV_SO + ".tmp%d" % os.getpid()
        _run(["g++"] + HOST_FLAGS + ["-fopenmp", "-Wno-misleading-indentation", "-shared", "-I", INCLUDE, src, "-o", tmp])
        os.replace(tmp, ORACLE_AOV_SO)
    return ORACLE_AOV_SO


ORACLE_LIGHTS_SO = os.path.join(ROOT, "build", "libezrt_oracle_lights.so")


def build_oracle_lights(force=False):
    """build/libezrt_oracle_lights.so: tests/oracle_lights.cpp, the CPU restatement of the light sampling mode (light table,
    bounded occlusion, integrator) over the oracle's functions (test infrastructure, loaded only by tests/oracle_lights.py)."""
    src = os.path.join(ROOT, "tests", "oracle_lights.cpp")
    deps = [src, os.path.join(ROOT, "oracle", "ezrt_oracle.cpp")] + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if force or _newer(ORACLE_LIGHTS_SO, deps):
        os.makedirs(os.path.dirname(ORACLE_LIGHTS_SO), exist_ok=True)
        tmp = ORACLE_LIGHTS_SO + ".tmp%d" % os.getpid()
        _run(["g++"] + HOST_FLAGS + ["-fopenmp", "-Wno-misleading-indentation", "-shared", "-I", INCLUDE, src, "-o", tmp])
        os.replace(tmp, ORACLE_LIGHTS_SO)
    return ORACLE_LIGHTS_SO


ORACLE_ENV_LIGHT_SO = os.path.join(ROOT, "build", "libezrt_oracle_env_light.so")


def build_oracle_env_light(force=False):
    """build/libezrt_oracle_env_light.so: tests/oracle_env_light.cpp, the CPU restatement of the environment map as a light
    (table, sampler, flagged integrator) over the light sampling mode's restatement (test infrastructure, loaded only by
    tests/oracle_env_light.py)."""
    src = os.path.join(ROOT, "tests", "oracle_env_light.cpp")
    deps = [src, os.path.join(ROOT, "tests", "oracle_lights.cpp"), os.path.join(ROOT, "oracle", "ezrt_oracle.cpp")] + \
        [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if force or _newer(ORACLE_ENV_LIGHT_SO, deps):
        os.makedirs(os.path.dirname(ORACLE_ENV_LIGHT_SO), exist_ok=True)
        tmp = ORACLE_ENV_LIGHT_SO + ".tmp%d" % os.getpid()
        _run(["g++"] + HOST_FLAGS + ["-fopenmp", "-Wno-misleading-indentation", "-shared", "-I", INCLUDE, src, "-o", tmp])
        os.replace(tmp, ORACLE_ENV_LIGHT_SO)
    return ORACLE_ENV_LIGHT_SO


ORACLE_TRANSMISSION_SO = os.path.join(ROOT, "build", "libezrt_oracle_transmission.so")


def build_oracle_transmission(force=False):
    """build/libezrt_oracle_transmission.so: tests/oracle_transmission.cpp, the CPU restatement of the materials' transmission
    (the mixture, its sampler, the flagged integrator with and without the map as a light) over the environment light's
    restatement (test infrastructure, loaded only by tests/oracle_transmission.py)."""
    src = os.path.join(ROOT, "tests", "oracle_transmission.cpp")
    deps = [src, os.path.join(ROOT, "tests", "oracle_env_light.cpp"), os.path.join(ROOT, "tests", "oracle_lights.cpp"),
            os.path.join(ROOT, "oracle", "ezrt_oracle.cpp")] + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if force or _newer(ORACLE_TRANSMISSION_SO, deps):
        os.makedirs(os.path.dirname(ORACLE_TRANSMISSION_SO), exist_ok=True)
        tmp = ORACLE_TRANSMISSION_SO + ".tmp%d" % os.getpid()
        _run(["g++"] + HOST_FLAGS + ["-fopenmp", "-Wno-misleading-indentation", "-shared", "-I", INCLUDE, src, "-o", tmp])
        os.replace(tmp, ORACLE_TRANSMISSION_SO)
    return ORACLE_TRANSMISSION_SO


ORACLE_LENS_SO = os.path.join(ROOT, "build", "libezrt_oracle_lens.so")


def build_oracle_lens(force=False):
    """build/libezrt_oracle_lens.so: tests/oracle_lens.cpp, the CPU restatement of the thin-lens camera (its ray, and every mode's
    render from the lens ray's first hit) over the transmission restatement (test infrastructure, loaded only by tests/oracle_lens.py)."""
    src = os.path.join(ROOT, "tests", "oracle_lens.cpp")
    deps = [src] + [os.path.join(ROOT, "tests", f) for f in ("oracle_transmission.cpp", "oracle_env_light.cpp", "oracle_lights.cpp")] + \
        [os.path.join(ROOT, "oracle", "ezrt_oracle.cpp")] + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if force or _newer(ORACLE_LENS_SO, deps):
        os.makedirs(os.path.dirname(ORACLE_LENS_SO), exist_ok=True)
        tmp = ORACLE_LENS_SO + ".tmp%d" % os.getpid()
        _run(["g++"] + HOST_FLAGS + ["-fopenmp", "-Wno-misleading-indentation", "-shared", "-I", INCLUDE, src, "-o", tmp])
        os.replace(tmp, ORACLE_LENS_SO)
    return ORACLE_LENS_SO


ORACLE_MEDIUM_SO = os.path.join(ROOT, "build", "libezrt_oracle_medium.so")


def build_oracle_medium(force=False):
    """build/libezrt_oracle_medium.so: tests/oracle_medium.cpp, the CPU restatement of the homogeneous medium (free flight, the
    phase function, the light samples' transmittance, the flagged render) over the lens restatement (test infrastructure, loaded only
    by tests/oracle_medium.py)."""
    src = os.path.join(ROOT, "tests", "oracle_medium.cpp")
    deps = [src] + [os.path.join(ROOT, "tests", f) for f in ("oracle_lens.cpp", "oracle_transmission.cpp", "oracle_env_light.cpp", "oracle_lights.cpp")] + \
        [os.path.join(ROOT, "oracle", "ezrt_oracle.cpp")] + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if force or _newer(ORACLE_MEDIUM_SO, deps):
        os.makedirs(os.path.dirname(ORACLE_MEDIUM_SO), exist_ok=True)
        tmp = ORACLE_MEDIUM_SO + ".tmp%d" % os.getpid()
        _run(["g++"] + HOST_FLAGS + ["-fopenmp", "-Wno-misleading-indentation", "-shared", "-I", INCLUDE, src, "-o", tmp])
        os.replace(tmp, ORACLE_MEDIUM_SO)
    return ORACLE_MEDIUM_SO


ORACLE_TEXTURES_SO = os.path.join(ROOT, "build", "libezrt_oracle_textures.so")


def build_oracle_textures(force=False):
    """build/libezrt_oracle_textures.so: tests/oracle_textures.cpp, the CPU restatement of base-colour textures (the barycentrics, the
    filter, the flagged render) over the medium restatement (test infrastructure, loaded only by tests/oracle_textures.py)."""
    src = os.path.join(ROOT, "tests", "oracle_textures.cpp")
    deps = [src] + [os.path.join(ROOT, "tests", f) for f in ("oracle_medium.cpp", "oracle_lens.cpp", "oracle_transmission.cpp", "oracle_env_light.cpp",
                                                              "oracle_lights.cpp")] + \
        [os.path.join(ROOT, "oracle", "ezrt_oracle.cpp")] + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if force or _newer(ORACLE_TEXTURES_SO, deps):
        os.makedirs(os.path.dirname(ORACLE_TEXTURES_SO), exist_ok=True)
        tmp = ORACLE_TEXTURES_SO + ".tmp%d" % os.getpid()
        _run(["g++"] + HOST_FLAGS + ["-fopenmp", "-Wno-misleading-indentation", "-shared", "-I", INCLUDE, src, "-o", tmp])
        os.replace(tmp, ORACLE_TEXTURES_SO)
    return ORACLE_TEXTURES_SO


ORACLE_MATERIAL_MAPS_SO = os.path.join(ROOT, "build", "libezrt_oracle_material_maps.so")


def build_oracle_material_maps(force=False):
    """build/libezrt_oracle_material_maps.so: tests/oracle_material_maps.cpp, the CPU restatement of the material maps (the table, the
    tangent frame, the mapped normal, the flagged render's medium and transmission loops) over the textures' restatement (test
    infrastructure, loaded only by tests/oracle_material_maps.py)."""
    src = os.path.join(ROOT, "tests", "oracle_material_maps.cpp")
    deps = [src] + [os.path.join(ROOT, "tests", f) for f in ("oracle_textures.cpp", "oracle_medium.cpp", "oracle_lens.cpp", "oracle_transmission.cpp",
                                                              "oracle_env_light.cpp", "oracle_lights.cpp")] + \
        [os.path.join(ROOT, "oracle", "ezrt_oracle.cpp")] + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if force or _newer(ORACLE_MATERIAL_MAPS_SO, deps):
        os.makedirs(os.path.dirname(ORACLE_MATERIAL_MAPS_SO), exist_ok=True)
        tmp = ORACLE_MATERIAL_MAPS_SO + ".tmp%d" % os.getpid()
        _run(["g++"] + HOST_FLAGS + ["-fopenmp", "-Wno-misleading-indentation", "-shared", "-I", INCLUDE, src, "-o", tmp])
        os.replace(tmp, ORACLE_MATERIAL_MAPS_SO)
    return ORACLE_MATERIAL_MAPS_SO


ORACLE_PUNCTUAL_SO = os.path.join(ROOT, "build", "libezrt_oracle_punctual.so")


def build_oracle_punctual(force=False):
    """build/libezrt_oracle_punctual.so: tests/oracle_punctual.cpp, the CPU restatement of the punctual lights (the table, the sample,
    the flagged render's medium and transmission loops with the category split) over the material maps' restatement (test
    infrastructure, loaded only by tests/oracle_punctual.py)."""
    src = os.path.join(ROOT, "tests", "oracle_punctual.cpp")
    deps = [src] + [os.path.join(ROOT, "tests", f) for f in ("oracle_material_maps.cpp", "oracle_textures.cpp", "oracle_medium.cpp", "oracle_lens.cpp",
                                                              "oracle_transmission.cpp", "oracle_env_light.cpp", "oracle_lights.cpp")] + \
        [os.path.join(ROOT, "oracle", "ezrt_oracle.cpp")] + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if force or _newer(ORACLE_PUNCTUAL_SO, deps):
        os.makedirs(os.path.dirname(ORACLE_PUNCTUAL_SO), exist_ok=True)
        tmp = ORACLE_PUNCTUAL_SO + ".tmp%d" % os.getpid()
        _run(["g++"] + HOST_FLAGS + ["-fopenmp", "-Wno-misleading-indentation", "-shared", "-I", INCLUDE, src, "-o", tmp])
        os.replace(tmp, ORACLE_PUNCTUAL_SO)
    return ORACLE_PUNCTUAL_SO


ORACLE_EMISSION_MAPS_SO = os.path.join(ROOT, "build", "libezrt_oracle_emission_maps.so")


def build_oracle_emission_maps(force=False):
    """build/libezrt_oracle_emission_maps.so: tests/oracle_emission_maps.cpp, the CPU restatement of the emission maps (the emission
    table, E(Q), the flagged render's medium and transmission loops) over the punctual lights' restatement (test infrastructure,
    loaded only by tests/oracle_emission_maps.py)."""
    src = os.path.join(ROOT, "tests", "oracle_emission_maps.cpp")
    deps = [src] + [os.path.join(ROOT, "tests", f) for f in ("oracle_punctual.cpp", "oracle_material_maps.cpp", "oracle_textures.cpp", "oracle_medium.cpp",
                                                              "oracle_lens.cpp", "oracle_transmission.cpp", "oracle_env_light.cpp", "oracle_lights.cpp")] + \
        [os.path.join(ROOT, "oracle", "ezrt_oracle.cpp")] + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if force or _newer(ORACLE_EMISSION_MAPS_SO, deps):
        os.makedirs(os.path.dirname(ORACLE_EMISSION_MAPS_SO), exist_ok=True)
        tmp = ORACLE_EMISSION_MAPS_SO + ".tmp%d" % os.getpid()
        _run(["g++"] + HOST_FLAGS + ["-fopenmp", "-Wno-misleading-indentation", "-shared", "-I", INCLUDE, src, "-o", tmp])
        os.replace(tmp, ORACLE_EMISSION_MAPS_SO)
    return ORACLE_EMISSION_MAPS_SO


ORACLE_LIGHT_TREE_SO = os.path.join(ROOT, "build", "libezrt_oracle_light_tree.so")


ORACLE_MEDIUM_GRID_SO = os.path.join(ROOT, "build", "libezrt_oracle_medium_grid.so")


def build_oracle_medium_grid(force=False):
    """build/libezrt_oracle_medium_grid.so: tests/oracle_medium_grid.cpp, the CPU restatement of the density grid (its brick maxima,
    lookup, free flight and transmittance with their majorant counters, and the flagged renders over the light tree's restatement;
    test infrastructure, loaded only by tests/oracle_medium_grid.py)."""
    src = os.path.join(ROOT, "tests", "oracle_medium_grid.cpp")
    deps = [src] + [os.path.join(ROOT, "tests", f) for f in ("oracle_light_tree.cpp", "oracle_emission_maps.cpp", "oracle_punctual.cpp",
                                                             "oracle_material_maps.cpp", "oracle_textures.cpp", "oracle_medium.cpp", "oracle_lens.cpp",
                                                             "oracle_transmission.cpp", "oracle_env_light.cpp", "oracle_lights.cpp")] + \
        [os.path.join(ROOT, "oracle", "ezrt_oracle.cpp")] + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if force or _newer(ORACLE_MEDIUM_GRID_SO, deps):
        os.makedirs(os.path.dirname(ORACLE_MEDIUM_GRID_SO), exist_ok=True)
        tmp = ORACLE_MEDIUM_GRID_SO + ".tmp%d" % os.getpid()
        _run(["g++"] + HOST_FLAGS + ["-fopenmp", "-Wno-misleading-indentation", "-shared", "-I", INCLUDE, src, "-o", tmp])
        os.replace(tmp, ORACLE_MEDIUM_GRID_SO)
    return ORACLE_MEDIUM_GRID_SO


ORACLE_VOLUMES_SO = os.path.join(ROOT, "build", "libezrt_oracle_volumes.so")


def build_oracle_volumes(force=False):
    """build/libezrt_oracle_volumes.so: tests/oracle_volumes.cpp, the CPU restatement of the volumes inside transmissive meshes (sigma_a,
    the interior test, the flagged render's transmission loop with the absorption) over the density grid's restatement (test
    infrastructure, loaded only by tests/oracle_volumes.py)."""
    src = os.path.join(ROOT, "tests", "oracle_volumes.cpp")
    deps = [src] + [os.path.join(ROOT, "tests", f) for f in ("oracle_medium_grid.cpp", "oracle_light_tree.cpp", "oracle_emission_maps.cpp",
                                                             "oracle_punctual.cpp", "oracle_material_maps.cpp", "oracle_textures.cpp",
                                                             "oracle_medium.cpp", "oracle_lens.cpp", "oracle_transmission.cpp", "oracle_env_light.cpp",
                                                             "oracle_lights.cpp")] + \
        [os.path.join(ROOT, "oracle", "ezrt_oracle.cpp")] + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if force or _newer(ORACLE_VOLUMES_SO, deps):
        os.makedirs(os.path.dirname(ORACLE_VOLUMES_SO), exist_ok=True)
        tmp = ORACLE_VOLUMES_SO + ".tmp%d" % os.getpid()
        _run(["g++"] + HOST_FLAGS + ["-fopenmp", "-Wno-misleading-indentation", "-shared", "-I", INCLUDE, src, "-o", tmp])
        os.replace(tmp, ORACLE_VOLUMES_SO)
    return ORACLE_VOLUMES_SO


def build_oracle_light_tree(force=False):
    """build/libezrt_oracle_light_tree.so: tests/oracle_light_tree.cpp, the CPU restatement of the light tree (the descent, the
    hit-side walk, the flagged render's medium and transmission loops) over the emission maps' restatement (test infrastructure,
    loaded only by tests/oracle_light_tree.py)."""
    src = os.path.join(ROOT, "tests", "oracle_light_tree.cpp")
    deps = [src] + [os.path.join(ROOT, "tests", f) for f in ("oracle_emission_maps.cpp", "oracle_punctual.cpp", "oracle_material_maps.cpp",
                                                              "oracle_textures.cpp", "oracle_medium.cpp", "oracle_lens.cpp", "oracle_transmission.cpp",
                                                              "oracle_env_light.cpp", "oracle_lights.cpp")] + \
        [os.path.join(ROOT, "oracle", "ezrt_oracle.cpp")] + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if force or _newer(ORACLE_LIGHT_TREE_SO, deps):
        os.makedirs(os.path.dirname(ORACLE_LIGHT_TREE_SO), exist_ok=True)
        tmp = ORACLE_LIGHT_TREE_SO + ".tmp%d" % os.getpid()
        _run(["g++"] + HOST_FLAGS + ["-fopenmp", "-Wno-misleading-indentation", "-shared", "-I", INCLUDE, src, "-o", tmp])
        os.replace(tmp, ORACLE_LIGHT_TREE_SO)
    return ORACLE_LIGHT_TREE_SO


def build_reference_hdrloader(force=False):
    return _oracle_recipes().build_reference_hdrloader(force)


def build_reference_shaders(force=False):
    return _oracle_recipes().build_reference_shaders(force)


def build_reference_host(force=False, part=5):
    return _oracle_recipes().build_reference_host(force, part)


EXAMPLE_BIN = os.path.join(ROOT, "examples", "ezrt_main")


def build_example(force=False):
    """examples/ezrt_main: the reference's main() + display() as a C++ host over the C ABI (links libezrt_b200.so)."""
    src = os.path.join(ROOT, "examples", "ezrt_main.cpp")
    if force or _newer(EXAMPLE_BIN, [src, PRODUCT_SO, os.path.join(INCLUDE, "ezrt.h")]):
        tmp = EXAMPLE_BIN + ".tmp%d" % os.getpid()
        _run(["g++", "-O2", "-std=c++17", "-Wall", "-I", INCLUDE, src, "-L", os.path.dirname(PRODUCT_SO), "-lezrt_b200",
              "-Wl,-rpath,$ORIGIN/../ezrt_b200", "-o", tmp])
        os.replace(tmp, EXAMPLE_BIN)
    return EXAMPLE_BIN


W8_MODEL_BIN = os.path.join(ROOT, "build", "w8_model")


def build_w8_model(force=False):
    """build/w8_model: CPU model of the W8 acceleration-tree traversal (tools/w8_model.cpp) over the PRODUCT tree builders --
    the not-gpu check that the quantised tree is conservative (closest hits equal brute force)."""
    srcs = [os.path.join(ROOT, "tools", "w8_model.cpp")] + [os.path.join(CSRC, f) for f in ("host_scene.cpp", "accel_w8.cpp", "errors.cpp")]
    if force or _newer(W8_MODEL_BIN, srcs + _headers()):
        os.makedirs(os.path.dirname(W8_MODEL_BIN), exist_ok=True)
        tmp = W8_MODEL_BIN + ".tmp%d" % os.getpid()
        _run(["g++"] + [f for f in HOST_FLAGS if f != "-fPIC"] + ["-fopenmp", "-pthread", "-I", INCLUDE, "-I", CSRC] + srcs + ["-o", tmp])
        os.replace(tmp, W8_MODEL_BIN)
    return W8_MODEL_BIN


W4_CHECK_BIN = os.path.join(ROOT, "build", "w4_check")


def build_w4_check(force=False):
    """build/w4_check: CPU check of the 4-wide acceleration-tree builder (tools/w4_check.cpp): thread-count independence, structure."""
    srcs = [os.path.join(ROOT, "tools", "w4_check.cpp")] + [os.path.join(CSRC, f) for f in ("host_scene.cpp", "accel_w8.cpp", "errors.cpp")]
    if force or _newer(W4_CHECK_BIN, srcs + _headers()):
        os.makedirs(os.path.dirname(W4_CHECK_BIN), exist_ok=True)
        tmp = W4_CHECK_BIN + ".tmp%d" % os.getpid()
        _run(["g++"] + [f for f in HOST_FLAGS if f != "-fPIC"] + ["-pthread", "-I", INCLUDE, "-I", CSRC] + srcs + ["-o", tmp])
        os.replace(tmp, W4_CHECK_BIN)
    return W4_CHECK_BIN


def build_all(force=False, verbose=False):
    build_product(force=force, verbose=verbose)
    build_oracle(force=force)
    build_oracle_adaptive(force=force)
    build_oracle_aov(force=force)
    build_oracle_lights(force=force)
    build_oracle_env_light(force=force)
    build_oracle_transmission(force=force)
    build_oracle_lens(force=force)
    build_oracle_medium(force=force)
    build_oracle_textures(force=force)
    build_oracle_material_maps(force=force)
    build_oracle_punctual(force=force)
    build_oracle_emission_maps(force=force)
    build_oracle_light_tree(force=force)
    build_oracle_volumes(force=force)
    build_example(force=force)
    build_reference_hdrloader(force=force)
    build_reference_shaders(force=force)
    for part in (3, 4, 5):
        build_reference_host(force=force, part=part)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built", PRODUCT_SO, ORACLE_SO)
