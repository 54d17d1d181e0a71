"""The cases of tests/golden/refshader.npz (frames rendered by the reference's own transpiled shaders),
shared by the generator (tests/golden/make_golden_refshader.py) and the CPU / GPU tests that replay them."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# (key, mode, max_bounce, hdr_linear, first_frame, spp): P3/P4 sample the map with GL_NEAREST, P5 with GL_LINEAR;
# max_bounce 2 / 4 / 2 are the shaders' own literals (P3/fsh:437, P4/fsh:541, P5/fsh:935).
CASES = [
    ("m0", 0, 2, False, 0, 3),
    ("m1", 1, 4, False, 0, 3),
    ("m2", 2, 2, True, 0, 3),
    ("m3", 3, 2, True, 0, 3),
    ("m3_b3_f7", 3, 3, True, 7, 2),  # continues an accumulation: lastFrame = the m3 image
]
W, H = 48, 32
SCENES = ("p3", "bunny", "grid")


def scene(name):
    """tris, nodes, eye, cam"""
    from ezrt_b200 import scenes
    if name == "p3":  # the reference's own P3 scene, arrays committed
        g = np.load(os.path.join(GOLDEN, "p3_scene.npz"))
        return g["tris"], g["nodes"], g["eye"], g["cam"]
    return scenes.s_bunny() if name == "bunny" else scenes.s_grid(3, 2, 2)


def environment():
    from ezrt_b200 import api, scenes
    hdr = scenes.synth_hdr(128, 64)
    return hdr, api.hdr_cache(hdr)


def config(case, eye, cam, **kw):
    from ezrt_b200 import api
    key, mode, mb, lin, first, spp = case
    return api.RenderConfig(width=W, height=H, spp=spp, max_bounce=mb, mode=mode, eye=tuple(eye), camera_rotate=tuple(cam),
                            first_frame=first, **kw)


def load():
    return np.load(os.path.join(GOLDEN, "refshader.npz"))


def load_refcompare():
    """what the reference's own code computed for the inputs of the comparison tests (tests/golden/make_golden_refcompare.py)"""
    return np.load(os.path.join(GOLDEN, "refcompare.npz"))
