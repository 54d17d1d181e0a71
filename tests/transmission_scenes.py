"""Scenes with transmissive materials for the transmission tests (RenderConfig.transmission, DESIGN.md section 12).  Every mesh
made glass here is closed and wound outward, as EZRT_PARAM_TRANSMISSION assumes."""
import numpy as np

from ezrt_b200 import api, scenes


def glass(roughness=0.3, ior=1.5, color=(1.0, 1.0, 1.0), transmission=1.0, metallic=0.0):
    return api.Material(baseColor=color, roughness=roughness, IOR=ior, transmission=transmission, metallic=metallic)


def _build(meshes, eye, cam):
    tl = api.TriangleList()
    for text, m, trans, smooth in meshes:
        tl.read_obj_text(text, m, trans, smooth)
    tris, nodes = tl.build_bvh(8)
    return np.asarray(tris, np.float32).reshape(-1, 36), nodes, eye, cam


def p3_glass(mesh="blob", material=None):
    """P3's scene (floor, emissive sphere) with its bunny ("bunny") or the closed blob ("blob") made of `material` (default rough
    glass, roughness 0.3, IOR 1.5)"""
    meshes = scenes.p3_bunny_meshes() if mesh == "bunny" else scenes.bunny_meshes()
    text, _, trans, smooth = meshes[0]
    meshes = [(text, material or glass(), trans, smooth)] + list(meshes[1:])
    eye, cam = api.camera_orbit(0.0, 0.0, 4.0)
    return _build(meshes, eye, cam)


def grid_glass(nx, nz, n_lights=4, roughness=(0.05, 0.3)):
    """scenes.s_grid's blob grid with every other blob glass (IOR 1.5), alternating the roughnesses given"""
    meshes = scenes.grid_meshes(nx, nz, n_lights)
    out, k = [], 0
    for i, (text, m, trans, smooth) in enumerate(meshes):
        if i < nx * nz and i % 2 == 1:
            m = glass(roughness[k % len(roughness)])
            k += 1
        out.append((text, m, trans, smooth))
    r = 0.62 * max(nx * 1.2, nz * 1.2) + 3.0
    eye, cam = api.camera_orbit(30.0, 25.0, r)
    return _build(out, eye, cam)

