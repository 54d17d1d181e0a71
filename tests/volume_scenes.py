"""Scenes with absorbing glass for the volume tests (RenderConfig.volumes, DESIGN.md section 21): tests/transmission_scenes.py's scenes
with volumes and their per-triangle ids, and the analytic slab.  Every mesh made glass here is closed, wound outward and not nested, as
EZRT_PARAM_VOLUMES assumes."""
import numpy as np

from ezrt_b200 import api, scenes
from tests import transmission_scenes as ts

# amber glass of a bottle: red and green pass, blue is absorbed within a fraction of the blob's size
AMBER = api.volume((0.9, 0.55, 0.15), 0.6)


def glass_ids(tris, vid=0):
    """volume id vid on every triangle whose material has transmission > 0, -1 elsewhere"""
    tris = np.asarray(tris, np.float32).reshape(-1, 36)
    return np.where(tris[:, 35] > 0, vid, -1).astype(np.int32)


def p3_coloured_glass(roughness=0.3, ior=1.5, volume=AMBER):
    """P3's scene with the blob made of coloured glass: (tris, nodes, eye, cam, volumes, volume_id)"""
    tris, nodes, eye, cam = ts.p3_glass("blob", ts.glass(roughness, ior))
    return tris, nodes, eye, cam, [volume], glass_ids(tris)


def grid_volumes(nx, nz, pitch=1.2):
    """three volumes, and the ids of transmission_scenes.grid_glass(nx, nz)'s triangles: glass blob k (row-major among the glass ones)
    has volume k mod 3, each triangle going to the glass blob whose grid cell centre is nearest (the glass blobs lie at least a
    diagonal pitch apart); the opaque blobs have id 0, which is ignored; the spheres and the floor -1"""
    vols = [AMBER, api.volume((0.3, 0.8, 0.5), 1.5), api.volume((0.6, 0.6, 0.95), 0.25)]
    cells = [i for i in range(nx * nz) if i % 2 == 1]
    centres = np.array([((i % nx - (nx - 1) / 2.0) * pitch, (i // nx - (nz - 1) / 2.0) * pitch) for i in cells])

    def ids(tris):
        tris = np.asarray(tris, np.float32).reshape(-1, 36)
        c = tris[:, 0:9].reshape(-1, 3, 3).mean(axis=1).astype(np.float64)
        out = np.full(tris.shape[0], -1, np.int32)
        glass = tris[:, 35] > 0
        cg = c[glass][:, [0, 2]]
        near = np.concatenate([np.argmin(((cg[k:k + 16384, None] - centres[None]) ** 2).sum(axis=2), axis=1) for k in range(0, len(cg), 16384)])
        out[glass] = near % 3
        blob = ~glass & (tris[:, 18:21].max(axis=1) == 0) & (c[:, 1] > -1.39)   # the opaque blobs (not the floor, not a light)
        out[blob] = 0
        return out
    return vols, ids


def grid_coloured_glass(nx, nz, n_lights=4):
    """transmission_scenes.grid_glass with three volumes over its blobs: (tris, nodes, eye, cam, volumes, volume_id)"""
    tris, nodes, eye, cam = ts.grid_glass(nx, nz, n_lights)
    vols, ids = grid_volumes(nx, nz)
    return tris, nodes, eye, cam, vols, ids(tris)


def slab(ior=1.0, roughness=0.0, thickness=0.4, emission=2.0):
    """a white glass slab (2.4 x 2.4 x thickness, front face at z = 0.7) between the camera (z = 4) and a black, non-reflecting square
    emitter (8 x 8 at z = -1.5) on a black environment: (tris, nodes, eye, cam); id 0 on the slab"""
    tl = api.TriangleList()
    tl.read_obj_text(scenes.box_obj(), ts.glass(roughness, ior), api.transform_matrix((0, 0, 0), (0, 0, 0.7 - thickness / 2), (2.4, 2.4, thickness)),
                     False)
    tl.read_obj_text(scenes.box_obj(), api.Material(emissive=(emission,) * 3, baseColor=(0, 0, 0), specular=0.0),
                     api.transform_matrix((0, 0, 0), (0, 0, -1.5), (8.0, 8.0, 0.02)), False)
    tris, nodes = tl.build_bvh(8)
    eye, cam = api.camera_orbit(0.0, 0.0, 4.0)
    return np.asarray(tris, np.float32).reshape(-1, 36), nodes, eye, cam


# fog around the P3 blob (EZRT_PARAM_MEDIUM): the blob and the space above the floor near it
FOG = dict(sigma_t=0.6, albedo=(0.9, 0.8, 0.7), g=0.4, box_min=(-1.6, -1.4, -1.6), box_max=(1.6, 1.2, 1.6))


def p3_glass_in_fog(roughness=0.3):
    """p3_coloured_glass inside homogeneous fog: (tris, nodes, eye, cam, volumes, volume_id, fog) with fog the keyword arguments of
    Scene.set_medium"""
    return p3_coloured_glass(roughness) + (dict(FOG),)


def p3_glass_in_smoke(n=32, seed=0, sigma_t=4.0):
    """p3_coloured_glass inside scenes.smoke_grid(n, seed) filling FOG's box: (tris, nodes, eye, cam, volumes, volume_id, medium, grid)"""
    return p3_coloured_glass() + (dict(FOG, sigma_t=sigma_t), scenes.smoke_grid(n, seed))


def clear_box_in_absorber(sigma_t=0.8):
    """slab(ior=1.0) (a clear, index-matched box 0.4 thick, front face at z = 0.7) inside a pure absorber (albedo 0) that fills
    z in [-1, 1.5] across the view, in front of the emitter at z = -1.5: (tris, nodes, eye, cam, medium)"""
    tris, nodes, eye, cam = slab(ior=1.0)
    return tris, nodes, eye, cam, dict(sigma_t=sigma_t, albedo=(0.0, 0.0, 0.0), g=0.0, box_min=(-20.0, -20.0, -1.0), box_max=(20.0, 20.0, 1.5))
