"""Synthetic scenes for the benchmark configurations of BASELINE.json (SURVEY.md 8d).

The named scenes use the Stanford bunny.  /root/reference (and its OBJ files) does not exist on the GPU box, so the
bunny travels as an indexed mesh asset (ezrt_b200/data/bunny.npz, 2503 vertices / 4968 faces, recovered from the
committed P3 scene arrays by tests/golden/make_bunny_asset.py); it is emitted as OBJ text and pushed through the same
readObj() parser, unit-box normalisation, transform and smooth-normal code as any mesh file.  sphere.obj (320
triangles) and quad.obj (a 12-triangle box) are regenerated procedurally with the same triangle counts.

  s_p3_bunny()   P3/main.cpp:690-701: bunny (4968) + floor (12) + emissive sphere (320) = 5300 tris     [C1, C2]
  s_1m_bunny()   SURVEY 8(d) "S-1M": 201 bunnies in the first 201 slots of a 15x14 grid + 4 emissive spheres + floor
                 = 201*4968 + 1280 + 12 = 999,860 triangles                                              [C3, C4, C5]

Second workload family kept from round 1 (a procedural stand-in mesh, "blob" = bumpy icosphere, 5120 triangles;
geometry uses only + - * / sqrt and integer hashing, so the OBJ text is identical on every machine):

  s_bunny()  blob (5120) + floor box (12) + emissive sphere (320) = 5452 tris
  s_1m()     195 blobs on a 15x13 grid + 4 emissive spheres + floor = 999,692 tris
"""
import os
import numpy as np

from . import api
from .api import Material, TriangleList, transform_matrix


def _wang(seed):
    seed = ((seed ^ 61) ^ (seed >> 16)) & 0xFFFFFFFF
    seed = (seed * 9) & 0xFFFFFFFF
    seed = (seed ^ (seed >> 4)) & 0xFFFFFFFF
    seed = (seed * 0x27d4eb2d) & 0xFFFFFFFF
    seed = (seed ^ (seed >> 15)) & 0xFFFFFFFF
    return seed


def _unit_randoms(seed, n):
    out = []
    s = seed | 1
    for _ in range(n):
        s = _wang(s)
        out.append(s / 4294967296.0)
    return out


def icosphere(subdiv):
    """Vertices (unit sphere, float64) and faces of an icosahedron subdivided `subdiv` times: 20*4^subdiv faces."""
    t = (1.0 + np.sqrt(5.0)) / 2.0
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
         (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    verts = [np.array(p, dtype=np.float64) / np.sqrt(1.0 + t * t) for p in v]
    faces = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
             (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10),
             (8, 6, 7), (9, 8, 1)]
    for _ in range(subdiv):
        cache = {}
        new_faces = []

        def mid(a, b):
            key = (a, b) if a < b else (b, a)
            if key not in cache:
                m = verts[a] + verts[b]
                m = m / np.sqrt(np.dot(m, m))
                verts.append(m)
                cache[key] = len(verts) - 1
            return cache[key]

        for a, b, c in faces:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            new_faces += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        faces = new_faces
    return np.array(verts), faces


def _obj_text(verts, faces):
    lines = ["v %.6f %.6f %.6f" % (p[0], p[1], p[2]) for p in verts]
    lines += ["f %d %d %d" % (a + 1, b + 1, c + 1) for a, b, c in faces]
    return "\n".join(lines) + "\n"


_CACHE = {}


def blob_obj(subdiv=4, seed=7):
    """Bumpy icosphere: r = 1 + sum_k a_k * max(0, 1 - |v-c_k|^2 / r_k^2)^2 (polynomial bumps)."""
    key = ("blob", subdiv, seed)
    if key not in _CACHE:
        verts, faces = icosphere(subdiv)
        u = _unit_randoms(seed * 7919 + 13, 5 * 12)
        r = np.ones(len(verts))
        for k in range(12):
            c = np.array([u[5 * k] * 2 - 1, u[5 * k + 1] * 2 - 1, u[5 * k + 2] * 2 - 1])
            c = c / np.sqrt(np.dot(c, c) + 1e-9)
            amp = 0.15 + 0.3 * u[5 * k + 3]
            if k % 3 == 2:
                amp = -0.5 * amp
            rad2 = (0.35 + 0.5 * u[5 * k + 4]) ** 2
            d2 = ((verts - c) ** 2).sum(axis=1)
            w = np.maximum(0.0, 1.0 - d2 / rad2)
            r = r + amp * w * w
        _CACHE[key] = _obj_text(verts * r[:, None] * np.array([1.0, 1.15, 0.85]), faces)
    return _CACHE[key]


def bunny_obj():
    """The Stanford bunny asset as OBJ text ("%.9g" round-trips fp32)."""
    key = ("bunny",)
    if key not in _CACHE:
        z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "bunny.npz"))
        lines = ["v %.9g %.9g %.9g" % (p[0], p[1], p[2]) for p in z["verts"]]
        lines += ["f %d %d %d" % (a + 1, b + 1, c + 1) for a, b, c in z["faces"]]
        _CACHE[key] = "\n".join(lines) + "\n"
    return _CACHE[key]


def _unit_ymin(text):
    """Lowest y of a mesh after readObj's unit-box normalisation (identity transform): instances are set on the floor with it."""
    key = ("ymin", hash(text))
    if key not in _CACHE:
        tl = TriangleList()
        tl.read_obj_text(text, Material(), transform_matrix(), False)
        _CACHE[key] = float(tl.encode_triangles()[:, :9].reshape(-1, 3)[:, 1].min())
    return _CACHE[key]


def sphere_obj(subdiv=2):
    """320-triangle sphere (same count as the reference's sphere.obj)."""
    key = ("sphere", subdiv)
    if key not in _CACHE:
        verts, faces = icosphere(subdiv)
        _CACHE[key] = _obj_text(verts, faces)
    return _CACHE[key]


def box_obj():
    """Unit cube centred at the origin, 8 v / 12 f (stands for the reference's quad.obj box)."""
    v = [(-.5, -.5, -.5), (.5, -.5, -.5), (.5, .5, -.5), (-.5, .5, -.5), (-.5, -.5, .5), (.5, -.5, .5), (.5, .5, .5), (-.5, .5, .5)]
    f = [(0, 2, 1), (0, 3, 2), (4, 5, 6), (4, 6, 7), (0, 1, 5), (0, 5, 4), (3, 7, 6), (3, 6, 2), (0, 4, 7), (0, 7, 3), (1, 2, 6), (1, 6, 5)]
    return _obj_text(np.array(v, dtype=np.float64), f)


# Eight Disney parameter sets spanning the reference's scene set-ups (P4/main.cpp:690-727, P5/main.cpp:803-817)
MATERIAL_PRESETS = [
    Material(baseColor=(1.0, 0.73, 0.25), roughness=0.5, specular=1.0, metallic=1.0, clearcoat=1.0, clearcoatGloss=0.0),
    Material(baseColor=(1.0, 0.5, 0.5), roughness=0.1, metallic=0.0, clearcoat=1.0, subsurface=1.0),
    Material(baseColor=(0.75, 0.7, 0.15), roughness=0.15, metallic=1.0, clearcoat=1.0),
    Material(baseColor=(0.5, 0.5, 1.0), roughness=0.1, metallic=0.0, clearcoat=1.0),
    Material(baseColor=(0.725, 0.71, 0.68), roughness=0.5),
    Material(baseColor=(0.2, 0.8, 0.3), roughness=0.3, metallic=0.7, sheen=0.5, sheenTint=0.8),
    Material(baseColor=(0.9, 0.9, 0.9), roughness=0.05, metallic=0.9, specularTint=0.5, anisotropic=0.6),
    Material(baseColor=(0.8, 0.3, 0.1), roughness=0.7, subsurface=0.5, clearcoat=0.5, clearcoatGloss=0.3),
]


def bunny_meshes():
    """P3's scene with the blob in place of the bunny (P3/main.cpp:688-701) as readObj calls:
    [(obj text, Material, trans, smooth)]"""
    return [
        (blob_obj(), Material(baseColor=(1, 1, 1)), transform_matrix((0, 0, 0), (0.3, -0.65, 0.0), (1.5, 1.5, 1.5)), True),
        (box_obj(), Material(baseColor=(0.725, 0.71, 0.68)), transform_matrix((0, 0, 0), (0, -1.4, 0), (18.83, 0.01, 18.83)), False),
        (sphere_obj(), Material(baseColor=(1, 1, 1), emissive=(30, 20, 10)), transform_matrix((0, 0, 0), (0.0, 0.9, 0.0), (1, 1, 1)), False),
    ]


def s_bunny(builder=api.BVH_SAH_FAST):
    """bunny_meshes() built with the default leaf size.  Returns (tris, nodes, eye, cam)."""
    tl = TriangleList()
    for text, m, trans, smooth in bunny_meshes():
        tl.read_obj_text(text, m, trans, smooth)
    tris, nodes = tl.build_bvh(8, builder)
    eye, cam = api.camera_orbit(0.0, 0.0, 4.0)  # P3/main.cpp:148-150
    return tris, nodes, eye, cam


def grid_meshes(nx, nz, n_lights=4, pitch=1.2, mesh="blob", count=None):
    """Instances of `mesh` ("blob" | "bunny") in the first `count` (default all) row-major slots of an nx x nz grid
    (y-rotation 360*u0 and scale 0.8+0.4*u1 from successive wang_hash outputs of seed (id*9781+1)|1, material preset
    id%8), `n_lights` emissive spheres above it and a floor box, as readObj calls: [(obj text, Material, trans, smooth)]"""
    out = []
    text = blob_obj() if mesh == "blob" else bunny_obj()
    ymin = None if mesh == "blob" else _unit_ymin(text)
    count = nx * nz if count is None else count
    inst = 0
    for iz in range(nz):
        for ix in range(nx):
            if inst >= count:
                break
            u = _unit_randoms(inst * 9781 + 1, 2)
            rot = 360.0 * u[0]
            sc = 0.8 + 0.4 * u[1]
            x = (ix - (nx - 1) / 2.0) * pitch
            z = (iz - (nz - 1) / 2.0) * pitch
            m = MATERIAL_PRESETS[inst % 8]
            y = (-1.4 + 0.6 * sc) if ymin is None else (-1.395 - sc * ymin)  # feet on the floor (top face at y = -1.395)
            out.append((text, m, transform_matrix((0, rot, 0), (x, y, z), (sc, sc, sc)), True))
            inst += 1
    light = Material(baseColor=(1, 1, 1), emissive=(20, 20, 20))
    sph = sphere_obj()
    span_x, span_z = nx * pitch, nz * pitch
    for k in range(n_lights):
        lx = (((k % 2) * 2 - 1) * 0.25) * span_x
        lz = (((k // 2) * 2 - 1) * 0.25) * span_z
        out.append((sph, light, transform_matrix((0, 0, 0), (lx, 2.5, lz), (1.5, 1.5, 1.5)), False))
    floor = Material(baseColor=(0.725, 0.71, 0.68), roughness=0.3, metallic=0.1)
    ext = max(span_x, span_z) * 1.5 + 4.0
    out.append((box_obj(), floor, transform_matrix((0, 0, 0), (0, -1.4, 0), (ext, 0.01, ext)), False))
    return out


def s_grid(nx, nz, n_lights=4, builder=api.BVH_SAH_FAST, pitch=1.2, mesh="blob", count=None):
    """grid_meshes() built with the default leaf size.  Returns (tris, nodes, eye, cam)."""
    tl = TriangleList()
    for text, m, trans, smooth in grid_meshes(nx, nz, n_lights, pitch, mesh, count):
        tl.read_obj_text(text, m, trans, smooth)
    tris, nodes = tl.build_bvh(8, builder)
    r = 0.62 * max(nx * pitch, nz * pitch) + 3.0
    eye, cam = api.camera_orbit(30.0, 25.0, r)
    return tris, nodes, eye, cam


def s_1m(builder=api.BVH_SAH_FAST):
    """195 blobs (15 x 13) + 4 spheres + floor = 195*5120 + 1280 + 12 = 999,692 triangles."""
    return s_grid(15, 13, 4, builder)


def s_1m_bunny(builder=api.BVH_SAH_FAST):
    """S-1M of SURVEY.md 8(d): 201 Stanford bunnies (15 x 14 grid, first 201 slots) + 4 spheres + floor = 999,860 triangles,
    camera orbit rotatAngle 30, upAngle 25."""
    return s_grid(15, 14, 4, builder, mesh="bunny", count=201)


def lamps_meshes(nx, nz, pitch=1.2, mesh="blob", count=None, rough=False, seed=5):
    """grid_meshes(nx, nz, 0, ...) with a small emissive sphere (320 triangles, scale 0.2) at y = 0.4 over each instance, in place of
    the four big ones.  Lamp i's colour is 0.4 + 0.6 u (per channel) and its intensity 2 * 100^u' (2 to 200), from
    seeded uniforms; rough=True sets every instance's roughness to at least 0.5 and its metallic to at most 0.5."""
    out = grid_meshes(nx, nz, 0, pitch, mesh, count)
    floor = out.pop()
    if rough:
        out = [(t, Material(**{**m.__dict__, "roughness": max(m.roughness, 0.5), "metallic": min(m.metallic, 0.5)}), tr, sm)
               for t, m, tr, sm in out]
    n = len(out)
    u = np.array(_unit_randoms(seed * 7919 + 3, 4 * n)).reshape(n, 4)
    sph = sphere_obj()
    for i in range(n):
        ix, iz = i % nx, i // nx
        x = (ix - (nx - 1) / 2.0) * pitch
        z = (iz - (nz - 1) / 2.0) * pitch
        E = (0.4 + 0.6 * u[i, :3]) * (2.0 * 100.0 ** u[i, 3])
        out.append((sph, Material(baseColor=(1, 1, 1), emissive=tuple(float(e) for e in E)),
                    transform_matrix((0, 0, 0), (x, 0.4, z), (0.2, 0.2, 0.2)), False))
    out.append(floor)
    return out


def s_lamps(nx, nz, builder=api.BVH_SAH_FAST, pitch=1.2, mesh="blob", count=None, rough=False, seed=5):
    """lamps_meshes() built with the default leaf size, camera as s_grid.  Returns (tris, nodes, eye, cam)."""
    tl = TriangleList()
    for text, m, trans, smooth in lamps_meshes(nx, nz, pitch, mesh, count, rough, seed):
        tl.read_obj_text(text, m, trans, smooth)
    tris, nodes = tl.build_bvh(8, builder)
    r = 0.62 * max(nx * pitch, nz * pitch) + 3.0
    eye, cam = api.camera_orbit(30.0, 25.0, r)
    return tris, nodes, eye, cam


def s_1m_lamps(builder=api.BVH_SAH_FAST):
    """S-1M's 201 bunnies with a lamp over each (s_lamps): 201 * 4968 + 201 * 320 + 12 = 1,062,900 triangles, 64,320 of them lights."""
    return s_lamps(15, 14, builder, mesh="bunny", count=201)


def p3_bunny_meshes():
    """P3's scene block (P3/main.cpp:690-701) with the real bunny."""
    return [
        (bunny_obj(), Material(baseColor=(1, 1, 1)), transform_matrix((0, 0, 0), (0.3, -1.6, 0.0), (1.5, 1.5, 1.5)), True),
        (box_obj(), Material(baseColor=(0.725, 0.71, 0.68)), transform_matrix((0, 0, 0), (0, -1.4, 0), (18.83, 0.01, 18.83)), False),
        (sphere_obj(), Material(baseColor=(1, 1, 1), emissive=(30, 20, 10)), transform_matrix((0, 0, 0), (0.0, 0.9, 0.0), (1, 1, 1)), False),
    ]


def s_p3_bunny(builder=api.BVH_SAH_FAST):
    """Stanford bunny 4968 + floor 12 + emissive sphere 320 = 5300 triangles, eye (0,0,4) (P3/main.cpp:148-150)."""
    tl = TriangleList()
    for text, m, trans, smooth in p3_bunny_meshes():
        tl.read_obj_text(text, m, trans, smooth)
    tris, nodes = tl.build_bvh(8, builder)
    eye, cam = api.camera_orbit(0.0, 0.0, 4.0)
    return tris, nodes, eye, cam


def synth_hdr(width=512, height=256, seed=3, n_lamps=16):
    """Procedural environment map: vertical gradient 0.2 -> 1.0 plus polynomial-falloff 'lamps' (peak 500)."""
    ys = (np.arange(height, dtype=np.float64) + 0.5) / height
    xs = (np.arange(width, dtype=np.float64) + 0.5) / width
    base = 1.0 - 0.8 * ys  # row 0 = top (zenith) bright
    img = np.zeros((height, width, 3), dtype=np.float64)
    img[:, :, 0] = base[:, None] * 0.9
    img[:, :, 1] = base[:, None] * 0.95
    img[:, :, 2] = base[:, None] * 1.0
    u = _unit_randoms(seed * 104729 + 7, 4 * n_lamps)
    for k in range(n_lamps):
        cx, cy = u[4 * k], 0.05 + 0.45 * u[4 * k + 1]
        rad = 0.01 + 0.03 * u[4 * k + 2]
        peak = 500.0 * (0.3 + 0.7 * u[4 * k + 3])
        dx = np.abs(xs - cx)
        dx = np.minimum(dx, 1.0 - dx)
        d2 = (dx[None, :] ** 2) * 4.0 + (ys[:, None] - cy) ** 2
        w = np.maximum(0.0, 1.0 - d2 / (rad * rad))
        lamp = peak * w * w
        img[:, :, 0] += lamp
        img[:, :, 1] += lamp * 0.9
        img[:, :, 2] += lamp * 0.7
    return img.astype(np.float32)


def procedural_textures(n=2, seed=11):
    """n seeded sRGB textures for EZRT_PARAM_TEXTURES, uint8 [H, W, 3] each: even indices an 8x8 checker of two colours (256 x 256),
    odd indices bilinear value noise on a 16x16 lattice (128 x 192)."""
    out = []
    for k in range(n):
        h, w = (256, 256) if k % 2 == 0 else (128, 192)
        r = _unit_randoms(seed * 7919 + k, 6 + 17 * 17 * 3)
        ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
        if k % 2 == 0:
            c0, c1 = np.array(r[0:3]) * 255.0, np.array(r[3:6]) * 255.0
            on = ((ys * 8 // h) + (xs * 8 // w)) % 2 == 1
            img = np.where(on[:, :, None], c1, c0)
        else:
            lat = np.array(r[6:]).reshape(17, 17, 3)
            fy, fx = ys * 16.0 / h, xs * 16.0 / w
            iy, ix = fy.astype(int), fx.astype(int)
            ty, tx = (fy - iy)[:, :, None], (fx - ix)[:, :, None]
            a = lat[iy, ix] * (1 - tx) + lat[iy, ix + 1] * tx
            b = lat[iy + 1, ix] * (1 - tx) + lat[iy + 1, ix + 1] * tx
            img = (a * (1 - ty) + b * ty) * 255.0
        out.append(np.clip(np.rint(img), 0, 255).astype(np.uint8))
    return out



def obj_with_vt(text, projection):
    """OBJ text with a vt line per vertex and every face as "f a/a b/b c/c": projection "spherical" (u = 2 x longitude, v = latitude
    about the mesh's bounding-box centre) or "planar" (u, v = x, z over the mesh's extent, 8 repeats)."""
    lines = text.splitlines()
    v = np.array([[float(x) for x in l.split()[1:4]] for l in lines if l.startswith("v ")], np.float64)
    lo, hi = v.min(0), v.max(0)
    d = v - (lo + hi) / 2
    if projection == "spherical":
        u = np.arctan2(d[:, 2], d[:, 0]) / np.pi + 1.0
        w = np.arcsin(np.clip(d[:, 1] / np.maximum(np.linalg.norm(d, axis=1), 1e-12), -1, 1)) / np.pi + 0.5
    else:
        ext = np.maximum(hi - lo, 1e-12)
        u, w = 8.0 * (v[:, 0] - lo[0]) / ext[0], 8.0 * (v[:, 2] - lo[2]) / ext[2]
    out = [l for l in lines if l.startswith("v ")] + ["vt %.9g %.9g" % (a, b) for a, b in zip(u, w)]
    for l in lines:
        if l.startswith("f "):
            out.append("f " + " ".join("%s/%s" % (t, t) for t in l.split()[1:]))
    return "\n".join(out) + "\n"


def _textured_list(meshes, n_textures, emissive_uv=False):
    """meshes of p3_bunny_meshes / grid_meshes read as textured OBJ text: emissive meshes untextured (emissive_uv: with spherical UVs
    for their emission maps), flat boxes planar with the last texture id, the other meshes spherical with ids cycling over the others"""
    tl = TriangleList()
    k = 0
    for text, m, trans, smooth in meshes:
        if any(c > 0 for c in m.emissive):
            if emissive_uv:
                tl.read_obj_text(obj_with_vt(text, "spherical"), m, trans, smooth, texture_id=-1)
            else:
                tl.read_obj_text(text, m, trans, smooth)
        elif text == box_obj():
            tl.read_obj_text(obj_with_vt(text, "planar"), m, trans, smooth, texture_id=n_textures - 1)
        else:
            tl.read_obj_text(obj_with_vt(text, "spherical"), m, trans, smooth, texture_id=k % max(1, n_textures - 1))
            k += 1
    return tl


def s_p3_bunny_textured(n_textures=2, builder=api.BVH_SAH_FAST):
    """s_p3_bunny with texture coordinates read from OBJ vt lines (the bunny spherical, the floor planar, the light untextured) and
    seeded procedural textures.  Returns (tris, nodes, eye, cam, textures, texcoords [N, 3, 2], texture_id [N]); the geometry is
    s_p3_bunny's byte for byte."""
    tl = _textured_list(p3_bunny_meshes(), n_textures)
    tris, nodes = tl.build_bvh(8, builder)
    uv, ids = tl.encode_texcoords()
    eye, cam = api.camera_orbit(0.0, 0.0, 4.0)
    return tris, nodes, eye, cam, procedural_textures(n_textures), uv, ids


def s_1m_bunny_textured(n_textures=2, builder=api.BVH_SAH_FAST):
    """s_1m_bunny with texture coordinates read from OBJ vt lines, as s_p3_bunny_textured (the bunnies' ids cycle over all textures
    but the last, the floor's)."""
    tl = _textured_list(grid_meshes(15, 14, 4, 1.2, "bunny", 201), n_textures)
    tris, nodes = tl.build_bvh(8, builder)
    uv, ids = tl.encode_texcoords()
    eye, cam = api.camera_orbit(30.0, 25.0, 0.62 * max(15 * 1.2, 14 * 1.2) + 3.0)
    return tris, nodes, eye, cam, procedural_textures(n_textures), uv, ids


def height_normal_map(seed=21, size=128, cells=8, strength=2.0):
    """a tangent-space normal map for EZRT_PARAM_MATERIAL_MAPS (uint8 [size, size, 4], OpenGL +Y, linear): the finite differences of a
    seeded periodic value-noise height field, so that the map tiles under wrap addressing"""
    lat = np.random.default_rng(seed).uniform(0, 1, (cells + 1, cells + 1))
    lat[-1, :], lat[:, -1] = lat[0, :], lat[:, 0]
    ys, xs = np.meshgrid(np.arange(size) * cells / size, np.arange(size) * cells / size, indexing="ij")
    iy, ix = ys.astype(int), xs.astype(int)
    ty, tx = ys - iy, xs - ix
    h = (lat[iy, ix] * (1 - tx) + lat[iy, ix + 1] * tx) * (1 - ty) + (lat[iy + 1, ix] * (1 - tx) + lat[iy + 1, ix + 1] * tx) * ty
    dx = (np.roll(h, -1, axis=1) - np.roll(h, 1, axis=1)) * 0.5 * strength
    dy = (np.roll(h, 1, axis=0) - np.roll(h, -1, axis=0)) * 0.5 * strength   # row 0 is the image's top: +v is -row
    n = np.stack([-dx, -dy, np.ones_like(h)], axis=2)
    n /= np.linalg.norm(n, axis=2, keepdims=True)
    out = np.empty((size, size, 4), np.uint8)
    out[:, :, :3] = np.clip(np.rint((n * 0.5 + 0.5) * 255.0), 0, 255)
    out[:, :, 3] = 255
    return out


def noise_mr_map(seed=22, size=64, cells=4):
    """a metallic-roughness map for EZRT_PARAM_MATERIAL_MAPS (uint8 [size, size, 4], linear, glTF's channels): R 0, G (the roughness
    factor) and B (the metallic factor) seeded value noise"""
    rng = np.random.default_rng(seed)
    out = np.zeros((size, size, 4), np.uint8)
    ys, xs = np.meshgrid(np.arange(size) * cells / size, np.arange(size) * cells / size, indexing="ij")
    iy, ix = ys.astype(int), xs.astype(int)
    ty, tx = ys - iy, xs - ix
    for c in (1, 2):
        lat = rng.uniform(0, 1, (cells + 1, cells + 1))
        v = (lat[iy, ix] * (1 - tx) + lat[iy, ix + 1] * tx) * (1 - ty) + (lat[iy + 1, ix] * (1 - tx) + lat[iy + 1, ix + 1] * tx) * ty
        out[:, :, c] = np.clip(np.rint(v * 255.0), 0, 255)
    out[:, :, 3] = 255
    return out


def _with_maps(textured):
    """a textured scene (s_*_textured's tuple) plus the two procedural maps appended to its textures and their ids: every textured
    triangle takes both maps, except every 7th (no metallic-roughness map) and every 11th (no normal map); untextured ones (the
    lights) none"""
    tris, nodes, eye, cam, tex, uv, ids = textured
    n = len(tex)
    k = np.arange(len(ids))
    on = ids >= 0
    mr = np.where(on & (k % 7 != 0), n, -1).astype(np.int32)
    nm = np.where(on & (k % 11 != 0), n + 1, -1).astype(np.int32)
    return tris, nodes, eye, cam, tex + [noise_mr_map(), height_normal_map()], uv, ids, mr, nm


def s_p3_bunny_mapped(n_textures=2, builder=api.BVH_SAH_FAST):
    """s_p3_bunny_textured plus a seeded metallic-roughness map and a tangent-space normal map (EZRT_PARAM_MATERIAL_MAPS).  Returns
    (tris, nodes, eye, cam, textures, texcoords, texture_id, metal_rough_id, normal_id); the geometry is s_p3_bunny_textured's byte for
    byte, and the maps are the last two textures."""
    return _with_maps(s_p3_bunny_textured(n_textures, builder))


def s_1m_bunny_mapped(n_textures=2, builder=api.BVH_SAH_FAST):
    """s_1m_bunny_textured plus the maps of s_p3_bunny_mapped"""
    return _with_maps(s_1m_bunny_textured(n_textures, builder))


def punctual_rig(tris, seed=0, n_points=3, power=1.0):
    """A seeded rig of punctual lights for RenderConfig.punctual_lights (Scene.set_punctual_lights), placed from the triangles' bounds:
    a sun from above at a seeded slant, a key spot above and in front of the centre aimed at it, and n_points coloured point lights
    around the scene.  power scales every intensity (the units are the render's; the scene's extent sets the point lights' scale)."""
    v = np.asarray(tris, np.float32).reshape(-1, 36)[:, :9].reshape(-1, 3).astype(np.float64)
    lo, hi = v.min(axis=0), v.max(axis=0)
    c, r = 0.5 * (lo + hi), 0.5 * float(np.linalg.norm(hi - lo))
    rng = np.random.default_rng(seed)
    a = rng.uniform(0, 2 * np.pi)
    sun_dir = (0.4 * np.cos(a), -1.0, 0.4 * np.sin(a))
    lights = [api.directional_light(sun_dir, color=(1.0, 0.95, 0.85), intensity=1.5 * power)]
    key = c + np.array([0.3 * r, 1.2 * r, 1.2 * r])
    lights.append(api.spot_light(key, c - key, color=(1.0, 0.9, 0.8), intensity=4.0 * r * r * power, inner_cone=0.25, outer_cone=0.6))
    for k in range(n_points):
        phi = 2 * np.pi * (k + rng.uniform()) / max(1, n_points)
        pos = c + r * np.array([1.1 * np.cos(phi), rng.uniform(0.2, 0.9), 1.1 * np.sin(phi)])
        col = rng.uniform(0.3, 1.0, 3)
        lights.append(api.point_light(pos, color=tuple(col), intensity=float(rng.uniform(0.5, 1.5) * r * r * power)))
    return lights


def emission_bands(seed=31, size=(64, 128)):
    """a high-contrast emission texture for EZRT_PARAM_EMISSION_MAPS (uint8 [H, W, 3], sRGB): seeded bright coloured bands across u on
    black, wide enough gaps that some triangles of a mapped sphere are black at all 64 points of their table weight"""
    h, w = size
    rng = np.random.default_rng(seed)
    img = np.zeros((h, w, 3), np.uint8)
    x = int(rng.integers(0, 8))
    while x < w:
        on, off = int(rng.integers(3, 10)), int(rng.integers(10, 26))
        img[:, x:x + on] = rng.integers(150, 256, 3)
        x += on + off
    return img


def _emission_mapped(textured_list, n_textures, builder):
    tris, nodes = textured_list.build_bvh(8, builder)
    uv, ids = textured_list.encode_texcoords()
    emissive = np.asarray(tris, np.float32).reshape(-1, 36)[:, 18:21]
    eid = np.where((emissive > 0).any(axis=1), n_textures, -1).astype(np.int32)
    return tris, nodes, uv, ids, eid


def s_p3_bunny_emission_mapped(n_textures=2, builder=api.BVH_SAH_FAST):
    """s_p3_bunny_textured with the emissive sphere read with spherical UVs and mapped by emission_bands (EZRT_PARAM_EMISSION_MAPS).
    Returns (tris, nodes, eye, cam, textures, texcoords, texture_id, emission_id); the geometry is s_p3_bunny's byte for byte, and the
    emission texture is the last one."""
    tris, nodes, uv, ids, eid = _emission_mapped(_textured_list(p3_bunny_meshes(), n_textures, emissive_uv=True), n_textures, builder)
    eye, cam = api.camera_orbit(0.0, 0.0, 4.0)
    return tris, nodes, eye, cam, procedural_textures(n_textures) + [emission_bands()], uv, ids, eid


def s_1m_bunny_emission_mapped(n_textures=2, builder=api.BVH_SAH_FAST):
    """s_1m_bunny_textured with its four emissive spheres mapped as s_p3_bunny_emission_mapped's; the geometry is s_1m_bunny's"""
    tl = _textured_list(grid_meshes(15, 14, 4, 1.2, "bunny", 201), n_textures, emissive_uv=True)
    tris, nodes, uv, ids, eid = _emission_mapped(tl, n_textures, builder)
    eye, cam = api.camera_orbit(30.0, 25.0, 0.62 * max(15 * 1.2, 14 * 1.2) + 3.0)
    return tris, nodes, eye, cam, procedural_textures(n_textures) + [emission_bands()], uv, ids, eid


def screen_image(seed=41, size=(72, 128)):
    """an image-like emission texture (uint8 [H, W, 3], sRGB): a seeded colour gradient with dark window bars and a few bright discs"""
    h, w = size
    rng = np.random.default_rng(seed)
    ys, xs = np.meshgrid(np.arange(h) / h, np.arange(w) / w, indexing="ij")
    c0, c1 = rng.uniform(0.2, 1.0, 3), rng.uniform(0.2, 1.0, 3)
    img = c0 * (1 - xs[..., None]) + c1 * xs[..., None]
    img *= (1.0 - 0.8 * ((ys * 6) % 1.0 < 0.15))[..., None]
    for _ in range(4):
        cy, cx, r = rng.uniform(0, 1), rng.uniform(0, 1), rng.uniform(0.05, 0.15)
        img[(ys - cy) ** 2 + ((xs - cx) * w / h) ** 2 < r * r] = rng.uniform(0.7, 1.0, 3)
    return np.clip(np.rint(img * 255.0), 0, 255).astype(np.uint8)


def screen_obj(width=3.0, height=1.8):
    """a quad in the z = 0 plane facing +z, centred at the origin, with UVs 0..1 (v = 0 at its bottom), as OBJ text"""
    x, y = width / 2.0, height / 2.0
    return ("v %r %r 0\nv %r %r 0\nv %r %r 0\nv %r %r 0\nvt 0 0\nvt 1 0\nvt 1 1\nvt 0 1\nf 1/1 2/2 3/3\nf 1/1 3/3 4/4\n"
            % (-x, -y, x, -y, x, y, -x, y))


def s_screen(bunny=True, builder=api.BVH_SAH_FAST, emission=(6.0, 6.0, 6.0)):
    """a "screen": a 3 x 1.8 quad emitter standing at the back edge of a floor, facing +z, mapped with screen_image, and the bunny
    (bunny=True) on the floor in front of it, lit by it and shadowing the floor in front.  readObj normalises every mesh to its unit
    box, so the meshes' sizes are set by their transforms' scales.
    Returns (tris, nodes, eye, cam, textures [screen_image()], texcoords, texture_id (all -1), emission_id (the quad 0, others -1))."""
    tl = TriangleList()
    top = -1.395   # the floor's top face
    # the floor ends at the screen's plane, so that no surface sees the screen's back
    floor = (box_obj(), Material(baseColor=(0.725, 0.71, 0.68)), transform_matrix((0, 0, 0), (0, -1.4, 1.8), (8.0, 0.01, 6.0)), False)
    meshes = [floor]
    if bunny:
        text, m, _, smooth = p3_bunny_meshes()[0]
        meshes.append((text, m, transform_matrix((0, 0, 0), (0.3, top - 1.5 * _unit_ymin(text), -0.2), (1.5, 1.5, 1.5)), smooth))
    for text, m, trans, smooth in meshes:
        tl.read_obj_text(obj_with_vt(text, "planar"), m, trans, smooth, texture_id=-1)
    tl.read_obj_text(screen_obj(), Material(baseColor=(0, 0, 0), emissive=tuple(emission)),
                     transform_matrix((0, 0, 0), (0.0, top + 0.95, -1.2), (3.0, 3.0, 3.0)), False, texture_id=-1)
    tris, nodes, uv, ids, eid = _emission_mapped(tl, 0, builder)
    eye, cam = api.camera_orbit(0.0, 15.0, 4.0)
    return tris, nodes, eye, cam, [screen_image()], uv, ids, eid


def smoke_grid(n=64, seed=0):
    """A seeded procedural plume for EZRT_PARAM_MEDIUM_GRID: float32 [n, n, n] densities ([z, y, x]) in [0, 1], deterministic in
    numpy.  Four octaves of value noise (seeded lattices of 4, 8, 16 and 32 cells, trilinearly upsampled; weights 1/2, 1/4, ...) shape a
    column that narrows and thins with height (y) and is empty near the grid's faces."""
    rng = np.random.default_rng(seed)
    t = np.linspace(0.0, 1.0, n)
    noise = np.zeros((n, n, n))
    for octave, cells in enumerate((4, 8, 16, 32)):
        lat = rng.random((cells + 1,) * 3)
        u = t * cells
        i = np.minimum(u.astype(np.int64), cells - 1)
        f = u - i
        acc = np.zeros((n, n, n))
        for dz in (0, 1):
            for dy in (0, 1):
                for dx in (0, 1):
                    w = (f if dz else 1 - f)[:, None, None] * (f if dy else 1 - f)[None, :, None] * (f if dx else 1 - f)[None, None, :]
                    acc += w * lat[np.ix_(i + dz, i + dy, i + dx)]
        noise += acc * 0.5 ** (octave + 1)
    z, y, x = np.meshgrid(t, t, t, indexing="ij")
    radius = 0.35 - 0.2 * y
    r2 = (x - 0.5) ** 2 + (z - 0.5) ** 2
    shape = np.clip(1.0 - r2 / radius ** 2, 0.0, None) * np.clip(1.0 - y, 0.0, None)
    return np.clip(shape * (2.0 * noise - 0.3), 0.0, None).astype(np.float32)


def s_p3_bunny_smoke(n=64, seed=0, sigma_t=6.0, builder=api.BVH_SAH_FAST):
    """s_p3_bunny with a smoke plume over the bunny: (tris, nodes, eye, cam, medium, grid), medium the keyword arguments of
    Scene.set_medium (its box holds the plume) and grid smoke_grid(n, seed)."""
    tris, nodes, eye, cam = s_p3_bunny(builder)
    medium = dict(sigma_t=sigma_t, albedo=(0.9, 0.9, 0.9), g=0.3, box_min=(-1.0, -1.0, -1.0), box_max=(1.0, 1.2, 1.0))
    return tris, nodes, eye, cam, medium, smoke_grid(n, seed)


def s_1m_smoke(n=128, seed=0, sigma_t=1.0, builder=api.BVH_SAH_FAST):
    """S-1M (s_1m) with a plume over its bounds: (tris, nodes, eye, cam, medium, grid) as s_p3_bunny_smoke."""
    tris, nodes, eye, cam = s_1m(builder)
    v = np.asarray(tris, np.float32).reshape(-1, 36)[:, :9].reshape(-1, 3)
    lo, hi = v.min(0), v.max(0)
    medium = dict(sigma_t=sigma_t, albedo=(0.9, 0.9, 0.9), g=0.3, box_min=tuple(lo), box_max=tuple(hi))
    return tris, nodes, eye, cam, medium, smoke_grid(n, seed)
