"""Host-side mirror of the reference's main()/display() for the path-tracing hot path.

Names follow the reference (P5/main.cpp): Material, readObj -> TriangleList.read_obj,
getTransformMatrix -> transform_matrix, buildBVHwithSAH -> TriangleList.build_bvh,
calculateHdrCache -> hdr_cache, display() -> Scene.render.  Everything calls the C ABI of
include/ezrt.h through ctypes; numpy carries host arrays, torch (optional) carries device
framebuffers and streams.
"""
import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _lib
from ._lib import AdaptiveParams, Counters, DenoiseParams, EzrtError, Medium, RenderParams, Texture, check, lib

MODE_DIFFUSE_P3 = 0
MODE_DISNEY_ANISO_P4 = 1
MODE_DISNEY_SOBOL_P5 = 2
MODE_DISNEY_IS_MIS_P5 = 3
MODE_DISNEY_LIGHTS = 4   # BRDF sampling + light sampling on the emissive triangles, MIS (DESIGN.md section 10)
PARAM_ACCUMULATE = 1   # ezrt_render_params.reserved[0] flags (include/ezrt.h)
PARAM_ENV_LIGHT = 2
PARAM_TRANSMISSION = 4
PARAM_THIN_LENS = 8
PARAM_MEDIUM = 16
PARAM_TEXTURES = 32
PARAM_MATERIAL_MAPS = 64
MODES = {"diffuse_p3": 0, "disney_aniso_p4": 1, "disney_sobol_p5": 2, "disney_is_mis_p5": 3, "disney_lights": 4}

TRAVERSE_ACCEL = 0
TRAVERSE_REFERENCE = 1
TRAVERSE_PRUNED = 2
PIPELINE_WAVEFRONT = 0
PIPELINE_MEGAKERNEL = 1

BVH_SAH_FAST = 0
BVH_SAH_LITERAL = 1
BVH_MEDIAN = 2

TRIANGLE_FLOATS = 36
BVHNODE_FLOATS = 12


def _fp(a):
    return a.ctypes.data_as(_lib.c_float_p)


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    if shape is not None:
        a = a.reshape(shape)
    return a


@dataclass
class Material:
    """struct Material, P5/main.cpp:27-42 (same defaults)."""
    emissive: tuple = (0.0, 0.0, 0.0)
    baseColor: tuple = (1.0, 1.0, 1.0)
    subsurface: float = 0.0
    metallic: float = 0.0
    specular: float = 0.5
    specularTint: float = 0.0
    roughness: float = 0.5
    anisotropic: float = 0.0
    sheen: float = 0.0
    sheenTint: float = 0.5
    clearcoat: float = 0.0
    clearcoatGloss: float = 1.0
    IOR: float = 1.0
    transmission: float = 0.0

    def as_array(self):
        return np.array(list(self.emissive) + list(self.baseColor) + [
            self.subsurface, self.metallic, self.specular, self.specularTint, self.roughness, self.anisotropic,
            self.sheen, self.sheenTint, self.clearcoat, self.clearcoatGloss, self.IOR, self.transmission], dtype=np.float32)


def transform_matrix(rotate=(0, 0, 0), translate=(0, 0, 0), scale=(1, 1, 1)):
    """getTransformMatrix(rotateCtrl, translateCtrl, scaleCtrl), P5/main.cpp:255-271 -> 16 floats, column-major."""
    out = np.zeros(16, dtype=np.float32)
    lib.ezrt_transform_matrix(_fp(_f32(rotate)), _fp(_f32(translate)), _fp(_f32(scale)), _fp(out))
    return out


def camera_orbit(rotate_angle=0.0, up_angle=0.0, r=4.0):
    """eye / cameraRotate of display(), P5/main.cpp:710-713."""
    eye = np.zeros(3, dtype=np.float32)
    cam = np.zeros(16, dtype=np.float32)
    lib.ezrt_camera_orbit(float(rotate_angle), float(up_angle), float(r), _fp(eye), _fp(cam))
    return eye, cam


def camera_look_at(eye, target=(0.0, 0.0, 0.0), up=(0.0, 1.0, 0.0), vfov=67.38013505195957, aspect=1.0):
    """(eye, cameraRotate) of a look-at camera with a vertical field of view vfov (degrees) and aspect = width / height
    (ezrt_camera_look_at).  The default vfov, 2 atan(2/3), is the pinhole's own: camera_orbit's view."""
    e = _f32(eye, (3,))
    cam = np.zeros(16, dtype=np.float32)
    check(lib.ezrt_camera_look_at(_fp(e), _fp(_f32(target, (3,))), _fp(_f32(up, (3,))), float(vfov), float(aspect), _fp(cam)))
    return e.copy(), cam


class TriangleList:
    """std::vector<Triangle> triangles of main() (P5/main.cpp:801) plus its BVH."""

    def __init__(self):
        self._h = lib.ezrt_trilist_create()
        if not self._h:
            raise MemoryError("ezrt_trilist_create")

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            lib.ezrt_trilist_destroy(h)

    def __len__(self):
        return check(lib.ezrt_trilist_size(self._h))

    def read_obj(self, path, material, trans, smooth_normal, texture_id=None):
        """readObj(filepath, triangles, material, trans, smoothNormal), P5/main.cpp:274-392.  texture_id (an int >= -1): also read the
        mesh's vt coordinates (ezrt_trilist_read_obj_textured); its triangles get that texture id where all three vertices carry a vt."""
        if texture_id is None:
            check(lib.ezrt_trilist_read_obj(self._h, str(path).encode(), _fp(material.as_array()), _fp(_f32(trans)), int(smooth_normal)))
        else:
            check(lib.ezrt_trilist_read_obj_textured(self._h, str(path).encode(), _fp(material.as_array()), _fp(_f32(trans)), int(smooth_normal),
                                                     int(texture_id)))
        return self

    def read_obj_text(self, text, material, trans, smooth_normal, texture_id=None):
        data = text.encode() if isinstance(text, str) else bytes(text)
        if texture_id is None:
            check(lib.ezrt_trilist_read_obj_text(self._h, data, len(data), _fp(material.as_array()), _fp(_f32(trans)), int(smooth_normal)))
        else:
            check(lib.ezrt_trilist_read_obj_textured_text(self._h, data, len(data), _fp(material.as_array()), _fp(_f32(trans)),
                                                          int(smooth_normal), int(texture_id)))
        return self

    def encode_texcoords(self):
        """(uv [N, 3, 2], texture id [N]) of the triangles in the list's current order (after build_bvh: the encoded triangles')."""
        uv = np.zeros((len(self), 3, 2), dtype=np.float32)
        ids = np.zeros(len(self), dtype=np.int32)
        check(lib.ezrt_trilist_encode_texcoords(self._h, _fp(uv), ids.ctypes.data_as(C.POINTER(C.c_int32))))
        return uv, ids

    def append_encoded(self, tris):
        tris = _f32(tris, (-1, TRIANGLE_FLOATS))
        check(lib.ezrt_trilist_append_encoded(self._h, _fp(tris), tris.shape[0]))
        return self

    def build_bvh(self, leaf_n=8, builder=BVH_SAH_FAST):
        """nodes{testNode}; buildBVHwithSAH(triangles, nodes, 0, N-1, 8) + encode (P5/main.cpp:830-871).
        Returns (triangles_encoded [N,36], nodes_encoded [M,12])."""
        n_nodes = check(lib.ezrt_trilist_build_bvh(self._h, int(leaf_n), int(builder)))
        return self.encode_triangles(), self.encode_nodes(n_nodes)

    def encode_triangles(self):
        out = np.zeros((len(self), TRIANGLE_FLOATS), dtype=np.float32)
        check(lib.ezrt_trilist_encode_triangles(self._h, _fp(out)))
        return out

    def encode_nodes(self, n_nodes=None):
        if n_nodes is None:
            n_nodes = check(lib.ezrt_trilist_node_count(self._h))
        out = np.zeros((n_nodes, BVHNODE_FLOATS), dtype=np.float32)
        check(lib.ezrt_trilist_encode_nodes(self._h, _fp(out)))
        return out


OBJ_HARDENED = 2


def host_sort_is_reference():
    """True if this host's std::sort reproduces libstdc++'s order of equal keys, i.e. build_bvh yields the reference's
    triangle order (ezrt_host_sort_is_reference, include/ezrt.h)."""
    return bool(lib.ezrt_host_sort_is_reference())


def load_scene_file(path):
    """Scene description file -> (TriangleList, (rotatAngle, upAngle, r), hdr path or None); see include/ezrt.h."""
    tl = TriangleList()
    cam = np.zeros(3, dtype=np.float32)
    buf = C.create_string_buffer(4096)
    check(lib.ezrt_scene_file_load(str(path).encode(), tl._h, _fp(cam), buf, 4096))
    hdr = buf.value.decode() or None
    return tl, tuple(float(x) for x in cam), hdr


def hdr_load(path):
    """HDRLoader::load, P5/lib/hdrloader.cpp:29-97 -> float32 [h, w, 3], row 0 = first scanline."""
    w, h = C.c_int(0), C.c_int(0)
    check(lib.ezrt_hdr_load(str(path).encode(), C.byref(w), C.byref(h), None))
    cols = np.zeros((h.value, w.value, 3), dtype=np.float32)
    check(lib.ezrt_hdr_load(str(path).encode(), C.byref(w), C.byref(h), _fp(cols)))
    return cols


def hdr_cache(hdr):
    """calculateHdrCache(HDR, width, height), P5/main.cpp:592-689."""
    hdr = _f32(hdr)
    h, w = hdr.shape[0], hdr.shape[1]
    out = np.zeros((h, w, 3), dtype=np.float32)
    check(lib.ezrt_hdr_cache(_fp(hdr), w, h, _fp(out)))
    return out


def hdr_cache_device(hdr, device=0):
    """calculateHdrCache on the GPU (bit-identical to hdr_cache).  Returns (cache, kernel milliseconds)."""
    hdr = _f32(hdr)
    h, w = hdr.shape[0], hdr.shape[1]
    out = np.zeros((h, w, 3), dtype=np.float32)
    ms = C.c_double(0.0)
    check(lib.ezrt_hdr_cache_device(int(device), _fp(hdr), w, h, _fp(out), C.byref(ms)))
    return out, ms.value


def partition_pixels(width, height, rank, count):
    return int(check(lib.ezrt_partition_pixels(width, height, rank, count)))


def partition_scatter_host(compact, full, width, height, channels, rank, count):
    compact = _f32(compact)
    assert full.dtype == np.float32 and full.flags.c_contiguous
    check(lib.ezrt_partition_scatter_host(_fp(compact), _fp(full), width, height, channels, rank, count))
    return full


@dataclass
class RenderConfig:
    """The uniforms display() sets plus the shader literals (ezrt_render_params)."""
    width: int = 512
    height: int = 512
    spp: int = 1
    first_frame: int = 0
    max_bounce: int = 2
    mode: int = MODE_DISNEY_SOBOL_P5
    eye: tuple = (0.0, 0.0, 4.0)
    camera_rotate: tuple = tuple(np.eye(4, dtype=np.float32).reshape(-1))
    env_color: tuple = (0.0, 0.0, 0.0)
    traverse: int = TRAVERSE_ACCEL
    pipeline: int = PIPELINE_WAVEFRONT
    out_channels: int = 3
    part_rank: int = 0
    part_count: int = 1
    frames_per_batch: int = 0
    profile: int = 0
    accumulate: bool = False   # EZRT_PARAM_ACCUMULATE: counters / kernel times continue from the previous render
    env_light: bool = False    # EZRT_PARAM_ENV_LIGHT (MODE_DISNEY_LIGHTS only): the HDR map is one more light (DESIGN.md section 11)
    transmission: bool = False  # EZRT_PARAM_TRANSMISSION (MODE_DISNEY_LIGHTS only): materials' IOR and transmission (DESIGN.md section 12)
    lens_radius: float = 0.0    # != 0: EZRT_PARAM_THIN_LENS, a thin-lens camera of this radius (DESIGN.md section 13); must be > 0
    focus_distance: float = None  # ... focused at this depth along the view (-column 2 of camera_rotate); required with a lens
    medium: bool = False        # EZRT_PARAM_MEDIUM (MODE_DISNEY_LIGHTS only): the scene's homogeneous medium (Scene.set_medium, DESIGN.md section 14)
    textures: bool = False      # EZRT_PARAM_TEXTURES (MODE_DISNEY_LIGHTS only): the scene's base-colour textures (Scene.set_textures, DESIGN.md section 15)
    material_maps: bool = False  # EZRT_PARAM_MATERIAL_MAPS (with textures): the scene's material maps (Scene.set_material_maps, DESIGN.md section 16)

    def to_struct(self):
        p = RenderParams()
        p.width, p.height, p.spp, p.first_frame = int(self.width), int(self.height), int(self.spp), int(self.first_frame)
        p.max_bounce, p.mode = int(self.max_bounce), int(self.mode)
        p.eye[:] = [float(x) for x in self.eye]
        p.camera_rotate[:] = [float(x) for x in np.asarray(self.camera_rotate, dtype=np.float32).reshape(-1)]
        p.env_color[:] = [float(x) for x in self.env_color]
        p.traverse, p.pipeline, p.out_channels = int(self.traverse), int(self.pipeline), int(self.out_channels)
        p.part_rank, p.part_count, p.frames_per_batch = int(self.part_rank), int(self.part_count), int(self.frames_per_batch)
        p.profile = int(self.profile)
        p.reserved[0] = ((PARAM_ACCUMULATE if self.accumulate else 0) | (PARAM_ENV_LIGHT if self.env_light else 0) |
                         (PARAM_TRANSMISSION if self.transmission else 0) | (PARAM_MEDIUM if self.medium else 0) |
                         (PARAM_TEXTURES if self.textures else 0) | (PARAM_MATERIAL_MAPS if self.material_maps else 0))
        if self.lens_radius != 0:   # a negative or NaN radius is set too, so that the library rejects it
            if self.focus_distance is None:
                raise ValueError("RenderConfig: a lens (lens_radius != 0) needs a focus_distance")
            p.reserved[0] |= PARAM_THIN_LENS
            p.reserved[1], p.reserved[2] = (int(x) for x in np.array([self.lens_radius, self.focus_distance], np.float32).view(np.int32))
        return p


def adaptive_params(threshold, min_spp, check_interval):
    """struct ezrt_adaptive_params (include/ezrt.h)."""
    a = AdaptiveParams()
    a.threshold, a.min_spp, a.check_interval, a.reserved = float(threshold), int(min_spp), int(check_interval), 0
    return a


# defaults of the denoiser (ezrt_denoise_params, DESIGN.md section 9)
DENOISE_DEFAULTS = dict(iterations=5, sigma_l=4.0, sigma_n=128.0, sigma_z=1.0, sigma_a=0.1)
AOV_CHANNELS = 8   # albedo.rgb, coverage, normal.xyz, depth


def denoise_params(iterations=5, sigma_l=4.0, sigma_n=128.0, sigma_z=1.0, sigma_a=0.1):
    """struct ezrt_denoise_params (include/ezrt.h)."""
    d = DenoiseParams()
    d.iterations, d.sigma_l, d.sigma_n, d.sigma_z, d.sigma_a, d.reserved = int(iterations), float(sigma_l), float(sigma_n), float(sigma_z), \
        float(sigma_a), 0
    return d


class Scene:
    """Device-resident scene: the two texture buffers + two HDR textures of P5/main.cpp:878-906."""

    def __init__(self, tris, nodes, hdr=None, hdr_cache_=None, device=0, hdr_filter_linear=True):
        self.tris = _f32(tris, (-1, TRIANGLE_FLOATS))
        self.nodes = _f32(nodes, (-1, BVHNODE_FLOATS))
        self.hdr = None if hdr is None else _f32(hdr)
        self.hdr_cache = None if hdr_cache_ is None else _f32(hdr_cache_)
        self.device = int(device)
        hw = hh = 0
        if self.hdr is not None:
            hh, hw = self.hdr.shape[0], self.hdr.shape[1]
        elif self.hdr_cache is not None:
            hh, hw = self.hdr_cache.shape[0], self.hdr_cache.shape[1]
        self._h = C.c_void_p()
        check(lib.ezrt_scene_create(self.device, _fp(self.tris), self.tris.shape[0], _fp(self.nodes), self.nodes.shape[0],
                                    None if self.hdr is None else _fp(self.hdr),
                                    None if self.hdr_cache is None else _fp(self.hdr_cache), hw, hh,
                                    int(bool(hdr_filter_linear)), C.byref(self._h)))

    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            lib.ezrt_scene_destroy(h)

    __del__ = close

    def set_medium(self, sigma_t, albedo=(1.0, 1.0, 1.0), g=0.0, box_min=None, box_max=None):
        """ezrt_scene_set_medium: the homogeneous medium RenderConfig.medium renders -- grey extinction sigma_t, RGB albedo,
        Henyey-Greenstein g, filling the box [box_min, box_max] (DESIGN.md section 14; both corners required).  set_medium(None)
        clears it.  Renders already enqueued keep the medium they were enqueued with."""
        if sigma_t is None:
            check(lib.ezrt_scene_set_medium(self._h, None))
            return
        if box_min is None or box_max is None:
            raise ValueError("Scene.set_medium: box_min and box_max are required (the medium fills that box)")
        m = Medium()
        m.sigma_t, m.g, m.reserved = float(sigma_t), float(g), 0
        m.albedo[:] = [float(x) for x in albedo]
        m.box_min[:] = [float(x) for x in box_min]
        m.box_max[:] = [float(x) for x in box_max]
        check(lib.ezrt_scene_set_medium(self._h, C.byref(m)))

    def set_textures(self, textures, texcoords=None, texture_id=None):
        """ezrt_scene_set_textures: the base-colour textures RenderConfig.textures renders (DESIGN.md section 15).  textures: uint8
        arrays [H, W, 3] or [H, W, 4] (row 0 on top, sRGB; alpha ignored; padded to RGBA); texcoords [N, 3, 2] or [N, 6] float (u, v
        per vertex, v = 0 at the image's bottom) and texture_id [N] int (-1: untextured), in the order of the scene's triangles.
        set_textures(None) clears them; with textures, texcoords and texture_id are required.  The call waits for the renders already enqueued on the device."""
        if textures is None:
            check(lib.ezrt_scene_set_textures(self._h, 0, None, None, None))
            return
        if texcoords is None or texture_id is None:
            raise ValueError("Scene.set_textures: texcoords and texture_id are required with textures")
        n = self.tris.shape[0]
        uv = np.ascontiguousarray(np.asarray(texcoords, np.float32).reshape(n, 6))
        ids = np.ascontiguousarray(np.asarray(texture_id, np.int32).reshape(n))
        keep, arr = [], (Texture * max(1, len(textures)))()
        for k, t in enumerate(textures):
            t = np.asarray(t)
            if t.dtype != np.uint8 or t.ndim != 3 or t.shape[2] not in (3, 4):
                raise ValueError("Scene.set_textures: texture %d must be a uint8 array [H, W, 3|4], got %s %s" % (k, t.dtype, t.shape))
            if t.shape[2] == 3:
                t = np.concatenate([t, np.full(t.shape[:2] + (1,), 255, np.uint8)], axis=2)
            t = np.ascontiguousarray(t)
            keep.append(t)
            arr[k].width, arr[k].height, arr[k].rgba, arr[k].reserved = t.shape[1], t.shape[0], t.ctypes.data, 0
        check(lib.ezrt_scene_set_textures(self._h, len(textures), arr, _fp(uv), ids.ctypes.data_as(C.POINTER(C.c_int32))))

    def sample_textures(self, tri, points):
        """ezrt_scene_sample_textures: the device's UV ([n, 2]) and textured base colour ([n, 3]) at points ([n, 3]) on reference triangles."""
        tri = np.ascontiguousarray(np.asarray(tri, np.int32).reshape(-1))
        pts = np.ascontiguousarray(np.asarray(points, np.float32).reshape(-1, 3))
        assert pts.shape[0] == tri.shape[0]
        uv = np.zeros((tri.shape[0], 2), np.float32)
        rgb = np.zeros((tri.shape[0], 3), np.float32)
        check(lib.ezrt_scene_sample_textures(self._h, tri.shape[0], tri.ctypes.data_as(C.POINTER(C.c_int32)), _fp(pts), _fp(uv), _fp(rgb)))
        return uv, rgb

    def set_material_maps(self, metal_rough_id, normal_id=None):
        """ezrt_scene_set_material_maps: the material maps RenderConfig.material_maps renders (DESIGN.md section 16).  metal_rough_id and
        normal_id [N] int: per triangle (in the order of the scene's triangles) the ids of its metallic-roughness and normal maps among
        the textures of set_textures (-1: no map).  set_material_maps(None) clears them.  set_textures clears them too."""
        if metal_rough_id is None:
            check(lib.ezrt_scene_set_material_maps(self._h, None, None))
            return
        if normal_id is None:
            raise ValueError("Scene.set_material_maps: normal_id is required with metal_rough_id")
        n = self.tris.shape[0]
        mr = np.ascontiguousarray(np.asarray(metal_rough_id, np.int32).reshape(n))
        nm = np.ascontiguousarray(np.asarray(normal_id, np.int32).reshape(n))
        check(lib.ezrt_scene_set_material_maps(self._h, mr.ctypes.data_as(C.POINTER(C.c_int32)), nm.ctypes.data_as(C.POINTER(C.c_int32))))

    def sample_materials(self, tri, o, d, t):
        """ezrt_scene_sample_materials: what the maps renders compute at hits of reference triangles tri ([n]) by rays (o [n, 3], d [n, 3],
        t [n]): a dict of uv [n, 2], base_color [n, 3], roughness [n], metallic [n] and normal [n, 3] (the final shading normal)."""
        tri = np.ascontiguousarray(np.asarray(tri, np.int32).reshape(-1))
        n = tri.shape[0]
        hits = np.ascontiguousarray(np.concatenate([np.asarray(o, np.float32).reshape(n, 3), np.asarray(d, np.float32).reshape(n, 3),
                                                    np.asarray(t, np.float32).reshape(n, 1)], axis=1))
        out = np.zeros((n, 10), np.float32)
        check(lib.ezrt_scene_sample_materials(self._h, n, tri.ctypes.data_as(C.POINTER(C.c_int32)), _fp(hits), _fp(out)))
        return dict(uv=out[:, 0:2], base_color=out[:, 2:5], roughness=out[:, 5], metallic=out[:, 6], normal=out[:, 7:10])

    def render(self, cfg, framebuffer=None):
        """render(width, height, spp) -> framebuffer: `spp` display() calls through HOST buffers
        (H2D of lastFrame when first_frame > 0, D2H of the result, synchronous)."""
        n = partition_pixels(cfg.width, cfg.height, cfg.part_rank, cfg.part_count)
        if framebuffer is None:
            framebuffer = np.zeros((n, cfg.out_channels), dtype=np.float32)
        assert framebuffer.dtype == np.float32 and framebuffer.size == n * cfg.out_channels and framebuffer.flags.c_contiguous
        p = cfg.to_struct()
        check(lib.ezrt_render(self._h, C.byref(p), _fp(framebuffer)))
        if cfg.part_count == 1:
            return framebuffer.reshape(cfg.height, cfg.width, cfg.out_channels)
        return framebuffer

    def render_device(self, cfg, d_framebuffer, stream=None):
        """Enqueue the render on a CUDA stream into a device buffer (torch tensor or raw pointer)."""
        ptr = d_framebuffer.data_ptr() if hasattr(d_framebuffer, "data_ptr") else int(d_framebuffer)
        st = 0 if stream is None else (stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream))
        p = cfg.to_struct()
        check(lib.ezrt_render_device(self._h, C.byref(p), C.c_void_p(ptr), C.c_void_p(st)))
        return d_framebuffer

    def render_adaptive(self, cfg, threshold, min_spp=16, check_interval=16):
        """Tile-adaptive render from frame 0 (ezrt_render_adaptive): cfg.spp is the frame cap; a 16x16 tile stops at the
        first test (after min_spp, then every check_interval frames) at which every pixel's relative standard error of
        luminance is <= threshold.  Returns host arrays (image, spp_map, luma2): [H, W, C], [H, W], [H, W] for one part,
        compact tile-major [n, C], [n], [n] otherwise.  spp_map = frames each pixel received, luma2 = running mean of the
        squared sample luminance."""
        n = partition_pixels(cfg.width, cfg.height, cfg.part_rank, cfg.part_count)
        img = np.zeros((n, cfg.out_channels), dtype=np.float32)
        spp = np.zeros(n, dtype=np.int32)
        luma2 = np.zeros(n, dtype=np.float32)
        p, a = cfg.to_struct(), adaptive_params(threshold, min_spp, check_interval)
        check(lib.ezrt_render_adaptive(self._h, C.byref(p), C.byref(a), _fp(img), spp.ctypes.data_as(_lib.c_int32_p), _fp(luma2)))
        if cfg.part_count == 1:
            return img.reshape(cfg.height, cfg.width, cfg.out_channels), spp.reshape(cfg.height, cfg.width), luma2.reshape(cfg.height, cfg.width)
        return img, spp, luma2

    def render_adaptive_device(self, cfg, threshold, min_spp, check_interval, d_framebuffer, d_spp, d_luma2, stream=None):
        """Enqueue a tile-adaptive render on a CUDA stream into device buffers (torch tensors or raw pointers): the
        framebuffer, int32 frames per pixel, float32 running mean of the squared luminance.  Synchronises the stream once per test."""
        ptr = lambda t: t.data_ptr() if hasattr(t, "data_ptr") else int(t)
        st = 0 if stream is None else (stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream))
        p, a = cfg.to_struct(), adaptive_params(threshold, min_spp, check_interval)
        check(lib.ezrt_render_adaptive_device(self._h, C.byref(p), C.byref(a), C.c_void_p(ptr(d_framebuffer)), C.c_void_p(ptr(d_spp)),
                                              C.c_void_p(ptr(d_luma2)), C.c_void_p(st)))
        return d_framebuffer, d_spp, d_luma2

    def render_aov(self, cfg, framebuffer=None, aov=None, luma2=None):
        """Plain render that also returns the first-hit feature buffers (ezrt_render_aov).  Returns host arrays
        (image, aov, luma2): [H, W, C], [H, W, 8], [H, W] for one part, compact tile-major [n, C], [n, 8], [n] otherwise.
        aov = running means of (albedo.rgb, coverage, normal.xyz, depth) of the first hit, 0 for a primary miss; luma2 =
        running mean of the squared sample luminance.  When cfg.first_frame > 0 pass the previous three arrays: they are in/out."""
        n = partition_pixels(cfg.width, cfg.height, cfg.part_rank, cfg.part_count)
        img = np.zeros((n, cfg.out_channels), np.float32) if framebuffer is None else framebuffer
        feat = np.zeros((n, AOV_CHANNELS), np.float32) if aov is None else aov
        m2 = np.zeros(n, np.float32) if luma2 is None else luma2
        for a, k in ((img, cfg.out_channels), (feat, AOV_CHANNELS), (m2, 1)):
            assert a.dtype == np.float32 and a.size == n * k and a.flags.c_contiguous
        p = cfg.to_struct()
        check(lib.ezrt_render_aov(self._h, C.byref(p), _fp(img), _fp(feat), _fp(m2)))
        if cfg.part_count == 1:
            return (img.reshape(cfg.height, cfg.width, cfg.out_channels), feat.reshape(cfg.height, cfg.width, AOV_CHANNELS),
                    m2.reshape(cfg.height, cfg.width))
        return img.reshape(n, cfg.out_channels), feat.reshape(n, AOV_CHANNELS), m2.reshape(n)

    def render_aov_device(self, cfg, d_framebuffer, d_aov, d_luma2, stream=None):
        """Enqueue a feature-buffer render on a CUDA stream into device buffers (torch tensors or raw pointers): the
        framebuffer, 8 float32 per pixel (16-byte aligned), float32 per pixel.  In/out when cfg.first_frame > 0."""
        ptr = lambda t: t.data_ptr() if hasattr(t, "data_ptr") else int(t)
        st = 0 if stream is None else (stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream))
        p = cfg.to_struct()
        check(lib.ezrt_render_aov_device(self._h, C.byref(p), C.c_void_p(ptr(d_framebuffer)), C.c_void_p(ptr(d_aov)),
                                         C.c_void_p(ptr(d_luma2)), C.c_void_p(st)))
        return d_framebuffer, d_aov, d_luma2

    def denoise(self, image, aov, luma2, n, out=None, **sigmas):
        """A-trous denoiser (ezrt_denoise) of a full image [H, W, 3 or 4] after n frames, with render_aov's aov [H, W, 8] and
        luma2 [H, W].  sigmas: iterations, sigma_l, sigma_n, sigma_z, sigma_a (DENOISE_DEFAULTS).  out may be image."""
        img = _f32(image)
        assert img.ndim == 3 and img.shape[2] in (3, 4)
        h, w, ch = img.shape
        feat, m2 = _f32(aov, (h, w, AOV_CHANNELS)), _f32(luma2, (h, w))
        if out is None:
            out = np.empty_like(img)
        assert out.dtype == np.float32 and out.shape == img.shape and out.flags.c_contiguous
        d = denoise_params(**{**DENOISE_DEFAULTS, **sigmas})
        check(lib.ezrt_denoise(self._h, C.byref(d), _fp(img), ch, _fp(feat), _fp(m2), w, h, int(n), _fp(out)))
        return out

    def denoise_device(self, d_image, channels, d_aov, d_luma2, width, height, n, d_out, stream=None, **sigmas):
        """Enqueue the denoiser on a CUDA stream over device buffers (torch tensors or raw pointers); d_out may be d_image."""
        ptr = lambda t: t.data_ptr() if hasattr(t, "data_ptr") else int(t)
        st = 0 if stream is None else (stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream))
        d = denoise_params(**{**DENOISE_DEFAULTS, **sigmas})
        check(lib.ezrt_denoise_device(self._h, C.byref(d), C.c_void_p(ptr(d_image)), int(channels), C.c_void_p(ptr(d_aov)),
                                      C.c_void_p(ptr(d_luma2)), int(width), int(height), int(n), C.c_void_p(ptr(d_out)), C.c_void_p(st)))
        return d_out

    def counters(self):
        c = Counters()
        check(lib.ezrt_get_counters(self._h, C.byref(c)))
        return c

    def kernel_times(self):
        """{class: (ms, launches)} of the last render with cfg.profile = 1."""
        ms = (C.c_double * 4)()
        n = (C.c_uint64 * 4)()
        check(lib.ezrt_get_kernel_times(self._h, ms, n))
        return {k: (ms[i], int(n[i])) for i, k in enumerate(("extend", "shade", "shadow", "other"))}

    def w8_phase_cycles(self):
        """{pass: {phase: SM cycles summed over warps}} of the last render with cfg.profile = 2 (ezrt_get_w8_phase_cycles)."""
        c = (C.c_uint64 * 8)()
        check(lib.ezrt_get_w8_phase_cycles(self._h, c))
        phases = ("refill", "node", "triangle", "ray_end")
        return {k: {ph: int(c[4 * i + j]) for j, ph in enumerate(phases)} for i, k in enumerate(("k_extend_w8", "k_shadow_w8"))}

    def w8_step_counts(self):
        """{pass: {count: n}} of the same render: the warps' node and triangle steps, the rays' node visits and triangle tests
        (ezrt_get_w8_step_counts)."""
        c = (C.c_uint64 * 8)()
        check(lib.ezrt_get_w8_step_counts(self._h, c))
        names = ("node_steps", "triangle_steps", "node_visits", "triangle_tests")
        return {k: {nm: int(c[4 * i + j]) for j, nm in enumerate(names)} for i, k in enumerate(("k_extend_w8", "k_shadow_w8"))}

    def trace_rays(self, origins, dirs, traverse=TRAVERSE_ACCEL, any_hit=False, p3_normal_fudge=False):
        """hitBVH for n rays on the device (P5/fsh:254-306)."""
        o = _f32(origins, (-1, 3))
        d = _f32(dirs, (-1, 3))
        n = o.shape[0]
        hit = np.zeros(n, dtype=np.int32); tri = np.zeros(n, dtype=np.int32); inside = np.zeros(n, dtype=np.int32)
        dist = np.zeros(n, dtype=np.float32); point = np.zeros((n, 3), dtype=np.float32); normal = np.zeros((n, 3), dtype=np.float32)
        ip = lambda a: a.ctypes.data_as(_lib.c_int32_p)
        check(lib.ezrt_trace_rays(self._h, n, _fp(o), _fp(d), int(traverse), int(bool(any_hit)), int(bool(p3_normal_fudge)),
                                  ip(hit), _fp(dist), ip(tri), ip(inside), _fp(point), _fp(normal)))
        return dict(hit=hit, distance=dist, triangle=tri, inside=inside, point=point, normal=normal)

    def camera_rays(self, cfg, px, py, frame):
        """ezrt_camera_rays: the render's camera rays (pinhole, or cfg's thin lens) of the samples (px[i], py[i], frame[i]) of
        cfg's image -> (origins [n, 3], dirs [n, 3]) float32.  For parity tests."""
        u = lambda a: np.ascontiguousarray(a, dtype=np.uint32).reshape(-1)
        px, py, frame = u(px), u(py), u(frame)
        n = px.size
        assert py.size == n and frame.size == n
        o, d = np.zeros((n, 3), np.float32), np.zeros((n, 3), np.float32)
        p = cfg.to_struct()
        up = lambda a: a.ctypes.data_as(_lib.c_uint32_p)
        check(lib.ezrt_camera_rays(self._h, C.byref(p), n, up(px), up(py), up(frame), _fp(o), _fp(d)))
        return o, d

    def lights(self):
        """The light table of MODE_DISNEY_LIGHTS (ezrt_scene_lights; built at the first call or render in that mode):
        (triangle indices int32 [K], cdf float32 [K], W = float64 sum of the weights)."""
        k = check(lib.ezrt_scene_lights(self._h, 0, None, None, None))
        tri = np.zeros(k, np.int32)
        cdf = np.zeros(k, np.float32)
        total = C.c_double(0.0)
        check(lib.ezrt_scene_lights(self._h, k, tri.ctypes.data_as(_lib.c_int32_p), _fp(cdf), C.byref(total)))
        return tri, cdf, total.value

    def env_light_table(self):
        """The environment table of RenderConfig.env_light (ezrt_scene_env_light; built at the first call or flagged render):
        (row_cdf float32 [H], col_cdf float32 [H, W], texel_pdf float32 [H, W], T = float64 sum of the texel weights), or None
        when the scene has no table (no map, or a black one)."""
        total = C.c_double(0.0)
        if not check(lib.ezrt_scene_env_light(self._h, None, None, None, C.byref(total))):
            return None
        h, w = self.hdr.shape[0], self.hdr.shape[1]
        row, col, pdf = np.zeros(h, np.float32), np.zeros((h, w), np.float32), np.zeros((h, w), np.float32)
        check(lib.ezrt_scene_env_light(self._h, _fp(row), _fp(col), _fp(pdf), None))
        return row, col, pdf, total.value

    def occluded_rays(self, origins, dirs, tmax, traverse=TRAVERSE_ACCEL):
        """ezrt_occluded_rays: 1 where nothing is accepted strictly before tmax along the ray (the render's shadow pass)."""
        o = _f32(origins, (-1, 3))
        d = _f32(dirs, (-1, 3))
        n = o.shape[0]
        t = _f32(np.broadcast_to(np.asarray(tmax, np.float32), (n,)))
        lit = np.zeros(n, np.int32)
        check(lib.ezrt_occluded_rays(self._h, n, _fp(o), _fp(d), _fp(t), int(traverse), lit.ctypes.data_as(_lib.c_int32_p)))
        return lit


def accel_build(tris, leaf_n=4, where="device", device=0):
    """The binary SAH tree ezrt_scene_create derives its acceleration tree from (ezrt_accel_build, include/ezrt.h):
    returns (links int32 [n,4], boxes float32 [n,6], order uint32 [n_triangles], ms).  where: "device" | "host"."""
    tris = _f32(tris).reshape(-1, 36)
    n = tris.shape[0]
    cap = 2 * n
    links = np.zeros((cap, 4), np.int32)
    boxes = np.zeros((cap, 6), np.float32)
    order = np.zeros(n, np.uint32)
    ms = C.c_double(0.0)
    rc = lib.ezrt_accel_build(device, _fp(tris), n, leaf_n, 1 if where == "host" else 0, links.ctypes.data_as(_lib.c_int32_p), _fp(boxes), cap,
                              order.ctypes.data_as(_lib.c_uint32_p), C.byref(ms))
    if rc < 0:
        check(rc)
    return links[:rc].copy(), boxes[:rc].copy(), order, ms.value


def post_tonemap(d_in, d_out=None, limit=1.5, stream=None):
    """pass3 (P5/shaders/pass3.fsh:14-25) on a device framebuffer (torch CUDA tensor [..., 3|4]) -> [..., 3]."""
    import torch
    channels = d_in.shape[-1]
    n = d_in.numel() // channels
    if d_out is None:
        d_out = torch.empty(tuple(d_in.shape[:-1]) + (3,), dtype=torch.float32, device=d_in.device)
    st = torch.cuda.current_stream() if stream is None else stream
    check(lib.ezrt_post_tonemap(C.c_void_p(d_in.data_ptr()), channels, C.c_void_p(d_out.data_ptr()), n, float(limit), C.c_void_p(st.cuda_stream)))
    return d_out


def write_png(path, framebuffer, tonemap=True):
    """Write a linear framebuffer [H, W, 3|4] (row 0 = bottom) as an 8-bit PNG (pass3 tone map + gamma when tonemap)."""
    fb = _f32(framebuffer)
    h, w, c = fb.shape
    check(lib.ezrt_write_png(str(path).encode(), _fp(fb), w, h, c, int(bool(tonemap))))


def eval_brdf(which, V, N, L, xi, materials, device=0):
    V = _f32(V, (-1, 3)); N = _f32(N, (-1, 3))
    L = None if L is None else _f32(L, (-1, 3))
    xi = None if xi is None else _f32(xi, (-1, 3))
    materials = _f32(materials, (-1, 18))
    out = np.zeros_like(V)
    check(lib.ezrt_eval_brdf(device, which, V.shape[0], _fp(V), _fp(N), None if L is None else _fp(L),
                             None if xi is None else _fp(xi), _fp(materials), _fp(out)))
    return out


def eval_bsdf(which, V, N, L, xi, inside, materials, device=0):
    """ezrt_eval_bsdf: the transmission mixture on the device, [n, 8] float32 (which 0: f, 1: pdf, 2: sample of xi [n, 4])."""
    V = _f32(V, (-1, 3)); N = _f32(N, (-1, 3))
    L = None if L is None else _f32(L, (-1, 3))
    xi = None if xi is None else _f32(xi, (-1, 4))
    inside = np.ascontiguousarray(inside, dtype=np.int32).reshape(-1)
    materials = _f32(materials, (-1, 18))
    out = np.zeros((V.shape[0], 8), np.float32)
    check(lib.ezrt_eval_bsdf(device, which, V.shape[0], _fp(V), _fp(N), None if L is None else _fp(L),
                             None if xi is None else _fp(xi), inside.ctypes.data_as(_lib.c_int32_p), _fp(materials), _fp(out)))
    return out


def eval_math(which, a, b=None, device=0):
    a = _f32(a).reshape(-1)
    b = None if b is None else _f32(b).reshape(-1)
    out = np.zeros_like(a)
    check(lib.ezrt_eval_math(device, which, a.size, _fp(a), None if b is None else _fp(b), _fp(out)))
    return out
