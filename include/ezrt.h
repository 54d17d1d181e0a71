/*
 * ezrt.h -- C ABI of ezrt_b200: the H100-native drop-in for EzRT's path-tracing hot path.
 *
 * The reference (AKGWSB/EzRT) has no plugin/FFI interface; its de-facto boundary is "what
 * main() hands to pass1 and what pass1 leaves in lastFrame" (SURVEY.md 8b).  Every entry
 * point below cites the reference code it replaces.  Path aliases: P2/ P3/ P4/ P5/ = the
 * "source code" directory of tutorial part 2..5; fsh = shaders/fshader.fsh.
 *
 * Conventions
 *   - plain C: pointers + sizes, no C++/torch types; all functions return 0 on success or
 *     a negative ezrt_status; ezrt_last_error() gives a thread-local message.  The
 *     reference prints and exit(-1)s (P5/main.cpp:178-182, :283-286); this ABI never exits.
 *   - the caller owns every input array and every output buffer; a scene handle owns its
 *     device allocations.  One handle = one CUDA device; calls on one handle are
 *     serialised by the caller; different handles may be driven from different threads.
 *   - "tris" is an array of Triangle_encoded (P5/main.cpp:60-69): 36 packed floats
 *     (p1 p2 p3 n1 n2 n3 emissive baseColor param1..param4), stride 144 B.
 *   - "nodes" is an array of BVHNode_encoded (P5/main.cpp:71-76): 12 packed floats
 *     (left,right,0)(n,index,0) AA BB, ints stored as floats; element 0 is the dummy
 *     testNode, the root is element 1 (P5/main.cpp:830-838, P5/fsh:263).
 *   - framebuffers are linear-radiance fp32, row 0 = bottom row (GL convention), the
 *     content of pass1's colour attachment 0 / lastFrame (P5/fsh:942-947) before any
 *     tone mapping.
 */
#ifndef EZRT_H
#define EZRT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EZRT_TRIANGLE_FLOATS 36 /* Triangle_encoded, P5/main.cpp:60-69 */
#define EZRT_BVHNODE_FLOATS 12  /* BVHNode_encoded,  P5/main.cpp:71-76 */
#define EZRT_MATERIAL_FLOATS 18 /* emissive, baseColor, 12 scalars: P5/main.cpp:27-42 */

typedef enum ezrt_status {
    EZRT_OK = 0,
    EZRT_ERR_INVALID = -1,   /* bad argument */
    EZRT_ERR_IO = -2,        /* file could not be opened / parsed */
    EZRT_ERR_CUDA = -3,      /* CUDA runtime error or no device */
    EZRT_ERR_BAD_TREE = -4,  /* node array is not a tree the traversal can walk */
    EZRT_ERR_NOMEM = -5
} ezrt_status;

/* Integrator modes: the four per-pixel loops the reference ships (SURVEY.md 8a), and mode 4, which adds light sampling
 * on the scene's emissive triangles to mode 3's BRDF sampling. */
typedef enum ezrt_mode {
    EZRT_MODE_DIFFUSE_P3 = 0,      /* P3/fsh:376-446  diffuse, uniform hemisphere, wang-hash   */
    EZRT_MODE_DISNEY_ANISO_P4 = 1, /* P4/fsh:478-550  anisotropic Disney, uniform hemisphere   */
    EZRT_MODE_DISNEY_SOBOL_P5 = 2, /* P5/fsh:762-807  Disney + Sobol/CP rotation               */
    EZRT_MODE_DISNEY_IS_MIS_P5 = 3, /* P5/fsh:810-890  BRDF + HDR importance sampling, MIS     */
    /* BRDF importance sampling + one light sample per bounce on the emissive triangles, balance-heuristic MIS (ezrt_math.h,
     * DESIGN.md section 10).  With or without an HDR map: the environment is reached by BRDF samples only, at weight 1,
     * unless reserved[0] has EZRT_PARAM_ENV_LIGHT.  Wavefront pipeline only.  The first render of a scene in this mode builds
     * its light table (ezrt_scene_lights), which synchronises the render's stream once. */
    EZRT_MODE_DISNEY_LIGHTS = 4
} ezrt_mode;

/* BVH traversal policy.  All three return bit-identical hits (tests assert it).
 * ACCEL (default): the device builds its own acceleration tree over the same triangles (the
 *   reference's sweep SAH without its INF = 114514 cost cut-off, P5/main.cpp:20,:493), finds the
 *   global closest hit there, keeps it when the shader's hitBVH provably reaches that triangle's
 *   leaf in the REFERENCE tree and no other triangle ties, and otherwise re-traces the ray with the
 *   exact reference-order traversal (DESIGN.md "accel").
 * REFERENCE walks every box the ray overlaps, exactly as P5/fsh:254-306 (no best-distance pruning).
 * PRUNED walks the reference tree in the shader's order but skips a sub-tree whose box entry lies
 *   beyond the current best hit by a conservative margin (DESIGN.md "pruning"). */
typedef enum ezrt_traverse {
    EZRT_TRAVERSE_ACCEL = 0,
    EZRT_TRAVERSE_REFERENCE = 1,
    EZRT_TRAVERSE_PRUNED = 2
} ezrt_traverse;

typedef enum ezrt_pipeline {
    EZRT_PIPELINE_WAVEFRONT = 0, /* generate / extend / shade / shadow / blend kernels */
    EZRT_PIPELINE_MEGAKERNEL = 1 /* one thread per pixel, literal loop (cross-check)   */
} ezrt_pipeline;

/* Everything display() passes to pass1 per frame (P5/main.cpp:709-745, :919-923) plus
 * the constants that are literals in the shaders. */
typedef struct ezrt_render_params {
    int32_t width, height;   /* uniform width,height  (P5/main.cpp:922-923)                  */
    int32_t spp;             /* number of consecutive display() calls to perform             */
    uint32_t first_frame;    /* frameCounter of the first call (P5/main.cpp:719); 0 = fresh  */
                             /* Frames count in the reference's uint arithmetic, modulo 2^32: frame 0xFFFFFFFF is
                              * blended with weight 1/float(frame + 1u) = 1/0 = +inf, which makes every blended
                              * value NaN (colour, features, luma2; alpha stays 1), and the frames after it (0, 1, ...)
                              * blend into NaN and leave it NaN; its Sobol index frame + 1 is 0. */
    int32_t max_bounce;      /* literal in main(): P5/fsh:935 (2), P4/fsh:540 (4), P3 (2)    */
    int32_t mode;            /* ezrt_mode                                                    */
    float eye[3];            /* uniform eye           (P5/main.cpp:710-711, :717)            */
    float camera_rotate[16]; /* uniform cameraRotate, column-major inverse(lookAt) (:712-718) */
    float env_color[3];      /* colour of a miss when the scene has no HDR map               */
    int32_t traverse;        /* ezrt_traverse                                                */
    int32_t pipeline;        /* ezrt_pipeline                                                */
    int32_t out_channels;    /* 3 (RGB) or 4 (RGBA, alpha = 1 as in P5/fsh:947)              */
    /* image partition for multi-GPU rendering: the image is cut into 16x16 tiles, tile
     * (tx,ty) belongs to part (tx+ty) % part_count; a part renders only its tiles and
     * writes them compactly (tile-major) unless part_count == 1. */
    int32_t part_rank, part_count;
    int32_t frames_per_batch; /* wavefront: display() calls traced concurrently (0 = auto)   */
    int32_t profile;          /* 1: bracket every kernel with CUDA events (ezrt_get_kernel_times);
                                 2: count the records the accel traversal fetches (ezrt_counters.node_visits / tri_tests;
                                    a slower instantiation of the same kernels -- never inside a timed region) */
    int32_t reserved[3];      /* [0]: flags, EZRT_PARAM_*; [1], [2]: with EZRT_PARAM_THIN_LENS the lens radius and the focus
                                 distance as IEEE-754 float bits, ignored otherwise */
} ezrt_render_params;

/* ezrt_render_params.reserved[0]: keep counting -- ezrt_get_counters / ezrt_get_kernel_times then report the sums over all
   renders since the last one issued without this flag (a benchmark loop reads them once, without a sync per render) */
#define EZRT_PARAM_ACCUMULATE 1
/* ezrt_render_params.reserved[0], EZRT_MODE_DISNEY_LIGHTS only (any other mode: EZRT_ERR_INVALID): the scene's HDR map is one
   more light.  Each shading point draws one light sample, from the map with probability 1/2 (1 when the scene has no emissive
   triangle) by an equirectangular table proportional to luminance in solid angle, else from the triangles as in mode 4; BRDF
   samples that leave the scene are MIS-weighted against it (ezrt_math.h, DESIGN.md section 11).  A scene without a map, or
   whose map is black, renders as mode 4.  Accepted by ezrt_render[_device], ezrt_render_adaptive[_device] and
   ezrt_render_aov[_device]; the first such render of a scene builds the map's table (ezrt_scene_env_light: about 8 bytes per
   texel of device memory), which synchronises the render's stream once. */
#define EZRT_PARAM_ENV_LIGHT 2
/* ezrt_render_params.reserved[0], EZRT_MODE_DISNEY_LIGHTS only (any other mode: EZRT_ERR_INVALID), with or without
   EZRT_PARAM_ENV_LIGHT: materials' IOR and transmission are rendered.  A material with t = clamp(transmission, 0, 1) *
   (1 - metallic) > 0 scatters by (1 - t) * the reference BRDF + t * a rough dielectric (GGX, exact Fresnel; reflection
   untinted, refraction tinted by baseColor; ezrt_math.h, DESIGN.md section 12).  The outside of every mesh is vacuum: a hit
   from the back of a triangle (geometric normal) leaves the medium of index IOR, so transmissive meshes must be closed and
   wound outward (so EZRT_PARAM_MEDIUM is rejected beside this flag).  |IOR - 1| <= 2^-8 is an index-matched pass-through; IOR <= 0 or not finite is opaque.  Light samples and
   shadow rays treat transmissive triangles as opaque: light through glass arrives by BSDF samples only.  A scene without a
   material of t > 0 renders as without the flag, bit for bit.  Accepted by ezrt_render[_device],
   ezrt_render_adaptive[_device] and ezrt_render_aov[_device]. */
#define EZRT_PARAM_TRANSMISSION 4
/* ezrt_render_params.reserved[0], any mode, policy and pipeline: a thin-lens camera (depth of field).  reserved[1] holds the
   bits of the lens radius R, reserved[2] those of the focus distance f (memcpy a float into each).  Each camera ray starts at a
   point of the disk of radius R around eye spanned by columns 0 and 1 of camera_rotate (normalised), and passes through the
   point the pinhole ray of the same pixel jitter reaches at depth f along -column 2; ezrt_math.h and DESIGN.md section 13 give
   the arithmetic.  The lens point is drawn from a random stream of its own, so the rest of every path draws what the pinhole
   render draws.  Invalid (EZRT_ERR_INVALID) unless R and f are finite and > 0 and columns 0, 1 and 2 have finite, non-zero
   length.  Accepted by ezrt_render[_device], ezrt_render_adaptive[_device] and ezrt_render_aov[_device]; a feature-buffer
   render's depth is the first hit's distance from the lens point. */
#define EZRT_PARAM_THIN_LENS 8
/* ezrt_render_params.reserved[0], EZRT_MODE_DISNEY_LIGHTS on the wavefront pipeline only, with or without EZRT_PARAM_ENV_LIGHT and
   EZRT_PARAM_THIN_LENS: the scene's homogeneous medium (ezrt_scene_set_medium) is rendered.  Every traced segment that overlaps the
   medium's box draws a free-flight distance; a path that scatters there takes a medium vertex (one bounce): a light sample evaluated
   with the Henyey-Greenstein phase function and a phase-function sample of the next direction.  Every light sample's contribution
   (from surfaces too) is multiplied by the transmittance of its shadow ray.  Opaque objects in the box stay surfaces; the feature
   buffers still describe the first surface along the camera ray.  ezrt_math.h and DESIGN.md section 14 give the arithmetic.
   Invalid (EZRT_ERR_INVALID) without a medium set on the scene, in another mode, with the megakernel, and with
   EZRT_PARAM_TRANSMISSION (glass is defined with vacuum outside; a medium around it would need a medium stack).  Accepted by
   ezrt_render[_device], ezrt_render_adaptive[_device] and ezrt_render_aov[_device]. */
#define EZRT_PARAM_MEDIUM 16
/* ezrt_render_params.reserved[0], EZRT_MODE_DISNEY_LIGHTS on the wavefront pipeline only, with or without EZRT_PARAM_ENV_LIGHT,
   EZRT_PARAM_TRANSMISSION, EZRT_PARAM_THIN_LENS and EZRT_PARAM_MEDIUM: the scene's base-colour textures (ezrt_scene_set_textures)
   are rendered.  Wherever the render reads the base colour of a surface hit -- the BRDF and the transmission mixture (evaluation,
   sampling, pdf), the light samples evaluated after the shadow pass, the feature buffers' albedo -- it uses the material's baseColor
   times the filtered linear colour of the triangle's texture at the hit's UV: barycentrics on the triangle's dominant plane, wrap
   addressing, RGBA8 texels decoded by the sRGB EOTF (alpha ignored), bilinear filtering (ezrt_math.h, DESIGN.md section 15).
   Emission is not textured, and no random number is drawn, so a render whose textures are all 1x1 white is the unflagged render's
   bit for bit.  Invalid (EZRT_ERR_INVALID) without textures set on the scene and in another mode.  Accepted by ezrt_render[_device],
   ezrt_render_adaptive[_device] and ezrt_render_aov[_device]; each shadow slot of a flagged render takes 16 bytes more. */
#define EZRT_PARAM_TEXTURES 32
/* ezrt_render_params.reserved[0], with EZRT_PARAM_TEXTURES (so in EZRT_MODE_DISNEY_LIGHTS on the wavefront pipeline only, with or
   without EZRT_PARAM_ENV_LIGHT, EZRT_PARAM_TRANSMISSION, EZRT_PARAM_THIN_LENS and EZRT_PARAM_MEDIUM): the scene's material maps
   (ezrt_scene_set_material_maps) are rendered.  At every surface hit but the last vertex, the metallic-roughness map (linear, glTF's
   channels) scales the material's roughness by its G and its metallic by its B, and the tangent-space normal map (linear, OpenGL's +Y)
   replaces the shading normal, in a per-triangle tangent frame from the triangle's edges and UV deltas (ezrt_math.h, DESIGN.md
   section 16).  The mapped values are used wherever the render reads them: the BRDF and the transmission mixture (evaluation,
   sampling, pdf, the lobe weights), the light samples' hemisphere tests and their evaluation after the shadow pass, the path's
   cosine, and the feature buffers' normal.  The emission's MIS and the inside test keep the geometric normal.  No random number is
   drawn.  Invalid (EZRT_ERR_INVALID) without EZRT_PARAM_TEXTURES or without maps set.  Accepted by ezrt_render[_device],
   ezrt_render_adaptive[_device] and ezrt_render_aov[_device].  Each shadow slot of a render takes 81 bytes, 97 with
   EZRT_PARAM_TEXTURES, 101 with EZRT_PARAM_MATERIAL_MAPS too. */
#define EZRT_PARAM_MATERIAL_MAPS 64

/* One texture of ezrt_scene_set_textures: width x height RGBA8 texels (4 bytes each, R first), row 0 the image's top row */
typedef struct ezrt_texture {
    int32_t width, height;   /* each in [1, 16384] */
    const uint8_t* rgba;     /* width * height * 4 bytes, sRGB-encoded colour; alpha is ignored */
    int32_t reserved;        /* 0 */
} ezrt_texture;

/* The homogeneous medium of EZRT_PARAM_MEDIUM: a grey extinction, an RGB single-scattering albedo and a Henyey-Greenstein
   asymmetry g (> 0: forward scattering), filling the axis-aligned box [box_min, box_max] (a box of zero extent on an axis holds
   no medium). */
typedef struct ezrt_medium {
    float sigma_t;     /* extinction per unit length, finite and >= 0 (0: the flagged render is mode 4's) */
    float albedo[3];   /* single-scattering albedo, each in [0, 1] */
    float g;           /* Henyey-Greenstein asymmetry, -1 < g < 1 */
    float box_min[3];  /* finite, box_min <= box_max on every axis */
    float box_max[3];
    int32_t reserved;  /* 0 */
} ezrt_medium;

typedef struct ezrt_counters {
    uint64_t rays;          /* hitBVH invocations: primary + bounce + shadow (SURVEY 8d)     */
    uint64_t primary_rays, bounce_rays, shadow_rays;
    uint64_t samples;       /* pixel-samples = fragment shader invocations                   */
    uint64_t kernel_launches;
    double device_ms;       /* CUDA-event time of the last render on its stream              */
    uint64_t deferred_rays; /* accel policy: rays re-traced by the exact reference-order pass */
    uint64_t node_visits;   /* profile = 2: acceleration-tree node records fetched ...       */
    uint64_t tri_tests;     /*              ... and triangle records (64 B) fetched by the accel kernels */
    uint64_t node_visits_96;/*              of node_visits: quantised records (16-bit planes, 96 B / W8, 80 B); the rest are 128-byte records */
    uint64_t node_bytes, tri_bytes; /*      96 B per quantised and 128 B per exact node visit, 64 B per triangle test: nominal
                                               figures, not bytes fetched (a W8 node is 80 B; a flat triangle test that fails its distance
                                               checks reads 16 B, an indexed one 32 B, and 48 B of vertices more past them) */
} ezrt_counters;

typedef struct ezrt_scene ezrt_scene; /* device-resident scene (replaces the two TBOs + 2 textures) */

const char* ezrt_last_error(void);
int ezrt_version(void);

/* ----------------------------------------------------------------------------------------
 * Device side: the hot path.
 * -------------------------------------------------------------------------------------- */

/* Replaces the texture-buffer uploads P5/main.cpp:878-906: copies the reference-layout
 * arrays to the GPU `device` and repacks them for the kernels.  hdr / hdr_cache may be
 * NULL (then hdr_w = hdr_h = 0).  hdr rows are stored top-to-bottom as HDRLoader returns
 * them (P5/lib/hdrloader.cpp:76-91); hdr_cache is calculateHdrCache()'s output
 * (P5/main.cpp:592-689).  hdr_filter_linear: 1 = GL_LINEAR (P5/main.cpp:196-199),
 * 0 = GL_NEAREST (P3/main.cpp:195-196). */
int ezrt_scene_create(int device, const float* tris, int n_triangles, const float* nodes, int n_nodes,
                      const float* hdr, const float* hdr_cache, int hdr_w, int hdr_h,
                      int hdr_filter_linear, ezrt_scene** out_scene);
int ezrt_scene_destroy(ezrt_scene* scene);
/* Sets the scene's homogeneous medium (a copy of *medium), or clears it (medium NULL).  Returns EZRT_ERR_INVALID, and keeps the
 * previous medium, for a non-finite or negative sigma_t, an albedo component outside [0, 1] or NaN, |g| >= 1 or NaN, a non-finite
 * box corner, box_min > box_max on an axis, or reserved != 0.  The medium travels to the kernels by value when a render is
 * enqueued: changing it afterwards does not affect renders already enqueued. */
int ezrt_scene_set_medium(ezrt_scene* scene, const ezrt_medium* medium);
/* Sets the scene's base-colour textures (EZRT_PARAM_TEXTURES): n_textures textures (copied), and per triangle, in the order of the
 * `tris` array given to ezrt_scene_create, 6 floats of texcoords (u1, v1, u2, v2, u3, v3: OBJ's convention, v = 0 at the image's
 * bottom) and a texture id in [-1, n_textures) (-1: the material's base colour).  textures NULL clears them.  Returns
 * EZRT_ERR_INVALID for a side outside [1, 16384], a null rgba, reserved != 0, an id out of range, more than 2^31 texels, or
 * n_textures < 1 with textures set; EZRT_ERR_NOMEM / EZRT_ERR_CUDA when the copies cannot be made.  On every error the previous
 * textures are kept.  The call first waits for every render already enqueued on the scene's device (it frees the
 * previous buffers those renders read), then uploads synchronously. */
int ezrt_scene_set_textures(ezrt_scene* scene, int n_textures, const ezrt_texture* textures, const float* texcoords, const int32_t* texture_id);
/* The textured base colour the kernels compute at n hit points: points[3 i..] on reference triangle tri[i] -> uv_out[2 i..] (the
 * interpolated UV) and rgb_out[3 i..] (the material's baseColor times the filtered texture; baseColor for texture id -1).  Host
 * arrays; synchronous.  EZRT_ERR_INVALID without textures set or for a triangle index out of range. */
int ezrt_scene_sample_textures(ezrt_scene* scene, int n, const int32_t* tri, const float* points, float* uv_out, float* rgb_out);
/* Sets the scene's material maps (EZRT_PARAM_MATERIAL_MAPS): per triangle, in the order of the `tris` array given to
 * ezrt_scene_create, the id of its metallic-roughness map and of its normal map among the textures of ezrt_scene_set_textures (-1: no
 * map).  Both NULL clears them.  Returns EZRT_ERR_INVALID without textures set, for exactly one NULL array, or for an id outside
 * [-1, n_textures) or of 65535 or more; on every error the previous maps are kept.  ezrt_scene_set_textures (also clearing) clears the
 * maps.  The call first waits for every render already enqueued on the scene's device, then writes the ids synchronously. */
int ezrt_scene_set_material_maps(ezrt_scene* scene, const int32_t* metal_rough_id, const int32_t* normal_id);
/* What the maps renders compute at n surface hits: reference triangle tri[i] hit by the ray hits[7 i..] = (o, d, t) -> out[10 i..] =
 * (u, v, the textured base colour (3), the mapped roughness, the mapped metallic, the final shading normal (3), flipped for a hit from
 * inside).  The maps set on the scene are used (none: the material's values and surface_hit's normal).  Host arrays; synchronous.
 * EZRT_ERR_INVALID without textures set or for a triangle index out of range. */
int ezrt_scene_sample_materials(ezrt_scene* scene, int n, const int32_t* tri, const float* hits, float* out);

/* render(width,height,spp) -> framebuffer: equals `spp` consecutive display() calls
 * (P5/main.cpp:697-748) each drawing pass1 (P5/fsh:894-949) and copying to lastFrame.
 * `framebuffer` is a HOST buffer, in/out: when first_frame > 0 it must hold lastFrame.
 * Size: n_pixels(part) * out_channels floats, see ezrt_partition_pixels(). */
int ezrt_render(ezrt_scene* scene, const ezrt_render_params* params, float* framebuffer);

/* Same, but `d_framebuffer` is DEVICE memory on the scene's GPU and the work is enqueued on
 * `cuda_stream` (a cudaStream_t, NULL = default stream).  Steady state: no host synchronisation.  The FIRST
 * call for a given (image size, partition, batch size) allocates the scene's scratch buffers (cudaMalloc synchronises
 * the device) and uploads the tile list (one stream synchronisation).  The scratch belongs to the scene: at most ONE
 * render of a scene may be in flight at a time -- enqueue renders of the same scene on one stream, or order them with
 * events; different scenes (one per GPU) are independent. */
int ezrt_render_device(ezrt_scene* scene, const ezrt_render_params* params, float* d_framebuffer,
                       void* cuda_stream);

/* Tile-adaptive sampling (DESIGN.md section 8; the criterion is defined in ezrt_math.h).  The image is rendered in 16x16
 * tiles; after min_spp frames and then every check_interval frames, each tile whose pixels all have a relative standard
 * error of luminance <= threshold stops, the others go on, up to params->spp frames.  Every tile holds exactly the bits a
 * plain render with spp = (the frames it received) gives it. */
typedef struct ezrt_adaptive_params {
    float threshold;        /* > 0: relative standard error of pixel luminance at which a tile stops */
    int32_t min_spp;        /* >= 2: frames before the first test */
    int32_t check_interval; /* >= 1: frames between tests */
    int32_t reserved;       /* 0 */
} ezrt_adaptive_params;

/* params->spp = frame cap, params->first_frame must be 0, wavefront pipeline only; any traversal policy, mode and partition
 * (the decision is per tile, so a part's tiles stop where they would in the whole image).
 * d_spp:   int32 per pixel, frames the pixel received.
 * d_luma2: float per pixel, the running mean of the squared sample luminance (M of the criterion).
 * Both use the framebuffer's pixel layout (tile-major compact when part_count > 1).  Device buffers, enqueued on cuda_stream
 * like ezrt_render_device, except that each test reads back 8 bytes (surviving tiles and pixels): one stream
 * synchronisation per test.  ezrt_get_counters reports the work done: samples = sum of the spp map, rays of active tiles
 * only; with params->profile = 1 the test kernel is timed in class 3 ("other"). */
int ezrt_render_adaptive_device(ezrt_scene* scene, const ezrt_render_params* params, const ezrt_adaptive_params* adaptive,
                                float* d_framebuffer, int32_t* d_spp, float* d_luma2, void* cuda_stream);
/* Same with host buffers (synchronous). */
int ezrt_render_adaptive(ezrt_scene* scene, const ezrt_render_params* params, const ezrt_adaptive_params* adaptive,
                         float* framebuffer, int32_t* spp, float* luma2);

/* Feature buffers (AOVs; DESIGN.md section 9): a plain render (params->spp frames from params->first_frame, the same
 * framebuffer bits as ezrt_render_device) that also returns, per pixel, running means over its frames with the colour's
 * weights (mix(acc, v, 1/(frame+1)) in frame order):
 *   d_aov:   8 floats: albedo.rgb (the first hit's base colour), coverage (1 hit, 0 miss), normal.xyz (the first hit's shading
 *            normal, flipped when hit from inside), depth (the first hit's distance); a primary miss contributes 0 to all 8.
 *            16-byte aligned.
 *   d_luma2: float, the running mean of the squared sample luminance (M of ezrt_math.h, bit for bit the adaptive render's).
 * When first_frame > 0 all three buffers are in/out.  Layout of the framebuffer's pixels (tile-major compact when
 * part_count > 1; ezrt_partition_scatter with channels = 8 / 1 scatters them).  Wavefront pipeline only.  The scratch
 * grows by 32 bytes per sample slot for these renders only. */
int ezrt_render_aov_device(ezrt_scene* scene, const ezrt_render_params* params, float* d_framebuffer, float* d_aov, float* d_luma2,
                           void* cuda_stream);
/* Same with host buffers (synchronous). */
int ezrt_render_aov(ezrt_scene* scene, const ezrt_render_params* params, float* framebuffer, float* aov, float* luma2);

/* Denoiser (DESIGN.md section 9; defined in ezrt_math.h): edge-avoiding a-trous wavelet filter with a variance-guided
 * luminance weight, over a full width x height image (row-major; gather the parts of a partitioned render first). */
typedef struct ezrt_denoise_params {
    int32_t iterations;   /* 1..10: passes with steps 1, 2, 4, ... */
    float sigma_l;        /* > 0: luminance weight, in standard deviations */
    float sigma_n;        /* > 0: normal weight, exponent of dot(n_p, n_q) */
    float sigma_z;        /* > 0: depth weight, relative depth difference per pixel of step */
    float sigma_a;        /* > 0: albedo weight, L1 distance */
    int32_t reserved;     /* 0 */
} ezrt_denoise_params;

/* d_color: channels (3 or 4) floats per pixel after n_frames frames; d_aov, d_luma2: ezrt_render_aov_device's outputs of the same
 * render.  d_out may be d_color; alpha is copied.  Enqueued on cuda_stream; the scratch (32 bytes per pixel) belongs to the scene
 * like the render's, so it is ordered with the scene's renders the same way. */
int ezrt_denoise_device(ezrt_scene* scene, const ezrt_denoise_params* params, const float* d_color, int channels, const float* d_aov,
                        const float* d_luma2, int width, int height, int n_frames, float* d_out, void* cuda_stream);
/* Same with host buffers (synchronous); out may be color. */
int ezrt_denoise(ezrt_scene* scene, const ezrt_denoise_params* params, const float* color, int channels, const float* aov,
                 const float* luma2, int width, int height, int n_frames, float* out);

/* Counters of the most recent render on this scene (synchronises the stream). */
int ezrt_get_counters(ezrt_scene* scene, ezrt_counters* out);

/* Per-kernel-class device time of the most recent render with params.profile = 1 (CUDA events on
 * the render's stream; synchronises).  Classes: 0 extend (hitBVH, closest hit), 1 shade,
 * 2 shadow (hitBVH, any hit), 3 other (generate, blend, tally).  ms[4], launches[4]. */
int ezrt_get_kernel_times(ezrt_scene* scene, double* ms, uint64_t* launches);

/* SM cycles the 8-wide accel kernels' warps spent per phase in the most recent render with params.profile = 2 (synchronises),
 * summed over warps: out[0..3] the bounce pass (k_extend_w8), out[4..7] the shadow pass (k_shadow_w8), each as refill, node
 * steps, triangle steps, ray ends.  All 0 for scenes traced without the 8-wide tree.  out[8]. */
int ezrt_get_w8_phase_cycles(ezrt_scene* scene, uint64_t* out);
/* Work of the same kernels in the same render: out[0..3] the bounce pass, out[4..7] the shadow pass, each as warp node steps,
 * warp triangle steps, node visits (per ray, summed) and triangle tests (per ray, summed).  All 0 as above.  out[8]. */
int ezrt_get_w8_step_counts(ezrt_scene* scene, uint64_t* out);

/* Number of pixels part `rank` of `count` owns for a width x height image. */
int64_t ezrt_partition_pixels(int width, int height, int rank, int count);
/* Device kernel: scatter the compact tile-major buffer of part `rank` into a full
 * width x height framebuffer (both device pointers, same channel count).  The device tile lists are cached per
 * (device, image size, rank, count) -- the gather runs once per render -- and live until ezrt_partition_cache_clear(). */
int ezrt_partition_scatter(const float* d_compact, float* d_full, int width, int height, int channels,
                           int rank, int count, void* cuda_stream);
/* Frees the tile lists ezrt_partition_scatter cached on the calling thread's current device (all devices: device < 0). */
int ezrt_partition_cache_clear(int device);
/* Host version of the same scatter (used by the CPU/gloo path and by tests). */
int ezrt_partition_scatter_host(const float* compact, float* full, int width, int height, int channels,
                                int rank, int count);

/* Single-function entry points of the hot path (device), for parity tests: trace `n` rays
 * (origins/dirs: n x 3 floats, host) through hitBVH (P5/fsh:254-306; C++ twin
 * P2/main.cpp:466-485) and return per ray: hit flag, distance, triangle index, isInside,
 * hit point, shading normal. any_hit=1 stops at the first hit (shadow rays, P5/fsh:826-829). */
int ezrt_trace_rays(ezrt_scene* scene, int n, const float* origins, const float* dirs, int traverse,
                    int any_hit, int p3_normal_fudge, int32_t* out_hit, float* out_distance,
                    int32_t* out_triangle, int32_t* out_inside, float* out_point, float* out_normal);

/* The light table of EZRT_MODE_DISNEY_LIGHTS (ezrt_math.h; built here if no render in that mode has built it yet, which
 * synchronises the device).  Returns K, the number of lights, or a negative status; writes min(K, cap) entries:
 * tri_out = the lights' triangle indices (caller's order), cdf_out = their cumulative distribution (the last entry 1),
 * and *total_out = W, the float64 sum of the weights.  Any output may be NULL. */
int ezrt_scene_lights(ezrt_scene* scene, int cap, int32_t* tri_out, float* cdf_out, double* total_out);

/* The environment table of EZRT_PARAM_ENV_LIGHT (ezrt_math.h; built here if no flagged render has built it yet, which
 * synchronises the device).  Returns 1 if the scene has a table, 0 if not (no map, or every texel weighs 0), or a negative
 * status.  With a table of the scene's W x H map, writes row_cdf[H], col_cdf[H * W] and texel_pdf[H * W] (row-major, row 0
 * at the top); *total = T, the float64 sum of the texel weights (0 without a table).  Any output may be NULL. */
int ezrt_scene_env_light(ezrt_scene* scene, float* row_cdf, float* col_cdf, float* texel_pdf, double* total);

/* Bounded occlusion of n rays (host arrays: origins, dirs n x 3, tmax n), for parity tests beside ezrt_trace_rays: runs the
 * shadow pass of the render for the traversal policy `traverse` -- the accel kernels with the exact pass over the rays they
 * defer, or the exact kernel -- and writes out_lit[i] = 1 iff no triangle the shader's hitBVH would test is accepted
 * with t < tmax[i].  When every tmax is +inf, mode 3's unbounded shadow kernels run instead (t < 114514, the shader's INF).
 * Not a general query API: it allocates and synchronises per call. */
int ezrt_occluded_rays(ezrt_scene* scene, int n, const float* origins, const float* dirs, const float* tmax, int traverse,
                       int32_t* out_lit);

/* Evaluate the BRDF functions on the device for n (V,N,L,material) tuples: which = 0
 * BRDF_Evaluate (P5/fsh:500-549), 1 BRDF_Evaluate aniso (P4/fsh:412-473), 2 BRDF_Pdf
 * (P5/fsh:715-752; result in out[3*i]), 3 SampleBRDF (P5/fsh:633-664; xi = n x 3). */
int ezrt_eval_brdf(int device, int which, int n, const float* V, const float* N, const float* L,
                   const float* xi, const float* materials, float* out);

/* Evaluate the mixture of EZRT_PARAM_TRANSMISSION (ezrt_math.h, DESIGN.md section 12) on the device for n (V, N, L, inside,
 * material) tuples (materials: 18 floats each, inside: 1 if the hit is from inside the medium).  out: 8 floats per tuple,
 * unused ones 0.  which = 0: f (3); 1: pdf (1); 2: the BSDF sample of xi[4 i .. 4 i + 3] = (xi_1, xi_2, xi_3, r_t), L unused:
 * L (3), the f (3), pdf and signed cosine the path carries, or 8 zeros if the path ends. */
int ezrt_eval_bsdf(int device, int which, int n, const float* V, const float* N, const float* L, const float* xi,
                   const int32_t* inside, const float* materials, float* out);

/* The camera rays of n samples (pixel px[i], py[i] of params' image, frame[i]; host arrays) as the render's kernels generate
 * them: the pinhole ray, or the thin-lens ray with EZRT_PARAM_THIN_LENS (validated as a render validates it).  origins_out,
 * dirs_out: n x 3 floats.  For parity tests, like ezrt_eval_bsdf: it allocates and synchronises per call. */
int ezrt_camera_rays(ezrt_scene* scene, const ezrt_render_params* params, int n, const uint32_t* px, const uint32_t* py,
                     const uint32_t* frame, float* origins_out, float* dirs_out);

/* Evaluate a ezrt_math.h function on the device for n inputs (parity of the arithmetic
 * definition): which = 0 sin, 1 cos, 2 log, 3 exp, 4 pow(a,b), 5 atan2(a,b), 6 asin, 7 floor. */
int ezrt_eval_math(int device, int which, int n, const float* a, const float* b, float* out);

/* The binary SAH tree ezrt_scene_create derives its acceleration tree from (NOT the reference's tree: the same
 * exhaustive sweep as buildBVHwithSAH, P5/main.cpp:458-589, without the INF = 114514 cost sentinel, leaves of <= leaf_n
 * triangles), built where = 0 on the GPU (csrc/accel_build.cu, what ezrt_scene_create uses) or where = 1 on the host
 * (host_scene.cpp); both produce the same array.  links_out: 4 ints per node (left, right, n, index; node 0 = root),
 * boxes_out: 6 floats per node (AA, BB), order_out: n_triangles triangle indices (the tree's triangle order); any may be
 * NULL.  nodes_cap = capacity of links_out / boxes_out in nodes.  Returns the node count or a negative status;
 * *ms = wall-clock of the build (device: upload of the triangles and read-back of the tree included). */
int ezrt_accel_build(int device, const float* tris, int n_triangles, int leaf_n, int where, int32_t* links_out,
                     float* boxes_out, int nodes_cap, uint32_t* order_out, double* ms);

/* ----------------------------------------------------------------------------------------
 * Post pass (SURVEY.md 8f "next" row 3): what the user sees.
 * -------------------------------------------------------------------------------------- */

/* pass3 (P5/shaders/pass3.fsh:14-25): toneMapping(c, limit) = c * 1.0 / (1.0 + lum/limit) with
 * lum = 0.3 r + 0.6 g + 0.1 b (limit = 1.5 in the shader), then pow(c, 1/2.2).  Device kernel:
 * d_in has `channels` (3 or 4) floats per pixel, d_out 3 floats per pixel. */
int ezrt_post_tonemap(const float* d_in, int channels, float* d_out, int64_t n_pixels, float limit, void* cuda_stream);
/* Host: write a linear framebuffer (row 0 = bottom, as ezrt_render returns it) as an 8-bit RGB PNG, top row
 * first; tonemap = 1 applies pass3 first; quantisation is P1's imshow(): (unsigned char)clamp(v*255, 0, 255)
 * (P1/main.cpp:173-194; P1 wrote its PNG with the vendored svpng.inc, this is an independent writer). */
int ezrt_write_png(const char* path, const float* framebuffer, int width, int height, int channels, int tonemap);

/* ----------------------------------------------------------------------------------------
 * Host side: the scene pipeline that feeds the path (stays on the CPU, north_star).
 * -------------------------------------------------------------------------------------- */

typedef struct ezrt_trilist ezrt_trilist; /* std::vector<Triangle> of P5/main.cpp:801 */

ezrt_trilist* ezrt_trilist_create(void);
void ezrt_trilist_destroy(ezrt_trilist* list);
int ezrt_trilist_size(const ezrt_trilist* list);

/* getTransformMatrix (P5/main.cpp:255-271): translate * rotate(x,y,z degrees) * scale,
 * column-major out[16]. */
void ezrt_transform_matrix(const float rotate_deg[3], const float translate[3], const float scale[3],
                           float out[16]);
/* readObj (P5/main.cpp:274-392) incl. its unit-box normalisation quirk (:317-318),
 * transform, smooth-normal generation and per-mesh material (18 floats: emissive,
 * baseColor, subsurface, metallic, specular, specularTint, roughness, anisotropic, sheen,
 * sheenTint, clearcoat, clearcoatGloss, IOR, transmission).  IOR and transmission are read only by
 * renders with EZRT_PARAM_TRANSMISSION. */
int ezrt_trilist_read_obj(ezrt_trilist* list, const char* path, const float material[EZRT_MATERIAL_FLOATS],
                          const float trans[16], int smooth_normal);
/* smooth_normal is a flag word: bit 0 = smoothNormal; EZRT_OBJ_HARDENED additionally accepts negative
 * (relative) vertex indices and fan-triangulates polygons -- the reference cuts a polygon to its first three
 * vertices (P5/main.cpp:321-336), which stays the default behaviour. */
#define EZRT_OBJ_HARDENED 2
/* Same parser on an in-memory OBJ text (synthetic meshes). */
int ezrt_trilist_read_obj_text(ezrt_trilist* list, const char* text, size_t len,
                               const float material[EZRT_MATERIAL_FLOATS], const float trans[16],
                               int smooth_normal);
/* ezrt_trilist_read_obj[_text] that also reads the mesh's texture coordinates, for EZRT_PARAM_TEXTURES: the "vt u v [w]" lines
 * (w ignored) and each face vertex's vt index ("v/vt" and "v/vt/vn"; with EZRT_OBJ_HARDENED also negative, relative ones, and the
 * UVs follow the fan).  A triangle whose three vertices all carry a vt gets their UVs and texture_id (>= 0, or -1), any other
 * texture id -1.  A vt index out of range is EZRT_ERR_IO.  Positions, normals and materials are exactly read_obj's. */
int ezrt_trilist_read_obj_textured(ezrt_trilist* list, const char* path, const float material[EZRT_MATERIAL_FLOATS],
                                   const float trans[16], int smooth_normal, int32_t texture_id);
int ezrt_trilist_read_obj_textured_text(ezrt_trilist* list, const char* text, size_t len, const float material[EZRT_MATERIAL_FLOATS],
                                        const float trans[16], int smooth_normal, int32_t texture_id);
/* Append already-built triangles in Triangle_encoded layout (texture id -1; also read_obj's triangles). */
int ezrt_trilist_append_encoded(ezrt_trilist* list, const float* tris, int n);
/* The texcoords (6 floats: u1, v1, u2, v2, u3, v3) and texture id of every triangle, in the list's current order: after
 * ezrt_trilist_build_bvh, the order of the encoded triangles, i.e. what ezrt_scene_set_textures takes. */
int ezrt_trilist_encode_texcoords(const ezrt_trilist* list, float* uv_out, int32_t* id_out);

typedef enum ezrt_bvh_builder {
    EZRT_BVH_SAH_FAST = 0,    /* same tree as SAH_LITERAL, keys pre-computed, subtrees in parallel */
    EZRT_BVH_SAH_LITERAL = 1, /* buildBVHwithSAH exactly as written (P5/main.cpp:458-589)   */
    EZRT_BVH_MEDIAN = 2,      /* buildBVH (P5/main.cpp:395-455)                              */
    EZRT_BVH_SAH_NO_SENTINEL = 3 /* NOT the reference tree: same sweep SAH without the INF = 114514
                                    cost cut-off (P5/main.cpp:20,:493); what the device builds
                                    internally as its acceleration tree (DESIGN.md "accel")      */
} ezrt_bvh_builder;

/* Sorts the list's triangles in place and builds the node array: nodes{testNode};
 * buildBVHwithSAH(triangles, nodes, 0, N-1, leaf_n) (P5/main.cpp:830-838).  Returns the
 * node count (incl. dummy node 0) or a negative status. */
int ezrt_trilist_build_bvh(ezrt_trilist* list, int leaf_n, int builder);
int ezrt_trilist_node_count(const ezrt_trilist* list);
/* 1 if this host's std::sort orders equal keys as libstdc++ does, i.e. the SAH_LITERAL / SAH_FAST / MEDIAN builders
 * reproduce the triangle order of the reference built with libstdc++ (its buildBVH* sort with order-only comparators,
 * P5/main.cpp:403-413, :560-568) and the goldens of this repository; 0 = the trees are valid but differ from the
 * reference's wherever centroid coordinates tie (ezrt_trilist_build_bvh then warns once on stderr). */
int ezrt_host_sort_is_reference(void);
/* Encode as P5/main.cpp:843-871 into caller buffers (36 floats/triangle, 12 floats/node). */
int ezrt_trilist_encode_triangles(const ezrt_trilist* list, float* tris_out);
int ezrt_trilist_encode_nodes(const ezrt_trilist* list, float* nodes_out);

/* Scene description file (SURVEY.md 8f row 4) in place of the hard-coded scene blocks of main()
 * (P3/main.cpp:688-701, P4/main.cpp:687-729, P5/main.cpp:795-823): directives `set <field> ...`, `reset`,
 * `mesh <obj> smooth|flat [hardened] rotate.. translate.. scale..`, `camera <rotatAngle> <upAngle> <r>`,
 * `hdr <path>`; appends the meshes to `list`; camera[3] and hdr_path (nullable) receive the other settings. */
int ezrt_scene_file_load(const char* path, ezrt_trilist* list, float camera[3], char* hdr_path, size_t hdr_path_cap);

/* HDRLoader::load (P5/lib/hdrloader.cpp:29-97): Radiance .hdr -> float RGB rows.  Call with
 * cols = NULL to query width/height.  Returns 0, or 1 when the pixel data ended early or was malformed (a run marker
 * with nothing to repeat, a run length beyond 32 bits): like the reference the rows decoded so far are kept and the
 * rest is zero, but unlike it nothing outside the scanline buffer is read; < 0 on errors. */
int ezrt_hdr_load(const char* path, int* width, int* height, float* cols);
/* calculateHdrCache (P5/main.cpp:592-689): (sample_x, sample_y, pdf) lookup texture. */
int ezrt_hdr_cache(const float* hdr, int width, int height, float* cache_out);

/* calculateHdrCache on the GPU `device` (SURVEY.md 8f row 1): same bits as ezrt_hdr_cache -- every fp32
 * sum keeps the reference's order -- host arrays in and out; device_ms (nullable) = kernel time. */
int ezrt_hdr_cache_device(int device, const float* hdr, int width, int height, float* cache_out, double* device_ms);

/* Camera of display() (P5/main.cpp:710-713): orbit angles in degrees + radius ->
 * eye, cameraRotate = inverse(lookAt(eye, 0, +y)), column-major. */
void ezrt_camera_orbit(float rotate_angle_deg, float up_angle_deg, float r, float eye[3],
                       float camera_rotate[16]);
/* A look-at camera with a vertical field of view (degrees, 0 < vfov_deg < 180) and an aspect ratio (width / height): the
 * cameraRotate whose columns are the orthonormal right, up and back vectors of lookAt(eye, target, up) (as camera_orbit's
 * inverse(lookAt)), column 0 scaled by aspect * tan(vfov/2) * 1.5 and column 1 by tan(vfov/2) * 1.5, column 3 = (eye, 1).
 * The pinhole kernels then render that field of view and aspect (they map the image to [-1, 1]^2 at depth 1.5).  Returns
 * EZRT_ERR_INVALID for a degenerate view (eye == target, up parallel to the view), vfov_deg outside (0, 180) or
 * aspect <= 0 or not finite. */
int ezrt_camera_look_at(const float eye[3], const float target[3], const float up[3], float vfov_deg, float aspect,
                        float cam_out[16]);

#ifdef __cplusplus
}
#endif
#endif /* EZRT_H */
