// device_scene.h -- HBM layouts of the repacked scene and per-render constants.
//
// The C ABI accepts the reference's layouts (Triangle_encoded 144 B, BVHNode_encoded 48 B,
// P5/main.cpp:60-76); ezrt_scene_create() repacks them once into 128-bit-aligned records:
//
//   inner node (64 B, "children in parent"): one 4 x float4 record per INNER node holding both
//       child boxes and both child references, so a traversal step is one 64-byte fetch instead
//       of the shader's three dependent 48-byte getBVHNode()s (P5/fsh:266,281,285).  Components
//       are paired for the packed FADD2/FMUL2 slab arithmetic:
//         q0 = (AA_l.x, AA_l.y, BB_l.x, BB_l.y)   q1 = (AA_r.x, AA_r.y, BB_r.x, BB_r.y)
//         q2 = (AA_l.z, BB_l.z, AA_r.z, BB_r.z)   q3 = (ref_left, ref_right, 0, 0)
//       ref >= 0 : index of an inner-node record;  ref < 0 : leaf, bits = 1|index(24)|n(7)
//   triangle geometry (64 B): q0 = (p1, N.x) q1 = (p2, N.y) q2 = (p3, N.z) q3 = (d0,0,0,0)
//       N = normalize(cross(p2-p1, p3-p1)) and d0 = dot(N,p1) are the ray-independent part of
//       hitTriangle (P5/fsh:172,184), evaluated once with the same fp32 operations.
//       (the accel-order copy of an 8-wide scene that shares its vertices is indexed instead, 32 B: (N, d0) (i1, i2, i3, 0)
//       into a 16-byte vertex array (x, y, z, 0); SceneDev::acc_tri_indexed, DESIGN.md section 4)
//   triangle shading (48 B): (n1, matId) (n2, 0) (n3, 0)  -- fetched only for the final hit
//   material table (80 B each): the 18-float material block de-duplicated (SURVEY.md 0: materials
//       are stored per triangle in the reference), padded to 5 x float4.
//   acceleration tree of the default traversal policy (DESIGN.md section 4): the device's own sentinel-free SAH tree over the
//       same triangles, as 4-wide nodes with exact boxes (128 B: four child boxes + four references, default) or as 8-wide
//       nodes with 8-bit quantised boxes (96 B, w8_node.h; env EZRT_ACCEL=8), plus geometry / shading records in its order.
#ifndef EZRT_DEVICE_SCENE_H
#define EZRT_DEVICE_SCENE_H

#include <cuda_runtime.h>
#include <stdint.h>

#include "ezrt_math.h"

#define EZRT_MAX_STACK 256       // >= validated tree depth + 1: the shader's own bound, int stack[256] (P5/fsh:260)
#define EZRT_LEAF_FLAG 0x80000000u
#define EZRT_LEAF_MAX_N 127
#define EZRT_TOP_NODES_MAX 1023   // 10 full levels; 80 B each in shared memory (bank-conflict padding)
#define EZRT_TRI_PENDING (-2)      // hit record of a ray the accel kernel deferred to the exact pass (a miss is -1)
#define EZRT_SIDE_CAP 65536u       // deferred rays per pass handled on the side stream beside k_shade; more: in line, as before
#define EZRT_ACCEL_STACK 64       // stack entries of the 4-wide accel kernel (<= 3 pushes per level): trees deeper than 20 levels are not built
#define EZRT_W8_SMEM_STACK 16      // per-lane W8 stack entries held in shared memory (8 B each x 1024 threads = 128 KB at most)
#define EZRT_TOP_STRIDE 5         // float4 per shared-memory record
#define EZRT_TILE 16             // == EZRT_PART_TILE
#define EZRT_TILE_PIXELS 256
#define EZRT_SORT_BITS 18         // ray sort key: direction octant (3) | 5-5-5 Morton cell of the origin
#define EZRT_SORT_BINS (1 << EZRT_SORT_BITS)

struct SceneDev {
    const float4* nodes;      // 4 float4 per inner node
    const float4* tri_geo;    // 4 float4 per triangle: (N, d0), (p1, 0), (p2, 0), (p3, 0)
    const float4* tri_shade;  // 3 float4 per triangle
    const float4* materials;  // 5 float4 per material
    const float* hdr;         // W*H*3 or null
    const float* hdr_cache;   // W*H*3 or null
    int hdr_w, hdr_h, hdr_linear;
    int root_ref;
    // acceleration tree (default traversal policy): sentinel-free SAH over the same triangles, boxes
    // inflated by 2*prune_delta; acc_tri_geo is tri_geo in the tree's own order, acc_tri_ref maps back
    const float4* acc_tri_geo;     // flat: 4 float4 per triangle as tri_geo; indexed: 2 per triangle, (N, d0) (i1, i2, i3, 0 as int bits)
    const float4* acc_tri_vert;    // indexed layout: the distinct vertex positions (x, y, z, 0) of acc_tri_geo, numbered by first use
    int acc_tri_indexed;           // 1: acc_tri_geo holds 32-byte indexed records (W8 scenes whose vertices are shared), 0: flat
    const uint32_t* acc_tri_ref;   // accel order -> reference triangle index
    const uint32_t* ref_to_acc;    // reference triangle index -> accel order
    const float4* acc_tri_shade;   // tri_shade in accel order (shading reads the arrays traversal keeps hot in L2)
    const int* acc_tri_leaf;       // reference leaf (slot in leaf_box) of every triangle, accel order
    const uint4* w8_nodes;         // the tree as 8-wide nodes with 8-bit quantised child boxes (80 B records, w8_node.h); null = none
    int w8_near_bit[3];            // significance of axis a in the slot index (octant order)
    int w8_stack_entries;          // per-lane stack entries kept in shared memory (>= depth of the 8-wide tree, or the smem cap)
    int w8_tri_weight;             // step vote of the W8 kernels: triangle step iff w8_tri_weight * min(pending_triangles, 32) >= lanes_with_a_node (env EZRT_TRI_W)
    uint32_t w8_decode_bits;       // W8_DECODE_BITS (passed as data: see w8_plane in device_functions.cuh)
    float w8_origin_limit;         // rays starting further out than this (any |coordinate|) go to the exact kernel (decode error bound)
    float quant_inv_limit;         // ... and rays with a larger |1/d_a| (decode range of the W8 or Q16 nodes: ezrt_quant_inv_limit, <= W8_INV_LIMIT)
    const float4* acc_wide_nodes;  // 4-wide nodes with exact boxes (128 B records): the accel form of scenes below 2^16 triangles (W8 above)
    int acc_wide_root_ref;
    const uint4* acc_wide_q16;     // the same 4-wide nodes with 16-bit quantised planes (96 B records, same numbering): bounce / shadow launches
    uint32_t q16_decode_bits;      // 0x4B000000, passed as data so that it stays in a register (see w8_plane)
    // reference leaf of every reference triangle + the leaves' boxes (AA, BB as float4 pairs)
    const int* tri_leaf;
    const float4* leaf_box;
    int n_triangles;
    int tri_l1_bypass;        // triangle records are read with LDG.NA (set for scenes whose geometry exceeds a few MB)
    int n_inner;
    int top_nodes;            // records [0, top_nodes) = the top tree levels, staged in shared memory
    float prune_delta;        // 2^-16 * max |vertex coordinate|
    int refill_thresh;        // persistent traversal tunables (env EZRT_REFILL_T / EZRT_INNER_T)
    int refill_thresh_camera; // the same for the camera pass, whose rays are coherent (env EZRT_REFILL_CAM; 0 = refill_thresh)
    int inner_thresh;
    int leaf_thresh;
    int work_chunk;           // rays a warp takes from the work counter at a time (env EZRT_CHUNK)
    int work_chunk_camera;    // the same for the camera pass (pixel-major order: 64 = the 16 samples of 4 pixels; env EZRT_CHUNK_CAM)
    float bmin[3];            // scene bounding box (ray-sort cells)
    float cell_scale[3];      // 32 / extent per axis
};

struct RenderDev {
    int width, height;
    int mode, max_bounce;
    int traverse;             // ezrt_traverse
    float eye[3];
    float cam[16];            // column-major cameraRotate
    float env[3];
    uint32_t first_frame;
    int out_channels;
    int compact_out;          // 1: write tile-major compact buffer (part_count > 1)
    int accel_space;          // 1: hit records hold acceleration-tree triangle indices (accel policy)
    int n_tiles;              // tiles owned by this part
};

// One owned 16x16 tile (clipped at the image border)
struct TileDev {
    int x0, y0, w, h;
    int pixel_offset;         // offset of the tile's first pixel in the compact buffer
};

// SoA path state of the wavefront pipeline (one set per queue; two queues ping-pong): 64 B per path + 8 B hit record.
struct PathQueue {
    float4* ray_o;    // (origin.xyz, rng seed as bits)
    float4* ray_d;    // (direction.xyz, sample slot as bits)
    float2* hit;      // written by extend: (hit distance, triangle index as int bits; -1 = miss)
    float4* hist;     // (history.xyz, cosine_i)
    float4* fr;       // (f_r.xyz, pdf)   pdf <= 0 marks "break after trace" (P5/fsh:865)
};

// The emissive-triangle light table of mode EZRT_MODE_DISNEY_LIGHTS (ezrt_math.h, DESIGN.md section 10), built at the first
// render in that mode.  Passed to k_shade / k_nee as a parameter of its own (not a SceneDev member, so the other kernels keep
// their parameter layout).  Light record k (64 B): (p1, material id as bits) (p2, reference triangle index as bits)
// (p3, accel-order triangle index as bits) (N, ez_luminance(emissive)).
struct LightsDev {
    const float4* rec;   // 4 float4 per light
    const float* cdf;    // n floats, cdf[n - 1] = 1
    int n;               // 0: no light (no light samples)
    float w_total;       // W_f = (float) sum of the weights
};

// The environment map's light table (EZRT_PARAM_ENV_LIGHT; ezrt_math.h, DESIGN.md section 11), built at the first flagged render
// of a scene with a map.  Passed to the k_shade instantiations as a parameter of its own, after LightsDev.
struct EnvDev {
    const float* row_cdf;     // H floats, row_cdf[H - 1] = 1
    const float* col_cdf;     // H x W floats, row-major
    const float* texel_pdf;   // H x W floats, row-major
    int w, h;
    float p_env;              // the probability of an environment sample: 1/2 beside triangle lights, 1 without
};

// The thin lens of EZRT_PARAM_THIN_LENS (ez_lens_setup, ezrt_math.h; DESIGN.md section 13): eye, the unit axes of the lens,
// the focus scale and the radius.  Passed to the lens instantiations (k_generate<true>, k_megakernel<.., true>) as a parameter
// of their own, after the others, so that no other kernel's parameter layout moves.
typedef ez_lens LensDev;

// The homogeneous medium of EZRT_PARAM_MEDIUM (ezrt_math.h, DESIGN.md section 14): sigma_t, albedo, g and the box, copied from the
// scene when the render is enqueued.  Passed to the medium instantiations (k_shade<.., MEDIUM>, k_nee<.., MEDIUM>) as a parameter of
// their own, after the others.  A medium vertex's shadow ray carries EZRT_MEDIUM_VERTEX as its material id (ShadowQueue::ray_d.w;
// no ~matId there, as EZRT_PARAM_TRANSMISSION is excluded) and its propagation direction d in place of V.
typedef ez_medium MediumDev;
#define EZRT_MEDIUM_VERTEX (-1)

// The base-colour textures of EZRT_PARAM_TEXTURES (ezrt_math.h, DESIGN.md section 15), set by ezrt_scene_set_textures.  Passed to the
// textured instantiations (k_shade<.., TEX>, k_nee<.., TEX>) as a parameter of their own, after the others.
//   rec / acc_rec: 32 bytes per triangle, (u1, v1, u2, v2) (u3, v3, texture id as bits, 0), in reference and in accel order (hit
//       records hold either index, RenderDev::accel_space)
//   table: per texture (offset of its first texel in texels, W, H, 0); texels: RGBA8 words; lut: ez_srgb_table, read through L1
//   sh_base: the textured base colour of every shadow slot's shading point (16 B per slot, carved beside the shadow queue for the
//       flagged renders only), read back by k_nee, which reloads the material from its id
struct TexDev {
    const float4* rec;
    const float4* acc_rec;
    const int4* table;
    const uint32_t* texels;
    const float* lut;
    float4* sh_base;
};
// The material maps of EZRT_PARAM_MATERIAL_MAPS (ezrt_math.h, DESIGN.md section 16), set by ezrt_scene_set_material_maps: their ids
// are the fourth word of TexDev's records, (metal_rough_id + 1) | (normal_id + 1) << 16 (0: no maps).  Passed to the maps
// instantiations (k_shade<.., TEX, MAPS>, k_nee<.., TEX, MAPS>) as one more parameter, after TexDev.
//   unorm: ez_unorm8_table, read through L1
//   sh_metal: the mapped metallic of every shadow slot's shading point (4 B per slot, after TexDev::sh_base, maps renders only); the
//       mapped roughness rides in sh_base[j].w
struct MapsDev {
    const float* unorm;
    float* sh_metal;
};

// A shadow ray and what k_nee needs to evaluate the light sample's contribution once the ray got through (nee_contrib):
// the BRDF / environment evaluation of the light sample is done after the shadow pass, for unoccluded rays only.
#define EZRT_SHADOW_SLOT_BYTES (5 * 16 + 1)
struct ShadowQueue {
    float4* ray_o;       // (origin.xyz, sample slot as bits)
    float4* ray_d;       // (direction to the light.xyz, material id as bits)
    float4* nrm;         // (shading normal N.xyz, -; bounded rays of the light sampling mode: tmax, EZ_INF for the environment)
    float4* view;        // (V = -incoming direction.xyz, -; light sampling mode: pdf of the light sample)
    float4* hist;        // (path history.xyz, -; light sampling mode: the light's material id as bits, -1 for the environment)
    unsigned char* lit;  // written by the shadow pass: 1 = nothing between the surface and the environment
};

#endif
