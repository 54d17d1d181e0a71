// kernels.cu -- sm_90a kernels of the wavefront path tracer and their launchers.
//
// Pipeline per batch of `nf` frames (= display() calls, P5/main.cpp:697-748) x owned pixels:
//   k_generate : camera rays (main(), P5/fsh:920-925) -> queue 0   (exact policies; the accel policy generates them inside
//                the first extend kernel, k_extend_accel_camera, and again in k_shade(0))
//   per bounce b = 0..maxBounce:
//     k_extend_accel : hitBVH for every queued ray on the device's 4-wide acceleration tree (persistent warps,
//                      per-lane refill, vote-driven inner / leaf phases); rays it cannot decide exactly are
//                      deferred to  k_extend  = the exact reference-order traversal (also the whole extend
//                      stage under the REFERENCE / PRUNED policies) -- on a side stream, followed by
//                      k_shade<MODE, LIST> over the deferred rays, beside the main k_shade ("deferred lane")
//     k_shade        : account the hit/miss, light sample + BRDF sampling, block-aggregated compaction -> queue b+1
//     k_shadow_accel / k_shadow : any-hit trace of the environment shadow rays (IS mode only): marks each ray lit / occluded
//     k_nee          : the lit light samples' contributions (BRDF, environment, MIS) -> Lo
//   k_blend    : running mean into the framebuffer in frame order (P5/fsh:942-947)
// Adaptive sampling adds k_blend<true> (also the running mean of the squared luminance and the spp map) and, at each test
// point, k_adaptive_check (drops converged tiles from the tile list the next batches run on).
// No host synchronisation inside a render: queue sizes live in device counters.
#include "kernels.h"

#include <cstdlib>
#include <map>
#include <mutex>
#include <type_traits>

#include "device_functions.cuh"

// ------------------------------------------------------------------------------------------
// slot <-> pixel mapping.  A sample slot is (frame_in_batch, tile, in_tile); in_tile enumerates
// the 16x16 tile as eight 8x4 sub-blocks so that a warp covers a compact 8x4 pixel block.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void in_tile_xy(int in_tile, int& ix, int& iy) {
    int sub = in_tile >> 5, lane = in_tile & 31;
    ix = (sub & 1) * 8 + (lane & 7);
    iy = (sub >> 1) * 4 + (lane >> 3);
}
__device__ __forceinline__ bool slot_pixel(const RenderDev& rd, const TileDev* __restrict__ tiles, uint32_t slot,
                                           uint32_t& px, uint32_t& py, uint32_t& frame_in_batch) {
    uint32_t per_frame = (uint32_t)rd.n_tiles * EZRT_TILE_PIXELS;
    frame_in_batch = slot / per_frame;
    uint32_t r = slot - frame_in_batch * per_frame;
    TileDev t = tiles[r >> 8];
    int ix, iy;
    in_tile_xy((int)(r & 255u), ix, iy);
    px = (uint32_t)(t.x0 + ix);
    py = (uint32_t)(t.y0 + iy);
    return ix < t.w && iy < t.h;
}

// block-aggregated append: returns this thread's position in the output queue (valid threads only).
// One atomicAdd per BLOCK: all queue appends of a kernel hit a single counter, and the L2 atomic unit
// serialises per address (~2 M warp-level atomics per step were a measurable part of k_shade/k_generate).
// Must be reached by every thread of the block (uniform loop trip counts).
__device__ __forceinline__ uint32_t block_append(bool valid, uint32_t* counter, uint32_t* s_scan /* [34] */) {
    const unsigned mask = __ballot_sync(0xffffffffu, valid);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, n_warps = (blockDim.x + 31) >> 5;
    if (lane == 0) s_scan[wid] = (uint32_t)__popc(mask);
    __syncthreads();
    if (wid == 0) {
        uint32_t v = (lane < n_warps) ? s_scan[lane] : 0u;
        uint32_t incl = v;
        for (int off = 1; off < 32; off <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, incl, off);
            if (lane >= off) incl += t;
        }
        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
        uint32_t base = 0;
        if (lane == 0 && total != 0u) base = atomicAdd(counter, total);
        base = __shfl_sync(0xffffffffu, base, 0);
        s_scan[lane] = base + incl - v;  // start of each warp's range
    }
    __syncthreads();
    const uint32_t pos = s_scan[wid] + (uint32_t)__popc(mask & ((1u << lane) - 1u));
    __syncthreads();  // s_scan is reused by the next append
    return pos;
}

// ------------------------------------------------------------------------------------------
// LENS (EZRT_PARAM_THIN_LENS): the thin-lens camera rays of `lens`, written to the same records; every policy traces them from
// the queue at bounce 0
template <bool LENS>
__global__ void __launch_bounds__(256) k_generate(RenderDev rd, const TileDev* __restrict__ tiles, uint32_t n_slots,
                                                  uint32_t batch_first_frame, PathQueue q, uint32_t* q_count, LensDev lens) {
    __shared__ uint32_t s_scan[34];
    uint32_t stride = gridDim.x * blockDim.x;
    uint32_t n_round = ((n_slots + blockDim.x - 1u) / blockDim.x) * blockDim.x;
    for (uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x; slot < n_round; slot += stride) {
        uint32_t px = 0, py = 0, fib = 0;
        bool valid = (slot < n_slots) && slot_pixel(rd, tiles, slot, px, py, fib);
        uint32_t pos = block_append(valid, q_count, s_scan);
        if (!valid) continue;
        uint32_t seed;
        vec3 o, d;
        camera_ray<LENS>(rd, lens, px, py, batch_first_frame + fib, seed, o, d);
        __stcs(q.ray_o + pos, make_float4(o.x, o.y, o.z, __uint_as_float(seed)));
        __stcs(q.ray_d + pos, make_float4(d.x, d.y, d.z, __uint_as_float(slot)));
    }
}

// ------------------------------------------------------------------------------------------
// extend: closest hit for every ray of the queue.  Persistent warps fetch 32 rays at a time from
// a global work counter so long traversals do not stall a statically assigned tail.
// ------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------
// Ray sort (bounce rays): counting sort of ray indices by key = direction octant | Morton cell of
// the origin.  Diffuse bounce rays leave the shade kernel in path order with unrelated directions;
// after the sort the 32 rays a warp fetches start close together and head the same way, so their
// traversals touch the same nodes (L1 hits, lanes finishing together).  Only the index permutation
// is sorted: rays and results stay where they are, and every ray's result is independent of the
// order in which rays are traced.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t spread5(uint32_t v) {  // 5 bits -> every third bit
    v &= 31u;
    v = (v | (v << 8)) & 0x100fu;
    v = (v | (v << 4)) & 0x10c3u;
    v = (v | (v << 2)) & 0x1249u;
    return v;
}
__device__ __forceinline__ uint32_t ray_sort_key(const SceneDev& sc, float4 o4, float4 d4) {
    int cx = min(31, max(0, (int)((o4.x - sc.bmin[0]) * sc.cell_scale[0])));
    int cy = min(31, max(0, (int)((o4.y - sc.bmin[1]) * sc.cell_scale[1])));
    int cz = min(31, max(0, (int)((o4.z - sc.bmin[2]) * sc.cell_scale[2])));
    uint32_t oct = (d4.x < 0.0f ? 1u : 0u) | (d4.y < 0.0f ? 2u : 0u) | (d4.z < 0.0f ? 4u : 0u);
    return (oct << 15) | spread5((uint32_t)cx) | (spread5((uint32_t)cy) << 1) | (spread5((uint32_t)cz) << 2);
}

__global__ void __launch_bounds__(256) k_sort_hist(SceneDev sc, PathQueue q, const uint32_t* __restrict__ q_count, uint32_t* __restrict__ keys,
                                                   uint32_t* __restrict__ bins) {
    const uint32_t n = *q_count;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        uint32_t key = ray_sort_key(sc, q.ray_o[i], q.ray_d[i]);
        keys[i] = key;
        atomicAdd(&bins[key], 1u);
    }
}

// exclusive scan of the EZRT_SORT_BINS counters, one block of 1024 threads
__global__ void __launch_bounds__(1024) k_sort_scan(uint32_t* __restrict__ bins) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t carry;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    constexpr int PER = 8;  // elements per thread per round
    for (uint32_t base = 0; base < EZRT_SORT_BINS; base += 1024 * PER) {
        uint32_t v[PER];
        uint32_t sum = 0;
        const uint32_t idx = base + (uint32_t)tid * PER;
#pragma unroll
        for (int k = 0; k < PER; k++) {
            v[k] = bins[idx + k];
            sum += v[k];
        }
        uint32_t incl = sum;
        for (int off = 1; off < 32; off <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, incl, off);
            if (lane >= off) incl += t;
        }
        if (lane == 31) warp_sums[wid] = incl;
        __syncthreads();
        if (wid == 0) {
            uint32_t w = warp_sums[lane];
            uint32_t wi = w;
            for (int off = 1; off < 32; off <<= 1) {
                uint32_t t = __shfl_up_sync(0xffffffffu, wi, off);
                if (lane >= off) wi += t;
            }
            warp_sums[lane] = wi - w;  // exclusive prefix of warp totals
        }
        __syncthreads();
        uint32_t excl = carry + warp_sums[wid] + (incl - sum);
#pragma unroll
        for (int k = 0; k < PER; k++) {
            bins[idx + k] = excl;
            excl += v[k];
        }
        __syncthreads();
        if (tid == 1023) carry = excl;  // total so far
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_sort_scatter(const uint32_t* __restrict__ q_count, const uint32_t* __restrict__ keys,
                                                      uint32_t* __restrict__ bins, uint32_t* __restrict__ perm) {
    const uint32_t n = *q_count;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        uint32_t pos = atomicAdd(&bins[keys[i]], 1u);
        perm[pos] = i;
    }
}

// the top levels of the tree a kernel walks, copied from global memory by every persistent block at start
extern __shared__ float4 g_smem_top[];
__device__ __forceinline__ void stage_top_nodes(const TreeView& tree) {
    const int n4 = tree.top_nodes * 4;
    for (int i = threadIdx.x; i < n4; i += blockDim.x) g_smem_top[(i >> 2) * EZRT_TOP_STRIDE + (i & 3)] = tree.nodes[i];
    __syncthreads();
}
__device__ __forceinline__ TreeView reference_tree(const SceneDev& sc) {
    TreeView t;
    t.nodes = sc.nodes; t.tri_geo = sc.tri_geo; t.root_ref = sc.root_ref; t.top_nodes = sc.top_nodes; t.wide = 0;
    return t;
}
// the 4-wide exact-box form (round-1 kernel, env EZRT_ACCEL=4).  Its kernels run only on scenes without a W8 tree, whose
// acc_tri_geo is always flat (the indexed layout is chosen for W8 scenes only: capi.cu)
__device__ __forceinline__ TreeView accel_tree(const SceneDev& sc) {
    TreeView t;
    t.nodes = sc.acc_wide_nodes; t.tri_geo = sc.acc_tri_geo; t.root_ref = sc.acc_wide_root_ref; t.top_nodes = 0; t.wide = 1;
    return t;
}

// ---- exact kernels: the reference tree in the shader's order (policies REFERENCE and PRUNED, and the
// fallback pass of the accel policy, which traces only the deferred ray indices in `perm`)
struct ExtendIO {
    PathQueue q;
    const uint32_t* perm;      // null: trace in queue order
    const uint32_t* to_accel;  // non-null (fallback pass of the accel policy): hits are stored as accel-order indices
    float2* side_hit;          // non-null (that pass on the side stream): hit i of the list goes to side_hit[i], not to the queue
    __device__ __forceinline__ bool load(uint32_t i, vec3& o, vec3& d) const {
        const uint32_t j = perm ? perm[i] : i;
        float4 o4 = __ldcs(q.ray_o + j), d4 = __ldcs(q.ray_d + j);  // queue data streams through the caches
        o = ez_v3(o4.x, o4.y, o4.z);
        d = ez_v3(d4.x, d4.y, d4.z);
        return true;
    }
    __device__ __forceinline__ void store(uint32_t i, HitRec h, bool, vec3, vec3, vec3) const {
        const uint32_t j = perm ? perm[i] : i;
        int tri = h.tri;
        if (to_accel && tri >= 0) tri = (int)__ldg(to_accel + tri);
        if (side_hit) side_hit[i] = make_float2(h.t, __int_as_float(tri));
        else __stcs(q.hit + j, make_float2(h.t, __int_as_float(tri)));
    }
    __device__ __forceinline__ void defer(uint32_t, vec3, vec3) const {}
};

// gate (the accel policy's pass over the deferred rays, DESIGN.md "deferred lane"): 0 = always; 1 = only if the list holds at most
// EZRT_SIDE_CAP rays (side stream, results to side_hit, no tree staging: a handful of rays, run beside k_shade); 2 = only if it holds
// more (in line, results to the queue).  Exactly one of the passes 1 and 2 does the work.
template <bool PRUNE, bool ANYHIT>
__global__ void __launch_bounds__(EZRT_EXTEND_MAX_THREADS, EZRT_EXTEND_LB_BLOCKS) k_extend(SceneDev sc, PathQueue q, const uint32_t* __restrict__ q_count,
                                                                uint32_t* work, const uint32_t* __restrict__ perm, int to_accel, float2* side_hit, int gate) {
    ExtendIO io;
    io.q = q;
    io.perm = perm;
    io.to_accel = to_accel ? sc.ref_to_acc : nullptr;
    io.side_hit = side_hit;
    const uint32_t n = *q_count;
    if (blockIdx.x * blockDim.x >= n) return;   // nothing for this block (the pass over an accel kernel's deferred rays is usually empty):
                                                // do not stage 80 KB of tree for it
    if ((gate == 1 && n > EZRT_SIDE_CAP) || (gate == 2 && n <= EZRT_SIDE_CAP)) return;
    TreeView tree = reference_tree(sc);
    if (gate == 1) tree.top_nodes = 0;
    stage_top_nodes(tree);
    extend_persistent<PRUNE, ANYHIT, false, false, 8, false, false>(sc, tree, n, work, io, g_smem_top);
}

// ---- accel kernels: the device's own SAH tree finds the global closest hit G; the result is kept when
// the shader's traversal provably reaches G's leaf and nothing ties with G, otherwise the ray index is
// appended to `defer_list` for the exact kernel (DESIGN.md "accel").
// LL = lanes per leaf in the cooperative leaf phase: 4 when the acceleration tree was built with leaves <= 4
// (the IO structs of the accel kernels -- queue rays, fused camera rays, shadow rays -- are shared by the 4-wide and the W8
// kernel: AccelExtendIO, AccelCameraIO, AccelShadowIO below)

// ---- shadow rays: any hit; the pass marks each ray lit / occluded, k_nee then adds the contribution of the lit ones (P5/fsh:829-841).
struct ShadowIO {
    ShadowQueue sq;
    float4* Lo;
    const uint32_t* perm;
    __device__ __forceinline__ bool load(uint32_t i, vec3& o, vec3& d) const {
        const uint32_t j = perm ? perm[i] : i;
        float4 o4 = __ldcs(sq.ray_o + j), d4 = __ldcs(sq.ray_d + j);
        o = ez_v3(o4.x, o4.y, o4.z);
        d = ez_v3(d4.x, d4.y, d4.z);
        return true;
    }
    // every shadow ray's flag is written exactly once per pass (here, or by the exact pass over the rays an accel kernel deferred)
    __device__ __forceinline__ void mark(uint32_t j, bool lit) const { sq.lit[j] = lit ? 1 : 0; }
    // bounded shadow rays (light sampling mode): the bound travels in nrm.w
    __device__ __forceinline__ float tmax(uint32_t i) const { return __ldcs(sq.nrm + (perm ? perm[i] : i)).w; }
    __device__ __forceinline__ void store(uint32_t i, HitRec h, bool, vec3, vec3, vec3) const { mark(perm ? perm[i] : i, h.tri < 0); }
    __device__ __forceinline__ void defer(uint32_t, vec3, vec3) const {}
};

// BOUNDED (light sampling mode): ray j only looks for occluders strictly before sq.nrm[j].w (extend_persistent)
template <bool PRUNE, bool BOUNDED = false>
__global__ void __launch_bounds__(EZRT_EXTEND_MAX_THREADS, EZRT_EXTEND_LB_BLOCKS) k_shadow(SceneDev sc, ShadowQueue sq, const uint32_t* __restrict__ s_count,
                                                                uint32_t* work, float4* __restrict__ Lo, const uint32_t* __restrict__ perm) {
    ShadowIO io;
    io.sq = sq;
    io.Lo = Lo;
    io.perm = perm;
    const uint32_t n = *s_count;
    if (blockIdx.x * blockDim.x >= n) return;
    const TreeView tree = reference_tree(sc);
    stage_top_nodes(tree);
    extend_persistent<PRUNE, true, false, false, 8, false, false, BOUNDED>(sc, tree, n, work, io, g_smem_top);
}

// ---- accel kernels: the device's own tree (4-wide exact boxes: extend_persistent<ACCEL, WIDE>; or W8: extend_w8 on the
// 8-wide quantised tree with per-lane stacks and the octant permutation table in shared memory) finds the global closest hit
// G; the result is kept when the shader's traversal provably reaches G's leaf and nothing ties with G, otherwise the ray
// index is appended to `defer_list` for the exact kernel (DESIGN.md "accel").
__device__ __forceinline__ void w8_smem_setup(unsigned char*& s_perm, uint2*& stack_sm) {
    unsigned char* base = reinterpret_cast<unsigned char*>(g_smem_top);
    s_perm = base;
    stack_sm = reinterpret_cast<uint2*>(base + 2048);
    for (int i = threadIdx.x; i < 2048; i += blockDim.x) {
        const int m = i >> 8, x = i & 255;
        int y = 0;
        for (int b = 0; b < 8; b++)
            if ((x >> b) & 1) y |= 1 << (b ^ m);
        s_perm[i] = (unsigned char)y;
    }
    __syncthreads();
}

struct AccelExtendIO {
    PathQueue q;
    const int* acc_tri_leaf;
    const float4* leaf_box;
    uint32_t* defer_list;
    uint32_t* defer_count;
    const uint32_t* perm;      // non-null (env EZRT_SORT_RAYS=1, experiment): trace the queue entries in this order
    __device__ __forceinline__ bool load(uint32_t i, vec3& o, vec3& d) const {
        const uint32_t j = perm ? perm[i] : i;
        float4 o4 = __ldcs(q.ray_o + j), d4 = __ldcs(q.ray_d + j);
        o = ez_v3(o4.x, o4.y, o4.z);
        d = ez_v3(d4.x, d4.y, d4.z);
        return true;
    }
    __device__ __forceinline__ void defer(uint32_t i, vec3, vec3) const {
        const uint32_t j = perm ? perm[i] : i;
        __stcs(q.hit + j, make_float2(0.0f, __int_as_float(EZRT_TRI_PENDING)));   // k_shade leaves it to the pass over the deferred rays
        defer_list[atomicAdd(defer_count, 1u)] = j;
    }
    __device__ __forceinline__ void store(uint32_t i, HitRec h, bool tie, vec3 o, vec3 d, vec3 inv) const {
        if (h.tri >= 0 && (tie || !reference_reaches_leaf_inv(acc_tri_leaf, leaf_box, h.tri, o, inv))) {
            defer(i, o, d);
            return;
        }
        __stcs(q.hit + (perm ? perm[i] : i), make_float2(h.t, __int_as_float(h.tri)));  // accel-order triangle index
    }
    // store() in two halves (extend_w8): leaf_of(h.tri) when the ray ends, finish() with its result at a later refill
    __device__ __forceinline__ int leaf_of(int tri) const { return __ldg(acc_tri_leaf + tri); }
    __device__ __forceinline__ void finish(uint32_t i, HitRec h, bool tie, vec3 o, vec3 d, vec3 inv, int leaf) const {
        if (h.tri >= 0 && (tie || !reference_reaches_leaf_box(leaf_box, leaf, o, inv))) {
            defer(i, o, d);
            return;
        }
        __stcs(q.hit + (perm ? perm[i] : i), make_float2(h.t, __int_as_float(h.tri)));
    }
};

// Camera pass with the ray generation fused in (main(), P5/fsh:920-925): ray `i` IS sample slot i, generated in the
// lane that traces it -- no k_generate pass, no 40-byte queue record written and read back per camera ray.  Slots of
// clipped edge tiles that lie outside the image are skipped.  Only a deferred ray is written to the queue, for the
// exact kernel that re-traces it.
struct AccelCameraIO {
    RenderDev rd;
    const TileDev* tiles;
    uint32_t batch_first_frame;
    uint32_t n_frames;       // frames of this batch; 0: trace the slots in slot order (frame-major)
    uint32_t per_frame;      // sample slots per frame
    PathQueue q;
    const int* acc_tri_leaf;
    const float4* leaf_box;
    uint32_t* defer_list;
    uint32_t* defer_count;
    // Work index -> sample slot.  Pixel-major order: consecutive work items are the n_frames samples of ONE pixel -- camera rays
    // that differ only by their sub-pixel jitter (P5/fsh:923) -- so the 32 rays of a warp walk the same nodes and hit the same
    // triangles almost always (frame-major order gives a warp an 8x4 pixel block of one frame, which splits at every silhouette).
    __device__ __forceinline__ uint32_t slot_of(uint32_t i) const {
        if (n_frames == 0u) return i;
        const uint32_t p = i / n_frames;
        return (i - p * n_frames) * per_frame + p;
    }
    __device__ __forceinline__ bool load(uint32_t i, vec3& o, vec3& d) const {
        uint32_t px, py, fib, seed;
        if (!slot_pixel(rd, tiles, slot_of(i), px, py, fib)) return false;
        primary_ray(rd, px, py, batch_first_frame + fib, seed, o, d);
        return true;
    }
    __device__ __forceinline__ void defer_slot(uint32_t slot, vec3 o, vec3 d) const {
        q.ray_o[slot] = make_float4(o.x, o.y, o.z, 0.0f);
        q.ray_d[slot] = make_float4(d.x, d.y, d.z, 0.0f);
        __stcs(q.hit + slot, make_float2(0.0f, __int_as_float(EZRT_TRI_PENDING)));
        defer_list[atomicAdd(defer_count, 1u)] = slot;
    }
    __device__ __forceinline__ void defer(uint32_t i, vec3 o, vec3 d) const { defer_slot(slot_of(i), o, d); }
    __device__ __forceinline__ void store(uint32_t i, HitRec h, bool tie, vec3 o, vec3 d, vec3 inv) const {
        const uint32_t slot = slot_of(i);
        if (h.tri >= 0 && (tie || !reference_reaches_leaf_inv(acc_tri_leaf, leaf_box, h.tri, o, inv))) {
            defer_slot(slot, o, d);
            return;
        }
        __stcs(q.hit + slot, make_float2(h.t, __int_as_float(h.tri)));
    }
};

template <bool COUNT, bool IDX>
__global__ void __launch_bounds__(EZRT_EXTEND_MAX_THREADS, EZRT_EXTEND_LB_BLOCKS) k_extend_w8_camera(SceneDev sc, RenderDev rd, const TileDev* __restrict__ tiles,
                                                                   uint32_t batch_first_frame, uint32_t n_slots, uint32_t n_frames, PathQueue q, uint32_t* work,
                                                                   uint32_t* defer_list, uint32_t* defer_count, W8Counts counts) {
    unsigned char* s_perm;
    uint2* stack_sm;
    w8_smem_setup(s_perm, stack_sm);
    AccelCameraIO io;
    io.rd = rd;
    io.tiles = tiles;
    io.batch_first_frame = batch_first_frame;
    io.n_frames = n_frames;
    io.per_frame = (uint32_t)rd.n_tiles * EZRT_TILE_PIXELS;
    io.q = q;
    io.acc_tri_leaf = sc.acc_tri_leaf;
    io.leaf_box = sc.leaf_box;
    io.defer_list = defer_list;
    io.defer_count = defer_count;
    extend_w8_bundle<COUNT, IDX>(sc, n_slots, work, io, s_perm, stack_sm, counts);
}

template <bool COUNT, bool IDX>
__global__ void __launch_bounds__(EZRT_EXTEND_MAX_THREADS, EZRT_EXTEND_LB_BLOCKS) k_extend_w8(SceneDev sc, PathQueue q, const uint32_t* __restrict__ q_count, uint32_t* work,
                                                                   uint32_t* defer_list, uint32_t* defer_count, W8Counts counts, const uint32_t* __restrict__ perm,
                                                                   unsigned long long* phase_cycles) {
    unsigned char* s_perm;
    uint2* stack_sm;
    w8_smem_setup(s_perm, stack_sm);
    AccelExtendIO io;
    io.q = q;
    io.acc_tri_leaf = sc.acc_tri_leaf;
    io.leaf_box = sc.leaf_box;
    io.defer_list = defer_list;
    io.defer_count = defer_count;
    io.perm = perm;
    extend_w8<false, COUNT, IDX>(sc, *q_count, work, io, s_perm, stack_sm, counts, phase_cycles);
}

struct AccelShadowIO {
    ShadowIO base;
    const int* acc_tri_leaf;
    const float4* leaf_box;
    uint32_t* defer_list;
    uint32_t* defer_count;
    __device__ __forceinline__ bool load(uint32_t i, vec3& o, vec3& d) const { return base.load(i, o, d); }
    __device__ __forceinline__ float tmax(uint32_t i) const { return base.tmax(i); }
    __device__ __forceinline__ void defer(uint32_t i, vec3, vec3) const { defer_list[atomicAdd(defer_count, 1u)] = i; }
    __device__ __forceinline__ void store(uint32_t i, HitRec h, bool, vec3 o, vec3 d, vec3 inv) const {
        if (h.tri < 0) {  // nothing accepted anywhere: the shader finds nothing either
            base.mark(i, true);
            return;
        }
        // occluded if the shader reaches the occluder's leaf; otherwise the exact kernel decides
        if (!reference_reaches_leaf_inv(acc_tri_leaf, leaf_box, h.tri, o, inv)) defer(i, o, d);
        else base.mark(i, false);
    }
    __device__ __forceinline__ int leaf_of(int tri) const { return __ldg(acc_tri_leaf + tri); }
    __device__ __forceinline__ void finish(uint32_t i, HitRec h, bool, vec3 o, vec3 d, vec3 inv, int leaf) const {
        if (h.tri < 0) base.mark(i, true);
        else if (!reference_reaches_leaf_box(leaf_box, leaf, o, inv)) defer(i, o, d);
        else base.mark(i, false);
    }
};

template <bool COUNT, bool IDX, bool BOUNDED = false>
__global__ void __launch_bounds__(EZRT_EXTEND_MAX_THREADS, EZRT_EXTEND_LB_BLOCKS) k_shadow_w8(SceneDev sc, ShadowQueue sq, const uint32_t* __restrict__ s_count, uint32_t* work,
                                                                   float4* __restrict__ Lo, uint32_t* defer_list, uint32_t* defer_count, W8Counts counts,
                                                                   unsigned long long* phase_cycles) {
    unsigned char* s_perm;
    uint2* stack_sm;
    w8_smem_setup(s_perm, stack_sm);
    AccelShadowIO io;
    io.base.sq = sq;
    io.base.Lo = Lo;
    io.base.perm = nullptr;
    io.acc_tri_leaf = sc.acc_tri_leaf;
    io.leaf_box = sc.leaf_box;
    io.defer_list = defer_list;
    io.defer_count = defer_count;
    extend_w8<true, COUNT, IDX, BOUNDED>(sc, *s_count, work, io, s_perm, stack_sm, counts, phase_cycles);
}

// ---- the same three passes on the 4-wide exact-box tree (default form, env EZRT_ACCEL): extend_persistent<ACCEL, WIDE>
template <bool COUNT, bool Q16>
__global__ void __launch_bounds__(EZRT_EXTEND_MAX_THREADS, EZRT_EXTEND_LB_BLOCKS) k_extend_accel(SceneDev sc, PathQueue q, const uint32_t* __restrict__ q_count, uint32_t* work,
                                                                      uint32_t* defer_list, uint32_t* defer_count, W8Counts counts, const uint32_t* __restrict__ perm) {
    AccelExtendIO io;
    io.q = q;
    io.acc_tri_leaf = sc.acc_tri_leaf;
    io.leaf_box = sc.leaf_box;
    io.defer_list = defer_list;
    io.defer_count = defer_count;
    io.perm = perm;
    extend_persistent<true, false, true, true, 4, COUNT, Q16>(sc, accel_tree(sc), *q_count, work, io, g_smem_top, counts);
}
template <bool COUNT>
__global__ void __launch_bounds__(EZRT_EXTEND_MAX_THREADS, EZRT_EXTEND_LB_BLOCKS) k_extend_accel_camera(SceneDev sc, RenderDev rd, const TileDev* __restrict__ tiles,
                                                                      uint32_t batch_first_frame, uint32_t n_slots, uint32_t n_frames, PathQueue q, uint32_t* work,
                                                                      uint32_t* defer_list, uint32_t* defer_count, W8Counts counts) {
    AccelCameraIO io;
    io.rd = rd;
    io.tiles = tiles;
    io.batch_first_frame = batch_first_frame;
    io.n_frames = n_frames;
    io.per_frame = (uint32_t)rd.n_tiles * EZRT_TILE_PIXELS;
    io.q = q;
    io.acc_tri_leaf = sc.acc_tri_leaf;
    io.leaf_box = sc.leaf_box;
    io.defer_list = defer_list;
    io.defer_count = defer_count;
    extend_persistent<true, false, true, true, 4, COUNT, false>(sc, accel_tree(sc), n_slots, work, io, g_smem_top, counts, sc.refill_thresh_camera, sc.work_chunk_camera);
}
template <bool COUNT, bool Q16, bool BOUNDED = false>
__global__ void __launch_bounds__(EZRT_EXTEND_MAX_THREADS, EZRT_EXTEND_LB_BLOCKS) k_shadow_accel(SceneDev sc, ShadowQueue sq, const uint32_t* __restrict__ s_count, uint32_t* work,
                                                                      float4* __restrict__ Lo, uint32_t* defer_list, uint32_t* defer_count, W8Counts counts) {
    AccelShadowIO io;
    io.base.sq = sq;
    io.base.Lo = Lo;
    io.base.perm = nullptr;
    io.acc_tri_leaf = sc.acc_tri_leaf;
    io.leaf_box = sc.leaf_box;
    io.defer_list = defer_list;
    io.defer_count = defer_count;
    extend_persistent<true, true, true, true, 4, COUNT, Q16, BOUNDED>(sc, accel_tree(sc), *s_count, work, io, g_smem_top, counts);
}

// ------------------------------------------------------------------------------------------
#ifndef EZRT_SHADE_REGROUP
#define EZRT_SHADE_REGROUP 0      // k_shade, bounces > 0: 1 = each block shades its 128 paths in the order hits | misses (exchange through shared
                                  // memory after the loads); 0 = queue order.
#endif
#define EZRT_SOBOL_TABLE 256      // frames per batch whose Sobol pairs a k_shade block keeps in shared memory
#define EZRT_SHADE_KEYS 18        // material id mod 16, "left the scene", "beyond the queue end"
#ifndef EZRT_SHADE_PREFETCH
#define EZRT_SHADE_PREFETCH 0     // k_shade: prefetch (L2) the triangle records of the path this thread shades in its next round
#endif
#ifndef EZRT_SHADE_MIN_BLOCKS
#define EZRT_SHADE_MIN_BLOCKS 8   // 64 registers: k_shade is latency-bound, 32 resident warps beat 20 despite small spills
#endif
// LIST (the pass over the accel policy's deferred rays, on the side stream beside the main k_shade): entry k is queue entry /
// sample slot list[k], its hit is side_hit[k]; nothing to do when the list overflowed (then the in-line exact pass filled the
// queue's hit records and the main k_shade found no pending ones).
// AOV (feature-buffer renders): at bounce 0 every surface hit also writes its first-hit record, 32 bytes per sample slot:
// aov_rec[2 slot] = (albedo, t), aov_rec[2 slot + 1] = (shading normal, 0).  A primary miss writes nothing (k_blend knows
// it from Lo.w == 1).  The plain instantiations never touch aov_rec.
// ENV (light sampling mode with EZRT_PARAM_ENV_LIGHT): the map is one more light, sampled from the table env (shade_step).
// TRANS (light sampling mode with EZRT_PARAM_TRANSMISSION): materials with a dielectric lobe (shade_step).
// MEDIUM (light sampling mode with EZRT_PARAM_MEDIUM): the homogeneous medium med (shade_step, medium_step).
// TEX (light sampling mode with EZRT_PARAM_TEXTURES): the base-colour textures tex (shade_step); every shadow slot also gets its
// shading point's textured base colour, tex.sh_base[spos].
// MAPS (with TEX; EZRT_PARAM_MATERIAL_MAPS): the material maps (shade_step); the slot also gets the mapped roughness in
// tex.sh_base[spos].w and the mapped metallic in maps.sh_metal[spos].
template <int MODE, bool LIST, bool AOV = false, bool ENV = false, bool TRANS = false, bool MEDIUM = false, bool TEX = false,
          bool MAPS = false>
__global__ void __launch_bounds__(128, EZRT_SHADE_MIN_BLOCKS) k_shade(SceneDev sc, RenderDev rd, const TileDev* __restrict__ tiles, int bounce,
                                               uint32_t batch_first_frame, PathQueue qin, const uint32_t* __restrict__ in_count,
                                               PathQueue qout, uint32_t* out_count, ShadowQueue sq, uint32_t* s_count,
                                               float4* __restrict__ Lo, float4* __restrict__ Le, uint32_t n_fused, uint32_t n_frames,
                                               const uint32_t* __restrict__ list, const float2* __restrict__ side_hit,
                                               float4* __restrict__ aov_rec, LightsDev lights, EnvDev env, MediumDev med, TexDev tex,
                                               MapsDev maps) {
    // The Sobol pair of (bounce, frame) is the same for every pixel of a frame (P5/fsh:361-376: up to 2 x 32 table XORs per path): each
    // block computes the pairs of the batch's frames once into shared memory (batches of more than EZRT_SOBOL_TABLE frames compute per path).
    __shared__ float2 s_sobol[EZRT_SOBOL_TABLE];
    const bool sobol_table = (MODE == EZRT_MODE_DISNEY_SOBOL_P5 || MODE == EZRT_MODE_DISNEY_IS_MIS_P5 || MODE == EZRT_MODE_DISNEY_LIGHTS) &&
                             n_frames <= EZRT_SOBOL_TABLE;
    if (sobol_table) {
        for (uint32_t f = threadIdx.x; f < n_frames; f += blockDim.x) s_sobol[f] = sobol_pair(bounce, batch_first_frame + f);
        __syncthreads();
    }
    // n_fused != 0 (bounce 0 of the W8 policy): entry i is sample slot i, its camera ray was generated inside
    // k_extend_w8_camera and is generated again here instead of being read from a queue; only q.hit[i] is read
    __shared__ uint32_t s_scan[34];
    const uint32_t n = (LIST || !n_fused) ? *in_count : n_fused;   // LIST: in_count = length of the list
    if (LIST && n > EZRT_SIDE_CAP) return;
    const uint32_t n_round = ((n + blockDim.x - 1u) / blockDim.x) * blockDim.x;
    const uint32_t stride = gridDim.x * blockDim.x;
#if EZRT_SHADE_REGROUP
    // Regrouping between bounces (north_star: "compact active rays and sort by material-id"), second version: every thread loads ITS queue
    // entry (all loads in flight at once, coalesced), the 128 entries of the block are then exchanged through shared memory into the order
    // surface hits | paths that left the scene | nothing to do, and thread t shades the t-th entry of that order: warps run one branch of the
    // integrator instead of both.  (First version: the block sorted on the hit record BEFORE loading the rest,
    // which serialised two memory latencies per path and lost 5 %.)  The result does not depend on the order.
    __shared__ float4 s_rg[4][128];
    __shared__ float2 s_rg_hit[128];
    __shared__ unsigned short s_rg_cnt[4][2];
#endif
    for (uint32_t i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < n_round; i0 += stride) {
        uint32_t i = i0;
#if EZRT_SHADE_PREFETCH
        int next_tri = -1;
        if (!LIST && i0 + stride < n) next_tri = __float_as_int(__ldcs(qin.hit + i0 + stride).y);
#endif
        bool alive = false;
        PathRegs p;
        ShadowRay sh;
        sh.valid = false;
        vec3 sh_base;   // TEX: the shading point's textured base colour
        float2 sh_rm;   // MAPS: its mapped roughness and metallic
        uint32_t slot = 0;
        uint32_t px = 0, py = 0, fib = 0;
        bool present = i < n;
        float2 hit = make_float2(0.0f, 0.0f);
        float4 o4 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), d4 = o4, h4 = o4, f4 = o4;
        bool staged = false;
#if EZRT_SHADE_REGROUP
        if (!LIST && bounce > 0) {   // camera paths are coherent as they are
            staged = true;
            hit = make_float2(0.0f, __int_as_float(EZRT_TRI_PENDING));
            if (present) {
                hit = __ldcs(qin.hit + i);
                o4 = __ldcs(qin.ray_o + i); d4 = __ldcs(qin.ray_d + i); h4 = __ldcs(qin.hist + i); f4 = __ldcs(qin.fr + i);
            }
            const int tri0 = __float_as_int(hit.y);
            const int key = (tri0 == EZRT_TRI_PENDING) ? 2 : (tri0 >= 0 ? 0 : 1);
            const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
            const unsigned lt = (1u << lane) - 1u;
            const unsigned m0 = __ballot_sync(0xffffffffu, key == 0), m1 = __ballot_sync(0xffffffffu, key == 1);
            if (lane == 0) { s_rg_cnt[wid][0] = (unsigned short)__popc(m0); s_rg_cnt[wid][1] = (unsigned short)__popc(m1); }
            __syncthreads();
            uint32_t n0 = 0, n1 = 0, b0 = 0, b1 = 0;
#pragma unroll
            for (int w = 0; w < 4; w++) {
                const uint32_t c0 = s_rg_cnt[w][0], c1 = s_rg_cnt[w][1];
                n0 += c0; n1 += c1;
                if (w < wid) { b0 += c0; b1 += c1; }
            }
            uint32_t dest;
            if (key == 0) dest = b0 + (uint32_t)__popc(m0 & lt);
            else if (key == 1) dest = n0 + b1 + (uint32_t)__popc(m1 & lt);
            else dest = n0 + n1 + ((uint32_t)wid * 32u - b0 - b1) + (uint32_t)__popc(~(m0 | m1) & lt);
            s_rg_hit[dest] = hit;
            s_rg[0][dest] = o4; s_rg[1][dest] = d4; s_rg[2][dest] = h4; s_rg[3][dest] = f4;
            __syncthreads();
            hit = s_rg_hit[threadIdx.x];
            o4 = s_rg[0][threadIdx.x]; d4 = s_rg[1][threadIdx.x]; h4 = s_rg[2][threadIdx.x]; f4 = s_rg[3][threadIdx.x];
            present = threadIdx.x < n0 + n1;   // the block_append barriers below separate these reads from the next round's writes
        }
#endif
        if (LIST && present) { hit = side_hit[i]; i = list[i]; }
        if (present && n_fused) present = slot_pixel(rd, tiles, i, px, py, fib);   // slots of clipped tiles outside the image
        if (present) {
            if (!LIST && !staged) hit = __ldcs(qin.hit + i);   // the other loads below do not wait for it
            if (n_fused) {
                slot = i;
                primary_ray(rd, px, py, batch_first_frame + fib, p.seed, p.o, p.d);
            } else {
                if (!staged) { o4 = __ldcs(qin.ray_o + i); d4 = __ldcs(qin.ray_d + i); }   // .w: rng seed / sample slot
                slot = __float_as_uint(d4.w);
                p.o = ez_v3(o4.x, o4.y, o4.z);
                p.d = ez_v3(d4.x, d4.y, d4.z);
                p.seed = __float_as_uint(o4.w);
                slot_pixel(rd, tiles, slot, px, py, fib);
            }
            vec3 lo = splat3(0.0f), le = splat3(0.0f);
            bool pmiss = false;
            float lo_w = 0.0f;   // Lo.w: 0 = Le absent (zero), 1 = the primary ray left the scene, 2 = Le[slot] holds the first hit's emission
            if (bounce > 0) {
                if (!staged) { h4 = __ldcs(qin.hist + i); f4 = __ldcs(qin.fr + i); }
                p.history = ez_v3(h4.x, h4.y, h4.z);
                p.cosine_i = h4.w;
                p.f_r = ez_v3(f4.x, f4.y, f4.z);
                p.pdf = f4.w;
                float4 l4 = Lo[slot];
                lo = ez_v3(l4.x, l4.y, l4.z);
                lo_w = l4.w;
            } else {
                p.history = splat3(1.0f);
                p.f_r = splat3(0.0f);
                p.cosine_i = 0.0f;
                p.pdf = 1.0f;
            }
            const float2 sob = sobol_table ? s_sobol[fib] : sobol_pair(bounce, batch_first_frame + fib);
#if EZRT_SHADE_PREFETCH
            // the geometry and shading records of the triangle this thread's NEXT path hit (its hit record was requested at the top of
            // this round): into L2 while this path is shaded -- the two random 48-byte gathers of surface_hit miss L2 three times in four
            if (!LIST && next_tri >= 0) {
                const float4* g = tri_geo_rec(sc, next_tri, rd.accel_space != 0);   // an indexed record's vertices are not prefetched
                const float4* sr = (rd.accel_space ? sc.acc_tri_shade : sc.tri_shade) + (size_t)next_tri * 3;
                asm volatile("prefetch.global.L2 [%0];" ::"l"(g));
                if (!(rd.accel_space && sc.acc_tri_indexed)) asm volatile("prefetch.global.L2 [%0];" ::"l"(g + 2));
                asm volatile("prefetch.global.L2 [%0];" ::"l"(sr));
                asm volatile("prefetch.global.L2 [%0];" ::"l"(sr + 2));
            }
#endif
            if (LIST || __float_as_int(hit.y) != EZRT_TRI_PENDING) {   // pending: deferred by the accel kernel, shaded by the LIST pass
                alive = shade_step<MODE, MODE == EZRT_MODE_DISNEY_IS_MIS_P5, AOV, ENV, TRANS, MEDIUM, TEX, MAPS>(sc, rd, bounce, p, hit.x, __float_as_int(hit.y), px, py,
                                                                                                          sob, lo, le, pmiss, sh, AOV ? aov_rec + 2 * (size_t)slot : nullptr,
                                                                                                          lights, env, med, tex, &sh_base, &sh_rm, maps);
                if (bounce == 0) {
                    // Le is zero for every surface that does not emit: it is stored (and read back by k_blend) only otherwise.
                    // color = Le + Lo with Le = +-0 is Lo bit for bit, because Lo is never -0.0 (it starts at +0.0 and only grows by additions)
                    lo_w = pmiss ? 1.0f : 0.0f;
                    if (le.x != 0.0f || le.y != 0.0f || le.z != 0.0f) {
                        Le[slot] = make_float4(le.x, le.y, le.z, 0.0f);
                        lo_w = 2.0f;
                    }
                }
                Lo[slot] = make_float4(lo.x, lo.y, lo.z, lo_w);
            }
        }
        uint32_t pos = block_append(alive, out_count, s_scan);
        if (alive) {
            __stcs(qout.ray_o + pos, make_float4(p.o.x, p.o.y, p.o.z, __uint_as_float(p.seed)));
            __stcs(qout.ray_d + pos, make_float4(p.d.x, p.d.y, p.d.z, __uint_as_float(slot)));
            __stcs(qout.hist + pos, make_float4(p.history.x, p.history.y, p.history.z, p.cosine_i));
            __stcs(qout.fr + pos, make_float4(p.f_r.x, p.f_r.y, p.f_r.z, p.pdf));
        }
        if (MODE == EZRT_MODE_DISNEY_IS_MIS_P5 || MODE == EZRT_MODE_DISNEY_LIGHTS) {
            constexpr bool LT = (MODE == EZRT_MODE_DISNEY_LIGHTS);   // light samples: tmax, pdf and the light's material in the .w words
            uint32_t spos = block_append(sh.valid, s_count, s_scan);
            if (sh.valid) {
                __stcs(sq.ray_o + spos, make_float4(sh.o.x, sh.o.y, sh.o.z, __uint_as_float(slot)));
                __stcs(sq.ray_d + spos, make_float4(sh.d.x, sh.d.y, sh.d.z, __int_as_float(sh.matId)));
                __stcs(sq.nrm + spos, make_float4(sh.N.x, sh.N.y, sh.N.z, LT ? sh.tmax : 0.0f));
                __stcs(sq.view + spos, make_float4(sh.V.x, sh.V.y, sh.V.z, LT ? sh.pdf : 0.0f));
                __stcs(sq.hist + spos, make_float4(sh.history.x, sh.history.y, sh.history.z, LT ? __int_as_float(sh.light_mat) : 0.0f));
                if constexpr (TEX) {   // a medium vertex's slot has no shading point: its entry is never read
                    if (sh.matId != EZRT_MEDIUM_VERTEX || !MEDIUM) {
                        __stcs(tex.sh_base + spos, make_float4(sh_base.x, sh_base.y, sh_base.z, MAPS ? sh_rm.x : 0.0f));
                        if constexpr (MAPS) __stcs(maps.sh_metal + spos, sh_rm.y);
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// k_nee: the light samples whose shadow ray got through (sq.lit) add their contribution to Lo -- the BRDF value and pdf of the
// light direction, the environment colour and pdf and the MIS weight (nee_contrib, P5/fsh:829-841) are evaluated here, after
// the shadow pass, instead of for every light sample in k_shade.  Each block compacts the lit rays of 512 queue entries in
// shared memory so that full warps evaluate.  One shadow ray per sample slot and bounce: no two threads touch one Lo entry.
// ------------------------------------------------------------------------------------------
// MODE = EZRT_MODE_DISNEY_LIGHTS: the light samples on the emissive triangles (nee_light_contrib; view.w = pdf, hist.w = the light's material);
// ENV: and on the environment map (hist.w = -1: the light's colour is the map's in the sample's direction).
// TRANS: evaluated with the mixture of the shading point's material (nee_trans_contrib); ray_d.w = ~matId for a hit from inside.
// MEDIUM: every contribution times the shadow ray's transmittance through the medium med; a medium vertex's (ray_d.w =
// EZRT_MEDIUM_VERTEX, view = d) is evaluated with the phase function (nee_medium_contrib).
// TEX: the shading point's material with the textured base colour k_shade left in tex.sh_base[j].
// MAPS: ... and the mapped roughness and metallic, tex.sh_base[j].w and maps.sh_metal[j]; the slot's N is already the mapped normal.
template <int MODE, bool ENV = false, bool TRANS = false, bool MEDIUM = false, bool TEX = false, bool MAPS = false>
__global__ void __launch_bounds__(128, 8) k_nee(SceneDev sc, RenderDev rd, ShadowQueue sq, const uint32_t* __restrict__ s_count, float4* __restrict__ Lo,
                                                MediumDev med, TexDev tex, MapsDev maps) {
    static_assert(MODE == EZRT_MODE_DISNEY_LIGHTS || !(ENV || TRANS || MEDIUM), "the options exist in the light sampling mode");
    static_assert(!(TRANS && MEDIUM), "the medium is rendered without transmission");
    __shared__ uint32_t s_scan[34];
    __shared__ uint32_t s_total;
    __shared__ uint32_t s_list[512];
    const uint32_t n = *s_count;
    for (uint32_t base = blockIdx.x * 512u; base < n; base += gridDim.x * 512u) {
        if (threadIdx.x == 0) s_total = 0u;
        __syncthreads();
#pragma unroll 1
        for (int k = 0; k < 4; k++) {
            const uint32_t j = base + (uint32_t)k * 128u + threadIdx.x;
            const bool lit = j < n && sq.lit[j] != 0;
            const uint32_t pos = block_append(lit, &s_total, s_scan);
            if (lit) s_list[pos] = j;
        }
        __syncthreads();
        const uint32_t total = s_total;
        for (uint32_t q = threadIdx.x; q < total; q += blockDim.x) {
            const uint32_t j = s_list[q];
            const float4 o4 = __ldcs(sq.ray_o + j), d4 = __ldcs(sq.ray_d + j), n4 = __ldcs(sq.nrm + j), v4 = __ldcs(sq.view + j), h4 = __ldcs(sq.hist + j);
            const uint32_t slot = __float_as_uint(o4.w);
            const int m_raw = __float_as_int(d4.w);
            const auto material = [&](int m_id) {
                MaterialDev m = load_material(sc, m_id);
                if constexpr (MAPS) {
                    const float4 b = __ldcs(tex.sh_base + j);
                    m.baseColor = f4xyz(b);
                    m.roughness = b.w;
                    m.metallic = __ldcs(maps.sh_metal + j);
                } else if constexpr (TEX) {
                    m.baseColor = f4xyz(__ldcs(tex.sh_base + j));
                }
                return m;
            };
            const vec3 V = ez_v3(v4.x, v4.y, v4.z), N = ez_v3(n4.x, n4.y, n4.z), Ld = ez_v3(d4.x, d4.y, d4.z), hist = ez_v3(h4.x, h4.y, h4.z);
            vec3 c;
            if constexpr (MODE == EZRT_MODE_DISNEY_LIGHTS) {
                const int lm = __float_as_int(h4.w);   // the light's material; -1: an environment sample
                const auto light_color = [&] { return (ENV && lm < 0) ? hdr_color(sc, rd, Ld, EZRT_MODE_DISNEY_LIGHTS) : load_emissive(sc, lm); };
                if constexpr (MEDIUM) {   // a medium vertex loads no material
                    const vec3 E = light_color();
                    if (m_raw == EZRT_MEDIUM_VERTEX) c = nee_medium_contrib(V, Ld, med.g, hist, E, v4.w);
                    else c = nee_light_contrib(V, N, Ld, material(m_raw), hist, E, v4.w);
                    c = ez_scale(c, ez_medium_transmittance(&med, ez_v3(o4.x, o4.y, o4.z), Ld, ez_medium_light_dist(n4.w, ENV && lm < 0)));
                } else {
                    const int m_id = (TRANS && m_raw < 0) ? ~m_raw : m_raw;
                    const MaterialDev mat = material(m_id);
                    if constexpr (TRANS) c = nee_trans_contrib(sc, V, N, Ld, m_id, mat, m_raw < 0, hist, light_color(), v4.w);
                    else c = nee_light_contrib(V, N, Ld, mat, hist, light_color(), v4.w);
                }
            } else {
                c = nee_contrib(sc, rd, EZRT_MODE_DISNEY_IS_MIS_P5, V, N, Ld, load_material(sc, m_raw), hist);
            }
            float4 lo = Lo[slot];
            lo.x += c.x; lo.y += c.y; lo.z += c.z;
            Lo[slot] = lo;
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------
// blend: color = Le + Li (or the sky for a primary miss), running mean in frame order
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ size_t fb_index(const RenderDev& rd, const TileDev& t, int ix, int iy) {
    if (rd.compact_out) return (size_t)t.pixel_offset + (size_t)iy * t.w + ix;
    return (size_t)(t.y0 + iy) * rd.width + (t.x0 + ix);
}

// ADAPTIVE: also the running mean of the squared sample luminance (luma2) and the frames the pixel received (spp_map), both
// indexed like the framebuffer's pixels (ezrt_math.h, "adaptive sampling").  The plain instantiation never touches them.
// AOV (with ADAPTIVE; no spp map): also the running means of the first-hit features, 8 floats per pixel (albedo, coverage,
// normal, depth; 0 for a primary miss) from the records k_shade<.., AOV> left in aov_rec, blended with the colour's weights.
template <bool ADAPTIVE, bool AOV = false>
__global__ void __launch_bounds__(256) k_blend(RenderDev rd, const TileDev* __restrict__ tiles, int nf, uint32_t batch_first_frame,
                                               const float4* __restrict__ Lo, const float4* __restrict__ Le, float* __restrict__ fb,
                                               float* __restrict__ luma2, int32_t* __restrict__ spp_map,
                                               const float4* __restrict__ aov_rec, float* __restrict__ aov) {
    uint32_t per_frame = (uint32_t)rd.n_tiles * EZRT_TILE_PIXELS;
    uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= per_frame) return;
    TileDev t = tiles[r >> 8];
    int ix, iy;
    in_tile_xy((int)(r & 255u), ix, iy);
    if (ix >= t.w || iy >= t.h) return;
    const size_t pix = fb_index(rd, t, ix, iy);
    size_t idx = pix * (size_t)rd.out_channels;
    // only the first batch of a render from frame 0 starts from nothing: a later batch that starts at frame 0 because the
    // uint32 frame counter wrapped blends onto the frames before it, as every display() call does
    const bool fresh = (batch_first_frame == 0u) && (rd.first_frame == 0u);
    vec3 acc = fresh ? splat3(0.0f) : ez_v3(fb[idx], fb[idx + 1], fb[idx + 2]);
    float m2 = 0.0f;
    if (ADAPTIVE && !fresh) m2 = luma2[pix];
    float feat[8];
    if (AOV) {
#pragma unroll
        for (int k = 0; k < 8; k++) feat[k] = fresh ? 0.0f : aov[pix * 8 + k];
    }
    for (int f = 0; f < nf; f++) {
        float4 lo = Lo[(size_t)f * per_frame + r];
        vec3 color = ez_v3(lo.x, lo.y, lo.z);   // primary miss: the sky; no emission at the first hit: 0 + Lo = Lo
        if (lo.w == 2.0f) {
            float4 le = Le[(size_t)f * per_frame + r];
            color = ez_add(ez_v3(le.x, le.y, le.z), color);
        }
        float a = EZ_DIV(1.0f, __uint2float_rn(batch_first_frame + (uint32_t)f + 1u));
        acc = ez_vmix(acc, color, a);
        if (ADAPTIVE) {
            const float y = ez_luminance(color);
            m2 = ez_mix(m2, y * y, a);
        }
        if (AOV) {
            float4 r0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), r1 = r0;
            float cov = 0.0f;
            if (lo.w != 1.0f) {   // Lo.w == 1: the primary ray left the scene
                const size_t s = (size_t)f * per_frame + r;
                r0 = aov_rec[2 * s];
                r1 = aov_rec[2 * s + 1];
                cov = 1.0f;
            }
            const float v[8] = {r0.x, r0.y, r0.z, cov, r1.x, r1.y, r1.z, r0.w};
#pragma unroll
            for (int k = 0; k < 8; k++) feat[k] = ez_mix(feat[k], v[k], a);
        }
    }
    fb[idx] = acc.x; fb[idx + 1] = acc.y; fb[idx + 2] = acc.z;
    if (rd.out_channels == 4) fb[idx + 3] = 1.0f;
    if (ADAPTIVE) luma2[pix] = m2;
    if (ADAPTIVE && !AOV) spp_map[pix] = (int32_t)(batch_first_frame + (uint32_t)nf);
    if (AOV) {
        float4* o = (float4*)(aov + pix * 8);
        o[0] = make_float4(feat[0], feat[1], feat[2], feat[3]);
        o[1] = make_float4(feat[4], feat[5], feat[6], feat[7]);
    }
}

// The convergence test of adaptive sampling: one block per active tile, one thread per pixel.  A tile survives unless every
// in-image pixel has err <= threshold (ez_adaptive_error; a NaN survives).  Each block leaves its verdict in keep[]; the last
// block to finish compacts the surviving tiles, in their input order, into tiles_out and writes (tiles, pixels) to counts.
// The input order is kept so that the tile order and the launch shapes of the next batches do not depend on block timing.
__global__ void __launch_bounds__(256) k_adaptive_check(RenderDev rd, const TileDev* __restrict__ tiles_in, int n_frames, float threshold,
                                                        const float* __restrict__ fb, const float* __restrict__ luma2,
                                                        unsigned char* __restrict__ keep, unsigned int* __restrict__ blocks_done,
                                                        TileDev* __restrict__ tiles_out, int32_t* __restrict__ counts) {
    __shared__ uint32_t s_scan[34];
    __shared__ uint32_t s_tiles, s_pixels;
    __shared__ bool s_last;
    const TileDev t = tiles_in[blockIdx.x];
    int ix, iy;
    in_tile_xy((int)threadIdx.x, ix, iy);
    bool ok = true;
    if (ix < t.w && iy < t.h) {
        const size_t pix = fb_index(rd, t, ix, iy);
        const size_t idx = pix * (size_t)rd.out_channels;
        const float err = ez_adaptive_error(luma2[pix], ez_v3(fb[idx], fb[idx + 1], fb[idx + 2]), n_frames);
        ok = (err <= threshold);
    }
    const bool converged = __syncthreads_and(ok) != 0;
    if (threadIdx.x == 0) {
        keep[blockIdx.x] = converged ? 0 : 1;
        __threadfence();
        s_last = (atomicAdd(blocks_done, 1u) == gridDim.x - 1);
    }
    __syncthreads();
    if (!s_last) return;
    // last block: order-preserving compaction of the surviving tiles.  block_append on a shared-memory counter ranks the
    // survivors of each chunk of 256 by thread index and the chunks run in order, so tiles_out keeps the order of tiles_in.
    __threadfence();
    if (threadIdx.x == 0) { s_tiles = 0u; s_pixels = 0u; }
    __syncthreads();
    for (uint32_t i0 = 0; i0 < gridDim.x; i0 += blockDim.x) {
        const uint32_t i = i0 + threadIdx.x;
        const bool k = (i < gridDim.x) && ((volatile const unsigned char*)keep)[i] != 0;
        const uint32_t pos = block_append(k, &s_tiles, s_scan);
        if (k) {
            const TileDev ti = tiles_in[i];
            tiles_out[pos] = ti;
            atomicAdd(&s_pixels, (uint32_t)(ti.w * ti.h));
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        counts[0] = (int32_t)s_tiles;
        counts[1] = (int32_t)s_pixels;
        *blocks_done = 0u;   // ready for the next test
    }
}

// totals[0..2] += primary, bounce, shadow rays of this batch; totals[3] += samples; totals[4] += deferred rays
__global__ void k_tally(const uint32_t* __restrict__ q_counts, const uint32_t* __restrict__ s_counts, const uint32_t* __restrict__ d_ext,
                        const uint32_t* __restrict__ d_sh, int n_stages, unsigned long long* totals, uint32_t n_primary) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    unsigned long long bounce = 0, shadow = 0, deferred = 0;
    for (int b = 1; b < n_stages; b++) bounce += q_counts[b];
    for (int b = 0; b < n_stages; b++) { shadow += s_counts[b]; deferred += d_ext[b] + d_sh[b]; }
    const unsigned long long primary = n_primary ? n_primary : q_counts[0];  // fused camera pass: no queue 0, the host knows the count
    totals[0] += primary;
    totals[1] += bounce;
    totals[2] += shadow;
    totals[3] += primary;
    totals[4] += deferred;
}

// ------------------------------------------------------------------------------------------
// megakernel: one thread = one pixel, all frames and bounces in registers (cross-check pipeline)
// ------------------------------------------------------------------------------------------
// LENS (EZRT_PARAM_THIN_LENS): the camera rays are the thin lens's
template <bool PRUNE, bool LENS>
__global__ void __launch_bounds__(128) k_megakernel(SceneDev sc, RenderDev rd, const TileDev* __restrict__ tiles, int spp,
                                                    float* __restrict__ fb, unsigned long long* totals, LensDev lens) {
    uint32_t per_frame = (uint32_t)rd.n_tiles * EZRT_TILE_PIXELS;
    uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= per_frame) return;
    TileDev t = tiles[r >> 8];
    int ix, iy;
    in_tile_xy((int)(r & 255u), ix, iy);
    if (ix >= t.w || iy >= t.h) return;
    uint32_t px = (uint32_t)(t.x0 + ix), py = (uint32_t)(t.y0 + iy);
    size_t idx = fb_index(rd, t, ix, iy) * (size_t)rd.out_channels;
    vec3 acc = (rd.first_frame == 0u) ? splat3(0.0f) : ez_v3(fb[idx], fb[idx + 1], fb[idx + 2]);
    unsigned long long n_primary = 0, n_bounce = 0, n_shadow = 0;
    for (int s = 0; s < spp; s++) {
        uint32_t frame = rd.first_frame + (uint32_t)s;
        PathRegs p;
        camera_ray<LENS>(rd, lens, px, py, frame, p.seed, p.o, p.d);
        p.history = splat3(1.0f);
        p.f_r = splat3(0.0f);
        p.cosine_i = 0.0f;
        p.pdf = 1.0f;
        vec3 lo = splat3(0.0f), le = splat3(0.0f);
        bool pmiss = false;
        for (int bounce = 0;; bounce++) {
            HitRec h = trace_ray<PRUNE, false>(sc, p.o, p.d);
            if (bounce == 0) n_primary++; else n_bounce++;
            ShadowRay sh;
            bool alive = shade_step<-1>(sc, rd, bounce, p, h.t, h.tri, px, py, sobol_pair(bounce, frame), lo, le, pmiss, sh);
            if (sh.valid) {
                HitRec hs = trace_ray<PRUNE, true>(sc, sh.o, sh.d);
                n_shadow++;
                if (hs.tri < 0) lo = ez_add(lo, sh.contrib);
            }
            if (!alive) break;
        }
        vec3 color = pmiss ? lo : ez_add(le, lo);
        float a = EZ_DIV(1.0f, __uint2float_rn(frame + 1u));
        acc = ez_vmix(acc, color, a);
    }
    fb[idx] = acc.x; fb[idx + 1] = acc.y; fb[idx + 2] = acc.z;
    if (rd.out_channels == 4) fb[idx + 3] = 1.0f;
    atomicAdd(&totals[0], n_primary);
    atomicAdd(&totals[1], n_bounce);
    atomicAdd(&totals[2], n_shadow);
    atomicAdd(&totals[3], n_primary);
}

// ------------------------------------------------------------------------------------------
// single-function entry points (parity tests)
// ------------------------------------------------------------------------------------------
// results of a traced ray queue -> the outputs of ezrt_trace_rays (tail of hitTriangle for the final hit)
__global__ void k_trace_finish(SceneDev sc, int n, PathQueue q, int p3fudge, int accel_space, int* hit, float* dist, int* tri, int* inside,
                               float* point, float* normal) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float4 o4 = q.ray_o[i], d4 = q.ray_d[i];
    const float2 h = q.hit[i];
    vec3 ro = ez_v3(o4.x, o4.y, o4.z), rdv = ez_v3(d4.x, d4.y, d4.z);
    const int ht = __float_as_int(h.y);  // triangle index in the policy's index space
    hit[i] = ht >= 0;
    dist[i] = h.x;
    tri[i] = (ht >= 0 && accel_space) ? (int)sc.acc_tri_ref[ht] : ht;
    vec3 P = splat3(0.0f), N = splat3(0.0f);
    int ins = 0;
    if (ht >= 0) {
        SurfaceHit s = surface_hit(sc, ro, rdv, h.x, ht, p3fudge != 0, accel_space != 0);
        P = s.P;
        N = s.N;
        vec3 Ng = f4xyz(ldg4(tri_geo_rec(sc, ht, accel_space != 0)));
        ins = ez_dot(Ng, rdv) > 0.0f;
    }
    inside[i] = ins;
    point[3 * i] = P.x; point[3 * i + 1] = P.y; point[3 * i + 2] = P.z;
    normal[3 * i] = N.x; normal[3 * i + 1] = N.y; normal[3 * i + 2] = N.z;
}

__device__ __forceinline__ MaterialDev material_from18(const float* m) {
    MaterialDev r;
    r.emissive = ez_v3(m[0], m[1], m[2]);
    r.baseColor = ez_v3(m[3], m[4], m[5]);
    r.subsurface = m[6]; r.metallic = m[7]; r.specular = m[8]; r.specularTint = m[9];
    r.roughness = m[10]; r.anisotropic = m[11]; r.sheen = m[12]; r.sheenTint = m[13];
    r.clearcoat = m[14]; r.clearcoatGloss = m[15];
    return r;
}

__global__ void k_eval_brdf(int which, int n, const float* V, const float* N, const float* L, const float* xi,
                            const float* materials, float* out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    vec3 v = ez_v3(V[3 * i], V[3 * i + 1], V[3 * i + 2]);
    vec3 nn = ez_v3(N[3 * i], N[3 * i + 1], N[3 * i + 2]);
    vec3 l = L ? ez_v3(L[3 * i], L[3 * i + 1], L[3 * i + 2]) : splat3(0.0f);
    MaterialDev m = material_from18(materials + (size_t)i * 18);
    vec3 r = splat3(0.0f);
    if (which == 0) r = brdf_evaluate<false>(v, nn, l, m);
    else if (which == 1) r = brdf_evaluate<true>(v, nn, l, m);
    else if (which == 2) r.x = brdf_pdf(v, nn, l, m);
    else if (which == 3) r = sample_brdf(xi[3 * i], xi[3 * i + 1], xi[3 * i + 2], v, nn, m);
    out[3 * i] = r.x; out[3 * i + 1] = r.y; out[3 * i + 2] = r.z;
}

// ezrt_eval_bsdf: the transmission mixture (ezrt_math.h, DESIGN.md section 12), 8 floats out per tuple:
// which 0: f (3), 1: pdf (1), 2: the sample of xi[4 i .. 4 i + 3] = (xi_1, xi_2, xi_3, r_t): L (3), f (3), pdf, signed cosine (0: the path ends)
__global__ void k_eval_bsdf(int which, int n, const float* V, const float* N, const float* L, const float* xi, const int* inside,
                            const float* materials, float* out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const vec3 v = ez_v3(V[3 * i], V[3 * i + 1], V[3 * i + 2]);
    const vec3 nn = ez_v3(N[3 * i], N[3 * i + 1], N[3 * i + 2]);
    const float* m18 = materials + (size_t)i * 18;
    const MaterialDev m = material_from18(m18);
    TransLobe tl;
    tl.t = ez_trans_weight(m18[17], m.metallic, m18[16]);
    tl.eta = ez_trans_eta(m18[16], inside[i]);
    tl.alpha = ez_max(0.001f, ez_sqr(m.roughness));
    tl.matched = ez_trans_matched(m18[16]) != 0;
    float r[8] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    if (which == 0 || which == 1) {
        float pdf;
        const vec3 f = bsdf_evaluate(v, nn, ez_v3(L[3 * i], L[3 * i + 1], L[3 * i + 2]), m, tl, pdf);
        if (which == 0) { r[0] = f.x; r[1] = f.y; r[2] = f.z; }
        else r[0] = pdf;
    } else {
        vec3 l = sample_brdf(xi[4 * i], xi[4 * i + 1], xi[4 * i + 2], v, nn, m), f = splat3(0.0f);
        float pdf = 0.0f, cosine = 0.0f;
        if (bsdf_sample(xi[4 * i], xi[4 * i + 1], xi[4 * i + 2], xi[4 * i + 3], v, nn, m, tl, l, f, pdf, cosine)) {
            r[0] = l.x; r[1] = l.y; r[2] = l.z; r[3] = f.x; r[4] = f.y; r[5] = f.z; r[6] = pdf; r[7] = cosine;
        }
    }
    for (int k = 0; k < 8; k++) out[8 * (size_t)i + k] = r[k];
}

// ezrt_camera_rays: the camera ray of sample (px[i], py[i], frame[i]), pinhole or thin lens (lens_on)
__global__ void k_camera_rays(RenderDev rd, int lens_on, int n, const uint32_t* px, const uint32_t* py, const uint32_t* frame, float* o_out,
                              float* d_out, LensDev lens) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t seed;
    vec3 o, d;
    if (lens_on) camera_ray<true>(rd, lens, px[i], py[i], frame[i], seed, o, d);
    else camera_ray<false>(rd, lens, px[i], py[i], frame[i], seed, o, d);
    const size_t k = 3 * (size_t)i;
    o_out[k] = o.x; o_out[k + 1] = o.y; o_out[k + 2] = o.z;
    d_out[k] = d.x; d_out[k + 1] = d.y; d_out[k + 2] = d.z;
}

__global__ void k_eval_math(int which, int n, const float* a, const float* b, float* out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float x = a[i], y = b ? b[i] : 0.0f, r = 0.0f;
    switch (which) {
        case 0: r = ez_sin(x); break;
        case 1: r = ez_cos(x); break;
        case 2: r = ez_log(x); break;
        case 3: r = ez_exp(x); break;
        case 4: r = ez_pow(x, y); break;
        case 5: r = ez_atan2(x, y); break;
        case 6: r = ez_asin(x); break;
        case 7: r = ez_floor(x); break;
    }
    out[i] = r;
}

// pass3: tone map + gamma (P5/shaders/pass3.fsh:14-25)
__global__ void __launch_bounds__(256) k_tonemap(const float* __restrict__ in, int channels, float* __restrict__ out, long long n, float limit) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    vec3 c = ez_v3(in[i * channels], in[i * channels + 1], in[i * channels + 2]);
    c = ez_tonemap_pass3(c, limit);
    out[i * 3] = c.x; out[i * 3 + 1] = c.y; out[i * 3 + 2] = c.z;
}

// compact tile-major part buffer -> full row-major framebuffer
__global__ void k_partition_scatter(const float* __restrict__ compact, float* __restrict__ full, const TileDev* __restrict__ tiles,
                                    int n_tiles, int width, int channels) {
    uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= (uint32_t)n_tiles * EZRT_TILE_PIXELS) return;
    TileDev t = tiles[r >> 8];
    int ix = (int)(r & 15u), iy = (int)((r & 255u) >> 4);
    if (ix >= t.w || iy >= t.h) return;
    size_t src = ((size_t)t.pixel_offset + (size_t)iy * t.w + ix) * channels;
    size_t dst = ((size_t)(t.y0 + iy) * width + (t.x0 + ix)) * channels;
    for (int c = 0; c < channels; c++) full[dst + c] = compact[src + c];
}

// ------------------------------------------------------------------------------------------
// denoiser (ezrt_math.h "denoiser", DESIGN.md section 9): k_denoise_init, then one k_atrous per iteration.  cv holds
// (colour, variance) per pixel; aov 2 float4 per pixel: (albedo, coverage), (normal, depth).  Full images, row-major.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_denoise_init(const float* __restrict__ color, int channels, const float* __restrict__ luma2,
                                                      int n_frames, long long n, float4* __restrict__ cv) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const vec3 c = ez_v3(color[i * channels], color[i * channels + 1], color[i * channels + 2]);
    cv[i] = make_float4(c.x, c.y, c.z, ez_denoise_var0(luma2[i], c, n_frames));
}

// One iteration, step s, one thread per pixel (16x16 blocks).  The last iteration writes the image (out, `channels` floats per
// pixel, alpha copied from color_in, which may be out itself) instead of cv_out.
__global__ void __launch_bounds__(256) k_atrous(int width, int height, int step, float sigma_l, float sigma_n, float sigma_z, float sigma_a,
                                                const float4* __restrict__ cv_in, const float4* __restrict__ aov, float4* __restrict__ cv_out,
                                                const float* color_in, float* out, int channels) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    const size_t p = (size_t)y * width + x;
    const float4 cp = cv_in[p];
    float4 res = cp;
    const float4 ap0 = aov[2 * p];
    if (ap0.w != 0.0f) {   // coverage 0: passed through
        const float4 ap1 = aov[2 * p + 1];
        const vec3 a_p = ez_v3(ap0.x, ap0.y, ap0.z), n_p = ez_v3(ap1.x, ap1.y, ap1.z);
        const float Y_p = ez_luminance(ez_v3(cp.x, cp.y, cp.z)), sd_p = EZ_SQRT(cp.w);
        float sw = 0.0f, sv = 0.0f;
        vec3 sc = splat3(0.0f);
#pragma unroll 1
        for (int j = -2; j <= 2; j++) {
            const int qy = y + step * j;
            if (qy < 0 || qy >= height) continue;
#pragma unroll
            for (int i = -2; i <= 2; i++) {
                const int qx = x + step * i;
                if (qx < 0 || qx >= width) continue;
                const float h = ez_b3(i) * ez_b3(j);
                float w;
                float4 cq;
                if (i == 0 && j == 0) {
                    w = h;
                    cq = cp;
                } else {
                    const size_t q = (size_t)qy * width + qx;
                    cq = cv_in[q];
                    const float4 aq0 = aov[2 * q];
                    if (aq0.w == 0.0f || !ez_finite(cq.x) || !ez_finite(cq.y) || !ez_finite(cq.z) || !ez_finite(cq.w)) continue;
                    const float4 aq1 = aov[2 * q + 1];
                    const int d = max(abs(i), abs(j));
                    w = ez_atrous_weight(h, (float)(step * d), n_p, ez_v3(aq1.x, aq1.y, aq1.z), ap1.w, aq1.w, Y_p, ez_luminance(ez_v3(cq.x, cq.y, cq.z)),
                                         sd_p, a_p, ez_v3(aq0.x, aq0.y, aq0.z), sigma_l, sigma_n, sigma_z, sigma_a);
                }
                sw = sw + w;
                sc = ez_add(sc, ez_scale(ez_v3(cq.x, cq.y, cq.z), w));
                sv = sv + (w * w) * cq.w;
            }
        }
        res = make_float4(EZ_DIV(sc.x, sw), EZ_DIV(sc.y, sw), EZ_DIV(sc.z, sw), EZ_DIV(sv, sw * sw));
    }
    if (out) {
        const size_t o = p * (size_t)channels;
        if (channels == 4) out[o + 3] = color_in[o + 3];
        out[o] = res.x; out[o + 1] = res.y; out[o + 2] = res.z;
    } else {
        cv_out[p] = res;
    }
}

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
static inline int div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

// run-time options -> template arguments: f(std::integral_constant<bool, b>...) for the bools b in order, so that each launcher
// names its kernel's instantiation once (combinations that are never instantiated are excluded by `if constexpr` inside f)
template <class F> static void with_bools(F&& f) { f(); }
template <class F, class... B> static void with_bools(F&& f, bool b, B... rest) {
    if (b) with_bools([&](auto... t) { f(std::true_type{}, t...); }, rest...);
    else with_bools([&](auto... t) { f(std::false_type{}, t...); }, rest...);
}

// persistent extend/shadow kernels: block size and resident blocks per SM (each block stages its own
// copy of the top tree levels in shared memory); env EZRT_EXTEND_THREADS / EZRT_EXTEND_BPS override
static int extend_threads() {
    static int v = 0;
    if (v == 0) {
        v = EZRT_EXTEND_THREADS;
        if (const char* e = getenv("EZRT_EXTEND_THREADS")) v = std::max(32, std::min(EZRT_EXTEND_MAX_THREADS, (atoi(e) / 32) * 32));
    }
    return v;
}
static int extend_blocks_per_sm() {
    static int v = 0;
    if (v == 0) {
        v = EZRT_EXTEND_BLOCKS_PER_SM;
        if (const char* e = getenv("EZRT_EXTEND_BPS")) v = std::max(1, std::min(16, atoi(e)));
    }
    return v;
}
void launch_generate(const RenderDev& rd, const TileDev* tiles, uint32_t n_slots, uint32_t batch_first_frame, PathQueue q,
                     uint32_t* q_count, int n_sms, cudaStream_t st, const LensDev* lens) {
    int blocks = std::min(div_up(n_slots, 256), n_sms * 8);
    const LensDev l = lens ? *lens : LensDev{};
    with_bools([&](auto L) { k_generate<L><<<blocks, 256, 0, st>>>(rd, tiles, n_slots, batch_first_frame, q, q_count, l); }, lens != nullptr);
}
// cudaFuncSetAttribute once per (kernel, size): the launchers run for every bounce of every batch
static void set_dynamic_smem(const void* kernel, size_t bytes) {
    static std::mutex mu;
    static std::map<const void*, size_t> done;
    std::lock_guard<std::mutex> lock(mu);
    auto it = done.find(kernel);
    if (it != done.end() && it->second >= bytes) return;   // the attribute is a maximum
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    done[kernel] = bytes;
}
template <class K>
static size_t smem_for(K kernel, int top_nodes) {
    size_t bytes = (size_t)top_nodes * EZRT_TOP_STRIDE * sizeof(float4) + (size_t)EZRT_SMEM_STACK * sizeof(int2) * extend_threads();
    set_dynamic_smem((const void*)kernel, std::max<size_t>(bytes, 1024));
    return bytes;
}
static int persistent_blocks(uint32_t n_max, int n_sms) {
    int blocks = std::min(div_up(n_max, extend_threads()), n_sms * extend_blocks_per_sm());
    return blocks < 1 ? 1 : blocks;
}

// exact traversal of the reference tree (policies REFERENCE / PRUNED, and the accel policy's fallback pass
// over the deferred indices in `perm`)
void launch_extend(const SceneDev& sc, bool prune, bool anyhit, PathQueue q, const uint32_t* q_count, uint32_t* work,
                   const uint32_t* perm, int to_accel, uint32_t n_max, int n_sms, cudaStream_t st, float2* side_hit, int gate) {
    int threads = extend_threads(), blocks = persistent_blocks(n_max, n_sms);
    int top = sc.top_nodes;
    if (gate == 1) {   // a few rays beside k_shade: small blocks find room on an SM as soon as one k_shade block retires
        threads = 128;
        blocks = std::max(1, std::min(div_up(n_max, threads), 64));
        top = 0;
    }
    with_bools([&](auto P, auto A) {
        k_extend<P, A><<<blocks, threads, smem_for(k_extend<P, A>, top), st>>>(sc, q, q_count, work, perm, to_accel, side_hit, gate);
    }, prune, anyhit);
}
template <class K>
static size_t w8_smem_for(K kernel, const SceneDev& sc) {
    size_t bytes = 2048 + (size_t)sc.w8_stack_entries * sizeof(uint2) * extend_threads();
    set_dynamic_smem((const void*)kernel, bytes);
    return bytes;
}
// the counters of the counting instantiations (counts != null, params.profile = 2): node visits to counts[2] when the kernel reads
// quantised nodes (W8, or the 4-wide tree's 96-byte form), to counts[0] when it reads the 128-byte exact nodes; triangle tests to counts[1]
static W8Counts w8_counts(unsigned long long* counts, bool quantised) {
    W8Counts c;
    c.node_visits = counts ? (quantised ? counts + 2 : counts) : nullptr;
    c.tri_tests = counts ? counts + 1 : nullptr;
    return c;
}
// accel policy: acceleration-tree pass (W8, or the round-1 4-wide kernel when the scene carries no W8 tree), then the
// exact pass over whatever it deferred.  counts != null selects the counting instantiation (params.profile = 2).
void launch_extend_accel(const SceneDev& sc, PathQueue q, const uint32_t* q_count, uint32_t* work, uint32_t* defer_list,
                         uint32_t* defer_count, uint32_t* defer_work, uint32_t n_max, int n_sms, unsigned long long* counts, const uint32_t* perm,
                         cudaStream_t st, int exact_gate) {
    const int threads = extend_threads(), blocks = persistent_blocks(n_max, n_sms);
    // incoherent rays on the 4-wide tree: the 96-byte quantised form of the nodes when the scene carries it (env EZRT_ACCEL_Q16=0: exact nodes)
    const W8Counts c = w8_counts(counts, sc.w8_nodes || sc.acc_wide_q16);
    if (sc.w8_nodes) {
        unsigned long long* const cyc = counts ? counts + EZRT_W8_PHASES_EXTEND : nullptr;
        with_bools([&](auto C, auto I) {
            k_extend_w8<C, I><<<blocks, threads, w8_smem_for(k_extend_w8<C, I>, sc), st>>>(sc, q, q_count, work, defer_list, defer_count, c, perm, cyc);
        }, counts != nullptr, sc.acc_tri_indexed != 0);
    } else {
        with_bools([&](auto C, auto Q) {
            k_extend_accel<C, Q><<<blocks, threads, smem_for(k_extend_accel<C, Q>, 0), st>>>(sc, q, q_count, work, defer_list, defer_count, c, perm);
        }, counts != nullptr, sc.acc_wide_q16 != 0);
    }
    launch_extend(sc, true, false, q, defer_count, defer_work, defer_list, 1, std::min<uint32_t>(n_max, 65536u), n_sms, st, nullptr, exact_gate);
}
// counting sort of the queue's ray indices into `perm` (3 kernels; bins must hold EZRT_SORT_BINS counters)
void launch_ray_sort(const SceneDev& sc, PathQueue q, const uint32_t* q_count, uint32_t* keys, uint32_t* bins, uint32_t* perm,
                     uint32_t n_max, int n_sms, cudaStream_t st) {
    cudaMemsetAsync(bins, 0, sizeof(uint32_t) * EZRT_SORT_BINS, st);
    int blocks = std::max(1, std::min(div_up(n_max, 256), n_sms * 8));
    k_sort_hist<<<blocks, 256, 0, st>>>(sc, q, q_count, keys, bins);
    k_sort_scan<<<1, 1024, 0, st>>>(bins);
    k_sort_scatter<<<blocks, 256, 0, st>>>(q_count, keys, bins, perm);
}
void launch_shadow(const SceneDev& sc, bool prune, ShadowQueue sq, const uint32_t* s_count, uint32_t* work, float4* Lo,
                   const uint32_t* perm, uint32_t n_max, int n_sms, cudaStream_t st, bool bounded) {
    const int threads = extend_threads(), blocks = persistent_blocks(n_max, n_sms);
    with_bools([&](auto P, auto B) {
        k_shadow<P, B><<<blocks, threads, smem_for(k_shadow<P, B>, sc.top_nodes), st>>>(sc, sq, s_count, work, Lo, perm);
    }, prune, bounded);
}
// camera pass of the W8 policy: rays generated in the kernel (slot i = ray i), then the exact pass over the deferred ones
void launch_extend_camera(const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, uint32_t batch_first_frame, uint32_t n_slots, uint32_t n_frames, PathQueue q,
                          uint32_t* work, uint32_t* defer_list, uint32_t* defer_count, uint32_t* defer_work, int n_sms, unsigned long long* counts,
                          cudaStream_t st, int exact_gate) {
    const int threads = extend_threads(), blocks = persistent_blocks(n_slots, n_sms);
    const W8Counts c = w8_counts(counts, sc.w8_nodes != nullptr);   // the 4-wide camera pass reads the 128-byte exact nodes
    if (sc.w8_nodes) {
        // s_perm + one stack of W8_BUNDLE_STACK entries per warp (extend_w8_bundle)
        const size_t smem = 2048 + (size_t)(threads / 32) * W8_BUNDLE_STACK * sizeof(uint2);
        with_bools([&](auto C, auto I) {
            set_dynamic_smem((const void*)k_extend_w8_camera<C, I>, smem);
            k_extend_w8_camera<C, I><<<blocks, threads, smem, st>>>(sc, rd, tiles, batch_first_frame, n_slots, n_frames, q, work, defer_list, defer_count, c);
        }, counts != nullptr, sc.acc_tri_indexed != 0);
    } else {
        with_bools([&](auto C) {
            k_extend_accel_camera<C><<<blocks, threads, smem_for(k_extend_accel_camera<C>, 0), st>>>(sc, rd, tiles, batch_first_frame, n_slots, n_frames, q, work, defer_list, defer_count, c);
        }, counts != nullptr);
    }
    launch_extend(sc, true, false, q, defer_count, defer_work, defer_list, 1, std::min<uint32_t>(n_slots, 65536u), n_sms, st, nullptr, exact_gate);
}
void launch_shadow_accel(const SceneDev& sc, ShadowQueue sq, const uint32_t* s_count, uint32_t* work, float4* Lo, uint32_t* defer_list,
                         uint32_t* defer_count, uint32_t* defer_work, uint32_t n_max, int n_sms, unsigned long long* counts, cudaStream_t st, bool bounded) {
    const int threads = extend_threads(), blocks = persistent_blocks(n_max, n_sms);
    const W8Counts c = w8_counts(counts, sc.w8_nodes || sc.acc_wide_q16);
    if (sc.w8_nodes) {
        unsigned long long* const cyc = counts ? counts + EZRT_W8_PHASES_SHADOW : nullptr;
        with_bools([&](auto C, auto I, auto B) {
            k_shadow_w8<C, I, B><<<blocks, threads, w8_smem_for(k_shadow_w8<C, I, B>, sc), st>>>(sc, sq, s_count, work, Lo, defer_list, defer_count, c, cyc);
        }, counts != nullptr, sc.acc_tri_indexed != 0, bounded);
    } else {
        with_bools([&](auto C, auto Q, auto B) {
            k_shadow_accel<C, Q, B><<<blocks, threads, smem_for(k_shadow_accel<C, Q, B>, 0), st>>>(sc, sq, s_count, work, Lo, defer_list, defer_count, c);
        }, counts != nullptr, sc.acc_wide_q16 != nullptr, bounded);
    }
    launch_shadow(sc, true, sq, defer_count, defer_work, Lo, defer_list, std::min<uint32_t>(n_max, 65536u), n_sms, st, bounded);
}
// k_shade over the queue, or (LIST) over the deferred lane's list with its hits in side_hit.  The instantiation follows the mode,
// aov_rec (non-null: AOV) and the light sampling mode's options; MODE = k_shade's mode template argument for rd.mode.
template <bool LIST>
static void launch_shade_t(int blocks, const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, int bounce, uint32_t batch_first_frame,
                           PathQueue qin, const uint32_t* in_count, PathQueue qout, uint32_t* out_count, ShadowQueue sq, uint32_t* s_count,
                           float4* Lo, float4* Le, uint32_t n_fused, uint32_t n_frames, const uint32_t* list, const float2* side_hit,
                           float4* aov_rec, const LightOptions& o, cudaStream_t st) {
    auto launch = [&](auto M) {
        with_bools([&](auto A, auto E, auto T, auto X, auto TX, auto MP) {
            // the options exist in the light sampling mode; the maps with the textures
            if constexpr ((M == EZRT_MODE_DISNEY_LIGHTS || !(E || T || X || TX)) && !(T && X) && (TX || !MP))
                k_shade<M, LIST, A, E, T, X, TX, MP><<<blocks, 128, 0, st>>>(sc, rd, tiles, bounce, batch_first_frame, qin, in_count, qout, out_count, sq,
                                                                             s_count, Lo, Le, n_fused, n_frames, list, side_hit, aov_rec, o.lights, o.env,
                                                                             o.med, o.tex, o.maps);
        }, aov_rec != nullptr, o.env_on, o.trans_on, o.medium_on, o.tex_on, o.maps_on);
    };
    switch (rd.mode) {
        case EZRT_MODE_DIFFUSE_P3: launch(std::integral_constant<int, EZRT_MODE_DIFFUSE_P3>{}); break;
        case EZRT_MODE_DISNEY_ANISO_P4: launch(std::integral_constant<int, EZRT_MODE_DISNEY_ANISO_P4>{}); break;
        case EZRT_MODE_DISNEY_SOBOL_P5: launch(std::integral_constant<int, EZRT_MODE_DISNEY_SOBOL_P5>{}); break;
        case EZRT_MODE_DISNEY_LIGHTS: launch(std::integral_constant<int, EZRT_MODE_DISNEY_LIGHTS>{}); break;
        default: launch(std::integral_constant<int, EZRT_MODE_DISNEY_IS_MIS_P5>{}); break;
    }
}
void launch_shade(const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, int bounce, uint32_t batch_first_frame,
                  PathQueue qin, const uint32_t* in_count, PathQueue qout, uint32_t* out_count, ShadowQueue sq,
                  uint32_t* s_count, float4* Lo, float4* Le, uint32_t n_max, uint32_t n_fused, uint32_t n_frames, int n_sms, cudaStream_t st,
                  float4* aov_rec, const LightOptions& o) {
    const int blocks = std::max(1, std::min(div_up(n_max, 128), n_sms * 4 * EZRT_SHADE_MIN_BLOCKS));
    launch_shade_t<false>(blocks, sc, rd, tiles, bounce, batch_first_frame, qin, in_count, qout, out_count, sq, s_count, Lo, Le, n_fused, n_frames,
                          nullptr, nullptr, aov_rec, o, st);
}
// The accel policy's deferred lane (side stream, beside the main k_shade of the same bounce): exact traversal of the deferred
// rays into side_hit, then their shading -- both do nothing if more than EZRT_SIDE_CAP rays were deferred (then
// launch_extend_accel / launch_extend_camera with exact_gate = 2 traced them in line).
void launch_deferred_lane(const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, int bounce, uint32_t batch_first_frame, PathQueue qin,
                          const uint32_t* defer_list, const uint32_t* defer_count, uint32_t* defer_work, float2* side_hit, PathQueue qout,
                          uint32_t* out_count, ShadowQueue sq, uint32_t* s_count, float4* Lo, float4* Le, uint32_t n_fused, uint32_t n_frames,
                          int n_sms, cudaStream_t st, float4* aov_rec, const LightOptions& o) {
    launch_extend(sc, true, false, qin, defer_count, defer_work, defer_list, 1, EZRT_SIDE_CAP, n_sms, st, side_hit, 1);
    launch_shade_t<true>(8, sc, rd, tiles, bounce, batch_first_frame, qin, defer_count, qout, out_count, sq, s_count, Lo, Le, n_fused, n_frames,
                         defer_list, side_hit, aov_rec, o, st);
}
void launch_nee(const SceneDev& sc, const RenderDev& rd, ShadowQueue sq, const uint32_t* s_count, float4* Lo, uint32_t n_max, int n_sms, cudaStream_t st,
                const LightOptions& o) {
    const int blocks = std::max(1, std::min(div_up(n_max, 512), n_sms * 8));
    with_bools([&](auto L, auto E, auto T, auto X, auto TX, auto MP) {
        // the options exist in the light sampling mode (the other mode here is mode 3); the maps with the textures
        if constexpr ((L || !(E || T || X || TX)) && !(T && X) && (TX || !MP))
            k_nee<L ? EZRT_MODE_DISNEY_LIGHTS : EZRT_MODE_DISNEY_IS_MIS_P5, E, T, X, TX, MP><<<blocks, 128, 0, st>>>(sc, rd, sq, s_count, Lo, o.med, o.tex, o.maps);
    }, rd.mode == EZRT_MODE_DISNEY_LIGHTS, o.env_on, o.trans_on, o.medium_on, o.tex_on, o.maps_on);
}

// ------------------------------------------------------------------------------------------
// light table of the light sampling mode (ezrt_math.h, DESIGN.md section 10): the weight of every triangle in the caller's
// order, the lights kept in that order, then their records.  One-off, at the first render in that mode.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_light_weights(SceneDev sc, float* __restrict__ w) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sc.n_triangles) return;
    vec3 p1, p2, p3;
    tri_vertices(sc, i, false, p1, p2, p3);
    w[i] = ez_light_weight(p1, p2, p3, load_emissive(sc, tri_material(sc, i)));
}
// stable compaction in one block: chunks of blockDim.x triangles in order, each ranked by thread index (block_append on a
// shared-memory counter), as k_adaptive_check's tail
__global__ void __launch_bounds__(1024) k_light_compact(const float* __restrict__ w, int n, int32_t* __restrict__ idx_out, float* __restrict__ w_out,
                                                        int32_t* __restrict__ count) {
    __shared__ uint32_t s_scan[34];
    __shared__ uint32_t s_count;
    if (threadIdx.x == 0) s_count = 0u;
    __syncthreads();
    for (int i0 = 0; i0 < n; i0 += blockDim.x) {
        const int i = i0 + threadIdx.x;
        const float wi = (i < n) ? w[i] : 0.0f;
        const bool keep = (i < n) && ez_is_light(wi);
        const uint32_t pos = block_append(keep, &s_count, s_scan);
        if (keep) { idx_out[pos] = i; w_out[pos] = wi; }
    }
    __syncthreads();
    if (threadIdx.x == 0) *count = (int32_t)s_count;
}
__global__ void __launch_bounds__(256) k_light_records(SceneDev sc, const int32_t* __restrict__ idx, int n, float4* __restrict__ rec) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const int tri = idx[k];
    vec3 p1, p2, p3;
    tri_vertices(sc, tri, false, p1, p2, p3);
    const int mat = tri_material(sc, tri);
    const vec3 N = f4xyz(ldg4(tri_geo_rec(sc, tri, false)));
    const int acc = sc.ref_to_acc ? (int)sc.ref_to_acc[tri] : tri;
    rec[4 * k] = make_float4(p1.x, p1.y, p1.z, __int_as_float(mat));
    rec[4 * k + 1] = make_float4(p2.x, p2.y, p2.z, __int_as_float(tri));
    rec[4 * k + 2] = make_float4(p3.x, p3.y, p3.z, __int_as_float(acc));
    rec[4 * k + 3] = make_float4(N.x, N.y, N.z, ez_luminance(load_emissive(sc, mat)));
}
// the environment table's texel weights (ezrt_math.h, DESIGN.md section 11): w[i * W + j] = ez_env_weight(texel (i, j) of the map)
__global__ void __launch_bounds__(256) k_env_weights(SceneDev sc, float* __restrict__ w) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= sc.hdr_w * sc.hdr_h) return;
    w[k] = ez_env_weight(texel3(sc.hdr, k), k / sc.hdr_w, sc.hdr_h);
}
void launch_env_weights(const SceneDev& sc, float* w, cudaStream_t st) {
    const int n = sc.hdr_w * sc.hdr_h;
    if (!sc.hdr || n <= 0) return;
    k_env_weights<<<div_up(n, 256), 256, 0, st>>>(sc, w);
}
void launch_light_weights(const SceneDev& sc, float* w, cudaStream_t st) {
    if (sc.n_triangles <= 0) return;
    k_light_weights<<<div_up(sc.n_triangles, 256), 256, 0, st>>>(sc, w);
}
void launch_light_compact(const float* w, int n, int32_t* idx_out, float* w_out, int32_t* count, cudaStream_t st) {
    k_light_compact<<<1, 1024, 0, st>>>(w, n, idx_out, w_out, count);
}
void launch_light_records(const SceneDev& sc, const int32_t* idx, int n, float4* rec, cudaStream_t st) {
    if (n <= 0) return;
    k_light_records<<<div_up(n, 256), 256, 0, st>>>(sc, idx, n, rec);
}
void launch_blend(const RenderDev& rd, const TileDev* tiles, int nf, uint32_t batch_first_frame, const float4* Lo, const float4* Le,
                  float* fb, float* luma2, int32_t* spp_map, const float4* aov_rec, float* aov, cudaStream_t st) {
    uint32_t per_frame = (uint32_t)rd.n_tiles * EZRT_TILE_PIXELS;
    with_bools([&](auto ADAPTIVE, auto AOV) {
        if constexpr (ADAPTIVE || !AOV)   // the feature buffers keep luma2
            k_blend<ADAPTIVE, AOV><<<div_up(per_frame, 256), 256, 0, st>>>(rd, tiles, nf, batch_first_frame, Lo, Le, fb, luma2, spp_map, aov_rec, aov);
    }, luma2 != nullptr, aov != nullptr);
}
void launch_adaptive_check(const RenderDev& rd, const TileDev* tiles_in, int n_frames, float threshold, const float* fb, const float* luma2,
                           unsigned char* keep, unsigned int* blocks_done, TileDev* tiles_out, int32_t* counts, cudaStream_t st) {
    if (rd.n_tiles <= 0) return;
    k_adaptive_check<<<rd.n_tiles, EZRT_TILE_PIXELS, 0, st>>>(rd, tiles_in, n_frames, threshold, fb, luma2, keep, blocks_done, tiles_out, counts);
}
void launch_tally(const uint32_t* q_counts, const uint32_t* s_counts, const uint32_t* d_ext, const uint32_t* d_sh, int n_stages,
                  unsigned long long* totals, uint32_t n_primary, cudaStream_t st) {
    k_tally<<<1, 32, 0, st>>>(q_counts, s_counts, d_ext, d_sh, n_stages, totals, n_primary);
}
void launch_megakernel(const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, bool prune, int spp, float* fb,
                       unsigned long long* totals, cudaStream_t st, const LensDev* lens) {
    uint32_t per_frame = (uint32_t)rd.n_tiles * EZRT_TILE_PIXELS;
    const LensDev l = lens ? *lens : LensDev{};
    with_bools([&](auto P, auto L) { k_megakernel<P, L><<<div_up(per_frame, 128), 128, 0, st>>>(sc, rd, tiles, spp, fb, totals, l); },
               prune, lens != nullptr);
}
void launch_camera_rays(const RenderDev& rd, const LensDev* lens, int n, const uint32_t* px, const uint32_t* py, const uint32_t* frame,
                        float* o, float* d, cudaStream_t st) {
    if (n <= 0) return;
    k_camera_rays<<<div_up(n, 128), 128, 0, st>>>(rd, lens ? 1 : 0, n, px, py, frame, o, d, lens ? *lens : LensDev{});
}
void launch_trace_finish(const SceneDev& sc, int n, PathQueue q, int p3fudge, int accel_space, int* hit, float* dist, int* tri, int* inside,
                         float* point, float* normal, cudaStream_t st) {
    k_trace_finish<<<div_up(n, 128), 128, 0, st>>>(sc, n, q, p3fudge, accel_space, hit, dist, tri, inside, point, normal);
}
void launch_eval_brdf(int which, int n, const float* V, const float* N, const float* L, const float* xi, const float* materials,
                      float* out, cudaStream_t st) {
    k_eval_brdf<<<div_up(n, 128), 128, 0, st>>>(which, n, V, N, L, xi, materials, out);
}
void launch_eval_bsdf(int which, int n, const float* V, const float* N, const float* L, const float* xi, const int* inside,
                      const float* materials, float* out, cudaStream_t st) {
    k_eval_bsdf<<<div_up(n, 128), 128, 0, st>>>(which, n, V, N, L, xi, inside, materials, out);
}
__global__ void k_tex_gather(const float4* __restrict__ rec, const uint32_t* __restrict__ acc_tri_ref, int n, float4* __restrict__ acc_rec) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n) return;
    const uint32_t r = acc_tri_ref[a];
    acc_rec[2 * (size_t)a] = rec[2 * (size_t)r];
    acc_rec[2 * (size_t)a + 1] = rec[2 * (size_t)r + 1];
}
void launch_tex_gather(const float4* rec, const uint32_t* acc_tri_ref, int n, float4* acc_rec, cudaStream_t st) {
    k_tex_gather<<<div_up(n, 256), 256, 0, st>>>(rec, acc_tri_ref, n, acc_rec);
}
// the textured base colour of the hits shade_step<.., TEX> computes, at the points of reference triangles (ezrt_scene_sample_textures)
__global__ void k_sample_textures(SceneDev sc, TexDev tex, int n, const int32_t* __restrict__ tri, const float* __restrict__ points,
                                  float* __restrict__ uv, float* __restrict__ rgb) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int t = tri[i];
    const vec3 P = ez_v3(points[3 * i], points[3 * i + 1], points[3 * i + 2]);
    const vec3 c = tex_base_color(sc, tex, t, false, P, load_material(sc, tri_material(sc, t)).baseColor, uv + 2 * (size_t)i);
    rgb[3 * i] = c.x; rgb[3 * i + 1] = c.y; rgb[3 * i + 2] = c.z;
}
void launch_sample_textures(const SceneDev& sc, const TexDev& tex, int n, const int32_t* tri, const float* points, float* uv, float* rgb,
                            cudaStream_t st) {
    k_sample_textures<<<div_up(n, 128), 128, 0, st>>>(sc, tex, n, tri, points, uv, rgb);
}
// what shade_step<.., TEX, MAPS> computes at hits (reference triangle, o, d, t) (ezrt_scene_sample_materials): the UV, the textured
// base colour, the mapped roughness and metallic and the final shading normal, 10 floats per hit
__global__ void k_sample_materials(SceneDev sc, TexDev tex, MapsDev maps, int n, const int32_t* __restrict__ tri, const float* __restrict__ odt,
                                   float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int t = tri[i];
    const float* r = odt + 7 * (size_t)i;
    const vec3 o = ez_v3(r[0], r[1], r[2]), d = ez_v3(r[3], r[4], r[5]);
    SurfaceHit hit = surface_hit(sc, o, d, r[6], t, false, false);
    MaterialDev mat = load_material(sc, hit.matId);
    float* w = out + 10 * (size_t)i;
    tex_material(sc, tex, maps, t, false, hit.P, ez_neg(d), hit.inside, mat, hit.N, w);
    w[2] = mat.baseColor.x; w[3] = mat.baseColor.y; w[4] = mat.baseColor.z;
    w[5] = mat.roughness; w[6] = mat.metallic;
    w[7] = hit.N.x; w[8] = hit.N.y; w[9] = hit.N.z;
}
void launch_sample_materials(const SceneDev& sc, const TexDev& tex, const MapsDev& maps, int n, const int32_t* tri, const float* odt, float* out,
                             cudaStream_t st) {
    k_sample_materials<<<div_up(n, 128), 128, 0, st>>>(sc, tex, maps, n, tri, odt, out);
}
// the maps' words of n triangles (reference order) into the fourth word of both texcoord record copies (ezrt_scene_set_material_maps)
__global__ void k_maps_set(const uint32_t* __restrict__ words, const uint32_t* __restrict__ acc_tri_ref, int n, float4* rec, float4* acc_rec) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    rec[2 * (size_t)i + 1].w = __uint_as_float(words[i]);
    if (acc_tri_ref) acc_rec[2 * (size_t)i + 1].w = __uint_as_float(words[acc_tri_ref[i]]);
}
void launch_maps_set(const uint32_t* words, const uint32_t* acc_tri_ref, int n, float4* rec, float4* acc_rec, cudaStream_t st) {
    k_maps_set<<<div_up(n, 256), 256, 0, st>>>(words, acc_tri_ref, n, rec, acc_rec);
}
void launch_eval_math(int which, int n, const float* a, const float* b, float* out, cudaStream_t st) {
    k_eval_math<<<div_up(n, 256), 256, 0, st>>>(which, n, a, b, out);
}
void launch_tonemap(const float* in, int channels, float* out, long long n, float limit, cudaStream_t st) {
    if (n <= 0) return;
    k_tonemap<<<div_up(n, 256), 256, 0, st>>>(in, channels, out, n, limit);
}
void launch_partition_scatter(const float* compact, float* full, const TileDev* tiles, int n_tiles, int width, int channels,
                              cudaStream_t st) {
    if (n_tiles <= 0) return;
    k_partition_scatter<<<div_up((long long)n_tiles * EZRT_TILE_PIXELS, 256), 256, 0, st>>>(compact, full, tiles, n_tiles, width, channels);
}
void launch_denoise(const float* color, int channels, const float* aov, const float* luma2, int n_frames, int width, int height, int iterations,
                    float sigma_l, float sigma_n, float sigma_z, float sigma_a, float4* cv0, float4* cv1, float* out, cudaStream_t st) {
    const long long n = (long long)width * height;
    if (n <= 0) return;
    k_denoise_init<<<div_up(n, 256), 256, 0, st>>>(color, channels, luma2, n_frames, n, cv0);
    const dim3 block(16, 16), grid(div_up(width, 16), div_up(height, 16));
    for (int k = 0; k < iterations; k++) {
        const bool last = (k == iterations - 1);
        k_atrous<<<grid, block, 0, st>>>(width, height, 1 << k, sigma_l, sigma_n, sigma_z, sigma_a, (k & 1) ? cv1 : cv0, (const float4*)aov,
                                         (k & 1) ? cv0 : cv1, color, last ? out : nullptr, channels);
    }
}
