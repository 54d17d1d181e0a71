// accel_build.cu -- the binary SAH acceleration tree of ezrt_scene_create, built on the GPU.
//
// Produces EXACTLY the tree of the host builder ezrt_build_accel (host_scene.cpp: exhaustive-sweep SAH without the reference's
// INF = 114514 sentinel, "sort once" per axis, median split below depth 32), node for node and bit for bit, so that everything
// measured on the host-built tree holds: the same fp32 cost expression (-fmad=false here, -ffp-contract=off there), the same
// tie rule (lowest cost, then lowest axis, then lowest split position), the same stable orders.  The reference's own tree
// (buildBVHwithSAH, P5/main.cpp:458-589) is NOT built here -- it arrives through the C ABI and is walked literally by the
// exact kernels; this is the device's own tree, which only has to be conservative (DESIGN.md section 4).
//
// Breadth-first, one level per round, every level as whole-array primitives over the n triangle positions:
//   sort      three cub radix sorts of the centroid coordinates (stable, like std::stable_sort on the host)
//   sweep     per axis a segmented prefix and a segmented suffix scan (cub::DeviceScan::InclusiveScanByKey, key = the node
//             that owns the position) of the triangle boxes in that axis' order = the host's lmin/lmax and rmin/rmax runs
//   choose    every split position of every axis computes its cost and atomicMin's a packed (cost | axis | position) word
//             into its node
//   partition the node's triangles are marked left/right along the chosen axis; the three orders are stable-partitioned with a
//             segmented exclusive sum of the "left" flags
// A node is identified by its slot in a sparse pre-order numbering -- node(base, l, r): left = base + 1, right = base +
// 2 * count(left) -- so no allocation counter is needed and a final compaction of the used slots yields the host builder's
// dense pre-order array.  The children's boxes fall out of the parent's sweep (prefix at the split, suffix after it).
//
// 1 M triangles: level rounds plus the read-back of the 660 k nodes, much faster than the threaded host builder.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <cub/cub.cuh>
#include <utility>
#include <vector>

#include "ezrt.h"
#include "ezrt_internal.h"
#include "ezrt_math.h"

namespace {

struct Box {
    float lo[3], hi[3];
};
struct BoxUnion {
    __host__ __device__ __forceinline__ Box operator()(const Box& a, const Box& b) const {
        Box r;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            r.lo[k] = ez_min(a.lo[k], b.lo[k]);
            r.hi[k] = ez_max(a.hi[k], b.hi[k]);
        }
        return r;
    }
};

// half_area2 of host_scene.cpp ("2.0 * (lx*ly + lx*lz + ly*lz)", P5/main.cpp:549)
__device__ __forceinline__ float box_area2(const Box& b) {
    const float lenx = b.hi[0] - b.lo[0], leny = b.hi[1] - b.lo[1], lenz = b.hi[2] - b.lo[2];
    return 2.0f * ((lenx * leny) + (lenx * lenz) + (leny * lenz));
}

struct BuildDev {
    int n, leaf_n, median_depth;
    const Box* tri_box;      // per triangle
    uint32_t* idx[3];        // triangle ids in centroid order of axis a, partitioned by node
    uint32_t* idx_new[3];
    int* seg;                // per position: slot of the node that owns it
    Box* L[3];               // per position: union of the node's boxes up to here, in axis order
    Box* Rrev[3];            // the same from the right; element j belongs to position n - 1 - j
    int* rank[3];            // per position: "left" flags before it within its node
    unsigned char* side;     // per triangle: 1 = right child
    // per slot (2n)
    int* nd_l;
    int* nd_r;
    int* nd_split;
    Box* nd_box;
    int* used;
    unsigned long long* best;
    int* counter;            // [0] = inner nodes created this level
};

__global__ void k_tri_boxes(const float* __restrict__ tris, int n, Box* __restrict__ box, float* __restrict__ key_x, float* __restrict__ key_y,
                            float* __restrict__ key_z, uint32_t* __restrict__ iota) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* t = tris + (size_t)i * EZRT_TRIANGLE_FLOATS;
    const ez_vec3 p1 = ez_v3(t[0], t[1], t[2]), p2 = ez_v3(t[3], t[4], t[5]), p3 = ez_v3(t[6], t[7], t[8]);
    const ez_vec3 c = ez_divs(ez_add(ez_add(p1, p2), p3), 3.0f);   // centroid(), host_scene.cpp (cmpx/cmpy/cmpz, P5/main.cpp:156-170)
    Box b;
    b.lo[0] = ez_min(p1.x, ez_min(p2.x, p3.x)); b.lo[1] = ez_min(p1.y, ez_min(p2.y, p3.y)); b.lo[2] = ez_min(p1.z, ez_min(p2.z, p3.z));
    b.hi[0] = ez_max(p1.x, ez_max(p2.x, p3.x)); b.hi[1] = ez_max(p1.y, ez_max(p2.y, p3.y)); b.hi[2] = ez_max(p1.z, ez_max(p2.z, p3.z));
    box[i] = b;
    // + 0.0f: -0.0 and +0.0 are one key, as for the host's `<` comparator
    key_x[i] = c.x + 0.0f;
    key_y[i] = c.y + 0.0f;
    key_z[i] = c.z + 0.0f;
    iota[i] = (uint32_t)i;
}

__global__ void k_init_root(BuildDev d) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < d.n) d.seg[i] = 0;
    if (i == 0) {
        d.nd_l[0] = 0;
        d.nd_r[0] = d.n - 1;
        d.used[0] = 1;
        d.best[0] = ~0ull;
        d.nd_split[0] = -1;
    }
}

struct GatherBox {
    const Box* box;
    const uint32_t* idx;
    __host__ __device__ __forceinline__ Box operator()(int i) const { return box[idx[i]]; }
};
struct GatherBoxRev {
    const Box* box;
    const uint32_t* idx;
    int last;
    __host__ __device__ __forceinline__ Box operator()(int j) const { return box[idx[last - j]]; }
};
struct KeyRev {
    const int* seg;
    int last;
    __host__ __device__ __forceinline__ int operator()(int j) const { return seg[last - j]; }
};
struct LeftFlag {
    const unsigned char* side;
    const uint32_t* idx;
    __host__ __device__ __forceinline__ int operator()(int i) const { return side[idx[i]] ? 0 : 1; }
};

// every split position of every axis: cost as in build_accel_presorted, packed so that an unsigned min picks the lowest cost,
// then the lowest axis, then the lowest position (the host loop keeps the first strictly smaller candidate)
__global__ void k_cost(BuildDev d) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = i < d.n;
    const int s = in ? d.seg[i] : -1;
    const int l = in ? d.nd_l[s] : 0, r = in ? d.nd_r[s] : 0;
    const bool active = in && (r - l + 1 > d.leaf_n) && i < r;
    unsigned long long bestw = ~0ull;
#pragma unroll
    for (int a = 0; a < 3 && active; a++) {
        const Box lb = d.L[a][i];
        const Box rb = d.Rrev[a][d.n - 1 - (i + 1)];
        float total = box_area2(lb) * (float)(i - l + 1) + box_area2(rb) * (float)(r - i);
        if (total < 3.0e38f) {
            total = total + 0.0f;   // -0.0 -> +0.0: the bit pattern orders like the value
            const unsigned long long w = ((unsigned long long)__float_as_uint(total) << 32) | ((unsigned long long)a << 30) | (unsigned long long)i;
            if (w < bestw) bestw = w;
        }
    }
    // one atomic per warp when the whole warp sits in one node (the big nodes of the top levels: n atomics on one word otherwise)
    const unsigned full = 0xffffffffu;
    const int s0 = __shfl_sync(full, s, 0);
    if (__all_sync(full, s == s0)) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const unsigned long long o = __shfl_xor_sync(full, bestw, off);
            if (o < bestw) bestw = o;
        }
        if ((threadIdx.x & 31) == 0 && bestw != ~0ull) atomicMin(&d.best[s], bestw);
    } else if (bestw != ~0ull) {
        atomicMin(&d.best[s], bestw);
    }
}

// per position: which side of its node's split it lies on; the node's first position also writes the two children
__global__ void k_split(BuildDev d, int level) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= d.n) return;
    const int s = d.seg[i];
    const int l = d.nd_l[s], r = d.nd_r[s];
    if (level == 0 && i == 0) d.nd_box[0] = d.L[0][d.n - 1];
    if (r - l + 1 <= d.leaf_n) return;
    const unsigned long long b = d.best[s];
    int axis = 0, split = (l + r) / 2;
    if (b != ~0ull) {
        axis = (int)((b >> 30) & 3ull);
        split = (int)(b & 0x3fffffffull);
    }
    if (d.median_depth > 0 && level >= d.median_depth) split = (l + r) / 2;   // coincident triangles: no O(n)-deep chains
    const uint32_t t = (axis == 0) ? d.idx[0][i] : (axis == 1) ? d.idx[1][i] : d.idx[2][i];
    d.side[t] = (i > split) ? 1 : 0;
    if (i != l) return;
    d.nd_split[s] = split;
    const int nleft = split - l + 1;
    const int cl = s + 1, cr = s + 2 * nleft;
    const Box* La = (axis == 0) ? d.L[0] : (axis == 1) ? d.L[1] : d.L[2];
    const Box* Ra = (axis == 0) ? d.Rrev[0] : (axis == 1) ? d.Rrev[1] : d.Rrev[2];
    d.nd_l[cl] = l; d.nd_r[cl] = split; d.nd_box[cl] = La[split]; d.used[cl] = 1; d.best[cl] = ~0ull; d.nd_split[cl] = -1;
    d.nd_l[cr] = split + 1; d.nd_r[cr] = r; d.nd_box[cr] = Ra[d.n - 1 - (split + 1)]; d.used[cr] = 1; d.best[cr] = ~0ull; d.nd_split[cr] = -1;
    int inner = 0;
    if (nleft > d.leaf_n) inner++;
    if (r - split > d.leaf_n) inner++;
    if (inner) atomicAdd(&d.counter[0], inner);
}

// stable partition of the three orders inside every split node; positions then belong to the children
__global__ void k_scatter(BuildDev d) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= d.n) return;
    const int s = d.seg[i];
    const int l = d.nd_l[s], r = d.nd_r[s];
    if (r - l + 1 <= d.leaf_n) {
#pragma unroll
        for (int a = 0; a < 3; a++) d.idx_new[a][i] = d.idx[a][i];
        return;
    }
    const int split = d.nd_split[s];
    const int nleft = split - l + 1;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const uint32_t t = d.idx[a][i];
        const int rk = d.rank[a][i];
        const int pos = d.side[t] ? (l + nleft + (i - l - rk)) : (l + rk);
        d.idx_new[a][pos] = t;
    }
    d.seg[i] = (i <= split) ? (s + 1) : (s + 2 * nleft);
}

__global__ void k_emit(BuildDev d, const int* __restrict__ dense, int n_slots, EzrtAccelNode* __restrict__ out) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots || !d.used[s]) return;
    EzrtAccelNode nd;
    const int l = d.nd_l[s], r = d.nd_r[s];
    if (r - l + 1 <= d.leaf_n) {
        nd.left = nd.right = 0;
        nd.n = r - l + 1;
        nd.index = l;
    } else {
        const int nleft = d.nd_split[s] - l + 1;
        nd.left = dense[s + 1];
        nd.right = dense[s + 2 * nleft];
        nd.n = 0;
        nd.index = 0;
    }
    const Box b = d.nd_box[s];
    for (int k = 0; k < 3; k++) { nd.AA[k] = b.lo[k]; nd.BB[k] = b.hi[k]; }
    out[dense[s]] = nd;
}

struct Arena {
    char* base = nullptr;
    size_t size = 0, off = 0;
    template <class T>
    T* take(size_t count) {
        off = (off + 255) & ~(size_t)255;
        T* p = (T*)(base + off);
        off += count * sizeof(T);
        return p;
    }
};

#define CUB_OK(call)                                                                                             \
    do {                                                                                                         \
        cudaError_t e_ = (call);                                                                                 \
        if (e_ != cudaSuccess) {                                                                                 \
            rc = ezrt_set_error(EZRT_ERR_CUDA, "accel build: %s: %s", #call, cudaGetErrorString(e_));            \
            goto done;                                                                                           \
        }                                                                                                        \
    } while (0)

}  // namespace

// d_tris: the caller's Triangle_encoded array on the device (36 floats per triangle).  nodes_out / order: as ezrt_build_accel.
int ezrt_build_accel_device(const float* d_tris, int n, int leaf_n, std::vector<EzrtAccelNode>& nodes_out, std::vector<uint32_t>& order,
                            int* levels_out) {
    if (!d_tris || n <= 0 || leaf_n < 1) return ezrt_set_error(EZRT_ERR_INVALID, "accel build: bad argument");
    int rc = EZRT_OK;
    EzrtLap lap("ezrt_build_accel_device");
    const int threads = 256, blocks = (n + threads - 1) / threads;
    const int n_slots = 2 * n;
    typedef cub::CountingInputIterator<int> Count;
    typedef cub::TransformInputIterator<Box, GatherBox, Count> BoxIt;
    typedef cub::TransformInputIterator<Box, GatherBoxRev, Count> BoxRevIt;
    typedef cub::TransformInputIterator<int, KeyRev, Count> KeyRevIt;
    typedef cub::TransformInputIterator<int, LeftFlag, Count> FlagIt;
    Arena ar;
    BuildDev d;
    memset(&d, 0, sizeof(d));
    d.n = n; d.leaf_n = leaf_n;
    d.median_depth = 32;   // as ezrt_build_accel: depth <= 32 + log2(n), the traversal stacks always suffice
    float* keys[3] = {nullptr, nullptr, nullptr};
    float* keys_out = nullptr;
    uint32_t* iota = nullptr;
    int* dense = nullptr;
    EzrtAccelNode* out_nodes = nullptr;
    Box* tri_box = nullptr;
    void* temp = nullptr;
    size_t temp_bytes = 0;
    int levels = 0, n_nodes = 0;
    // ---- temp storage: the largest request of the cub calls below ----
    {
        size_t b = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, b, (const float*)nullptr, (float*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr, n);
        temp_bytes = std::max(temp_bytes, b);
        GatherBox g{nullptr, nullptr};
        cub::DeviceScan::InclusiveScanByKey(nullptr, b, (const int*)nullptr, BoxIt(Count(0), g), (Box*)nullptr, BoxUnion(), n);
        temp_bytes = std::max(temp_bytes, b);
        GatherBoxRev gr{nullptr, nullptr, 0};
        KeyRev kr{nullptr, 0};
        cub::DeviceScan::InclusiveScanByKey(nullptr, b, KeyRevIt(Count(0), kr), BoxRevIt(Count(0), gr), (Box*)nullptr, BoxUnion(), n);
        temp_bytes = std::max(temp_bytes, b);
        LeftFlag lf{nullptr, nullptr};
        cub::DeviceScan::ExclusiveSumByKey(nullptr, b, (const int*)nullptr, FlagIt(Count(0), lf), (int*)nullptr, n);
        temp_bytes = std::max(temp_bytes, b);
        cub::DeviceScan::ExclusiveSum(nullptr, b, (const int*)nullptr, (int*)nullptr, n_slots);
        temp_bytes = std::max(temp_bytes, b);
    }
    {
        const size_t N = (size_t)n, S = (size_t)n_slots;
        size_t need = temp_bytes + 256;
        need += (N * sizeof(Box) + 256);                     // tri_box
        need += 4 * (N * sizeof(float) + 256);                // keys, keys_out
        need += (N * 4 + 256);                                // iota
        need += 6 * (N * 4 + 256);                            // idx, idx_new
        need += (N * 4 + 256);                                // seg
        need += 6 * (N * sizeof(Box) + 256);                  // L, Rrev
        need += 3 * (N * 4 + 256);                            // rank
        need += (N + 256);                                    // side
        need += 4 * (S * 4 + 256) + (S * sizeof(Box) + 256) + (S * 8 + 256);   // per-slot arrays
        need += (S * 4 + 256);                                // dense
        need += (S / 2 + 1) * 2 * sizeof(EzrtAccelNode) + 256;   // out_nodes: at most 2n - 1 nodes
        need += 1024;
        ar.size = need;
        if (cudaMalloc((void**)&ar.base, need) != cudaSuccess) {
            cudaGetLastError();
            return ezrt_set_error(EZRT_ERR_NOMEM, "accel build: %.1f MB of device scratch", need / 1048576.0);
        }
    }
    lap("scratch allocation");
    temp = ar.take<char>(temp_bytes);
    tri_box = ar.take<Box>(n);
    for (int a = 0; a < 3; a++) keys[a] = ar.take<float>(n);
    keys_out = ar.take<float>(n);
    iota = ar.take<uint32_t>(n);
    for (int a = 0; a < 3; a++) { d.idx[a] = ar.take<uint32_t>(n); d.idx_new[a] = ar.take<uint32_t>(n); }
    d.seg = ar.take<int>(n);
    for (int a = 0; a < 3; a++) { d.L[a] = ar.take<Box>(n); d.Rrev[a] = ar.take<Box>(n); d.rank[a] = ar.take<int>(n); }
    d.side = ar.take<unsigned char>(n);
    d.nd_l = ar.take<int>(n_slots); d.nd_r = ar.take<int>(n_slots); d.nd_split = ar.take<int>(n_slots); d.used = ar.take<int>(n_slots);
    d.nd_box = ar.take<Box>(n_slots);
    d.best = ar.take<unsigned long long>(n_slots);
    d.counter = ar.take<int>(4);
    dense = ar.take<int>(n_slots);
    out_nodes = ar.take<EzrtAccelNode>(n_slots);
    d.tri_box = tri_box;

    CUB_OK(cudaMemsetAsync(d.used, 0, (size_t)n_slots * sizeof(int)));
    CUB_OK(cudaMemsetAsync(d.side, 0, (size_t)n));   // read by the partition scan for the triangles of finished leaves as well
    k_tri_boxes<<<blocks, threads>>>(d_tris, n, tri_box, keys[0], keys[1], keys[2], iota);
    for (int a = 0; a < 3; a++) {
        size_t b = temp_bytes;
        CUB_OK(cub::DeviceRadixSort::SortPairs(temp, b, (const float*)keys[a], keys_out, (const uint32_t*)iota, d.idx[a], n));
    }
    k_init_root<<<blocks, threads>>>(d);
    if (lap.on) { cudaDeviceSynchronize(); lap("boxes, three sorts"); }
    for (int level = 0;; level++) {
        levels = level + 1;
        for (int a = 0; a < 3; a++) {
            size_t b = temp_bytes;
            GatherBox g{tri_box, d.idx[a]};
            CUB_OK(cub::DeviceScan::InclusiveScanByKey(temp, b, (const int*)d.seg, BoxIt(Count(0), g), d.L[a], BoxUnion(), n));
            b = temp_bytes;
            GatherBoxRev gr{tri_box, d.idx[a], n - 1};
            KeyRev kr{d.seg, n - 1};
            CUB_OK(cub::DeviceScan::InclusiveScanByKey(temp, b, KeyRevIt(Count(0), kr), BoxRevIt(Count(0), gr), d.Rrev[a], BoxUnion(), n));
        }
        CUB_OK(cudaMemsetAsync(d.counter, 0, sizeof(int)));
        k_cost<<<blocks, threads>>>(d);
        k_split<<<blocks, threads>>>(d, level);
        for (int a = 0; a < 3; a++) {
            size_t b = temp_bytes;
            LeftFlag lf{d.side, d.idx[a]};
            CUB_OK(cub::DeviceScan::ExclusiveSumByKey(temp, b, (const int*)d.seg, FlagIt(Count(0), lf), d.rank[a], n));
        }
        k_scatter<<<blocks, threads>>>(d);
        for (int a = 0; a < 3; a++) std::swap(d.idx[a], d.idx_new[a]);
        int inner_next = 0;
        CUB_OK(cudaMemcpy(&inner_next, d.counter, sizeof(int), cudaMemcpyDeviceToHost));
        if (inner_next == 0) break;
        if (level > 4096) { rc = ezrt_set_error(EZRT_ERR_BAD_TREE, "accel build: runaway depth"); goto done; }
    }
    lap("levels");
    {
        size_t b = temp_bytes;
        CUB_OK(cub::DeviceScan::ExclusiveSum(temp, b, (const int*)d.used, dense, n_slots));
        k_emit<<<(n_slots + threads - 1) / threads, threads>>>(d, dense, n_slots, out_nodes);
        int last_dense = 0, last_used = 0;
        CUB_OK(cudaMemcpy(&last_dense, dense + n_slots - 1, sizeof(int), cudaMemcpyDeviceToHost));
        CUB_OK(cudaMemcpy(&last_used, d.used + n_slots - 1, sizeof(int), cudaMemcpyDeviceToHost));
        n_nodes = last_dense + last_used;
        nodes_out.resize(n_nodes);
        order.resize(n);
        CUB_OK(cudaMemcpy(nodes_out.data(), out_nodes, (size_t)n_nodes * sizeof(EzrtAccelNode), cudaMemcpyDeviceToHost));
        CUB_OK(cudaMemcpy(order.data(), d.idx[0], (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        CUB_OK(cudaGetLastError());
        lap("compaction, read-back");
    }
    if (levels_out) *levels_out = levels;
    rc = n_nodes;
done:
    cudaFree(ar.base);
    lap("free");
    return rc;
}
