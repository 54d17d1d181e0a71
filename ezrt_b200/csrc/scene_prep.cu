// scene_prep.cu -- the per-triangle part of ezrt_scene_create on the GPU: from the caller's Triangle_encoded array (36 floats
// per triangle, P5/main.cpp:60-69, :843-861) in device memory to the records the kernels read (device_scene.h), the run
// structure of the materials (for the de-duplicated material table), the scene bounds, and the same records gathered into
// the acceleration tree's triangle order.  Replaces ~120 ms of single-threaded host loops and ~350 MB of uploads at 1 M
// triangles by one 144 MB upload and four kernels.
//
// The arithmetic is the host's: N = normalize(cross(p2 - p1, p3 - p1)) and d0 = dot(N, p1) with the ezrt_math.h primitives
// (hitTriangle, P5/fsh:172, :184), compiled -fmad=false.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <cub/cub.cuh>
#include <map>
#include <string>
#include <vector>

#include "ezrt.h"
#include "ezrt_internal.h"
#include "ezrt_math.h"

namespace {

// total order on floats as unsigned integers (-0.0 below +0.0)
__device__ __forceinline__ uint32_t f2ord(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord2f(uint32_t o) {
    const uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}

// bounds[0] = max |coordinate| (float bits), [1..3] = min xyz (ordered), [4..6] = max xyz (ordered)
__global__ void k_records(const float* __restrict__ raw, int n, float4* __restrict__ geo, float4* __restrict__ shade, int* __restrict__ head,
                          uint32_t* __restrict__ bounds) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t amax = 0u, lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0u, 0u, 0u};
    if (i < n) {
        const float* s = raw + (size_t)i * EZRT_TRIANGLE_FLOATS;
        float v[18];
#pragma unroll
        for (int k = 0; k < 18; k++) v[k] = s[k];
        const ez_vec3 p1 = ez_v3(v[0], v[1], v[2]), p2 = ez_v3(v[3], v[4], v[5]), p3 = ez_v3(v[6], v[7], v[8]);
#pragma unroll
        for (int k = 0; k < 9; k++) {
            const float x = v[k];
            if (x == x) {   // the host's `<` updates skip NaN
                const uint32_t a = __float_as_uint(x) & 0x7fffffffu;
                amax = max(amax, a);
                const uint32_t o = f2ord(x);
                lo[k % 3] = min(lo[k % 3], o);
                hi[k % 3] = max(hi[k % 3], o);
            }
        }
        const ez_vec3 N = ez_normalize(ez_cross(ez_sub(p2, p1), ez_sub(p3, p1)));   // hitTriangle, P5/fsh:172
        const float d0 = ez_dot(N, p1);                                              // P5/fsh:184
        geo[(size_t)i * 4 + 0] = make_float4(N.x, N.y, N.z, d0);   // first: the distance checks of tri_test_t read only this
        geo[(size_t)i * 4 + 1] = make_float4(p1.x, p1.y, p1.z, 0.0f);
        geo[(size_t)i * 4 + 2] = make_float4(p2.x, p2.y, p2.z, 0.0f);
        geo[(size_t)i * 4 + 3] = make_float4(p3.x, p3.y, p3.z, 0.0f);
        shade[(size_t)i * 3 + 0] = make_float4(v[9], v[10], v[11], 0.0f);
        shade[(size_t)i * 3 + 1] = make_float4(v[12], v[13], v[14], 0.0f);
        shade[(size_t)i * 3 + 2] = make_float4(v[15], v[16], v[17], 0.0f);
        // first triangle of a run of equal materials (bit comparison, as the host's byte-string key)
        int h = (i == 0) ? 1 : 0;
        if (i > 0) {
            const uint32_t* m = (const uint32_t*)(s + 18);
            const uint32_t* q = m - EZRT_TRIANGLE_FLOATS;
#pragma unroll
            for (int k = 0; k < EZRT_MATERIAL_FLOATS; k++) h |= (m[k] != q[k]) ? 1 : 0;
        }
        head[i] = h;
    }
    // block reduction of the bounds, one atomic per block and value
    typedef cub::BlockReduce<uint32_t, 256> Reduce;
    __shared__ typename Reduce::TempStorage tmp;
    uint32_t r = Reduce(tmp).Reduce(amax, cub::Max());
    if (threadIdx.x == 0) atomicMax(&bounds[0], r);
    for (int k = 0; k < 3; k++) {
        __syncthreads();
        r = Reduce(tmp).Reduce(lo[k], cub::Min());
        if (threadIdx.x == 0) atomicMin(&bounds[1 + k], r);
        __syncthreads();
        r = Reduce(tmp).Reduce(hi[k], cub::Max());
        if (threadIdx.x == 0) atomicMax(&bounds[4 + k], r);
    }
}

// run[i] = inclusive sum of head = 1-based index of i's run; the heads copy their material out
__global__ void k_head_materials(const float* __restrict__ raw, int n, const int* __restrict__ head, const int* __restrict__ run,
                                 float* __restrict__ head_mat) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !head[i]) return;
    const float* m = raw + (size_t)i * EZRT_TRIANGLE_FLOATS + 18;
    float* o = head_mat + (size_t)(run[i] - 1) * EZRT_MATERIAL_FLOATS;
    for (int k = 0; k < EZRT_MATERIAL_FLOATS; k++) o[k] = m[k];
}

__global__ void k_assign_material(float4* __restrict__ shade, int n, const int* __restrict__ run, const int* __restrict__ head_id) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ((int*)&shade[(size_t)i * 3])[3] = head_id[run[i] - 1];
}

__global__ void k_gather(const float4* __restrict__ geo, const float4* __restrict__ shade, const int* __restrict__ tri_leaf,
                         const uint32_t* __restrict__ order, int n, float4* __restrict__ acc_geo, float4* __restrict__ acc_shade,
                         int* __restrict__ acc_leaf, uint32_t* __restrict__ ref_to_acc) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t r = order[i];
#pragma unroll
    for (int k = 0; k < 4; k++) acc_geo[(size_t)i * 4 + k] = geo[(size_t)r * 4 + k];
#pragma unroll
    for (int k = 0; k < 3; k++) acc_shade[(size_t)i * 3 + k] = shade[(size_t)r * 3 + k];
    acc_leaf[i] = tri_leaf[r];
    ref_to_acc[r] = (uint32_t)i;
}

// Vertex de-duplication of the accel-order records.  Position j = 3 i + k is vertex k + 1 of triangle i (acc_geo[4 i + 1 + k]);
// positions are equal iff their (x, y, z) BIT PATTERNS are (+0 and -0 differ, NaNs are equal only with the same payload), and the
// vertices are numbered by first occurrence in j.  Two stable radix sorts (z, then x:y) order the positions by key with equal
// keys in ascending j, so the head of every run of equal keys is its first occurrence.
__device__ __forceinline__ uint4 pos_bits(const float4* __restrict__ acc_geo, uint32_t j) {
    const float4 p = acc_geo[(size_t)(j / 3u) * 4 + 1 + j % 3u];
    return make_uint4(__float_as_uint(p.x), __float_as_uint(p.y), __float_as_uint(p.z), 0u);
}
__global__ void k_pos_z(const float4* __restrict__ acc_geo, uint32_t m, uint32_t* __restrict__ key_z, uint32_t* __restrict__ idx) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    key_z[j] = pos_bits(acc_geo, j).z;
    idx[j] = j;
}
__global__ void k_pos_xy(const float4* __restrict__ acc_geo, uint32_t m, const uint32_t* __restrict__ idx, unsigned long long* __restrict__ key_xy) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    const uint4 b = pos_bits(acc_geo, idx[p]);
    key_xy[p] = ((unsigned long long)b.x << 32) | b.y;
}
// head[p] = 1 iff sorted position p starts a run of equal keys; first[j] = 1 iff position j is that run's first occurrence
__global__ void k_pos_heads(const float4* __restrict__ acc_geo, uint32_t m, const uint32_t* __restrict__ idx, uint32_t* __restrict__ head,
                            uint32_t* __restrict__ first) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    const uint32_t j = idx[p];
    bool h = p == 0;
    if (!h) {
        const uint4 a = pos_bits(acc_geo, j), b = pos_bits(acc_geo, idx[p - 1]);
        h = a.x != b.x || a.y != b.y || a.z != b.z;
    }
    head[p] = h ? 1u : 0u;
    if (h) first[j] = 1u;
}
// num = exclusive scan of first (vertex id of every first occurrence), run = inclusive scan of head (1-based run of p)
__global__ void k_run_ids(uint32_t m, const uint32_t* __restrict__ idx, const uint32_t* __restrict__ head, const uint32_t* __restrict__ run,
                          const uint32_t* __restrict__ num, uint32_t* __restrict__ run_vid, uint32_t* __restrict__ vert_src) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m || !head[p]) return;
    const uint32_t j = idx[p], v = num[j];
    run_vid[run[p] - 1] = v;
    vert_src[v] = j;
}
__global__ void k_vertex_ids(uint32_t m, const uint32_t* __restrict__ idx, const uint32_t* __restrict__ run, const uint32_t* __restrict__ run_vid,
                             uint32_t* __restrict__ vid) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    vid[idx[p]] = run_vid[run[p] - 1];
}
// indexed records (N, d0) (i1, i2, i3, 0) and the vertex array (x, y, z, 0)
__global__ void k_indexed(const float4* __restrict__ acc_geo, int n, const uint32_t* __restrict__ vid, float4* __restrict__ rec) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    rec[(size_t)i * 2] = acc_geo[(size_t)i * 4];
    rec[(size_t)i * 2 + 1] = make_float4(__uint_as_float(vid[(size_t)i * 3]), __uint_as_float(vid[(size_t)i * 3 + 1]), __uint_as_float(vid[(size_t)i * 3 + 2]), 0.0f);
}
__global__ void k_vertices(const float4* __restrict__ acc_geo, uint32_t n_vert, const uint32_t* __restrict__ vert_src, float4* __restrict__ vert) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n_vert) return;
    const uint32_t j = vert_src[v];
    const float4 p = acc_geo[(size_t)(j / 3u) * 4 + 1 + j % 3u];
    vert[v] = make_float4(p.x, p.y, p.z, 0.0f);
}

}  // namespace

#define PREP_OK(call)                                                                                           \
    do {                                                                                                         \
        cudaError_t e_ = (call);                                                                                 \
        if (e_ != cudaSuccess) {                                                                                 \
            rc = ezrt_set_error(EZRT_ERR_CUDA, "scene prep: %s: %s", #call, cudaGetErrorString(e_));             \
            goto done;                                                                                           \
        }                                                                                                        \
    } while (0)

int ezrt_prep_records(const float* d_raw, int n, void* d_geo, void* d_shade, EzrtPrepInfo& info) {
    int rc = EZRT_OK;
    EzrtLap lap("ezrt_prep_records");
    const int threads = 256, blocks = (n + threads - 1) / threads;
    char* scratch = nullptr;
    int* head = nullptr;
    int* run = nullptr;
    uint32_t* bounds = nullptr;
    float* head_mat = nullptr;
    int* head_id = nullptr;
    void* temp = nullptr;
    size_t temp_bytes = 0;
    uint32_t hb[8];
    int n_heads = 0;
    const size_t N = (size_t)n;
    cub::DeviceScan::InclusiveSum(nullptr, temp_bytes, (const int*)nullptr, (int*)nullptr, n);
    const size_t off_run = (N * 4 + 255) / 256 * 256, off_bounds = off_run * 2, off_temp = off_bounds + 256;
    PREP_OK(cudaMalloc((void**)&scratch, off_temp + temp_bytes + 256));
    head = (int*)scratch; run = (int*)(scratch + off_run); bounds = (uint32_t*)(scratch + off_bounds); temp = scratch + off_temp;
    {
        const uint32_t init[8] = {0u, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u, 0u};
        PREP_OK(cudaMemcpy(bounds, init, sizeof(init), cudaMemcpyHostToDevice));
    }
    lap("scratch allocation");
    k_records<<<blocks, threads>>>(d_raw, n, (float4*)d_geo, (float4*)d_shade, head, bounds);
    PREP_OK(cub::DeviceScan::InclusiveSum(temp, temp_bytes, (const int*)head, run, n));
    PREP_OK(cudaMemcpy(&n_heads, run + (n - 1), sizeof(int), cudaMemcpyDeviceToHost));
    PREP_OK(cudaMemcpy(hb, bounds, sizeof(hb), cudaMemcpyDeviceToHost));
    {
        uint32_t a = hb[0];
        memcpy(&info.max_abs, &a, 4);
        for (int k = 0; k < 3; k++) {
            // the host loop starts from +-3.0e38 and only moves on `<`: values beyond stay clamped there
            const float lo = ord2f(hb[1 + k]), hi = ord2f(hb[4 + k]);
            info.bmin[k] = (hb[1 + k] != 0xffffffffu && lo < 3.0e38f) ? lo : 3.0e38f;
            info.bmax[k] = (hb[4 + k] != 0u && hi > -3.0e38f) ? hi : -3.0e38f;
        }
    }
    lap("records kernel, run scan, bounds read-back");
    // material table: the run heads in order, de-duplicated on the host (ids in order of first occurrence, as the host map did)
    PREP_OK(cudaMalloc((void**)&head_mat, (size_t)n_heads * EZRT_MATERIAL_FLOATS * sizeof(float)));
    k_head_materials<<<blocks, threads>>>(d_raw, n, head, run, head_mat);
    {
        std::vector<float> hm((size_t)n_heads * EZRT_MATERIAL_FLOATS);
        PREP_OK(cudaMemcpy(hm.data(), head_mat, hm.size() * sizeof(float), cudaMemcpyDeviceToHost));
        std::vector<int> ids(n_heads);
        std::map<std::string, int> seen;
        info.materials.clear();
        for (int h = 0; h < n_heads; h++) {
            const float* m = &hm[(size_t)h * EZRT_MATERIAL_FLOATS];
            std::string key((const char*)m, sizeof(float) * EZRT_MATERIAL_FLOATS);
            auto it = seen.find(key);
            if (it == seen.end()) {
                ids[h] = (int)seen.size();
                seen.emplace(key, ids[h]);
                info.materials.insert(info.materials.end(), m, m + EZRT_MATERIAL_FLOATS);
            } else {
                ids[h] = it->second;
            }
        }
        info.n_materials = (int)seen.size();
        PREP_OK(cudaMalloc((void**)&head_id, (size_t)n_heads * sizeof(int)));
        PREP_OK(cudaMemcpy(head_id, ids.data(), (size_t)n_heads * sizeof(int), cudaMemcpyHostToDevice));
    }
    k_assign_material<<<blocks, threads>>>((float4*)d_shade, n, run, head_id);
    PREP_OK(cudaDeviceSynchronize());
    lap("materials");
done:
    cudaFree(scratch);
    cudaFree(head_mat);
    cudaFree(head_id);
    return rc;
}

int ezrt_prep_gather(const void* d_geo, const void* d_shade, const int* d_tri_leaf, const uint32_t* d_order, int n, void* d_acc_geo,
                     void* d_acc_shade, int* d_acc_leaf, uint32_t* d_ref_to_acc) {
    const int threads = 256, blocks = (n + threads - 1) / threads;
    k_gather<<<blocks, threads>>>((const float4*)d_geo, (const float4*)d_shade, d_tri_leaf, d_order, n, (float4*)d_acc_geo, (float4*)d_acc_shade,
                                  d_acc_leaf, d_ref_to_acc);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return ezrt_set_error(EZRT_ERR_CUDA, "scene prep: gather: %s", cudaGetErrorString(e));
    return EZRT_OK;
}

int ezrt_prep_vertex_ids(const void* d_acc_geo, int n, uint32_t* d_vid, uint32_t* d_vert_src, int& n_vert) {
    int rc = EZRT_OK;
    const uint32_t m = 3u * (uint32_t)n;
    const int threads = 256, blocks = (int)((m + threads - 1) / threads);
    const float4* geo = (const float4*)d_acc_geo;
    char* scratch = nullptr;
    size_t t_sort_z = 0, t_sort_xy = 0, t_scan = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, t_sort_z, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)m);
    cub::DeviceRadixSort::SortPairs(nullptr, t_sort_xy, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)m);
    cub::DeviceScan::InclusiveSum(nullptr, t_scan, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)m);
    const size_t temp_bytes = std::max(t_sort_z, std::max(t_sort_xy, t_scan));
    const size_t a4 = ((size_t)m * 4 + 255) / 256 * 256, a8 = 2 * a4;
    // u32 arrays: key_z, key_z_sorted, idx0, idx1, idx2, head, run, first, num, run_vid; u64: key_xy, key_xy_sorted
    PREP_OK(cudaMalloc((void**)&scratch, 10 * a4 + 2 * a8 + temp_bytes + 256));
    {
        uint32_t* key_z = (uint32_t*)scratch;
        uint32_t* key_z_s = (uint32_t*)(scratch + a4);
        uint32_t* idx0 = (uint32_t*)(scratch + 2 * a4);
        uint32_t* idx1 = (uint32_t*)(scratch + 3 * a4);
        uint32_t* idx2 = (uint32_t*)(scratch + 4 * a4);
        uint32_t* head = (uint32_t*)(scratch + 5 * a4);
        uint32_t* run = (uint32_t*)(scratch + 6 * a4);
        uint32_t* first = (uint32_t*)(scratch + 7 * a4);
        uint32_t* num = (uint32_t*)(scratch + 8 * a4);
        uint32_t* run_vid = (uint32_t*)(scratch + 9 * a4);
        unsigned long long* key_xy = (unsigned long long*)(scratch + 10 * a4);
        unsigned long long* key_xy_s = (unsigned long long*)(scratch + 10 * a4 + a8);
        void* temp = scratch + 10 * a4 + 2 * a8;
        size_t tb = temp_bytes;
        uint32_t last[2] = {0u, 0u};
        k_pos_z<<<blocks, threads>>>(geo, m, key_z, idx0);
        PREP_OK(cub::DeviceRadixSort::SortPairs(temp, tb, key_z, key_z_s, idx0, idx1, (int)m));
        k_pos_xy<<<blocks, threads>>>(geo, m, idx1, key_xy);
        tb = temp_bytes;
        PREP_OK(cub::DeviceRadixSort::SortPairs(temp, tb, key_xy, key_xy_s, idx1, idx2, (int)m));   // stable: equal keys stay in ascending j
        PREP_OK(cudaMemset(first, 0, (size_t)m * 4));
        k_pos_heads<<<blocks, threads>>>(geo, m, idx2, head, first);
        tb = temp_bytes;
        PREP_OK(cub::DeviceScan::InclusiveSum(temp, tb, head, run, (int)m));
        tb = temp_bytes;
        PREP_OK(cub::DeviceScan::ExclusiveSum(temp, tb, first, num, (int)m));
        PREP_OK(cudaMemcpy(&last[0], num + (m - 1), 4, cudaMemcpyDeviceToHost));
        PREP_OK(cudaMemcpy(&last[1], first + (m - 1), 4, cudaMemcpyDeviceToHost));
        n_vert = (int)(last[0] + last[1]);
        k_run_ids<<<blocks, threads>>>(m, idx2, head, run, num, run_vid, d_vert_src);
        k_vertex_ids<<<blocks, threads>>>(m, idx2, run, run_vid, d_vid);
        PREP_OK(cudaDeviceSynchronize());
    }
done:
    cudaFree(scratch);
    return rc;
}

int ezrt_prep_indexed(const void* d_acc_geo, int n, const uint32_t* d_vid, const uint32_t* d_vert_src, int n_vert, void* d_rec, void* d_vert) {
    const int threads = 256;
    k_indexed<<<(n + threads - 1) / threads, threads>>>((const float4*)d_acc_geo, n, d_vid, (float4*)d_rec);
    k_vertices<<<(n_vert + threads - 1) / threads, threads>>>((const float4*)d_acc_geo, (uint32_t)n_vert, d_vert_src, (float4*)d_vert);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return ezrt_set_error(EZRT_ERR_CUDA, "scene prep: indexed records: %s", cudaGetErrorString(e));
    return EZRT_OK;
}
