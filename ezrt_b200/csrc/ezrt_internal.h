// ezrt_internal.h -- shared between the translation units of libezrt_b200.so (not installed).
#ifndef EZRT_INTERNAL_H
#define EZRT_INTERNAL_H

#include "ezrt.h"

#ifdef __cplusplus
extern "C" {
#endif

// records a thread-local message for ezrt_last_error() and returns `code`
int ezrt_set_error(int code, const char* fmt, ...)
#if defined(__GNUC__)
    __attribute__((format(printf, 2, 3)))
#endif
    ;

#ifdef __cplusplus
}
#endif

#ifdef __cplusplus
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <chrono>

#include <vector>
// host threads for the scene-setup stages: min(16, CPUs this process may use (affinity, cgroup cpu.max)); env EZRT_HOST_THREADS
int ezrt_host_threads();
// env EZRT_VERBOSE >= 2: wall-clock of the sub-stages of the scene setup on stderr
struct EzrtLap {
    const char* tag;
    bool on;
    std::chrono::steady_clock::time_point tp;
    explicit EzrtLap(const char* tag_) : tag(tag_), on(getenv("EZRT_VERBOSE") && atoi(getenv("EZRT_VERBOSE")) > 1), tp(std::chrono::steady_clock::now()) {}
    void operator()(const char* what) {
        if (!on) return;
        const auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[%s] %-40s %7.1f ms\n", tag, what, std::chrono::duration<double, std::milli>(now - tp).count());
        tp = now;
    }
};

// a plain array without value-initialisation: the big host arrays of the scene setup are written exactly once, by several
// threads; zero-filling them first (std::vector) costs a single-threaded pass of page faults
template <class T>
struct EzrtRawArray {
    T* p = nullptr;
    size_t n = 0;
    EzrtRawArray() {}
    EzrtRawArray(const EzrtRawArray&) = delete;
    EzrtRawArray& operator=(const EzrtRawArray&) = delete;
    ~EzrtRawArray() { free(p); }
    bool resize_uninit(size_t count) {
        free(p);
        p = count ? (T*)malloc(count * sizeof(T)) : nullptr;
        n = p ? count : 0;
        return count == 0 || p != nullptr;
    }
    void clear() { free(p); p = nullptr; n = 0; }
    T* data() { return p; }
    const T* data() const { return p; }
    size_t size() const { return n; }
    bool empty() const { return n == 0; }
    T& operator[](size_t i) { return p[i]; }
    const T& operator[](size_t i) const { return p[i]; }
};

struct EzrtAccelNode {
    int left, right, n, index;  // children (0 = none; the root is node 0 and never a child), leaf range
    float AA[3], BB[3];
};
// host_scene.cpp: sentinel-free SAH tree over the triangles of a Triangle_encoded array
int ezrt_build_accel(const float* tris, int n_tris, int leaf_n, std::vector<EzrtAccelNode>& nodes, std::vector<uint32_t>& order);

// accel_build.cu: the same tree, node for node, built on the GPU from the Triangle_encoded array in device memory (the
// current device).  Returns the node count or a negative status; *levels = depth of the tree.
int ezrt_build_accel_device(const float* d_tris, int n_tris, int leaf_n, std::vector<EzrtAccelNode>& nodes, std::vector<uint32_t>& order,
                            int* levels);

// scene_prep.cu (current device): per-triangle records from the Triangle_encoded array in device memory.
// d_geo: 4 float4 per triangle (N|d0, p1, p2, p3), d_shade: 3 float4 (n1|material id, n2, n3); info: scene bounds and
// the de-duplicated material table (ids in order of first occurrence).
struct EzrtPrepInfo {
    float max_abs = 0.0f, bmin[3] = {0, 0, 0}, bmax[3] = {0, 0, 0};
    int n_materials = 0;
    std::vector<float> materials;   // EZRT_MATERIAL_FLOATS per material
};
int ezrt_prep_records(const float* d_raw, int n, void* d_geo, void* d_shade, EzrtPrepInfo& info);
// the same records gathered into the acceleration tree's triangle order (d_order[i] = caller index of tree triangle i)
int ezrt_prep_gather(const void* d_geo, const void* d_shade, const int* d_tri_leaf, const uint32_t* d_order, int n, void* d_acc_geo,
                     void* d_acc_shade, int* d_acc_leaf, uint32_t* d_ref_to_acc);
// indexed layout of the accel-order records d_acc_geo (flat, 4 float4 per triangle): d_vid[3 i + k] = vertex id of vertex k + 1 of
// triangle i, vertices = the distinct (x, y, z) bit patterns numbered by first occurrence, d_vert_src[v] = its first position
// (both 3 n entries; n_vert of d_vert_src are written) ...
int ezrt_prep_vertex_ids(const void* d_acc_geo, int n, uint32_t* d_vid, uint32_t* d_vert_src, int& n_vert);
// ... and from them the 32-byte records (N, d0) (i1, i2, i3, 0) and the vertex array (x, y, z, 0)
int ezrt_prep_indexed(const void* d_acc_geo, int n, const uint32_t* d_vid, const uint32_t* d_vert_src, int n_vert, void* d_rec, void* d_vert);

// accel_w8.cpp: SAH-optimal collapse of the binary tree to `width`-wide nodes (dynamic programming; shared by the 4-wide
// exact-box form and the 8-wide quantised form)
struct EzrtCollapse {
    const std::vector<EzrtAccelNode>* an = nullptr;
    int width = 0;
    std::vector<int> first, count;   // per binary node: first triangle / triangle count of its sub-tree (in the binary tree's order)
    std::vector<char> as_leaf;       // per binary node: as a child of a wide node it is ONE leaf (all its triangles)
    EzrtRawArray<float> C;           // C[n * 8 + i]: cost of representing n's sub-tree by <= i roots
    int build(const std::vector<EzrtAccelNode>& an, int width, int max_leaf, double cost_node, double cost_tri, int threads = 1);
    int collect(int n0, int k0, int* roots) const;
    int children(int b, int* ch) const;   // b: an inner binary node that is not as_leaf; returns the child count (<= width)
};

// accel_w8.cpp: the 4-wide form (default of the accel kernels): 128-byte nodes with exact fp32 child boxes (8 float4: lo.xy|hi.xy
// of the four children, lo.z|hi.z pairs, four references) and the same nodes with 16-bit planes in 96 bytes (24 words, "Q16";
// empty if not wanted or if a node does not fit the grid).  Depth-first pre-order numbering, root = node `root`.
// greedy: round 1's collapse rule instead of the SAH-optimal one.  The result does not depend on `threads`.
struct EzrtW4Tree {
    EzrtRawArray<float> nodes;
    EzrtRawArray<uint32_t> q16;
    int root = 0, depth = 0;
    EzrtCollapse col;
};
int ezrt_build_w4(const std::vector<EzrtAccelNode>& an, float pad, float max_abs_coord, bool greedy, bool want_q16, int threads, EzrtW4Tree& out);

// accel_w8.cpp: the same tree collapsed to 8-wide nodes with 8-bit quantised child boxes (w8_node.h)
struct EzrtW8Tree {
    std::vector<uint32_t> nodes;       // W8_NODE_WORDS words per node; node 0 = root; breadth-first numbering
    std::vector<uint32_t> tri_order;   // triangle i of the tree = tri_order[i] of the caller's triangle array
    std::vector<int> leaf_first;       // per binary node: first triangle (new order) of that leaf, -1 for inner nodes
    int depth;                         // levels of 8-wide nodes
    int n_nodes;
    long long n_children;              // occupied slots over all nodes (fill statistics)
};
// `order_in`: triangle order of the binary tree (ezrt_build_accel); `pad`: box inflation (2 * prune_delta);
// axis_bit[a]: significance (0..2) of axis a in the slot index (largest scene extent -> bit 2); cost_tri: the collapse's price
// of a triangle test, a node visit costing 1 (the product's: W8_COST_TRI); threads: the collapse's (the result does not
// depend on them).  Returns 0 or < 0.
void ezrt_w8_axis_bits(const float bmin[3], const float bmax[3], int axis_bit[3]);
int ezrt_build_w8(const std::vector<EzrtAccelNode>& an, const std::vector<uint32_t>& order_in, float pad, float max_abs_coord,
                  const int axis_bit[3], double cost_tri, int threads, EzrtW8Tree& out);

// accel_w8.cpp: the largest |1/d_a| a quantised tree may be walked with (w8_node.h, "decode range"): a power of two, at most
// W8_INV_LIMIT, small enough that the decode's terms bias * scale * |1/d_a| and 5 * max|coordinate| * |1/d_a| stay finite for
// the largest per-axis scale of the tree.  Rays with a larger |1/d_a| go to the exact kernel.
float ezrt_quant_inv_limit(double max_scale, double bias, float max_abs_coord);
float ezrt_w8_max_scale(const uint32_t* nodes, size_t n_nodes);    // W8 records (W8_NODE_WORDS words each)
float ezrt_q16_max_scale(const uint32_t* nodes, size_t n_nodes);   // Q16 records (24 words each)
#endif

// Image partition shared by host and device code (ezrt_render_params.part_rank/part_count):
// 16x16 tiles, tile (tx,ty) -> part (tx+ty) % count; a part stores its tiles in row-major
// tile order, pixels row-major inside a tile (edge tiles are clipped).
#define EZRT_PART_TILE 16

#endif
