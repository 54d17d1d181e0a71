// accel_w8.cpp -- host builder of the 8-wide quantised acceleration tree (layout and rationale: w8_node.h).
// Input is the binary sentinel-free SAH tree of ezrt_build_accel (host_scene.cpp); this file collapses it to
// 8-wide nodes, puts the children into octant-ordered slots, renumbers the triangles so that the leaf children
// of a node are consecutive, and quantises the child boxes conservatively.  The reference has no counterpart
// (its hitBVH walks the 48-byte binary nodes, P5/fsh:254-306); results stay the reference's through the
// deferral rule of the accel policy (DESIGN.md section 4).
#include <math.h>
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <thread>
#include <utility>
#include <vector>

#include "ezrt_internal.h"
#include "w8_node.h"

namespace {

inline float box_area(const EzrtAccelNode& c) {
    const float x = c.BB[0] - c.AA[0], y = c.BB[1] - c.AA[1], z = c.BB[2] - c.AA[2];
    return x * y + x * z + y * z;
}

}  // namespace

int ezrt_host_threads() {
    if (const char* e = getenv("EZRT_HOST_THREADS")) return std::max(1, std::min(256, atoi(e)));
    int n = (int)std::thread::hardware_concurrency();
#ifdef __linux__
    cpu_set_t set;
    CPU_ZERO(&set);
    if (sched_getaffinity(0, sizeof(set), &set) == 0) n = std::min(n > 0 ? n : 1 << 20, CPU_COUNT(&set));
    if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {   // cgroup v2 quota: "<quota> <period>" or "max <period>"
        char q[64];
        long period = 0;
        if (fscanf(f, "%63s %ld", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0) n = std::min(n, (int)std::max(1L, atol(q) / period));
        fclose(f);
    }
#endif
    return std::max(1, std::min(16, n));
}

// Significance of the axes in the slot index: the axis of largest scene extent decides first (bit 2).
void ezrt_w8_axis_bits(const float bmin[3], const float bmax[3], int axis_bit[3]) {
    int idx[3] = {0, 1, 2};
    float ext[3] = {bmax[0] - bmin[0], bmax[1] - bmin[1], bmax[2] - bmin[2]};
    std::stable_sort(idx, idx + 3, [&](int a, int b) { return ext[a] < ext[b]; });  // ascending extent
    for (int k = 0; k < 3; k++) axis_bit[idx[k]] = k;
}

// Decode range of a quantised tree (w8_node.h): the decode forms A = fma(-bias, B, (origin - o) * inv) with B = scale * inv, so
// bias * scale * |inv| and |origin - o| * |inv| <= 5 max|coordinate| * |inv| must stay finite.  The limit keeps the larger of
// the two at or below 2^124, a factor 16 below the overflow threshold 2^128.
float ezrt_quant_inv_limit(double max_scale, double bias, float max_abs_coord) {
    const double m = std::max(bias * max_scale, 5.0 * (double)max_abs_coord);
    double lim = (double)W8_INV_LIMIT;
    while (lim * m > ldexp(1.0, 124) && lim > ldexp(1.0, -126)) lim *= 0.5;
    return (float)lim;
}

float ezrt_w8_max_scale(const uint32_t* nodes, size_t n_nodes) {
    uint32_t e = 0;
    for (size_t i = 0; i < n_nodes; i++)
        for (int a = 0; a < 3; a++) e = std::max(e, W8_SCALE_BITS(nodes[i * W8_NODE_WORDS + W8_W_EXP_IMASK], a));
    float s;
    memcpy(&s, &e, 4);
    return s;
}

float ezrt_q16_max_scale(const uint32_t* nodes, size_t n_nodes) {
    float s = 0.0f;
    for (size_t i = 0; i < n_nodes; i++)
        for (int a = 0; a < 3; a++) {
            float v;
            memcpy(&v, &nodes[i * 24 + 3 + a], 4);
            s = std::max(s, v);
        }
    return s;
}

// ------------------------------------------------------------------------------------------
// Optimal collapse of the binary tree to `width`-wide nodes by dynamic programming over the binary tree (surface-area
// heuristic, after Ylitie et al. 2017 section 3.1; children have larger indices than their parent):
//   C(n,1) = min(cost of n as ONE leaf (<= max_leaf triangles, consecutive), area(n) * cost_node + best split of n into <= width roots)
//   C(n,i) = min(C(n,i-1), min_k C(left,k) + C(right,i-k))          i = 2..width-1: n's sub-tree represented by <= i roots
// Visiting a wide node costs cost_node, testing one triangle cost_tri (the 8-wide form's prices: w8_node.h, W8_COST_TRI).
// ------------------------------------------------------------------------------------------
int EzrtCollapse::build(const std::vector<EzrtAccelNode>& an_, int width_, int max_leaf, double cost_node, double cost_tri, int threads) {
    an = &an_;
    width = width_;
    const int NB = (int)an_.size();
    first.assign(NB, 0);
    count.assign(NB, 0);
    as_leaf.assign(NB, 0);
    if (!C.resize_uninit((size_t)NB * 8)) return -4;
    if (width < 2 || width > 8) return -1;
    auto step = [&](int i) -> int {
        const EzrtAccelNode& nd = an_[i];
        const double area = (double)box_area(nd);
        float* c = &C[(size_t)i * 8];
        if (nd.n > 0) {
            if (nd.n > max_leaf) return -3;
            first[i] = nd.index;
            count[i] = nd.n;
            as_leaf[i] = 1;
            for (int k = 1; k <= 7; k++) c[k] = (float)(area * nd.n * cost_tri);
            return 0;
        }
        const float *cl = &C[(size_t)nd.left * 8], *cr = &C[(size_t)nd.right * 8];
        first[i] = std::min(first[nd.left], first[nd.right]);
        count[i] = count[nd.left] + count[nd.right];
        float dist[9];
        for (int j = 2; j <= width; j++) {
            float best = 3.0e38f;
            for (int k = 1; k < j; k++)
                if (k <= width - 1 && j - k <= width - 1) best = std::min(best, cl[k] + cr[j - k]);
            dist[j] = best;
        }
        const float c_internal = (float)(area * cost_node) + dist[width];
        const float c_leaf = (count[i] <= max_leaf && first[nd.left] + count[nd.left] == first[nd.right]) ? (float)(area * count[i] * cost_tri) : 3.0e38f;
        as_leaf[i] = c_leaf <= c_internal;
        c[1] = std::min(c_leaf, c_internal);
        for (int j = 2; j <= width - 1; j++) c[j] = std::min(c[j - 1], dist[j]);
        for (int j = width; j <= 7; j++) c[j] = c[width - 1];
        return 0;
    };
    // Children have larger indices than their parent and a sub-tree is one contiguous index range (pre-order): the sub-trees
    // hanging below binary depth 6 are processed on separate threads (each range backwards), then the few nodes above them.
    std::vector<std::pair<int, int>> ranges;   // [begin, end) of the sub-trees handed to threads
    std::vector<int> top;                      // nodes above them, in increasing index order
    {
        struct It { int n, end, depth; };
        std::vector<It> stk;
        stk.push_back({0, NB, 0});
        while (!stk.empty()) {
            const It it = stk.back();
            stk.pop_back();
            if (threads <= 1 || it.depth >= 6 || an_[it.n].n > 0 || it.end - it.n < 4096) { ranges.push_back({it.n, it.end}); continue; }
            top.push_back(it.n);
            stk.push_back({an_[it.n].right, it.end, it.depth + 1});
            stk.push_back({an_[it.n].left, an_[it.n].right, it.depth + 1});
        }
    }
    std::atomic<int> next(0), status(0);
    auto worker = [&]() {
        for (;;) {
            const int r = next.fetch_add(1);
            if (r >= (int)ranges.size()) return;
            for (int i = ranges[r].second - 1; i >= ranges[r].first; i--) {
                const int rc = step(i);
                if (rc) { status.store(rc); return; }
            }
        }
    };
    {
        std::vector<std::thread> pool;
        const int nt = std::max(1, std::min(threads, (int)ranges.size()));
        for (int t = 1; t < nt; t++) {
            try { pool.emplace_back(worker); } catch (...) { break; }   // no more threads: the ones we have take all the ranges
        }
        worker();
        for (auto& t : pool) t.join();
    }
    if (status.load()) return status.load();
    std::sort(top.begin(), top.end());
    for (int k = (int)top.size() - 1; k >= 0; k--) {
        const int rc = step(top[k]);
        if (rc) return rc;
    }
    return 0;
}

// roots of the best representation of sub-tree n0 by <= k0 roots (left to right)
int EzrtCollapse::collect(int n0, int k0, int* roots) const {
    const std::vector<EzrtAccelNode>& a = *an;
    struct Pick { int n, k; };
    int cnt = 0;
    Pick stack[32];
    int sp = 0;
    stack[sp++] = {n0, k0};
    while (sp > 0) {
        Pick p = stack[--sp];
        const float* c = &C[(size_t)p.n * 8];
        while (p.k > 1 && c[p.k] == c[p.k - 1]) p.k--;
        if (p.k == 1 || a[p.n].n > 0) { roots[cnt++] = p.n; continue; }
        const EzrtAccelNode& nd = a[p.n];
        const float *cl = &C[(size_t)nd.left * 8], *cr = &C[(size_t)nd.right * 8];
        int bk = 1;
        float best = 3.0e38f;
        for (int k = 1; k < p.k; k++)
            if (cl[k] + cr[p.k - k] < best) { best = cl[k] + cr[p.k - k]; bk = k; }
        stack[sp++] = {nd.right, p.k - bk};   // right first on the stack: the left roots come out first
        stack[sp++] = {nd.left, bk};
    }
    return cnt;
}

// children (binary nodes; as_leaf[] says which become leaves) of the wide node made from inner binary node b
int EzrtCollapse::children(int b, int* ch) const {
    const std::vector<EzrtAccelNode>& a = *an;
    const EzrtAccelNode& nd = a[b];
    const float *cl = &C[(size_t)nd.left * 8], *cr = &C[(size_t)nd.right * 8];
    int bk = 1;
    float best = 3.0e38f;
    for (int k = 1; k <= width - 1; k++)
        if (cl[k] + cr[width - k] < best) { best = cl[k] + cr[width - k]; bk = k; }
    int cnt = collect(nd.left, bk, ch);
    cnt += collect(nd.right, width - bk, ch + cnt);
    return cnt;
}

int ezrt_build_w8(const std::vector<EzrtAccelNode>& an, const std::vector<uint32_t>& order_in, float pad, float max_abs_coord,
                  const int axis_bit[3], double cost_tri, int threads, EzrtW8Tree& out) {
    out.nodes.clear();
    out.tri_order.clear();
    out.leaf_first.assign(an.size(), -1);
    out.depth = 0;
    out.n_nodes = 0;
    out.n_children = 0;
    if (an.empty()) return -1;
    const int NB = (int)an.size();
    const double min_step = (double)max_abs_coord * (double)W8_MIN_STEP_REL;
    EzrtCollapse col;
    const int crc = col.build(an, 8, W8_MAX_LEAF_TRIS, 1.0, cost_tri, threads);
    if (crc) return crc;
    const std::vector<int>& first = col.first;
    const std::vector<int>& count = col.count;
    const std::vector<char>& as_leaf = col.as_leaf;

    struct Item { int bnode, level; };
    std::vector<Item> queue;   // wide node i is built from queue[i] (breadth-first: a node's inner children are consecutive)
    queue.push_back({0, 1});
    out.tri_order.reserve(order_in.size());
    std::vector<int> new_pos(order_in.size(), -1);   // position in order_in -> position in the new order
    for (size_t wi = 0; wi < queue.size(); wi++) {
        const int b = queue[wi].bnode, level = queue[wi].level;
        out.depth = std::max(out.depth, level);
        // ---- the node's children: the best split of b's sub-tree into <= 8 roots
        int ch[8];
        int cnt = 0;
        if (an[b].n > 0 || (wi == 0 && as_leaf[b])) {  // the whole tree is one leaf slot
            ch[cnt++] = b;
        } else {
            cnt = col.children(b, ch);
        }
        // ---- octant-ordered slots: greedy assignment of (child, slot) pairs by dot(child centre - node centre, slot corner)
        double nlo[3] = {3.0e38, 3.0e38, 3.0e38}, nhi[3] = {-3.0e38, -3.0e38, -3.0e38};  // union of the padded child boxes (exact in double)
        for (int k = 0; k < cnt; k++)
            for (int a = 0; a < 3; a++) {
                nlo[a] = std::min(nlo[a], (double)an[ch[k]].AA[a] - (double)pad);
                nhi[a] = std::max(nhi[a], (double)an[ch[k]].BB[a] + (double)pad);
            }
        int slot_child[8];
        for (int s = 0; s < 8; s++) slot_child[s] = -1;
        {
            double cost[8][8];
            for (int k = 0; k < cnt; k++)
                for (int s = 0; s < 8; s++) {
                    double c = 0.0;
                    for (int a = 0; a < 3; a++) {
                        const double off = 0.5 * ((double)an[ch[k]].AA[a] + (double)an[ch[k]].BB[a]) - 0.5 * (nlo[a] + nhi[a]);
                        c += ((s >> axis_bit[a]) & 1) ? off : -off;
                    }
                    cost[k][s] = c;
                }
            bool child_done[8] = {false, false, false, false, false, false, false, false};
            for (int round = 0; round < cnt; round++) {
                int bk = -1, bs = -1;
                double bc = -1.0e300;
                for (int k = 0; k < cnt; k++) {
                    if (child_done[k]) continue;
                    for (int s = 0; s < 8; s++)
                        if (slot_child[s] < 0 && cost[k][s] > bc) { bc = cost[k][s]; bk = k; bs = s; }
                }
                child_done[bk] = true;
                slot_child[bs] = ch[bk];
            }
        }
        // ---- record
        uint32_t w[W8_NODE_WORDS];
        memset(w, 0, sizeof(w));
        uint8_t qlo[3][8], qhi[3][8], meta[8];
        memset(meta, 0, sizeof(meta));
        float origin[3], scale[3];
        for (int a = 0; a < 3; a++) {
            // 252 steps span the extent; the stored planes lie at least W8_SLACK_STEPS outside the exact ones (decode rounding, w8_node.h)
            double step = (nhi[a] - nlo[a]) / 252.0;
            int e;
            frexp(std::max(step, 1.0e-300), &e);            // 2^e > step
            double sc = ldexp(1.0, e);
            while (sc < min_step) sc *= 2.0;
            scale[a] = (float)sc;                            // a power of two: exact
            float org = (float)(nlo[a] - sc);
            while ((double)org > nlo[a] - sc) org = nextafterf(org, -3.0e38f);  // never above: low planes must not move up
            origin[a] = org;
            for (int s = 0; s < 8; s++) {
                const int c = slot_child[s];
                if (c < 0) { qlo[a][s] = 255; qhi[a][s] = 0; continue; }  // inverted: never hit
                const double lo = (double)an[c].AA[a] - (double)pad, hi = (double)an[c].BB[a] + (double)pad;
                double ql = floor((lo - (double)org) / sc - W8_SLACK_STEPS);
                double qh = ceil((hi - (double)org) / sc + W8_SLACK_STEPS);
                if (ql < 0.0 || qh > 255.0 || ql > qh) return -2;  // cannot happen with the 252-step rule; refuse rather than clamp
                qlo[a][s] = (uint8_t)ql;
                qhi[a][s] = (uint8_t)qh;
            }
        }
        uint32_t imask = 0;
        const uint32_t tri_base = (uint32_t)out.tri_order.size();
        const uint32_t child_base = (uint32_t)queue.size();
        for (int s = 0; s < 8; s++) {
            const int c = slot_child[s];
            if (c < 0) continue;
            out.n_children++;
            if (as_leaf[c]) {  // one leaf slot: all triangles of c's sub-tree (consecutive in order_in)
                const uint32_t off = (uint32_t)out.tri_order.size() - tri_base;
                if (count[c] > W8_MAX_LEAF_TRIS || off + (uint32_t)count[c] > W8_MAX_NODE_TRIS) return -3;
                meta[s] = (uint8_t)(((uint32_t)count[c] << 5) | off);
                for (int k = 0; k < count[c]; k++) {
                    new_pos[(size_t)first[c] + k] = (int)out.tri_order.size();
                    out.tri_order.push_back(order_in[(size_t)first[c] + k]);
                }
            } else {
                imask |= 1u << s;
                queue.push_back({c, level + 1});
            }
        }
        memcpy(&w[W8_W_ORIGIN], origin, 12);
        uint32_t exp_imask = imask << 24;
        for (int a = 0; a < 3; a++) {   // a normal power of two is its exponent byte alone
            uint32_t bits;
            memcpy(&bits, &scale[a], 4);
            if ((bits & 0x007fffffu) != 0u || (bits >> 23) == 0u || (bits >> 23) >= 255u) return -5;
            exp_imask |= (bits >> 23) << (8 * a);
        }
        w[W8_W_EXP_IMASK] = exp_imask;
        w[W8_W_CHILD_BASE] = child_base;
        w[W8_W_TRI_BASE] = tri_base;
        for (int a = 0; a < 3; a++) {
            memcpy(&w[W8_W_QLO + 2 * a], qlo[a], 8);
            memcpy(&w[W8_W_QHI + 2 * a], qhi[a], 8);
        }
        memcpy(&w[W8_W_META], meta, 8);
        out.nodes.insert(out.nodes.end(), w, w + W8_NODE_WORDS);
    }
    out.n_nodes = (int)queue.size();
    if (out.tri_order.size() != order_in.size()) return -4;
    for (int i = 0; i < NB; i++)
        if (an[i].n > 0) out.leaf_first[i] = new_pos[an[i].index];
    return 0;
}

// ------------------------------------------------------------------------------------------
// The 4-wide form (the default of the accel kernels): exact fp32 child boxes in 128-byte nodes and, beside them, the same
// nodes with 16-bit planes in 96 bytes (device_functions.cuh "Q16").  Nodes are numbered in depth-first pre-order (a
// sub-tree is contiguous in memory).  The sub-trees below wide depth 3 are built on separate threads into their own arrays
// with local numbering and spliced in pre-order, so the result does not depend on the thread count.
// ------------------------------------------------------------------------------------------
namespace {

#define W4_LEAF_FLAG 0x80000000u   // EZRT_LEAF_FLAG of device_scene.h

struct W4Ctx {
    const std::vector<EzrtAccelNode>* an;
    const EzrtCollapse* col;
    float pad;
    double q16_min_step;
    bool greedy, want_q16;
};
struct W4Part {
    std::vector<float> nodes;     // 32 floats per node
    std::vector<uint32_t> q16;    // 24 words per node (want_q16)
    int depth = 0;
    bool q16_ok = true;
};

// children of the wide node made from inner binary node b
int w4_children(const W4Ctx& cx, int b, int* ch) {
    const std::vector<EzrtAccelNode>& an = *cx.an;
    if (!cx.greedy) return cx.col->children(b, ch);
    // round 1's rule: replace the inner child of largest area by its two children until there are four
    ch[0] = an[b].left; ch[1] = an[b].right;
    int cnt = 2;
    while (cnt < 4) {
        int best = -1;
        float ba = -1.0f;
        for (int k = 0; k < cnt; k++)
            if (an[ch[k]].n <= 0 && box_area(an[ch[k]]) > ba) { ba = box_area(an[ch[k]]); best = k; }
        if (best < 0) break;
        const int c = ch[best];
        for (int k = cnt; k > best + 1; k--) ch[k] = ch[k - 1];
        ch[best] = an[c].left;
        ch[best + 1] = an[c].right;
        cnt++;
    }
    return cnt;
}
inline bool w4_is_leaf(const W4Ctx& cx, int c) { return cx.greedy ? ((*cx.an)[c].n > 0) : (cx.col->as_leaf[c] != 0); }
inline uint32_t w4_leaf_ref(const W4Ctx& cx, int c) { return W4_LEAF_FLAG | ((uint32_t)cx.col->first[c] << 7) | (uint32_t)cx.col->count[c]; }

// one node: children ch[0..cnt), refs[k] already final for leaves, any value for inner children (patched by the caller)
void w4_pack(const W4Ctx& cx, const int* ch, int cnt, const int* refs, float* rec, uint32_t* w, bool& q16_ok) {
    const std::vector<EzrtAccelNode>& an = *cx.an;
    const float pad = cx.pad;
    for (int k = 0; k < 4; k++) {
        float AA[3] = {3.0e38f, 3.0e38f, 3.0e38f}, BB[3] = {3.0e38f, 3.0e38f, 3.0e38f};  // absent: a far-away point box (min/max slab test)
        if (k < cnt) {
            const EzrtAccelNode& c = an[ch[k]];
            for (int a = 0; a < 3; a++) { AA[a] = c.AA[a] - pad; BB[a] = c.BB[a] + pad; }
        }
        rec[4 * k + 0] = AA[0]; rec[4 * k + 1] = AA[1]; rec[4 * k + 2] = BB[0]; rec[4 * k + 3] = BB[1];
        rec[16 + 2 * k] = AA[2]; rec[16 + 2 * k + 1] = BB[2];
    }
    memcpy(&rec[24], refs, 16);
    for (int k = 24 + 4; k < 32; k++) rec[k] = 0.0f;
    if (!w) return;
    memset(w, 0, sizeof(uint32_t) * 24);
    for (int a = 0; a < 3; a++) {
        double nlo = 3.0e38, nhi = -3.0e38;
        for (int k = 0; k < cnt; k++) {
            nlo = std::min(nlo, (double)an[ch[k]].AA[a] - (double)pad);
            nhi = std::max(nhi, (double)an[ch[k]].BB[a] + (double)pad);
        }
        int e;
        frexp(std::max((nhi - nlo) / 65000.0, 1.0e-300), &e);
        double sc = ldexp(1.0, e);
        while (sc < cx.q16_min_step) sc *= 2.0;
        float org = (float)(nlo - 2.0 * sc);
        while ((double)org > nlo - 2.0 * sc) org = nextafterf(org, -3.0e38f);
        const float scf = (float)sc;
        memcpy(&w[a], &org, 4);
        memcpy(&w[3 + a], &scf, 4);
        for (int k = 0; k < 4; k++) {
            uint32_t ql = 65535u, qh = 65535u;   // absent: a point at the far corner of the grid, outside every real child
            if (k < cnt) {
                const double lo = (double)an[ch[k]].AA[a] - (double)pad, hi = (double)an[ch[k]].BB[a] + (double)pad;
                const double l = floor((lo - (double)org) / sc - 1.25), h = ceil((hi - (double)org) / sc + 1.25);
                if (l < 0.0 || h > 65534.0 || l > h) q16_ok = false;
                ql = (uint32_t)std::max(0.0, l);
                qh = (uint32_t)std::min(65535.0, h);
            }
            w[6 + 3 * k + a] = ql | (qh << 16);
        }
    }
    for (int k = 0; k < 4; k++) w[18 + k] = (k < cnt) ? (uint32_t)refs[k] : (W4_LEAF_FLAG | (1u << 7));  // absent: an empty leaf, should the point ever be hit
}

// the sub-tree of inner binary node b into `out`, local pre-order numbering; returns the local id
int w4_subtree(const W4Ctx& cx, int b, int depth, W4Part& out) {
    out.depth = std::max(out.depth, depth);
    const int id = (int)(out.nodes.size() / 32);
    out.nodes.resize(out.nodes.size() + 32, 0.0f);
    if (cx.want_q16) out.q16.resize(out.q16.size() + 24, 0u);
    int ch[8] = {-1, -1, -1, -1, -1, -1, -1, -1};
    const int cnt = w4_children(cx, b, ch);
    int refs[4];
    for (int k = 0; k < 4; k++) {
        refs[k] = (int)W4_LEAF_FLAG;   // EZRT_REF_DONE, never followed
        if (k < cnt) refs[k] = w4_is_leaf(cx, ch[k]) ? (int)w4_leaf_ref(cx, ch[k]) : w4_subtree(cx, ch[k], depth + 1, out);
    }
    float rec[32];
    uint32_t w[24];
    w4_pack(cx, ch, cnt, refs, rec, cx.want_q16 ? w : nullptr, out.q16_ok);
    memcpy(&out.nodes[(size_t)id * 32], rec, sizeof(rec));
    if (cx.want_q16) memcpy(&out.q16[(size_t)id * 24], w, sizeof(w));
    return id;
}

}  // namespace

int ezrt_build_w4(const std::vector<EzrtAccelNode>& an, float pad, float max_abs_coord, bool greedy, bool want_q16, int threads, EzrtW4Tree& out) {
    out.nodes.clear();
    out.q16.clear();
    out.root = 0;
    out.depth = 0;
    if (an.empty() || an[0].n > 0) return -1;
    threads = (an.size() < 65536 && !getenv("EZRT_W4_FORCE_THREADS")) ? 1 : std::max(1, threads);   // small trees: not worth starting threads
    EzrtLap lap("ezrt_build_w4");
    int crc = out.col.build(an, 4, W8_MAX_LEAF_TRIS, 1.0, 0.3, threads);
    lap("collapse (dynamic programme)");
    if (crc) return crc;
    W4Ctx cx;
    cx.an = &an; cx.col = &out.col; cx.pad = pad;
    cx.q16_min_step = (double)max_abs_coord * (double)W8_MIN_STEP_REL;
    cx.greedy = greedy; cx.want_q16 = want_q16;
    // ---- the top of the wide tree (depth <= 3) here, every sub-tree below it as a task ----
    struct Top { int b, depth, cnt, ch[4], kind[4], arg[4]; };   // kind: 0 leaf (arg = ref), 1 top node (arg = index in tops), 2 task (arg = task)
    std::vector<Top> tops;
    std::vector<std::pair<int, int>> tasks;   // (binary node, wide depth)
    const int top_levels = (threads > 1) ? 3 : 0;
    std::vector<int> todo;
    if (top_levels == 0) {
        tasks.push_back({0, 1});
    } else {
        tops.push_back(Top());
        tops[0].b = 0; tops[0].depth = 1;
        for (size_t t = 0; t < tops.size(); t++) {
            int ch[8];
            const int cnt = w4_children(cx, tops[t].b, ch);
            tops[t].cnt = cnt;
            for (int k = 0; k < cnt; k++) {
                tops[t].ch[k] = ch[k];
                if (w4_is_leaf(cx, ch[k])) {
                    tops[t].kind[k] = 0; tops[t].arg[k] = (int)w4_leaf_ref(cx, ch[k]);
                } else if (tops[t].depth < top_levels) {
                    Top nt;
                    nt.b = ch[k]; nt.depth = tops[t].depth + 1;
                    tops[t].kind[k] = 1; tops[t].arg[k] = (int)tops.size();
                    tops.push_back(nt);   // note: invalidates references into tops
                } else {
                    tops[t].kind[k] = 2; tops[t].arg[k] = (int)tasks.size();
                    tasks.push_back({ch[k], tops[t].depth + 1});
                }
            }
        }
    }
    std::vector<W4Part> parts(tasks.size());
    {
        std::atomic<int> next(0);
        auto worker = [&]() {
            for (;;) {
                const int t = next.fetch_add(1);
                if (t >= (int)tasks.size()) return;
                w4_subtree(cx, tasks[t].first, tasks[t].second, parts[t]);
            }
        };
        std::vector<std::thread> pool;
        const int nt = std::max(1, std::min(threads, (int)tasks.size()));
        for (int t = 1; t < nt; t++) {
            try { pool.emplace_back(worker); } catch (...) { break; }   // no more threads: the ones we have take all the ranges
        }
        worker();
        for (auto& t : pool) t.join();
    }
    lap("sub-trees");
    bool q16_ok = true;
    for (const W4Part& p : parts) { out.depth = std::max(out.depth, p.depth); q16_ok = q16_ok && p.q16_ok; }
    if (top_levels == 0) {
        if (!out.nodes.resize_uninit(parts[0].nodes.size()) || !out.q16.resize_uninit(parts[0].q16.size())) return -4;
        memcpy(out.nodes.data(), parts[0].nodes.data(), parts[0].nodes.size() * sizeof(float));
        if (!parts[0].q16.empty()) memcpy(out.q16.data(), parts[0].q16.data(), parts[0].q16.size() * sizeof(uint32_t));
    } else {
        // ---- final ids in depth-first pre-order over tops and tasks ----
        std::vector<int> top_id(tops.size(), -1), task_base(tasks.size(), -1);
        int counter = 0;
        {
            struct Fr { int t, k; };
            std::vector<Fr> stk;
            top_id[0] = counter++;
            stk.push_back({0, 0});
            while (!stk.empty()) {
                Fr& f = stk.back();
                if (f.k >= tops[f.t].cnt) { stk.pop_back(); continue; }
                const int k = f.k++;
                const Top& T = tops[f.t];
                if (T.kind[k] == 1) {
                    top_id[T.arg[k]] = counter++;
                    stk.push_back({T.arg[k], 0});
                } else if (T.kind[k] == 2) {
                    task_base[T.arg[k]] = counter;
                    counter += (int)(parts[T.arg[k]].nodes.size() / 32);
                }
            }
        }
        if (!out.nodes.resize_uninit((size_t)counter * 32)) return -4;
        if (want_q16 && !out.q16.resize_uninit((size_t)counter * 24)) return -4;
        for (size_t t = 0; t < tops.size(); t++) {
            const Top& T = tops[t];
            out.depth = std::max(out.depth, T.depth);
            int refs[4];
            for (int k = 0; k < 4; k++) {
                refs[k] = (int)W4_LEAF_FLAG;
                if (k < T.cnt) refs[k] = (T.kind[k] == 0) ? T.arg[k] : (T.kind[k] == 1) ? top_id[T.arg[k]] : task_base[T.arg[k]];
            }
            w4_pack(cx, T.ch, T.cnt, refs, &out.nodes[(size_t)top_id[t] * 32], want_q16 ? &out.q16[(size_t)top_id[t] * 24] : nullptr, q16_ok);
        }
        // sub-trees: copy with the inner references moved by the base (threads again: it is a 50 MB copy)
        std::atomic<int> next(0);
        auto copier = [&]() {
            for (;;) {
                const int t = next.fetch_add(1);
                if (t >= (int)tasks.size()) return;
                const W4Part& p = parts[t];
                const int base = task_base[t], nn = (int)(p.nodes.size() / 32);
                float* dst = &out.nodes[(size_t)base * 32];
                memcpy(dst, p.nodes.data(), p.nodes.size() * sizeof(float));
                for (int i = 0; i < nn; i++) {
                    int refs[4];
                    memcpy(refs, dst + (size_t)i * 32 + 24, 16);
                    for (int k = 0; k < 4; k++)
                        if (refs[k] >= 0) refs[k] += base;
                    memcpy(dst + (size_t)i * 32 + 24, refs, 16);
                }
                if (want_q16) {
                    uint32_t* q = &out.q16[(size_t)base * 24];
                    memcpy(q, p.q16.data(), p.q16.size() * sizeof(uint32_t));
                    for (int i = 0; i < nn; i++)
                        for (int k = 0; k < 4; k++)
                            if (!(q[(size_t)i * 24 + 18 + k] & W4_LEAF_FLAG)) q[(size_t)i * 24 + 18 + k] += (uint32_t)base;
                }
            }
        };
        std::vector<std::thread> pool;
        const int nt = std::max(1, std::min(threads, (int)tasks.size()));
        for (int t = 1; t < nt; t++) {
            try { pool.emplace_back(copier); } catch (...) { break; }
        }
        copier();
        for (auto& t : pool) t.join();
    }
    lap("top and splice");
    if (!want_q16 || !q16_ok) out.q16.clear();
    return 0;
}
