// light_tree.cpp -- the light tree of EZRT_PARAM_LIGHT_TREE (ezrt_math.h, DESIGN.md section 19): a binary tree over the lights of a
// light table, built on the host in one deterministic pass.  The renders upload this function's output unchanged.
//
// Split: binned power-weighted SAH.  Each node's lights are binned by centroid into 16 equal bins along each axis of the centroids'
// bounds; the split between bins minimising phi_L * area(box_L) + phi_R * area(box_R) (float64) over the three axes wins, the lowest
// axis and bin on ties.  A node whose centroids coincide, whose best split leaves one side empty, or that lies 32 levels deep or more
// is split at the median of its lights ordered by (centroid along the centroids' widest axis, light index) -- so the depth is at most
// 32 + ceil(log2 K) <= 64 for every K < 2^31.  Leaves hold one light each.
#include <math.h>

#include <algorithm>
#include <vector>

#include "ezrt_internal.h"
#include "ezrt_math.h"

namespace {

constexpr int kBins = 16;
constexpr int kSahDepth = 32;

struct Builder {
    const float* verts;
    const float* w;
    std::vector<double> cen, nrm;   // per light: the centroid and the unit geometric normal (float64)
    std::vector<int> idx;           // the lights, reordered in place by the splits
    float* nodes;                   // 12 floats per node
    uint32_t* paths;                // 4 words per light: path bits (low, high), depth, area
    int next = 1;                   // the next free node pair

    void leaf_or_split(int node, int b, int e, int depth, uint64_t path) {
        float* nd = nodes + 12 * (size_t)node;
        // bounds, power and cone of lights idx[b, e)
        float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
        double phi = 0.0, ax[3] = {0.0, 0.0, 0.0};
        const double* n0 = &nrm[3 * (size_t)idx[b]];
        for (int i = b; i < e; i++) {
            const int k = idx[i];
            for (int v = 0; v < 3; v++)
                for (int c = 0; c < 3; c++) {
                    lo[c] = std::min(lo[c], verts[9 * (size_t)k + 3 * v + c]);
                    hi[c] = std::max(hi[c], verts[9 * (size_t)k + 3 * v + c]);
                }
            phi += (double)w[k];
            const double* n = &nrm[3 * (size_t)k];
            const double s = (n[0] * n0[0] + n[1] * n0[1] + n[2] * n0[2] < 0.0) ? -1.0 : 1.0;   // lines: orient towards the first
            for (int c = 0; c < 3; c++) ax[c] += s * n[c];
        }
        double len = sqrt(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]);
        float a[3];
        for (int c = 0; c < 3; c++) a[c] = (len > 0.0) ? (float)(ax[c] / len) : (c == 2 ? 1.0f : 0.0f);
        double cmin = 1.0;   // the cone: the least |dot(N_k, a)| over the lights, with the fp32 axis as stored
        for (int i = b; i < e; i++) {
            const double* n = &nrm[3 * (size_t)idx[i]];
            cmin = std::min(cmin, fabs(n[0] * a[0] + n[1] * a[1] + n[2] * a[2]));
        }
        // stored rounded down, with a margin for normals computed in another order
        float cos_o = (float)(cmin - 1e-6);
        if ((double)cos_o > cmin - 1e-6) cos_o = nextafterf(cos_o, -INFINITY);
        cos_o = std::max(cos_o, 0.0f);
        for (int c = 0; c < 3; c++) {
            nd[c] = lo[c];
            nd[4 + c] = hi[c];
            nd[8 + c] = a[c];
        }
        nd[3] = (float)phi;
        nd[7] = cos_o;
        if (e - b == 1) {
            const int k = idx[b];
            nd[11] = ez_u2f((uint32_t)~k);
            paths[4 * (size_t)k] = (uint32_t)path;
            paths[4 * (size_t)k + 1] = (uint32_t)(path >> 32);
            paths[4 * (size_t)k + 2] = (uint32_t)depth;
            const float* p = verts + 9 * (size_t)k;
            paths[4 * (size_t)k + 3] = ez_f2u(ez_triangle_area(ez_v3(p[0], p[1], p[2]), ez_v3(p[3], p[4], p[5]), ez_v3(p[6], p[7], p[8])));
            return;
        }
        const int m = split(b, e, depth);
        const int c = next;
        next += 2;
        nd[11] = ez_u2f((uint32_t)c);
        leaf_or_split(c, b, m, depth + 1, path);
        leaf_or_split(c + 1, m, e, depth + 1, path | ((uint64_t)1 << depth));
    }

    // reorders idx[b, e) and returns the first index of the right child, b < m < e
    int split(int b, int e, int depth) {
        double clo[3] = {INFINITY, INFINITY, INFINITY}, chi[3] = {-INFINITY, -INFINITY, -INFINITY};
        for (int i = b; i < e; i++)
            for (int c = 0; c < 3; c++) {
                clo[c] = std::min(clo[c], cen[3 * (size_t)idx[i] + c]);
                chi[c] = std::max(chi[c], cen[3 * (size_t)idx[i] + c]);
            }
        if (depth < kSahDepth) {
            double best = INFINITY;
            int best_axis = -1, best_bin = -1;
            for (int ax = 0; ax < 3; ax++) {
                const double ext = chi[ax] - clo[ax];
                if (!(ext > 0.0)) continue;
                double blo[kBins][3], bhi[kBins][3], bphi[kBins];
                int bn[kBins];
                for (int j = 0; j < kBins; j++) {
                    bphi[j] = 0.0;
                    bn[j] = 0;
                    for (int c = 0; c < 3; c++) { blo[j][c] = INFINITY; bhi[j][c] = -INFINITY; }
                }
                for (int i = b; i < e; i++) {
                    const int k = idx[i];
                    const int j = bin_of(cen[3 * (size_t)k + ax], clo[ax], ext);
                    bphi[j] += (double)w[k];
                    bn[j]++;
                    for (int v = 0; v < 3; v++)
                        for (int c = 0; c < 3; c++) {
                            blo[j][c] = std::min(blo[j][c], (double)verts[9 * (size_t)k + 3 * v + c]);
                            bhi[j][c] = std::max(bhi[j][c], (double)verts[9 * (size_t)k + 3 * v + c]);
                        }
                }
                // suffix sums of the right side, then a sweep of the left
                double rcost[kBins];
                double rlo[3] = {INFINITY, INFINITY, INFINITY}, rhi[3] = {-INFINITY, -INFINITY, -INFINITY}, rphi = 0.0;
                int rn = 0;
                for (int j = kBins - 1; j >= 1; j--) {
                    rphi += bphi[j];
                    rn += bn[j];
                    for (int c = 0; c < 3; c++) { rlo[c] = std::min(rlo[c], blo[j][c]); rhi[c] = std::max(rhi[c], bhi[j][c]); }
                    rcost[j] = rn ? rphi * area(rlo, rhi) : INFINITY;
                }
                double llo[3] = {INFINITY, INFINITY, INFINITY}, lhi[3] = {-INFINITY, -INFINITY, -INFINITY}, lphi = 0.0;
                int ln = 0;
                for (int j = 0; j < kBins - 1; j++) {
                    lphi += bphi[j];
                    ln += bn[j];
                    for (int c = 0; c < 3; c++) { llo[c] = std::min(llo[c], blo[j][c]); lhi[c] = std::max(lhi[c], bhi[j][c]); }
                    if (!ln || ln == e - b) continue;
                    const double cost = lphi * area(llo, lhi) + rcost[j + 1];
                    if (cost < best) { best = cost; best_axis = ax; best_bin = j; }
                }
            }
            if (best_axis >= 0) {
                const double lo = clo[best_axis], ext = chi[best_axis] - clo[best_axis];
                const int* mid = std::stable_partition(idx.data() + b, idx.data() + e, [&](int k) {
                    return bin_of(cen[3 * (size_t)k + best_axis], lo, ext) <= best_bin;
                });
                const int m = (int)(mid - idx.data());
                if (m > b && m < e) return m;
            }
        }
        int ax = 0;
        for (int c = 1; c < 3; c++)
            if (chi[c] - clo[c] > chi[ax] - clo[ax]) ax = c;
        std::sort(idx.begin() + b, idx.begin() + e, [&](int x, int y) {
            const double cx = cen[3 * (size_t)x + ax], cy = cen[3 * (size_t)y + ax];
            return (cx < cy) || (cx == cy && x < y);
        });
        return b + (e - b) / 2;
    }

    static int bin_of(double x, double lo, double ext) {
        const int j = (int)((x - lo) / ext * kBins);
        return std::min(std::max(j, 0), kBins - 1);
    }
    static double area(const double* lo, const double* hi) {
        const double dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
        return 2.0 * (dx * dy + dy * dz + dz * dx);
    }
};

}  // namespace

int ezrt_light_tree_build(int n, const float* verts, const float* weights, int cap, float* nodes_out, uint32_t* paths_out) {
    if (n < 0 || (n > 0 && (!verts || !weights))) return ezrt_set_error(EZRT_ERR_INVALID, "light_tree_build: bad argument");
    for (int k = 0; k < n; k++)
        if (!ez_is_light(weights[k])) return ezrt_set_error(EZRT_ERR_INVALID, "light_tree_build: light %d has weight %g (not finite and > 0)", k, weights[k]);
    for (size_t i = 0; i < 9 * (size_t)n; i++)
        if (!ez_finite(verts[i])) return ezrt_set_error(EZRT_ERR_INVALID, "light_tree_build: vertex coordinate %zu is not finite", i);
    if (n == 0) return 0;
    const int M = 2 * n - 1;
    if (cap < M || !nodes_out || !paths_out) return M;   // the size only
    Builder bd;
    bd.verts = verts;
    bd.w = weights;
    bd.nodes = nodes_out;
    bd.paths = paths_out;
    bd.cen.resize(3 * (size_t)n);
    bd.nrm.resize(3 * (size_t)n);
    bd.idx.resize(n);
    for (int k = 0; k < n; k++) {
        const float* p = verts + 9 * (size_t)k;
        double e1[3], e2[3];
        for (int c = 0; c < 3; c++) {
            bd.cen[3 * (size_t)k + c] = ((double)p[c] + (double)p[3 + c] + (double)p[6 + c]) / 3.0;
            e1[c] = (double)p[3 + c] - (double)p[c];
            e2[c] = (double)p[6 + c] - (double)p[c];
        }
        double N[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
        const double len = sqrt(N[0] * N[0] + N[1] * N[1] + N[2] * N[2]);
        for (int c = 0; c < 3; c++) bd.nrm[3 * (size_t)k + c] = (len > 0.0) ? N[c] / len : 0.0;
        bd.idx[k] = k;
    }
    bd.leaf_or_split(0, 0, n, 0, 0);
    return M;
}
