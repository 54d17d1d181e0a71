// w8_model.cpp -- CPU model of the W8 acceleration-tree traversal (development + test tool; not product, not oracle).
// Builds the tree with the PRODUCT builders (ezrt_build_accel + ezrt_build_w8), then walks it with exactly the decode
// arithmetic and visit rule of the device kernel (w8_node.h, device_functions.cuh: octant-ordered hit masks, group
// stack, triangle masks) and checks every ray's closest-hit distance against brute force over all triangles
// (small scenes) or against the exact-box traversal of the binary tree (large scenes).  Prints work counts per ray, the
// triangles pending per node visit and a warp-level replay of the kernel's schedule (serial vs cooperative triangle step).
//   g++ -O2 -std=c++17 -fopenmp -ffp-contract=off -mfma -Iinclude -Iezrt_b200/csrc tools/w8_model.cpp \
//       ezrt_b200/csrc/host_scene.cpp ezrt_b200/csrc/accel_w8.cpp ezrt_b200/csrc/errors.cpp -o build/w8_model
//   build/w8_model tris.f32 n_tris rays.f32 [brute] [bundle] [sweep] [prices=N,T]   rays: 7-float records (o, d, kind) as oracle_set_ray_dump writes
//   The tree is the product's (binary leaves of W8_BINARY_LEAF_TRIS, triangle price W8_COST_TRI); sweep: the same walk on every tree of
//   binary leaf size 1, 2, 4 times collapse triangle price 0.4, 0.7, 1.0, 1.3, 1.6, then one summary line per tree.  prices=N,T: the
//   bounce kernel's measured warp cycles per node step and per triangle step (tools/bench_extend_phases.py), which turn the warp
//   replay's steps into predicted cycles per 32 bounce rays.
//   bundle: also walk every 32 consecutive rays as bundles (a ray joins the first pending ray's sub-bundle when each component of
//   its 1/d has the same sign and lies within a factor 2) -- one stack, one conservative interval test per slot for all
//   member rays, then every candidate triangle tested by every member in serial order -- and check it against the per-ray walk:
//   equal (t, triangle, tie), and every node / triangle of the per-ray walk visited / tested by the bundle.
//   The bundle bound and its arithmetic: w8_node.h "Bundle bound".  Kind-2 (shadow) rays stay out of the bundles: the camera
//   pass never traces them.
//   Kind-2 rays are walked any-hit, as extend_w8<ANYHIT = true> (k_shadow_w8) walks them: unbounded (P5's shadow rays), the first
//   strict hit ends the ray after the node it was found in, and the check is hit / miss against brute force (or the exact
//   boxes).  Their triangle tests have two totals: min, the serial order's (up to and including the first strict hit), and
//   max, every triangle pending at that node.  The kernel's cooperative step tests an owner's run of pairs at once and where
//   the run splits depends on the rays sharing the warp, so its count lies between the two; node visits are exact.
//   Machine-readable lines after the summary (integers; test_w8_tree.py, test_gpu_w8_counts.py parse them):
//     totals <camera|bounce|shadow> rays R gate G ties T visits V tests N tests_max M   (per kind: rays walked, rays left to the
//       exact kernel, rays with a tie, node visits, triangle tests; tests_max = tests except for shadow rays)
//     bundle totals bundles B members K visits V tests N   (bundle mode: (sub-)bundle node visits, member x candidate tests --
//       what extend_w8_bundle counts: one visit per warp per node, one test per member lane per candidate triangle)
//   per_ray: also "ray <index> <kind> <visits> <tests> <tests_max> <hit>" for every walked ray and (bundle mode) "bundle_at <first
//     record> <visits> <tests>" for every 32 records holding a bundle, in record order.
//   threads=a,b,...: rebuild the 8-wide tree with ezrt_build_w8 on each thread count and check that the node words, tri_order and
//     leaf_first equal those of the ezrt_host_threads() build ("threads <t>: identical" / "differs"; exit 7 if any differs).
#include <fenv.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "ezrt.h"
#include "ezrt_internal.h"
#include "ezrt_math.h"
#include "w8_node.h"

struct TriRec { ez_vec3 p1, p2, p3, N; float d0; };

// tri_test_t<TIES> of device_functions.cuh (hitTriangle P5/fsh:160-217 on the repacked record); *passed: the test got past the
// distance checks, i.e. the device loaded the vertices
static int tri_test(const TriRec& r, ez_vec3 o, ez_vec3 d, float best, float& tout, bool* passed = nullptr) {
    float nd = ez_dot(r.N, d);
    if (ez_abs(nd) < 0.00001f) return 0;
    float t = EZ_DIV(r.d0 - ez_dot(o, r.N), nd);
    if (t < 0.0005f) return 0;
    if (!(t <= best)) return 0;
    if (passed) *passed = true;
    ez_vec3 P = ez_add(o, ez_scale(d, t));
    float s1 = ez_dot(ez_cross(ez_sub(r.p2, r.p1), ez_sub(P, r.p1)), r.N);
    float s2 = ez_dot(ez_cross(ez_sub(r.p3, r.p2), ez_sub(P, r.p2)), r.N);
    float s3 = ez_dot(ez_cross(ez_sub(r.p1, r.p3), ez_sub(P, r.p3)), r.N);
    bool r1 = (s1 > 0.0f && s2 > 0.0f && s3 > 0.0f), r2 = (s1 < 0.0f && s2 < 0.0f && s3 < 0.0f);
    if (!(r1 || r2)) return 0;
    tout = t;
    return (t == best) ? 2 : 1;
}

// Warp-level replay of extend_w8's schedule (device_functions.cuh) for rays in queue order: a warp takes `chunk` rays at a
// time, refills its idle lanes when fewer than `refill` are busy, and every iteration votes for ONE step -- a node step
// (every lane holding a node visits it) or a triangle step.  Serial triangle step: one test per lane with pending triangles;
// cooperative: up to 32 (lane, triangle) pairs of all lanes, lowest lane first.  Vote: triangle step iff
// tri_w * (lanes served by a triangle step) >= lanes holding a node.  trace[r] = triangles pending after each node visit of ray r.
struct Replay { double node_steps = 0, tri_steps = 0, node_lanes = 0, tri_lanes = 0; };
static Replay replay(const std::vector<const std::vector<uint8_t>*>& trace, bool coop, int tri_w, int refill, int chunk) {
    Replay R;
    const size_t n = trace.size();
    int ray[32], vi[32], pend[32];
    for (int l = 0; l < 32; l++) ray[l] = -1;
    size_t next = 0, chunk_pos = 0, chunk_end = 0;
    bool exhausted = false;
    auto after = [&](int l) { if (pend[l] == 0 && vi[l] == (int)trace[ray[l]]->size()) ray[l] = -1; };   // nothing left: ray done
    while (true) {
        int need = 0;
        for (int l = 0; l < 32; l++) need += ray[l] < 0;
        if (need && !exhausted) {
            if (chunk_pos >= chunk_end) {
                chunk_pos = next;
                next += chunk;
                chunk_end = std::min(chunk_pos + chunk, n);
                if (chunk_pos >= n) exhausted = true;
            }
            if (!exhausted) {
                size_t idx = chunk_pos;
                for (int l = 0; l < 32; l++)
                    if (ray[l] < 0 && idx < chunk_end) { ray[l] = (int)idx++; vi[l] = 0; pend[l] = 0; }
                chunk_pos = std::min(chunk_pos + need, chunk_end);
            }
        }
        int busy = 0;
        for (int l = 0; l < 32; l++) busy += ray[l] >= 0;
        if (!busy) { if (exhausted) break; continue; }
        do {
            int nn = 0, nt = 0, pairs = 0;
            for (int l = 0; l < 32; l++)
                if (ray[l] >= 0) { nn += pend[l] == 0; nt += pend[l] > 0; pairs += pend[l]; }
            const int served = coop ? std::min(pairs, 32) : nt;
            if (nn && tri_w * served < nn) {
                R.node_steps++; R.node_lanes += nn;
                for (int l = 0; l < 32; l++)
                    if (ray[l] >= 0 && pend[l] == 0) { pend[l] = (*trace[ray[l]])[vi[l]++]; after(l); }
            } else {
                R.tri_steps++; R.tri_lanes += served;
                int slots = 32;
                for (int l = 0; l < 32; l++)
                    if (ray[l] >= 0 && pend[l] > 0) {
                        const int take = coop ? std::min(pend[l], slots) : 1;
                        slots -= take;
                        pend[l] -= take;
                        after(l);
                    }
            }
            busy = 0;
            for (int l = 0; l < 32; l++) busy += ray[l] >= 0;
        } while (busy && (exhausted || busy >= refill));
    }
    return R;
}

// the bundle bound of w8_node.h with its directed roundings (the device's __fadd_rd, __fsub_ru, __fmul_rd, ...)
static float rnd(int mode, char op, float a, float b) {
    fesetround(mode);
    volatile float x = a, y = b;
    volatile float r = op == '+' ? x + y : (op == '-' ? x - y : x * y);
    fesetround(FE_TONEAREST);
    return r;
}
static void bundle_axis(float lo, float hi, int sign, float omin, float omax, float vmin, float vmax, float& entry, float& exit) {
    if (sign == 0) { entry = -EZ_INF; exit = EZ_INF; return; }
    const bool pos = sign == 1;
    const float pn = pos ? lo : hi, pf = pos ? hi : lo;
    const float xe = pos ? rnd(FE_DOWNWARD, '-', pn, omax) : rnd(FE_UPWARD, '-', pn, omin);
    const float xx = pos ? rnd(FE_UPWARD, '-', pf, omin) : rnd(FE_DOWNWARD, '-', pf, omax);
    entry = rnd(FE_DOWNWARD, '*', xe, xe >= 0.0f ? vmin : vmax);
    exit = rnd(FE_UPWARD, '*', xx, xx >= 0.0f ? vmax : vmin);
}
struct RayResult { float t; int tri; bool tie; std::vector<int> nodes, tris; };

// what one tree's walk of the rays costs (the sweep's summary)
struct TreeStats {
    int depth = 0, n_nodes = 0, max_sp = 0;
    double nv = 0, nt = 0, npass = 0, node_steps = 0, tri_steps = 0;   // bounce rays: per ray; warp replay (cooperative step): per 32 rays
    double cam_nodes = 0, cam_cands = 0;                                // bundle mode: camera bundles' node visits, triangle candidates per 32 rays
    float inv_limit = 0.0f;
};

struct Options { bool brute = false, bundle = false, per_ray = false; std::vector<int> threads; };
static int model(const std::vector<float>& tris, int n, const std::vector<float>& rays, const Options& opt, int leaf_n, double cost_tri,
                 TreeStats& S);

int main(int argc, char** argv) {
    if (argc < 4) { fprintf(stderr, "usage: w8_model tris.f32 n_tris rays.f32 [brute] [bundle] [sweep] [per_ray] [prices=N,T] [threads=a,b,...]\n"); return 2; }
    const int n = atoi(argv[2]);
    Options opt;
    bool sweep = false;
    double price_node = 0.0, price_tri = 0.0;
    for (int i = 4; i < argc; i++) {
        opt.brute |= !strcmp(argv[i], "brute");
        opt.bundle |= !strcmp(argv[i], "bundle");
        opt.per_ray |= !strcmp(argv[i], "per_ray");
        sweep |= !strcmp(argv[i], "sweep");
        if (!strncmp(argv[i], "prices=", 7) && sscanf(argv[i] + 7, "%lf,%lf", &price_node, &price_tri) != 2) { fprintf(stderr, "prices=N,T\n"); return 2; }
        if (!strncmp(argv[i], "threads=", 8))
            for (const char* c = argv[i] + 8; *c;) {
                char* e;
                const long t = strtol(c, &e, 10);
                if (e == c || t < 1) { fprintf(stderr, "threads=a,b,...\n"); return 2; }
                opt.threads.push_back((int)t);
                c = *e == ',' ? e + 1 : e;
            }
    }
    std::vector<float> tris((size_t)n * 36);
    FILE* f = fopen(argv[1], "rb");
    if (!f || fread(tris.data(), 4, tris.size(), f) != tris.size()) { fprintf(stderr, "cannot read triangles\n"); return 1; }
    fclose(f);
    std::vector<float> rays;
    {
        FILE* rf = fopen(argv[3], "rb");
        float r[7];
        while (rf && fread(r, 4, 7, rf) == 7) rays.insert(rays.end(), r, r + 7);
        if (rf) fclose(rf);
    }
    if (!sweep) {
        TreeStats S;
        return model(tris, n, rays, opt, W8_BINARY_LEAF_TRIS, W8_COST_TRI, S);
    }
    struct Row { int leaf; double cost; TreeStats S; };
    std::vector<Row> rows;
    for (int leaf : {1, 2, 4})
        for (double cost : {0.4, 0.7, 1.0, 1.3, 1.6}) {
            printf("==== binary leaves <= %d, collapse triangle price %.1f\n", leaf, cost);
            Row r{leaf, cost, TreeStats()};
            const int rc = model(tris, n, rays, opt, leaf, cost, r.S);
            if (rc) return rc;
            rows.push_back(r);
        }
    printf("sweep: leaf, price, W8 depth, nodes, max stack, decode range; bounce rays per ray: node visits, triangle tests, distance-check "
           "passes; per 32 bounce rays: node steps, triangle steps, predicted warp cycles (prices %.1f, %.1f); camera bundles per 32 rays: "
           "node visits, triangle candidates\n", price_node, price_tri);
    for (const Row& r : rows)
        printf("sweep %d %.1f | %d %d %d %g | %.3f %.3f %.3f | %.2f %.2f %.0f | %.2f %.2f\n", r.leaf, r.cost, r.S.depth, r.S.n_nodes, r.S.max_sp,
               r.S.inv_limit, r.S.nv, r.S.nt, r.S.npass, r.S.node_steps, r.S.tri_steps, r.S.node_steps * price_node + r.S.tri_steps * price_tri,
               r.S.cam_nodes, r.S.cam_cands);
    return 0;
}

static int model(const std::vector<float>& tris, int n, const std::vector<float>& rays, const Options& opt, int leaf_n, double cost_tri,
                 TreeStats& S) {
    const bool brute = opt.brute, bundle = opt.bundle;
    const int NR = (int)(rays.size() / 7);
    float maxc = 0, bmin[3] = {3e38f, 3e38f, 3e38f}, bmax[3] = {-3e38f, -3e38f, -3e38f};
    for (int i = 0; i < n; i++)
        for (int k = 0; k < 9; k++) {
            const float v = tris[(size_t)i * 36 + k];
            maxc = fmaxf(maxc, fabsf(v));
            bmin[k % 3] = fminf(bmin[k % 3], v);
            bmax[k % 3] = fmaxf(bmax[k % 3], v);
        }
    const float delta = maxc * 1.52587890625e-05f, pad = 2.0f * delta;
    int axis_bit[3];
    ezrt_w8_axis_bits(bmin, bmax, axis_bit);

    std::vector<EzrtAccelNode> an;
    std::vector<uint32_t> order;
    ezrt_build_accel(tris.data(), n, leaf_n, an, order);
    EzrtW8Tree w8;
    const int rc = ezrt_build_w8(an, order, pad, maxc, axis_bit, cost_tri, ezrt_host_threads(), w8);
    if (rc) { fprintf(stderr, "ezrt_build_w8 failed: %d\n", rc); return 1; }
    printf("binary nodes %zu, 8-wide nodes %d (%.1f MB), depth %d, mean fill %.2f, axis bits x%d y%d z%d\n", an.size(), w8.n_nodes,
           w8.n_nodes * (double)W8_NODE_BYTES / 1e6, w8.depth, (double)w8.n_children / w8.n_nodes, axis_bit[0], axis_bit[1], axis_bit[2]);
    // the kernel's gate on |1/d_a| (capi.cu: SceneDev::quant_inv_limit)
    const float max_scale = ezrt_w8_max_scale(w8.nodes.data(), (size_t)w8.n_nodes);
    const float inv_limit = ezrt_quant_inv_limit(max_scale, W8_DECODE_BIAS, maxc);
    printf("largest node scale %g, decode range |1/d| <= %g\n", max_scale, inv_limit);
    bool threads_differ = false;
    for (int t : opt.threads) {   // the collapse's result must not depend on its thread count
        EzrtW8Tree w;
        if (ezrt_build_w8(an, order, pad, maxc, axis_bit, cost_tri, t, w)) { fprintf(stderr, "ezrt_build_w8 failed on %d threads\n", t); return 1; }
        const bool same = w.n_nodes == w8.n_nodes && w.depth == w8.depth && w.nodes == w8.nodes && w.tri_order == w8.tri_order && w.leaf_first == w8.leaf_first;
        printf("threads %d: %s\n", t, same ? "identical" : "differs");
        threads_differ |= !same;
    }
    S.depth = w8.depth;
    S.n_nodes = w8.n_nodes;
    S.inv_limit = inv_limit;
    {   // the 4-wide collapse the default kernel uses (same dynamic programme, width 4): every triangle in exactly one leaf of <= 4
        EzrtCollapse c4;
        if (c4.build(an, 4, W8_MAX_LEAF_TRIS, 1.0, 0.3) != 0) { fprintf(stderr, "4-wide collapse failed\n"); return 1; }
        std::vector<char> seen(n, 0);
        long nodes4 = 0, kids = 0, bad = 0;
        std::vector<int> todo;
        if (an[0].n <= 0 && !c4.as_leaf[0]) todo.push_back(0);
        while (!todo.empty()) {
            const int b = todo.back();
            todo.pop_back();
            int ch[8];
            const int cnt = c4.children(b, ch);
            nodes4++;
            kids += cnt;
            if (cnt < 2 || cnt > 4) bad++;
            for (int k = 0; k < cnt; k++) {
                if (c4.as_leaf[ch[k]]) {
                    if (c4.count[ch[k]] < 1 || c4.count[ch[k]] > W8_MAX_LEAF_TRIS) bad++;
                    for (int t = 0; t < c4.count[ch[k]]; t++) { if (seen[c4.first[ch[k]] + t]++) bad++; }
                } else {
                    todo.push_back(ch[k]);
                }
            }
        }
        if (nodes4 > 0) for (int i = 0; i < n; i++) if (seen[i] != 1) bad++;
        printf("4-wide collapse: %ld nodes, mean fill %.2f, violations %ld\n", nodes4, nodes4 ? (double)kids / nodes4 : 0.0, bad);
        if (bad) return 4;
    }
    std::vector<TriRec> rec(n);
    for (int i = 0; i < n; i++) {
        const float* s = &tris[(size_t)w8.tri_order[i] * 36];
        TriRec& r = rec[i];
        r.p1 = ez_v3(s[0], s[1], s[2]); r.p2 = ez_v3(s[3], s[4], s[5]); r.p3 = ez_v3(s[6], s[7], s[8]);
        r.N = ez_normalize(ez_cross(ez_sub(r.p2, r.p1), ez_sub(r.p3, r.p1)));
        r.d0 = ez_dot(r.N, r.p1);
    }

    // experiment switches (environment): W8M_SORT=1 visit hit children by entry distance instead of octant order;
    // W8M_GMIN=1 keep the smallest entry distance of a pushed group and drop the group at pop when it is beyond the best hit;
    // W8M_EXACT=1 exact child boxes instead of the quantised ones (how much the 8-bit planes cost)
    const bool x_sort = getenv("W8M_SORT") && atoi(getenv("W8M_SORT")), x_gmin = getenv("W8M_GMIN") && atoi(getenv("W8M_GMIN"));
    double nv[3] = {0, 0, 0}, nt[3] = {0, 0, 0}, npass[3] = {0, 0, 0}, npush[3] = {0, 0, 0}, cntk[3] = {0, 0, 0};
    long long tot_rays[3] = {0, 0, 0}, tot_gate[3] = {0, 0, 0}, tot_ties[3] = {0, 0, 0}, tot_nv[3] = {0, 0, 0}, tot_nt[3] = {0, 0, 0}, tot_nt_max[3] = {0, 0, 0};
    std::vector<long long> ray_nv(opt.per_ray ? NR : 0), ray_nt(opt.per_ray ? NR : 0), ray_nt_max(opt.per_ray ? NR : 0);
    std::vector<char> ray_hit(opt.per_ray ? NR : 0);
    long mismatch = 0, skipped = 0, ties = 0, hits = 0;
    int max_sp = 0;
    std::vector<std::vector<uint8_t>> trace(NR);   // triangles pending after each node visit, for the warp replay
    std::vector<int> ray_kind(NR, -1);              // -1: left to the exact kernel
    std::vector<RayResult> res(bundle ? NR : 0);    // bundle mode: the per-ray walk's result, nodes and triangles
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : mismatch, skipped, ties, hits) reduction(max : max_sp)
    for (int r = 0; r < NR; r++) {
        const float* R = &rays[(size_t)r * 7];
        const ez_vec3 o = ez_v3(R[0], R[1], R[2]), d = ez_v3(R[3], R[4], R[5]);
        const int kind = std::min(2, std::max(0, (int)R[6]));
        const float inv[3] = {EZ_DIV(1.0f, d.x), EZ_DIV(1.0f, d.y), EZ_DIV(1.0f, d.z)}, oo[3] = {o.x, o.y, o.z}, dd[3] = {d.x, d.y, d.z};
        const float ax = fabsf(inv[0]), ay = fabsf(inv[1]), az = fabsf(inv[2]);
        const float olim = W8_ORIGIN_LIMIT_REL * maxc;
        if (!(ax <= inv_limit && ay <= inv_limit && az <= inv_limit && ax >= W8_INV_MIN && ay >= W8_INV_MIN && az >= W8_INV_MIN) || !(fabsf(oo[0]) <= olim && fabsf(oo[1]) <= olim && fabsf(oo[2]) <= olim)) {
            skipped++;  // the kernel hands these to the exact traversal
#pragma omp atomic
            tot_gate[kind]++;
            continue;
        }
        ray_kind[r] = kind;
        const bool anyhit = kind == 2;
        long long my_nt_max = -1;   // any-hit: tests up to the end of the node of the first strict hit (-1: no hit yet)
        const float slack = delta * fmaxf(ax, fmaxf(ay, az));
        uint32_t near_mask = 0;
        for (int a = 0; a < 3; a++) if (dd[a] >= 0.0f) near_mask |= 1u << axis_bit[a];
        float best = EZ_INF;
        bool tie = false;
        int best_tri = -1;
        struct Group { uint32_t base, bits; float tmin; uint32_t order; float ts[8]; } st[64];
        float g_ts[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const bool x_tsel = getenv("W8M_TSEL") && atoi(getenv("W8M_TSEL"));  // per-child entry distance kept with the group (ideal pop pruning)
        const bool x_exact = getenv("W8M_EXACT") && atoi(getenv("W8M_EXACT"));
        float g_tmin = 0.0f;
        uint32_t g_order = 0;   // W8M_SORT: slots in visit order, 4 bits each, first = lowest nibble
        int sp = 0;
        uint32_t g_base = 0, g_bits = 0;   // bits: imask (low 8) | hits in priority positions (bits 8..15)
        int node = 0;
        double my_nv = 0, my_nt = 0, my_pass = 0, my_push = 0;
        while (true) {
            uint32_t t_base = 0, t_mask = 0;
            if (node >= 0) {
                const uint32_t* w = &w8.nodes[(size_t)node * W8_NODE_WORDS];
                my_nv += 1;
                if (bundle) res[r].nodes.push_back(node);
                const float limit = best + (best * 0.000244140625f + slack);
                float A[3], B[3];
                for (int a = 0; a < 3; a++) {
                    float org, sc;
                    const uint32_t sc_bits = W8_SCALE_BITS(w[W8_W_EXP_IMASK], a);
                    memcpy(&org, &w[W8_W_ORIGIN + a], 4);
                    memcpy(&sc, &sc_bits, 4);
                    B[a] = sc * inv[a];
                    A[a] = fmaf(-W8_DECODE_BIAS, B[a], (org - oo[a]) * inv[a]);
                }
                const uint8_t* qlo = (const uint8_t*)&w[W8_W_QLO];
                const uint8_t* qhi = (const uint8_t*)&w[W8_W_QHI];
                const uint8_t* meta = (const uint8_t*)&w[W8_W_META];
                const uint32_t imask = w[W8_W_EXP_IMASK] >> 24;
                uint32_t hits8 = 0;
                float tmin_s[8];
                for (int s = 0; s < 8; s++) {
                    float tn[3], tf[3];
                    for (int a = 0; a < 3; a++) {
                        const uint8_t lo = qlo[8 * a + s], hi = qhi[8 * a + s];
                        const uint8_t nr = dd[a] >= 0.0f ? lo : hi, fr = dd[a] >= 0.0f ? hi : lo;
                        tn[a] = fmaf(W8_DECODE_BIAS + (float)nr + (x_exact ? (dd[a] >= 0.0f ? 1.5f : -1.5f) : 0.0f), B[a], A[a]);
                        tf[a] = fmaf(W8_DECODE_BIAS + (float)fr + (x_exact ? (dd[a] >= 0.0f ? -1.5f : 1.5f) : 0.0f), B[a], A[a]);
                    }
                    const float tmin = fmaxf(fmaxf(tn[0], tn[1]), fmaxf(tn[2], 0.0f));
                    const float tmax = fminf(fminf(tf[0], tf[1]), fminf(tf[2], limit));
                    if (tmin <= tmax) hits8 |= 1u << s;
                    tmin_s[s] = tmin;
                }
                uint32_t inner = hits8 & imask, leaf = hits8 & ~imask, perm = 0;
                for (int s = 0; s < 8; s++) if (inner >> s & 1) perm |= 1u << (s ^ near_mask);
                for (int s = 0; s < 8; s++)
                    if (leaf >> s & 1) t_mask |= ((1u << (meta[s] >> 5)) - 1u) << (meta[s] & 31u);
                t_base = w[W8_W_TRI_BASE];
                trace[r].push_back((uint8_t)__builtin_popcount(t_mask));
                if (g_bits >> 8) { st[sp].base = g_base; st[sp].bits = g_bits; st[sp].tmin = g_tmin; st[sp].order = g_order; memcpy(st[sp].ts, g_ts, sizeof(g_ts)); sp++; my_push += 1; max_sp = std::max(max_sp, sp); }
                g_base = w[W8_W_CHILD_BASE];
                g_bits = imask | (perm << 8);
                g_tmin = 3.0e38f;
                for (int s = 0; s < 8; s++) if (inner >> s & 1) g_tmin = fminf(g_tmin, tmin_s[s]);
                memcpy(g_ts, tmin_s, sizeof(g_ts));
                if (x_sort) {  // hit inner slots by ascending entry distance; bits 8.. = slot mask (unpermuted)
                    int idx[8], m = 0;
                    for (int s = 0; s < 8; s++) if (inner >> s & 1) idx[m++] = s;
                    std::sort(idx, idx + m, [&](int a, int b) { return tmin_s[a] < tmin_s[b]; });
                    g_order = 0;
                    for (int k = m - 1; k >= 0; k--) g_order = (g_order << 4) | (uint32_t)idx[k];
                    g_bits = imask | (inner << 8);
                }
            }
            const long long node_end = (long long)my_nt + __builtin_popcount(t_mask);
            while (t_mask) {  // the node's triangles, lowest offset first
                const int k = __builtin_ctz(t_mask);
                t_mask &= t_mask - 1;
                my_nt += 1;
                float t;
                bool passed = false;
                const int h = tri_test(rec[t_base + k], o, d, best, t, &passed);
                my_pass += passed ? 1 : 0;
                if (bundle) res[r].tris.push_back((int)(t_base + k));
                if (h == 2) tie = true;
                else if (h == 1) { best = t; tie = false; best_tri = (int)(t_base + k); }
                if (anyhit && h == 1) { my_nt_max = node_end; break; }   // the first strict hit ends a shadow ray
            }
            if (my_nt_max >= 0) break;
            bool done = false;
            while ((g_bits >> 8) == 0) {
                if (sp == 0) { done = true; break; }
                --sp;
                g_base = st[sp].base;
                g_bits = st[sp].bits;
                g_tmin = st[sp].tmin;
                g_order = st[sp].order;
                memcpy(g_ts, st[sp].ts, sizeof(g_ts));
                if (x_gmin && g_tmin > best + (best * 0.000244140625f + slack)) g_bits &= 255u;  // the whole group lies beyond the best hit
            }
            if (done) break;
            int slot;
            if (x_sort) {
                slot = (int)(g_order & 15u);
                g_order >>= 4;
                g_bits ^= 1u << (8 + slot);
            } else {
                const int p = 31 - __builtin_clz(g_bits >> 8);      // highest priority position
                g_bits ^= 1u << (8 + p);
                slot = p ^ (int)near_mask;
            }
            if (x_tsel && g_ts[slot] > best + (best * 0.000244140625f + slack)) { node = -1; continue; }
            if (x_gmin) {  // entry distance of what stays behind in the group (model: exact minimum over the remaining hit slots)
                // NOTE: needs the t values of the node the group came from; the model keeps them only for the node just visited,
                // so the minimum is taken when the group is created (below) and is a lower bound afterwards
            }
            node = (int)(g_base + __builtin_popcount(g_bits & 255u & ((1u << slot) - 1u)));
        }
        if (tie) ties++;
        if (bundle) { res[r].t = best; res[r].tri = best_tri; res[r].tie = tie; }
        // ---- check
        float want = EZ_INF;
        if (brute) {
            for (int i = 0; i < n; i++) { float t; if (tri_test(rec[i], o, d, want, t) != 0) want = t; }
        } else {  // exact (padded) boxes of the binary tree, pruned
            int stk[128], sp2 = 0, cur = 0;
            while (true) {
                const EzrtAccelNode& nd = an[cur];
                bool descend = false;
                if (nd.n > 0) {
                    const int first = w8.leaf_first[cur];
                    for (int k = 0; k < nd.n; k++) { float t; if (tri_test(rec[first + k], o, d, want, t) != 0) want = t; }
                } else {
                    const float limit = want + (want * 0.000244140625f + slack);
                    int c[2] = {nd.left, nd.right};
                    bool hit[2];
                    for (int j = 0; j < 2; j++) {
                        float t0 = -3e38f, t1 = 3e38f;
                        for (int a = 0; a < 3; a++) {
                            const float ta = ((an[c[j]].AA[a] - pad) - oo[a]) * inv[a], tb = ((an[c[j]].BB[a] + pad) - oo[a]) * inv[a];
                            t0 = fmaxf(t0, fminf(ta, tb)); t1 = fminf(t1, fmaxf(ta, tb));
                        }
                        hit[j] = t1 >= t0 && t1 > 0.0f && !(t0 > limit);
                    }
                    if (hit[0] && hit[1]) { stk[sp2++] = c[1]; cur = c[0]; descend = true; }
                    else if (hit[0]) { cur = c[0]; descend = true; }
                    else if (hit[1]) { cur = c[1]; descend = true; }
                }
                if (descend) continue;
                if (sp2 == 0) break;
                cur = stk[--sp2];
            }
        }
        if (anyhit ? (want < EZ_INF) != (best < EZ_INF) : memcmp(&want, &best, 4) != 0) mismatch++;
        if (want < EZ_INF) hits++;
        if (my_nt_max < 0) my_nt_max = (long long)my_nt;
        if (opt.per_ray) { ray_nv[r] = (long long)my_nv; ray_nt[r] = (long long)my_nt; ray_nt_max[r] = my_nt_max; ray_hit[r] = best < EZ_INF; }
#pragma omp critical
        {
            nv[kind] += my_nv; nt[kind] += my_nt; npass[kind] += my_pass; npush[kind] += my_push; cntk[kind] += 1;
            tot_rays[kind]++; tot_ties[kind] += tie; tot_nv[kind] += (long long)my_nv; tot_nt[kind] += (long long)my_nt; tot_nt_max[kind] += my_nt_max;
        }
    }
    const char* names[3] = {"camera", "bounce", "shadow"};
    if (cntk[1] > 0) { S.nv = nv[1] / cntk[1]; S.nt = nt[1] / cntk[1]; S.npass = npass[1] / cntk[1]; }
    S.max_sp = max_sp;
    for (int k = 0; k < 3; k++)
        if (cntk[k] > 0)
            printf("%s rays %.0f: %.2f node visits, %.2f triangle tests, %.2f pushes per ray; %.3f of the tests pass the distance checks\n", names[k], cntk[k],
                   nv[k] / cntk[k], nt[k] / cntk[k], npush[k] / cntk[k], nt[k] > 0 ? npass[k] / nt[k] : 0.0);
    for (int k = 0; k < 3; k++)   // 128-bit loads of the device kernel: five per node visit, one per triangle test and three per vertex stage
        if (cntk[k] > 0)
            printf("%s rays: %.1f 16-byte loads per ray (%.1f with the 96-byte node and the 64-byte triangle loaded whole)\n", names[k],
                   (W8_NODE_BYTES / 16 * nv[k] + nt[k] + 3 * npass[k]) / cntk[k], (6 * nv[k] + 4 * nt[k]) / cntk[k]);
    for (int k = 0; k < 3; k++) {   // triangles pending per node visit that pends any
        long hist[W8_MAX_NODE_TRIS + 1] = {0}, visits = 0;
        for (int r = 0; r < NR; r++)
            if (ray_kind[r] == k)
                for (uint8_t c : trace[r]) { hist[c]++; visits++; }
        long pending = 0, sum = 0;
        for (int c = 1; c <= W8_MAX_NODE_TRIS; c++) { pending += hist[c]; sum += (long)c * hist[c]; }
        if (!pending) continue;
        printf("%s rays: %.3f of the node visits pend triangles, %.2f on average; distribution", names[k], (double)pending / visits, (double)sum / pending);
        for (int c = 1; c <= W8_MAX_NODE_TRIS; c++)
            if (hist[c]) printf(" %d:%.3f", c, (double)hist[c] / pending);
        printf("\n");
    }
    // the replay uses the device's defaults (capi.cu: w8_tri_weight, refill_thresh, work_chunk); W8M_TRI_W / W8M_REFILL override
    // (the serial step is replayed with its own tuned weight, 2)
    const int tri_w = getenv("W8M_TRI_W") ? atoi(getenv("W8M_TRI_W")) : 1, refill = getenv("W8M_REFILL") ? atoi(getenv("W8M_REFILL")) : 24;
    for (int k = 0; k < 3; k++) {
        std::vector<const std::vector<uint8_t>*> q;
        for (int r = 0; r < NR; r++)
            if (ray_kind[r] == k) q.push_back(&trace[r]);
        if (q.size() < 32) continue;
        for (int coop = 0; coop < 2; coop++) {
            const Replay R = replay(q, coop != 0, coop ? tri_w : 2, refill, 32);
            const double per = 32.0 / q.size();
            if (k == 1 && coop) { S.node_steps = R.node_steps * per; S.tri_steps = R.tri_steps * per; }
            printf("%s rays, warp replay, %s triangle step (tri_w %d, refill %d): per 32 rays %.1f node steps (%.1f lanes busy), "
                   "%.1f triangle steps (%.1f lanes busy); 2 x node + triangle steps = %.1f\n", names[k], coop ? "cooperative" : "serial", coop ? tri_w : 2, refill,
                   R.node_steps * per, R.node_lanes / R.node_steps, R.tri_steps * per, R.tri_lanes / R.tri_steps, (2 * R.node_steps + R.tri_steps) * per);
        }
    }
    if (bundle) {   // 32 consecutive rays, one stack, one bundle test per slot, serial triangle tests per member (see the top of the file)
        long b_nodes = 0, b_cands = 0, b_tests = 0, r_tests = 0, n_members = 0, n_bundles = 0, bad_result = 0, bad_nodes = 0, bad_tris = 0;
        std::vector<long long> at_nv(opt.per_ray ? (NR + 31) / 32 : 0), at_nt(at_nv.size());   // per_ray: per 32 records
#pragma omp parallel for schedule(dynamic, 4) reduction(+ : b_nodes, b_cands, b_tests, r_tests, n_members, n_bundles, bad_result, bad_nodes, bad_tris)
        for (int b0 = 0; b0 < NR; b0 += 32) {
            const int nb = std::min(32, NR - b0);
            int pend[32], np_ = 0;
            for (int j = 0; j < nb; j++) if (ray_kind[b0 + j] >= 0 && ray_kind[b0 + j] != 2) pend[np_++] = b0 + j;
            // sub-bundles: a ray joins the first pending ray's when every component of its 1/d has the leader's sign and lies
            // within a factor 2 of the leader's (extend_w8_bundle)
            while (np_ > 0) {
            int mem[32], nm = 0, rest = 0;
            float lead[3];
            for (int a = 0; a < 3; a++) lead[a] = EZ_DIV(1.0f, rays[(size_t)pend[0] * 7 + 3 + a]);
            for (int k = 0; k < np_; k++) {
                bool in = true;
                for (int a = 0; a < 3; a++) {
                    const float v = EZ_DIV(1.0f, rays[(size_t)pend[k] * 7 + 3 + a]), w = lead[a];
                    in = in && (v > 0.0f) == (w > 0.0f) && fabsf(v) <= 2.0f * fabsf(w) && fabsf(w) <= 2.0f * fabsf(v);
                }
                if (in) mem[nm++] = pend[k]; else pend[rest++] = pend[k];
            }
            np_ = rest;
            n_bundles++;
            float bo[3][4];   // per axis: omin, omax, vmin, vmax
            int sign[3];
            float best[32], slack[32], inv[32][3];
            int btri[32];
            bool tie[32];
            for (int a = 0; a < 3; a++) { bo[a][0] = INFINITY; bo[a][1] = -INFINITY; bo[a][2] = INFINITY; bo[a][3] = -INFINITY; }
            int npos[3] = {0, 0, 0};
            for (int k = 0; k < nm; k++) {
                const float* R = &rays[(size_t)mem[k] * 7];
                for (int a = 0; a < 3; a++) {
                    inv[k][a] = EZ_DIV(1.0f, R[3 + a]);
                    bo[a][0] = fminf(bo[a][0], R[a]); bo[a][1] = fmaxf(bo[a][1], R[a]);
                    bo[a][2] = fminf(bo[a][2], inv[k][a]); bo[a][3] = fmaxf(bo[a][3], inv[k][a]);
                    npos[a] += R[3 + a] >= 0.0f;
                }
                slack[k] = delta * fmaxf(fabsf(inv[k][0]), fmaxf(fabsf(inv[k][1]), fabsf(inv[k][2])));
                best[k] = EZ_INF; btri[k] = -1; tie[k] = false;
            }
            for (int a = 0; a < 3; a++) sign[a] = npos[a] == nm ? 1 : (npos[a] == 0 ? 2 : 0);
            uint32_t near_mask = 0;
            for (int a = 0; a < 3; a++) if (rays[(size_t)mem[0] * 7 + 3 + a] >= 0.0f) near_mask |= 1u << axis_bit[a];
            std::vector<int> vis, cand;
            float L = EZ_INF;
            uint32_t st_base[64], st_bits[64];
            int sp = 0;
            uint32_t node = 0, g_base = 0, g_bits = 0;
            while (true) {
                const uint32_t* w = &w8.nodes[(size_t)node * W8_NODE_WORDS];
                vis.push_back((int)node);
                const uint8_t* qlo = (const uint8_t*)&w[W8_W_QLO];
                const uint8_t* qhi = (const uint8_t*)&w[W8_W_QHI];
                const uint8_t* meta = (const uint8_t*)&w[W8_W_META];
                uint32_t hits = 0;
                for (int sl = 0; sl < 8; sl++) {
                    float en[3], ex[3];
                    for (int a = 0; a < 3; a++) {
                        float org, sc;
                        const uint32_t sc_bits = W8_SCALE_BITS(w[W8_W_EXP_IMASK], a);
                        memcpy(&org, &w[W8_W_ORIGIN + a], 4);
                        memcpy(&sc, &sc_bits, 4);
                        const float lo = rnd(FE_DOWNWARD, '+', org, ((float)qlo[8 * a + sl] - 0.25f) * sc);
                        const float hi = rnd(FE_UPWARD, '+', org, ((float)qhi[8 * a + sl] + 0.25f) * sc);
                        bundle_axis(lo, hi, sign[a], bo[a][0], bo[a][1], bo[a][2], bo[a][3], en[a], ex[a]);
                    }
                    if (fmaxf(fmaxf(en[0], en[1]), fmaxf(en[2], 0.0f)) <= fminf(fminf(ex[0], ex[1]), fminf(ex[2], L))) hits |= 1u << sl;
                }
                const uint32_t imask = w[W8_W_EXP_IMASK] >> 24, inner = hits & imask;
                uint32_t leaf = hits & ~imask, perm = 0, t_mask = 0;
                for (int sl = 0; sl < 8; sl++) if (inner >> sl & 1) perm |= 1u << (sl ^ near_mask);
                if (g_bits >> 8) { st_base[sp] = g_base; st_bits[sp] = g_bits; sp++; }
                g_base = w[W8_W_CHILD_BASE];
                g_bits = imask | (perm << 8);
                for (int sl = 0; sl < 8; sl++) if (leaf >> sl & 1) t_mask |= ((1u << (meta[sl] >> 5)) - 1u) << (meta[sl] & 31u);
                if (t_mask) {
                    while (t_mask) {
                        const int tri = (int)w[W8_W_TRI_BASE] + __builtin_ctz(t_mask);
                        t_mask &= t_mask - 1;
                        cand.push_back(tri);
                        for (int k = 0; k < nm; k++) {
                            const float* R = &rays[(size_t)mem[k] * 7];
                            float t;
                            const int h = tri_test(rec[tri], ez_v3(R[0], R[1], R[2]), ez_v3(R[3], R[4], R[5]), best[k], t);
                            if (h == 2) tie[k] = true;
                            else if (h == 1) { best[k] = t; btri[k] = tri; tie[k] = false; }
                        }
                    }
                    L = 0.0f;
                    for (int k = 0; k < nm; k++) L = fmaxf(L, best[k] + (best[k] * 0.000244140625f + slack[k]));
                }
                if ((g_bits >> 8) == 0) {
                    if (sp == 0) break;
                    --sp;
                    g_base = st_base[sp];
                    g_bits = st_bits[sp];
                }
                const int p = 31 - __builtin_clz(g_bits >> 8);
                g_bits ^= 1u << (8 + p);
                const uint32_t slot = (uint32_t)p ^ near_mask;
                node = g_base + (uint32_t)__builtin_popcount(g_bits & 255u & ((1u << slot) - 1u));
            }
            b_nodes += (long)vis.size();
            b_cands += (long)cand.size();
            b_tests += (long)cand.size() * nm;
            if (opt.per_ray) { at_nv[b0 / 32] += (long long)vis.size(); at_nt[b0 / 32] += (long long)cand.size() * nm; }
            n_members += nm;
            std::sort(vis.begin(), vis.end());
            std::sort(cand.begin(), cand.end());
            for (int k = 0; k < nm; k++) {
                const RayResult& q = res[mem[k]];
                r_tests += (long)q.tris.size();
                if (memcmp(&q.t, &best[k], 4) != 0 || q.tie != tie[k] || (!q.tie && q.tri != btri[k])) bad_result++;
                for (int x : q.nodes) if (!std::binary_search(vis.begin(), vis.end(), x)) { bad_nodes++; break; }
                for (int x : q.tris) if (!std::binary_search(cand.begin(), cand.end(), x)) { bad_tris++; break; }
            }
            }
        }
        if (n_members > 0) {
            const double per32 = 32.0 / n_members;
            S.cam_nodes = b_nodes * per32;
            S.cam_cands = b_cands * per32;
            printf("bundle: %ld (sub-)bundles, %ld member rays; per 32 rays %.2f node visits, %.2f triangle candidates; (ray, triangle) tests per ray %.2f "
                   "(per-ray walk %.2f); warp steps per 32 rays %.2f node + %.2f triangle\n", n_bundles, n_members, b_nodes * per32, b_cands * per32,
                   (double)b_tests / n_members, (double)r_tests / n_members, b_nodes * per32, b_cands * per32);
            printf("bundle checks: results differing %ld, rays with a node missing %ld, rays with a triangle missing %ld\n", bad_result, bad_nodes, bad_tris);
        }
        printf("bundle totals bundles %ld members %ld visits %ld tests %ld\n", n_bundles, n_members, b_nodes, b_tests);
        for (size_t b = 0; b < at_nv.size(); b++)
            if (at_nv[b]) printf("bundle_at %zu %lld %lld\n", 32 * b, at_nv[b], at_nt[b]);
        if (n_members > 0) {
            if (bad_result) return 6;
            if (bad_nodes || bad_tris) return 5;
        }
    }
    printf("max stack depth %d, rays left to the exact kernel %ld, rays with a tie %ld\n", max_sp, skipped, ties);
    printf("closest-hit distances differing from %s: %ld of %d rays (%ld of them hit)\n", brute ? "brute force" : "the exact-box traversal", mismatch, NR, hits);
    for (int k = 0; k < 3; k++)
        printf("totals %s rays %lld gate %lld ties %lld visits %lld tests %lld tests_max %lld\n", names[k], tot_rays[k], tot_gate[k], tot_ties[k], tot_nv[k],
               tot_nt[k], tot_nt_max[k]);
    if (opt.per_ray)
        for (int r = 0; r < NR; r++)
            if (ray_kind[r] >= 0) printf("ray %d %d %lld %lld %lld %d\n", r, ray_kind[r], ray_nv[r], ray_nt[r], ray_nt_max[r], (int)ray_hit[r]);
    if (mismatch) return 3;
    return threads_differ ? 7 : 0;
}
