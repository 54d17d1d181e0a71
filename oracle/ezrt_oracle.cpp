// ezrt_oracle.cpp -- CPU ORACLE of EzRT's per-pixel path-tracing inner loop.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT.  Only tests/, __graft_entry__.smoke() and bench.py's
// *** cpu_baseline / --impl reference legs may load this library.  ezrt_b200 never does.
//
// PARITY PIN.  The reference (AKGWSB/EzRT @51cf8774) ships no test, golden vector or known-answer
// value for this path (SURVEY.md 4, 8c) and its hot path is a GLSL fragment shader that needs an
// OpenGL 4.3 context plus glm/GLEW/freeglut (none installed, no network).  What pins this file:
//   1. the reference's OWN SHADER SOURCE run on the CPU: oracle/ref_shader/ transpiles
//      P3|P4|P5/shaders/fshader.fsh from where they lie (literal suffixes, swizzle accessors,
//      qualifiers -- statements, expression order, control flow, constants and tables untouched)
//      and this file must equal it bit for bit in all four integrator modes
//      (tests/test_ref_shader.py; frames committed in tests/golden/refshader.npz);
//   2. constants: wang_hash chain, Sobol/Joe-Kuo points, PI literal (tests/test_kat.py), and the one
//      ray of P2/main.cpp:581-586 (BVH result == brute force).
// What stays OURS by definition, because GLSL does not specify it bit-wise: the built-in functions
// (-> include/ezrt_math.h), texture filtering, the rasteriser's `pix` and the left-to-right
// evaluation of call arguments (list below).  Both sides of pin 1 share those definitions.
// This file is a plain scalar C++ restatement of the reference's algorithm, function by function,
// each citing the file:line it follows
// (P2/ P3/ P4/ P5/ = "source code" directory of tutorial part 2..5, fsh = shaders/fshader.fsh).
//
// Arithmetic is the normative fp32 definition of include/ezrt_math.h (GLSL built-ins are not
// bit-specified), compiled with -ffp-contract=off -mfma so it is comparable bit-for-bit with
// the CUDA kernels, which are written separately (ezrt_b200/csrc/*.cu) against the same
// primitives.
//
// Fixed conventions where the reference leaves a choice (SURVEY.md 8b):
//   - pixel (px,py), py = 0 bottom row:  pix = ((px+.5)/W*2-1, (py+.5)/H*2-1); the seed terms
//     uint((pix.x*.5+.5)*width) are px / py; lastFrame is read at the pixel's own texel.
//   - GLSL evaluates call arguments left to right (SampleHdr(rand(), rand()), AA).
//   - texture2D: fp32 bilinear with texel centres at +0.5 and CLAMP_TO_EDGE (P5), or nearest
//     (P3/P4), selected by hdr_linear.
//   - the material of a hit is fetched once for the final closest hit (the shader re-fetches on
//     every improvement, P5/fsh:245-248; same value).
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "ezrt.h"
#include "ezrt_math.h"

#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

typedef ez_vec3 vec3;

struct Material {  // P5/fsh:50-65
    vec3 emissive, baseColor;
    float subsurface, metallic, specular, specularTint, roughness, anisotropic, sheen, sheenTint, clearcoat,
        clearcoatGloss, IOR, transmission;
};
struct Ray {  // P5/fsh:68-71
    vec3 startPoint, direction;
};
struct HitResult {  // P5/fsh:74-82
    bool isHit, isInside;
    float distance;
    vec3 hitPoint, normal, viewDir;
    int triangle;  // index of the triangle (stands for `material`, fetched by getMaterial at the end)
};
struct BVHNode {  // P5/fsh:41-47
    int left, right, n, index;
    vec3 AA, BB;
};

struct Counters {
    uint64_t rays[3];    // primary, bounce, shadow
    uint64_t nodes;      // N_node: nodes fetched (popped + children tested), SURVEY 8d
    uint64_t tris;       // N_tri : triangles tested
    uint64_t hits;       // H     : rays that hit
    uint64_t hdr_lookups;
    uint64_t max_stack;
    uint64_t innerByDepth[64];  // inner-node visits by tree depth (root = 0)
};

struct Scene {
    const float* tris; int nTriangles;
    const float* nodes; int nNodes;
    const float* hdr; const float* hdrCache; int hdrW, hdrH; int hdrLinear;
    vec3 envColor;
    int mode;       // ezrt_mode
    int traverse;   // ezrt_traverse
    float pruneDelta;  // absolute slack of the pruned policy (DESIGN.md "pruning")
};

// ---------------------------------------------------------------- decode, P5/fsh:93-155
inline vec3 texel(const float* base, int i) { return ez_v3(base[3 * i], base[3 * i + 1], base[3 * i + 2]); }

struct Triangle { vec3 p1, p2, p3, n1, n2, n3; };

inline Triangle getTriangle(const Scene& sc, int i) {
    int offset = i * 12;
    Triangle t;
    t.p1 = texel(sc.tris, offset + 0); t.p2 = texel(sc.tris, offset + 1); t.p3 = texel(sc.tris, offset + 2);
    t.n1 = texel(sc.tris, offset + 3); t.n2 = texel(sc.tris, offset + 4); t.n3 = texel(sc.tris, offset + 5);
    return t;
}
inline Material getMaterial(const Scene& sc, int i) {
    int offset = i * 12;
    Material m;
    vec3 param1 = texel(sc.tris, offset + 8), param2 = texel(sc.tris, offset + 9);
    vec3 param3 = texel(sc.tris, offset + 10), param4 = texel(sc.tris, offset + 11);
    m.emissive = texel(sc.tris, offset + 6);
    m.baseColor = texel(sc.tris, offset + 7);
    m.subsurface = param1.x; m.metallic = param1.y; m.specular = param1.z;
    m.specularTint = param2.x; m.roughness = param2.y; m.anisotropic = param2.z;
    m.sheen = param3.x; m.sheenTint = param3.y; m.clearcoat = param3.z;
    m.clearcoatGloss = param4.x; m.IOR = param4.y; m.transmission = param4.z;
    return m;
}
inline BVHNode getBVHNode(const Scene& sc, int i) {
    int offset = i * 4;
    BVHNode node;
    vec3 childs = texel(sc.nodes, offset + 0), leafInfo = texel(sc.nodes, offset + 1);
    node.left = (int)childs.x; node.right = (int)childs.y;
    node.n = (int)leafInfo.x; node.index = (int)leafInfo.y;
    node.AA = texel(sc.nodes, offset + 2);
    node.BB = texel(sc.nodes, offset + 3);
    return node;
}

// ---------------------------------------------------------------- hitTriangle
// P5/fsh:160-217 (GLSL), P2/main.cpp:212-238 (C++ twin), P3/fsh:228-282 (normal fudge variant)
HitResult hitTriangle(const Triangle& triangle, const Ray& ray, bool p3Fudge) {
    HitResult res;
    res.distance = EZ_INF;
    res.isHit = false;
    res.isInside = false;
    res.triangle = -1;
    res.hitPoint = res.normal = res.viewDir = ez_v3(0, 0, 0);

    vec3 p1 = triangle.p1, p2 = triangle.p2, p3 = triangle.p3;
    vec3 S = ray.startPoint, d = ray.direction;
    vec3 N = ez_normalize(ez_cross(ez_sub(p2, p1), ez_sub(p3, p1)));
    if (ez_dot(N, d) > 0.0f) {
        N = ez_neg(N);
        res.isInside = true;
    }
    if (ez_abs(ez_dot(N, d)) < 0.00001f) return res;
    float t = EZ_DIV(ez_dot(N, p1) - ez_dot(S, N), ez_dot(d, N));
    if (t < 0.0005f) return res;
    vec3 P = ez_add(S, ez_scale(d, t));
    vec3 c1 = ez_cross(ez_sub(p2, p1), ez_sub(P, p1));
    vec3 c2 = ez_cross(ez_sub(p3, p2), ez_sub(P, p2));
    vec3 c3 = ez_cross(ez_sub(p1, p3), ez_sub(P, p3));
    bool r1 = (ez_dot(c1, N) > 0 && ez_dot(c2, N) > 0 && ez_dot(c3, N) > 0);
    bool r2 = (ez_dot(c1, N) < 0 && ez_dot(c2, N) < 0 && ez_dot(c3, N) < 0);
    if (r1 || r2) {
        res.isHit = true;
        res.hitPoint = P;
        res.distance = t;
        res.normal = N;
        res.viewDir = d;
        float alpha, beta;
        if (!p3Fudge) {  // P5/fsh:206-207
            alpha = EZ_DIV((-(P.x - p2.x)) * (p3.y - p2.y) + (P.y - p2.y) * (p3.x - p2.x),
                           ((-(p1.x - p2.x)) * (p3.y - p2.y) + (p1.y - p2.y) * (p3.x - p2.x)) + 1e-7f);
            beta = EZ_DIV((-(P.x - p3.x)) * (p1.y - p3.y) + (P.y - p3.y) * (p1.x - p3.x),
                          ((-(p2.x - p3.x)) * (p1.y - p3.y) + (p2.y - p3.y) * (p1.x - p3.x)) + 1e-7f);
        } else {  // P3/fsh:273-274, P4/fsh (same lines)
            alpha = EZ_DIV((-(P.x - p2.x)) * (p3.y - p2.y) + (P.y - p2.y) * (p3.x - p2.x),
                           (-((p1.x - p2.x) - 0.00005f)) * ((p3.y - p2.y) + 0.00005f) +
                               ((p1.y - p2.y) + 0.00005f) * ((p3.x - p2.x) + 0.00005f));
            beta = EZ_DIV((-(P.x - p3.x)) * (p1.y - p3.y) + (P.y - p3.y) * (p1.x - p3.x),
                          (-((p2.x - p3.x) - 0.00005f)) * ((p1.y - p3.y) + 0.00005f) +
                              ((p2.y - p3.y) + 0.00005f) * ((p1.x - p3.x) + 0.00005f));
        }
        float gama = (1.0f - alpha) - beta;
        vec3 Nsmooth = ez_add(ez_add(ez_scale(triangle.n1, alpha), ez_scale(triangle.n2, beta)),
                              ez_scale(triangle.n3, gama));
        Nsmooth = ez_normalize(Nsmooth);
        res.normal = res.isInside ? ez_neg(Nsmooth) : Nsmooth;
    }
    return res;
}

// ---------------------------------------------------------------- hitAABB
// P5/fsh:220-233, P2/main.cpp:449-463.  t0out = slab entry distance (used only by the pruned policy).
float hitAABB(const Ray& r, vec3 AA, vec3 BB, float* t0out) {
    vec3 invdir = ez_v3(EZ_DIV(1.0f, r.direction.x), EZ_DIV(1.0f, r.direction.y), EZ_DIV(1.0f, r.direction.z));
    vec3 f = ez_mul(ez_sub(BB, r.startPoint), invdir);
    vec3 n = ez_mul(ez_sub(AA, r.startPoint), invdir);
    vec3 tmax = ez_vmax(f, n);
    vec3 tmin = ez_vmin(f, n);
    float t1 = ez_min(tmax.x, ez_min(tmax.y, tmax.z));
    float t0 = ez_max(tmin.x, ez_max(tmin.y, tmin.z));
    *t0out = t0;
    return (t1 >= t0) ? ((t0 > 0.0f) ? t0 : t1) : -1.0f;
}

// ---------------------------------------------------------------- hitArray, P5/fsh:238-251
HitResult hitArray(const Scene& sc, const Ray& ray, int l, int r, Counters& cn) {
    HitResult res;
    res.isHit = false;
    res.isInside = false;
    res.distance = EZ_INF;
    res.triangle = -1;
    res.hitPoint = res.normal = res.viewDir = ez_v3(0, 0, 0);
    bool fudge = (sc.mode == EZRT_MODE_DIFFUSE_P3 || sc.mode == EZRT_MODE_DISNEY_ANISO_P4);
    for (int i = l; i <= r; i++) {
        Triangle triangle = getTriangle(sc, i);
        cn.tris++;
        HitResult rr = hitTriangle(triangle, ray, fudge);
        if (rr.isHit && rr.distance < res.distance) {
            res = rr;
            res.triangle = i;
        }
    }
    return res;
}

// Per-ray slack of the pruned policy: a sub-tree is skipped only if its box entry distance
// t0 exceeds  best + (|best| * 2^-12 + pruneDelta * max_k |1/d_k|).  See DESIGN.md "pruning".
inline float pruneSlack(const Scene& sc, const Ray& ray) {
    float ix = ez_abs(EZ_DIV(1.0f, ray.direction.x)), iy = ez_abs(EZ_DIV(1.0f, ray.direction.y)),
          iz = ez_abs(EZ_DIV(1.0f, ray.direction.z));
    float m = ez_max(ix, ez_max(iy, iz));
    return sc.pruneDelta * m;
}
inline bool pruned(float t0, float best, float slack) {
    // NaN-safe: any NaN makes the comparison false => not pruned
    return t0 > (best + (best * 0.000244140625f + slack));
}

// ---------------------------------------------------------------- hitBVH, P5/fsh:254-306
// (identical in P3/fsh:319-371 and P4/fsh:243-295).  P2's recursive C++ twin (P2/main.cpp:
// 466-485) swaps n/index in its leaf call (:471); that bug is documented, not reproduced.
float* g_rayDump = nullptr;  // see oracle_set_ray_dump
uint64_t g_rayDumpCap = 0, g_rayDumpCount = 0;

HitResult hitBVH(const Scene& sc, const Ray& ray, Counters& cn, int kind) {
    cn.rays[kind]++;
    HitResult res;
    res.isHit = false;
    res.isInside = false;
    res.distance = EZ_INF;
    res.triangle = -1;
    res.hitPoint = res.normal = res.viewDir = ez_v3(0, 0, 0);

    if (g_rayDump) {  // development aid (tools/accel_stats.cpp): record the rays a render traces, kind = 0 primary, 1 bounce, 2 shadow
        const uint64_t k = __atomic_fetch_add(&g_rayDumpCount, 1, __ATOMIC_RELAXED);
        if (k < g_rayDumpCap) {
            float* r = g_rayDump + 7 * k;
            r[0] = ray.startPoint.x; r[1] = ray.startPoint.y; r[2] = ray.startPoint.z;
            r[3] = ray.direction.x; r[4] = ray.direction.y; r[5] = ray.direction.z; r[6] = (float)kind;
        }
    }

    const bool prune = (sc.traverse != EZRT_TRAVERSE_REFERENCE);  // the oracle has no accel tree: ACCEL == PRUNED here
    const float slack = prune ? pruneSlack(sc, ray) : 0.0f;

    int stack[256];
    float stackT0[256];
    int stackDepth[256];
    int sp = 0;
    stackT0[sp] = -1.0f;
    stackDepth[sp] = 0;
    stack[sp++] = 1;
    cn.nodes++;  // the root is fetched once
    while (sp > 0) {
        if ((uint64_t)sp > cn.max_stack) cn.max_stack = (uint64_t)sp;
        int top = stack[--sp];
        const int depth = stackDepth[sp];
        if (prune && pruned(stackT0[sp], res.distance, slack)) continue;
        BVHNode node = getBVHNode(sc, top);
        if (node.n > 0) {
            int L = node.index;
            int R = node.index + node.n - 1;
            HitResult r = hitArray(sc, ray, L, R, cn);
            if (r.isHit && r.distance < res.distance) res = r;
            continue;
        }
        float d1 = EZ_INF, d2 = EZ_INF;
        float e1 = -1.0f, e2 = -1.0f;
        cn.innerByDepth[depth < 63 ? depth : 63]++;
        if (node.left > 0) {
            BVHNode leftNode = getBVHNode(sc, node.left);
            cn.nodes++;
            d1 = hitAABB(ray, leftNode.AA, leftNode.BB, &e1);
        }
        if (node.right > 0) {
            BVHNode rightNode = getBVHNode(sc, node.right);
            cn.nodes++;
            d2 = hitAABB(ray, rightNode.AA, rightNode.BB, &e2);
        }
        bool h1 = d1 > 0, h2 = d2 > 0;
        if (prune) {  // drop a child whose box starts beyond the current best hit
            if (h1 && pruned(e1, res.distance, slack)) h1 = false;
            if (h2 && pruned(e2, res.distance, slack)) h2 = false;
            if (h1 && h2) {
                if (d1 < d2) { stackT0[sp] = e2; stackDepth[sp] = depth + 1; stack[sp++] = node.right; stackT0[sp] = e1; stackDepth[sp] = depth + 1; stack[sp++] = node.left; }
                else         { stackT0[sp] = e1; stackDepth[sp] = depth + 1; stack[sp++] = node.left;  stackT0[sp] = e2; stackDepth[sp] = depth + 1; stack[sp++] = node.right; }
            } else if (h1) { stackT0[sp] = e1; stackDepth[sp] = depth + 1; stack[sp++] = node.left; }
            else if (h2)   { stackT0[sp] = e2; stackDepth[sp] = depth + 1; stack[sp++] = node.right; }
            continue;
        }
        if (h1 && h2) {
            stackDepth[sp] = stackDepth[sp + 1] = depth + 1;
            if (d1 < d2) { stack[sp++] = node.right; stack[sp++] = node.left; }
            else         { stack[sp++] = node.left;  stack[sp++] = node.right; }
        } else if (h1) {
            stackDepth[sp] = depth + 1;
            stack[sp++] = node.left;
        } else if (h2) {
            stackDepth[sp] = depth + 1;
            stack[sp++] = node.right;
        }
    }
    if (res.isHit) cn.hits++;
    return res;
}

// ---------------------------------------------------------------- RNG, P5/fsh:315-331
inline uint32_t wang_hash(uint32_t& seed) {
    seed = (seed ^ 61u) ^ (seed >> 16);
    seed *= 9u;
    seed = seed ^ (seed >> 4);
    seed *= 0x27d4eb2du;
    seed = seed ^ (seed >> 15);
    return seed;
}
inline float u2unit(uint32_t h) { return ez_u32_to_float(h) * 2.3283064365386963e-10f; }  // / 4294967296.0
struct Rng {
    uint32_t seed;
    float rand() { return u2unit(wang_hash(seed)); }
};

// ---------------------------------------------------------------- Sobol, P5/fsh:351-376
const uint32_t V[8 * 32] = {
#include "ezrt_sobol_table.inc"
};
inline uint32_t grayCode(uint32_t i) { return i ^ (i >> 1); }
inline float sobol(uint32_t d, uint32_t i) {
    uint32_t result = 0;
    uint32_t offset = d * 32;
    for (uint32_t j = 0; i != 0; i >>= 1, j++)
        if ((i & 1) != 0) result ^= V[(j + offset) & 255u];  // d >= 8 is out of bounds in the shader; wraps here
    return ez_u32_to_float(result) * (1.0f / 4294967296.0f);  // 1.0f/float(0xFFFFFFFFU), float(0xFFFFFFFF)=2^32
}
inline void sobolVec2(uint32_t i, uint32_t b, float* u, float* v) {
    *u = sobol(b * 2, grayCode(i));
    *v = sobol(b * 2 + 1, grayCode(i));
}
// P5/fsh:378-396
inline void CranleyPattersonRotation(float* px, float* py, uint32_t pixx, uint32_t pixy) {
    uint32_t pseed = (pixx * 1973u + pixy * 9277u + (uint32_t)(114514 / 1919) * 26699u) | 1u;
    float u = u2unit(wang_hash(pseed));
    float v = u2unit(wang_hash(pseed));
    float x = *px, y = *py;
    x += u;
    if (x > 1) x -= 1;
    if (x < 0) x += 1;
    y += v;
    if (y > 1) y -= 1;
    if (y < 0) y += 1;
    *px = x;
    *py = y;
}

// ---------------------------------------------------------------- Disney BRDF, P5/fsh:400-549
inline float SchlickFresnel(float u) {
    float m = ez_clamp(1.0f - u, 0.0f, 1.0f);
    float m2 = m * m;
    return m2 * m2 * m;
}
inline float GTR1(float NdotH, float a) {
    if (a >= 1) return EZ_DIV(1.0f, EZ_PI);
    float a2 = a * a;
    float t = 1.0f + (a2 - 1.0f) * NdotH * NdotH;
    return EZ_DIV(a2 - 1.0f, EZ_PI * ez_log(a2) * t);
}
inline float GTR2(float NdotH, float a) {
    float a2 = a * a;
    float t = 1.0f + (a2 - 1.0f) * NdotH * NdotH;
    return EZ_DIV(a2, EZ_PI * t * t);
}
inline float GTR2_aniso(float NdotH, float HdotX, float HdotY, float ax, float ay) {
    return EZ_DIV(1.0f, EZ_PI * ax * ay * ez_sqr(ez_sqr(EZ_DIV(HdotX, ax)) + ez_sqr(EZ_DIV(HdotY, ay)) + NdotH * NdotH));
}
inline float smithG_GGX(float NdotV, float alphaG) {
    float a = alphaG * alphaG;
    float b = NdotV * NdotV;
    return EZ_DIV(1.0f, NdotV + EZ_SQRT(a + b - a * b));
}
inline float smithG_GGX_aniso(float NdotV, float VdotX, float VdotY, float ax, float ay) {
    return EZ_DIV(1.0f, NdotV + EZ_SQRT(ez_sqr(VdotX * ax) + ez_sqr(VdotY * ay) + ez_sqr(NdotV)));
}
inline vec3 splat(float s) { return ez_v3(s, s, s); }

// P5/fsh:500-549 BRDF_Evaluate (== body of BRDF_Evaluate_aniso :437-498, whose aniso block is
// commented out) when aniso == false;  P4/fsh:412-473 when aniso == true.
vec3 BRDF_Evaluate(vec3 Vv, vec3 N, vec3 L, vec3 X, vec3 Y, const Material& material, bool aniso) {
    float NdotL = ez_dot(N, L);
    float NdotV = ez_dot(N, Vv);
    if (NdotL < 0 || NdotV < 0) return splat(0);

    vec3 H = ez_normalize(ez_add(L, Vv));
    float NdotH = ez_dot(N, H);
    float LdotH = ez_dot(L, H);

    vec3 Cdlin = material.baseColor;
    float Cdlum = 0.3f * Cdlin.x + 0.6f * Cdlin.y + 0.1f * Cdlin.z;
    vec3 Ctint = (Cdlum > 0) ? ez_divs(Cdlin, Cdlum) : splat(1);
    vec3 Cspec = ez_scale(ez_vmix(splat(1), Ctint, material.specularTint), material.specular);
    vec3 Cspec0 = ez_vmix(ez_scale(Cspec, 0.08f), Cdlin, material.metallic);
    vec3 Csheen = ez_vmix(splat(1), Ctint, material.sheenTint);

    float Fd90 = 0.5f + 2.0f * LdotH * LdotH * material.roughness;
    float FL = SchlickFresnel(NdotL);
    float FV = SchlickFresnel(NdotV);
    float Fd = ez_mix(1.0f, Fd90, FL) * ez_mix(1.0f, Fd90, FV);

    float Fss90 = LdotH * LdotH * material.roughness;
    float Fss = ez_mix(1.0f, Fss90, FL) * ez_mix(1.0f, Fss90, FV);
    float ss = 1.25f * (Fss * (EZ_DIV(1.0f, NdotL + NdotV) - 0.5f) + 0.5f);

    float Ds, FH, Gs;
    vec3 Fs;
    if (!aniso) {
        float alpha = ez_max(0.001f, ez_sqr(material.roughness));
        Ds = GTR2(NdotH, alpha);
        FH = SchlickFresnel(LdotH);
        Fs = ez_vmix(Cspec0, splat(1), FH);
        Gs = smithG_GGX(NdotL, material.roughness);
        Gs *= smithG_GGX(NdotV, material.roughness);
    } else {
        float aspect = EZ_SQRT(1.0f - material.anisotropic * 0.9f);
        float ax = ez_max(0.001f, EZ_DIV(ez_sqr(material.roughness), aspect));
        float ay = ez_max(0.001f, ez_sqr(material.roughness) * aspect);
        Ds = GTR2_aniso(NdotH, ez_dot(H, X), ez_dot(H, Y), ax, ay);
        FH = SchlickFresnel(LdotH);
        Fs = ez_vmix(Cspec0, splat(1), FH);
        Gs = smithG_GGX_aniso(NdotL, ez_dot(L, X), ez_dot(L, Y), ax, ay);
        Gs *= smithG_GGX_aniso(NdotV, ez_dot(Vv, X), ez_dot(Vv, Y), ax, ay);
    }

    float Dr = GTR1(NdotH, ez_mix(0.1f, 0.001f, material.clearcoatGloss));
    float Fr = ez_mix(0.04f, 1.0f, FH);
    float Gr = smithG_GGX(NdotL, 0.25f) * smithG_GGX(NdotV, 0.25f);

    vec3 Fsheen = ez_scale(Csheen, FH * material.sheen);

    vec3 diffuse = ez_add(ez_scale(Cdlin, EZ_DIV(1.0f, EZ_PI) * ez_mix(Fd, ss, material.subsurface)), Fsheen);
    vec3 specular = ez_scale(ez_scale(Fs, Gs), Ds);  // GLSL "Gs * Fs * Ds" = (Gs*Fs)*Ds
    vec3 clearcoat = splat(0.25f * Gr * Fr * Dr * material.clearcoat);

    return ez_add(ez_add(ez_scale(diffuse, 1.0f - material.metallic), specular), clearcoat);
}

// P5/fsh:553-558 (P4/fsh:341-352)
inline void getTangent(vec3 N, vec3* tangent, vec3* bitangent) {
    vec3 helper = ez_v3(1, 0, 0);
    if (ez_abs(N.x) > 0.999f) helper = ez_v3(0, 0, 1);
    *bitangent = ez_normalize(ez_cross(N, helper));
    *tangent = ez_normalize(ez_cross(N, *bitangent));
}
// P5/fsh:561-567
inline vec3 toNormalHemisphere(vec3 v, vec3 N) {
    vec3 helper = ez_v3(1, 0, 0);
    if (ez_abs(N.x) > 0.999f) helper = ez_v3(0, 0, 1);
    vec3 tangent = ez_normalize(ez_cross(N, helper));
    vec3 bitangent = ez_normalize(ez_cross(N, tangent));
    return ez_add(ez_add(ez_scale(tangent, v.x), ez_scale(bitangent, v.y)), ez_scale(N, v.z));
}
// P5/fsh:570-576
inline vec3 SampleHemisphere(float xi_1, float xi_2) {
    float z = xi_1;
    float r = ez_max(0.0f, EZ_SQRT(1.0f - z * z));
    float phi = 2.0f * EZ_PI * xi_2;
    return ez_v3(r * ez_cos(phi), r * ez_sin(phi), z);
}
// P5/fsh:579-590
inline vec3 SampleCosineHemisphere(float xi_1, float xi_2, vec3 N) {
    float r = EZ_SQRT(xi_1);
    float theta = xi_2 * 2.0f * EZ_PI;
    float x = r * ez_cos(theta);
    float y = r * ez_sin(theta);
    float z = EZ_SQRT(1.0f - x * x - y * y);
    return toNormalHemisphere(ez_v3(x, y, z), N);
}
// P5/fsh:593-610
inline vec3 SampleGTR2(float xi_1, float xi_2, vec3 Vv, vec3 N, float alpha) {
    float phi_h = 2.0f * EZ_PI * xi_1;
    float sin_phi_h = ez_sin(phi_h);
    float cos_phi_h = ez_cos(phi_h);
    float cos_theta_h = EZ_SQRT(EZ_DIV(1.0f - xi_2, 1.0f + (alpha * alpha - 1.0f) * xi_2));
    float sin_theta_h = EZ_SQRT(ez_max(0.0f, 1.0f - cos_theta_h * cos_theta_h));
    vec3 H = ez_v3(sin_theta_h * cos_phi_h, sin_theta_h * sin_phi_h, cos_theta_h);
    H = toNormalHemisphere(H, N);
    return ez_reflect(ez_neg(Vv), H);
}
// P5/fsh:613-630
inline vec3 SampleGTR1(float xi_1, float xi_2, vec3 Vv, vec3 N, float alpha) {
    float phi_h = 2.0f * EZ_PI * xi_1;
    float sin_phi_h = ez_sin(phi_h);
    float cos_phi_h = ez_cos(phi_h);
    float cos_theta_h = EZ_SQRT(EZ_DIV(1.0f - ez_pow(alpha * alpha, 1.0f - xi_2), 1.0f - alpha * alpha));
    float sin_theta_h = EZ_SQRT(ez_max(0.0f, 1.0f - cos_theta_h * cos_theta_h));
    vec3 H = ez_v3(sin_theta_h * cos_phi_h, sin_theta_h * sin_phi_h, cos_theta_h);
    H = toNormalHemisphere(H, N);
    return ez_reflect(ez_neg(Vv), H);
}
// P5/fsh:633-664
vec3 SampleBRDF(float xi_1, float xi_2, float xi_3, vec3 Vv, vec3 N, const Material& material) {
    float alpha_GTR1 = ez_mix(0.1f, 0.001f, material.clearcoatGloss);
    float alpha_GTR2 = ez_max(0.001f, ez_sqr(material.roughness));
    float r_diffuse = (1.0f - material.metallic);
    float r_specular = 1.0f;
    float r_clearcoat = 0.25f * material.clearcoat;
    float r_sum = r_diffuse + r_specular + r_clearcoat;
    float p_diffuse = EZ_DIV(r_diffuse, r_sum);
    float p_specular = EZ_DIV(r_specular, r_sum);
    float rd = xi_3;
    if (rd <= p_diffuse) return SampleCosineHemisphere(xi_1, xi_2, N);
    else if (p_diffuse < rd && rd <= p_diffuse + p_specular) return SampleGTR2(xi_1, xi_2, Vv, N, alpha_GTR2);
    else if (p_diffuse + p_specular < rd) return SampleGTR1(xi_1, xi_2, Vv, N, alpha_GTR1);
    return ez_v3(0, 1, 0);
}
// P5/fsh:715-752
float BRDF_Pdf(vec3 Vv, vec3 N, vec3 L, const Material& material) {
    float NdotL = ez_dot(N, L);
    float NdotV = ez_dot(N, Vv);
    if (NdotL < 0 || NdotV < 0) return 0;
    vec3 H = ez_normalize(ez_add(L, Vv));
    float NdotH = ez_dot(N, H);
    float alpha = ez_max(0.001f, ez_sqr(material.roughness));
    float Ds = GTR2(NdotH, alpha);
    float Dr = GTR1(NdotH, ez_mix(0.1f, 0.001f, material.clearcoatGloss));
    float pdf_diffuse = EZ_DIV(NdotL, EZ_PI);
    float pdf_specular = EZ_DIV(Ds * NdotH, 4.0f * ez_dot(L, H));
    float pdf_clearcoat = EZ_DIV(Dr * NdotH, 4.0f * ez_dot(L, H));
    float r_diffuse = (1.0f - material.metallic);
    float r_specular = 1.0f;
    float r_clearcoat = 0.25f * material.clearcoat;
    float r_sum = r_diffuse + r_specular + r_clearcoat;
    float p_diffuse = EZ_DIV(r_diffuse, r_sum);
    float p_specular = EZ_DIV(r_specular, r_sum);
    float p_clearcoat = EZ_DIV(r_clearcoat, r_sum);
    float pdf = p_diffuse * pdf_diffuse + p_specular * pdf_specular + p_clearcoat * pdf_clearcoat;
    pdf = ez_max(1e-10f, pdf);
    return pdf;
}
// P5/fsh:754-757
inline float misMixWeight(float a, float b) {
    float t = a * a;
    return EZ_DIV(t, b * b + t);
}

// ---------------------------------------------------------------- textures
// texture2D on an RGB32F W x H image with CLAMP_TO_EDGE; row 0 <-> v = 0.
vec3 tex2D(const float* img, int W, int H, float u, float v, bool linear) {
    if (!linear) return texel(img, ez_env_texel(u, v, W, H));  // GL_NEAREST
    float x = u * (float)W - 0.5f, y = v * (float)H - 0.5f;
    float fx0 = ez_floor(x), fy0 = ez_floor(y);
    float ax = x - fx0, ay = y - fy0;
    // indices clamped in float: a NaN coordinate reads texel 0 and weighs it by NaN
    const int x0 = ez_texel_clamp(fx0, W), x1 = ez_texel_clamp(fx0 + 1.0f, W);
    const int y0 = ez_texel_clamp(fy0, H), y1 = ez_texel_clamp(fy0 + 1.0f, H);
    vec3 t00 = texel(img, y0 * W + x0), t10 = texel(img, y0 * W + x1);
    vec3 t01 = texel(img, y1 * W + x0), t11 = texel(img, y1 * W + x1);
    return ez_vmix(ez_vmix(t00, t10, ax), ez_vmix(t01, t11, ax), ay);
}

// P5/fsh:684-690
inline void toSphericalCoord(vec3 v, float* ou, float* ov) {
    float u = ez_atan2(v.z, v.x), w = ez_asin(v.y);
    u = EZ_DIV(u, 2.0f * EZ_PI);
    w = EZ_DIV(w, EZ_PI);
    u += 0.5f;
    w += 0.5f;
    w = 1.0f - w;
    *ou = u;
    *ov = w;
}
// P5/fsh:693-697 hdrColor; P3/fsh:151-156 sampleHdr (clamped to 10); P4/fsh:366-371 (unclamped)
vec3 hdrColor(const Scene& sc, vec3 L, Counters& cn) {
    vec3 color;
    if (!sc.hdr) {
        color = sc.envColor;
    } else {
        float u, v;
        toSphericalCoord(ez_normalize(L), &u, &v);
        cn.hdr_lookups++;
        color = tex2D(sc.hdr, sc.hdrW, sc.hdrH, u, v, sc.hdrLinear != 0);
    }
    if (sc.mode == EZRT_MODE_DIFFUSE_P3) color = ez_vmin(color, splat(10.0f));
    return color;
}
// P5/fsh:667-679
vec3 SampleHdr(const Scene& sc, float xi_1, float xi_2, Counters& cn) {
    vec3 c = tex2D(sc.hdrCache, sc.hdrW, sc.hdrH, xi_1, xi_2, sc.hdrLinear != 0);
    cn.hdr_lookups++;
    float x = c.x, y = c.y;
    y = 1.0f - y;
    float phi = 2.0f * EZ_PI * (x - 0.5f);
    float theta = EZ_PI * (y - 0.5f);
    return ez_v3(ez_cos(theta) * ez_cos(phi), ez_sin(theta), ez_cos(theta) * ez_sin(phi));
}
// P5/fsh:701-712
float hdrPdf(const Scene& sc, vec3 L, int hdrResolution, Counters& cn) {
    float u, v;
    toSphericalCoord(ez_normalize(L), &u, &v);
    cn.hdr_lookups++;
    float pdf = tex2D(sc.hdrCache, sc.hdrW, sc.hdrH, u, v, sc.hdrLinear != 0).z;
    float theta = EZ_PI * (0.5f - v);
    float sin_theta = ez_max(ez_sin(theta), 1e-10f);
    float p_convert = EZ_DIV((float)(hdrResolution * hdrResolution / 2), 2.0f * EZ_PI * EZ_PI * sin_theta);
    return pdf * p_convert;
}

// ---------------------------------------------------------------- integrators
struct PixelCtx {
    uint32_t px, py, frameCounter;
    Rng rng;
};

// Lo += a*b*c*s/p  with GLSL's left-to-right evaluation:  ((((a*b)*c)*s)/p)
inline vec3 contrib(vec3 a, vec3 b, vec3 c, float s, float p) {
    return ez_divs(ez_scale(ez_mul(ez_mul(a, b), c), s), p);
}

// P3/fsh:376-413 (diffuse), P4/fsh:478-517 (aniso Disney), P5/fsh:762-807 (Sobol Disney)
vec3 pathTracing(const Scene& sc, HitResult hit, int maxBounce, PixelCtx& px, Counters& cn) {
    vec3 Lo = splat(0);
    vec3 history = splat(1);
    for (int bounce = 0; bounce < maxBounce; bounce++) {
        vec3 Vv = ez_neg(hit.viewDir);
        vec3 N = hit.normal;
        Material material = getMaterial(sc, hit.triangle);
        vec3 L;
        if (sc.mode == EZRT_MODE_DISNEY_SOBOL_P5) {
            float u, v;
            sobolVec2(px.frameCounter + 1u, (uint32_t)bounce, &u, &v);
            CranleyPattersonRotation(&u, &v, px.px, px.py);
            L = SampleHemisphere(u, v);
        } else {  // P3/fsh:110-115, P4/fsh:325-329: z = rand() first, then phi
            float z = px.rng.rand();
            float r = ez_max(0.0f, EZ_SQRT(1.0f - z * z));
            float phi = 2.0f * EZ_PI * px.rng.rand();
            L = ez_v3(r * ez_cos(phi), r * ez_sin(phi), z);
        }
        L = toNormalHemisphere(L, hit.normal);
        float pdf = EZ_DIV(1.0f, 2.0f * EZ_PI);
        float cosine_i = ez_max(0.0f, ez_dot(L, N));
        vec3 f_r;
        if (sc.mode == EZRT_MODE_DIFFUSE_P3) {
            f_r = ez_divs(material.baseColor, EZ_PI);
        } else {
            vec3 tangent, bitangent;
            getTangent(N, &tangent, &bitangent);
            f_r = BRDF_Evaluate(Vv, N, L, tangent, bitangent, material, sc.mode == EZRT_MODE_DISNEY_ANISO_P4);
        }
        Ray randomRay;
        randomRay.startPoint = hit.hitPoint;
        randomRay.direction = L;
        HitResult newHit = hitBVH(sc, randomRay, cn, 1);
        if (!newHit.isHit) {
            vec3 skyColor = hdrColor(sc, randomRay.direction, cn);
            Lo = ez_add(Lo, contrib(history, skyColor, f_r, cosine_i, pdf));
            break;
        }
        vec3 Le = getMaterial(sc, newHit.triangle).emissive;
        Lo = ez_add(Lo, contrib(history, Le, f_r, cosine_i, pdf));
        hit = newHit;
        history = ez_mul(history, ez_divs(ez_scale(f_r, cosine_i), pdf));
    }
    return Lo;
}

// P5/fsh:810-890
vec3 pathTracingImportanceSampling(const Scene& sc, HitResult hit, int maxBounce, PixelCtx& px, Counters& cn) {
    vec3 Lo = splat(0);
    vec3 history = splat(1);
    const int hdrResolution = sc.hdrW;
    for (int bounce = 0; bounce < maxBounce; bounce++) {
        vec3 Vv = ez_neg(hit.viewDir);
        vec3 N = hit.normal;
        Material material = getMaterial(sc, hit.triangle);

        Ray hdrTestRay;
        hdrTestRay.startPoint = hit.hitPoint;
        float r1 = px.rng.rand();
        float r2 = px.rng.rand();
        hdrTestRay.direction = SampleHdr(sc, r1, r2, cn);
        if (ez_dot(N, hdrTestRay.direction) > 0.0f) {
            HitResult hdrHit = hitBVH(sc, hdrTestRay, cn, 2);
            if (!hdrHit.isHit) {
                vec3 L = hdrTestRay.direction;
                vec3 color = hdrColor(sc, L, cn);
                float pdf_light = hdrPdf(sc, L, hdrResolution, cn);
                vec3 f_r = BRDF_Evaluate(Vv, N, L, splat(0), splat(0), material, false);
                float pdf_brdf = BRDF_Pdf(Vv, N, L, material);
                float mis_weight = misMixWeight(pdf_light, pdf_brdf);
                // mis_weight * history * color * f_r * dot(N, L) / pdf_light
                vec3 c = ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, mis_weight), color), f_r), ez_dot(N, L)), pdf_light);
                Lo = ez_add(Lo, c);
            }
        }

        float xi_1, xi_2;
        sobolVec2(px.frameCounter + 1u, (uint32_t)bounce, &xi_1, &xi_2);
        CranleyPattersonRotation(&xi_1, &xi_2, px.px, px.py);
        float xi_3 = px.rng.rand();

        vec3 L = SampleBRDF(xi_1, xi_2, xi_3, Vv, N, material);
        float NdotL = ez_dot(N, L);
        if (NdotL <= 0.0f) break;

        Ray randomRay;
        randomRay.startPoint = hit.hitPoint;
        randomRay.direction = L;
        HitResult newHit = hitBVH(sc, randomRay, cn, 1);

        vec3 f_r = BRDF_Evaluate(Vv, N, L, splat(0), splat(0), material, false);
        float pdf_brdf = BRDF_Pdf(Vv, N, L, material);
        if (pdf_brdf <= 0.0f) break;

        if (!newHit.isHit) {
            vec3 color = hdrColor(sc, L, cn);
            float pdf_light = hdrPdf(sc, L, hdrResolution, cn);
            float mis_weight = misMixWeight(pdf_brdf, pdf_light);
            vec3 c = ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, mis_weight), color), f_r), NdotL), pdf_brdf);
            Lo = ez_add(Lo, c);
            break;
        }
        vec3 Le = getMaterial(sc, newHit.triangle).emissive;
        Lo = ez_add(Lo, contrib(history, Le, f_r, NdotL, pdf_brdf));
        hit = newHit;
        history = ez_mul(history, ez_divs(ez_scale(f_r, NdotL), pdf_brdf));
    }
    return Lo;
}

// main(), P5/fsh:894-949 (P4/fsh:521-550, P3/fsh:417-446): one fragment = one sample of one pixel
vec3 shadePixel(const Scene& sc, const ezrt_render_params& p, uint32_t ipx, uint32_t ipy, uint32_t frameCounter,
                Counters& cn) {
    PixelCtx px;
    px.px = ipx; px.py = ipy; px.frameCounter = frameCounter;
    px.rng.seed = (ipx * 1973u + ipy * 9277u + frameCounter * 26699u) | 1u;

    float pixx = EZ_DIV((float)ipx + 0.5f, (float)p.width) * 2.0f - 1.0f;
    float pixy = EZ_DIV((float)ipy + 0.5f, (float)p.height) * 2.0f - 1.0f;

    Ray ray;
    ray.startPoint = ez_v3(p.eye[0], p.eye[1], p.eye[2]);
    float aax = EZ_DIV(px.rng.rand() - 0.5f, (float)p.width);
    float aay = EZ_DIV(px.rng.rand() - 0.5f, (float)p.height);
    float vx = pixx + aax, vy = pixy + aay, vz = -1.5f, vw = 0.0f;
    const float* m = p.camera_rotate;  // column-major: m[col*4+row]
    vec3 dir = ez_v3(((m[0] * vx + m[4] * vy) + m[8] * vz) + m[12] * vw,
                     ((m[1] * vx + m[5] * vy) + m[9] * vz) + m[13] * vw,
                     ((m[2] * vx + m[6] * vy) + m[10] * vz) + m[14] * vw);
    ray.direction = ez_normalize(dir);

    HitResult firstHit = hitBVH(sc, ray, cn, 0);
    vec3 color;
    if (!firstHit.isHit) {
        color = hdrColor(sc, ray.direction, cn);
    } else {
        vec3 Le = getMaterial(sc, firstHit.triangle).emissive;
        vec3 Li = (sc.mode == EZRT_MODE_DISNEY_IS_MIS_P5)
                      ? pathTracingImportanceSampling(sc, firstHit, p.max_bounce, px, cn)
                      : pathTracing(sc, firstHit, p.max_bounce, px, cn);
        color = ez_add(Le, Li);
    }
    return color;
}

inline float maxAbsCoord(const float* tris, int n) {
    float m = 0.0f;
    for (int i = 0; i < n; i++)
        for (int k = 0; k < 9; k++) {
            float a = ez_abs(tris[(size_t)i * 36 + k]);
            if (a > m) m = a;
        }
    return m;
}

uint64_t g_innerByDepth[64];  // accumulated by oracle_render (diagnostic: where traversal time goes)

Scene makeScene(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr,
                const float* hdrCache, int hdrW, int hdrH, int hdrLinear, const float envColor[3], int mode,
                int traverse) {
    Scene sc;
    sc.tris = tris; sc.nTriangles = nTriangles; sc.nodes = nodes; sc.nNodes = nNodes;
    sc.hdr = hdr; sc.hdrCache = hdrCache; sc.hdrW = hdrW; sc.hdrH = hdrH; sc.hdrLinear = hdrLinear;
    sc.envColor = envColor ? ez_v3(envColor[0], envColor[1], envColor[2]) : ez_v3(0, 0, 0);
    sc.mode = mode; sc.traverse = traverse;
    sc.pruneDelta = maxAbsCoord(tris, nTriangles) * 1.52587890625e-05f;  // 2^-16 * scene extent
    return sc;
}

}  // namespace

extern "C" {

// counters_out[0..8] = rays_primary, rays_bounce, rays_shadow, N_node, N_tri, H, hdr_lookups, samples, max_stack
// Window form: only the pixels [x0,x1) x [y0,y1) of the width x height grid are rendered, into a framebuffer of
// (y1-y0) x (x1-x0) pixels (row 0 = row y0).  Pixel (px,py) gets exactly the value the full render gives it: seed,
// Sobol index and Cranley-Patterson shift depend only on (px, py, frame) (P5/fsh:315-318, :379-382).  This lets the
// parity tests check the BASELINE configs on their OWN pixel grid (1920x1080, 1024x1024) at a cost of seconds.
int oracle_render_window(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr,
                         const float* hdrCache, int hdrW, int hdrH, int hdrLinear, const ezrt_render_params* p,
                         int x0, int y0, int x1, int y1, float* framebuffer, uint64_t* counters_out, int n_threads) {
    if (!tris || !nodes || !p || !framebuffer || nTriangles <= 0 || nNodes < 2) return -1;
    if (x0 < 0 || y0 < 0 || x1 > p->width || y1 > p->height || x1 <= x0 || y1 <= y0) return -1;
    if (p->mode == EZRT_MODE_DISNEY_IS_MIS_P5 && (!hdr || !hdrCache)) return -1;
    Scene sc = makeScene(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p->env_color, p->mode,
                         p->traverse);
    const int C = (p->out_channels == 4) ? 4 : 3;
    Counters total;
    memset(&total, 0, sizeof(total));
#ifdef _OPENMP
    if (n_threads > 0) omp_set_num_threads(n_threads);
#endif
#pragma omp parallel
    {
        Counters cn;
        memset(&cn, 0, sizeof(cn));
#pragma omp for schedule(dynamic, 1)
        for (int py = y0; py < y1; py++) {
            for (int pxl = x0; pxl < x1; pxl++) {
                float* dst = framebuffer + ((size_t)(py - y0) * (x1 - x0) + (pxl - x0)) * C;
                vec3 acc = ez_v3(dst[0], dst[1], dst[2]);
                if (p->first_frame == 0) acc = ez_v3(0, 0, 0);
                for (int s = 0; s < p->spp; s++) {
                    uint32_t frameCounter = p->first_frame + (uint32_t)s;
                    vec3 color = shadePixel(sc, *p, (uint32_t)pxl, (uint32_t)py, frameCounter, cn);
                    // P5/fsh:943-944: mix(lastColor, color, 1.0/float(frameCounter+1))
                    float a = EZ_DIV(1.0f, ez_u32_to_float(frameCounter + 1u));
                    acc = ez_vmix(acc, color, a);
                }
                dst[0] = acc.x; dst[1] = acc.y; dst[2] = acc.z;
                if (C == 4) dst[3] = 1.0f;
            }
        }
#pragma omp critical
        {
            for (int k = 0; k < 3; k++) total.rays[k] += cn.rays[k];
            total.nodes += cn.nodes; total.tris += cn.tris; total.hits += cn.hits;
            total.hdr_lookups += cn.hdr_lookups;
            for (int k = 0; k < 64; k++) g_innerByDepth[k] += cn.innerByDepth[k];
            if (cn.max_stack > total.max_stack) total.max_stack = cn.max_stack;
        }
    }
    if (counters_out) {
        counters_out[0] = total.rays[0]; counters_out[1] = total.rays[1]; counters_out[2] = total.rays[2];
        counters_out[3] = total.nodes; counters_out[4] = total.tris; counters_out[5] = total.hits;
        counters_out[6] = total.hdr_lookups; counters_out[7] = (uint64_t)(x1 - x0) * (y1 - y0) * (uint64_t)p->spp;
        counters_out[8] = total.max_stack;
    }
    return 0;
}

int oracle_render(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr,
                  const float* hdrCache, int hdrW, int hdrH, int hdrLinear, const ezrt_render_params* p,
                  float* framebuffer, uint64_t* counters_out, int n_threads) {
    if (!p) return -1;
    return oracle_render_window(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p, 0, 0, p->width, p->height,
                                framebuffer, counters_out, n_threads);
}

// hitBVH for n rays; brute = 1 runs hitArray over all triangles instead (P2/main.cpp:585's cross-check).
int oracle_trace_rays(const float* tris, int nTriangles, const float* nodes, int nNodes, int n, const float* origins,
                      const float* dirs, int traverse, int p3_fudge, int brute, int32_t* out_hit, float* out_distance,
                      int32_t* out_triangle, int32_t* out_inside, float* out_point, float* out_normal,
                      uint64_t* counters_out) {
    Scene sc = makeScene(tris, nTriangles, nodes, nNodes, nullptr, nullptr, 0, 0, 0, nullptr,
                         p3_fudge ? EZRT_MODE_DIFFUSE_P3 : EZRT_MODE_DISNEY_SOBOL_P5, traverse);
    Counters cn;
    memset(&cn, 0, sizeof(cn));
    for (int i = 0; i < n; i++) {
        Ray ray;
        ray.startPoint = ez_v3(origins[3 * i], origins[3 * i + 1], origins[3 * i + 2]);
        ray.direction = ez_v3(dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2]);
        HitResult r = brute ? hitArray(sc, ray, 0, nTriangles - 1, cn) : hitBVH(sc, ray, cn, 0);
        out_hit[i] = r.isHit ? 1 : 0;
        out_distance[i] = r.distance;
        out_triangle[i] = r.triangle;
        out_inside[i] = r.isInside ? 1 : 0;
        out_point[3 * i] = r.hitPoint.x; out_point[3 * i + 1] = r.hitPoint.y; out_point[3 * i + 2] = r.hitPoint.z;
        out_normal[3 * i] = r.normal.x; out_normal[3 * i + 1] = r.normal.y; out_normal[3 * i + 2] = r.normal.z;
    }
    if (counters_out) {
        counters_out[0] = cn.rays[0]; counters_out[1] = cn.nodes; counters_out[2] = cn.tris;
        counters_out[3] = cn.hits; counters_out[4] = cn.max_stack;
    }
    return 0;
}

static Material materialFrom18(const float* m) {
    Material r;
    r.emissive = ez_v3(m[0], m[1], m[2]);
    r.baseColor = ez_v3(m[3], m[4], m[5]);
    r.subsurface = m[6]; r.metallic = m[7]; r.specular = m[8];
    r.specularTint = m[9]; r.roughness = m[10]; r.anisotropic = m[11];
    r.sheen = m[12]; r.sheenTint = m[13]; r.clearcoat = m[14];
    r.clearcoatGloss = m[15]; r.IOR = m[16]; r.transmission = m[17];
    return r;
}

// which: 0 BRDF_Evaluate (P5), 1 BRDF_Evaluate aniso (P4, frame from getTangent), 2 BRDF_Pdf, 3 SampleBRDF
int oracle_eval_brdf(int which, int n, const float* Vv, const float* Nn, const float* Ll, const float* xi,
                     const float* materials, float* out) {
    for (int i = 0; i < n; i++) {
        vec3 V3 = ez_v3(Vv[3 * i], Vv[3 * i + 1], Vv[3 * i + 2]);
        vec3 N3 = ez_v3(Nn[3 * i], Nn[3 * i + 1], Nn[3 * i + 2]);
        vec3 L3 = Ll ? ez_v3(Ll[3 * i], Ll[3 * i + 1], Ll[3 * i + 2]) : ez_v3(0, 0, 0);
        Material m = materialFrom18(materials + (size_t)i * 18);
        vec3 r = ez_v3(0, 0, 0);
        if (which == 0) r = BRDF_Evaluate(V3, N3, L3, splat(0), splat(0), m, false);
        else if (which == 1) {
            vec3 t, b;
            getTangent(N3, &t, &b);
            r = BRDF_Evaluate(V3, N3, L3, t, b, m, true);
        } else if (which == 2) r.x = BRDF_Pdf(V3, N3, L3, m);
        else if (which == 3) r = SampleBRDF(xi[3 * i], xi[3 * i + 1], xi[3 * i + 2], V3, N3, m);
        else return -1;
        out[3 * i] = r.x; out[3 * i + 1] = r.y; out[3 * i + 2] = r.z;
    }
    return 0;
}

// which: 0 sin, 1 cos, 2 log, 3 exp, 4 pow, 5 atan2, 6 asin, 7 floor
int oracle_eval_math(int which, int n, const float* a, const float* b, float* out) {
    for (int i = 0; i < n; i++) {
        float x = a[i], y = b ? b[i] : 0.0f, r;
        switch (which) {
            case 0: r = ez_sin(x); break;
            case 1: r = ez_cos(x); break;
            case 2: r = ez_log(x); break;
            case 3: r = ez_exp(x); break;
            case 4: r = ez_pow(x, y); break;
            case 5: r = ez_atan2(x, y); break;
            case 6: r = ez_asin(x); break;
            case 7: r = ez_floor(x); break;
            default: return -1;
        }
        out[i] = r;
    }
    return 0;
}

// KAT helpers (tests/test_kat.py): wang_hash chain / rand(), sobol, CP rotation
void oracle_wang_chain(uint32_t seed, int n, uint32_t* hashes, float* rands) {
    Rng r;
    r.seed = seed;
    for (int i = 0; i < n; i++) {
        uint32_t h = wang_hash(r.seed);
        hashes[i] = h;
        rands[i] = u2unit(h);
    }
}
float oracle_sobol(uint32_t d, uint32_t i) { return sobol(d, grayCode(i)); }
void oracle_cp_rotation(float* xy, uint32_t px, uint32_t py) { CranleyPattersonRotation(&xy[0], &xy[1], px, py); }
float oracle_pi(void) { return EZ_PI; }
// pass3.fsh:14-25 on n pixels (`channels` floats in, 3 floats out)
void oracle_tonemap(const float* in, int channels, float* out, long long n, float limit) {
    for (long long i = 0; i < n; i++) {
        vec3 c = ez_tonemap_pass3(ez_v3(in[i * channels], in[i * channels + 1], in[i * channels + 2]), limit);
        out[i * 3] = c.x; out[i * 3 + 1] = c.y; out[i * 3 + 2] = c.z;
    }
}
// development aid: while `buf` is set, every hitBVH call appends (origin, direction, kind) -- 7 floats -- to it (up to `cap`
// rays); returns the number of rays seen since the previous call and resets the counter
uint64_t oracle_set_ray_dump(float* buf, uint64_t cap) {
    const uint64_t seen = g_rayDumpCount;
    g_rayDump = buf;
    g_rayDumpCap = cap;
    g_rayDumpCount = 0;
    return seen;
}

// inner-node visits by depth accumulated over all oracle_render calls since the last reset
void oracle_depth_hist(uint64_t* out64, int reset) {
    for (int k = 0; k < 64; k++) { out64[k] = g_innerByDepth[k]; if (reset) g_innerByDepth[k] = 0; }
}

}  // extern "C"
