// device_functions.cuh -- sm_90a device code of the hot path: BVH traversal, ray/triangle and
// ray/box tests, Disney BRDF evaluate/sample/pdf, wang-hash + Sobol samplers, HDR lookups.
// Replaces the GLSL of P5/shaders/fshader.fsh (and its P3/P4 variants) and the C++ twins
// hitTriangle/hitAABB/hitBVH of P2/main.cpp:212-238,:449-485.  Every function cites the
// reference lines it must agree with; arithmetic is the normative fp32 of ezrt_math.h
// (compile with -fmad=false: FMA only where EZ_FMA spells it).
#ifndef EZRT_DEVICE_FUNCTIONS_CUH
#define EZRT_DEVICE_FUNCTIONS_CUH

#include "device_scene.h"
#include "ezrt.h"
#include "ezrt_math.h"
#include "w8_node.h"

__constant__ uint32_t c_sobolV[8 * 32] = {
#include "ezrt_sobol_table.inc"
};

typedef ez_vec3 vec3;

__device__ __forceinline__ vec3 f4xyz(float4 q) { return ez_v3(q.x, q.y, q.z); }
__device__ __forceinline__ vec3 splat3(float s) { return ez_v3(s, s, s); }
__device__ __forceinline__ float4 ldg4(const float4* p) { return __ldg(p); }

// The transcendental functions of ezrt_math.h are 35-100 instructions each and the integrators call them at up to twenty sites;
// inlined everywhere they made k_shade<IS/MIS> 5104 instructions (80 KB), whose largest stall is instruction fetch
// (`no_instruction` was the largest stall).  EZRT_MATH_NOINLINE=1 routes the calls through one out-of-line
// copy per function (same code, same bits).
#ifndef EZRT_MATH_NOINLINE
#define EZRT_MATH_NOINLINE 0
#endif
#if EZRT_MATH_NOINLINE
#define EZD_MATH __device__ __noinline__
#else
#define EZD_MATH __device__ __forceinline__
#endif
EZD_MATH float ezd_sin(float x) { return ez_sin(x); }
EZD_MATH float ezd_cos(float x) { return ez_cos(x); }
EZD_MATH float ezd_log(float x) { return ez_log(x); }
EZD_MATH float ezd_pow(float x, float y) { return ez_pow(x, y); }
EZD_MATH float ezd_atan2(float y, float x) { return ez_atan2(y, x); }
EZD_MATH float ezd_asin(float x) { return ez_asin(x); }

// ------------------------------------------------------------------------------------------
// RNG + low-discrepancy samplers
// ------------------------------------------------------------------------------------------
// wang_hash / rand, P5/fsh:320-331
__device__ __forceinline__ uint32_t wang_hash(uint32_t& seed) {
    seed = (seed ^ 61u) ^ (seed >> 16);
    seed *= 9u;
    seed = seed ^ (seed >> 4);
    seed *= 0x27d4eb2du;
    seed = seed ^ (seed >> 15);
    return seed;
}
__device__ __forceinline__ float rand01(uint32_t& seed) {
    return __uint2float_rn(wang_hash(seed)) * 2.3283064365386963e-10f;  // float(h) / 4294967296.0
}
// seed initialiser, P5/fsh:315-318
__device__ __forceinline__ uint32_t pixel_seed(uint32_t px, uint32_t py, uint32_t frame) {
    return (px * 1973u + py * 9277u + frame * 26699u) | 1u;
}
// sobol(d, grayCode(i)), P5/fsh:356-369
__device__ __forceinline__ float sobol_gray(uint32_t d, uint32_t i) {
    uint32_t g = i ^ (i >> 1);
    uint32_t result = 0;
    uint32_t offset = (d * 32u) & 255u;
    for (uint32_t j = 0; g != 0; g >>= 1, j++)
        if (g & 1u) result ^= c_sobolV[(j + offset) & 255u];
    return __uint2float_rn(result) * 2.3283064365386963e-10f;  // * (1.0f/float(0xFFFFFFFFU))
}
// CranleyPattersonRotation, P5/fsh:378-396
__device__ __forceinline__ void cp_rotate(float& x, float& y, uint32_t px, uint32_t py) {
    uint32_t pseed = (px * 1973u + py * 9277u + 59u * 26699u) | 1u;  // uint(114514/1919) = 59
    float u = rand01(pseed);
    float v = rand01(pseed);
    x += u;
    if (x > 1.0f) x -= 1.0f;
    if (x < 0.0f) x += 1.0f;
    y += v;
    if (y > 1.0f) y -= 1.0f;
    if (y < 0.0f) y += 1.0f;
}

// ------------------------------------------------------------------------------------------
// BVH traversal (hitBVH P5/fsh:254-306, hitArray :238-251, hitTriangle :160-217, hitAABB :220-233)
// ------------------------------------------------------------------------------------------
struct HitRec {
    float t;    // EZ_INF on miss
    int tri;    // -1 on miss
};

// ---- fp32 pairs in one 64-bit register pair: the slab constants of a ray and the (x, y) / (lo, hi) halves of a node
// record travel together.  Hopper has no packed fp32x2 add / mul, so each operation is two scalar IEEE-rn instructions
// (explicitly _rn: never contracted into an FMA).
typedef unsigned long long pk2;
__device__ __forceinline__ pk2 pk2_make(float lo, float hi) {
    pk2 r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ void pk2_split(pk2 v, float& lo, float& hi) {
    asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ pk2 pk2_add(pk2 a, pk2 b) {
    float a0, a1, b0, b1;
    pk2_split(a, a0, a1);
    pk2_split(b, b0, b1);
    return pk2_make(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ pk2 pk2_mul(pk2 a, pk2 b) {
    float a0, a1, b0, b1;
    pk2_split(a, a0, a1);
    pk2_split(b, b0, b1);
    return pk2_make(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}

// 32-byte read-only global loads (32-byte aligned): two 128-bit loads, the widest Hopper has
#ifndef EZRT_NODE_L1_POLICY
#define EZRT_NODE_L1_POLICY 0   // 1: node records are loaded with L1::evict_last (experiment)
#endif
__device__ __forceinline__ void ldg256_b64(const void* p, ulonglong2& a, ulonglong2& b) {
    const char* c = static_cast<const char*>(p);
#if EZRT_NODE_L1_POLICY == 1
    asm("ld.global.nc.L1::evict_last.v2.b64 {%0, %1}, [%2];" : "=l"(a.x), "=l"(a.y) : "l"(c));
    asm("ld.global.nc.L1::evict_last.v2.b64 {%0, %1}, [%2];" : "=l"(b.x), "=l"(b.y) : "l"(c + 16));
#else
    asm("ld.global.nc.v2.b64 {%0, %1}, [%2];" : "=l"(a.x), "=l"(a.y) : "l"(c));
    asm("ld.global.nc.v2.b64 {%0, %1}, [%2];" : "=l"(b.x), "=l"(b.y) : "l"(c + 16));
#endif
}
__device__ __forceinline__ uint4 ldg128_u32(const uint4* p) {
    uint4 a;
#if EZRT_NODE_L1_POLICY == 1
    asm("ld.global.nc.L1::evict_last.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w) : "l"(p));
#else
    asm("ld.global.nc.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w) : "l"(p));
#endif
    return a;
}
// ldg4 without allocating the line in L1 (LDG.NA): triangle records of a large scene are touched once per ray,
// the L1 is better spent on node records (a scene whose triangles fit in L1/L2-near caches loses with it, so
// SceneDev::tri_l1_bypass is set by size).  volatile: the load stays behind the branches that guard it.
__device__ __forceinline__ float4 ldg4_na(const float4* p) {
    float4 a;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(a.x), "=f"(a.y), "=f"(a.z), "=f"(a.w) : "l"(p));
    return a;
}

// Per-ray constants of the slab test: -origin and 1/direction as register pairs.
struct RaySlab {
    pk2 no_xy, no_zz, inv_xy, inv_zz;
};
__device__ __forceinline__ RaySlab make_ray_slab(vec3 o, vec3 inv) {
    RaySlab r;
    r.no_xy = pk2_make(-o.x, -o.y);
    r.no_zz = pk2_make(-o.z, -o.z);
    r.inv_xy = pk2_make(inv.x, inv.y);
    r.inv_zz = pk2_make(inv.z, inv.z);
    return r;
}

struct NodeVisit {
    bool h1, h2;        // would the shader push the left / right child (hitAABB > 0, P5/fsh:290-302)
    float d1, d2;       // hitAABB distances the children are ordered by
    float e1, e2;       // slab entry distances (pruning only)
    int rl, rr;         // child references
};

// hitAABB (P5/fsh:220-233) for both children of one inner node: (BB - S) * invdir and
// (AA - S) * invdir as 6 pair additions + 6 pair products ((x - s) == (x + (-s)) exactly), then min/max.
// FAST: all 1/d finite, no NaN can arise, FMNMX equals the GLSL ternaries; otherwise the
// ternaries are evaluated literally (NaN behaviour of the oracle).
template <bool FAST>
__device__ __forceinline__ NodeVisit node_visit_q(ulonglong2 q0, ulonglong2 q1, ulonglong2 q2, ulonglong2 q3, const RaySlab& rs);

// record from global memory: four 128-bit loads.  The traversal is bound by L1 wavefronts -- every lane
// reads a different line.
template <bool FAST>
__device__ __forceinline__ NodeVisit node_visit(const float4* __restrict__ nd, const RaySlab& rs) {
    ulonglong2 q0, q1, q2, q3;
    ldg256_b64(nd, q0, q1);
    ldg256_b64(nd + 2, q2, q3);
    return node_visit_q<FAST>(q0, q1, q2, q3, rs);
}
// record of the top tree levels from shared memory (stride EZRT_TOP_STRIDE float4 = 80 B, so the
// 16-byte pieces of different records spread over the banks), else from global memory
template <bool FAST>
__device__ __forceinline__ NodeVisit node_visit_top(const float4* __restrict__ nodes, const float4* smem_top, int top_nodes, int ref, const RaySlab& rs) {
    ulonglong2 q0, q1, q2, q3;
    if (ref < top_nodes) {
        const ulonglong2* p = reinterpret_cast<const ulonglong2*>(smem_top + ref * EZRT_TOP_STRIDE);
        q0 = p[0]; q1 = p[1]; q2 = p[2]; q3 = p[3];
    } else {
        const float4* nd = nodes + (size_t)ref * 4;
        ldg256_b64(nd, q0, q1);
        ldg256_b64(nd + 2, q2, q3);
    }
    return node_visit_q<FAST>(q0, q1, q2, q3, rs);
}

template <bool FAST>
__device__ __forceinline__ NodeVisit node_visit_q(ulonglong2 q0, ulonglong2 q1, ulonglong2 q2, ulonglong2 q3, const RaySlab& rs) {
    int2 refs = make_int2((int)(unsigned)(q3.x & 0xffffffffull), (int)(unsigned)(q3.x >> 32));
    float lnx, lny, lfx, lfy, rnx, rny, rfx, rfy, lnz, lfz, rnz, rfz;
    pk2_split(pk2_mul(pk2_add(q0.x, rs.no_xy), rs.inv_xy), lnx, lny);  // left  (AA - S) * inv, x y
    pk2_split(pk2_mul(pk2_add(q0.y, rs.no_xy), rs.inv_xy), lfx, lfy);  // left  (BB - S) * inv, x y
    pk2_split(pk2_mul(pk2_add(q1.x, rs.no_xy), rs.inv_xy), rnx, rny);  // right (AA - S) * inv, x y
    pk2_split(pk2_mul(pk2_add(q1.y, rs.no_xy), rs.inv_xy), rfx, rfy);  // right (BB - S) * inv, x y
    pk2_split(pk2_mul(pk2_add(q2.x, rs.no_zz), rs.inv_zz), lnz, lfz);  // left  z: (AA.z, BB.z)
    pk2_split(pk2_mul(pk2_add(q2.y, rs.no_zz), rs.inv_zz), rnz, rfz);  // right z
    float lt1, lt0, rt1, rt0;
    if (FAST) {
        lt1 = fminf(fmaxf(lfx, lnx), fminf(fmaxf(lfy, lny), fmaxf(lfz, lnz)));
        lt0 = fmaxf(fminf(lfx, lnx), fmaxf(fminf(lfy, lny), fminf(lfz, lnz)));
        rt1 = fminf(fmaxf(rfx, rnx), fminf(fmaxf(rfy, rny), fmaxf(rfz, rnz)));
        rt0 = fmaxf(fminf(rfx, rnx), fmaxf(fminf(rfy, rny), fminf(rfz, rnz)));
    } else {
        lt1 = ez_min(ez_max(lfx, lnx), ez_min(ez_max(lfy, lny), ez_max(lfz, lnz)));
        lt0 = ez_max(ez_min(lfx, lnx), ez_max(ez_min(lfy, lny), ez_min(lfz, lnz)));
        rt1 = ez_min(ez_max(rfx, rnx), ez_min(ez_max(rfy, rny), ez_max(rfz, rnz)));
        rt0 = ez_max(ez_min(rfx, rnx), ez_max(ez_min(rfy, rny), ez_min(rfz, rnz)));
    }
    NodeVisit v;
    v.e1 = lt0;
    v.e2 = rt0;
    v.d1 = (lt1 >= lt0) ? ((lt0 > 0.0f) ? lt0 : lt1) : -1.0f;
    v.d2 = (rt1 >= rt0) ? ((rt0 > 0.0f) ? rt0 : rt1) : -1.0f;
    v.h1 = v.d1 > 0.0f;
    v.h2 = v.d2 > 0.0f;
    v.rl = refs.x;
    v.rr = refs.y;
    return v;
}

// ---- 4-wide node of the acceleration tree (128-byte record, DESIGN.md "accel"):
//   q0..q3 : child c = (AA.x, AA.y, BB.x, BB.y)      q4 : (AA.z0, BB.z0, AA.z1, BB.z1)
//   q5     : (AA.z2, BB.z2, AA.z3, BB.z3)            q6 : the four child references
// An absent child has an inverted box (never hit).  The acceleration tree is free to visit children
// in any order, so they are ordered by slab entry distance; one dependent fetch now decides two levels.
struct WideVisit {
    float k0, k1, k2, k3;   // entry distance of each child, +inf when missed / pruned
    int r0, r1, r2, r3;
};
__device__ __forceinline__ void slab_xy(pk2 lo, pk2 hi, const RaySlab& rs, float& t0, float& t1) {
    float nx, ny, fx, fy;
    pk2_split(pk2_mul(pk2_add(lo, rs.no_xy), rs.inv_xy), nx, ny);
    pk2_split(pk2_mul(pk2_add(hi, rs.no_xy), rs.inv_xy), fx, fy);
    t0 = fmaxf(fminf(fx, nx), fminf(fy, ny));
    t1 = fminf(fmaxf(fx, nx), fmaxf(fy, ny));
}
__device__ __forceinline__ float wide_key(float t0, float t1, float nz, float fz, float limit) {
    t0 = fmaxf(t0, fminf(fz, nz));
    t1 = fminf(t1, fmaxf(fz, nz));
    const bool ok = (t1 >= t0) && (t1 > 0.0f) && !(t0 > limit);  // hitAABB > 0 and not beyond the best hit
    return ok ? t0 : 3.0e38f;
}
__device__ __forceinline__ WideVisit wide_visit(const float4* __restrict__ nd, const RaySlab& rs, float limit) {
    ulonglong2 q0, q1, q2, q3, q4, q5;
    ldg256_b64(nd, q0, q1);
    ldg256_b64(nd + 2, q2, q3);
    ldg256_b64(nd + 4, q4, q5);
    const int4 refs = __ldg(reinterpret_cast<const int4*>(nd + 6));
    float a0, b0, a1, b1, a2, b2, a3, b3;
    slab_xy(q0.x, q0.y, rs, a0, b0);
    slab_xy(q1.x, q1.y, rs, a1, b1);
    slab_xy(q2.x, q2.y, rs, a2, b2);
    slab_xy(q3.x, q3.y, rs, a3, b3);
    float z0n, z0f, z1n, z1f, z2n, z2f, z3n, z3f;
    pk2_split(pk2_mul(pk2_add(q4.x, rs.no_zz), rs.inv_zz), z0n, z0f);
    pk2_split(pk2_mul(pk2_add(q4.y, rs.no_zz), rs.inv_zz), z1n, z1f);
    pk2_split(pk2_mul(pk2_add(q5.x, rs.no_zz), rs.inv_zz), z2n, z2f);
    pk2_split(pk2_mul(pk2_add(q5.y, rs.no_zz), rs.inv_zz), z3n, z3f);
    WideVisit v;
    v.k0 = wide_key(a0, b0, z0n, z0f, limit);
    v.k1 = wide_key(a1, b1, z1n, z1f, limit);
    v.k2 = wide_key(a2, b2, z2n, z2f, limit);
    v.k3 = wide_key(a3, b3, z3n, z3f, limit);
    v.r0 = refs.x; v.r1 = refs.y; v.r2 = refs.z; v.r3 = refs.w;
    return v;
}
// ---- the same node with 16-bit quantised planes (96 B = three 256-bit loads instead of 3.5; DESIGN.md section 4, "Q16"):
//   w0..2 origin.xyz   w3..5 scale.xyz (powers of two)   w6 + 3 c + a : child c, axis a, (lo | hi << 16)   w18..21 references
// plane = origin + q * scale, stored floor(x - 1.25) / ceil(x + 1.25) steps: supersets of the exact boxes under the decode
//   t = fma(as_float(0x4B000000 | q), scale * inv_d, fma(-2^23, scale * inv_d, (origin - o) * inv_d))
// (error bound as in w8_node.h with the A term rounded at magnitude 2^23 * B: half a step; the builder keeps scale >=
// W8_MIN_STEP_REL * max|coordinate|).  The bounce / shadow launches are bound by the L1 gather rate, and a 96-byte record is
// gathered faster than the 128-byte one; the decode costs ~24 instructions.
// Near / far planes are picked by the PRMT selector: sel_a = 0x7510 takes the low half (the lo plane), 0x7532 the high half; the
// ray keeps the NEAR selector per axis (lo iff d_a >= 0), the far one is near ^ 0x0022 -- no min/max per axis.
__device__ __forceinline__ float q16_plane(uint32_t w, uint32_t bias, uint32_t sel, float B, float A) {
    uint32_t f;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(f) : "r"(w), "r"(bias), "r"(sel));
    return __fmaf_rn(__uint_as_float(f), B, A);
}
struct Q16Ray {
    uint32_t nx, ny, nz;   // near-plane selectors
};
__device__ __forceinline__ Q16Ray make_q16_ray(vec3 d) {
    Q16Ray r;
    r.nx = (d.x >= 0.0f) ? 0x7510u : 0x7532u;
    r.ny = (d.y >= 0.0f) ? 0x7510u : 0x7532u;
    r.nz = (d.z >= 0.0f) ? 0x7510u : 0x7532u;
    return r;
}
__device__ __forceinline__ float q16_child(uint32_t wx, uint32_t wy, uint32_t wz, uint32_t bias, const Q16Ray& qr, uint32_t fx, uint32_t fy, uint32_t fz, float Bx,
                                           float By, float Bz, float Ax, float Ay, float Az, float limit) {
    const float t0 = fmaxf(fmaxf(q16_plane(wx, bias, qr.nx, Bx, Ax), q16_plane(wy, bias, qr.ny, By, Ay)), q16_plane(wz, bias, qr.nz, Bz, Az));
    const float t1 = fminf(fminf(q16_plane(wx, bias, fx, Bx, Ax), q16_plane(wy, bias, fy, By, Ay)), q16_plane(wz, bias, fz, Bz, Az));
    const bool ok = (t1 >= t0) && (t1 > 0.0f) && !(t0 > limit);
    return ok ? t0 : 3.0e38f;
}
__device__ __forceinline__ WideVisit wide_visit_q16(const uint4* __restrict__ nd, vec3 o, const RaySlab& rs, float limit, uint32_t bias, const Q16Ray& qr) {
    ulonglong2 a, b;
    ldg256_b64(nd, a, b);
    const uint32_t w0 = (uint32_t)a.x, w1 = (uint32_t)(a.x >> 32), w2 = (uint32_t)a.y, w3 = (uint32_t)(a.y >> 32);
    const uint32_t w4 = (uint32_t)b.x, w5 = (uint32_t)(b.x >> 32), w6 = (uint32_t)b.y, w7 = (uint32_t)(b.y >> 32);
    ldg256_b64(nd + 2, a, b);
    const uint32_t w8 = (uint32_t)a.x, w9 = (uint32_t)(a.x >> 32), w10 = (uint32_t)a.y, w11 = (uint32_t)(a.y >> 32);
    const uint32_t w12 = (uint32_t)b.x, w13 = (uint32_t)(b.x >> 32), w14 = (uint32_t)b.y, w15 = (uint32_t)(b.y >> 32);
    ldg256_b64(nd + 4, a, b);
    const uint32_t w16 = (uint32_t)a.x, w17 = (uint32_t)(a.x >> 32);
    float ix, iy, iz, iz2;
    pk2_split(rs.inv_xy, ix, iy);
    pk2_split(rs.inv_zz, iz, iz2);
    const float Bx = __uint_as_float(w3) * ix, By = __uint_as_float(w4) * iy, Bz = __uint_as_float(w5) * iz;
    const float Ax = __fmaf_rn(-8388608.0f, Bx, (__uint_as_float(w0) - o.x) * ix);
    const float Ay = __fmaf_rn(-8388608.0f, By, (__uint_as_float(w1) - o.y) * iy);
    const float Az = __fmaf_rn(-8388608.0f, Bz, (__uint_as_float(w2) - o.z) * iz);
    const uint32_t fx = qr.nx ^ 0x0022u, fy = qr.ny ^ 0x0022u, fz = qr.nz ^ 0x0022u;
    WideVisit v;
    v.k0 = q16_child(w6, w7, w8, bias, qr, fx, fy, fz, Bx, By, Bz, Ax, Ay, Az, limit);
    v.k1 = q16_child(w9, w10, w11, bias, qr, fx, fy, fz, Bx, By, Bz, Ax, Ay, Az, limit);
    v.k2 = q16_child(w12, w13, w14, bias, qr, fx, fy, fz, Bx, By, Bz, Ax, Ay, Az, limit);
    v.k3 = q16_child(w15, w16, w17, bias, qr, fx, fy, fz, Bx, By, Bz, Ax, Ay, Az, limit);
    v.r0 = (int)a.y; v.r1 = (int)(a.y >> 32); v.r2 = (int)b.x; v.r3 = (int)(b.x >> 32);
    return v;
}
__device__ __forceinline__ void cswap(float& ka, int& ra, float& kb, int& rb) {  // ascending by key
    const bool sw = kb < ka;
    const float tk = sw ? kb : ka, uk = sw ? ka : kb;
    const int tr = sw ? rb : ra, ur = sw ? ra : rb;
    ka = tk; kb = uk; ra = tr; rb = ur;
}

// Ray/triangle test against the repacked record (N, d0), p1, p2, p3.  Accepts exactly the hits hitTriangle accepts
// that are also strictly closer than `best` (the only ones hitArray/hitBVH can keep).
// TIES (accel policy): a hit at exactly t == best is also reported (return 2) so the caller can
// detect that two triangles tie and let the exact reference-order traversal decide.
// The distance checks need only the first 16 bytes; the vertices are loaded for the candidates that pass them.
template <bool TIES>
__device__ __forceinline__ int tri_test_t(const float4* __restrict__ rec, vec3 o, vec3 d, float best, float& tout, const bool l1_bypass = false) {
    const float4 q0 = l1_bypass ? ldg4_na(rec) : ldg4(rec);   // l1_bypass is warp-uniform
    vec3 N = f4xyz(q0);
    float nd = ez_dot(N, d);
    if (ez_abs(nd) < 0.00001f) return 0;                        // :181 (|dot(+-N,d)| is sign-free)
    float t = EZ_DIV(q0.w - ez_dot(o, N), nd);                  // :184 (sign of N cancels exactly)
    if (t < 0.0005f) return 0;                                  // :185
    if (TIES ? !(t <= best) : !(t < best)) return 0;            // :245, :273 strict <, first wins
    float4 q1, q2, q3;
    if (l1_bypass) {
        q1 = ldg4_na(rec + 1); q2 = ldg4_na(rec + 2); q3 = ldg4_na(rec + 3);
    } else {
        q1 = ldg4(rec + 1); q2 = ldg4(rec + 2); q3 = ldg4(rec + 3);
    }
    vec3 p1 = f4xyz(q1), p2 = f4xyz(q2), p3 = f4xyz(q3);
    vec3 P = ez_add(o, ez_scale(d, t));                         // :188
    float s1 = ez_dot(ez_cross(ez_sub(p2, p1), ez_sub(P, p1)), N);  // :191-195 (N unflipped: r1/r2 swap)
    float s2 = ez_dot(ez_cross(ez_sub(p3, p2), ez_sub(P, p2)), N);
    float s3 = ez_dot(ez_cross(ez_sub(p1, p3), ez_sub(P, p3)), N);
    bool r1 = (s1 > 0.0f && s2 > 0.0f && s3 > 0.0f);
    bool r2 = (s1 < 0.0f && s2 < 0.0f && s3 < 0.0f);
    if (!(r1 || r2)) return 0;
    tout = t;
    return (TIES && t == best) ? 2 : 1;
}
// The same test, statement for statement, on an indexed record (N, d0) (i1, i2, i3, 0) and the vertex array: both halves of
// the record are loaded together (one 32-byte sector); the three vertices, independent of each other, for the candidates past
// the distance checks.  The vertices are read through L1 even where the records bypass it: the triangles of a leaf, tested by
// neighbouring lanes and steps, share them (C3, H100: 3 % faster than with the vertices past L1, which was no faster than flat).
template <bool TIES>
__device__ __forceinline__ int tri_test_idx_t(const float4* __restrict__ rec, const float4* __restrict__ vert, vec3 o, vec3 d, float best, float& tout,
                                              const bool l1_bypass) {
    const float4 q0 = l1_bypass ? ldg4_na(rec) : ldg4(rec);
    const float4 qi = l1_bypass ? ldg4_na(rec + 1) : ldg4(rec + 1);
    vec3 N = f4xyz(q0);
    float nd = ez_dot(N, d);
    if (ez_abs(nd) < 0.00001f) return 0;
    float t = EZ_DIV(q0.w - ez_dot(o, N), nd);
    if (t < 0.0005f) return 0;
    if (TIES ? !(t <= best) : !(t < best)) return 0;
    const float4* v1 = vert + __float_as_uint(qi.x);
    const float4* v2 = vert + __float_as_uint(qi.y);
    const float4* v3 = vert + __float_as_uint(qi.z);
    const float4 q1 = ldg4(v1), q2 = ldg4(v2), q3 = ldg4(v3);   // through L1 whatever l1_bypass: the triangles of a leaf share them
    vec3 p1 = f4xyz(q1), p2 = f4xyz(q2), p3 = f4xyz(q3);
    vec3 P = ez_add(o, ez_scale(d, t));
    float s1 = ez_dot(ez_cross(ez_sub(p2, p1), ez_sub(P, p1)), N);
    float s2 = ez_dot(ez_cross(ez_sub(p3, p2), ez_sub(P, p2)), N);
    float s3 = ez_dot(ez_cross(ez_sub(p1, p3), ez_sub(P, p3)), N);
    bool r1 = (s1 > 0.0f && s2 > 0.0f && s3 > 0.0f);
    bool r2 = (s1 < 0.0f && s2 < 0.0f && s3 < 0.0f);
    if (!(r1 || r2)) return 0;
    tout = t;
    return (TIES && t == best) ? 2 : 1;
}
__device__ __forceinline__ bool tri_test(const float4* __restrict__ rec, vec3 o, vec3 d, float best, float& tout) {
    return tri_test_t<false>(rec, o, d, best, tout) != 0;
}

__device__ __forceinline__ bool prune_test(float t0, float best, float slack) {
    return t0 > (best + (best * 0.000244140625f + slack));
}

// hitBVH.  PRUNE: skip sub-trees whose box entry lies beyond the best hit (+ conservative slack);
// ANYHIT: return on the first accepted triangle (shadow rays only need isHit, P5/fsh:826-829).
// tmax: a bounded ray (light samples) starts with best = tmax, so only hits strictly closer than tmax are accepted.
template <bool PRUNE, bool ANYHIT, bool FAST>
__device__ __forceinline__ HitRec trace_impl(const SceneDev& sc, vec3 o, vec3 d, vec3 inv, float slack, float tmax = EZ_INF) {
    HitRec res;
    res.t = tmax;
    res.tri = -1;
    int stack[EZRT_MAX_STACK];
    float stack_t0[PRUNE ? EZRT_MAX_STACK : 1];
    int sp = 0;
    int ref = sc.root_ref;
    float ref_t0 = -1.0f;
    const RaySlab rs = make_ray_slab(o, inv);
    while (true) {
        if (ref < 0) {  // leaf: hitArray(index, index+n-1)
            uint32_t bits = (uint32_t)ref & 0x7fffffffu;
            int n = (int)(bits & 127u);
            int first = (int)(bits >> 7);
            const float4* rec = sc.tri_geo + (size_t)first * 4;
            for (int i = 0; i < n; i++, rec += 4) {
                float t;
                if (tri_test(rec, o, d, res.t, t)) {
                    res.t = t;
                    res.tri = first + i;
                    if (ANYHIT) return res;
                }
            }
        } else {
            NodeVisit nv = node_visit<FAST>(sc.nodes + (size_t)ref * 4, rs);
            bool h1 = nv.h1, h2 = nv.h2;
            const float d1 = nv.d1, d2 = nv.d2, e1 = nv.e1, e2 = nv.e2;
            const int rl = nv.rl, rr = nv.rr;
            if (PRUNE) {
                if (h1 && prune_test(e1, res.t, slack)) h1 = false;
                if (h2 && prune_test(e2, res.t, slack)) h2 = false;
            }
            if (h1 && h2) {  // near child first, far child pushed (P5/fsh:290-297)
                bool leftFirst = d1 < d2;
                int nearRef = leftFirst ? rl : rr, farRef = leftFirst ? rr : rl;
                if (PRUNE) stack_t0[sp] = leftFirst ? e2 : e1;
                stack[sp++] = farRef;
                ref = nearRef;
                if (PRUNE) ref_t0 = leftFirst ? e1 : e2;
                continue;
            } else if (h1) {
                ref = rl;
                if (PRUNE) ref_t0 = e1;
                continue;
            } else if (h2) {
                ref = rr;
                if (PRUNE) ref_t0 = e2;
                continue;
            }
        }
        // pop
        while (true) {
            if (sp == 0) return res;
            --sp;
            ref = stack[sp];
            if (PRUNE) {
                ref_t0 = stack_t0[sp];
                if (prune_test(ref_t0, res.t, slack)) continue;
            }
            break;
        }
    }
}

template <bool PRUNE, bool ANYHIT>
__device__ __forceinline__ HitRec trace_ray(const SceneDev& sc, vec3 o, vec3 d) {
    vec3 inv = ez_v3(EZ_DIV(1.0f, d.x), EZ_DIV(1.0f, d.y), EZ_DIV(1.0f, d.z));  // hitAABB :221
    float ax = ez_abs(inv.x), ay = ez_abs(inv.y), az = ez_abs(inv.z);
    float m = ez_max(ax, ez_max(ay, az));
    bool finite = (ax < 3.0e38f) && (ay < 3.0e38f) && (az < 3.0e38f);  // false for inf and NaN
    float slack = sc.prune_delta * m;
    if (finite) return trace_impl<PRUNE, ANYHIT, true>(sc, o, d, inv, slack);
    return trace_impl<PRUNE, ANYHIT, false>(sc, o, d, inv, slack);
}

// ------------------------------------------------------------------------------------------
// Persistent-warp traversal ("while-while" with per-lane refill).  Incoherent bounce rays have
// very different traversal lengths; a warp that waits for its longest ray runs at ~4 of 32
// lanes (ncu).  Here a lane that finishes its ray takes the next one from the
// global work counter (warp-aggregated atomicAdd) while its neighbours keep traversing, and the
// inner-node loop is separated from the leaf loop so lanes at inner nodes do not wait for lanes
// testing triangles.  Per ray the visit order -- and therefore the result -- is exactly that
// of trace_impl / the shader's hitBVH.
//   io.load(i, o, d) fetches ray i; io.store(i, hit) receives its result.
// ------------------------------------------------------------------------------------------
#ifndef EZRT_LEAF_SERIAL
#define EZRT_LEAF_SERIAL 0  // 1: lane-serial leaf tests in the accel kernels instead of the cooperative quads (A/B)
#endif
#ifndef EZRT_IS_DEDUPE
#define EZRT_IS_DEDUPE 0    // IS/MIS integrator: 1 = evaluate the BRDF of the light and the BRDF sample in one non-unrolled loop
#endif
#ifndef EZRT_SMEM_STACK
#define EZRT_SMEM_STACK 0   // stack entries kept in shared memory (experiment; 0 = all in local memory)
#endif
#ifndef EZRT_NODE_PREFETCH
#define EZRT_NODE_PREFETCH 0   // 1: prefetch the next 4-wide node into L1 as soon as it is chosen (experiment)
#endif
#ifndef EZRT_WIDE_SORT
#define EZRT_WIDE_SORT 1    // 1: fully sort the children of a 4-wide node before pushing; 0: nearest first, the others
                            // unsorted (CPU model: +1 % visits, 20 instructions less per visit)
#endif
#define EZRT_REF_DONE ((int)0x80000000)   // leaf flag with n == 0: no real leaf has this encoding

// the tree a persistent traversal walks: the reference tree or the device's acceleration tree
struct TreeView {
    const float4* nodes;     // binary records (64 B), or 4-wide records (128 B) when `wide`
    const float4* tri_geo;
    int root_ref;
    int top_nodes;
    int wide;
};

// Would the shader's hitBVH have reached the leaf that holds reference triangle `ref_tri`?  Yes iff
// the leaf's own box passes hitAABB > 0: the fp32 slab values are monotone in the box bounds
// (rounding is monotone), every ancestor box contains the leaf box, so it passes whenever the leaf
// does (DESIGN.md "accel").  Exact hitAABB arithmetic; only called for rays with finite 1/d.
__device__ __forceinline__ bool reference_reaches_leaf(const int* __restrict__ tri_leaf, const float4* __restrict__ leaf_box, int tri, vec3 o,
                                                       const RaySlab& rs) {
    const int leaf = __ldg(tri_leaf + tri);  // tri_leaf in the same index space as `tri`
    const float4 a = ldg4(leaf_box + 2 * (size_t)leaf), b = ldg4(leaf_box + 2 * (size_t)leaf + 1);
    float ix, iy, iz, iz2;
    pk2_split(rs.inv_xy, ix, iy);
    pk2_split(rs.inv_zz, iz, iz2);
    float fx = (b.x - o.x) * ix, fy = (b.y - o.y) * iy, fz = (b.z - o.z) * iz;
    float nx = (a.x - o.x) * ix, ny = (a.y - o.y) * iy, nz = (a.z - o.z) * iz;
    float t1 = fminf(fmaxf(fx, nx), fminf(fmaxf(fy, ny), fmaxf(fz, nz)));
    float t0 = fmaxf(fminf(fx, nx), fmaxf(fminf(fy, ny), fminf(fz, nz)));
    float d = (t1 >= t0) ? ((t0 > 0.0f) ? t0 : t1) : -1.0f;
    return d > 0.0f;
}

// the same test on a leaf index the caller fetched earlier (tri_leaf[tri]), so that the two dependent loads need not be waited on together
__device__ __forceinline__ bool reference_reaches_leaf_box(const float4* __restrict__ leaf_box, int leaf, vec3 o, vec3 inv) {
    const float4 a = ldg4(leaf_box + 2 * (size_t)leaf), b = ldg4(leaf_box + 2 * (size_t)leaf + 1);
    float fx = (b.x - o.x) * inv.x, fy = (b.y - o.y) * inv.y, fz = (b.z - o.z) * inv.z;
    float nx = (a.x - o.x) * inv.x, ny = (a.y - o.y) * inv.y, nz = (a.z - o.z) * inv.z;
    float t1 = fminf(fmaxf(fx, nx), fminf(fmaxf(fy, ny), fmaxf(fz, nz)));
    float t0 = fmaxf(fminf(fx, nx), fmaxf(fminf(fy, ny), fminf(fz, nz)));
    float d = (t1 >= t0) ? ((t0 > 0.0f) ? t0 : t1) : -1.0f;
    return d > 0.0f;
}

__device__ __forceinline__ bool reference_reaches_leaf_inv(const int* __restrict__ tri_leaf, const float4* __restrict__ leaf_box, int tri, vec3 o, vec3 inv) {
    return reference_reaches_leaf_box(leaf_box, __ldg(tri_leaf + tri), o, inv);
}

// ACCEL: `tree` is the device's own acceleration tree, not the reference tree: the closest hit it
// finds is the global minimum over all triangles; ties (two triangles at exactly the same t) and rays
// with non-finite 1/d are handed to io.defer() and re-traced by the exact reference-order kernel.
struct W8Counts {   // COUNT instantiations only (bench.py roofline: records fetched on the kernel's own layout)
    unsigned long long* node_visits;
    unsigned long long* tri_tests;
};

// BOUNDED (shadow rays of the light sampling mode): ray i starts with best = io.tmax(i) instead of EZ_INF, so a triangle occludes
// only if it is accepted strictly before tmax.  A hit at exactly tmax is not accepted: it must not end an any-hit traversal.
template <bool BOUNDED, class RayIO>
__device__ __forceinline__ float ray_tmax(const RayIO& io, uint32_t i) {
    if constexpr (BOUNDED) return io.tmax(i);
    else return EZ_INF;
}

template <bool PRUNE, bool ANYHIT, bool ACCEL, bool WIDE, int LL, bool COUNT, bool Q16, bool BOUNDED = false, class RayIO>
__device__ __forceinline__ void extend_persistent(const SceneDev& sc, const TreeView tree, uint32_t n, uint32_t* work, RayIO io,
                                                  const float4* smem_top, W8Counts counts = W8Counts{nullptr, nullptr}, int refill_override = 0,
                                                  int chunk_override = 0) {
    unsigned long long n_visits = 0, n_tests = 0;
    const int top_nodes = tree.top_nodes;
    const bool tri_na = sc.tri_l1_bypass != 0;
    __shared__ unsigned char s_owner_all[(EZRT_EXTEND_MAX_THREADS / 32) * 8];   // leaf phase: rank -> owner lane, 8 bytes per warp
    unsigned char* const s_owner = s_owner_all + (threadIdx.x >> 5) * 8;
    bool tie = false;          // ACCEL: another triangle was accepted at exactly the best distance
    const int refill_thresh = refill_override ? refill_override : sc.refill_thresh;  // go back to refill when fewer lanes than this are busy
    const int inner_thresh = sc.inner_thresh;    // leave the inner-node phase when fewer lanes than this walk
    const int leaf_thresh = sc.leaf_thresh;      // ... or when at least this many lanes wait at a leaf
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const unsigned lt_mask = (1u << lane) - 1u;
    // stack of (child reference, slab entry distance bits).  Entries below EZRT_SMEM_STACK live in shared
    // memory at [entry][thread] (a lane always hits its own banks: 2 wavefronts per warp access however the
    // lanes' stack pointers differ), deeper ones in local memory.
    int2 stack_local[ACCEL ? EZRT_ACCEL_STACK : EZRT_MAX_STACK];
#if EZRT_SMEM_STACK > 0
    int2* const stack_sm = reinterpret_cast<int2*>(const_cast<float4*>(smem_top) + (size_t)tree.top_nodes * EZRT_TOP_STRIDE) + threadIdx.x;
    const int stack_stride = blockDim.x;
#define STACK_PUSH(e) do { const int2 e__ = (e); if (sp < EZRT_SMEM_STACK) stack_sm[sp * stack_stride] = e__; else stack_local[sp] = e__; ++sp; } while (0)
#define STACK_POP() ((--sp < EZRT_SMEM_STACK) ? stack_sm[sp * stack_stride] : stack_local[sp])
#else
#define STACK_PUSH(e) do { stack_local[sp++] = (e); } while (0)
#define STACK_POP() (stack_local[--sp])
#endif
    int sp = 0;
    int ray = -1;              // index of the ray this lane is tracing, -1 = idle
    int ref = EZRT_REF_DONE;
    vec3 o = splat3(0.0f), d = splat3(0.0f), inv = splat3(0.0f);
    RaySlab rs = make_ray_slab(o, inv);
    Q16Ray qr = make_q16_ray(d);
    float slack = 0.0f, best = EZ_INF;
    int best_tri = -1;
    bool exhausted = false;    // warp-uniform: the work counter has run past n
    uint32_t chunk_pos = 0, chunk_end = 0;  // warp-uniform: this warp's current range of ray indices
    const uint32_t chunk = (uint32_t)(chunk_override ? chunk_override : sc.work_chunk);

    while (true) {
        // ---------------- refill idle lanes ----------------
        // Work is taken in per-warp chunks of `chunk` consecutive rays (one atomicAdd per chunk): the
        // lanes of a warp keep tracing neighbours of the (sorted) ray order even as they refill.
        unsigned need = __ballot_sync(FULL, ray < 0);
        if (need != 0u && !exhausted) {
            if (chunk_pos >= chunk_end) {
                uint32_t base = 0;
                if (lane == 0) base = atomicAdd(work, chunk);
                base = __shfl_sync(FULL, base, 0);
                chunk_pos = base;
                chunk_end = (base + chunk < n) ? base + chunk : n;
                if (base >= n) exhausted = true;
            }
            if (!exhausted && ray < 0) {
                uint32_t idx = chunk_pos + (uint32_t)__popc(need & lt_mask);
                if (idx < chunk_end && io.load(idx, o, d)) {
                    inv = ez_v3(EZ_DIV(1.0f, d.x), EZ_DIV(1.0f, d.y), EZ_DIV(1.0f, d.z));
                    float ax = ez_abs(inv.x), ay = ez_abs(inv.y), az = ez_abs(inv.z);
                    slack = sc.prune_delta * ez_max(ax, ez_max(ay, az));
                    bool traceable = (ax < 3.0e38f) && (ay < 3.0e38f) && (az < 3.0e38f);
                    if (Q16) {   // the quantised planes are conservative only within the decode error bound (w8_node.h): the rest goes to the exact kernel
                        const float ao = fmaxf(ez_abs(o.x), fmaxf(ez_abs(o.y), ez_abs(o.z)));
                        traceable = traceable && (fmaxf(ax, fmaxf(ay, az)) <= sc.quant_inv_limit) && (fminf(ax, fminf(ay, az)) >= W8_INV_MIN) && (ao <= sc.w8_origin_limit);
                    }
                    if (traceable) {
                        rs = make_ray_slab(o, inv);
                        if (Q16) qr = make_q16_ray(d);
                        ray = (int)idx;
                        ref = tree.root_ref;
                        sp = 0;
                        best = ray_tmax<BOUNDED>(io, idx);
                        best_tri = -1;
                        tie = false;
                    } else if (ACCEL) {  // exact kernel handles the literal ternary min/max path
                        io.defer(idx, o, d);
                    } else {  // a zero / NaN direction component: literal ternary min/max path (rare)
                        io.store(idx, trace_impl<PRUNE, ANYHIT, false>(sc, o, d, inv, slack, ray_tmax<BOUNDED>(io, idx)), false, o, d, inv);
                    }
                }
            }
            if (!exhausted) {
                uint32_t take = (uint32_t)__popc(need);
                chunk_pos = (chunk_pos + take < chunk_end) ? chunk_pos + take : chunk_end;
            }
        }
        if (__ballot_sync(FULL, ray >= 0) == 0u) {
            if (exhausted) break;
            continue;
        }
        // ---------------- traverse ----------------
        // Two warp-synchronous phases per macro-step ("while-while" with votes):
        //   inner phase: lanes standing at an inner node visit it, one node per iteration, for as
        //                long as at least `inner_thresh` lanes want to (lanes that reached a leaf or
        //                finished wait) -- or until nobody waits at a leaf;
        //   leaf phase : every lane standing at a leaf tests its triangles and pops.
        // Measured before this split: 70% of all issued instructions were inner-node
        // visits running at 5.8 of 32 lanes, because the warp waited for its longest walk per leaf.
        unsigned busy;
        do {
            const unsigned m_busy = __ballot_sync(FULL, ray >= 0);  // constant during the inner phase
            while (true) {
                const bool at_inner = (ray >= 0) && (ref >= 0);
                const unsigned m_inner = __ballot_sync(FULL, at_inner);
                if (m_inner == 0u) break;
                const unsigned m_wait = m_busy & ~m_inner;  // busy lanes standing at a leaf (or done)
                if (m_wait != 0u && (__popc(m_inner) < inner_thresh || __popc(m_wait) >= leaf_thresh)) break;
                if (WIDE) {
                    if (at_inner) {  // 4-wide acceleration-tree node: nearest child next, the others pushed far-to-near
                        const float limit = best + (best * 0.000244140625f + slack);
                        const WideVisit w = Q16 ? wide_visit_q16(sc.acc_wide_q16 + (size_t)ref * 6, o, rs, limit, sc.q16_decode_bits, qr)
                                                : wide_visit(tree.nodes + (size_t)ref * 8, rs, limit);
                        if (COUNT) n_visits++;
#if EZRT_WIDE_SORT
                        WideVisit v = w;
                        cswap(v.k0, v.r0, v.k1, v.r1);
                        cswap(v.k2, v.r2, v.k3, v.r3);
                        cswap(v.k0, v.r0, v.k2, v.r2);
                        cswap(v.k1, v.r1, v.k3, v.r3);
                        cswap(v.k1, v.r1, v.k2, v.r2);
                        if (v.k3 < 3.0e38f) STACK_PUSH(make_int2(v.r3, __float_as_int(v.k3)));
                        if (v.k2 < 3.0e38f) STACK_PUSH(make_int2(v.r2, __float_as_int(v.k2)));
                        if (v.k1 < 3.0e38f) STACK_PUSH(make_int2(v.r1, __float_as_int(v.k1)));
                        const bool descend = v.k0 < 3.0e38f;
                        const int next = v.r0;
#else
                        const float km = fminf(fminf(w.k0, w.k1), fminf(w.k2, w.k3));
                        const bool descend = km < 3.0e38f;
                        const int m = (w.k0 == km) ? 0 : (w.k1 == km) ? 1 : (w.k2 == km) ? 2 : 3;
                        if (m != 0 && w.k0 < 3.0e38f) STACK_PUSH(make_int2(w.r0, __float_as_int(w.k0)));
                        if (m != 1 && w.k1 < 3.0e38f) STACK_PUSH(make_int2(w.r1, __float_as_int(w.k1)));
                        if (m != 2 && w.k2 < 3.0e38f) STACK_PUSH(make_int2(w.r2, __float_as_int(w.k2)));
                        if (m != 3 && w.k3 < 3.0e38f) STACK_PUSH(make_int2(w.r3, __float_as_int(w.k3)));
                        const int next = (m == 0) ? w.r0 : (m == 1) ? w.r1 : (m == 2) ? w.r2 : w.r3;
#endif
                        if (descend) {
                            ref = next;
#if EZRT_NODE_PREFETCH
                            if (next >= 0) {   // the next node record (Q16: 96 bytes, may straddle two lines) ...
                                if (Q16) {
                                    asm volatile("prefetch.global.L1 [%0];" ::"l"(sc.acc_wide_q16 + (size_t)next * 6));
                                    asm volatile("prefetch.global.L1 [%0];" ::"l"(sc.acc_wide_q16 + (size_t)next * 6 + 4));
                                } else {
                                    asm volatile("prefetch.global.L1 [%0];" ::"l"(tree.nodes + (size_t)next * 8));
                                }
                            }
#if EZRT_NODE_PREFETCH >= 2
                            else if (next != EZRT_REF_DONE) {   // ... or the first triangles of the leaf this lane will wait at
                                const uint32_t lb = (uint32_t)next & 0x7fffffffu;
                                asm volatile("prefetch.global.L2 [%0];" ::"l"(tree.tri_geo + (size_t)(lb >> 7) * 4));
                                asm volatile("prefetch.global.L2 [%0];" ::"l"(tree.tri_geo + (size_t)(lb >> 7) * 4 + 8));
                            }
#endif
#endif
                        } else {  // pop
                            ref = EZRT_REF_DONE;
                            while (sp > 0) {
                                const int2 e = STACK_POP();
                                if (prune_test(__int_as_float(e.y), best, slack)) continue;
                                ref = e.x;
                                break;
                            }
                        }
                    }
                } else if (at_inner) {
                    NodeVisit nv = node_visit_top<true>(tree.nodes, smem_top, top_nodes, ref, rs);
                    bool h1 = nv.h1, h2 = nv.h2;
                    const float d1 = nv.d1, d2 = nv.d2, e1 = nv.e1, e2 = nv.e2;
                    const int rl = nv.rl, rr = nv.rr;
                    if (PRUNE) {
                        if (h1 && prune_test(e1, best, slack)) h1 = false;
                        if (h2 && prune_test(e2, best, slack)) h2 = false;
                    }
                    if (h1 && h2) {
                        bool leftFirst = d1 < d2;
                        STACK_PUSH(make_int2(leftFirst ? rr : rl, __float_as_int(leftFirst ? e2 : e1)));
                        ref = leftFirst ? rl : rr;
                    } else if (h1) {
                        ref = rl;
                    } else if (h2) {
                        ref = rr;
                    } else {  // pop
                        ref = EZRT_REF_DONE;
                        while (sp > 0) {
                            const int2 e = STACK_POP();
                            if (PRUNE && prune_test(__int_as_float(e.y), best, slack)) continue;
                            ref = e.x;
                            break;
                        }
                    }
                }
            }
            // ---- leaf phase, warp-cooperative: the warp takes up to G = 32/LL waiting leaves at a time and gives
            // each a group of LL lanes, one triangle per lane (LL = 8: leaves of reference-built trees hold <= 8
            // triangles; LL = 4: the acceleration tree built with leaves <= 4 -- a ray visits ~2.5 leaves whatever
            // their size, so twice the leaves per pass halves the passes; longer leaves take several passes).
            // The owner's ray travels by shuffle; the group's winning distance is a log2(LL)-step integer min of
            // the t bits (t > 0, so bit order = value order) and the winning triangle is the lowest lane holding
            // it -- hitArray's "strictly closer, first index wins" rule (P5/fsh:242-249); more than one holder,
            // or a hit at exactly the old best, is a tie (ACCEL).
            constexpr int G = 32 / LL;
            const bool at_leaf = (ray >= 0) && (ref < 0) && (ref != EZRT_REF_DONE);
            unsigned m_leaf = __ballot_sync(FULL, at_leaf);
            const uint32_t my_bits = (uint32_t)ref & 0x7fffffffu;
            int leaf_cnt = at_leaf ? (int)(my_bits & 127u) : 0;
            int leaf_first = (int)(my_bits >> 7);
            const bool long_leaves = __ballot_sync(FULL, leaf_cnt > LL) != 0u;
            bool stop = false;
            const int q = lane / LL, k = lane % LL;
#if EZRT_LEAF_SERIAL   // experiment: every lane tests the triangles of its own leaf one after the other (accel kernels, leaves <= 4)
            if (ACCEL) {
                m_leaf = 0u;
                int cnt = leaf_cnt, first = leaf_first;
                while (__ballot_sync(FULL, cnt > 0 && !stop) != 0u) {
                    if (cnt > 0 && !stop) {
                        float t;
                        if (COUNT) n_tests++;
                        const int r = tri_test_t<true>(tree.tri_geo + (size_t)first * 4, o, d, best, t, tri_na);
                        if (r == 2) tie = true;
                        else if (r == 1) { best = t; best_tri = first; if (ANYHIT) stop = true; }
                        first++;
                        cnt--;
                    }
                }
            }
#endif
            while (m_leaf != 0u) {
                // the G lowest waiting lanes own this pass: lane with rank g (g-th set bit of m_leaf) serves group g.  The
                // rank -> lane map goes through a few bytes of shared memory (one STS / LDS per pass; the unrolled
                // find-first-set loop it replaces was 16 % of the kernel's instructions)
                const int my_rank = __popc(m_leaf & lt_mask);
                const unsigned taken = __ballot_sync(FULL, ((m_leaf >> lane) & 1u) != 0u && my_rank < G);   // the G lowest waiting lanes
                const unsigned rest = m_leaf & ~taken;
                __syncwarp();
                if ((taken >> lane) & 1u) s_owner[my_rank] = (unsigned char)lane;
                __syncwarp();
                const int owner = (q < __popc(taken)) ? (int)s_owner[q] : -1;
                m_leaf = rest;
                const int src = (owner < 0) ? lane : owner;
                vec3 ro, rdir;
                ro.x = __shfl_sync(FULL, o.x, src); ro.y = __shfl_sync(FULL, o.y, src); ro.z = __shfl_sync(FULL, o.z, src);
                rdir.x = __shfl_sync(FULL, d.x, src); rdir.y = __shfl_sync(FULL, d.y, src); rdir.z = __shfl_sync(FULL, d.z, src);
                const float rbest = __shfl_sync(FULL, best, src);
                const int rfirst = __shfl_sync(FULL, leaf_first, src);
                const int rcnt = __shfl_sync(FULL, leaf_cnt, src);
                unsigned tb = 0xffffffffu;  // t bits of this lane's triangle, or "no hit"
                if (owner >= 0 && k < rcnt) {
                    float t;
                    if (COUNT) n_tests++;
                    if (tri_test_t<ACCEL>(tree.tri_geo + (size_t)(rfirst + k) * 4, ro, rdir, rbest, t, tri_na) != 0) tb = __float_as_uint(t);
                }
                unsigned mn = tb;
                mn = min(mn, __shfl_xor_sync(FULL, mn, 1));
                mn = min(mn, __shfl_xor_sync(FULL, mn, 2));
                if (LL == 8) mn = min(mn, __shfl_xor_sync(FULL, mn, 4));
                const unsigned win = __ballot_sync(FULL, tb == mn && tb != 0xffffffffu);  // holders of the winning distance
                const int pos = ((taken >> lane) & 1u) ? __popc(taken & lt_mask) : -1;    // which group served this lane's leaf
                const unsigned res = __shfl_sync(FULL, mn, (pos < 0) ? lane : pos * LL);
                if (pos >= 0) {  // this lane owns one of the leaves just tested
                    const unsigned mq = (win >> (LL * pos)) & ((1u << LL) - 1u);
                    if (mq != 0u) {
                        const float tn = __uint_as_float(res);
                        const bool strict = !ACCEL || tn < best;
                        if (ACCEL && (__popc(mq) > 1 || tn == best)) tie = true;
                        if (strict) {  // ACCEL accepts t == best only to flag the tie
                            best = tn;
                            best_tri = leaf_first + __ffs(mq) - 1;
                        }
                        if (ANYHIT && (!BOUNDED || strict)) stop = true;   // bounded: a hit at exactly tmax does not end the ray
                    }
                    leaf_first += LL;
                    leaf_cnt -= LL;
                }
                if (long_leaves) m_leaf |= __ballot_sync(FULL, pos >= 0 && leaf_cnt > 0 && !stop);  // next pass of a long leaf
            }
            if (at_leaf) {  // pop (hitBVH continues with the next stack entry)
                ref = EZRT_REF_DONE;
                if (!stop) {
                    while (sp > 0) {
                        const int2 e = STACK_POP();
                        if (PRUNE && prune_test(__int_as_float(e.y), best, slack)) continue;
                        ref = e.x;
                        break;
                    }
                }
            }
            if (ray >= 0 && ref == EZRT_REF_DONE) {  // ray finished
                HitRec h;
                h.t = best;
                h.tri = best_tri;
                float ix, iy, iz, iz2;   // 1/d lives in the slab constants (no extra registers across the loop)
                pk2_split(rs.inv_xy, ix, iy);
                pk2_split(rs.inv_zz, iz, iz2);
                io.store((uint32_t)ray, h, tie, o, d, ez_v3(ix, iy, iz));
                ray = -1;
            }
            busy = __ballot_sync(FULL, ray >= 0);
        } while (busy != 0u && (exhausted || __popc(busy) >= refill_thresh));
    }
    if (COUNT) {
        atomicAdd(counts.node_visits, n_visits);
        atomicAdd(counts.tri_tests, n_tests);
    }
}

#undef STACK_PUSH
#undef STACK_POP

// ------------------------------------------------------------------------------------------
// W8: the default traversal of the accel policy.  8-wide nodes with 8-bit quantised child boxes (80-byte records,
// five 128-bit loads; layout, decode arithmetic and error bound in w8_node.h), children visited in octant order
// from a hit bit mask -- no distance sort, at most one stack push per node visit -- and a per-lane stack of
// (child base | slot masks) groups in SHARED memory at [entry][thread].  The triangles of all hit leaf slots of a node
// are collected in a bit mask; a triangle step tests up to 32 of the warp's pending triangles, one per lane, whichever
// lanes they belong to.
// Like the 4-wide kernel it only has to find the globally closest accepted triangle (and notice ties); what it
// cannot decide exactly goes to io.defer() (DESIGN.md section 4).  Measured ceiling for its access pattern on an H100: at
// most one divergent 128-bit load per lane per SM-cycle (tools/gather_bench.cu, DESIGN.md section 4).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
    return r;
}
// byte K of `w` -> the float 2^15 + q (w8_node.h "Decode").  `bias` = W8_DECODE_BITS held in a REGISTER so that the
// selector can be the instruction's immediate (with the constant as immediate ptxas moves 46 selectors per node visit
// through registers).
template <int K>
__device__ __forceinline__ float w8_plane(uint32_t w, uint32_t bias) {
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(w), "r"(bias), "n"(0x7604 | (K << 4)));
    return __uint_as_float(r);
}
// one slot: entry / exit distances from the six decoded planes; hit iff the clamped interval is non-empty
template <int K>
__device__ __forceinline__ bool w8_slot_hit(uint32_t nx, uint32_t ny, uint32_t nz, uint32_t fx, uint32_t fy, uint32_t fz, float Bx, float By, float Bz,
                                            float Ax, float Ay, float Az, float limit, uint32_t bias) {
    const float tnx = __fmaf_rn(w8_plane<K>(nx, bias), Bx, Ax), tny = __fmaf_rn(w8_plane<K>(ny, bias), By, Ay), tnz = __fmaf_rn(w8_plane<K>(nz, bias), Bz, Az);
    const float tfx = __fmaf_rn(w8_plane<K>(fx, bias), Bx, Ax), tfy = __fmaf_rn(w8_plane<K>(fy, bias), By, Ay), tfz = __fmaf_rn(w8_plane<K>(fz, bias), Bz, Az);
    const float tmin = fmaxf(fmaxf(tnx, tny), fmaxf(tnz, 0.0f));
    const float tmax = fminf(fminf(tfx, tfy), fminf(tfz, limit));
    return tmin <= tmax;
}

// position of the r-th lowest set bit of m (r < popc(m))
__device__ __forceinline__ int nth_set_bit(uint32_t m, int r) {
    int pos = 0, c = __popc(m & 0xffffu);
    if (r >= c) { r -= c; m >>= 16; pos += 16; }
    c = __popc(m & 0xffu);
    if (r >= c) { r -= c; m >>= 8; pos += 8; }
    c = __popc(m & 0xfu);
    if (r >= c) { r -= c; m >>= 4; pos += 4; }
    c = __popc(m & 0x3u);
    if (r >= c) { r -= c; m >>= 2; pos += 2; }
    return pos + ((r >= (int)(m & 1u)) ? 1 : 0);
}

// SM clock for the phase sums of the COUNT instantiations; the memory clobber keeps the compiler from moving loads and stores across it
__device__ __forceinline__ uint32_t w8_clock() {
    uint32_t t;
    asm volatile("mov.u32 %0, %%clock;" : "=r"(t) : : "memory");
    return t;
}

// s_perm: 8 x 256 bytes in shared memory, s_perm[m * 256 + x] = the bits of x moved from position s to position s ^ m
// stack : uint2 [entries][blockDim.x] in shared memory
// IDX: the scene's triangle records are indexed (SceneDev::acc_tri_indexed; one instantiation per layout keeps each within 64
// registers without spilling)
#define W8_ENDED (-2)   // extend_w8: `node` of a lane whose ray is traced and waits for its leaf check at the next refill
// phase_cycles (COUNT only): += the SM cycles each warp spends in [0] refill, [1] node steps, [2] triangle steps, [3] ray ends,
// then the warp's [4] node steps and [5] triangle steps and its lanes' [6] node visits and [7] triangle tests
template <bool ANYHIT, bool COUNT, bool IDX, bool BOUNDED = false, class RayIO>
__device__ __forceinline__ void extend_w8(const SceneDev& sc, uint32_t n, uint32_t* work, RayIO io, const unsigned char* s_perm, uint2* stack_sm,
                                          W8Counts counts, unsigned long long* phase_cycles) {
    const bool tri_na = sc.tri_l1_bypass != 0;
    const int refill_thresh = sc.refill_thresh, leaf_thresh = sc.w8_tri_weight;
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const unsigned lt_mask = (1u << lane) - 1u;
    const int stack_stride = blockDim.x;
    const int stack_cap = sc.w8_stack_entries;
    uint2 stack_local[W8_LOCAL_STACK];   // entries beyond the shared-memory part (trees deeper than the smem stack)
    uint2* const my_stack = stack_sm + threadIdx.x;
    const uint4* __restrict__ nodes = sc.w8_nodes;
    const float origin_limit = sc.w8_origin_limit, inv_limit = sc.quant_inv_limit;
    const uint32_t bias = sc.w8_decode_bits;   // = W8_DECODE_BITS; a run-time value so that ptxas keeps it in a register (see w8_plane)
    __shared__ unsigned char s_owner_all[EZRT_EXTEND_MAX_THREADS];   // triangle step: first tested pair -> owner lane, 32 bytes per warp
    unsigned char* const s_owner = s_owner_all + (threadIdx.x & ~31u);

    int ray = -1;                 // index of the ray this lane traces, -1 = idle
    int node = -1;                // next node to visit, -1 = none (waiting for the triangle phase, or idle), W8_ENDED = ray traced
    int end_leaf = 0;             // W8_ENDED: reference leaf of best_tri, loaded at the ray's end and first read at the next refill
    int sp = 0;
    vec3 o = splat3(0.0f), d = splat3(0.0f), inv = splat3(0.0f);
    float slack = 0.0f, best = EZ_INF;
    int best_tri = -1;
    bool tie = false;
    uint32_t near_mask = 0;       // bit of axis a set iff d_a >= 0 (children towards -a come first)
    uint32_t g_base = 0, g_bits = 0;   // current group: first inner child | imask (bits 0..7), unvisited hit slots in priority positions (bits 8..15)
    uint32_t t_base = 0, t_mask = 0;   // pending triangles of the node just visited
    uint32_t n_visits = 0, n_tests = 0;   // per lane; 32 bits keep the COUNT instantiations within 64 registers
    uint32_t cyc_refill = 0, cyc_node = 0, cyc_tri = 0, cyc_end = 0;   // COUNT: the warp's phase sums (phase_cycles)
    uint32_t n_node_steps = 0, n_tri_steps = 0;                        // COUNT: the warp's steps of each kind
    uint32_t end_dt = 0, t_mark = COUNT ? w8_clock() : 0u;             // COUNT: this lane's ray-end span; end of the last phase
    bool exhausted = false;
    uint32_t chunk_pos = 0, chunk_end = 0;
    const uint32_t chunk = (uint32_t)sc.work_chunk;

#define W8_PUSH(e) do { const uint2 e__ = (e); if (sp < stack_cap) my_stack[sp * stack_stride] = e__; else stack_local[sp - stack_cap] = e__; ++sp; } while (0)
#define W8_POP() ((--sp < stack_cap) ? my_stack[sp * stack_stride] : stack_local[sp - stack_cap])
    // next node of this lane's ray from the current group / the stack; finishes the ray when nothing is left
    // A finished ray's leaf check (io.store) is two dependent loads.  Waited on where the ray ends, they would stall every lane of
    // the warp in most steps; so the ray only issues the first load here and becomes W8_ENDED (no longer busy, not yet idle), and
    // the next refill, which waits on memory anyway, finishes it with io.finish before it takes a new ray.
    auto select_next = [&]() {
        if ((g_bits >> 8) == 0u) {
            if (sp == 0) {  // ray finished
                const uint32_t te = COUNT ? w8_clock() : 0u;
                if (best_tri >= 0) end_leaf = io.leaf_of(best_tri);
                if (COUNT) end_dt = w8_clock() - te;
                node = W8_ENDED;
                return;
            }
            const uint2 e = W8_POP();
            g_base = e.x;
            g_bits = e.y;
        }
        const int p = 23 - __clz(g_bits);                  // highest priority position among bits 8..15
        g_bits ^= 0x100u << p;
        const uint32_t slot = (uint32_t)p ^ near_mask;
        node = (int)(g_base + __popc(g_bits & 0xffu & ((1u << slot) - 1u)));
    };

    while (true) {
        // ---------------- refill idle lanes (per-warp chunks of the global work counter, as extend_persistent) ----------------
        const bool ended = node == W8_ENDED;
        const unsigned need = __ballot_sync(FULL, ray < 0 || ended);
        const bool claim = need != 0u && !exhausted && chunk_pos >= chunk_end;
        uint32_t base = 0;
        if (claim && lane == 0) base = atomicAdd(work, chunk);   // issued before the leaf checks, so that their round trips overlap
        if (ended) {
            HitRec h;
            h.t = best;
            h.tri = best_tri;
            const uint32_t te = COUNT ? w8_clock() : 0u;
            io.finish((uint32_t)ray, h, tie, o, d, inv, end_leaf);
            if (COUNT) end_dt = w8_clock() - te;
            ray = -1;
            node = -1;
        }
        if (need != 0u && !exhausted) {
            if (claim) {
                base = __shfl_sync(FULL, base, 0);
                chunk_pos = base;
                chunk_end = (base + chunk < n) ? base + chunk : n;
                if (base >= n) exhausted = true;
            }
            if (!exhausted && ray < 0) {
                uint32_t idx = chunk_pos + (uint32_t)__popc(need & lt_mask);
                if (idx < chunk_end && io.load(idx, o, d)) {
                    inv = ez_v3(EZ_DIV(1.0f, d.x), EZ_DIV(1.0f, d.y), EZ_DIV(1.0f, d.z));
                    const float ax = ez_abs(inv.x), ay = ez_abs(inv.y), az = ez_abs(inv.z);
                    const float ao = fmaxf(ez_abs(o.x), fmaxf(ez_abs(o.y), ez_abs(o.z)));
                    const float amin = fminf(ax, fminf(ay, az)), amax = fmaxf(ax, fmaxf(ay, az));
                    if ((amax <= inv_limit) && (amin >= W8_INV_MIN) && (ao <= origin_limit)) {  // false for inf / NaN
                        slack = sc.prune_delta * ez_max(ax, ez_max(ay, az));
                        near_mask = (d.x >= 0.0f ? (1u << sc.w8_near_bit[0]) : 0u) | (d.y >= 0.0f ? (1u << sc.w8_near_bit[1]) : 0u) |
                                    (d.z >= 0.0f ? (1u << sc.w8_near_bit[2]) : 0u);
                        ray = (int)idx;
                        node = 0;
                        sp = 0;
                        g_bits = 0u;
                        t_mask = 0u;
                        best = ray_tmax<BOUNDED>(io, idx);   // bounded: a hit at exactly tmax is a tie, which does not end the ray
                        best_tri = -1;
                        tie = false;
                    } else {  // outside the decode error bound: the exact kernel traces it
                        io.defer(idx, o, d);
                    }
                }
            }
            if (!exhausted) {
                uint32_t take = (uint32_t)__popc(need);
                chunk_pos = (chunk_pos + take < chunk_end) ? chunk_pos + take : chunk_end;
            }
        }
        if (COUNT) {
            const uint32_t now = w8_clock(), e = __reduce_max_sync(FULL, end_dt);   // the leaf checks of the ended rays run side by side
            end_dt = 0u;
            cyc_end += e;
            cyc_refill += now - t_mark - e;
            t_mark = now;
        }
        if (__ballot_sync(FULL, ray >= 0) == 0u) {
            if (exhausted) break;
            continue;
        }
        // ---------------- traverse: every iteration the warp runs ONE of two steps, chosen by a vote ----------------
        //   node step     : every lane holding a node visits it (five 128-bit loads, eight slab tests; ~200 instructions)
        //   triangle step : the warp tests up to 32 pending (lane, triangle) pairs, one per lane (one 128-bit load, three more
        //                   past the distance checks, plus the shuffles that hand out the pairs)
        // A lane with pending triangles cannot take a node step (its next node depends on them), so the warp takes the
        // triangle step as soon as  tri_weight * min(pending pairs, 32) >= (lanes with a node).  A node step costs about two
        // triangle steps, but a triangle step also frees its lanes for the next node step: 1 measured best (env EZRT_TRI_W).
        const int tri_weight = leaf_thresh;
        unsigned busy;
        do {
            const bool at_node = node >= 0;
            const unsigned m_node = __ballot_sync(FULL, at_node);
            const uint32_t pairs = __reduce_add_sync(FULL, (uint32_t)__popc(t_mask));
            if (m_node == 0u && pairs == 0u) { busy = 0u; break; }
            const bool node_step = m_node != 0u && tri_weight * (int)min(pairs, 32u) < __popc(m_node);
            if (node_step) {
                if (at_node) {
                    // the 20 words of the record (w8_node.h): h = w0..3, c = w4..7, l = w8..11, m = w12..15, u = w16..19
                    const uint4* nd = nodes + (size_t)node * (W8_NODE_WORDS / 4);
                    const uint4 h = ldg128_u32(nd), c = ldg128_u32(nd + 1), l = ldg128_u32(nd + 2), m = ldg128_u32(nd + 3), u = ldg128_u32(nd + 4);
                    if (COUNT) n_visits++;
                    const float limit = best + (best * 0.000244140625f + slack);
                    // B = scale * inv, A = fma(-2^15, B, (origin - o) * inv)
                    const float Bx = __uint_as_float(W8_SCALE_BITS(h.w, 0)) * inv.x, By = __uint_as_float(W8_SCALE_BITS(h.w, 1)) * inv.y,
                                Bz = __uint_as_float(W8_SCALE_BITS(h.w, 2)) * inv.z;
                    const float Ax = __fmaf_rn(-W8_DECODE_BIAS, Bx, (__uint_as_float(h.x) - o.x) * inv.x);
                    const float Ay = __fmaf_rn(-W8_DECODE_BIAS, By, (__uint_as_float(h.y) - o.y) * inv.y);
                    const float Az = __fmaf_rn(-W8_DECODE_BIAS, Bz, (__uint_as_float(h.z) - o.z) * inv.z);
                    // near / far plane words per axis (slots 0..3 | 4..7): low planes are near iff d >= 0
                    // qlo_x = c.z, c.w  qlo_y = l.x, l.y  qlo_z = l.z, l.w   qhi_x = m.z, m.w  qhi_y = u.x, u.y  qhi_z = u.z, u.w
                    const bool px = d.x >= 0.0f, py = d.y >= 0.0f, pz = d.z >= 0.0f;
                    const uint32_t nx0 = px ? c.z : m.z, nx1 = px ? c.w : m.w, fx0 = px ? m.z : c.z, fx1 = px ? m.w : c.w;
                    const uint32_t ny0 = py ? l.x : u.x, ny1 = py ? l.y : u.y, fy0 = py ? u.x : l.x, fy1 = py ? u.y : l.y;
                    const uint32_t nz0 = pz ? l.z : u.z, nz1 = pz ? l.w : u.w, fz0 = pz ? u.z : l.z, fz1 = pz ? u.w : l.w;
                    uint32_t hits = 0u;
                    if (w8_slot_hit<0>(nx0, ny0, nz0, fx0, fy0, fz0, Bx, By, Bz, Ax, Ay, Az, limit, bias)) hits |= 1u;
                    if (w8_slot_hit<1>(nx0, ny0, nz0, fx0, fy0, fz0, Bx, By, Bz, Ax, Ay, Az, limit, bias)) hits |= 2u;
                    if (w8_slot_hit<2>(nx0, ny0, nz0, fx0, fy0, fz0, Bx, By, Bz, Ax, Ay, Az, limit, bias)) hits |= 4u;
                    if (w8_slot_hit<3>(nx0, ny0, nz0, fx0, fy0, fz0, Bx, By, Bz, Ax, Ay, Az, limit, bias)) hits |= 8u;
                    if (w8_slot_hit<0>(nx1, ny1, nz1, fx1, fy1, fz1, Bx, By, Bz, Ax, Ay, Az, limit, bias)) hits |= 16u;
                    if (w8_slot_hit<1>(nx1, ny1, nz1, fx1, fy1, fz1, Bx, By, Bz, Ax, Ay, Az, limit, bias)) hits |= 32u;
                    if (w8_slot_hit<2>(nx1, ny1, nz1, fx1, fy1, fz1, Bx, By, Bz, Ax, Ay, Az, limit, bias)) hits |= 64u;
                    if (w8_slot_hit<3>(nx1, ny1, nz1, fx1, fy1, fz1, Bx, By, Bz, Ax, Ay, Az, limit, bias)) hits |= 128u;
                    const uint32_t imask = h.w >> 24;
                    const uint32_t inner = hits & imask;
                    uint32_t leaf = hits & ~imask;
                    // the rest of the group this node came from waits on the stack
                    if ((g_bits >> 8) != 0u) W8_PUSH(make_uint2(g_base, g_bits));
                    g_base = c.x;
                    g_bits = imask | ((uint32_t)s_perm[near_mask * 256u + inner] << 8);
                    // triangles of the hit leaf slots: meta byte = (count << 5) | offset
                    t_base = c.y;
                    t_mask = 0u;
                    while (leaf != 0u) {
                        const int s = __ffs(leaf) - 1;
                        leaf &= leaf - 1u;
                        const uint32_t mb = ((s < 4 ? m.x : m.y) >> ((s & 3) * 8)) & 0xffu;
                        t_mask |= ((1u << (mb >> 5)) - 1u) << (mb & 31u);
                    }
                    node = -1;
                    if (t_mask == 0u) select_next();
                }
            } else {
                // Cooperative triangle step.  The warp's pending (lane, triangle) pairs are numbered lane by lane, lowest triangle
                // first; lane j tests pair j with its owner's ray and best distance (by shuffle).  Pairs from 32 on stay pending.
                // Each owner then applies its pairs' results with the semantics of testing them one after the other in that
                // order (tri_test_t<true>: t <= best accepted, t == best reported as a tie):
                //   closest hit: m = the least accepted t.  m < best: best = m, best_tri = the first triangle holding m, tie iff
                //   a second one holds it (the serial order clears `tie` at the first holder's strict improvement and sets it
                //   again at the second).  m == best: tie.
                //   ANYHIT: the first strict hit ends the ray (with `tie` cleared); without one, a hit at exactly best is a tie.
                // The pairs are tested against the owner's best from before the step, not the best after the earlier pairs.  That
                // changes no result: a stale best is never smaller, so every triangle the serial order accepts is still accepted
                // at the same t; an extra one lies beyond the best the serial order had reached at it, so strictly above m: it
                // changes neither the minimum nor its holders.  ANYHIT rays keep best until their first strict hit: nothing is stale.
                const uint32_t cnt = (uint32_t)__popc(t_mask);
                uint32_t incl = cnt;                               // inclusive prefix sum of the pending counts
#pragma unroll
                for (int s = 1; s < 32; s <<= 1) {
                    const uint32_t v = __shfl_up_sync(FULL, incl, s);
                    if (lane >= s) incl += v;
                }
                const uint32_t first = incl - cnt;                 // this lane's pairs are numbered first, first + 1, ...
                const bool owns = cnt != 0u && first < 32u;        // ... and some of them are tested in this step
                const unsigned starts = __reduce_or_sync(FULL, owns ? 1u << first : 0u);
                __syncwarp();
                if (owns) s_owner[first] = (unsigned char)lane;   // the first lane testing an owner's pairs -> owner
                __syncwarp();
                const int start = 31 - __clz(starts & (FULL >> (31 - lane)));   // first lane of the owner this lane tests for
                const bool act = (uint32_t)lane < pairs;
                const int src = act ? (int)s_owner[start] : lane;
                vec3 ro, rd;
                ro.x = __shfl_sync(FULL, o.x, src); ro.y = __shfl_sync(FULL, o.y, src); ro.z = __shfl_sync(FULL, o.z, src);
                rd.x = __shfl_sync(FULL, d.x, src); rd.y = __shfl_sync(FULL, d.y, src); rd.z = __shfl_sync(FULL, d.z, src);
                const float rbest = __shfl_sync(FULL, best, src);
                const uint32_t rmask = __shfl_sync(FULL, t_mask, src);
                const int k = nth_set_bit(rmask, lane - start);
                const int tri = (int)__shfl_sync(FULL, t_base, src) + k;
                float t = 0.0f;
                int r = 0;
                if (act) {
                    if (COUNT) n_tests++;
                    r = IDX ? tri_test_idx_t<true>(sc.acc_tri_geo + (size_t)tri * 2, sc.acc_tri_vert, ro, rd, rbest, t, tri_na)
                            : tri_test_t<true>(sc.acc_tri_geo + (size_t)tri * 4, ro, rd, rbest, t, tri_na);
                }
                const uint32_t taken = owns ? min(cnt, 32u - first) : 0u;   // this lane's pairs tested in this step ...
                const unsigned seg = (taken == 32u) ? FULL : ((1u << taken) - 1u) << (first & 31u);   // ... by these lanes
                bool stop = false;
                if (ANYHIT) {
                    const unsigned strict = __ballot_sync(FULL, r == 1) & seg, level = __ballot_sync(FULL, r == 2) & seg;
                    const int p = strict ? __ffs(strict) - 1 : lane;
                    const float tw = __shfl_sync(FULL, t, p);
                    const int triw = __shfl_sync(FULL, tri, p);
                    if (strict) {
                        best = tw;
                        best_tri = triw;
                        tie = false;
                        stop = true;
                    } else if (level) {
                        tie = true;
                    }
                } else {
                    // per-owner minimum of the t bits (t > 0, so bit order = value order): a suffix minimum within each owner's
                    // run of lanes leaves the run's minimum in its first lane
                    const unsigned tb = (r != 0) ? __float_as_uint(t) : 0xffffffffu;
                    const unsigned above = starts & ~(FULL >> (31 - lane));
                    const int end = above ? __ffs(above) - 1 : (int)min(pairs, 32u);
                    unsigned mn = tb;
#pragma unroll
                    for (int s = 1; s < 32; s <<= 1) {
                        const unsigned v = __shfl_down_sync(FULL, mn, s);
                        if (lane + s < end) mn = min(mn, v);
                    }
                    const unsigned run_min = __shfl_sync(FULL, mn, start);
                    const unsigned win = __ballot_sync(FULL, act && tb != 0xffffffffu && tb == run_min) & seg;   // holders of the minimum
                    const int p = win ? __ffs(win) - 1 : lane;   // the first holder
                    const int triw = __shfl_sync(FULL, tri, p);
                    const float tn = __uint_as_float(__shfl_sync(FULL, tb, p));
                    if (win) {
                        if (tn < best) {
                            best = tn;
                            best_tri = triw;
                            tie = __popc(win) > 1;
                        } else {
                            tie = true;   // tn == best
                        }
                    }
                }
                const int k_last = __shfl_sync(FULL, k, 31);   // the last pair tested: its owner keeps the triangles above it
                if (owns) {
                    t_mask = (taken < cnt && !stop) ? t_mask & ~((2u << k_last) - 1u) : 0u;
                    if (stop) { g_bits = 0u; sp = 0; }   // any accepted hit ends a shadow ray
                    if (t_mask == 0u) select_next();
                }
            }
            busy = __ballot_sync(FULL, ray >= 0 && node != W8_ENDED);
            if (COUNT) {
                const uint32_t now = w8_clock(), e = __reduce_max_sync(FULL, end_dt);   // the ray ends of a step run side by side
                end_dt = 0u;
                cyc_end += e;
                if (node_step) { cyc_node += now - t_mark - e; n_node_steps++; }
                else { cyc_tri += now - t_mark - e; n_tri_steps++; }
                t_mark = now;
            }
        } while (busy != 0u && (exhausted || __popc(busy) >= refill_thresh));
    }
#undef W8_PUSH
#undef W8_POP
    if (COUNT) {
        atomicAdd(counts.node_visits, (unsigned long long)n_visits);
        atomicAdd(counts.tri_tests, (unsigned long long)n_tests);
        atomicAdd(phase_cycles + 6, (unsigned long long)n_visits);
        atomicAdd(phase_cycles + 7, (unsigned long long)n_tests);
        if (lane == 0) {
            atomicAdd(phase_cycles + 0, (unsigned long long)cyc_refill);
            atomicAdd(phase_cycles + 1, (unsigned long long)cyc_node);
            atomicAdd(phase_cycles + 2, (unsigned long long)cyc_tri);
            atomicAdd(phase_cycles + 3, (unsigned long long)cyc_end);
            atomicAdd(phase_cycles + 4, (unsigned long long)n_node_steps);
            atomicAdd(phase_cycles + 5, (unsigned long long)n_tri_steps);
        }
    }
}

// ------------------------------------------------------------------------------------------
// W8 camera pass: the warp traces its 32 work items as ONE bundle.  In pixel-major order those are the jittered samples of
// one or two pixels, which share the eye and walk the same nodes, so the node work is done once per warp: one warp-uniform
// stack, and lanes 0..7 each test one slot of the node with the bundle bound of w8_node.h (conservative for every member
// ray).  The triangles of the hit leaf slots are then tested one after the other, every member lane its own ray (tri_test_t
// in its serial order: t <= best accepted, t == best a tie).
// The result of every ray equals the per-ray traversal's: the bundle reaches every slot the ray's exact segment reaches
// within its limit, so it tests every triangle the ray accepts at or below its final best -- the minimum and its holders
// (best, tie) are the same, and best_tri is the first holder, which matters only without a tie.
// ------------------------------------------------------------------------------------------
template <int K>
__device__ __forceinline__ float warp_reduce_f(float v) {   // K = 0: minimum, 1: maximum, over all 32 lanes
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        const float u = __shfl_xor_sync(0xffffffffu, v, s);
        v = K ? fmaxf(v, u) : fminf(v, u);
    }
    return v;
}
// one axis of the bundle bound (w8_node.h): entry / exit bounds of the slab [lo, hi] for every member ray
__device__ __forceinline__ void w8_bundle_axis(float lo, float hi, uint32_t sign, const float4 b, float& entry, float& exit) {
    const float omin = b.x, omax = b.y, vmin = b.z, vmax = b.w;
    const bool pos = sign == 1u;
    const float pn = pos ? lo : hi, pf = pos ? hi : lo;
    const float xe = pos ? __fsub_rd(pn, omax) : __fsub_ru(pn, omin);
    const float xx = pos ? __fsub_ru(pf, omin) : __fsub_rd(pf, omax);
    entry = sign ? __fmul_rd(xe, xe >= 0.0f ? vmin : vmax) : -EZ_INF;   // sign 0: the members' d_a differ in sign
    exit = sign ? __fmul_ru(xx, xx >= 0.0f ? vmax : vmin) : EZ_INF;
}

template <bool COUNT, bool IDX, class RayIO>
__device__ __forceinline__ void extend_w8_bundle(const SceneDev& sc, uint32_t n, uint32_t* work, RayIO io, const unsigned char* s_perm, uint2* stack_sm,
                                                 W8Counts counts) {
    const bool tri_na = sc.tri_l1_bypass != 0;
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    uint2* const stack = stack_sm + (threadIdx.x >> 5) * W8_BUNDLE_STACK;   // the warp's stack: every lane writes the same entry
    __shared__ float4 s_bnd_all[(EZRT_EXTEND_MAX_THREADS / 32) * 3];
    float4* const bnd = s_bnd_all + (threadIdx.x >> 5) * 3;
    __shared__ unsigned s_pend_all[EZRT_EXTEND_MAX_THREADS / 32];
    unsigned* const s_pend = s_pend_all + (threadIdx.x >> 5);
    const uint4* __restrict__ nodes = sc.w8_nodes;
    const float origin_limit = sc.w8_origin_limit, inv_limit = sc.quant_inv_limit;
    uint32_t n_tests = 0;
    __shared__ uint32_t s_visits_all[EZRT_EXTEND_MAX_THREADS / 32];   // COUNT: node visits of the warp (lane 0), in shared memory
    uint32_t* const s_visits = s_visits_all + (threadIdx.x >> 5);
    if (COUNT && lane == 0) *s_visits = 0u;
    // slot of this lane in a node step (lanes 0..7) and its byte in the plane words
    const bool slot_hi = (lane & 7) >= 4;
    const uint32_t slot_shift = (uint32_t)(lane & 3) * 8u;
    auto slot_byte = [&](uint32_t w0, uint32_t w1) { return (float)(((slot_hi ? w1 : w0) >> slot_shift) & 0xffu); };

    while (true) {
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(work, 32u);
        base = __shfl_sync(FULL, base, 0);
        if (base >= n) break;
        const uint32_t idx = base + (uint32_t)lane;
        vec3 o = splat3(0.0f), d = splat3(0.0f), inv = splat3(0.0f);
        bool member = false;
        if (idx < n && io.load(idx, o, d)) {
            inv = ez_v3(EZ_DIV(1.0f, d.x), EZ_DIV(1.0f, d.y), EZ_DIV(1.0f, d.z));
            const float ax = ez_abs(inv.x), ay = ez_abs(inv.y), az = ez_abs(inv.z);
            const float ao = fmaxf(ez_abs(o.x), fmaxf(ez_abs(o.y), ez_abs(o.z)));
            const float amin = fminf(ax, fminf(ay, az)), amax = fmaxf(ax, fmaxf(ay, az));
            if ((amax <= inv_limit) && (amin >= W8_INV_MIN) && (ao <= origin_limit)) member = true;   // false for inf / NaN
            else io.defer(idx, o, d);   // outside the decode error bound: the exact kernel traces it
        }
        // Sub-bundles: a member joins the first pending member's sub-bundle when every component of its 1/d has the leader's sign
        // and lies within a factor 2 of the leader's.  Camera rays of neighbouring pixels almost always form one sub-bundle; where
        // a component of d crosses zero its 1/d spreads without bound, and one bundle over such rays would bound nothing on that
        // axis (and their slack makes the limit huge): those rays go in sub-bundles of their own.
        // (the pending mask lives in shared memory, like the bundle's intervals: 64 registers without spilling)
        *s_pend = __ballot_sync(FULL, member);
        while (*s_pend != 0u) {
        const unsigned pending = *s_pend;
        const int lead = __ffs(pending) - 1;
        const float lx = __shfl_sync(FULL, inv.x, lead), ly = __shfl_sync(FULL, inv.y, lead), lz = __shfl_sync(FULL, inv.z, lead);
        auto close = [](float v, float w) { return (v > 0.0f) == (w > 0.0f) && ez_abs(v) <= 2.0f * ez_abs(w) && ez_abs(w) <= 2.0f * ez_abs(v); };
        member = ((pending >> lane) & 1u) && close(inv.x, lx) && close(inv.y, ly) && close(inv.z, lz);
        const unsigned members = __ballot_sync(FULL, member);
        *s_pend = pending & ~members;
        float best = EZ_INF;
        int best_tri = -1;
        bool tie = false;
        // the bundle's intervals (w8_node.h "Bundle bound"): (omin, omax, vmin, vmax) per axis in shared memory, and the sign of
        // axis a in bits 2a..2a+1: 1 all members d_a >= 0, 2 all d_a < 0, 0 mixed
        uint32_t signs = 0u;
        {
            const float oa[3] = {o.x, o.y, o.z}, da[3] = {d.x, d.y, d.z}, va[3] = {inv.x, inv.y, inv.z};
#pragma unroll
            for (int a = 0; a < 3; a++) {
                const unsigned p = __ballot_sync(FULL, member && da[a] >= 0.0f);
                signs |= (p == members ? 1u : (p == 0u ? 2u : 0u)) << (2 * a);
                const float4 b = make_float4(warp_reduce_f<0>(member ? oa[a] : INFINITY), warp_reduce_f<1>(member ? oa[a] : -INFINITY),
                                             warp_reduce_f<0>(member ? va[a] : INFINITY), warp_reduce_f<1>(member ? va[a] : -INFINITY));
                bnd[a] = b;   // every lane writes the same value and reads back its own write
            }
        }
        // visit order: the octant order of the first member's ray (any order is correct)
        const uint32_t near_mask = __shfl_sync(FULL, (d.x >= 0.0f ? (1u << sc.w8_near_bit[0]) : 0u) | (d.y >= 0.0f ? (1u << sc.w8_near_bit[1]) : 0u) |
                                                         (d.z >= 0.0f ? (1u << sc.w8_near_bit[2]) : 0u), __ffs(members) - 1);
        float L = EZ_INF;   // the largest per-ray limit best + best 2^-12 + slack of the members
        int sp = 0;
        uint32_t node = 0, g_base = 0, g_bits = 0;
        while (true) {
            const uint4* nd = nodes + (size_t)node * (W8_NODE_WORDS / 4);
            const uint4 h = ldg128_u32(nd), c = ldg128_u32(nd + 1), l = ldg128_u32(nd + 2), m = ldg128_u32(nd + 3), u = ldg128_u32(nd + 4);
            if (COUNT && lane == 0) ++*s_visits;
            bool hit = false;
            if (lane < 8) {
                const float sx = __uint_as_float(W8_SCALE_BITS(h.w, 0)), sy = __uint_as_float(W8_SCALE_BITS(h.w, 1)), sz = __uint_as_float(W8_SCALE_BITS(h.w, 2));
                const float ox = __uint_as_float(h.x), oy = __uint_as_float(h.y), oz = __uint_as_float(h.z);
                float ex, ey, ez, xx, xy, xz;
                w8_bundle_axis(__fadd_rd(ox, (slot_byte(c.z, c.w) - 0.25f) * sx), __fadd_ru(ox, (slot_byte(m.z, m.w) + 0.25f) * sx), signs & 3u, bnd[0], ex, xx);
                w8_bundle_axis(__fadd_rd(oy, (slot_byte(l.x, l.y) - 0.25f) * sy), __fadd_ru(oy, (slot_byte(u.x, u.y) + 0.25f) * sy), (signs >> 2) & 3u, bnd[1], ey, xy);
                w8_bundle_axis(__fadd_rd(oz, (slot_byte(l.z, l.w) - 0.25f) * sz), __fadd_ru(oz, (slot_byte(u.z, u.w) + 0.25f) * sz), signs >> 4, bnd[2], ez, xz);
                hit = fmaxf(fmaxf(ex, ey), fmaxf(ez, 0.0f)) <= fminf(fminf(xx, xy), fminf(xz, L));
            }
            const uint32_t hits = __ballot_sync(FULL, hit) & 0xffu;
            const uint32_t imask = h.w >> 24;
            const uint32_t inner = hits & imask;
            uint32_t leaf = hits & ~imask;
            if ((g_bits >> 8) != 0u) stack[sp++] = make_uint2(g_base, g_bits);   // the rest of the group this node came from
            g_base = c.x;
            g_bits = imask | ((uint32_t)s_perm[near_mask * 256u + inner] << 8);
            // triangles of the hit leaf slots (meta byte = (count << 5) | offset), every member lane its own ray, lowest first
            uint32_t t_mask = 0u;
            while (leaf != 0u) {
                const int s = __ffs(leaf) - 1;
                leaf &= leaf - 1u;
                const uint32_t mb = ((s < 4 ? m.x : m.y) >> ((s & 3) * 8)) & 0xffu;
                t_mask |= ((1u << (mb >> 5)) - 1u) << (mb & 31u);
            }
            if (t_mask != 0u) {
                while (t_mask != 0u) {
                    const int tri = (int)c.y + __ffs(t_mask) - 1;
                    t_mask &= t_mask - 1u;
                    if (member) {
                        if (COUNT) n_tests++;
                        float t = 0.0f;
                        const int r = IDX ? tri_test_idx_t<true>(sc.acc_tri_geo + (size_t)tri * 2, sc.acc_tri_vert, o, d, best, t, tri_na)
                                          : tri_test_t<true>(sc.acc_tri_geo + (size_t)tri * 4, o, d, best, t, tri_na);
                        if (r == 2) tie = true;
                        else if (r == 1) { best = t; best_tri = tri; tie = false; }
                    }
                }
                // the per-ray limit (slack recomputed here: one register less); >= 0, so the bits order as the values
                const float slack = sc.prune_delta * fmaxf(ez_abs(inv.x), fmaxf(ez_abs(inv.y), ez_abs(inv.z)));
                const float lim = member ? best + (best * 0.000244140625f + slack) : 0.0f;
                L = __uint_as_float(__reduce_max_sync(FULL, __float_as_uint(lim)));
            }
            // next node: from the current group, else from the stack
            if ((g_bits >> 8) == 0u) {
                if (sp == 0) break;
                const uint2 e = stack[--sp];
                g_base = e.x;
                g_bits = e.y;
            }
            const int p = 23 - __clz(g_bits);
            g_bits ^= 0x100u << p;
            const uint32_t slot = (uint32_t)p ^ near_mask;
            node = g_base + (uint32_t)__popc(g_bits & 0xffu & ((1u << slot) - 1u));
        }
        if (member) {
            HitRec hr;
            hr.t = best;
            hr.tri = best_tri;
            io.store(idx, hr, tie, o, d, inv);
        }
        }
    }
    if (COUNT) {
        if (lane == 0) atomicAdd(counts.node_visits, (unsigned long long)*s_visits);
        atomicAdd(counts.tri_tests, (unsigned long long)n_tests);
    }
}

// ------------------------------------------------------------------------------------------
// hit geometry + material for the final closest hit (tail of hitTriangle :198-214, getMaterial :110-135)
// ------------------------------------------------------------------------------------------
struct MaterialDev {
    vec3 emissive, baseColor;
    float subsurface, metallic, specular, specularTint, roughness, anisotropic, sheen, sheenTint, clearcoat,
        clearcoatGloss;
};

__device__ __forceinline__ MaterialDev load_material(const SceneDev& sc, int matId) {
    const float4* m = sc.materials + (size_t)matId * 5;
    float4 a = ldg4(m), b = ldg4(m + 1), c = ldg4(m + 2), d = ldg4(m + 3);
    MaterialDev r;
    r.emissive = ez_v3(a.x, a.y, a.z);
    r.baseColor = ez_v3(a.w, b.x, b.y);
    r.subsurface = b.z; r.metallic = b.w; r.specular = c.x; r.specularTint = c.y;
    r.roughness = c.z; r.anisotropic = c.w; r.sheen = d.x; r.sheenTint = d.y;
    r.clearcoat = d.z; r.clearcoatGloss = d.w;
    return r;
}
__device__ __forceinline__ vec3 load_emissive(const SceneDev& sc, int matId) {
    float4 a = ldg4(sc.materials + (size_t)matId * 5);
    return ez_v3(a.x, a.y, a.z);
}

struct SurfaceHit {
    vec3 P, N;   // hitPoint, shading normal (flipped when hit from inside)
    int matId;
    bool inside; // hit from inside: dot(Ng, d) > 0
};

// Recomputes P and the interpolated normal for (ray, t, tri).  p3fudge selects the P3/P4
// barycentric denominators (P3/fsh:273-274) instead of P5's "+1e-7" (P5/fsh:206-207).
// The (N, d0) quad of triangle `tri` in the policy's index space: the first 16 bytes of its flat or indexed record.
__device__ __forceinline__ const float4* tri_geo_rec(const SceneDev& sc, int tri, bool accel_space) {
    return accel_space ? sc.acc_tri_geo + (size_t)tri * (sc.acc_tri_indexed ? 2 : 4) : sc.tri_geo + (size_t)tri * 4;
}
__device__ __forceinline__ SurfaceHit surface_hit(const SceneDev& sc, vec3 o, vec3 d, float t, int tri, bool p3fudge, bool accel_space = false) {
    // vertices: v[i1], v[i2], v[i3] of the vertex array (indexed record) or g[1], g[2], g[3] (flat record)
    const float4* g = tri_geo_rec(sc, tri, accel_space);
    const float4* v = g;
    uint32_t i1 = 1u, i2 = 2u, i3 = 3u;
    if (accel_space && sc.acc_tri_indexed) {
        const uint4 qi = __ldg(reinterpret_cast<const uint4*>(g + 1));
        v = sc.acc_tri_vert; i1 = qi.x; i2 = qi.y; i3 = qi.z;
    }
    float4 q0 = ldg4(g), q1 = ldg4(v + i1), q2 = ldg4(v + i2), q3 = ldg4(v + i3);
    const float4* s = (accel_space ? sc.acc_tri_shade : sc.tri_shade) + (size_t)tri * 3;
    float4 m0 = ldg4(s), m1 = ldg4(s + 1), m2 = ldg4(s + 2);
    vec3 p1 = f4xyz(q1), p2 = f4xyz(q2), p3 = f4xyz(q3);
    vec3 Ng = f4xyz(q0);
    bool inside = ez_dot(Ng, d) > 0.0f;  // :175
    vec3 P = ez_add(o, ez_scale(d, t));
    float alpha, beta;
    float an = (-(P.x - p2.x)) * (p3.y - p2.y) + (P.y - p2.y) * (p3.x - p2.x);
    float bn = (-(P.x - p3.x)) * (p1.y - p3.y) + (P.y - p3.y) * (p1.x - p3.x);
    if (!p3fudge) {
        alpha = EZ_DIV(an, ((-(p1.x - p2.x)) * (p3.y - p2.y) + (p1.y - p2.y) * (p3.x - p2.x)) + 1e-7f);
        beta = EZ_DIV(bn, ((-(p2.x - p3.x)) * (p1.y - p3.y) + (p2.y - p3.y) * (p1.x - p3.x)) + 1e-7f);
    } else {
        alpha = EZ_DIV(an, (-((p1.x - p2.x) - 0.00005f)) * ((p3.y - p2.y) + 0.00005f) +
                               ((p1.y - p2.y) + 0.00005f) * ((p3.x - p2.x) + 0.00005f));
        beta = EZ_DIV(bn, (-((p2.x - p3.x) - 0.00005f)) * ((p1.y - p3.y) + 0.00005f) +
                              ((p2.y - p3.y) + 0.00005f) * ((p1.x - p3.x) + 0.00005f));
    }
    float gama = (1.0f - alpha) - beta;
    vec3 Ns = ez_add(ez_add(ez_scale(f4xyz(m0), alpha), ez_scale(f4xyz(m1), beta)), ez_scale(f4xyz(m2), gama));
    Ns = ez_normalize(Ns);
    SurfaceHit r;
    r.P = P;
    r.N = inside ? ez_neg(Ns) : Ns;
    r.matId = __float_as_int(m0.w);
    r.inside = inside;
    return r;
}
__device__ __forceinline__ int tri_material(const SceneDev& sc, int tri) {
    return __float_as_int(ldg4(sc.tri_shade + (size_t)tri * 3).w);
}

// ------------------------------------------------------------------------------------------
// Disney principled BRDF, P5/fsh:400-549 (isotropic) and P4/fsh:375-473 (anisotropic)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float SchlickFresnel(float u) {
    float m = ez_clamp(1.0f - u, 0.0f, 1.0f);
    float m2 = m * m;
    return m2 * m2 * m;
}
__device__ __forceinline__ float GTR1(float NdotH, float a) {
    if (a >= 1.0f) return EZ_DIV(1.0f, EZ_PI);
    float a2 = a * a;
    float t = 1.0f + (a2 - 1.0f) * NdotH * NdotH;
    return EZ_DIV(a2 - 1.0f, EZ_PI * ezd_log(a2) * t);
}
__device__ __forceinline__ float GTR2(float NdotH, float a) {
    float a2 = a * a;
    float t = 1.0f + (a2 - 1.0f) * NdotH * NdotH;
    return EZ_DIV(a2, EZ_PI * t * t);
}
__device__ __forceinline__ float GTR2_aniso(float NdotH, float HdotX, float HdotY, float ax, float ay) {
    float s = ez_sqr(EZ_DIV(HdotX, ax)) + ez_sqr(EZ_DIV(HdotY, ay)) + NdotH * NdotH;
    return EZ_DIV(1.0f, EZ_PI * ax * ay * ez_sqr(s));
}
__device__ __forceinline__ float smithG_GGX(float NdotV, float alphaG) {
    float a = alphaG * alphaG;
    float b = NdotV * NdotV;
    return EZ_DIV(1.0f, NdotV + EZ_SQRT(a + b - a * b));
}
__device__ __forceinline__ float smithG_GGX_aniso(float NdotV, float VdotX, float VdotY, float ax, float ay) {
    return EZ_DIV(1.0f, NdotV + EZ_SQRT(ez_sqr(VdotX * ax) + ez_sqr(VdotY * ay) + ez_sqr(NdotV)));
}
// getTangent, P5/fsh:553-558
__device__ __forceinline__ void get_tangent(vec3 N, vec3& tangent, vec3& bitangent) {
    vec3 helper = ez_v3(1.0f, 0.0f, 0.0f);
    if (ez_abs(N.x) > 0.999f) helper = ez_v3(0.0f, 0.0f, 1.0f);
    bitangent = ez_normalize(ez_cross(N, helper));
    tangent = ez_normalize(ez_cross(N, bitangent));
}

template <bool ANISO>
__device__ __forceinline__ vec3 brdf_evaluate(vec3 V, vec3 N, vec3 L, const MaterialDev& mat) {
    float NdotL = ez_dot(N, L);
    float NdotV = ez_dot(N, V);
    if (NdotL < 0.0f || NdotV < 0.0f) return splat3(0.0f);

    vec3 H = ez_normalize(ez_add(L, V));
    float NdotH = ez_dot(N, H);
    float LdotH = ez_dot(L, H);

    vec3 Cdlin = mat.baseColor;
    float Cdlum = 0.3f * Cdlin.x + 0.6f * Cdlin.y + 0.1f * Cdlin.z;
    vec3 Ctint = (Cdlum > 0.0f) ? ez_divs(Cdlin, Cdlum) : splat3(1.0f);
    vec3 Cspec = ez_scale(ez_vmix(splat3(1.0f), Ctint, mat.specularTint), mat.specular);
    vec3 Cspec0 = ez_vmix(ez_scale(Cspec, 0.08f), Cdlin, mat.metallic);
    vec3 Csheen = ez_vmix(splat3(1.0f), Ctint, mat.sheenTint);

    float Fd90 = 0.5f + 2.0f * LdotH * LdotH * mat.roughness;
    float FL = SchlickFresnel(NdotL);
    float FV = SchlickFresnel(NdotV);
    float Fd = ez_mix(1.0f, Fd90, FL) * ez_mix(1.0f, Fd90, FV);

    float Fss90 = LdotH * LdotH * mat.roughness;
    float Fss = ez_mix(1.0f, Fss90, FL) * ez_mix(1.0f, Fss90, FV);
    float ss = 1.25f * (Fss * (EZ_DIV(1.0f, NdotL + NdotV) - 0.5f) + 0.5f);

    float Ds, Gs;
    float FH = SchlickFresnel(LdotH);
    vec3 Fs = ez_vmix(Cspec0, splat3(1.0f), FH);
    if (!ANISO) {
        float alpha = ez_max(0.001f, ez_sqr(mat.roughness));
        Ds = GTR2(NdotH, alpha);
        Gs = smithG_GGX(NdotL, mat.roughness);
        Gs *= smithG_GGX(NdotV, mat.roughness);
    } else {
        vec3 X, Y;
        get_tangent(N, X, Y);
        float aspect = EZ_SQRT(1.0f - mat.anisotropic * 0.9f);
        float ax = ez_max(0.001f, EZ_DIV(ez_sqr(mat.roughness), aspect));
        float ay = ez_max(0.001f, ez_sqr(mat.roughness) * aspect);
        Ds = GTR2_aniso(NdotH, ez_dot(H, X), ez_dot(H, Y), ax, ay);
        Gs = smithG_GGX_aniso(NdotL, ez_dot(L, X), ez_dot(L, Y), ax, ay);
        Gs *= smithG_GGX_aniso(NdotV, ez_dot(V, X), ez_dot(V, Y), ax, ay);
    }

    float Dr = GTR1(NdotH, ez_mix(0.1f, 0.001f, mat.clearcoatGloss));
    float Fr = ez_mix(0.04f, 1.0f, FH);
    float Gr = smithG_GGX(NdotL, 0.25f) * smithG_GGX(NdotV, 0.25f);

    vec3 Fsheen = ez_scale(Csheen, FH * mat.sheen);
    vec3 diffuse = ez_add(ez_scale(Cdlin, EZ_DIV(1.0f, EZ_PI) * ez_mix(Fd, ss, mat.subsurface)), Fsheen);
    vec3 specular = ez_scale(ez_scale(Fs, Gs), Ds);
    vec3 clearcoat = splat3(0.25f * Gr * Fr * Dr * mat.clearcoat);
    return ez_add(ez_add(ez_scale(diffuse, 1.0f - mat.metallic), specular), clearcoat);
}

// BRDF_Pdf, P5/fsh:715-752
__device__ __forceinline__ float brdf_pdf(vec3 V, vec3 N, vec3 L, const MaterialDev& mat) {
    float NdotL = ez_dot(N, L);
    float NdotV = ez_dot(N, V);
    if (NdotL < 0.0f || NdotV < 0.0f) return 0.0f;
    vec3 H = ez_normalize(ez_add(L, V));
    float NdotH = ez_dot(N, H);
    float alpha = ez_max(0.001f, ez_sqr(mat.roughness));
    float Ds = GTR2(NdotH, alpha);
    float Dr = GTR1(NdotH, ez_mix(0.1f, 0.001f, mat.clearcoatGloss));
    float LH4 = 4.0f * ez_dot(L, H);
    float pdf_diffuse = EZ_DIV(NdotL, EZ_PI);
    float pdf_specular = EZ_DIV(Ds * NdotH, LH4);
    float pdf_clearcoat = EZ_DIV(Dr * NdotH, LH4);
    float r_diffuse = 1.0f - mat.metallic;
    float r_specular = 1.0f;
    float r_clearcoat = 0.25f * mat.clearcoat;
    float r_sum = r_diffuse + r_specular + r_clearcoat;
    float p_diffuse = EZ_DIV(r_diffuse, r_sum);
    float p_specular = EZ_DIV(r_specular, r_sum);
    float p_clearcoat = EZ_DIV(r_clearcoat, r_sum);
    float pdf = p_diffuse * pdf_diffuse + p_specular * pdf_specular + p_clearcoat * pdf_clearcoat;
    return ez_max(1e-10f, pdf);
}
__device__ __forceinline__ float mis_mix_weight(float a, float b) {  // P5/fsh:754-757
    float t = a * a;
    return EZ_DIV(t, b * b + t);
}

// ------------------------------------------------------------------------------------------
// transmission (EZRT_PARAM_TRANSMISSION; ezrt_math.h, DESIGN.md section 12): the reference BRDF mixed with a rough dielectric
// ------------------------------------------------------------------------------------------
struct TransLobe {
    float t, eta, alpha;   // the lobe's weight, eta_L / eta_V, the GGX alpha
    bool matched;          // index-matched: a pass-through
};
// the dielectric lobe of material matId at a hit from `inside` (the record's fifth quad: IOR, transmission)
__device__ __forceinline__ TransLobe trans_lobe(const SceneDev& sc, int matId, const MaterialDev& mat, bool inside) {
    const float4 e = ldg4(sc.materials + (size_t)matId * 5 + 4);
    TransLobe r;
    r.t = ez_trans_weight(e.y, mat.metallic, e.x);
    r.eta = ez_trans_eta(e.x, inside);
    r.alpha = ez_max(0.001f, ez_sqr(mat.roughness));
    r.matched = ez_trans_matched(e.x) != 0;
    return r;
}
// the mixture's f at L and its pdf
__device__ __forceinline__ vec3 bsdf_evaluate(vec3 V, vec3 N, vec3 L, const MaterialDev& mat, const TransLobe& tl, float& pdf) {
    vec3 f_ref = splat3(0.0f), f_diel = splat3(0.0f);
    float pdf_ref = 0.0f, pdf_diel = 0.0f;
    if (ez_dot(N, L) > 0.0f) { f_ref = brdf_evaluate<false>(V, N, L, mat); pdf_ref = brdf_pdf(V, N, L, mat); }
    if (!tl.matched) f_diel = ez_diel_eval(V, N, L, mat.baseColor, tl.alpha, tl.eta, &pdf_diel);
    return ez_trans_mix(f_ref, pdf_ref, f_diel, pdf_diel, tl.t, &pdf);
}

// ------------------------------------------------------------------------------------------
// direction samplers, P5/fsh:561-664
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ vec3 to_normal_hemisphere(vec3 v, vec3 N) {
    vec3 helper = ez_v3(1.0f, 0.0f, 0.0f);
    if (ez_abs(N.x) > 0.999f) helper = ez_v3(0.0f, 0.0f, 1.0f);
    vec3 tangent = ez_normalize(ez_cross(N, helper));
    vec3 bitangent = ez_normalize(ez_cross(N, tangent));
    return ez_add(ez_add(ez_scale(tangent, v.x), ez_scale(bitangent, v.y)), ez_scale(N, v.z));
}
__device__ __forceinline__ vec3 sample_hemisphere(float xi_1, float xi_2) {
    float z = xi_1;
    float r = ez_max(0.0f, EZ_SQRT(1.0f - z * z));
    float phi = 2.0f * EZ_PI * xi_2;
    return ez_v3(r * ezd_cos(phi), r * ezd_sin(phi), z);
}
__device__ __forceinline__ vec3 half_vector_to_L(float sin_theta_h, float cos_theta_h, float phi_h, vec3 V, vec3 N) {
    float sin_phi_h = ezd_sin(phi_h);
    float cos_phi_h = ezd_cos(phi_h);
    vec3 H = ez_v3(sin_theta_h * cos_phi_h, sin_theta_h * sin_phi_h, cos_theta_h);
    H = to_normal_hemisphere(H, N);
    return ez_reflect(ez_neg(V), H);
}
// SampleBRDF, P5/fsh:633-664
__device__ __forceinline__ vec3 sample_brdf(float xi_1, float xi_2, float xi_3, vec3 V, vec3 N, const MaterialDev& mat) {
    float alpha_GTR1 = ez_mix(0.1f, 0.001f, mat.clearcoatGloss);
    float alpha_GTR2 = ez_max(0.001f, ez_sqr(mat.roughness));
    float r_diffuse = 1.0f - mat.metallic;
    float r_specular = 1.0f;
    float r_clearcoat = 0.25f * mat.clearcoat;
    float r_sum = r_diffuse + r_specular + r_clearcoat;
    float p_diffuse = EZ_DIV(r_diffuse, r_sum);
    float p_specular = EZ_DIV(r_specular, r_sum);
    float rd = xi_3;
    if (rd <= p_diffuse) {  // SampleCosineHemisphere :579-590
        float r = EZ_SQRT(xi_1);
        float theta = xi_2 * 2.0f * EZ_PI;
        float x = r * ezd_cos(theta);
        float y = r * ezd_sin(theta);
        float z = EZ_SQRT(1.0f - x * x - y * y);
        return to_normal_hemisphere(ez_v3(x, y, z), N);
    } else if (p_diffuse < rd && rd <= p_diffuse + p_specular) {  // SampleGTR2 :593-610
        float phi_h = 2.0f * EZ_PI * xi_1;
        float cos_theta_h = EZ_SQRT(EZ_DIV(1.0f - xi_2, 1.0f + (alpha_GTR2 * alpha_GTR2 - 1.0f) * xi_2));
        float sin_theta_h = EZ_SQRT(ez_max(0.0f, 1.0f - cos_theta_h * cos_theta_h));
        return half_vector_to_L(sin_theta_h, cos_theta_h, phi_h, V, N);
    } else if (p_diffuse + p_specular < rd) {  // SampleGTR1 :613-630
        float phi_h = 2.0f * EZ_PI * xi_1;
        float a2 = alpha_GTR1 * alpha_GTR1;
        float cos_theta_h = EZ_SQRT(EZ_DIV(1.0f - ezd_pow(a2, 1.0f - xi_2), 1.0f - a2));
        float sin_theta_h = EZ_SQRT(ez_max(0.0f, 1.0f - cos_theta_h * cos_theta_h));
        return half_vector_to_L(sin_theta_h, cos_theta_h, phi_h, V, N);
    }
    return ez_v3(0.0f, 1.0f, 0.0f);
}
// The mixture's sample (ezrt_math.h, DESIGN.md section 12) at a hit with tl.t > 0: L, and what the path carries -- f, pdf and
// the cosine |dot(N, L)| with the sign of dot(N, L) (< 0: below the surface).  Returns false when the path ends.  On entry L is
// sample_brdf(xi_1, xi_2, xi_3, V, N, mat), the reference lobe's sample, which the caller has already drawn.
__device__ __forceinline__ bool bsdf_sample(float xi_1, float xi_2, float xi_3, float r_t, vec3 V, vec3 N, const MaterialDev& mat,
                                            const TransLobe& tl, vec3& L, vec3& f, float& pdf, float& cosine) {
    if (r_t < tl.t) {
        if (tl.matched) {   // pass-through: weight baseColor
            L = ez_neg(V);
            f = mat.baseColor;
            pdf = 1.0f;
            cosine = -1.0f;
            return true;
        }
        if (!ez_diel_sample(xi_1, xi_2, xi_3, V, N, tl.alpha, tl.eta, &L)) return false;
    } else if (!(ez_dot(N, L) > 0.0f)) {
        return false;
    }
    f = bsdf_evaluate(V, N, L, mat, tl, pdf);
    cosine = ez_dot(N, L);
    return true;
}

// ------------------------------------------------------------------------------------------
// HDR environment: texture2D restated as plain loads (fp32 bilinear / nearest, CLAMP_TO_EDGE)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ vec3 texel3(const float* img, int idx) {
    const float* p = img + (size_t)idx * 3;
    return ez_v3(__ldg(p), __ldg(p + 1), __ldg(p + 2));
}
__device__ __forceinline__ vec3 tex2d(const float* img, int W, int H, float u, float v, int linear) {
    if (!linear) return texel3(img, ez_env_texel(u, v, W, H));
    float x = u * (float)W - 0.5f, y = v * (float)H - 0.5f;
    float fx0 = ez_floor(x), fy0 = ez_floor(y);
    float ax = x - fx0, ay = y - fy0;
    // indices clamped in float: a NaN coordinate reads texel 0 and weighs it by NaN
    const int x0 = ez_texel_clamp(fx0, W), x1 = ez_texel_clamp(fx0 + 1.0f, W);
    const int y0 = ez_texel_clamp(fy0, H), y1 = ez_texel_clamp(fy0 + 1.0f, H);
    vec3 t00 = texel3(img, y0 * W + x0), t10 = texel3(img, y0 * W + x1);
    vec3 t01 = texel3(img, y1 * W + x0), t11 = texel3(img, y1 * W + x1);
    return ez_vmix(ez_vmix(t00, t10, ax), ez_vmix(t01, t11, ax), ay);
}
// toSphericalCoord, P5/fsh:684-690
__device__ __forceinline__ void to_spherical(vec3 v, float& ou, float& ov) {
    float u = ezd_atan2(v.z, v.x), w = ezd_asin(v.y);
    u = EZ_DIV(u, 2.0f * EZ_PI);
    w = EZ_DIV(w, EZ_PI);
    u += 0.5f;
    w += 0.5f;
    ou = u;
    ov = 1.0f - w;
}
// hdrColor P5/fsh:693-697; sampleHdr P3/fsh:151-156 (clamped to 10) / P4/fsh:366-371
__device__ __forceinline__ vec3 hdr_color(const SceneDev& sc, const RenderDev& rd, vec3 L, int mode) {
    vec3 color;
    if (!sc.hdr) {
        color = ez_v3(rd.env[0], rd.env[1], rd.env[2]);
    } else {
        float u, v;
        to_spherical(ez_normalize(L), u, v);
        color = tex2d(sc.hdr, sc.hdr_w, sc.hdr_h, u, v, sc.hdr_linear);
    }
    if (mode == EZRT_MODE_DIFFUSE_P3) color = ez_vmin(color, splat3(10.0f));
    return color;
}
// SampleHdr, P5/fsh:667-679
__device__ __forceinline__ vec3 sample_hdr(const SceneDev& sc, float xi_1, float xi_2) {
    vec3 c = tex2d(sc.hdr_cache, sc.hdr_w, sc.hdr_h, xi_1, xi_2, sc.hdr_linear);
    float x = c.x, y = 1.0f - c.y;
    float phi = 2.0f * EZ_PI * (x - 0.5f);
    float theta = EZ_PI * (y - 0.5f);
    float ct = ezd_cos(theta);
    return ez_v3(ct * ezd_cos(phi), ezd_sin(theta), ct * ezd_sin(phi));
}
// hdrPdf, P5/fsh:701-712
__device__ __forceinline__ float hdr_pdf(const SceneDev& sc, vec3 L) {
    float u, v;
    to_spherical(ez_normalize(L), u, v);
    float pdf = tex2d(sc.hdr_cache, sc.hdr_w, sc.hdr_h, u, v, sc.hdr_linear).z;
    float theta = EZ_PI * (0.5f - v);
    float sin_theta = ez_max(ezd_sin(theta), 1e-10f);
    int res = sc.hdr_w;
    float p_convert = EZ_DIV((float)(res * res / 2), 2.0f * EZ_PI * EZ_PI * sin_theta);
    return pdf * p_convert;
}

// ------------------------------------------------------------------------------------------
// camera ray, main() P5/fsh:920-925
// ------------------------------------------------------------------------------------------
// the pinhole direction M (vx, vy, -1.5, 0) before normalisation; seed leaves with the two jitter draws taken
__device__ __forceinline__ vec3 pinhole_dir(const RenderDev& rd, uint32_t px, uint32_t py, uint32_t frame, uint32_t& seed) {
    seed = pixel_seed(px, py, frame);
    float pixx = EZ_DIV((float)px + 0.5f, (float)rd.width) * 2.0f - 1.0f;
    float pixy = EZ_DIV((float)py + 0.5f, (float)rd.height) * 2.0f - 1.0f;
    float aax = EZ_DIV(rand01(seed) - 0.5f, (float)rd.width);
    float aay = EZ_DIV(rand01(seed) - 0.5f, (float)rd.height);
    float vx = pixx + aax, vy = pixy + aay, vz = -1.5f, vw = 0.0f;
    const float* m = rd.cam;
    return ez_v3(((m[0] * vx + m[4] * vy) + m[8] * vz) + m[12] * vw,
                 ((m[1] * vx + m[5] * vy) + m[9] * vz) + m[13] * vw,
                 ((m[2] * vx + m[6] * vy) + m[10] * vz) + m[14] * vw);
}
__device__ __forceinline__ void primary_ray(const RenderDev& rd, uint32_t px, uint32_t py, uint32_t frame, uint32_t& seed,
                                            vec3& o, vec3& d) {
    const vec3 dir = pinhole_dir(rd, px, py, frame, seed);
    o = ez_v3(rd.eye[0], rd.eye[1], rd.eye[2]);
    d = ez_normalize(dir);
}
// the thin-lens camera ray (EZRT_PARAM_THIN_LENS; ezrt_math.h, DESIGN.md section 13): the pinhole's seed, jitter and direction,
// then the lens point from the lens stream; seed leaves as primary_ray leaves it
__device__ __forceinline__ void lens_ray(const RenderDev& rd, const LensDev& lens, uint32_t px, uint32_t py, uint32_t frame, uint32_t& seed,
                                         vec3& o, vec3& d) {
    const vec3 dir = pinhole_dir(rd, px, py, frame, seed);
    float r_a, r_b;
    ez_lens_draws(px, py, frame, &r_a, &r_b);
    ez_lens_ray(&lens, dir, r_a, r_b, &o, &d);
}
// the camera ray of a render: the pinhole's, or the thin lens's (LENS)
template <bool LENS>
__device__ __forceinline__ void camera_ray(const RenderDev& rd, const LensDev& lens, uint32_t px, uint32_t py, uint32_t frame, uint32_t& seed,
                                           vec3& o, vec3& d) {
    if (LENS) lens_ray(rd, lens, px, py, frame, seed, o, d);
    else primary_ray(rd, px, py, frame, seed, o, d);
}

// ------------------------------------------------------------------------------------------
// one bounce of the integrators (P3/fsh:381-410, P4/fsh:483-514, P5/fsh:767-804, P5/fsh:815-887)
// ------------------------------------------------------------------------------------------
struct PathRegs {
    vec3 o, d;          // current ray
    uint32_t seed;
    vec3 history, f_r;  // throughput before this bounce, BRDF value of this bounce
    float cosine_i, pdf;
};
struct ShadowRay {
    bool valid;
    vec3 o, d, contrib;      // contrib: DEFER_NEE = false
    vec3 N, V, history;      // DEFER_NEE = true: the inputs of nee_contrib, evaluated only if the shadow ray gets through (k_nee)
    int matId;
    float tmax, pdf;         // light sampling mode: the shadow ray's bound and the light sample's pdf ...
    int light_mat;           // ... and the light's material id (nee_light_contrib)
};

// Lo += a*b*c*s/p evaluated left to right as GLSL does
__device__ __forceinline__ vec3 contrib3(vec3 a, vec3 b, vec3 c, float s, float p) {
    return ez_divs(ez_scale(ez_mul(ez_mul(a, b), c), s), p);
}

// Account for the result (t,tri) of tracing p's ray, which was generated at bounce-1 (bounce==0:
// the primary ray), then -- if the path continues -- sample the next direction and fill p with the
// next ray.  Returns false when the path ends.  Lo/Le/primary_miss are the sample's accumulators.
// MODE >= 0: the integrator is a compile-time constant (k_shade<MODE>: each instantiation carries only its own
// integrator -- the four-in-one kernel was 7288 instructions = 116 KB and instruction-fetch bound in the IS/MIS mode,
// ncu); MODE < 0: rd.mode at run time (megakernel).
// (sob_u, sob_v) = sobolVec2(frame + 1, bounce) (P5/fsh:372-376), the same for every pixel of a frame: the caller looks it
// up (k_shade: a per-block table) or computes it (sobol_pair).
__device__ __forceinline__ float2 sobol_pair(int bounce, uint32_t frame) {
    return make_float2(sobol_gray((uint32_t)bounce * 2u, frame + 1u), sobol_gray((uint32_t)bounce * 2u + 1u, frame + 1u));
}
// The environment sample's contribution if its shadow ray gets through (P5/fsh:829-841): history * mis * color * f_r * NdotL / pdf_light,
// left to right.  One definition for the in-line evaluation (megakernel) and the deferred one (k_nee, after the shadow pass).
__device__ __forceinline__ vec3 nee_contrib(const SceneDev& sc, const RenderDev& rd, int mode, vec3 V, vec3 N, vec3 Lh, const MaterialDev& mat,
                                            vec3 history) {
    const float NdotLh = ez_dot(N, Lh);
    const vec3 fr_h = brdf_evaluate<false>(V, N, Lh, mat);
    const float pdf_h = brdf_pdf(V, N, Lh, mat);
    const vec3 color = hdr_color(sc, rd, Lh, mode);
    const float pdf_light = hdr_pdf(sc, Lh);
    const float mis_weight = mis_mix_weight(pdf_light, pdf_h);
    return ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, mis_weight), color), fr_h), NdotLh), pdf_light);
}
// The light sampling mode's light sample (ezrt_math.h, DESIGN.md section 10), evaluated by k_nee<EZRT_MODE_DISNEY_LIGHTS> for the lit
// rays: history * mis(pdf_l, BRDF_Pdf) * E * f_r * dot(N, L) / pdf_l, left to right as nee_contrib.
__device__ __forceinline__ vec3 nee_light_contrib(vec3 V, vec3 N, vec3 L, const MaterialDev& mat, vec3 history, vec3 E, float pdf_l) {
    const float NdotL = ez_dot(N, L);
    const vec3 fr = brdf_evaluate<false>(V, N, L, mat);
    const float pdf_b = brdf_pdf(V, N, L, mat);
    const float mis_weight = mis_mix_weight(pdf_l, pdf_b);
    return ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, mis_weight), E), fr), NdotL), pdf_l);
}
// ... with EZRT_PARAM_TRANSMISSION: the same product with the mixture's f and pdf, and nee_light_contrib's bits where t == 0
__device__ __forceinline__ vec3 nee_trans_contrib(const SceneDev& sc, vec3 V, vec3 N, vec3 L, int matId, const MaterialDev& mat, bool inside,
                                                  vec3 history, vec3 E, float pdf_l) {
    const TransLobe tl = trans_lobe(sc, matId, mat, inside);
    if (tl.t == 0.0f) return nee_light_contrib(V, N, L, mat, history, E, pdf_l);
    const float NdotL = ez_dot(N, L);
    float pdf_b;
    const vec3 fr = bsdf_evaluate(V, N, L, mat, tl, pdf_b);
    const float mis_weight = mis_mix_weight(pdf_l, pdf_b);
    return ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, mis_weight), E), fr), NdotL), pdf_l);
}
// ... at a medium vertex (EZRT_PARAM_MEDIUM; ezrt_math.h, DESIGN.md section 14), before the shadow ray's transmittance: the phase
// function in place of f_r and the cosine 1; d = the path's propagation direction at the vertex
__device__ __forceinline__ vec3 nee_medium_contrib(vec3 d, vec3 L, float g, vec3 history, vec3 E, float pdf_l) {
    const float p = ez_hg_pdf(d, L, g);
    const float mis_weight = mis_mix_weight(pdf_l, p);
    return ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, mis_weight), E), splat3(p)), 1.0f), pdf_l);
}
// the cosine a path record carries: with TRANS its sign is the bit "the BSDF sample went below the surface"
template <bool TRANS>
__device__ __forceinline__ float path_cos(float c) { return TRANS ? ez_abs(c) : c; }
// the three vertices of triangle `tri` in the policy's index space (flat or indexed record)
__device__ __forceinline__ void tri_vertices(const SceneDev& sc, int tri, bool accel_space, vec3& p1, vec3& p2, vec3& p3) {
    const float4* g = tri_geo_rec(sc, tri, accel_space);
    const float4* v = g;
    uint32_t i1 = 1u, i2 = 2u, i3 = 3u;
    if (accel_space && sc.acc_tri_indexed) {
        const uint4 qi = __ldg(reinterpret_cast<const uint4*>(g + 1));
        v = sc.acc_tri_vert; i1 = qi.x; i2 = qi.y; i3 = qi.z;
    }
    p1 = f4xyz(ldg4(v + i1)); p2 = f4xyz(ldg4(v + i2)); p3 = f4xyz(ldg4(v + i3));
}
// EZRT_PARAM_TEXTURES (ezrt_math.h, DESIGN.md section 15): the base colour `base` of the hit at P on triangle `tri` (the policy's index
// space) times its texture's filtered colour at the hit's UV; `base` itself for texture id -1.  One 32-byte texcoord record as two
// 128-bit loads, the triangle's records again (L1 hits after surface_hit), four texel words and twelve table reads through L1.
__device__ __forceinline__ vec3 tex_base_color(const SceneDev& sc, const TexDev& tex, int tri, bool accel_space, vec3 P, vec3 base, float* uv_out = nullptr) {
    const float4* r = (accel_space ? tex.acc_rec : tex.rec) + (size_t)tri * 2;
    const float4 a = ldg4(r), b = ldg4(r + 1);
    const int id = __float_as_int(b.z);
    vec3 p1, p2, p3;
    tri_vertices(sc, tri, accel_space, p1, p2, p3);
    const vec3 Ng = f4xyz(ldg4(tri_geo_rec(sc, tri, accel_space)));
    float w1, w2, w3, u, v;
    ez_tri_bary(P, p1, p2, p3, Ng, &w1, &w2, &w3);
    const float uv6[6] = {a.x, a.y, a.z, a.w, b.x, b.y};
    ez_tex_uv(w1, w2, w3, uv6, &u, &v);
    if (uv_out) { uv_out[0] = u; uv_out[1] = v; }
    if (id < 0) return base;
    const int4 t = __ldg(tex.table + id);
    return ez_mul(base, ez_tex_sample(tex.texels + t.x, t.y, t.z, u, v, tex.lut));
}
// EZRT_PARAM_MATERIAL_MAPS (ezrt_math.h, DESIGN.md section 16): the whole lookup of a hit in one place -- mat's base colour textured
// as tex_base_color's, its roughness and metallic by the metallic-roughness map, and N (surface_hit's, for a hit from `inside`,
// viewed from V) replaced by the normal map's.  The same loads as tex_base_color, plus four texel words per map.
__device__ __forceinline__ void tex_material(const SceneDev& sc, const TexDev& tex, const MapsDev& maps_dev, int tri, bool accel_space, vec3 P, vec3 V, bool inside,
                                             MaterialDev& mat, vec3& N, float* uv_out = nullptr) {
    const float4* r = (accel_space ? tex.acc_rec : tex.rec) + (size_t)tri * 2;
    const float4 a = ldg4(r), b = ldg4(r + 1);
    const int id = __float_as_int(b.z);
    const uint32_t maps = __float_as_uint(b.w);
    vec3 p1, p2, p3;
    tri_vertices(sc, tri, accel_space, p1, p2, p3);
    const vec3 Ng = f4xyz(ldg4(tri_geo_rec(sc, tri, accel_space)));
    float w1, w2, w3, u, v;
    ez_tri_bary(P, p1, p2, p3, Ng, &w1, &w2, &w3);
    const float uv6[6] = {a.x, a.y, a.z, a.w, b.x, b.y};
    ez_tex_uv(w1, w2, w3, uv6, &u, &v);
    if (uv_out) { uv_out[0] = u; uv_out[1] = v; }
    if (id >= 0) {
        const int4 t = __ldg(tex.table + id);
        mat.baseColor = ez_mul(mat.baseColor, ez_tex_sample(tex.texels + t.x, t.y, t.z, u, v, tex.lut));
    }
    const int mr = ez_maps_mr_id(maps), nm = ez_maps_normal_id(maps);
    if (mr >= 0) {
        const int4 t = __ldg(tex.table + mr);
        ez_mr_apply(ez_tex_sample(tex.texels + t.x, t.y, t.z, u, v, maps_dev.unorm), &mat.roughness, &mat.metallic);
    }
    if (nm >= 0) {
        const int4 t = __ldg(tex.table + nm);
        N = ez_normal_map(p1, p2, p3, uv6, u, v, ez_tex_sample(tex.texels + t.x, t.y, t.z, u, v, maps_dev.unorm), N, inside, V);
    }
}

// A medium vertex (EZRT_PARAM_MEDIUM; ezrt_math.h, DESIGN.md section 14): p's segment scattered at t_s before its hit (hit_t,
// hit_tri) or its miss.  The weights of the segment (bounce >= 1) and the albedo enter the history; then, below max_bounce, one light
// sample from P as at a surface but without the hemisphere test and the self exclusion (its shadow ray carries EZRT_MEDIUM_VERTEX
// and d), and the phase function's sample as the next ray with the record (splat(p), p, 1).  Returns false when the path ends.
// TEX: the first-hit record's albedo is the textured base colour.  MAPS: ... and its normal the mapped one.
template <bool AOV, bool ENV, bool TEX = false, bool MAPS = false>
__device__ __forceinline__ bool medium_step(const SceneDev& sc, const RenderDev& rd, int bounce, PathRegs& p, float t_s, float hit_t,
                                            int hit_tri, vec3& Lo, vec3& Le, bool& primary_miss, ShadowRay& sh, float4* aov_rec,
                                            const LightsDev& lights, const EnvDev& env, const MediumDev& med, const TexDev& tex = TexDev{},
                                            const MapsDev& maps = MapsDev{}) {
    if (bounce == 0) {
        Lo = splat3(0.0f);
        Le = splat3(0.0f);
        primary_miss = hit_tri < 0;   // k_blend: a camera ray that left the scene, its colour the Lo of its medium vertices
        if (AOV && hit_tri >= 0) {    // the feature buffers describe the first surface behind the medium
            SurfaceHit hit = surface_hit(sc, p.o, p.d, hit_t, hit_tri, false, rd.accel_space != 0);
            MaterialDev mat = load_material(sc, hit.matId);
            if constexpr (MAPS) tex_material(sc, tex, maps, hit_tri, rd.accel_space != 0, hit.P, ez_neg(p.d), hit.inside, mat, hit.N);
            else if constexpr (TEX) mat.baseColor = tex_base_color(sc, tex, hit_tri, rd.accel_space != 0, hit.P, mat.baseColor);
            aov_rec[0] = make_float4(mat.baseColor.x, mat.baseColor.y, mat.baseColor.z, hit_t);
            aov_rec[1] = make_float4(hit.N.x, hit.N.y, hit.N.z, 0.0f);
        }
    } else {
        p.history = ez_mul(p.history, ez_divs(ez_scale(p.f_r, p.cosine_i), p.pdf));
    }
    p.history = ez_mul(p.history, med.albedo);
    if (bounce >= rd.max_bounce) return false;
    const vec3 P = ez_add(p.o, ez_scale(p.d, t_s));
    const float r_sel = rand01(p.seed);
    const float r_1 = rand01(p.seed);
    const float r_2 = rand01(p.seed);
    bool env_pick = false;
    float r_tri = r_sel;
    if constexpr (ENV) {
        const bool half = (env.p_env == 0.5f);
        env_pick = (env.p_env == 1.0f) || (half && r_sel < 0.5f);
        if (half) r_tri = (r_sel - 0.5f) * 2.0f;
        if (env_pick) {
            int texel;
            const vec3 Le_dir = ez_env_sample(env.row_cdf, env.col_cdf, env.w, env.h, r_1, r_2, &texel);
            const float pdf_e = env.p_env * ez_env_pdf(env.texel_pdf, env.w, env.h, Le_dir);
            if (ez_finite(pdf_e) && pdf_e > 0.0f) {
                sh.valid = true;
                sh.d = Le_dir;
                sh.tmax = EZ_INF;
                sh.pdf = pdf_e;
                sh.light_mat = -1;
            }
        }
    }
    if (!env_pick && lights.n > 0) {
        const float4* lr = lights.rec + 4 * (size_t)ez_light_select(lights.cdf, lights.n, r_tri);
        const float4 a = ldg4(lr), b = ldg4(lr + 1), c = ldg4(lr + 2), e = ldg4(lr + 3);
        const vec3 D = ez_sub(ez_triangle_point(f4xyz(a), f4xyz(b), f4xyz(c), r_1, r_2), P);
        const float dist = EZ_SQRT(ez_dot(D, D));
        const vec3 Ll = ez_normalize(D);
        const float cos_l = ez_abs(ez_dot(f4xyz(e), Ll));
        if (cos_l != 0.0f && dist != 0.0f) {
            sh.valid = true;
            sh.d = Ll;
            sh.tmax = ez_light_tmax(dist);
            sh.pdf = ez_light_pdf(e.w, lights.w_total, dist, cos_l);
            if constexpr (ENV) sh.pdf = sh.pdf * (1.0f - env.p_env);
            sh.light_mat = __float_as_int(a.w);
        }
    }
    if (sh.valid) {
        sh.o = P;
        sh.N = splat3(0.0f); sh.V = p.d; sh.history = p.history; sh.matId = EZRT_MEDIUM_VERTEX;
    }
    const float h_1 = rand01(p.seed);
    const float h_2 = rand01(p.seed);
    const vec3 L = ez_hg_sample(p.d, med.g, h_1, h_2);
    const float pdf = ez_hg_pdf(p.d, L, med.g);
    p.f_r = splat3(pdf);
    p.pdf = pdf;
    p.cosine_i = 1.0f;
    p.o = P;
    p.d = L;
    return true;
}

// DEFER_NEE (wavefront pipeline, IS/MIS mode): the shadow ray carries the inputs of nee_contrib instead of its value -- the
// BRDF / environment evaluation of the light sample runs after the shadow pass, only for the rays that got through, and is
// no longer part of k_shade (5104 instructions, instruction-fetch bound).
// AOV: at bounce 0 a surface hit also writes its first-hit record to aov_rec[0..1] = (base colour, t), (shading normal as
// surface_hit returns it, 0) -- as soon as they are known, so that they are not held through the rest of the step.  A primary
// miss writes nothing.
// ENV (light sampling mode with EZRT_PARAM_ENV_LIGHT, ezrt_math.h, DESIGN.md section 11): the map is one more light, sampled
// with probability env.p_env from the table env; its samples travel as bounded shadow rays with tmax = EZ_INF and light
// material -1.
// TRANS (light sampling mode with EZRT_PARAM_TRANSMISSION, ezrt_math.h, DESIGN.md section 12): a hit on a material with t > 0
// samples and evaluates the mixture with the rough dielectric.  p.cosine_i keeps dot(N, L)'s sign: a BSDF sample below the
// surface weighs 1 where it hits an emitter or leaves the scene.  The shadow ray's material id is ~matId for a hit from inside.
// MEDIUM (light sampling mode with EZRT_PARAM_MEDIUM, ezrt_math.h, DESIGN.md section 14; not with TRANS): the free flight of the
// traced segment comes first; a path that scatters takes a medium vertex (medium_step) instead of its hit or miss.
// TEX (light sampling mode with EZRT_PARAM_TEXTURES, ezrt_math.h, DESIGN.md section 15): every use of the hit's base colour -- the
// BRDF / mixture's evaluation, sampling and pdf, the first-hit record -- takes the textured one (tex_base_color); a light sample's
// shadow ray carries it out through *sh_base, for k_nee.
// MAPS (with TEX; EZRT_PARAM_MATERIAL_MAPS, ezrt_math.h, DESIGN.md section 16): the hit's roughness and metallic are the
// metallic-roughness map's and its shading normal N the normal map's (tex_material), everywhere N and the material are read after
// the lookup: the BSDF, the lobe weights, the light samples' hemisphere tests, the path record's cosine, the shadow ray's N and the
// first-hit record; the emission's MIS and the inside test keep the geometric normal.  *sh_rm carries (roughness, metallic) to k_nee.
template <int MODE, bool DEFER_NEE = false, bool AOV = false, bool ENV = false, bool TRANS = false, bool MEDIUM = false, bool TEX = false,
          bool MAPS = false>
__device__ __forceinline__ bool shade_step(const SceneDev& sc, const RenderDev& rd, int bounce, PathRegs& p, float hit_t,
                                           int hit_tri, uint32_t px, uint32_t py, float2 sob, vec3& Lo, vec3& Le,
                                           bool& primary_miss, ShadowRay& sh, float4* aov_rec = nullptr, LightsDev lights = LightsDev{},
                                           EnvDev env = EnvDev{}, MediumDev med = MediumDev{}, TexDev tex = TexDev{}, vec3* sh_base = nullptr,
                                           float2* sh_rm = nullptr, MapsDev maps = MapsDev{}) {
    sh.valid = false;
    const int mode = (MODE < 0) ? rd.mode : MODE;
    const bool is_mode = (mode == EZRT_MODE_DISNEY_IS_MIS_P5);
    // the light sampling mode exists only as k_shade<EZRT_MODE_DISNEY_LIGHTS> (the megakernel, MODE < 0, rejects it)
    constexpr bool lights_mode = (MODE == EZRT_MODE_DISNEY_LIGHTS);
    const bool below = TRANS && p.cosine_i < 0.0f;   // the BSDF sample went below the surface: no light strategy reaches it
    static_assert(lights_mode || !TEX, "textures are rendered in the light sampling mode");
    static_assert(TEX || !MAPS, "material maps are rendered with the textures");
    if constexpr (MEDIUM) {
        static_assert(lights_mode && !TRANS, "the medium is rendered in the light sampling mode, without transmission");
        if (bounce > 0 && p.pdf <= 0.0f) return false;   // P5/fsh:865, before the free flight's draw
        float t_s;
        const float t_end = (hit_tri < 0) ? __int_as_float(0x7f800000) : hit_t;
        if (ez_medium_flight(&med, p.o, p.d, t_end, &p.seed, &t_s))
            return medium_step<AOV, ENV, TEX, MAPS>(sc, rd, bounce, p, t_s, hit_t, hit_tri, Lo, Le, primary_miss, sh, aov_rec, lights, env, med, tex, maps);
    }
    if (bounce == 0) {
        Lo = splat3(0.0f);
        Le = splat3(0.0f);
        primary_miss = false;
        if (hit_tri < 0) {  // P5/fsh:931-933
            Lo = hdr_color(sc, rd, p.d, mode);
            primary_miss = true;
            return false;
        }
    } else {
        if ((is_mode || lights_mode) && p.pdf <= 0.0f) return false;  // P5/fsh:865
        if (hit_tri < 0) {  // miss: sky contribution, then break
            vec3 sky = hdr_color(sc, rd, p.d, mode);
            if (is_mode) {  // P5/fsh:868-878
                float pdf_light = hdr_pdf(sc, p.d);
                float mis_weight = mis_mix_weight(p.pdf, pdf_light);
                vec3 c = ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(p.history, mis_weight), sky), p.f_r), p.cosine_i), p.pdf);
                Lo = ez_add(Lo, c);
            } else if (ENV) {   // the map is a light: MIS against its sampling density, in mode 3's order
                const float w = (env.p_env > 0.0f && !below) ? mis_mix_weight(p.pdf, env.p_env * ez_env_pdf(env.texel_pdf, env.w, env.h, p.d)) : 1.0f;
                Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(p.history, w), sky), p.f_r), path_cos<TRANS>(p.cosine_i)), p.pdf));
            } else {
                Lo = ez_add(Lo, contrib3(p.history, sky, p.f_r, path_cos<TRANS>(p.cosine_i), p.pdf));
            }
            return false;
        }
    }
    const bool fudge = (mode == EZRT_MODE_DIFFUSE_P3 || mode == EZRT_MODE_DISNEY_ANISO_P4);
    SurfaceHit hit = surface_hit(sc, p.o, p.d, hit_t, hit_tri, fudge, rd.accel_space != 0);
    MaterialDev mat = load_material(sc, hit.matId);
    if constexpr (TEX) {   // not at the last vertex, where only the emission is read
        if ((AOV && bounce == 0) || bounce < rd.max_bounce) {
            if constexpr (MAPS) {
                tex_material(sc, tex, maps, hit_tri, rd.accel_space != 0, hit.P, ez_neg(p.d), hit.inside, mat, hit.N);
                *sh_rm = make_float2(mat.roughness, mat.metallic);
            } else {
                mat.baseColor = tex_base_color(sc, tex, hit_tri, rd.accel_space != 0, hit.P, mat.baseColor);
            }
            *sh_base = mat.baseColor;
        }
    }
    if (bounce == 0) {
        Le = mat.emissive;  // P5/fsh:936
        if (AOV) {
            aov_rec[0] = make_float4(mat.baseColor.x, mat.baseColor.y, mat.baseColor.z, hit_t);
            aov_rec[1] = make_float4(hit.N.x, hit.N.y, hit.N.z, 0.0f);
        }
    } else {
        if (lights_mode) {   // a BRDF sample that hit a light: MIS against the light sampling pdf of the hit point
            float w = 1.0f;
            const float lum = ez_luminance(mat.emissive);
            if (lum > 0.0f && !below) {   // lum <= 0: the weight area * lum is never a light; below: weight 1
                vec3 p1, p2, p3;
                tri_vertices(sc, hit_tri, rd.accel_space != 0, p1, p2, p3);
                if (ez_is_light(ez_light_weight(p1, p2, p3, mat.emissive))) {
                    const vec3 Ng = f4xyz(ldg4(tri_geo_rec(sc, hit_tri, rd.accel_space != 0)));
                    if constexpr (ENV) w = mis_mix_weight(p.pdf, (1.0f - env.p_env) * ez_light_pdf(lum, lights.w_total, hit_t, ez_abs(ez_dot(Ng, p.d))));
                    else w = mis_mix_weight(p.pdf, ez_light_pdf(lum, lights.w_total, hit_t, ez_abs(ez_dot(Ng, p.d))));
                }
            }
            Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(p.history, w), mat.emissive), p.f_r), path_cos<TRANS>(p.cosine_i)), p.pdf));
        } else {
            Lo = ez_add(Lo, contrib3(p.history, mat.emissive, p.f_r, p.cosine_i, p.pdf));
        }
        p.history = ez_mul(p.history, ez_divs(ez_scale(p.f_r, path_cos<TRANS>(p.cosine_i)), p.pdf));
    }
    if (bounce >= rd.max_bounce) return false;

    vec3 V = ez_neg(p.d);
    vec3 N = hit.N;
    vec3 L;
    if (lights_mode) {
        // one light sample on the emissive triangles (ezrt_math.h, DESIGN.md section 10), then mode 3's BRDF sample.  The three
        // draws of the light sample come first and are made whether or not the scene has a light.
        const float r_sel = rand01(p.seed);
        const float r_1 = rand01(p.seed);
        const float r_2 = rand01(p.seed);
        float xi_1 = sob.x, xi_2 = sob.y;
        cp_rotate(xi_1, xi_2, px, py);
        const float xi_3 = rand01(p.seed);
        L = sample_brdf(xi_1, xi_2, xi_3, V, N, mat);
        float NdotL = ez_dot(N, L);
        vec3 fr_l = splat3(0.0f);
        float pdf_l = 0.0f;
        if (NdotL > 0.0f) { fr_l = brdf_evaluate<false>(V, N, L, mat); pdf_l = brdf_pdf(V, N, L, mat); }
        bool go = !(NdotL <= 0.0f);   // the path continues
        if constexpr (TRANS) {   // a material with a dielectric lobe: the mixture's sample instead, with one more draw, r_t
            const TransLobe tl = trans_lobe(sc, hit.matId, mat, hit.inside);
            if (tl.t != 0.0f) go = bsdf_sample(xi_1, xi_2, xi_3, rand01(p.seed), V, N, mat, tl, L, fr_l, pdf_l, NdotL);
        }
        const int sh_mat = (TRANS && hit.inside) ? ~hit.matId : hit.matId;   // k_nee<.., TRANS> needs the side for eta
        bool env_pick = false;
        float r_tri = r_sel;   // the triangle light's selection number
        if constexpr (ENV) {   // the environment with probability p_env: r_sel < 0.5 beside triangle lights, always without
            const bool half = (env.p_env == 0.5f);
            env_pick = (env.p_env == 1.0f) || (half && r_sel < 0.5f);
            if (half) r_tri = (r_sel - 0.5f) * 2.0f;
            if (env_pick) {
                int texel;
                const vec3 Le_dir = ez_env_sample(env.row_cdf, env.col_cdf, env.w, env.h, r_1, r_2, &texel);
                const float pdf_e = env.p_env * ez_env_pdf(env.texel_pdf, env.w, env.h, Le_dir);
                if (ez_finite(pdf_e) && pdf_e > 0.0f && ez_dot(N, Le_dir) > 0.0f) {
                    sh.valid = true;
                    sh.o = hit.P;
                    sh.d = Le_dir;
                    sh.N = N; sh.V = V; sh.history = p.history; sh.matId = sh_mat;
                    sh.tmax = EZ_INF;
                    sh.pdf = pdf_e;
                    sh.light_mat = -1;
                }
            }
        }
        if (!env_pick && lights.n > 0) {
            const float4* lr = lights.rec + 4 * (size_t)ez_light_select(lights.cdf, lights.n, r_tri);
            const float4 a = ldg4(lr), b = ldg4(lr + 1), c = ldg4(lr + 2), e = ldg4(lr + 3);
            const int self = __float_as_int(rd.accel_space ? c.w : b.w);   // the light's triangle in the hit's index space
            const vec3 D = ez_sub(ez_triangle_point(f4xyz(a), f4xyz(b), f4xyz(c), r_1, r_2), hit.P);
            const float dist = EZ_SQRT(ez_dot(D, D));
            const vec3 Ll = ez_normalize(D);
            const float cos_l = ez_abs(ez_dot(f4xyz(e), Ll));
            if (self != hit_tri && ez_dot(N, Ll) > 0.0f && cos_l != 0.0f && dist != 0.0f) {
                sh.valid = true;
                sh.o = hit.P;
                sh.d = Ll;
                sh.N = N; sh.V = V; sh.history = p.history; sh.matId = sh_mat;
                sh.tmax = ez_light_tmax(dist);
                sh.pdf = ez_light_pdf(e.w, lights.w_total, dist, cos_l);
                if constexpr (ENV) sh.pdf = sh.pdf * (1.0f - env.p_env);
                sh.light_mat = __float_as_int(a.w);
            }
        }
        if (!go) return false;
        p.f_r = fr_l;
        p.pdf = pdf_l;   // <= 0: traced, then break
        p.cosine_i = NdotL;   // TRANS: < 0 below the surface
    } else if (is_mode) {
        // environment importance sample + shadow ray (P5/fsh:820-842), then the BRDF sample (:845-865).  The three
        // random numbers are drawn in the shader's order (two for SampleHdr :822, one for the lobe choice :849); the BRDF
        // value and pdf of the two directions are evaluated by ONE copy of the code (a two-trip loop that is not unrolled)
        float r1 = rand01(p.seed);
        float r2 = rand01(p.seed);
        float xi_1 = sob.x, xi_2 = sob.y;
        cp_rotate(xi_1, xi_2, px, py);
        float xi_3 = rand01(p.seed);
        const vec3 Lh = sample_hdr(sc, r1, r2);
        const float NdotLh = ez_dot(N, Lh);
        L = sample_brdf(xi_1, xi_2, xi_3, V, N, mat);
        const float NdotL = ez_dot(N, L);
        vec3 fr_l = splat3(0.0f);
        float pdf_l = 0.0f;
        if (NdotL > 0.0f) { fr_l = brdf_evaluate<false>(V, N, L, mat); pdf_l = brdf_pdf(V, N, L, mat); }
        if (NdotLh > 0.0f) {
            sh.valid = true;
            sh.o = hit.P;
            sh.d = Lh;
            if (DEFER_NEE) {
                sh.N = N; sh.V = V; sh.history = p.history; sh.matId = hit.matId;
            } else {
                sh.contrib = nee_contrib(sc, rd, mode, V, N, Lh, mat, p.history);
            }
        }
        if (NdotL <= 0.0f) return false;  // :854
        p.f_r = fr_l;
        p.pdf = pdf_l;   // <= 0: traced, then break (:860-865)
        p.cosine_i = NdotL;
    } else {
        vec3 Lh;
        if (mode == EZRT_MODE_DISNEY_SOBOL_P5) {  // P5/fsh:771-776
            float u = sob.x, v = sob.y;
            cp_rotate(u, v, px, py);
            Lh = sample_hemisphere(u, v);
        } else {  // P3/fsh:110-115: z = rand(), then phi
            float z = rand01(p.seed);
            float r = ez_max(0.0f, EZ_SQRT(1.0f - z * z));
            float phi = 2.0f * EZ_PI * rand01(p.seed);
            Lh = ez_v3(r * ezd_cos(phi), r * ezd_sin(phi), z);
        }
        L = to_normal_hemisphere(Lh, N);
        p.pdf = EZ_DIV(1.0f, 2.0f * EZ_PI);
        p.cosine_i = ez_max(0.0f, ez_dot(L, N));
        if (mode == EZRT_MODE_DIFFUSE_P3) p.f_r = ez_divs(mat.baseColor, EZ_PI);
        else if (mode == EZRT_MODE_DISNEY_ANISO_P4) p.f_r = brdf_evaluate<true>(V, N, L, mat);
        else p.f_r = brdf_evaluate<false>(V, N, L, mat);
    }
    p.o = hit.P;
    p.d = L;
    return true;
}

#endif
