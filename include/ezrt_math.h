/*
 * ezrt_math.h -- the NORMATIVE fp32 arithmetic of the EzRT path-tracing hot path.
 *
 * The reference (AKGWSB/EzRT) runs this path as GLSL (P5/shaders/fshader.fsh) on top of
 * driver-implemented built-ins (normalize, cross, mix, sin, cos, atan, asin, log, pow ...)
 * and glm on the host; neither is bit-specified, and the reference ships no test that pins
 * them (SURVEY.md 8c; how parity is pinned nevertheless: DESIGN.md section 2).  This header therefore DEFINES every such
 * operation as a fixed sequence of IEEE-754 binary32  + - * / sqrt fma  operations, so the
 * same source gives bit-identical results under g++ (host, -ffp-contract=off -mfma) and
 * nvcc (device, -fmad=false, default -prec-div/-prec-sqrt/-ftz=false).
 *
 * Rules:
 *   - every fused multiply-add is spelled EZ_FMA(); nothing else may be contracted;
 *   - min/max are the GLSL/glm ternaries: min(x,y) = (y<x)?y:x, max(x,y) = (x<y)?y:x
 *     (P5/fsh:226-230; glm/detail/func_common.inl);
 *   - dot/cross use FMA chains (what a GPU shader compiler emits for the GLSL built-ins);
 *   - transcendental functions are Cephes-style single-precision kernels (published
 *     algorithm, S. Moshier, "Cephes Mathematical Library", sinf/cosf/logf/expf/atanf/
 *     asinf) restated with explicit operation order.
 *
 * Used by: the CUDA kernels (ezrt_b200/csrc), the host scene pipeline, and the CPU oracle
 * (oracle/), which must share these primitive definitions to be comparable bit-for-bit.
 */
#ifndef EZRT_MATH_H
#define EZRT_MATH_H

#include <stdint.h>
#include <string.h>
#include <math.h>

#if defined(__CUDACC__)
#define EZ_HD __host__ __device__ __forceinline__
#else
#define EZ_HD static inline
#endif

#if defined(__CUDA_ARCH__)
#define EZ_FMA(a, b, c) __fmaf_rn((a), (b), (c))
#define EZ_SQRT(a) __fsqrt_rn(a)
#define EZ_DIV(a, b) __fdiv_rn((a), (b))
#else
#define EZ_FMA(a, b, c) __builtin_fmaf((a), (b), (c))
#define EZ_SQRT(a) __builtin_sqrtf(a)
#define EZ_DIV(a, b) ((a) / (b))
#endif

/* the shader's constants: P5/fsh:27-28 (PI is one ulp below float(pi)) */
#define EZ_PI 3.1415926f
#define EZ_INF 114514.0f

/* ------------------------------------------------------------------ bit casts */
EZ_HD uint32_t ez_f2u(float f) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    uint32_t u; memcpy(&u, &f, 4); return u;
#endif
}
EZ_HD float ez_u2f(uint32_t u) {
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}

/* ------------------------------------------------------------------ scalar helpers */
EZ_HD float ez_min(float x, float y) { return (y < x) ? y : x; }
EZ_HD float ez_max(float x, float y) { return (x < y) ? y : x; }
EZ_HD float ez_abs(float x) { return ez_u2f(ez_f2u(x) & 0x7fffffffu); }
EZ_HD float ez_clamp(float x, float lo, float hi) { return ez_min(ez_max(x, lo), hi); }
/* GLSL mix(x,y,a) = x*(1-a) + y*a */
EZ_HD float ez_mix(float x, float y, float a) { return x * (1.0f - a) + y * a; }
EZ_HD float ez_sqr(float x) { return x * x; }
/* floor, exact for every input: NaN, +-inf and every |x| >= 2^23 are whole already and return themselves (no conversion to int
 * out of its range, which the host leaves undefined and the device saturates); floor(-0) = +0 */
EZ_HD float ez_floor(float x) {
    if (!(ez_abs(x) < 8388608.0f)) return x;
    float t = (float)(int)x;
    return (t > x) ? (t - 1.0f) : t;
}
/* a texel index in [0, n): f a whole number (ez_floor's result) or NaN, clamped in float before the conversion, so that NaN and
 * f < 0 give 0 and f > n - 1 gives n - 1 for every f */
EZ_HD int ez_texel_clamp(float f, int n) {
    const int i = (f > 0.0f) ? (int)ez_min(f, 2147483520.0f) : 0;
    return (i > n - 1) ? n - 1 : i;
}
/* uint -> float, round to nearest even (GLSL float(uint)) */
EZ_HD float ez_u32_to_float(uint32_t u) {
#if defined(__CUDA_ARCH__)
    return __uint2float_rn(u);
#else
    return (float)u;
#endif
}

/* ------------------------------------------------------------------ vec3 */
struct ez_vec3 {
    float x, y, z;
};
typedef struct ez_vec3 ez_vec3;

EZ_HD ez_vec3 ez_v3(float x, float y, float z) { ez_vec3 v; v.x = x; v.y = y; v.z = z; return v; }
EZ_HD ez_vec3 ez_add(ez_vec3 a, ez_vec3 b) { return ez_v3(a.x + b.x, a.y + b.y, a.z + b.z); }
EZ_HD ez_vec3 ez_sub(ez_vec3 a, ez_vec3 b) { return ez_v3(a.x - b.x, a.y - b.y, a.z - b.z); }
EZ_HD ez_vec3 ez_mul(ez_vec3 a, ez_vec3 b) { return ez_v3(a.x * b.x, a.y * b.y, a.z * b.z); }
EZ_HD ez_vec3 ez_scale(ez_vec3 a, float s) { return ez_v3(a.x * s, a.y * s, a.z * s); }
EZ_HD ez_vec3 ez_divs(ez_vec3 a, float s) { return ez_v3(EZ_DIV(a.x, s), EZ_DIV(a.y, s), EZ_DIV(a.z, s)); }
EZ_HD ez_vec3 ez_neg(ez_vec3 a) { return ez_v3(-a.x, -a.y, -a.z); }
EZ_HD ez_vec3 ez_vmin(ez_vec3 a, ez_vec3 b) { return ez_v3(ez_min(a.x, b.x), ez_min(a.y, b.y), ez_min(a.z, b.z)); }
EZ_HD ez_vec3 ez_vmax(ez_vec3 a, ez_vec3 b) { return ez_v3(ez_max(a.x, b.x), ez_max(a.y, b.y), ez_max(a.z, b.z)); }
EZ_HD ez_vec3 ez_vmix(ez_vec3 a, ez_vec3 b, float t) {
    return ez_v3(ez_mix(a.x, b.x, t), ez_mix(a.y, b.y, t), ez_mix(a.z, b.z, t));
}
/* dot = fma(z,z, fma(y,y, x*x)) */
EZ_HD float ez_dot(ez_vec3 a, ez_vec3 b) { return EZ_FMA(a.z, b.z, EZ_FMA(a.y, b.y, a.x * b.x)); }
/* cross: each component a*b - c*d = fma(a, b, -(c*d)) */
EZ_HD ez_vec3 ez_cross(ez_vec3 a, ez_vec3 b) {
    return ez_v3(EZ_FMA(a.y, b.z, -(a.z * b.y)),
                 EZ_FMA(a.z, b.x, -(a.x * b.z)),
                 EZ_FMA(a.x, b.y, -(a.y * b.x)));
}
/* normalize(v) = v * (1/sqrt(dot(v,v)))   (glm: v * inversesqrt(dot(v,v))) */
EZ_HD ez_vec3 ez_normalize(ez_vec3 v) {
    float inv = EZ_DIV(1.0f, EZ_SQRT(ez_dot(v, v)));
    return ez_v3(v.x * inv, v.y * inv, v.z * inv);
}
/* reflect(I,N) = I - 2*dot(N,I)*N */
EZ_HD ez_vec3 ez_reflect(ez_vec3 I, ez_vec3 N) {
    float k = 2.0f * ez_dot(N, I);
    return ez_v3(I.x - k * N.x, I.y - k * N.y, I.z - k * N.z);
}

/* ------------------------------------------------------------------ frexp / ldexp */
/* x = m * 2^e, m in [0.5,1); x must be finite and > 0 */
EZ_HD float ez_frexp_pos(float x, int* e) {
    uint32_t u = ez_f2u(x);
    int bias = 0;
    if ((u & 0x7f800000u) == 0u) { /* denormal: scale by 2^24 (exact) */
        x = x * 16777216.0f;
        u = ez_f2u(x);
        bias = -24;
    }
    *e = (int)((u >> 23) & 0xffu) - 126 + bias;
    return ez_u2f((u & 0x807fffffu) | 0x3f000000u);
}
/* z * 2^n, z finite; two-step so that the intermediate scale factors stay normal */
EZ_HD float ez_ldexp(float z, int n) {
    if (n > 254) n = 254;
    if (n < -252) n = -252;
    int n1 = n / 2;
    int n2 = n - n1;
    float s1 = ez_u2f((uint32_t)(n1 + 127) << 23);
    float s2 = ez_u2f((uint32_t)(n2 + 127) << 23);
    return (z * s1) * s2;
}

/* ------------------------------------------------------------------ sin / cos */
#define EZ_FOPI 1.27323954473516f
#define EZ_DP1 0.78515625f
#define EZ_DP2 2.4187564849853515625e-4f
#define EZ_DP3 3.77489497744594108e-8f

EZ_HD float ez_sin_poly(float x, float z) {
    float y = ((-1.9515295891e-4f * z + 8.3321608736e-3f) * z - 1.6666654611e-1f) * z * x;
    return y + x;
}
EZ_HD float ez_cos_poly(float z) {
    float y = ((2.443315711809948e-5f * z - 1.388731625493765e-3f) * z + 4.166664568298827e-2f) * z * z;
    y = y - 0.5f * z;
    return y + 1.0f;
}
/* valid for |x| < 8192 (the path only produces |x| <= 4*pi); larger arguments return 0 / 1 */
EZ_HD float ez_sin(float xx) {
    float sign = 1.0f;
    float x = xx;
    if (x < 0.0f) { sign = -1.0f; x = -x; }
    if (!(x < 8192.0f)) return 0.0f;
    int j = (int)(EZ_FOPI * x);
    float y = (float)j;
    if (j & 1) { j += 1; y += 1.0f; }
    j &= 7;
    if (j > 3) { sign = -sign; j -= 4; }
    x = ((x - y * EZ_DP1) - y * EZ_DP2) - y * EZ_DP3;
    float z = x * x;
    float r = (j == 1 || j == 2) ? ez_cos_poly(z) : ez_sin_poly(x, z);
    return (sign < 0.0f) ? -r : r;
}
EZ_HD float ez_cos(float xx) {
    float sign = 1.0f;
    float x = xx;
    if (x < 0.0f) x = -x;
    if (!(x < 8192.0f)) return 1.0f;
    int j = (int)(EZ_FOPI * x);
    float y = (float)j;
    if (j & 1) { j += 1; y += 1.0f; }
    j &= 7;
    if (j > 3) { j -= 4; sign = -sign; }
    if (j > 1) sign = -sign;
    x = ((x - y * EZ_DP1) - y * EZ_DP2) - y * EZ_DP3;
    float z = x * x;
    float r = (j == 1 || j == 2) ? ez_sin_poly(x, z) : ez_cos_poly(z);
    return (sign < 0.0f) ? -r : r;
}

/* ------------------------------------------------------------------ log / exp / pow */
/* natural log; x <= 0 or NaN returns -EZ_HUGE (x==0) or NaN */
EZ_HD float ez_log(float x) {
    if (!(x > 0.0f)) {
        if (x == 0.0f) return -3.402823466e38f;
        return ez_u2f(0x7fc00000u);
    }
    if (ez_f2u(x) >= 0x7f800000u) return x; /* +inf */
    int e;
    x = ez_frexp_pos(x, &e);
    if (x < 0.707106781186547524f) { e -= 1; x = x + x - 1.0f; }
    else { x = x - 1.0f; }
    float z = x * x;
    float y = ((((((((7.0376836292e-2f * x - 1.1514610310e-1f) * x + 1.1676998740e-1f) * x
                    - 1.2420140846e-1f) * x + 1.4249322787e-1f) * x - 1.6668057665e-1f) * x
                 + 2.0000714765e-1f) * x - 2.4999993993e-1f) * x + 3.3333331174e-1f) * x * z;
    float fe = (float)e;
    if (e != 0) y = y + (-2.12194440e-4f) * fe;
    y = y + (-0.5f) * z;
    z = x + y;
    if (e != 0) z = z + 0.693359375f * fe;
    return z;
}
EZ_HD float ez_exp(float x) {
    if (x != x) return x;
    if (x > 88.72283905206835f) return ez_u2f(0x7f800000u);
    if (x < -103.278929903431851103f) return 0.0f;
    float z = ez_floor(1.44269504088896341f * x + 0.5f);
    x = x - z * 0.693359375f;
    x = x - z * (-2.12194440e-4f);
    int n = (int)z;
    z = x * x;
    z = (((((1.9875691500e-4f * x + 1.3981999507e-3f) * x + 8.3334519073e-3f) * x
           + 4.1665795894e-2f) * x + 1.6666665459e-1f) * x + 5.0000001201e-1f) * z + x + 1.0f;
    return ez_ldexp(z, n);
}
/* GLSL pow(x,y), x > 0:  exp(y*log(x)); pow(0,y>0) = 0; undefined (NaN) for x < 0 */
EZ_HD float ez_pow(float x, float y) {
    if (x == 0.0f) return (y > 0.0f) ? 0.0f : ((y == 0.0f) ? 1.0f : ez_u2f(0x7f800000u));
    if (x < 0.0f) return ez_u2f(0x7fc00000u);
    return ez_exp(y * ez_log(x));
}

/* ------------------------------------------------------------------ atan / asin */
#define EZ_TRUE_PI 3.14159265358979323846f
#define EZ_PIO2 1.5707963267948966192f
#define EZ_PIO4 0.7853981633974483096f

EZ_HD float ez_atan(float xx) {
    float sign = 1.0f;
    float x = xx;
    if (x < 0.0f) { sign = -1.0f; x = -x; }
    float y;
    if (x > 2.414213562373095f) { y = EZ_PIO2; x = -EZ_DIV(1.0f, x); }
    else if (x > 0.4142135623730950f) { y = EZ_PIO4; x = EZ_DIV(x - 1.0f, x + 1.0f); }
    else { y = 0.0f; }
    float z = x * x;
    y = y + ((((8.05374449538e-2f * z - 1.38776856032e-1f) * z + 1.99777106478e-1f) * z
              - 3.33329491539e-1f) * z * x + x);
    return (sign < 0.0f) ? -y : y;
}
/* GLSL atan(y,x) */
EZ_HD float ez_atan2(float y, float x) {
    if (x == 0.0f) {
        if (y > 0.0f) return EZ_PIO2;
        if (y < 0.0f) return -EZ_PIO2;
        return 0.0f;
    }
    if (y == 0.0f) return (x < 0.0f) ? EZ_TRUE_PI : 0.0f;
    float w = 0.0f;
    if (x < 0.0f) w = (y < 0.0f) ? -EZ_TRUE_PI : EZ_TRUE_PI;
    float z = ez_atan(EZ_DIV(y, x));
    return w + z;
}
/* GLSL asin(x); |x|>1 (undefined in GLSL) is treated as |x|=1 */
EZ_HD float ez_asin(float xx) {
    float sign = 1.0f;
    float a = xx;
    if (a < 0.0f) { sign = -1.0f; a = -a; }
    if (a != a) return a;
    if (a > 1.0f) a = 1.0f;
    if (a < 1.0e-4f) return xx;
    float x, z;
    int flag;
    if (a > 0.5f) { z = 0.5f * (1.0f - a); x = EZ_SQRT(z); flag = 1; }
    else { x = a; z = x * x; flag = 0; }
    z = ((((4.2163199048e-2f * z + 2.4181311049e-2f) * z + 4.5470025998e-2f) * z
          + 7.4953002686e-2f) * z + 1.6666752422e-1f) * z * x + x;
    if (flag) { z = z + z; z = EZ_PIO2 - z; }
    return (sign < 0.0f) ? -z : z;
}

/* ------------------------------------------------------------------ post pass */
/* the luminance of pass3.fsh:16 */
EZ_HD float ez_luminance(ez_vec3 c) { return 0.3f * c.x + 0.6f * c.y + 0.1f * c.z; }

/* pass3.fsh:14-25: toneMapping(c, limit) = c * 1.0 / (1.0 + lum / limit), then pow(c, vec3(1.0/2.2)) */
EZ_HD ez_vec3 ez_tonemap_pass3(ez_vec3 c, float limit) {
    float luminance = ez_luminance(c);
    float den = 1.0f + EZ_DIV(luminance, limit);
    ez_vec3 t = ez_v3(EZ_DIV(c.x * 1.0f, den), EZ_DIV(c.y * 1.0f, den), EZ_DIV(c.z * 1.0f, den));
    const float g = EZ_DIV(1.0f, 2.2f);
    return ez_v3(ez_pow(t.x, g), ez_pow(t.y, g), ez_pow(t.z, g));
}

/* ------------------------------------------------------------------ adaptive sampling (DESIGN.md section 8)
 * Per pixel after n frames (frames 0 .. n-1):  y = ez_luminance(c) of each sample colour c;  M = running mean of y*y,
 * updated in frame order as the colour is (M = ez_mix(M, y*y, 1/(frame+1)), from +0);  Y = ez_luminance of the mean colour.
 *   var = max(M - Y*Y, 0) (NaN stays NaN),   err = sqrt(var / n) / (Y + EZRT_ADAPTIVE_LUMA_FLOOR)
 * A 16x16 tile has converged when err <= threshold holds for every pixel of it inside the image (a NaN fails).
 * The floor lets black pixels with zero variance converge. */
#define EZRT_ADAPTIVE_LUMA_FLOOR 1e-3f

/* the per-sample variance of the luminance: max(M - Y*Y, 0), NaN stays NaN */
EZ_HD float ez_luma_variance(float M, float Y) {
    float var = M - Y * Y;
    return (var < 0.0f) ? 0.0f : var;
}

EZ_HD float ez_adaptive_error(float M, ez_vec3 mean, int n) {
    float Y = ez_luminance(mean);
    float var = ez_luma_variance(M, Y);
    return EZ_DIV(EZ_SQRT(EZ_DIV(var, (float)n)), Y + EZRT_ADAPTIVE_LUMA_FLOOR);
}

/* ------------------------------------------------------------------ denoiser (DESIGN.md section 9)
 * Edge-avoiding a-trous wavelet filter (Dammertz et al. 2010) with SVGF's variance-guided luminance weight (Schied et al.
 * 2017), no temporal part.  Per pixel: colour c, variance v of the mean's luminance, and the first-hit feature buffers of
 * the render (albedo a, coverage, normal n, depth z; means over the frames).  Start:  c = colour, v = ez_denoise_var0.
 * Iteration k (step s = 2^k): taps q = p + s*(i, j), j outer, i inner, both -2..2; taps outside the image are skipped.
 *   centre tap:  w = h = b3(i) * b3(j)
 *   other taps:  skipped if coverage_p == 0 or coverage_q == 0 or c_q / v_q is not finite; else w = ez_atrous_weight(...)
 *   c' = (sum w c_q) / (sum w),   v' = (sum (w*w) v_q) / ((sum w) * (sum w)),   sums in tap order, plain fp32 adds.
 * A pixel with coverage 0 (no surface in any frame) is passed through unchanged. */
#define EZRT_DENOISE_LUMA_EPS 1e-4f

EZ_HD int ez_finite(float x) { return (ez_f2u(x) & 0x7f800000u) != 0x7f800000u; }
/* the B3 spline {1/16, 1/4, 3/8, 1/4, 1/16} at i = -2..2 */
EZ_HD float ez_b3(int i) { return (i == 0) ? 0.375f : ((i == 1 || i == -1) ? 0.25f : 0.0625f); }
/* start variance: that of the mean's luminance after n frames, max(M - Y*Y, 0) / n (the term inside ez_adaptive_error) */
EZ_HD float ez_denoise_var0(float M, ez_vec3 mean, int n) { return EZ_DIV(ez_luma_variance(M, ez_luminance(mean)), (float)n); }
/* weight of tap q of pixel p: h = b3(i) b3(j), s_dist = s * max(|i|, |j|), sd_p = sqrt(v_p), Y = ez_luminance(c) */
EZ_HD float ez_atrous_weight(float h, float s_dist, ez_vec3 n_p, ez_vec3 n_q, float z_p, float z_q, float Y_p, float Y_q, float sd_p,
                             ez_vec3 a_p, ez_vec3 a_q, float sigma_l, float sigma_n, float sigma_z, float sigma_a) {
    const float d = ez_dot(n_p, n_q);
    const float w_n = (d > 0.0f) ? ez_pow(d, sigma_n) : 0.0f;
    const float w_z = ez_exp(-EZ_DIV(ez_abs(z_p - z_q), (sigma_z * z_p) * s_dist));
    const float w_l = ez_exp(-EZ_DIV(ez_abs(Y_p - Y_q), sigma_l * sd_p + EZRT_DENOISE_LUMA_EPS));
    const float da = (ez_abs(a_p.x - a_q.x) + ez_abs(a_p.y - a_q.y)) + ez_abs(a_p.z - a_q.z);
    const float w_a = ez_exp(-EZ_DIV(da, sigma_a));
    return (((h * w_n) * w_z) * w_l) * w_a;
}

/* ------------------------------------------------------------------ emissive-triangle light sampling (DESIGN.md section 10)
 * Mode EZRT_MODE_DISNEY_LIGHTS.  Light table: light k is the k-th triangle (caller's order) whose weight
 * w = ez_light_weight(p1, p2, p3, emissive) passes ez_is_light; W = sum of the weights in float64 in triangle order,
 * cdf_k = (float)(S_k / W) with the last entry exactly 1.0f, W_f = (float)W.
 * Per shading point of a bounce b < max_bounce, after mode 3's emission accounting:
 *   r_sel, r_1, r_2 = three rand01 draws (in place of mode 3's two SampleHdr draws; drawn even when there is no light), then
 *   mode 3's Sobol pair with CP rotation, xi_3 = rand01, L = SampleBRDF(...).
 *   k = the first entry with r_sel < cdf_k;  Q = ez_triangle_point(p1_k, p2_k, p3_k, r_1, r_2)
 *   D = Q - P, dist = sqrt(dot(D, D)), L_l = ez_normalize(D), cos_l = |dot(N_k, L_l)| (N_k: the light's geometric normal)
 *   pdf_l = ez_light_pdf(ez_luminance(E_k), W_f, dist, cos_l)
 *   no sample if k is the hit triangle, dot(N, L_l) <= 0, cos_l == 0 or dist == 0; else a shadow ray P -> L_l with
 *   tmax = ez_light_tmax(dist), lit iff no triangle is accepted with t < tmax (strict), and if lit
 *   Lo += history * mis(pdf_l, BRDF_Pdf(V, N, L_l)) * E_k * f_r(V, N, L_l) * dot(N, L_l) / pdf_l   (left to right)
 * A BRDF sample's emission hit at bounce >= 1 on a light T weighs mis(p.pdf, ez_light_pdf(ez_luminance(E_T), W_f, t, |dot(N_T, d)|));
 * every other emission hit weighs 1.  mis = the balance heuristic mis_mix_weight (P5/fsh:754-757). */
/* area = 0.5 * length(cross(p2 - p1, p3 - p1)) */
EZ_HD float ez_triangle_area(ez_vec3 p1, ez_vec3 p2, ez_vec3 p3) {
    const ez_vec3 c = ez_cross(ez_sub(p2, p1), ez_sub(p3, p1));
    return 0.5f * EZ_SQRT(ez_dot(c, c));
}
EZ_HD float ez_light_weight(ez_vec3 p1, ez_vec3 p2, ez_vec3 p3, ez_vec3 emissive) { return ez_triangle_area(p1, p2, p3) * ez_luminance(emissive); }
/* a light: finite weight > 0 (zero-area, black, negative and NaN emitters are not) */
EZ_HD int ez_is_light(float w) { return ez_finite(w) && w > 0.0f; }
/* uniform point of the triangle: s = sqrt(r_1), b0 = 1 - s, b1 = r_2 * s, Q = p1 b0 + p2 b1 + p3 (1 - b0 - b1) */
EZ_HD ez_vec3 ez_triangle_point(ez_vec3 p1, ez_vec3 p2, ez_vec3 p3, float r_1, float r_2) {
    const float s = EZ_SQRT(r_1);
    const float b0 = 1.0f - s, b1 = r_2 * s;
    const float b2 = (1.0f - b0) - b1;
    return ez_add(ez_add(ez_scale(p1, b0), ez_scale(p2, b1)), ez_scale(p3, b2));
}
/* solid-angle pdf of a point at distance dist seen at cosine cos_l: ((lum / W_f) * (dist * dist)) / cos_l */
EZ_HD float ez_light_pdf(float lum, float W_f, float dist, float cos_l) { return EZ_DIV(EZ_DIV(lum, W_f) * (dist * dist), cos_l); }
/* the shadow ray's bound: dist * (1 - 2^-10), so that the light's own triangle and its coplanar neighbours do not occlude */
EZ_HD float ez_light_tmax(float dist) { return dist * 0.9990234375f; }
/* index of the selected light: the first k with r < cdf[k] (cdf non-decreasing, cdf[n - 1] = 1 > r) */
EZ_HD int ez_light_select(const float* cdf, int n, float r) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (r < cdf[mid]) hi = mid;
        else lo = mid + 1;
    }
    return lo;
}

/* ------------------------------------------------------------------ the environment map as a light (DESIGN.md section 11)
 * Mode EZRT_MODE_DISNEY_LIGHTS with EZRT_PARAM_ENV_LIGHT.  The map is W x H texels, row 0 at the top (tex2d's indexing).
 * Table: w_ij = ez_env_weight(texel_ij, i, H); R_i = float64 sum of row i in column order, T = float64 sum of the R_i in row
 * order; no table if T is not finite or not > 0.  Otherwise, each cast from float64 to float:
 *   row_cdf_i = (float)((R_0 + ... + R_i) / T),  col_cdf_ij = (float)((w_i0 + ... + w_ij) / R_i) (0 where R_i = 0),
 *   texel_pdf_ij = (float)(w_ij / T);  the last entry of row_cdf and of every row of col_cdf with R_i > 0 is exactly 1.
 * Per shading point of a bounce b < max_bounce: P_env = 1/2 with K > 0 triangle lights, 1 with none (0 without a table:
 * then the render is mode 4's).  The draws are mode 4's: r_sel, r_1, r_2, the Sobol pair, xi_3.  The environment is
 * sampled if P_env == 1 or r_sel < 0.5:
 *   L_e = ez_env_sample(r_1, r_2), pdf_e = P_env * ez_env_pdf(L_e); no sample if pdf_e is not finite or <= 0, or
 *   dot(N, L_e) <= 0; else a shadow ray bounded at EZ_INF (mode 3's), and if lit
 *   Lo += history * mis(pdf_e, BRDF_Pdf(V, N, L_e)) * hdrColor(L_e) * f_r(V, N, L_e) * dot(N, L_e) / pdf_e   (left to right)
 * otherwise mode 4's triangle sample with the selection number (r_sel - 0.5) * 2 and pdf_l * (1 - P_env).
 * A BRDF sample that leaves the scene at bounce >= 1 weighs mis(p.pdf, P_env * ez_env_pdf(d)) (mode 3's order); one that hits
 * a light T weighs mis(p.pdf, (1 - P_env) * ez_light_pdf(...)); a camera ray that leaves the scene weighs 1. */
/* toSphericalCoord (P5/fsh:684-690): the device's to_spherical and the oracle's toSphericalCoord are this sequence of operations */
EZ_HD void ez_to_spherical(ez_vec3 v, float* ou, float* ov) {
    float u = ez_atan2(v.z, v.x), w = ez_asin(v.y);
    u = EZ_DIV(u, 2.0f * EZ_PI);
    w = EZ_DIV(w, EZ_PI);
    u += 0.5f;
    w += 0.5f;
    *ou = u;
    *ov = 1.0f - w;
}
/* weight of texel (i, j) in row i of H: luminance times the cosine of the row centre's elevation (solid angle), 0 unless
 * finite and > 0 */
EZ_HD float ez_env_weight(ez_vec3 texel, int i, int H) {
    const float e = EZ_PI * (0.5f - EZ_DIV((float)i + 0.5f, (float)H));
    const float w = ez_luminance(texel) * ez_cos(e);
    return (ez_finite(w) && w > 0.0f) ? w : 0.0f;
}
/* the first k with r < cdf[k] (ez_light_select) and the offset of r inside entry k, clamped below 1 */
EZ_HD int ez_env_select(const float* cdf, int n, float r, float* offset) {
    const int k = ez_light_select(cdf, n, r);
    const float lo = (k > 0) ? cdf[k - 1] : 0.0f;
    const float a = EZ_DIV(r - lo, cdf[k] - lo);
    *offset = ez_min(a, 0.99999994f);
    return k;
}
/* the direction of the sample (r_1, r_2); *texel = i * W + j, the texel it was drawn from */
EZ_HD ez_vec3 ez_env_sample(const float* row_cdf, const float* col_cdf, int W, int H, float r_1, float r_2, int* texel) {
    float a, b;
    const int i = ez_env_select(row_cdf, H, r_1, &a);
    const int j = ez_env_select(col_cdf + (size_t)i * W, W, r_2, &b);
    *texel = i * W + j;
    const float u = EZ_DIV((float)j + b, (float)W), v = EZ_DIV((float)i + a, (float)H);
    const float phi = 2.0f * EZ_PI * (u - 0.5f);
    const float e = EZ_PI * (0.5f - v);
    const float ce = ez_cos(e);
    return ez_v3(ce * ez_cos(phi), ez_sin(e), ce * ez_sin(phi));
}
/* the texel tex2d's nearest lookup reads at (u, v) */
EZ_HD int ez_env_texel(float u, float v, int W, int H) {
    return ez_texel_clamp(ez_floor(v * (float)H), H) * W + ez_texel_clamp(ez_floor(u * (float)W), W);
}
/* solid-angle density of ez_env_sample at direction L: texel_pdf * W * H / (2 pi^2 cos e), 0 if the texel's pdf or cos e is 0 */
EZ_HD float ez_env_pdf(const float* texel_pdf, int W, int H, ez_vec3 L) {
    const ez_vec3 n = ez_normalize(L);
    float u, v;
    ez_to_spherical(n, &u, &v);
    const float p = texel_pdf[ez_env_texel(u, v, W, H)];
    const float ce = EZ_SQRT(n.x * n.x + n.z * n.z);
    if (p == 0.0f || ce == 0.0f) return 0.0f;
    return EZ_DIV(p * (float)(W * H), (2.0f * EZ_PI * EZ_PI) * ce);
}

/* ------------------------------------------------------------------ transmission (DESIGN.md section 12)
 * Mode EZRT_MODE_DISNEY_LIGHTS with EZRT_PARAM_TRANSMISSION: a rough dielectric lobe (Walter et al. 2007) beside the reference
 * BRDF.  At a hit: V = -d, N = the shading normal as the hit returns it (flipped towards V by the geometric test), inside = that
 * test (dot(Ng, d) > 0: the ray leaves the medium).  The outside is vacuum; eta = eta_L / eta_V = IOR entering, 1 / IOR leaving.
 *   t = ez_trans_weight(transmission, metallic, IOR).  t == 0: the hit is mode 4's, draws, arithmetic and bits.
 *   BSDF  f = (1 - t) f_ref + t f_diel,  pdf = (1 - t) pdf_ref + t pdf_diel  (ez_trans_mix), f_ref / pdf_ref = the reference's
 *         BRDF_Evaluate / BRDF_Pdf where dot(N, L) > 0 and 0 elsewhere; f_diel / pdf_diel = ez_diel_eval.
 *   alpha = max(0.001, roughness^2); D = the reference's GTR2; G = Smith GGX G1(V) G1(L); F = exact unpolarised Fresnel (TIR: 1).
 *   reflection (dot(N, L) > 0): h = normalize(V + L),
 *         f_diel = F D G / (4 |N.V| |N.L|) (untinted),  pdf_diel = F D (N.h) / (4 V.h)
 *   refraction (dot(N, L) < 0): h = normalize(-(V + eta L)) turned to the N side, den = V.h + eta L.h,
 *         f_diel = baseColor (1 - F) D G (V.h) |L.h| / (|N.V| |N.L| den^2),  pdf_diel = (1 - F) D (N.h) eta^2 |L.h| / den^2
 *     This is the radiance convention: f(V, L) / eta_V^2 = f(L, V) / eta_L^2, and a smooth refraction carries (1 - F) / eta^2.
 *   f_diel = pdf_diel = 0 unless dot(N, V) > 0, N.h > 0, V.h > 0 and L.h on L's side, or where a value is not finite.
 *   Index-matched (|IOR - 1| <= 2^-8): f_diel is a pass-through, F = 0, L = -V, weight baseColor; it adds nothing to f and pdf
 *   at any other direction.
 * Sampling, after mode 4's draws (r_sel, r_1, r_2, the Sobol pair, xi_3): r_t = rand01.
 *   r_t < t: index-matched: L = d, the path carries (f, pdf, |cos|) = (baseColor, 1, 1); else L = ez_diel_sample(xi, xi_3).
 *   otherwise: L = SampleBRDF as mode 4, the path ends unless dot(N, L) > 0.
 *   The path then carries f and pdf of the mixture at L and |dot(N, L)|.  A failed dielectric sample ends the path.
 * Light samples are evaluated with the mixture at L (dot(N, L) > 0) and MIS-weighted with its pdf.  A BSDF sample with
 * dot(N, L) < 0 (a refraction or a pass-through) cannot be drawn by a light sample: the emission it hits, or the environment it
 * leaves to, weighs 1.  The path record keeps this bit as the sign of its cosine. */
#define EZ_TRANS_MATCHED 0.00390625f   /* 2^-8 */
/* the weight of the dielectric lobe: clamp(transmission, 0, 1) * (1 - metallic), clamped to [0, 1]; 0 if transmission or the
 * product is not finite, or IOR is not finite or <= 0 (opaque) */
EZ_HD float ez_trans_weight(float transmission, float metallic, float IOR) {
    if (!ez_finite(transmission) || !ez_finite(IOR) || !(IOR > 0.0f)) return 0.0f;
    const float t = ez_clamp(transmission, 0.0f, 1.0f) * (1.0f - metallic);
    return (ez_finite(t) && t > 0.0f) ? ez_min(t, 1.0f) : 0.0f;
}
/* eta = eta_L / eta_V of a refraction from V's side: IOR entering, 1 / IOR leaving (inside) */
EZ_HD float ez_trans_eta(float IOR, int inside) { return inside ? EZ_DIV(1.0f, IOR) : IOR; }
EZ_HD int ez_trans_matched(float IOR) { return ez_abs(IOR - 1.0f) <= EZ_TRANS_MATCHED; }
/* the exact unpolarised Fresnel reflectance at cos_i = |V.h| for the relative index eta; total internal reflection gives 1 */
EZ_HD float ez_fresnel_dielectric(float cos_i, float eta) {
    const float c = ez_min(ez_abs(cos_i), 1.0f);
    const float s2 = EZ_DIV(1.0f - c * c, eta * eta);
    if (!(s2 < 1.0f)) return 1.0f;
    const float ct = EZ_SQRT(1.0f - s2);
    const float rs = EZ_DIV(c - eta * ct, c + eta * ct);
    const float rp = EZ_DIV(eta * c - ct, eta * c + ct);
    return 0.5f * (rs * rs + rp * rp);
}
/* the reference's GTR2 (GGX D) */
EZ_HD float ez_ggx_D(float NdotH, float a) {
    const float a2 = a * a;
    const float t = 1.0f + (a2 - 1.0f) * NdotH * NdotH;
    return EZ_DIV(a2, EZ_PI * t * t);
}
/* Smith GGX masking of one direction at cosine c > 0: 2 c / (c + sqrt(a^2 + c^2 - a^2 c^2)) */
EZ_HD float ez_ggx_G1(float c, float a) {
    const float a2 = a * a, c2 = c * c;
    return EZ_DIV(2.0f * c, c + EZ_SQRT(a2 + c2 - a2 * c2));
}
/* the reference's toNormalHemisphere */
EZ_HD ez_vec3 ez_to_normal_hemisphere(ez_vec3 v, ez_vec3 N) {
    ez_vec3 helper = ez_v3(1.0f, 0.0f, 0.0f);
    if (ez_abs(N.x) > 0.999f) helper = ez_v3(0.0f, 0.0f, 1.0f);
    const ez_vec3 tangent = ez_normalize(ez_cross(N, helper));
    const ez_vec3 bitangent = ez_normalize(ez_cross(N, tangent));
    return ez_add(ez_add(ez_scale(tangent, v.x), ez_scale(bitangent, v.y)), ez_scale(N, v.z));
}
/* the reference's GTR2 half-vector law (SampleGTR2 before its reflection): density D(h) (N.h) */
EZ_HD ez_vec3 ez_ggx_half(float xi_1, float xi_2, ez_vec3 N, float a) {
    const float phi_h = 2.0f * EZ_PI * xi_1;
    const float sin_phi_h = ez_sin(phi_h), cos_phi_h = ez_cos(phi_h);
    const float cos_theta_h = EZ_SQRT(EZ_DIV(1.0f - xi_2, 1.0f + (a * a - 1.0f) * xi_2));
    const float sin_theta_h = EZ_SQRT(ez_max(0.0f, 1.0f - cos_theta_h * cos_theta_h));
    return ez_to_normal_hemisphere(ez_v3(sin_theta_h * cos_phi_h, sin_theta_h * sin_phi_h, cos_theta_h), N);
}
/* f_diel(V, L) of unit vectors (rough lobe; not for the index-matched case) and its density *pdf */
EZ_HD ez_vec3 ez_diel_eval(ez_vec3 V, ez_vec3 N, ez_vec3 L, ez_vec3 baseColor, float a, float eta, float* pdf) {
    const ez_vec3 zero = ez_v3(0.0f, 0.0f, 0.0f);
    *pdf = 0.0f;
    const float NdotV = ez_dot(N, V), NdotL = ez_dot(N, L);
    if (!(NdotV > 0.0f) || !(NdotL != 0.0f) || !ez_finite(NdotL)) return zero;
    const int refr = NdotL < 0.0f;
    ez_vec3 H = ez_normalize(refr ? ez_neg(ez_add(V, ez_scale(L, eta))) : ez_add(V, L));
    float NdotH = ez_dot(N, H);
    if (NdotH < 0.0f) { H = ez_neg(H); NdotH = -NdotH; }
    const float VdotH = ez_dot(V, H), LdotH = ez_dot(L, H);
    if (!(NdotH > 0.0f) || !(VdotH > 0.0f) || (refr ? !(LdotH < 0.0f) : !(LdotH > 0.0f))) return zero;
    const float F = ez_fresnel_dielectric(VdotH, eta);
    const float D = ez_ggx_D(NdotH, a);
    const float G = ez_ggx_G1(NdotV, a) * ez_ggx_G1(ez_abs(NdotL), a);
    float f, p;
    if (!refr) {
        f = EZ_DIV(F * D * G, 4.0f * NdotV * NdotL);
        p = EZ_DIV(F * D * NdotH, 4.0f * VdotH);
    } else {
        const float T = 1.0f - F, aL = ez_abs(LdotH);
        const float den = VdotH + eta * LdotH;
        const float den2 = den * den;
        if (!(T > 0.0f) || !(den2 > 0.0f)) return zero;
        f = EZ_DIV(T * D * G * VdotH * aL, NdotV * ez_abs(NdotL) * den2);
        p = EZ_DIV(T * D * NdotH * (eta * eta) * aL, den2);
    }
    if (!ez_finite(f) || !ez_finite(p) || !(p > 0.0f)) return zero;
    *pdf = p;
    return refr ? ez_scale(baseColor, f) : ez_v3(f, f, f);
}
/* the dielectric lobe's sample: h by ez_ggx_half(xi_1, xi_2), reflect if xi_3 < F(V.h), refract otherwise.  Returns 1 with *L,
 * or 0 (the path ends) if dot(N, V) <= 0, V.h <= 0, or L lands on the wrong side of N for its lobe */
EZ_HD int ez_diel_sample(float xi_1, float xi_2, float xi_3, ez_vec3 V, ez_vec3 N, float a, float eta, ez_vec3* L) {
    if (!(ez_dot(N, V) > 0.0f)) return 0;
    const ez_vec3 H = ez_ggx_half(xi_1, xi_2, N, a);
    const float VdotH = ez_dot(V, H);
    if (!(VdotH > 0.0f)) return 0;
    const float F = ez_fresnel_dielectric(VdotH, eta);
    if (xi_3 < F) {
        *L = ez_reflect(ez_neg(V), H);
        return ez_dot(N, *L) > 0.0f;
    }
    /* F < 1: no total internal reflection, s2 < 1 as in ez_fresnel_dielectric */
    const float c = ez_min(VdotH, 1.0f);
    const float s2 = EZ_DIV(1.0f - c * c, eta * eta);
    const float ct = EZ_SQRT(1.0f - s2);
    const float ie = EZ_DIV(1.0f, eta);
    *L = ez_normalize(ez_add(ez_scale(V, -ie), ez_scale(H, ie * c - ct)));
    return ez_dot(N, *L) < 0.0f;
}
/* the mixture: f = (1 - t) f_ref + t f_diel, *pdf = (1 - t) pdf_ref + t pdf_diel */
EZ_HD ez_vec3 ez_trans_mix(ez_vec3 f_ref, float pdf_ref, ez_vec3 f_diel, float pdf_diel, float t, float* pdf) {
    const float s = 1.0f - t;
    *pdf = s * pdf_ref + t * pdf_diel;
    return ez_add(ez_scale(f_ref, s), ez_scale(f_diel, t));
}

/* ------------------------------------------------------------------ thin-lens camera (DESIGN.md section 13)
 * EZRT_PARAM_THIN_LENS, any mode: lens radius R = reserved[1], focus distance f = reserved[2] (IEEE-754 bits of floats).
 * M = camera_rotate (column-major), c_i = column i, eye = params.eye.  Per sample (px, py, frame):
 *   the pinhole's seed, jitter draws, vx, vy and dir_pin = M (vx, vy, -1.5, 0), bit for bit (primary_ray, P5/fsh:915-925);
 *   F = eye + dir_pin * k,  k = f / (1.5 |c2|)        the point at depth f along -c2 (ez_lens_setup: k, u0, u1)
 *   (lx, ly) = ez_concentric_disk(r_a, r_b),  (r_a, r_b) = ez_lens_draws(px, py, frame)
 *   o = eye + (lx u0 + ly u1) R,  u0 = c0 / |c0|, u1 = c1 / |c1|;   d = normalize(F - o)
 * |c| = sqrt(dot(c, c)).  The lens draws come from a stream of their own, so every draw of the path after the jitter is the
 * pinhole render's.  The flag is valid iff R and f are finite and > 0, |c0|, |c1|, |c2| are finite and > 0, and k is finite. */
#define EZRT_LENS_SALT 0x4c454e53u   /* "LENS" */
/* wang_hash / rand (P5/fsh:320-331) */
EZ_HD uint32_t ez_wang_hash(uint32_t* seed) {
    uint32_t s = *seed;
    s = (s ^ 61u) ^ (s >> 16);
    s *= 9u;
    s = s ^ (s >> 4);
    s *= 0x27d4eb2du;
    s = s ^ (s >> 15);
    *seed = s;
    return s;
}
EZ_HD float ez_rand01(uint32_t* seed) { return ez_u32_to_float(ez_wang_hash(seed)) * 2.3283064365386963e-10f; }
/* the lens stream: two rand draws from the pixel seed (P5/fsh:315-318) XOR EZRT_LENS_SALT; a function of (px, py, frame) only */
EZ_HD void ez_lens_draws(uint32_t px, uint32_t py, uint32_t frame, float* r_a, float* r_b) {
    uint32_t s = ((px * 1973u + py * 9277u + frame * 26699u) | 1u) ^ EZRT_LENS_SALT;
    *r_a = ez_rand01(&s);
    *r_b = ez_rand01(&s);
}
/* Shirley-Chiu concentric map of [0, 1]^2 onto the unit disk (uniform in area) */
EZ_HD void ez_concentric_disk(float u1, float u2, float* x, float* y) {
    const float a = 2.0f * u1 - 1.0f, b = 2.0f * u2 - 1.0f;
    if (a == 0.0f && b == 0.0f) { *x = 0.0f; *y = 0.0f; return; }
    float r, phi;
    if (ez_abs(a) > ez_abs(b)) { r = a; phi = EZ_PIO4 * EZ_DIV(b, a); }
    else { r = b; phi = EZ_PIO2 - EZ_PIO4 * EZ_DIV(a, b); }
    *x = r * ez_cos(phi);
    *y = r * ez_sin(phi);
}
struct ez_lens {
    ez_vec3 eye, u0, u1;   /* the lens centre and its unit axes */
    float k, R;            /* focus scale f / (1.5 |c2|), lens radius */
};
typedef struct ez_lens ez_lens;
/* the lens of (eye, camera_rotate, R, f); returns 0 (and leaves *L unset) if the flag's parameters are invalid */
EZ_HD int ez_lens_setup(const float eye[3], const float cam[16], float R, float f, ez_lens* L) {
    const ez_vec3 c0 = ez_v3(cam[0], cam[1], cam[2]), c1 = ez_v3(cam[4], cam[5], cam[6]), c2 = ez_v3(cam[8], cam[9], cam[10]);
    const float n0 = EZ_SQRT(ez_dot(c0, c0)), n1 = EZ_SQRT(ez_dot(c1, c1)), n2 = EZ_SQRT(ez_dot(c2, c2));
    if (!(ez_finite(R) && R > 0.0f && ez_finite(f) && f > 0.0f)) return 0;
    if (!(ez_finite(n0) && n0 > 0.0f && ez_finite(n1) && n1 > 0.0f && ez_finite(n2) && n2 > 0.0f)) return 0;
    const float k = EZ_DIV(f, 1.5f * n2);
    if (!ez_finite(k)) return 0;
    L->eye = ez_v3(eye[0], eye[1], eye[2]);
    L->u0 = ez_divs(c0, n0);
    L->u1 = ez_divs(c1, n1);
    L->k = k;
    L->R = R;
    return 1;
}
/* the lens ray through the pinhole direction dir_pin with the lens draws (r_a, r_b) */
EZ_HD void ez_lens_ray(const ez_lens* L, ez_vec3 dir_pin, float r_a, float r_b, ez_vec3* o, ez_vec3* d) {
    const ez_vec3 F = ez_add(L->eye, ez_scale(dir_pin, L->k));
    float lx, ly;
    ez_concentric_disk(r_a, r_b, &lx, &ly);
    *o = ez_add(L->eye, ez_scale(ez_add(ez_scale(L->u0, lx), ez_scale(L->u1, ly)), L->R));
    *d = ez_normalize(ez_sub(F, *o));
}

/* ------------------------------------------------------------------ homogeneous medium (DESIGN.md section 14)
 * Mode EZRT_MODE_DISNEY_LIGHTS with EZRT_PARAM_MEDIUM: grey extinction sigma_t, albedo, Henyey-Greenstein g, box [bmin, bmax].
 * Free flight, on every traced segment (origin o, direction d, hit distance t_hit, or a miss) of a path, camera rays included:
 *   t_end = t_hit, or +inf for a miss.  At the start of the shading step (at bounce >= 1 after the check of the previous sample's
 *   pdf), ez_medium_flight: if sigma_t > 0 and ez_box_overlap(o, d, bmin, bmax, t_end) = [t0, t1] with t0 < t1, one draw
 *   r_m = rand01 and t_s = t0 + ez_free_flight(r_m, sigma_t); the path scatters iff t_s < t1.  A segment without overlap draws
 *   nothing.  A path that does not scatter reaches its hit, or leaves the scene, exactly as in mode 4.
 * Medium vertex (the path scatters) at bounce b, P = o + d t_s:
 *   b == 0: Lo = 0, no emission; a camera ray that missed is a primary miss (its colour is Lo), one that hit keeps its first-hit
 *   features.  b >= 1: history *= f_r cos / pdf as at a surface.  Then history *= albedo; b >= max_bounce: the path ends.
 *   Draws: r_sel, r_1, r_2, then h_1, h_2 (rand01 each).  The light sample is the surface's (sections 10, 11: the map with P_env,
 *   else the triangles) at P with neither the hemisphere test nor the self exclusion: a triangle sample needs cos_l != 0 and
 *   dist != 0, a map sample a finite pdf_e > 0.  If its shadow ray is lit (p = ez_hg_pdf(d, L_l, g)):
 *     Lo += ((history * mis(pdf_l, p) * E * splat(p)) * 1 / pdf_l) * T   (left to right; T = ez_medium_transmittance)
 *   L = ez_hg_sample(d, g, h_1, h_2); the path record is (f_r, pdf, cos) = (splat(p), p, 1) with p = ez_hg_pdf(d, L, g), so that the
 *   emission and environment it reaches are MIS-weighted by mode 4's code unchanged.
 * Every lit light sample (surface or medium vertex) is multiplied by T = ez_medium_transmittance(o, L_l, ez_medium_light_dist(tmax,
 * map)) of its shadow ray after its mode-4 value: the contribution times T, with T = 1 when the ray does not overlap the box.
 * Limit: rays from a medium vertex are traced like every other ray, so a triangle closer than the traversal's minimum hit distance
 * (0.0005, the reference's hitTriangle) is not seen by them.  A vertex within 0.0005 of a surface can send its phase sample or its
 * shadow ray through that surface: with a mean free path near or below 0.0005 (sigma_t >~ 2000) light leaks into and past opaque
 * objects.  The definition is what the kernels compute either way; it is the physics that degrades there. */
struct ez_medium {
    float sigma_t;
    ez_vec3 albedo;
    float g;
    ez_vec3 bmin, bmax;
};
typedef struct ez_medium ez_medium;
/* the overlap [*t0, *t1] of the segment o + t d, 0 <= t <= t_end, with the box; 1 iff it has positive length (t0 < t1) and the box
 * has positive extent on every axis.  Per axis a: d_a == 0: no overlap if o_a < bmin_a or o_a > bmax_a, else no bound; otherwise
 * ta = (bmin_a - o_a) / d_a, tb = (bmax_a - o_a) / d_a, t0 = max(t0, min(ta, tb)), t1 = min(t1, max(ta, tb)) (from 0, t_end) */
EZ_HD int ez_box_overlap(ez_vec3 o, ez_vec3 d, ez_vec3 bmin, ez_vec3 bmax, float t_end, float* t0, float* t1) {
    const float oo[3] = {o.x, o.y, o.z}, dd[3] = {d.x, d.y, d.z};
    const float lo[3] = {bmin.x, bmin.y, bmin.z}, hi[3] = {bmax.x, bmax.y, bmax.z};
    float a = 0.0f, b = t_end;
    for (int k = 0; k < 3; k++) {
        if (!(lo[k] < hi[k])) return 0;
        if (dd[k] == 0.0f) {
            if (oo[k] < lo[k] || oo[k] > hi[k]) return 0;
            continue;
        }
        const float ta = EZ_DIV(lo[k] - oo[k], dd[k]), tb = EZ_DIV(hi[k] - oo[k], dd[k]);
        a = ez_max(a, ez_min(ta, tb));
        b = ez_min(b, ez_max(ta, tb));
    }
    *t0 = a;
    *t1 = b;
    return a < b;
}
/* the free-flight distance of the draw r: -log(1 - r) / sigma_t */
EZ_HD float ez_free_flight(float r, float sigma_t) { return EZ_DIV(-ez_log(1.0f - r), sigma_t); }
/* the free flight of a segment (t_end: the hit distance, +inf for a miss): 1 with *t_s if the path scatters.  Draws r_m from *seed
 * only when the segment overlaps the medium. */
EZ_HD int ez_medium_flight(const ez_medium* m, ez_vec3 o, ez_vec3 d, float t_end, uint32_t* seed, float* t_s) {
    float t0, t1;
    if (!(m->sigma_t > 0.0f) || !ez_box_overlap(o, d, m->bmin, m->bmax, t_end, &t0, &t1)) return 0;
    const float t = t0 + ez_free_flight(ez_rand01(seed), m->sigma_t);
    *t_s = t;
    return t < t1;
}
/* the transmittance of the shadow ray o + t d, 0 <= t <= L: exp(-sigma_t |[0, L] & box|), exactly 1 without overlap */
EZ_HD float ez_medium_transmittance(const ez_medium* m, ez_vec3 o, ez_vec3 d, float L) {
    float t0, t1;
    if (!(m->sigma_t > 0.0f) || !ez_box_overlap(o, d, m->bmin, m->bmax, L, &t0, &t1)) return 1.0f;
    return ez_exp(-(m->sigma_t * (t1 - t0)));
}
/* L of a light sample's shadow ray: the light's distance recovered from the bound tmax = ez_light_tmax(dist), or +inf for the map
 * (the box exit) */
EZ_HD float ez_medium_light_dist(float tmax, int map) { return map ? ez_u2f(0x7f800000u) : EZ_DIV(tmax, 0.9990234375f); }
/* Henyey-Greenstein density (per steradian) of the direction L after propagation along d (unit vectors; cos = their angle's cosine):
 * (1 - g^2) / (4 pi den^1.5), den = 1 + g^2 - 2 g cos, evaluated without cancellation as (1 - g)^2 + g |d - L|^2 for g >= 0 and
 * (1 + g)^2 - g |d + L|^2 for g < 0 (|d -+ L|^2 = 2 (1 -+ cos)) */
EZ_HD float ez_hg_pdf(ez_vec3 d, ez_vec3 L, float g) {
    float den;
    if (g >= 0.0f) {
        const ez_vec3 v = ez_sub(d, L);
        den = (1.0f - g) * (1.0f - g) + g * ez_dot(v, v);
    } else {
        const ez_vec3 v = ez_add(d, L);
        den = (1.0f + g) * (1.0f + g) - g * ez_dot(v, v);
    }
    return EZ_DIV((1.0f - g) * (1.0f + g), (4.0f * EZ_PI) * (den * EZ_SQRT(den)));
}
/* the exact inversion of the Henyey-Greenstein law of cos (h_1 = its cdf) and phi = 2 pi h_2, in the frame of d
 * (ez_to_normal_hemisphere).  With a = 1 - g + 2 g h_1 (> 0):  1 - cos = 2 (1 - g)^2 (1 - h_1) (1 + g h_1) / a^2,
 * 1 + cos = 2 (1 + g)^2 h_1 (1 - g + g h_1) / a^2;  cos from the smaller of the two, sin = sqrt((1 - cos)(1 + cos)) */
EZ_HD ez_vec3 ez_hg_sample(ez_vec3 d, float g, float h_1, float h_2) {
    const float a = (1.0f - g) + (2.0f * g) * h_1;
    const float a2 = a * a;
    const float qm = EZ_DIV((2.0f * ((1.0f - g) * (1.0f - g))) * ((1.0f - h_1) * (1.0f + g * h_1)), a2);
    const float qp = EZ_DIV((2.0f * ((1.0f + g) * (1.0f + g))) * (h_1 * ((1.0f - g) + g * h_1)), a2);
    const float c = (qm < qp) ? 1.0f - qm : qp - 1.0f;
    const float s = EZ_SQRT(qm * qp);
    const float phi = 2.0f * EZ_PI * h_2;
    return ez_to_normal_hemisphere(ez_v3(s * ez_cos(phi), s * ez_sin(phi), c), d);
}

/* ------------------------------------------------------------------ base-colour textures (EZRT_PARAM_TEXTURES, DESIGN.md section 15)
 * A textured triangle carries three UVs and a texture index; the base colour of a hit on it is mat.baseColor * the texture's filtered
 * linear colour at the hit's UV, per channel.  Texture index -1: the material's base colour.  No random number is drawn.
 * Barycentrics (ez_tri_bary): drop the axis k of the largest |Ng_k| (the first on ties), 2D edge functions on the axes (k+1, k+2) mod 3:
 *   w1 = e(p2, p3, P) / A, w2 = e(p3, p1, P) / A, w3 = (1 - w1) - w2 with A = e(p1, p2, p3); A == 0 or not finite: 1/3 each.
 *   (surface_hit's weights are the reference's xy-projected ones, which collapse on triangles of degenerate xy projection.)
 *   uv = (w1 uv1 + w2 uv2) + w3 uv3.
 * Filter (ez_tex_sample): wrap in both axes, s = u - floor(u), t = v - floor(v); x = s W - 0.5, y = (1 - t) H - 0.5 (texel row 0 is
 *   the image's top row, OBJ's v = 0 its bottom); x0 = floor(x), weight x - x0, x0 and x0 + 1 reduced modulo W (s may round to
 *   1.0); the same for y.  Texels are RGBA8 (alpha ignored), each channel decoded by ez_srgb_table (the sRGB EOTF in float64, rounded
 *   to fp32), then filtered bilinearly with lerp(a, b, f) = a + (b - a) f, so that four equal texels give that texel exactly.  A
 *   non-finite u or v gives exactly (1, 1, 1); every finite |u| >= 2^23 is whole, so s = 0 there and the texel indices stay in range. */
static const float ez_srgb_table[256] = {
#include "ezrt_srgb_table.inc"
};
EZ_HD float ez_tex_axis(const ez_vec3 v, int a) { return a == 0 ? v.x : (a == 1 ? v.y : v.z); }
/* the 2D edge function of (p, q) at r on the axes (a, b) */
EZ_HD float ez_tex_edge(ez_vec3 p, ez_vec3 q, ez_vec3 r, int a, int b) {
    return (ez_tex_axis(q, a) - ez_tex_axis(p, a)) * (ez_tex_axis(r, b) - ez_tex_axis(p, b)) -
           (ez_tex_axis(q, b) - ez_tex_axis(p, b)) * (ez_tex_axis(r, a) - ez_tex_axis(p, a));
}
EZ_HD void ez_tri_bary(ez_vec3 P, ez_vec3 p1, ez_vec3 p2, ez_vec3 p3, ez_vec3 Ng, float* w1, float* w2, float* w3) {
    int k = 0;
    float m = ez_abs(Ng.x);
    if (ez_abs(Ng.y) > m) { k = 1; m = ez_abs(Ng.y); }
    if (ez_abs(Ng.z) > m) k = 2;
    const int a = (k + 1) % 3, b = (k + 2) % 3;
    const float A = ez_tex_edge(p1, p2, p3, a, b);
    if (A == 0.0f || !ez_finite(A)) {
        *w1 = *w2 = *w3 = 1.0f / 3.0f;
        return;
    }
    *w1 = EZ_DIV(ez_tex_edge(p2, p3, P, a, b), A);
    *w2 = EZ_DIV(ez_tex_edge(p3, p1, P, a, b), A);
    *w3 = (1.0f - *w1) - *w2;
}
EZ_HD float ez_tex_lerp(float a, float b, float f) { return a + (b - a) * f; }
/* i in [-1, n] reduced modulo n */
EZ_HD int ez_tex_wrap(int i, int n) { return i < 0 ? i + n : (i >= n ? i - n : i); }
EZ_HD ez_vec3 ez_tex_texel(const uint32_t* texels, int idx, const float* lut) {
#if defined(__CUDA_ARCH__)
    const uint32_t c = __ldg(texels + idx);
    return ez_v3(__ldg(lut + (c & 255u)), __ldg(lut + ((c >> 8) & 255u)), __ldg(lut + ((c >> 16) & 255u)));
#else
    const uint32_t c = texels[idx];
    return ez_v3(lut[c & 255u], lut[(c >> 8) & 255u], lut[(c >> 16) & 255u]);
#endif
}
/* the filtered linear colour of the W x H texture `texels` (RGBA8 as little-endian words, row 0 on top) at (u, v); lut = ez_srgb_table */
EZ_HD ez_vec3 ez_tex_sample(const uint32_t* texels, int W, int H, float u, float v, const float* lut) {
    if (!ez_finite(u) || !ez_finite(v)) return ez_v3(1.0f, 1.0f, 1.0f);
    const float s = u - ez_floor(u), t = v - ez_floor(v);
    const float x = s * (float)W - 0.5f, y = (1.0f - t) * (float)H - 0.5f;
    const float fx0 = ez_floor(x), fy0 = ez_floor(y);
    const float ax = x - fx0, ay = y - fy0;
    const int x0 = ez_tex_wrap((int)fx0, W), x1 = ez_tex_wrap((int)fx0 + 1, W);
    const int y0 = ez_tex_wrap((int)fy0, H), y1 = ez_tex_wrap((int)fy0 + 1, H);
    const ez_vec3 t00 = ez_tex_texel(texels, y0 * W + x0, lut), t10 = ez_tex_texel(texels, y0 * W + x1, lut);
    const ez_vec3 t01 = ez_tex_texel(texels, y1 * W + x0, lut), t11 = ez_tex_texel(texels, y1 * W + x1, lut);
    const ez_vec3 top = ez_v3(ez_tex_lerp(t00.x, t10.x, ax), ez_tex_lerp(t00.y, t10.y, ax), ez_tex_lerp(t00.z, t10.z, ax));
    const ez_vec3 bot = ez_v3(ez_tex_lerp(t01.x, t11.x, ax), ez_tex_lerp(t01.y, t11.y, ax), ez_tex_lerp(t01.z, t11.z, ax));
    return ez_v3(ez_tex_lerp(top.x, bot.x, ay), ez_tex_lerp(top.y, bot.y, ay), ez_tex_lerp(top.z, bot.z, ay));
}
/* the interpolated UV of barycentrics (w1, w2, w3) over the triangle's (u1, v1, u2, v2) (u3, v3) */
EZ_HD void ez_tex_uv(float w1, float w2, float w3, const float* uv6, float* u, float* v) {
    *u = (w1 * uv6[0] + w2 * uv6[2]) + w3 * uv6[4];
    *v = (w1 * uv6[1] + w2 * uv6[3]) + w3 * uv6[5];
}

/* ------------------------------------------------------------------ material maps (EZRT_PARAM_MATERIAL_MAPS, DESIGN.md section 16)
 * Two more per-triangle texture ids into the textures of EZRT_PARAM_TEXTURES, looked up at the same UV as the base colour with
 * ez_tex_sample(..., ez_unorm8_table): the maps are linear data (c / 255 in float64, rounded to fp32), not sRGB.  Id -1: no map.
 * Metallic-roughness map (glTF's channels): roughness = mat.roughness * G, metallic = mat.metallic * B (ez_mr_apply).
 * Normal map (tangent space, OpenGL +Y), ez_normal_map; N is surface_hit's shading normal, No = N, negated for a hit from inside:
 *   e1 = p2 - p1, e2 = p3 - p1, (du1, dv1) = uv2 - uv1, (du2, dv2) = uv3 - uv1, det = du1 dv2 - du2 dv1;
 *   T = (dv2 e1 - dv1 e2) / det, B_uv = (du1 e2 - du2 e1) / det (each component: (a x - b y) / det);
 *   T' = normalize(T - dot(No, T) No), B = cross(No, T'), negated when dot(B, B_uv) < 0;
 *   n_t = 2 f - 1 per channel of the filtered colour f; n = normalize((n_t.x T' + n_t.y B) + n_t.z No), negated for a hit from inside.
 *   N itself, bit for bit, when u or v is not finite, det is 0 or not finite, dot(T - dot(No, T) No, itself) is 0 or not finite,
 *   dot(B, B_uv) is 0 or not finite, n is not finite, or dot(n, V) <= 0 (the view stays on the shading side) -- in that order.
 * The tangent is per triangle (not MikkTSpace): maps baked against smooth per-vertex tangents show faint seams between facets. */
static const float ez_unorm8_table[256] = {
#include "ezrt_unorm8_table.inc"
};
/* the metallic-roughness map's filtered colour f applied to a material's roughness and metallic */
EZ_HD void ez_mr_apply(ez_vec3 f, float* roughness, float* metallic) {
    *roughness = *roughness * f.y;
    *metallic = *metallic * f.z;
}
EZ_HD int ez_finite3(ez_vec3 v) { return ez_finite(v.x) && ez_finite(v.y) && ez_finite(v.z); }
/* (a x - b y) / det per component */
EZ_HD ez_vec3 ez_tangent_comb(float a, ez_vec3 x, float b, ez_vec3 y, float det) {
    return ez_divs(ez_sub(ez_scale(x, a), ez_scale(y, b)), det);
}
/* the triangle's tangent frame (T', B) about the unflipped shading normal No; 0 when it falls back */
EZ_HD int ez_tangent_frame(ez_vec3 p1, ez_vec3 p2, ez_vec3 p3, const float* uv6, ez_vec3 No, ez_vec3* T, ez_vec3* B) {
    const ez_vec3 e1 = ez_sub(p2, p1), e2 = ez_sub(p3, p1);
    const float du1 = uv6[2] - uv6[0], dv1 = uv6[3] - uv6[1], du2 = uv6[4] - uv6[0], dv2 = uv6[5] - uv6[1];
    const float det = du1 * dv2 - du2 * dv1;
    if (det == 0.0f || !ez_finite(det)) return 0;
    const ez_vec3 Tu = ez_tangent_comb(dv2, e1, dv1, e2, det);
    const ez_vec3 Bu = ez_tangent_comb(du1, e2, du2, e1, det);
    const ez_vec3 Tp = ez_sub(Tu, ez_scale(No, ez_dot(No, Tu)));
    const float l2 = ez_dot(Tp, Tp);
    if (l2 == 0.0f || !ez_finite(l2)) return 0;
    *T = ez_normalize(Tp);
    ez_vec3 b = ez_cross(No, *T);
    const float s = ez_dot(b, Bu);
    if (s == 0.0f || !ez_finite(s)) return 0;
    *B = (s < 0.0f) ? ez_neg(b) : b;
    return 1;
}
/* the mapped shading normal of a hit at (u, v) on (p1, p2, p3) with the triangle's UVs uv6: f the normal map's filtered colour, N
 * surface_hit's shading normal, inside the hit's side, V = -d */
EZ_HD ez_vec3 ez_normal_map(ez_vec3 p1, ez_vec3 p2, ez_vec3 p3, const float* uv6, float u, float v, ez_vec3 f, ez_vec3 N, int inside, ez_vec3 V) {
    if (!ez_finite(u) || !ez_finite(v)) return N;
    const ez_vec3 No = inside ? ez_neg(N) : N;
    ez_vec3 T, B;
    if (!ez_tangent_frame(p1, p2, p3, uv6, No, &T, &B)) return N;
    const float tx = 2.0f * f.x - 1.0f, ty = 2.0f * f.y - 1.0f, tz = 2.0f * f.z - 1.0f;
    ez_vec3 n = ez_normalize(ez_add(ez_add(ez_scale(T, tx), ez_scale(B, ty)), ez_scale(No, tz)));
    if (!ez_finite3(n)) return N;
    if (inside) n = ez_neg(n);
    if (!(ez_dot(n, V) > 0.0f)) return N;
    return n;
}
/* the material-maps word of a texcoord record (its fourth float's bits): (metal_rough_id + 1) | (normal_id + 1) << 16 */
EZ_HD int ez_maps_mr_id(uint32_t w) { return (int)(w & 0xffffu) - 1; }
EZ_HD int ez_maps_normal_id(uint32_t w) { return (int)(w >> 16) - 1; }

#endif /* EZRT_MATH_H */
