// glsl_emul.h -- the subset of GLSL 4.30 that EzRT's fragment shaders use, as C++17.
//
// *** TEST INFRASTRUCTURE (oracle/), NOT PRODUCT.  See oracle/README.md.
//
// Purpose: compile the reference's own shader SOURCE TEXT (shaders/fshader.fsh of tutorial parts 3, 4
// and 5, read from /root/reference at build time by transpile.py, never copied into this repository)
// for the CPU, so the hand-written oracle (oracle/ezrt_oracle.cpp) and the CUDA kernels can be checked
// against the statements, expression order and control flow the reference actually contains.
//
// What is NOT taken from the reference here is exactly what GLSL leaves unspecified bit-wise: the
// built-in functions.  Each maps to the normative fp32 definition in include/ezrt_math.h (the same
// one the oracle and the kernels use); operators are IEEE fp32 (compile with -ffp-contract=off).
// Texture filtering follows the conventions stated in oracle/ezrt_oracle.cpp's header.
#ifndef EZRT_GLSL_EMUL_H
#define EZRT_GLSL_EMUL_H

#include <stdint.h>

#include "ezrt_math.h"

namespace glsl {

typedef unsigned int uint;

struct vec2 {
    union { float x, r; };
    union { float y, g; };
    vec2() : x(0.0f), y(0.0f) {}
    explicit vec2(float s) : x(s), y(s) {}
    vec2(float a, float b) : x(a), y(b) {}
    vec2& operator+=(float s) { x = x + s; y = y + s; return *this; }
    vec2& operator+=(vec2 o) { x = x + o.x; y = y + o.y; return *this; }
    vec2& operator/=(vec2 o) { x = x / o.x; y = y / o.y; return *this; }
};
inline vec2 operator+(vec2 a, vec2 b) { return vec2(a.x + b.x, a.y + b.y); }
inline vec2 operator+(vec2 a, float s) { return vec2(a.x + s, a.y + s); }
inline vec2 operator-(vec2 a, vec2 b) { return vec2(a.x - b.x, a.y - b.y); }
inline vec2 operator*(vec2 a, float s) { return vec2(a.x * s, a.y * s); }
inline vec2 operator*(float s, vec2 a) { return vec2(s * a.x, s * a.y); }

struct vec3 {
    union { float x, r; };
    union { float y, g; };
    union { float z, b; };
    vec3() : x(0.0f), y(0.0f), z(0.0f) {}
    explicit vec3(float s) : x(s), y(s), z(s) {}
    vec3(float a, float b_, float c) : x(a), y(b_), z(c) {}
    vec3(ez_vec3 v) : x(v.x), y(v.y), z(v.z) {}
    ez_vec3 ez() const { return ez_v3(x, y, z); }
    vec2 xy() const { return vec2(x, y); }
    vec3 xyz() const { return *this; }
    vec3 rgb() const { return *this; }
    vec3& operator+=(vec3 o) { x = x + o.x; y = y + o.y; z = z + o.z; return *this; }
    vec3& operator*=(vec3 o) { x = x * o.x; y = y * o.y; z = z * o.z; return *this; }
    vec3& operator*=(float s) { x = x * s; y = y * s; z = z * s; return *this; }
};
inline vec3 operator+(vec3 a, vec3 b) { return vec3(a.x + b.x, a.y + b.y, a.z + b.z); }
inline vec3 operator-(vec3 a, vec3 b) { return vec3(a.x - b.x, a.y - b.y, a.z - b.z); }
inline vec3 operator-(vec3 a) { return vec3(-a.x, -a.y, -a.z); }
inline vec3 operator*(vec3 a, vec3 b) { return vec3(a.x * b.x, a.y * b.y, a.z * b.z); }
inline vec3 operator*(vec3 a, float s) { return vec3(a.x * s, a.y * s, a.z * s); }
inline vec3 operator*(float s, vec3 a) { return vec3(s * a.x, s * a.y, s * a.z); }
inline vec3 operator/(vec3 a, float s) { return vec3(a.x / s, a.y / s, a.z / s); }
inline vec3 operator/(vec3 a, vec3 b) { return vec3(a.x / b.x, a.y / b.y, a.z / b.z); }
inline vec3 operator/(float s, vec3 a) { return vec3(s / a.x, s / a.y, s / a.z); }

struct vec4 {
    union { float x, r; };
    union { float y, g; };
    union { float z, b; };
    union { float w, a; };
    vec4() : x(0.0f), y(0.0f), z(0.0f), w(0.0f) {}
    explicit vec4(float s) : x(s), y(s), z(s), w(s) {}
    vec4(float a_, float b_, float c, float d) : x(a_), y(b_), z(c), w(d) {}
    vec4(vec3 v, float d) : x(v.x), y(v.y), z(v.z), w(d) {}
    vec4(vec2 v, float c, float d) : x(v.x), y(v.y), z(c), w(d) {}
    vec3 xyz() const { return vec3(x, y, z); }
    vec3 rgb() const { return vec3(x, y, z); }
    vec2 xy() const { return vec2(x, y); }
    vec2 rg() const { return vec2(x, y); }
};

struct ivec3 {
    int x, y, z;
    explicit ivec3(vec3 v) : x((int)v.x), y((int)v.y), z((int)v.z) {}  // float -> int truncates
};

// column-major like GLSL / glm::value_ptr.  mat4 * vec4: the products of one row are summed left to
// right (column 0 first), every operation rounded -- the convention of oracle/ezrt_oracle.cpp main().
struct mat4 {
    float m[16];
};
inline vec4 operator*(const mat4& M, vec4 v) {
    const float* m = M.m;
    return vec4(((m[0] * v.x + m[4] * v.y) + m[8] * v.z) + m[12] * v.w,
                ((m[1] * v.x + m[5] * v.y) + m[9] * v.z) + m[13] * v.w,
                ((m[2] * v.x + m[6] * v.y) + m[10] * v.z) + m[14] * v.w,
                ((m[3] * v.x + m[7] * v.y) + m[11] * v.z) + m[15] * v.w);
}

// ---- built-in functions -> include/ezrt_math.h ----
inline float abs(float x) { return ez_abs(x); }
inline float sqrt(float x) { return EZ_SQRT(x); }
inline float sin(float x) { return ez_sin(x); }
inline float cos(float x) { return ez_cos(x); }
inline float log(float x) { return ez_log(x); }
inline float exp(float x) { return ez_exp(x); }
inline float pow(float x, float y) { return ez_pow(x, y); }
inline vec3 pow(vec3 x, vec3 y) { return vec3(ez_pow(x.x, y.x), ez_pow(x.y, y.y), ez_pow(x.z, y.z)); }
inline float asin(float x) { return ez_asin(x); }
inline float atan(float y, float x) { return ez_atan2(y, x); }
inline float min(float a, float b) { return ez_min(a, b); }
inline float max(float a, float b) { return ez_max(a, b); }
inline vec3 min(vec3 a, vec3 b) { return vec3(ez_vmin(a.ez(), b.ez())); }
inline vec3 max(vec3 a, vec3 b) { return vec3(ez_vmax(a.ez(), b.ez())); }
inline float clamp(float x, float lo, float hi) { return ez_clamp(x, lo, hi); }
inline float mix(float a, float b, float t) { return ez_mix(a, b, t); }
inline vec3 mix(vec3 a, vec3 b, float t) { return vec3(ez_vmix(a.ez(), b.ez(), t)); }
inline float dot(vec3 a, vec3 b) { return ez_dot(a.ez(), b.ez()); }
inline vec3 cross(vec3 a, vec3 b) { return vec3(ez_cross(a.ez(), b.ez())); }
inline vec3 normalize(vec3 v) { return vec3(ez_normalize(v.ez())); }
inline vec3 reflect(vec3 I, vec3 N) { return vec3(ez_reflect(I.ez(), N.ez())); }

// ---- samplers ----
// samplerBuffer over GL_RGB32F texels (P5/main.cpp glTexBuffer(GL_TEXTURE_BUFFER, GL_RGB32F, tbo))
struct samplerBuffer {
    const float* texels;
};
inline vec4 texelFetch(const samplerBuffer& s, int i) {
    return vec4(s.texels[3 * (long long)i], s.texels[3 * (long long)i + 1], s.texels[3 * (long long)i + 2], 1.0f);
}

// sampler2D over an RGB32F image with `channels` floats per texel, CLAMP_TO_EDGE, row 0 <-> v = 0.
// filter: 0 = GL_NEAREST, 1 = GL_LINEAR (fp32 bilinear, texel centres at +0.5).
struct sampler2D {
    const float* img;
    int w, h, channels, filter;
};
inline vec3 texel2D(const sampler2D& s, int ix, int iy) {
    const float* p = s.img + ((long long)iy * s.w + ix) * s.channels;
    return vec3(p[0], p[1], p[2]);
}
inline vec4 texture2D(const sampler2D& s, vec2 uv) {
    if (s.filter == 0) {
        int ix = ez_texel_clamp(ez_floor(uv.x * (float)s.w), s.w);
        int iy = ez_texel_clamp(ez_floor(uv.y * (float)s.h), s.h);
        return vec4(texel2D(s, ix, iy), 1.0f);
    }
    float x = uv.x * (float)s.w - 0.5f, y = uv.y * (float)s.h - 0.5f;
    float fx0 = ez_floor(x), fy0 = ez_floor(y);
    float ax = x - fx0, ay = y - fy0;
    int x0 = ez_texel_clamp(fx0, s.w), x1 = ez_texel_clamp(fx0 + 1.0f, s.w);
    int y0 = ez_texel_clamp(fy0, s.h), y1 = ez_texel_clamp(fy0 + 1.0f, s.h);
    vec3 t00 = texel2D(s, x0, y0), t10 = texel2D(s, x1, y0), t01 = texel2D(s, x0, y1), t11 = texel2D(s, x1, y1);
    return vec4(mix(mix(t00, t10, ax), mix(t01, t11, ax), ay), 1.0f);
}

// uniforms of all three shaders (P3/P4 use a subset); set by the host harness per frame
struct Uniforms {
    uint frameCounter;
    int nTriangles, nNodes, width, height, hdrResolution;
    samplerBuffer triangles, nodes;
    sampler2D lastFrame, hdrMap, hdrCache;
    sampler2D texPass0, texPass1, texPass2, texPass3, texPass4, texPass5, texPass6;  // pass2/pass3 inputs (RenderPass::draw)
    vec3 eye;
    mat4 cameraRotate;
};

}  // namespace glsl

#endif
