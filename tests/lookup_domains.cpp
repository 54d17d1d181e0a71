// lookup_domains.cpp -- the render path's lookups and ezrt_math.h's functions over their whole input domains, on the host.
//
//   lookup_domains lookups        every texture, HDR-map and environment-table lookup at hostile coordinates: UVs at 0, +-2^23,
//                                 2^31 - 128, +-2^31, +-3e9, +-2^40, +-FLT_MAX, +-inf and NaN, each paired with every other, on
//                                 textures of 1x1, 1x7, 5x1, 3x5 and 16384x1 texels held in arrays of exactly their size, and the
//                                 environment's pdf at every direction built from those values (NaN and zero-length ones included).
//                                 Built with -fsanitize=address,undefined,float-cast-overflow, it must report nothing; it prints
//                                 one line of counts and checks what the definition promises of each result.
//   lookup_domains scan FN        the largest error of FN (sin cos log exp asin atan) against float64 libm over every fp32 input of
//                                 its domain, in ulps of the exact result, on all hardware threads; sin and cos also print the
//                                 largest absolute error over |x| < 8192.
//
// *** TEST INFRASTRUCTURE (tests/test_lookup_domains.py, tests/test_kat.py).
#include "../oracle/ezrt_oracle.cpp"

#include <float.h>
#include <math.h>
#include <stdio.h>

#include <thread>

namespace {

int g_failures = 0;

void fail(const char* what, float u, float v, int W, int H) {
    if (g_failures++ < 20) fprintf(stderr, "FAIL %s at (%a, %a) on %d x %d\n", what, u, v, W, H);
}

bool in01(vec3 c) { return c.x >= 0.0f && c.x <= 1.0f && c.y >= 0.0f && c.y <= 1.0f && c.z >= 0.0f && c.z <= 1.0f; }

const float kValues[] = {0.0f, 8388608.0f, -8388608.0f, 2147483520.0f, 2147483648.0f, -2147483648.0f, 3e9f, -3e9f,
                         1099511627776.0f, -1099511627776.0f, FLT_MAX, -FLT_MAX, INFINITY, -INFINITY, NAN};
const int kN = sizeof(kValues) / sizeof(kValues[0]);
const int kSizes[][2] = {{1, 1}, {1, 7}, {5, 1}, {3, 5}, {16384, 1}};

uint32_t hash32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}

int lookups() {
    long calls = 0;
    for (const auto& sz : kSizes) {
        const int W = sz[0], H = sz[1];
        std::vector<uint32_t> texels((size_t)W * H);
        for (size_t i = 0; i < texels.size(); i++) texels[i] = hash32((uint32_t)i + 1u);
        std::vector<float> img((size_t)W * H * 3), pdf((size_t)W * H);
        for (size_t i = 0; i < img.size(); i++) img[i] = (float)(hash32((uint32_t)i + 77u) & 0xffffu) / 65536.0f;
        for (size_t i = 0; i < pdf.size(); i++) pdf[i] = 1.0f / (float)pdf.size();
        for (int a = 0; a < kN; a++)
            for (int b = 0; b < kN; b++) {
                const float u = kValues[a], v = kValues[b];
                const bool finite = ez_finite(u) && ez_finite(v);
                const bool scaled = ez_finite(u * (float)W - 0.5f) && ez_finite(v * (float)H - 0.5f);
                // the textures' filter: a texel-weighted colour in [0, 1] for every finite UV, exactly white otherwise
                for (const float* lut : {ez_srgb_table, ez_unorm8_table}) {
                    const vec3 c = ez_tex_sample(texels.data(), W, H, u, v, lut);
                    calls++;
                    if (finite ? !in01(c) : !(c.x == 1.0f && c.y == 1.0f && c.z == 1.0f)) fail("ez_tex_sample", u, v, W, H);
                }
                // the normal map at the hit (u, v) of a triangle whose UVs are (u, v) and its unit offsets
                const float uv6[6] = {u, v, u + 1.0f, v, u, v + 1.0f};
                const vec3 N = ez_v3(0.0f, 0.0f, 1.0f);
                const vec3 f = ez_tex_sample(texels.data(), W, H, u, v, ez_unorm8_table);
                for (int inside = 0; inside < 2; inside++) {
                    const vec3 n = ez_normal_map(ez_v3(0, 0, 0), ez_v3(1, 0, 0), ez_v3(0, 1, 0), uv6, u, v, f, inside ? ez_neg(N) : N, inside,
                                                 ez_v3(0.0f, 0.6f, 0.8f));
                    calls++;
                    if (!ez_finite3(n)) fail("ez_normal_map", u, v, W, H);
                }
                // the HDR map's lookups (the oracle's tex2D): nearest reads a texel; bilinear is a texel mix, NaN (a weight of
                // inf - inf or NaN) where u W or v H is not finite
                const vec3 t0 = tex2D(img.data(), W, H, u, v, false), t1 = tex2D(img.data(), W, H, u, v, true);
                calls += 2;
                if (!in01(t0)) fail("tex2D nearest", u, v, W, H);
                if (scaled ? !in01(t1) : !(t1.x != t1.x && t1.y != t1.y && t1.z != t1.z)) fail("tex2D bilinear", u, v, W, H);
                const int k = ez_env_texel(u, v, W, H);
                calls++;
                if (k < 0 || k >= W * H) fail("ez_env_texel", u, v, W, H);
                if ((u != u && k % W != 0) || (v != v && k / W != 0)) fail("ez_env_texel NaN axis", u, v, W, H);
                for (int c = 0; c < kN; c++) {
                    const float p = ez_env_pdf(pdf.data(), W, H, ez_v3(u, v, kValues[c]));
                    calls++;
                    if (p < 0.0f) fail("ez_env_pdf", u, v, W, H);
                }
            }
        // unit directions and the zero vector
        const vec3 dirs[] = {ez_v3(0, 0, 0), ez_v3(-0.0f, 0, -0.0f), ez_v3(0, 1, 0), ez_v3(0, -1, 0), ez_v3(1, 0, 0), ez_v3(0, 0, -1),
                             ez_v3(1e-30f, 1e-30f, 1e-30f), ez_v3(NAN, 0, 0)};
        for (const vec3& d : dirs) {
            float u, v;
            ez_to_spherical(ez_normalize(d), &u, &v);
            calls += 3;
            const int k = ez_env_texel(u, v, W, H);
            if (k < 0 || k >= W * H) fail("ez_env_texel of a direction", u, v, W, H);
            const float p = ez_env_pdf(pdf.data(), W, H, d);
            if (p < 0.0f) fail("ez_env_pdf of a direction", u, v, W, H);
            const vec3 t = tex2D(img.data(), W, H, u, v, false);
            if (!in01(t)) fail("tex2D nearest of a direction", u, v, W, H);
        }
    }
    printf("lookups %ld failures %d\n", calls, g_failures);
    return g_failures ? 1 : 0;
}

// ulps of the exact result r between got and r: |got - r| / 2^(e - 23) with 2^e <= |r| < 2^(e + 1), e >= -126
double ulp_error(float got, double r) {
    if (std::isnan(r)) return std::isnan(got) ? 0.0 : INFINITY;
    if (std::isinf(r)) return ((double)got == r) ? 0.0 : INFINITY;
    int e;
    frexp(fabs(r), &e);
    return fabs((double)got - r) / ldexp(1.0, (e - 1 < -126 ? -126 : e - 1) - 23);
}

int scan(const char* fn) {
    const int which = !strcmp(fn, "sin") ? 0 : !strcmp(fn, "cos") ? 1 : !strcmp(fn, "log") ? 2 : !strcmp(fn, "exp") ? 3
                    : !strcmp(fn, "asin") ? 4 : !strcmp(fn, "atan") ? 5 : -1;
    if (which < 0) return 2;
    struct Result { double ulp = 0, abs = 0; uint32_t ulp_at = 0, abs_at = 0; uint64_t n = 0; };
    const int T = (int)std::thread::hardware_concurrency() > 0 ? (int)std::thread::hardware_concurrency() : 1;
    std::vector<Result> res(T);
    std::vector<std::thread> pool;
    for (int t = 0; t < T; t++)
        pool.emplace_back([&, t] {
            Result r;
            for (uint64_t i = (uint64_t)t; i < (1ull << 32); i += (uint64_t)T) {
                const float x = ez_u2f((uint32_t)i);
                if (x != x) continue;
                float got;
                double want;
                bool ulp_domain = true;
                switch (which) {
                    case 0: case 1:
                        if (!(fabsf(x) < 8192.0f)) continue;
                        got = which ? ez_cos(x) : ez_sin(x);
                        want = which ? cos((double)x) : sin((double)x);
                        ulp_domain = fabsf(x) <= 4.0f * 3.14159265358979f;
                        if (fabs((double)got - want) > r.abs) { r.abs = fabs((double)got - want); r.abs_at = (uint32_t)i; }
                        break;
                    case 2: if (!(x > 0.0f)) continue; got = ez_log(x); want = log((double)x); break;
                    case 3: if (!(x <= 88.72283f)) continue; got = ez_exp(x); want = exp((double)x); break;
                    case 4: if (!(fabsf(x) <= 1.0f)) continue; got = ez_asin(x); want = asin((double)x); break;
                    default: got = ez_atan(x); want = atan((double)x); break;
                }
                if (!ulp_domain) continue;
                r.n++;
                const double e = ulp_error(got, want);
                if (e > r.ulp) { r.ulp = e; r.ulp_at = (uint32_t)i; }
            }
            res[t] = r;
        });
    for (auto& th : pool) th.join();
    Result best;
    for (const Result& r : res) {
        best.n += r.n;
        if (r.ulp > best.ulp) { best.ulp = r.ulp; best.ulp_at = r.ulp_at; }
        if (r.abs > best.abs) { best.abs = r.abs; best.abs_at = r.abs_at; }
    }
    printf("scan %s inputs %llu max_ulp %.6g at %a max_abs %.6g at %a\n", fn, (unsigned long long)best.n, best.ulp,
           (double)ez_u2f(best.ulp_at), best.abs, (double)ez_u2f(best.abs_at));
    return 0;
}

}  // namespace

int main(int argc, char** argv) {
    if (argc >= 2 && !strcmp(argv[1], "lookups")) return lookups();
    if (argc >= 3 && !strcmp(argv[1], "scan")) return scan(argv[2]);
    fprintf(stderr, "usage: %s lookups | scan sin|cos|log|exp|asin|atan\n", argv[0]);
    return 2;
}
