// oracle_transmission.cpp -- CPU restatement of the materials' transmission (EZRT_PARAM_TRANSMISSION in EZRT_MODE_DISNEY_LIGHTS,
// ezrt_math.h, DESIGN.md section 12): the mixture of the reference BRDF with the rough dielectric, its sampler, and the flagged
// per-pixel integrator with and without EZRT_PARAM_ENV_LIGHT, over the environment light's restatement (tests/oracle_env_light.cpp,
// included unchanged) and the oracle's functions.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT, like the oracle it compiles in (build/libezrt_oracle_transmission.so,
// tests/oracle_transmission.py).
//
// bsdf_only (a switch of the restatement only): no light samples, and every emission and environment hit of a BSDF sample weighs 1
// -- an independent estimator of the same integral, for the unbiasedness tests.
#include "oracle_env_light.cpp"

namespace {

struct TransLobe {
    float t, eta, alpha;
    bool matched;
};

TransLobe transLobe(const Material& m, bool inside) {
    TransLobe r;
    r.t = ez_trans_weight(m.transmission, m.metallic, m.IOR);
    r.eta = ez_trans_eta(m.IOR, inside ? 1 : 0);
    r.alpha = ez_max(0.001f, ez_sqr(m.roughness));
    r.matched = ez_trans_matched(m.IOR) != 0;
    return r;
}

// the mixture's f at L and its pdf
vec3 BSDF_Evaluate(vec3 Vv, vec3 N, vec3 L, const Material& m, const TransLobe& tl, float* pdf) {
    vec3 f_ref = splat(0), f_diel = splat(0);
    float pdf_ref = 0.0f, pdf_diel = 0.0f;
    if (ez_dot(N, L) > 0.0f) { f_ref = BRDF_Evaluate(Vv, N, L, splat(0), splat(0), m, false); pdf_ref = BRDF_Pdf(Vv, N, L, m); }
    if (!tl.matched) f_diel = ez_diel_eval(Vv, N, L, m.baseColor, tl.alpha, tl.eta, &pdf_diel);
    return ez_trans_mix(f_ref, pdf_ref, f_diel, pdf_diel, tl.t, pdf);
}

// the mixture's sample: L and the f, pdf and signed cosine the path carries; false: the path ends.  On entry *L is SampleBRDF's
// sample of (xi_1, xi_2, xi_3), the reference lobe's.
bool SampleBSDF(float xi_1, float xi_2, float xi_3, float r_t, vec3 Vv, vec3 N, const Material& m, const TransLobe& tl, vec3* L, vec3* f,
                float* pdf, float* cosine) {
    if (r_t < tl.t) {
        if (tl.matched) {
            *L = ez_neg(Vv);
            *f = m.baseColor;
            *pdf = 1.0f;
            *cosine = -1.0f;
            return true;
        }
        if (!ez_diel_sample(xi_1, xi_2, xi_3, Vv, N, tl.alpha, tl.eta, L)) return false;
    } else if (!(ez_dot(N, *L) > 0.0f)) {
        return false;
    }
    *f = BSDF_Evaluate(Vv, N, *L, m, tl, pdf);
    *cosine = ez_dot(N, *L);
    return true;
}

// a light sample's contribution: the reference BRDF where t == 0, the mixture otherwise
vec3 lightContrib(vec3 history, vec3 Vv, vec3 N, vec3 Ll, const Material& m, const TransLobe& tl, vec3 E, float pdf_light) {
    vec3 f_r;
    float pdf_b;
    if (tl.t == 0.0f) {
        f_r = BRDF_Evaluate(Vv, N, Ll, splat(0), splat(0), m, false);
        pdf_b = BRDF_Pdf(Vv, N, Ll, m);
    } else {
        f_r = BSDF_Evaluate(Vv, N, Ll, m, tl, &pdf_b);
    }
    const float mis_weight = misMixWeight(pdf_light, pdf_b);
    return ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, mis_weight), E), f_r), ez_dot(N, Ll)), pdf_light);
}

// pathTracingEnvLights (tests/oracle_env_light.cpp) with the transmission mixture; env.ok false: the light samples are mode 4's
vec3 pathTracingTrans(const Scene& sc, const LightTable& lt, const EnvTable& env, HitResult hit, int maxBounce, PixelCtx& px, Counters& cn,
                      bool bsdfOnly) {
    vec3 Lo = splat(0);
    vec3 history = splat(1);
    const int K = (int)lt.tri.size();
    const float P_env = env.ok ? (K > 0 ? 0.5f : 1.0f) : 0.0f;
    for (int bounce = 0; bounce < maxBounce; bounce++) {
        vec3 Vv = ez_neg(hit.viewDir);
        vec3 N = hit.normal;
        Material material = getMaterial(sc, hit.triangle);
        const TransLobe tl = transLobe(material, hit.isInside);

        const float r_sel = px.rng.rand();
        const float r_1 = px.rng.rand();
        const float r_2 = px.rng.rand();
        const bool envPick = (P_env == 1.0f) || (P_env == 0.5f && r_sel < 0.5f);
        const float r_tri = (P_env == 0.5f) ? (r_sel - 0.5f) * 2.0f : r_sel;
        if (bsdfOnly) {
        } else if (envPick) {
            int texel;
            const vec3 Le = ez_env_sample(env.row.data(), env.col.data(), env.W, env.H, r_1, r_2, &texel);
            const float pdf_env = P_env * ez_env_pdf(env.pdf.data(), env.W, env.H, Le);
            if (ez_finite(pdf_env) && pdf_env > 0.0f && ez_dot(N, Le) > 0.0f) {
                Ray sray;
                sray.startPoint = hit.hitPoint;
                sray.direction = Le;
                if (!occludedBounded(sc, sray, EZ_INF, cn)) Lo = ez_add(Lo, lightContrib(history, Vv, N, Le, material, tl, hdrColor(sc, Le, cn), pdf_env));
            }
        } else if (K > 0) {
            const int k = ez_light_select(lt.cdf.data(), K, r_tri);
            const int tk = lt.tri[k];
            const Triangle T = getTriangle(sc, tk);
            const vec3 E = getMaterial(sc, tk).emissive;
            const vec3 D = ez_sub(ez_triangle_point(T.p1, T.p2, T.p3, r_1, r_2), hit.hitPoint);
            const float dist = EZ_SQRT(ez_dot(D, D));
            const vec3 Ll = ez_normalize(D);
            const float cos_l = ez_abs(ez_dot(geoNormal(T), Ll));
            if (tk != hit.triangle && ez_dot(N, Ll) > 0.0f && cos_l != 0.0f && dist != 0.0f) {
                Ray sray;
                sray.startPoint = hit.hitPoint;
                sray.direction = Ll;
                if (!occludedBounded(sc, sray, ez_light_tmax(dist), cn)) {
                    const float pdf_light = ez_light_pdf(ez_luminance(E), lt.total_f, dist, cos_l) * (1.0f - P_env);
                    Lo = ez_add(Lo, lightContrib(history, Vv, N, Ll, material, tl, E, pdf_light));
                }
            }
        }

        float xi_1, xi_2;
        sobolVec2(px.frameCounter + 1u, (uint32_t)bounce, &xi_1, &xi_2);
        CranleyPattersonRotation(&xi_1, &xi_2, px.px, px.py);
        float xi_3 = px.rng.rand();
        vec3 L = SampleBRDF(xi_1, xi_2, xi_3, Vv, N, material), f_r;
        float pdf_b, cosine;
        if (tl.t == 0.0f) {   // mode 4's sample
            cosine = ez_dot(N, L);
            if (cosine <= 0.0f) break;
        } else {
            const float r_t = px.rng.rand();
            if (!SampleBSDF(xi_1, xi_2, xi_3, r_t, Vv, N, material, tl, &L, &f_r, &pdf_b, &cosine)) break;
        }

        Ray randomRay;
        randomRay.startPoint = hit.hitPoint;
        randomRay.direction = L;
        HitResult newHit = hitBVH(sc, randomRay, cn, 1);
        if (tl.t == 0.0f) {
            f_r = BRDF_Evaluate(Vv, N, L, splat(0), splat(0), material, false);
            pdf_b = BRDF_Pdf(Vv, N, L, material);
        }
        if (pdf_b <= 0.0f) break;
        const bool below = cosine < 0.0f;   // no light strategy reaches it: weight 1
        const float ac = ez_abs(cosine);
        if (!newHit.isHit) {
            const float w = (P_env > 0.0f && !below && !bsdfOnly) ? misMixWeight(pdf_b, P_env * ez_env_pdf(env.pdf.data(), env.W, env.H, L)) : 1.0f;
            Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), hdrColor(sc, L, cn)), f_r), ac), pdf_b));
            break;
        }
        const vec3 Le = getMaterial(sc, newHit.triangle).emissive;
        float w = 1.0f;
        const float lum = ez_luminance(Le);
        if (lum > 0.0f && !below && !bsdfOnly) {
            const Triangle T = getTriangle(sc, newHit.triangle);
            if (ez_is_light(ez_light_weight(T.p1, T.p2, T.p3, Le)))
                w = misMixWeight(pdf_b, (1.0f - P_env) * ez_light_pdf(lum, lt.total_f, newHit.distance, ez_abs(ez_dot(geoNormal(T), L))));
        }
        Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), Le), f_r), ac), pdf_b));
        hit = newHit;
        history = ez_mul(history, ez_divs(ez_scale(f_r, ac), pdf_b));
    }
    return Lo;
}

vec3 shadePixelTrans(const Scene& sc, const LightTable& lt, const EnvTable& env, const ezrt_render_params& p, uint32_t ipx, uint32_t ipy,
                     uint32_t frameCounter, Counters& cn, bool bsdfOnly) {
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
    const float* m = p.camera_rotate;
    vec3 dir = ez_v3(((m[0] * vx + m[4] * vy) + m[8] * vz) + m[12] * vw,
                     ((m[1] * vx + m[5] * vy) + m[9] * vz) + m[13] * vw,
                     ((m[2] * vx + m[6] * vy) + m[10] * vz) + m[14] * vw);
    ray.direction = ez_normalize(dir);
    HitResult firstHit = hitBVH(sc, ray, cn, 0);
    if (!firstHit.isHit) return hdrColor(sc, ray.direction, cn);
    return ez_add(getMaterial(sc, firstHit.triangle).emissive, pathTracingTrans(sc, lt, env, firstHit, p.max_bounce, px, cn, bsdfOnly));
}

}  // namespace

extern "C" {

// which: 0 f, 1 pdf, 2 the sample of xi[4 i ..] = (xi_1, xi_2, xi_3, r_t); out as ezrt_eval_bsdf's (8 floats per tuple)
int oracle_eval_bsdf(int which, int n, const float* Vv, const float* Nn, const float* Ll, const float* xi, const int32_t* inside,
                     const float* materials, float* out) {
    for (int i = 0; i < n; i++) {
        const vec3 V3 = ez_v3(Vv[3 * i], Vv[3 * i + 1], Vv[3 * i + 2]);
        const vec3 N3 = ez_v3(Nn[3 * i], Nn[3 * i + 1], Nn[3 * i + 2]);
        const Material m = materialFrom18(materials + (size_t)i * 18);
        const TransLobe tl = transLobe(m, inside[i] != 0);
        float r[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (which == 0 || which == 1) {
            float pdf;
            const vec3 f = BSDF_Evaluate(V3, N3, ez_v3(Ll[3 * i], Ll[3 * i + 1], Ll[3 * i + 2]), m, tl, &pdf);
            if (which == 0) { r[0] = f.x; r[1] = f.y; r[2] = f.z; }
            else r[0] = pdf;
        } else if (which == 2) {
            vec3 L = SampleBRDF(xi[4 * i], xi[4 * i + 1], xi[4 * i + 2], V3, N3, m), f;
            float pdf, cosine;
            if (SampleBSDF(xi[4 * i], xi[4 * i + 1], xi[4 * i + 2], xi[4 * i + 3], V3, N3, m, tl, &L, &f, &pdf, &cosine)) {
                r[0] = L.x; r[1] = L.y; r[2] = L.z; r[3] = f.x; r[4] = f.y; r[5] = f.z; r[6] = pdf; r[7] = cosine;
            }
        } else {
            return -1;
        }
        for (int k = 0; k < 8; k++) out[8 * (size_t)i + k] = r[k];
    }
    return 0;
}

// ez_fresnel_dielectric of n (cos_i, eta) pairs
void oracle_fresnel(int n, const float* cos_i, const float* eta, float* out) {
    for (int i = 0; i < n; i++) out[i] = ez_fresnel_dielectric(cos_i[i], eta[i]);
}

// oracle_render_env_light (tests/oracle_env_light.cpp) with EZRT_PARAM_TRANSMISSION read from p->reserved[0]: mode 4 with the flag
// runs the mixture (with the map as a light if EZRT_PARAM_ENV_LIGHT is set too), anything else what oracle_render_env_light runs.
int oracle_render_transmission(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache,
                               int hdrW, int hdrH, int hdrLinear, const ezrt_render_params* p, int x0, int y0, int x1, int y1, float* framebuffer,
                               float* luma2, uint64_t* counters_out, int n_threads, int bsdf_only) {
    const bool flagged = p && p->mode == EZRT_MODE_DISNEY_LIGHTS && (p->reserved[0] & EZRT_PARAM_TRANSMISSION);
    if (!flagged)
        return oracle_render_env_light(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p, x0, y0, x1, y1, framebuffer,
                                       luma2, counters_out, n_threads);
    if (!tris || !nodes || !framebuffer || !luma2 || nTriangles <= 0 || nNodes < 2) return -1;
    if (x0 < 0 || y0 < 0 || x1 > p->width || y1 > p->height || x1 <= x0 || y1 <= y0) return -1;
    Scene sc = makeScene(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p->env_color, p->mode, p->traverse);
    const LightTable lt = buildLights(sc);
    const EnvTable env = (p->reserved[0] & EZRT_PARAM_ENV_LIGHT) ? buildEnv(hdr, hdrW, hdrH) : EnvTable();
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
                const size_t k = (size_t)(py - y0) * (x1 - x0) + (pxl - x0);
                float* dst = framebuffer + k * C;
                vec3 acc = ez_v3(dst[0], dst[1], dst[2]);
                float m2 = luma2[k];
                if (p->first_frame == 0) { acc = ez_v3(0, 0, 0); m2 = 0.0f; }
                for (int s = 0; s < p->spp; s++) {
                    const uint32_t frame = p->first_frame + (uint32_t)s;
                    const vec3 color = shadePixelTrans(sc, lt, env, *p, (uint32_t)pxl, (uint32_t)py, frame, cn, bsdf_only != 0);
                    const float a = EZ_DIV(1.0f, ez_u32_to_float(frame + 1u));
                    acc = ez_vmix(acc, color, a);
                    const float y = ez_luminance(color);
                    m2 = ez_mix(m2, y * y, a);
                }
                dst[0] = acc.x; dst[1] = acc.y; dst[2] = acc.z;
                if (C == 4) dst[3] = 1.0f;
                luma2[k] = m2;
            }
        }
#pragma omp critical
        {
            for (int k = 0; k < 3; k++) total.rays[k] += cn.rays[k];
            total.nodes += cn.nodes; total.tris += cn.tris; total.hits += cn.hits;
            total.hdr_lookups += cn.hdr_lookups;
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

}  // extern "C"
