// oracle_punctual.cpp -- CPU restatement of the punctual lights (EZRT_PARAM_PUNCTUAL_LIGHTS in EZRT_MODE_DISNEY_LIGHTS, ezrt_math.h,
// DESIGN.md section 17): the table (ezrt_punctual.h, the library's own builder) and the category split of every light sample, over
// the material maps' restatement (tests/oracle_material_maps.cpp, included unchanged).  Its two loops -- the homogeneous medium's
// (mode 4's when there is no medium) and the transmission mixture's -- are restated with the punctual category beside the map and
// the triangle lights, with every other option: the environment light, the thin lens, the medium, textures and maps.
// Plain/window, feature-buffer and adaptive forms.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT, like the oracle it compiles in (build/libezrt_oracle_punctual.so, tests/oracle_punctual.py).
//
// A render without EZRT_PARAM_TEXTURES runs with every texture id and map id -1, which changes no material and no normal; a render
// without EZRT_PARAM_PUNCTUAL_LIGHTS (or with a table of J = 0) has P_p = 0 and is the maps restatement's, bit for bit.
#include "oracle_material_maps.cpp"

#include "ezrt_punctual.h"

namespace {

struct PunctSet {
    EzPunctTable t;
    int J = 0;
};

// P_p of a render: 0 without punctual lights, 1 without triangle lights and map table, 1/2 otherwise
float punctProb(const PunctSet& pt, int K, bool envOn) { return pt.J == 0 ? 0.0f : ((K > 0 || envOn) ? 0.5f : 1.0f); }

// The category split of r_sel: true (punctual) with *r_p, false with *r_env for the map-or-triangle rule
bool punctPick(float P_p, float r_sel, float* r_p, float* r_env) {
    *r_env = r_sel;
    if (P_p == 0.0f) return false;
    if (P_p == 1.0f || r_sel < 0.5f) {
        *r_p = (P_p == 1.0f) ? r_sel : r_sel * 2.0f;
        return true;
    }
    *r_env = (r_sel - 0.5f) * 2.0f;
    return false;
}

// the vertex box of the caller's triangles, as the library's scene preparation computes it (moves on < and > from +-3e38)
void vertexBox(const float* tris, int n, float bmin[3], float bmax[3]) {
    for (int k = 0; k < 3; k++) { bmin[k] = 3.0e38f; bmax[k] = -3.0e38f; }
    for (int i = 0; i < n; i++)
        for (int v = 0; v < 3; v++)
            for (int k = 0; k < 3; k++) {
                const float x = tris[(size_t)i * EZRT_TRIANGLE_FLOATS + 3 * v + k];
                if (x < bmin[k]) bmin[k] = x;
                if (x > bmax[k]) bmax[k] = x;
            }
}

// shadePixelMapsMedium (tests/oracle_material_maps.cpp) with the punctual category
vec3 shadePixelPunctMedium(const Scene& sc, const Tables& tb, const TexSet& ts, const MapSet& ms, const PunctSet& pt, const ez_medium& med,
                           const ezrt_render_params& p, const ez_lens* lens, uint32_t ipx, uint32_t ipy, uint32_t frameCounter, Counters& cn,
                           First* first) {
    PixelCtx px;
    px.px = ipx; px.py = ipy; px.frameCounter = frameCounter;
    Ray ray = cameraRay(p, lens, px);
    const bool envOn = (p.reserved[0] & EZRT_PARAM_ENV_LIGHT) && tb.env.ok;
    const int K = (int)tb.lt.tri.size();
    const float P_env = envOn ? (K > 0 ? 0.5f : 1.0f) : 0.0f;
    const float P_p = punctProb(pt, K, envOn);
    vec3 Lo = splat(0), Le = splat(0), history = splat(1), f_r = splat(0);
    float pdf = 1.0f, cosine = 0.0f;
    for (int bounce = 0;; bounce++) {
        const HitResult h = hitBVH(sc, ray, cn, bounce == 0 ? 0 : 1);
        if (bounce == 0) firstOf(sc, ts, ms, h, first);
        if (bounce > 0 && pdf <= 0.0f) break;
        float t_s;
        const float t_end = h.isHit ? h.distance : ez_u2f(0x7f800000u);
        const bool scatter = ez_medium_flight(&med, ray.startPoint, ray.direction, t_end, &px.rng.seed, &t_s) != 0;
        if (!scatter && !h.isHit) {
            if (bounce == 0) return hdrColor(sc, ray.direction, cn);
            float w = 1.0f;
            if (P_env > 0.0f) {
                const float pe = P_env * ez_env_pdf(tb.env.pdf.data(), tb.env.W, tb.env.H, ray.direction);
                w = (P_p > 0.0f) ? misMixWeight(pdf, (1.0f - P_p) * pe) : misMixWeight(pdf, pe);
            }
            Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), hdrColor(sc, ray.direction, cn)), f_r), cosine), pdf));
            break;
        }
        if (!scatter) {
            const vec3 E = getMaterial(sc, h.triangle).emissive;
            if (bounce == 0) {
                Le = E;
            } else {
                float w = 1.0f;
                const float lum = ez_luminance(E);
                if (lum > 0.0f) {
                    const Triangle T = getTriangle(sc, h.triangle);
                    if (ez_is_light(ez_light_weight(T.p1, T.p2, T.p3, E))) {
                        float pl = ez_light_pdf(lum, tb.lt.total_f, h.distance, ez_abs(ez_dot(geoNormal(T), ray.direction)));
                        if (envOn) pl = (1.0f - P_env) * pl;
                        w = (P_p > 0.0f) ? misMixWeight(pdf, (1.0f - P_p) * pl) : misMixWeight(pdf, pl);
                    }
                }
                Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), E), f_r), cosine), pdf));
                history = ez_mul(history, ez_divs(ez_scale(f_r, cosine), pdf));
            }
        } else {
            if (bounce > 0) history = ez_mul(history, ez_divs(ez_scale(f_r, cosine), pdf));
            history = ez_mul(history, med.albedo);
        }
        if (bounce >= p.max_bounce) break;
        const vec3 P = scatter ? ez_add(ray.startPoint, ez_scale(ray.direction, t_s)) : h.hitPoint;
        const vec3 d = ray.direction;
        const vec3 Vv = ez_neg(h.viewDir);
        vec3 N = h.normal;
        Material material = scatter ? Material() : getMaterial(sc, h.triangle);
        if (!scatter) mapMaterial(sc, ts, ms, h.triangle, h.hitPoint, Vv, h.isInside, &material, &N);
        const float r_sel = px.rng.rand();
        const float r_1 = px.rng.rand();
        const float r_2 = px.rng.rand();
        float r_p = 0.0f, r_env;
        const bool punct = punctPick(P_p, r_sel, &r_p, &r_env);
        const bool envPick = !punct && ((P_env == 1.0f) || (P_env == 0.5f && r_env < 0.5f));
        const float r_tri = (P_env == 0.5f) ? (r_env - 0.5f) * 2.0f : r_env;
        if (punct) {
            const float* rec = pt.t.rec.data() + 16 * (size_t)ez_light_select(pt.t.cdf.data(), pt.J, r_p);
            vec3 Ll;
            float tmax, s;
            if (ez_punct_sample(rec, P_p * rec[12], P, N, scatter ? 1 : 0, &Ll, &tmax, &s)) {
                Ray sray;
                sray.startPoint = P;
                sray.direction = Ll;
                if (!occludedBounded(sc, sray, tmax, cn)) {
                    vec3 f;
                    float cl = 1.0f;
                    if (scatter) {
                        f = splat(ez_hg_pdf(d, Ll, med.g));
                    } else {
                        f = BRDF_Evaluate(Vv, N, Ll, splat(0), splat(0), material, false);
                        cl = ez_dot(N, Ll);
                    }
                    const vec3 c = ez_punct_contrib(history, f, cl, ez_v3(rec[8], rec[9], rec[10]), s);
                    Lo = ez_add(Lo, ez_scale(c, ez_medium_transmittance(&med, P, Ll, ez_medium_light_dist(tmax, rec[3] == 2.0f))));
                }
            }
        } else if (envPick) {
            int texel;
            const vec3 Ld = ez_env_sample(tb.env.row.data(), tb.env.col.data(), tb.env.W, tb.env.H, r_1, r_2, &texel);
            const float pdf_env = P_env * ez_env_pdf(tb.env.pdf.data(), tb.env.W, tb.env.H, Ld);
            if (ez_finite(pdf_env) && pdf_env > 0.0f && (scatter || ez_dot(N, Ld) > 0.0f)) {
                Ray sray;
                sray.startPoint = P;
                sray.direction = Ld;
                if (!occludedBounded(sc, sray, EZ_INF, cn)) {
                    const float pl = (P_p > 0.0f) ? pdf_env * (1.0f - P_p) : pdf_env;
                    const vec3 c = mediumLightContrib(history, scatter, d, Vv, N, Ld, material, med.g, hdrColor(sc, Ld, cn), pl);
                    Lo = ez_add(Lo, ez_scale(c, ez_medium_transmittance(&med, P, Ld, ez_medium_light_dist(EZ_INF, 1))));
                }
            }
        } else if (K > 0) {
            const int k = ez_light_select(tb.lt.cdf.data(), K, r_tri);
            const int tk = tb.lt.tri[k];
            const Triangle T = getTriangle(sc, tk);
            const vec3 E = getMaterial(sc, tk).emissive;
            const vec3 D = ez_sub(ez_triangle_point(T.p1, T.p2, T.p3, r_1, r_2), P);
            const float dist = EZ_SQRT(ez_dot(D, D));
            const vec3 Ll = ez_normalize(D);
            const float cos_l = ez_abs(ez_dot(geoNormal(T), Ll));
            if ((scatter || (tk != h.triangle && ez_dot(N, Ll) > 0.0f)) && cos_l != 0.0f && dist != 0.0f) {
                Ray sray;
                sray.startPoint = P;
                sray.direction = Ll;
                const float tmax = ez_light_tmax(dist);
                if (!occludedBounded(sc, sray, tmax, cn)) {
                    float pdf_light = ez_light_pdf(ez_luminance(E), tb.lt.total_f, dist, cos_l);
                    if (envOn) pdf_light = pdf_light * (1.0f - P_env);
                    if (P_p > 0.0f) pdf_light = pdf_light * (1.0f - P_p);
                    const vec3 c = mediumLightContrib(history, scatter, d, Vv, N, Ll, material, med.g, E, pdf_light);
                    Lo = ez_add(Lo, ez_scale(c, ez_medium_transmittance(&med, P, Ll, ez_medium_light_dist(tmax, 0))));
                }
            }
        }
        vec3 L;
        if (scatter) {
            const float h_1 = px.rng.rand();
            const float h_2 = px.rng.rand();
            L = ez_hg_sample(d, med.g, h_1, h_2);
            pdf = ez_hg_pdf(d, L, med.g);
            f_r = splat(pdf);
            cosine = 1.0f;
        } else {
            float xi_1, xi_2;
            sobolVec2(px.frameCounter + 1u, (uint32_t)bounce, &xi_1, &xi_2);
            CranleyPattersonRotation(&xi_1, &xi_2, px.px, px.py);
            const float xi_3 = px.rng.rand();
            L = SampleBRDF(xi_1, xi_2, xi_3, Vv, N, material);
            cosine = ez_dot(N, L);
            if (cosine <= 0.0f) break;
            f_r = BRDF_Evaluate(Vv, N, L, splat(0), splat(0), material, false);
            pdf = BRDF_Pdf(Vv, N, L, material);
        }
        ray.startPoint = P;
        ray.direction = L;
    }
    return ez_add(Le, Lo);
}

// pathTracingTransMaps (tests/oracle_material_maps.cpp) with the punctual category
vec3 pathTracingTransPunct(const Scene& sc, const TexSet& ts, const MapSet& ms, const PunctSet& pt, const LightTable& lt, const EnvTable& env,
                           HitResult hit, int maxBounce, PixelCtx& px, Counters& cn) {
    vec3 Lo = splat(0);
    vec3 history = splat(1);
    const int K = (int)lt.tri.size();
    const float P_env = env.ok ? (K > 0 ? 0.5f : 1.0f) : 0.0f;
    const float P_p = punctProb(pt, K, env.ok);
    for (int bounce = 0; bounce < maxBounce; bounce++) {
        vec3 Vv = ez_neg(hit.viewDir);
        vec3 N = hit.normal;
        Material material = getMaterial(sc, hit.triangle);
        mapMaterial(sc, ts, ms, hit.triangle, hit.hitPoint, Vv, hit.isInside, &material, &N);
        const TransLobe tl = transLobe(material, hit.isInside);

        const float r_sel = px.rng.rand();
        const float r_1 = px.rng.rand();
        const float r_2 = px.rng.rand();
        float r_p = 0.0f, r_env;
        const bool punct = punctPick(P_p, r_sel, &r_p, &r_env);
        const bool envPick = !punct && ((P_env == 1.0f) || (P_env == 0.5f && r_env < 0.5f));
        const float r_tri = (P_env == 0.5f) ? (r_env - 0.5f) * 2.0f : r_env;
        if (punct) {
            const float* rec = pt.t.rec.data() + 16 * (size_t)ez_light_select(pt.t.cdf.data(), pt.J, r_p);
            vec3 Ll;
            float tmax, s;
            if (ez_punct_sample(rec, P_p * rec[12], hit.hitPoint, N, 0, &Ll, &tmax, &s)) {
                Ray sray;
                sray.startPoint = hit.hitPoint;
                sray.direction = Ll;
                if (!occludedBounded(sc, sray, tmax, cn)) {
                    float pdf_unused;
                    const vec3 f = (tl.t == 0.0f) ? BRDF_Evaluate(Vv, N, Ll, splat(0), splat(0), material, false)
                                                  : BSDF_Evaluate(Vv, N, Ll, material, tl, &pdf_unused);
                    Lo = ez_add(Lo, ez_punct_contrib(history, f, ez_dot(N, Ll), ez_v3(rec[8], rec[9], rec[10]), s));
                }
            }
        } else if (envPick) {
            int texel;
            const vec3 Le = ez_env_sample(env.row.data(), env.col.data(), env.W, env.H, r_1, r_2, &texel);
            const float pdf_env = P_env * ez_env_pdf(env.pdf.data(), env.W, env.H, Le);
            if (ez_finite(pdf_env) && pdf_env > 0.0f && ez_dot(N, Le) > 0.0f) {
                Ray sray;
                sray.startPoint = hit.hitPoint;
                sray.direction = Le;
                const float pl = (P_p > 0.0f) ? pdf_env * (1.0f - P_p) : pdf_env;
                if (!occludedBounded(sc, sray, EZ_INF, cn)) Lo = ez_add(Lo, lightContrib(history, Vv, N, Le, material, tl, hdrColor(sc, Le, cn), pl));
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
                    float pdf_light = ez_light_pdf(ez_luminance(E), lt.total_f, dist, cos_l) * (1.0f - P_env);
                    if (P_p > 0.0f) pdf_light = pdf_light * (1.0f - P_p);
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
            float w = 1.0f;
            if (P_env > 0.0f && !below) {
                const float pe = P_env * ez_env_pdf(env.pdf.data(), env.W, env.H, L);
                w = (P_p > 0.0f) ? misMixWeight(pdf_b, (1.0f - P_p) * pe) : misMixWeight(pdf_b, pe);
            }
            Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), hdrColor(sc, L, cn)), f_r), ac), pdf_b));
            break;
        }
        const vec3 Le = getMaterial(sc, newHit.triangle).emissive;
        float w = 1.0f;
        const float lum = ez_luminance(Le);
        if (lum > 0.0f && !below) {
            const Triangle T = getTriangle(sc, newHit.triangle);
            if (ez_is_light(ez_light_weight(T.p1, T.p2, T.p3, Le))) {
                const float pl = (1.0f - P_env) * ez_light_pdf(lum, lt.total_f, newHit.distance, ez_abs(ez_dot(geoNormal(T), L)));
                w = (P_p > 0.0f) ? misMixWeight(pdf_b, (1.0f - P_p) * pl) : misMixWeight(pdf_b, pl);
            }
        }
        Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), Le), f_r), ac), pdf_b));
        hit = newHit;
        history = ez_mul(history, ez_divs(ez_scale(f_r, ac), pdf_b));
    }
    return Lo;
}

// one sample of a punctual render: the transmission loop with EZRT_PARAM_TRANSMISSION, the medium loop otherwise
vec3 shadePixelPunct(const Scene& sc, const Tables& tb, const TexSet& ts, const MapSet& ms, const PunctSet& pt, const ez_medium& med,
                     const ezrt_render_params& p, const ez_lens* lens, uint32_t ipx, uint32_t ipy, uint32_t frameCounter, Counters& cn, First* first) {
    if (!(p.reserved[0] & EZRT_PARAM_TRANSMISSION)) return shadePixelPunctMedium(sc, tb, ts, ms, pt, med, p, lens, ipx, ipy, frameCounter, cn, first);
    PixelCtx px;
    px.px = ipx; px.py = ipy; px.frameCounter = frameCounter;
    const Ray ray = cameraRay(p, lens, px);
    const HitResult firstHit = hitBVH(sc, ray, cn, 0);
    firstOf(sc, ts, ms, firstHit, first);
    if (!firstHit.isHit) return hdrColor(sc, ray.direction, cn);
    return ez_add(getMaterial(sc, firstHit.triangle).emissive, pathTracingTransPunct(sc, ts, ms, pt, tb.lt, tb.env, firstHit, p.max_bounce, px, cn));
}

// The validated set-up: textures and maps (all ids -1 without EZRT_PARAM_TEXTURES / EZRT_PARAM_MATERIAL_MAPS), the medium and the
// punctual table; -2 where the library returns EZRT_ERR_INVALID
struct Setup {
    ez_medium med;
    TexSet ts;
    MapSet ms;
    PunctSet pt;
    std::vector<int32_t> none;   // -1 per triangle
    std::vector<float> uv0;      // 0 per texcoord
};

int punctSetup(const ezrt_render_params* p, const ezrt_medium* m, int nTex, const ezrt_texture* tex, const float* uv, const int32_t* id,
               const int32_t* mr, const int32_t* nm, const float* tris, int nTriangles, int nLights, const ezrt_punctual_light* lights, Setup* s) {
    const int f = p->reserved[0];
    if (p->mode != EZRT_MODE_DISNEY_LIGHTS || p->pipeline == EZRT_PIPELINE_MEGAKERNEL) return -2;
    s->none.assign((size_t)nTriangles, -1);
    s->uv0.assign(6 * (size_t)nTriangles, 0.0f);
    if (f & EZRT_PARAM_TEXTURES) {
        if (!texSetOf(nTex, tex, uv, id, nTriangles, &s->ts)) return -2;
    } else {
        s->ts.uv = s->uv0.data();
        s->ts.id = s->none.data();
    }
    if (f & EZRT_PARAM_MATERIAL_MAPS) {
        if (!(f & EZRT_PARAM_TEXTURES) || !mapSetOf(mr, nm, nTex, nTriangles, &s->ms)) return -2;
    } else {
        s->ms.mr = s->none.data();
        s->ms.normal = s->none.data();
    }
    memset(&s->med, 0, sizeof(s->med));
    if (f & EZRT_PARAM_MEDIUM) {
        if (f & EZRT_PARAM_TRANSMISSION) return -2;
        if (!mediumOf(m, &s->med)) return -2;
    }
    if (f & EZRT_PARAM_PUNCTUAL_LIGHTS) {
        if (!lights || nLights < 0) return -2;
        float bmin[3], bmax[3];
        vertexBox(tris, nTriangles, bmin, bmax);
        const char* why;
        if (ez_punct_build(nLights, lights, bmin, bmax, &s->pt.t, &why) >= 0) return -2;
        s->pt.J = (int)s->pt.t.index.size();
    }
    return 0;
}

}  // namespace

extern "C" {

// The table of n lights over the triangles' vertex box: returns J (writing min(J, cap) entries) or -1 - k for invalid light k
int oracle_punct_table(const float* tris, int nTriangles, int n, const ezrt_punctual_light* lights, int cap, int32_t* index_out, float* cdf_out,
                       float* q_out, float* rec_out, double* total_out) {
    float bmin[3], bmax[3];
    vertexBox(tris, nTriangles, bmin, bmax);
    EzPunctTable t;
    const char* why;
    const int bad = ez_punct_build(n, lights, bmin, bmax, &t, &why);
    if (bad >= 0) return -1 - bad;
    const int J = (int)t.index.size();
    for (int j = 0; j < J && j < cap; j++) {
        if (index_out) index_out[j] = t.index[j];
        if (cdf_out) cdf_out[j] = t.cdf[j];
        if (q_out) q_out[j] = t.q[j];
        if (rec_out) memcpy(rec_out + 16 * j, t.rec.data() + 16 * j, 16 * sizeof(float));
    }
    if (total_out) *total_out = t.W;
    return J;
}

// ez_punct_sample of n rows: rec (16 floats), pq, P (3), N (3), medium -> ok, L (3), tmax, s
void oracle_punct_sample(int n, const float* rec, const float* pq, const float* P, const float* N, const int32_t* medium, int32_t* ok, float* L,
                         float* tmax, float* s) {
    for (int i = 0; i < n; i++) {
        vec3 l = splat(0);
        float t = 0.0f, sc = 0.0f;
        ok[i] = ez_punct_sample(rec + 16 * (size_t)i, pq[i], ez_v3(P[3 * i], P[3 * i + 1], P[3 * i + 2]), ez_v3(N[3 * i], N[3 * i + 1], N[3 * i + 2]),
                                medium[i], &l, &t, &sc);
        L[3 * i] = l.x; L[3 * i + 1] = l.y; L[3 * i + 2] = l.z;
        tmax[i] = t;
        s[i] = sc;
    }
}

// The window [x0,x1) x [y0,y1) as oracle_render_material_maps, with the punctual lights of ezrt_scene_set_punctual_lights (used with
// EZRT_PARAM_PUNCTUAL_LIGHTS); the textures and maps are read only with their flags; aov (8 floats per pixel): the first hit's features
int oracle_render_punctual(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache, int hdrW,
                           int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, int nTex, const ezrt_texture* tex,
                           const float* uv, const int32_t* id, const int32_t* mr, const int32_t* nm, int nLights, const ezrt_punctual_light* lights,
                           int x0, int y0, int x1, int y1, float* framebuffer, float* aov, float* luma2, uint64_t* counters_out, int n_threads) {
    if (!p || !tris) return -1;
    Setup su;
    int rc = punctSetup(p, m, nTex, tex, uv, id, mr, nm, tris, nTriangles, nLights, lights, &su);
    if (rc) return rc;
    ez_lens lens;
    bool on;
    rc = checkRender(tris, nTriangles, nodes, nNodes, hdr, hdrCache, p, x0, y0, x1, y1, &lens, &on);
    if (rc) return rc;
    if (!framebuffer || !luma2) return -1;
    Scene sc = makeScene(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p->env_color, p->mode, p->traverse);
    const Tables tb = makeTables(sc, *p, hdr, hdrW, hdrH);
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
                float* feat = aov ? aov + k * 8 : nullptr;
                vec3 acc = ez_v3(dst[0], dst[1], dst[2]);
                float m2 = luma2[k];
                if (p->first_frame == 0) {
                    acc = ez_v3(0, 0, 0);
                    m2 = 0.0f;
                    if (feat)
                        for (int c = 0; c < 8; c++) feat[c] = 0.0f;
                }
                for (int s = 0; s < p->spp; s++) {
                    const uint32_t frame = p->first_frame + (uint32_t)s;
                    First f;
                    const vec3 color = shadePixelPunct(sc, tb, su.ts, su.ms, su.pt, su.med, *p, on ? &lens : nullptr, (uint32_t)pxl, (uint32_t)py, frame,
                                                       cn, &f);
                    const float a = EZ_DIV(1.0f, ez_u32_to_float(frame + 1u));
                    acc = ez_vmix(acc, color, a);
                    const float y = ez_luminance(color);
                    m2 = ez_mix(m2, y * y, a);
                    if (feat) {
                        float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                        if (f.h.isHit) {
                            v[0] = f.albedo.x; v[1] = f.albedo.y; v[2] = f.albedo.z; v[3] = 1.0f;
                            v[4] = f.normal.x; v[5] = f.normal.y; v[6] = f.normal.z; v[7] = f.h.distance;
                        }
                        for (int c = 0; c < 8; c++) feat[c] = ez_mix(feat[c], v[c], a);
                    }
                }
                dst[0] = acc.x; dst[1] = acc.y; dst[2] = acc.z;
                if (C == 4) dst[3] = 1.0f;
                luma2[k] = m2;
            }
        }
#pragma omp critical
        addCounters(total, cn);
    }
    writeCounters(counters_out, total, (uint64_t)(x1 - x0) * (y1 - y0) * (uint64_t)p->spp);
    return 0;
}

// The adaptive form (tests/oracle_material_maps.cpp's loop with this file's sample function)
int oracle_render_punctual_adaptive(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache,
                                    int hdrW, int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, int nTex,
                                    const ezrt_texture* tex, const float* uv, const int32_t* id, const int32_t* mr, const int32_t* nm, int nLights,
                                    const ezrt_punctual_light* lights, const ezrt_adaptive_params* ap, int x0, int y0, int x1, int y1,
                                    float* framebuffer, int32_t* spp_out, float* luma2_out, uint64_t* counters_out, int n_threads) {
    if (!p || !tris) return -1;
    Setup su;
    int rc = punctSetup(p, m, nTex, tex, uv, id, mr, nm, tris, nTriangles, nLights, lights, &su);
    if (rc) return rc;
    ez_lens lens;
    bool on;
    rc = checkRender(tris, nTriangles, nodes, nNodes, hdr, hdrCache, p, x0, y0, x1, y1, &lens, &on);
    if (rc) return rc;
    if (!ap || !framebuffer || !spp_out || !luma2_out) return -1;
    if (p->first_frame != 0 || ap->min_spp < 2 || ap->check_interval < 1 || !(ap->threshold > 0.0f)) return -1;
    if (x0 % EZRT_TILE_SIZE || y0 % EZRT_TILE_SIZE || (x1 % EZRT_TILE_SIZE && x1 != p->width) || (y1 % EZRT_TILE_SIZE && y1 != p->height)) return -1;
    Scene sc = makeScene(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p->env_color, p->mode, p->traverse);
    const Tables tb = makeTables(sc, *p, hdr, hdrW, hdrH);
    const int C = (p->out_channels == 4) ? 4 : 3;
    const int W = x1 - x0;
    const int tx0 = x0 / EZRT_TILE_SIZE, ty0 = y0 / EZRT_TILE_SIZE;
    const int tnx = (x1 - x0 + EZRT_TILE_SIZE - 1) / EZRT_TILE_SIZE, tny = (y1 - y0 + EZRT_TILE_SIZE - 1) / EZRT_TILE_SIZE;
    Counters total;
    memset(&total, 0, sizeof(total));
    uint64_t samples = 0;
#ifdef _OPENMP
    if (n_threads > 0) omp_set_num_threads(n_threads);
#endif
#pragma omp parallel
    {
        Counters cn;
        memset(&cn, 0, sizeof(cn));
        uint64_t my_samples = 0;
        std::vector<vec3> acc;
        std::vector<float> m2;
#pragma omp for schedule(dynamic, 1)
        for (int t = 0; t < tnx * tny; t++) {
            const int bx = (tx0 + t % tnx) * EZRT_TILE_SIZE, by = (ty0 + t / tnx) * EZRT_TILE_SIZE;
            const int tw = (p->width - bx < EZRT_TILE_SIZE) ? p->width - bx : EZRT_TILE_SIZE;
            const int th = (p->height - by < EZRT_TILE_SIZE) ? p->height - by : EZRT_TILE_SIZE;
            acc.assign((size_t)tw * th, ez_v3(0, 0, 0));
            m2.assign((size_t)tw * th, 0.0f);
            int n = 0, next = ap->min_spp;
            for (;;) {
                const int stop = (p->spp < next) ? p->spp : next;
                for (int i = 0; i < tw * th; i++) {
                    const uint32_t px = (uint32_t)(bx + i % tw), py = (uint32_t)(by + i / tw);
                    for (int f = n; f < stop; f++) {
                        const vec3 color = shadePixelPunct(sc, tb, su.ts, su.ms, su.pt, su.med, *p, on ? &lens : nullptr, px, py, (uint32_t)f, cn, nullptr);
                        const float a = EZ_DIV(1.0f, ez_u32_to_float((uint32_t)f + 1u));
                        acc[i] = ez_vmix(acc[i], color, a);
                        const float y = ez_luminance(color);
                        m2[i] = ez_mix(m2[i], y * y, a);
                    }
                }
                n = stop;
                if (n >= p->spp) break;
                bool converged = true;
                for (int i = 0; i < tw * th && converged; i++) converged = ez_adaptive_error(m2[i], acc[i], n) <= ap->threshold;
                if (converged) break;
                next += ap->check_interval;
            }
            for (int i = 0; i < tw * th; i++) {
                const size_t k = (size_t)(by + i / tw - y0) * W + (size_t)(bx + i % tw - x0);
                float* dst = framebuffer + k * C;
                dst[0] = acc[i].x; dst[1] = acc[i].y; dst[2] = acc[i].z;
                if (C == 4) dst[3] = 1.0f;
                spp_out[k] = n;
                luma2_out[k] = m2[i];
            }
            my_samples += (uint64_t)n * (uint64_t)(tw * th);
        }
#pragma omp critical
        {
            addCounters(total, cn);
            samples += my_samples;
        }
    }
    writeCounters(counters_out, total, samples);
    return 0;
}

}  // extern "C"
