// oracle_emission_maps.cpp -- CPU restatement of the emission maps (EZRT_PARAM_EMISSION_MAPS in EZRT_MODE_DISNEY_LIGHTS, ezrt_math.h,
// DESIGN.md section 18): the emission table and E(Q) at every place mode 4 reads emission, over the punctual lights' restatement
// (tests/oracle_punctual.cpp, included unchanged).  Its two loops -- the homogeneous medium's (mode 4's when there is no medium) and
// the transmission mixture's -- are restated with E(Q) at the camera ray's hit, at BSDF-sample emission hits and in the triangle light
// samples, and with the emission table as the render's light table, with every other option: the environment light, the thin lens,
// the medium, textures, material maps and punctual lights.  Plain/window, feature-buffer and adaptive forms.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT, like the oracle it compiles in (build/libezrt_oracle_emission_maps.so,
// tests/oracle_emission_maps.py).
//
// A render without EZRT_PARAM_EMISSION_MAPS runs with every emission id -1 and mode 4's table, and is the punctual restatement's, bit
// for bit.
#include "oracle_punctual.cpp"

namespace {

// The emission maps of a render: the ids, each triangle's lum_eff (ez_emit_lum_eff for a mapped emitter, lum(E) otherwise), the
// emission table and its lights' record luminance (the records' fourth word)
struct EmitSet {
    const int32_t* id = nullptr;
    const TexSet* ts = nullptr;
    std::vector<float> lumEff;
    LightTable lt;
    std::vector<float> lightLum;
    float misScale = 1.0f;   // test-only: a mapped light's lum_eff in the emission hits' MIS weights times this
};

// a mapped emitter: lum(E_T) > 0 and an emission id
bool emitMapped(const Scene& sc, const EmitSet& es, int tri) { return es.id[tri] >= 0 && ez_luminance(getMaterial(sc, tri).emissive) > 0.0f; }

// lum_eff of triangle tri with emission texture k
float emitLumEff(const Scene& sc, const TexSet& ts, int tri, int k) {
    return ez_emit_lum_eff(getMaterial(sc, tri).emissive, ts.uv + 6 * (size_t)tri, ts.texels.data() + ts.off[k], ts.W[k], ts.H[k], ez_srgb_table);
}

// the emission table of ids `id` (lumIn: test-only lum_eff per triangle in place of ez_emit_lum_eff's), in section 10's layout
void emitSetOf(const Scene& sc, const TexSet& ts, const int32_t* id, const float* lumIn, EmitSet* es) {
    es->id = id;
    es->ts = &ts;
    es->lumEff.assign((size_t)sc.nTriangles, 0.0f);
    std::vector<float> w;
    for (int i = 0; i < sc.nTriangles; i++) {
        const Triangle t = getTriangle(sc, i);
        const vec3 E = getMaterial(sc, i).emissive;
        const bool mapped = emitMapped(sc, *es, i);
        es->lumEff[i] = mapped ? (lumIn ? lumIn[i] : emitLumEff(sc, ts, i, id[i])) : ez_luminance(E);
        const float wi = mapped ? ez_triangle_area(t.p1, t.p2, t.p3) * es->lumEff[i] : ez_light_weight(t.p1, t.p2, t.p3, E);
        if (!ez_is_light(wi)) continue;
        es->lt.tri.push_back(i);
        es->lightLum.push_back(es->lumEff[i]);
        w.push_back(wi);
    }
    for (float x : w) es->lt.total += (double)x;
    double S = 0.0;
    for (float x : w) {
        S += (double)x;
        es->lt.cdf.push_back((float)(S / es->lt.total));
    }
    if (!es->lt.cdf.empty()) es->lt.cdf.back() = 1.0f;
    es->lt.total_f = (float)es->lt.total;
}

// E(Q) at Q on triangle tri; *mapped: the triangle is a mapped emitter
vec3 emitAt(const Scene& sc, const TexSet& ts, const EmitSet& es, int tri, vec3 Q, bool* mapped) {
    const vec3 E = getMaterial(sc, tri).emissive;
    *mapped = emitMapped(sc, es, tri);
    if (!*mapped) return E;
    const Triangle T = getTriangle(sc, tri);
    const int k = es.id[tri];
    return ez_emit_eval(E, Q, T.p1, T.p2, T.p3, geoNormal(T), ts.uv + 6 * (size_t)tri, ts.texels.data() + ts.off[k], ts.W[k], ts.H[k], ez_srgb_table);
}

// E(Q) of the light sample on light triangle tk at ez_triangle_point(r_1, r_2) (every light has lum(E) > 0)
vec3 emitLight(const Scene& sc, const TexSet& ts, const EmitSet& es, int tk, float r_1, float r_2) {
    const Triangle T = getTriangle(sc, tk);
    bool mapped;
    return emitAt(sc, ts, es, tk, ez_triangle_point(T.p1, T.p2, T.p3, r_1, r_2), &mapped);
}

bool emitBlack(vec3 E) { return E.x == 0.0f && E.y == 0.0f && E.z == 0.0f; }

// an emission hit's membership: the table's own (area * lum_eff) on a mapped triangle, section 10's otherwise
bool emitIsLight(const Scene& sc, const EmitSet& es, int tri, bool mapped) {
    const Triangle T = getTriangle(sc, tri);
    if (mapped) return ez_is_light(ez_triangle_area(T.p1, T.p2, T.p3) * es.lumEff[tri]);
    return ez_is_light(ez_light_weight(T.p1, T.p2, T.p3, getMaterial(sc, tri).emissive));
}

// the luminance of an emission hit's MIS pdf: lum_eff (times the test-only misScale) on a mapped triangle, lum(E_T) otherwise
float emitMisLum(const EmitSet& es, int tri, float lum, bool mapped) { return mapped ? es.lumEff[tri] * es.misScale : lum; }

// The two pdfs of a point on a light that must agree (before the 1 - P_env and 1 - P_p factors).  A light sample's: light k of the
// table lt, its point at distance dist along L from the shading point.
float emitSamplePdf(const Scene& sc, const EmitSet& es, const LightTable& lt, int k, float dist, vec3 L) {
    const Triangle T = getTriangle(sc, lt.tri[k]);
    return ez_light_pdf(es.lightLum[k], lt.total_f, dist, ez_abs(ez_dot(geoNormal(T), L)));
}
// A BSDF sample's emission hit at distance t along d on triangle tri: false when tri is not a light of the table
bool emitHitPdf(const Scene& sc, const EmitSet& es, const LightTable& lt, int tri, float t, vec3 d, float* pdf) {
    const float lum = ez_luminance(getMaterial(sc, tri).emissive);
    if (!(lum > 0.0f)) return false;
    const bool mapped = emitMapped(sc, es, tri);
    if (!emitIsLight(sc, es, tri, mapped)) return false;
    const Triangle T = getTriangle(sc, tri);
    *pdf = ez_light_pdf(emitMisLum(es, tri, lum, mapped), lt.total_f, t, ez_abs(ez_dot(geoNormal(T), d)));
    return true;
}

// shadePixelPunctMedium (tests/oracle_punctual.cpp) with E(Q) and the emission table (tb.lt)
vec3 shadePixelEmitMedium(const Scene& sc, const Tables& tb, const TexSet& ts, const MapSet& ms, const PunctSet& pt, const EmitSet& es, const ez_medium& med,
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
            bool mapped;
            const vec3 E = emitAt(sc, ts, es, h.triangle, h.hitPoint, &mapped);
            if (bounce == 0) {
                Le = E;
            } else {
                float w = 1.0f, pl;
                if (emitHitPdf(sc, es, tb.lt, h.triangle, h.distance, ray.direction, &pl)) {
                    if (envOn) pl = (1.0f - P_env) * pl;
                    w = (P_p > 0.0f) ? misMixWeight(pdf, (1.0f - P_p) * pl) : misMixWeight(pdf, pl);
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
            const vec3 E = emitLight(sc, ts, es, tk, r_1, r_2);
            const vec3 D = ez_sub(ez_triangle_point(T.p1, T.p2, T.p3, r_1, r_2), P);
            const float dist = EZ_SQRT(ez_dot(D, D));
            const vec3 Ll = ez_normalize(D);
            const float cos_l = ez_abs(ez_dot(geoNormal(T), Ll));
            if ((scatter || (tk != h.triangle && ez_dot(N, Ll) > 0.0f)) && cos_l != 0.0f && dist != 0.0f && !emitBlack(E)) {
                Ray sray;
                sray.startPoint = P;
                sray.direction = Ll;
                const float tmax = ez_light_tmax(dist);
                if (!occludedBounded(sc, sray, tmax, cn)) {
                    float pdf_light = emitSamplePdf(sc, es, tb.lt, k, dist, Ll);
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

// pathTracingTransPunct (tests/oracle_punctual.cpp) with E(Q) and the emission table lt
vec3 pathTracingTransEmit(const Scene& sc, const TexSet& ts, const MapSet& ms, const PunctSet& pt, const EmitSet& es, const LightTable& lt, const EnvTable& env,
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
            const vec3 E = emitLight(sc, ts, es, tk, r_1, r_2);
            const vec3 D = ez_sub(ez_triangle_point(T.p1, T.p2, T.p3, r_1, r_2), hit.hitPoint);
            const float dist = EZ_SQRT(ez_dot(D, D));
            const vec3 Ll = ez_normalize(D);
            const float cos_l = ez_abs(ez_dot(geoNormal(T), Ll));
            if (tk != hit.triangle && ez_dot(N, Ll) > 0.0f && cos_l != 0.0f && dist != 0.0f && !emitBlack(E)) {
                Ray sray;
                sray.startPoint = hit.hitPoint;
                sray.direction = Ll;
                if (!occludedBounded(sc, sray, ez_light_tmax(dist), cn)) {
                    float pdf_light = emitSamplePdf(sc, es, lt, k, dist, Ll) * (1.0f - P_env);
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
        bool mapped;
        const vec3 Le = emitAt(sc, ts, es, newHit.triangle, newHit.hitPoint, &mapped);
        float w = 1.0f, pl;
        if (!below && emitHitPdf(sc, es, lt, newHit.triangle, newHit.distance, L, &pl)) {
            pl = (1.0f - P_env) * pl;
            w = (P_p > 0.0f) ? misMixWeight(pdf_b, (1.0f - P_p) * pl) : misMixWeight(pdf_b, pl);
        }
        Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), Le), f_r), ac), pdf_b));
        hit = newHit;
        history = ez_mul(history, ez_divs(ez_scale(f_r, ac), pdf_b));
    }
    return Lo;
}

// one sample of an emission-map render: the transmission loop with EZRT_PARAM_TRANSMISSION, the medium loop otherwise
vec3 shadePixelEmit(const Scene& sc, const Tables& tb, const TexSet& ts, const MapSet& ms, const PunctSet& pt, const EmitSet& es, const ez_medium& med,
                    const ezrt_render_params& p, const ez_lens* lens, uint32_t ipx, uint32_t ipy, uint32_t frameCounter, Counters& cn, First* first) {
    if (!(p.reserved[0] & EZRT_PARAM_TRANSMISSION)) return shadePixelEmitMedium(sc, tb, ts, ms, pt, es, med, p, lens, ipx, ipy, frameCounter, cn, first);
    PixelCtx px;
    px.px = ipx; px.py = ipy; px.frameCounter = frameCounter;
    const Ray ray = cameraRay(p, lens, px);
    const HitResult firstHit = hitBVH(sc, ray, cn, 0);
    firstOf(sc, ts, ms, firstHit, first);
    if (!firstHit.isHit) return hdrColor(sc, ray.direction, cn);
    bool mapped;
    return ez_add(emitAt(sc, ts, es, firstHit.triangle, firstHit.hitPoint, &mapped),
                  pathTracingTransEmit(sc, ts, ms, pt, es, tb.lt, tb.env, firstHit, p.max_bounce, px, cn));
}


}  // namespace

extern "C" {

// ez_emit_lum_eff of n triangles (E: 3 floats, uv6: 6 floats each) over one W x H texture (RGBA8 words), sRGB-decoded
void oracle_emit_lum_eff(int n, const float* E, const float* uv6, const uint32_t* texels, int W, int H, float* out) {
    for (int i = 0; i < n; i++)
        out[i] = ez_emit_lum_eff(ez_v3(E[3 * i], E[3 * i + 1], E[3 * i + 2]), uv6 + 6 * (size_t)i, texels, W, H, ez_srgb_table);
}

// ez_emit_eval of n points: E (3), Q (3), p1..p3 (9), Ng (3), uv6 (6) each, over one texture -> rgb (3 each)
void oracle_emit_eval(int n, const float* E, const float* Q, const float* P, const float* Ng, const float* uv6, const uint32_t* texels, int W, int H,
                      float* rgb) {
    for (int i = 0; i < n; i++) {
        const float* p = P + 9 * (size_t)i;
        const vec3 c = ez_emit_eval(ez_v3(E[3 * i], E[3 * i + 1], E[3 * i + 2]), ez_v3(Q[3 * i], Q[3 * i + 1], Q[3 * i + 2]), ez_v3(p[0], p[1], p[2]),
                                    ez_v3(p[3], p[4], p[5]), ez_v3(p[6], p[7], p[8]), ez_v3(Ng[3 * i], Ng[3 * i + 1], Ng[3 * i + 2]), uv6 + 6 * (size_t)i,
                                    texels, W, H, ez_srgb_table);
        rgb[3 * i] = c.x; rgb[3 * i + 1] = c.y; rgb[3 * i + 2] = c.z;
    }
}

// The emission table of the scene's triangles with textures (tex, uv) and emission ids emit_id: returns K (writing min(K, cap) entries
// of tri_out, cdf_out, lum_out -- the records' fourth word -- and hit_lum_out, the luminance an emission hit on that light's triangle
// uses in its MIS pdf) or -2 where ezrt_scene_set_emission_maps returns EZRT_ERR_INVALID
int oracle_emission_table(const float* tris, int nTriangles, const float* nodes, int nNodes, int nTex, const ezrt_texture* tex, const float* uv,
                          const int32_t* emit_id, int cap, int32_t* tri_out, float* cdf_out, float* lum_out, float* hit_lum_out, double* total_out) {
    std::vector<int32_t> none((size_t)nTriangles, -1);
    TexSet ts;
    if (!texSetOf(nTex, tex, uv, none.data(), nTriangles, &ts)) return -2;
    for (int i = 0; i < nTriangles; i++)
        if (emit_id[i] < -1 || emit_id[i] >= nTex) return -2;
    const Scene sc = makeScene(tris, nTriangles, nodes, nNodes, nullptr, nullptr, 0, 0, 0, nullptr, EZRT_MODE_DISNEY_LIGHTS, EZRT_TRAVERSE_ACCEL);
    EmitSet es;
    emitSetOf(sc, ts, emit_id, nullptr, &es);
    const int K = (int)es.lt.tri.size();
    for (int k = 0; k < K && k < cap; k++) {
        const int t = es.lt.tri[k];
        const bool mapped = emitMapped(sc, es, t);
        if (tri_out) tri_out[k] = t;
        if (cdf_out) cdf_out[k] = es.lt.cdf[k];
        if (lum_out) lum_out[k] = es.lightLum[k];
        if (hit_lum_out) hit_lum_out[k] = emitMisLum(es, t, ez_luminance(getMaterial(sc, t).emissive), mapped);
    }
    if (total_out) *total_out = es.lt.total;
    return K;
}

// For every light k of the emission table and n_pts shading points (P: 3 floats each, one set for every light), a point Q of the
// light (r: 2 draws per point) and both pdfs of it through the render's own code paths: sample_pdf (emitSamplePdf at the light
// sample's dist and direction), hit_pdf (emitHitPdf at the same distance and direction; -1 where the triangle is no light), traced_pdf
// (emitHitPdf at the distance of the ray P -> Q traced through the scene, -1 where it hits another triangle first), all [K, n_pts].
// Returns K, or -2 as oracle_emission_table.
int oracle_emission_pdf_pairs(const float* tris, int nTriangles, const float* nodes, int nNodes, int nTex, const ezrt_texture* tex, const float* uv,
                              const int32_t* emit_id, int cap, int n_pts, const float* P, const float* r, float* sample_pdf, float* hit_pdf,
                              float* traced_pdf) {
    std::vector<int32_t> none((size_t)nTriangles, -1);
    TexSet ts;
    if (!texSetOf(nTex, tex, uv, none.data(), nTriangles, &ts)) return -2;
    for (int i = 0; i < nTriangles; i++)
        if (emit_id[i] < -1 || emit_id[i] >= nTex) return -2;
    const Scene sc = makeScene(tris, nTriangles, nodes, nNodes, nullptr, nullptr, 0, 0, 0, nullptr, EZRT_MODE_DISNEY_LIGHTS, EZRT_TRAVERSE_REFERENCE);
    EmitSet es;
    emitSetOf(sc, ts, emit_id, nullptr, &es);
    const int K = (int)es.lt.tri.size();
    Counters cn;
    memset(&cn, 0, sizeof(cn));
    for (int k = 0; k < K && k < cap; k++) {
        const Triangle T = getTriangle(sc, es.lt.tri[k]);
        for (int j = 0; j < n_pts; j++) {
            const size_t o = (size_t)k * n_pts + j;
            const vec3 Pj = ez_v3(P[3 * j], P[3 * j + 1], P[3 * j + 2]);
            const vec3 D = ez_sub(ez_triangle_point(T.p1, T.p2, T.p3, r[2 * o], r[2 * o + 1]), Pj);
            const float dist = EZ_SQRT(ez_dot(D, D));
            const vec3 L = ez_normalize(D);
            sample_pdf[o] = emitSamplePdf(sc, es, es.lt, k, dist, L);
            float pl;
            hit_pdf[o] = emitHitPdf(sc, es, es.lt, es.lt.tri[k], dist, L, &pl) ? pl : -1.0f;
            Ray ray;
            ray.startPoint = Pj;
            ray.direction = L;
            const HitResult h = hitBVH(sc, ray, cn, 1);
            traced_pdf[o] = (h.isHit && h.triangle == es.lt.tri[k] && emitHitPdf(sc, es, es.lt, h.triangle, h.distance, L, &pl)) ? pl : -1.0f;
        }
    }
    return K;
}

// The window [x0,x1) x [y0,y1) as oracle_render_punctual, with the emission maps of ezrt_scene_set_emission_maps (emit_id, used with
// EZRT_PARAM_EMISSION_MAPS).  Test-only inputs: lum_eff (null: the table's own, ez_emit_lum_eff) replaces each mapped emitter's lum_eff
// in the table and in every pdf, so that a test renders with other valid weights; mis_scale (1: none) scales a mapped light's lum_eff
// in the MIS weights of emission hits only
int oracle_render_emission_maps(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache, int hdrW,
                           int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, int nTex, const ezrt_texture* tex,
                           const float* uv, const int32_t* id, const int32_t* mr, const int32_t* nm, int nLights, const ezrt_punctual_light* lights,
                           const int32_t* emit_id, const float* lum_eff, float mis_scale, int x0, int y0, int x1, int y1, float* framebuffer, float* aov, float* luma2, uint64_t* counters_out, int n_threads) {
    if (!p || !tris) return -1;
    Setup su;
    int rc = punctSetup(p, m, nTex, tex, uv, id, mr, nm, tris, nTriangles, nLights, lights, &su);
    if (rc) return rc;
    if ((p->reserved[0] & EZRT_PARAM_EMISSION_MAPS) && (!(p->reserved[0] & EZRT_PARAM_TEXTURES) || !emit_id)) return -2;
    if (emit_id)
        for (int i = 0; i < nTriangles; i++)
            if (emit_id[i] < -1 || emit_id[i] >= nTex) return -2;
    ez_lens lens;
    bool on;
    rc = checkRender(tris, nTriangles, nodes, nNodes, hdr, hdrCache, p, x0, y0, x1, y1, &lens, &on);
    if (rc) return rc;
    if (!framebuffer || !luma2) return -1;
    Scene sc = makeScene(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p->env_color, p->mode, p->traverse);
    Tables tb = makeTables(sc, *p, hdr, hdrW, hdrH);
    EmitSet es;
    es.misScale = mis_scale;
    emitSetOf(sc, su.ts, (p->reserved[0] & EZRT_PARAM_EMISSION_MAPS) ? emit_id : su.none.data(), lum_eff, &es);
    if (p->reserved[0] & EZRT_PARAM_EMISSION_MAPS) tb.lt = es.lt;
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
                    const vec3 color = shadePixelEmit(sc, tb, su.ts, su.ms, su.pt, es, su.med, *p, on ? &lens : nullptr, (uint32_t)pxl, (uint32_t)py, frame,
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
int oracle_render_emission_maps_adaptive(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache,
                                    int hdrW, int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, int nTex,
                                    const ezrt_texture* tex, const float* uv, const int32_t* id, const int32_t* mr, const int32_t* nm, int nLights,
                                    const ezrt_punctual_light* lights, const int32_t* emit_id, const float* lum_eff, float mis_scale,
                                    const ezrt_adaptive_params* ap, int x0, int y0, int x1, int y1,
                                    float* framebuffer, int32_t* spp_out, float* luma2_out, uint64_t* counters_out, int n_threads) {
    if (!p || !tris) return -1;
    Setup su;
    int rc = punctSetup(p, m, nTex, tex, uv, id, mr, nm, tris, nTriangles, nLights, lights, &su);
    if (rc) return rc;
    if ((p->reserved[0] & EZRT_PARAM_EMISSION_MAPS) && (!(p->reserved[0] & EZRT_PARAM_TEXTURES) || !emit_id)) return -2;
    if (emit_id)
        for (int i = 0; i < nTriangles; i++)
            if (emit_id[i] < -1 || emit_id[i] >= nTex) return -2;
    ez_lens lens;
    bool on;
    rc = checkRender(tris, nTriangles, nodes, nNodes, hdr, hdrCache, p, x0, y0, x1, y1, &lens, &on);
    if (rc) return rc;
    if (!ap || !framebuffer || !spp_out || !luma2_out) return -1;
    if (p->first_frame != 0 || ap->min_spp < 2 || ap->check_interval < 1 || !(ap->threshold > 0.0f)) return -1;
    if (x0 % EZRT_TILE_SIZE || y0 % EZRT_TILE_SIZE || (x1 % EZRT_TILE_SIZE && x1 != p->width) || (y1 % EZRT_TILE_SIZE && y1 != p->height)) return -1;
    Scene sc = makeScene(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p->env_color, p->mode, p->traverse);
    Tables tb = makeTables(sc, *p, hdr, hdrW, hdrH);
    EmitSet es;
    es.misScale = mis_scale;
    emitSetOf(sc, su.ts, (p->reserved[0] & EZRT_PARAM_EMISSION_MAPS) ? emit_id : su.none.data(), lum_eff, &es);
    if (p->reserved[0] & EZRT_PARAM_EMISSION_MAPS) tb.lt = es.lt;
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
                        const vec3 color = shadePixelEmit(sc, tb, su.ts, su.ms, su.pt, es, su.med, *p, on ? &lens : nullptr, px, py, (uint32_t)f, cn, nullptr);
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
