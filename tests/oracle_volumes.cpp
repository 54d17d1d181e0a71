// oracle_volumes.cpp -- CPU restatement of the volumes inside transmissive meshes (EZRT_PARAM_VOLUMES in EZRT_MODE_DISNEY_LIGHTS with
// EZRT_PARAM_TRANSMISSION, ezrt_math.h, DESIGN.md section 21) over the density grid's restatement (tests/oracle_medium_grid.cpp, and
// through it the light tree's, emission maps', punctual lights', material maps', textures', lens' and transmission's, included
// unchanged).  One sample function for the flag: the transmission loop of tests/oracle_light_tree.cpp and tests/oracle_emission_maps.cpp
// (the triangle light chosen by the light tree or by the table, with every other option), with the absorption of every interior segment
// -- the camera ray's and the BSDF samples' -- applied to the path's history, and at the camera ray's hit to its emission, before the
// hit is shaded.  Plain/window, feature-buffer and adaptive forms.
//
// With EZRT_PARAM_MEDIUM too (sigma_t > 0), a second sample function: the medium loop with the mixture at surfaces, in which an interior
// segment draws no free flight, through the homogeneous medium or the density grid of oracle_grid_render_set.
//
// test_flags (switches of the restatement only): 1, no light samples, and every emission and environment hit of a BSDF sample weighs 1
// -- an independent estimator of the same integral, for the unbiasedness tests; 2, a mutation: the first BSDF sample's hit is not
// absorbed; 4, a mutation: interior segments draw the medium's free flight (the analytic checks must fail with either).
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT (build/libezrt_oracle_volumes.so, tests/oracle_volumes.py).
//
// A render without EZRT_PARAM_VOLUMES is the light tree's restatement's, bit for bit.
#include "oracle_medium_grid.cpp"

namespace {

// The volumes of a render: sigma_a (3 floats per volume) and each triangle's volume id (-1: none); on false: no volumes (every interior
// clear)
struct VolSet {
    bool on = false;
    const float* sigma = nullptr;
    const int32_t* id = nullptr;
};

// The absorption of the traced segment that ends at h: true with T = exp(-sigma_a t) per channel when h ends an interior segment
// (a hit from inside on a triangle whose material record has a dielectric weight > 0) on a triangle with a volume
bool volAbsorb(const Scene& sc, const VolSet& vs, const HitResult& h, vec3* T) {
    if (!vs.on || !h.isHit || !h.isInside) return false;
    const int v = vs.id[h.triangle];
    if (v < 0) return false;
    const Material m = getMaterial(sc, h.triangle);
    if (!(ez_trans_weight(m.transmission, m.metallic, m.IOR) > 0.0f)) return false;
    const float* s = vs.sigma + 3 * (size_t)v;
    *T = ez_v3(ez_volume_transmittance(s[0], h.distance), ez_volume_transmittance(s[1], h.distance), ez_volume_transmittance(s[2], h.distance));
    return true;
}

// The transmission loop from the camera ray's hit `hit` with the history `history` (its absorption applied): the triangle light
// sample chosen by the tree tr (treeOn) or by the table lt, every BSDF sample's hit absorbed before its emission is added
vec3 pathTracingTransVol(const Scene& sc, const TexSet& ts, const MapSet& ms, const PunctSet& pt, const EmitSet& es, const TreeSet& tr, bool treeOn,
                         const LightTable& lt, const EnvTable& env, const VolSet& vs, HitResult hit, vec3 history, int maxBounce, PixelCtx& px,
                         Counters& cn, bool bsdfOnly, bool mutate) {
    vec3 Lo = splat(0);
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
        if (bsdfOnly) {
        } else if (punct) {
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
            float p_sel = 0.0f;
            const int k = treeOn ? ez_ltree_descend(tr.nodes, hit.hitPoint, r_tri, &p_sel) : ez_light_select(lt.cdf.data(), K, r_tri);
            const int tk = lt.tri[k < 0 ? 0 : k];
            const Triangle T = getTriangle(sc, tk);
            const vec3 E = emitLight(sc, ts, es, tk, r_1, r_2);
            const vec3 D = ez_sub(ez_triangle_point(T.p1, T.p2, T.p3, r_1, r_2), hit.hitPoint);
            const float dist = EZ_SQRT(ez_dot(D, D));
            const vec3 Ll = ez_normalize(D);
            const float cos_l = ez_abs(ez_dot(geoNormal(T), Ll));
            if (k >= 0 && tk != hit.triangle && ez_dot(N, Ll) > 0.0f && cos_l != 0.0f && dist != 0.0f && !emitBlack(E)) {
                Ray sray;
                sray.startPoint = hit.hitPoint;
                sray.direction = Ll;
                if (!occludedBounded(sc, sray, ez_light_tmax(dist), cn)) {
                    float pdf_light = (treeOn ? ez_ltree_pdf(p_sel, ez_triangle_area(T.p1, T.p2, T.p3), dist, cos_l) : emitSamplePdf(sc, es, lt, k, dist, Ll)) *
                                      (1.0f - P_env);
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
            if (P_env > 0.0f && !below && !bsdfOnly) {
                const float pe = P_env * ez_env_pdf(env.pdf.data(), env.W, env.H, L);
                w = (P_p > 0.0f) ? misMixWeight(pdf_b, (1.0f - P_p) * pe) : misMixWeight(pdf_b, pe);
            }
            Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), hdrColor(sc, L, cn)), f_r), ac), pdf_b));
            break;
        }
        vec3 T_vol;
        if (!(mutate && bounce == 0) && volAbsorb(sc, vs, newHit, &T_vol)) history = ez_mul(history, T_vol);   // before newHit is shaded
        bool mapped;
        const vec3 Le = emitAt(sc, ts, es, newHit.triangle, newHit.hitPoint, &mapped);
        float w = 1.0f, pl;
        if (!below && !bsdfOnly &&
            (treeOn ? treeHitPdf(sc, tr, newHit.triangle, hit.hitPoint, newHit.distance, L, &pl) : emitHitPdf(sc, es, lt, newHit.triangle, newHit.distance, L, &pl))) {
            pl = (1.0f - P_env) * pl;
            w = (P_p > 0.0f) ? misMixWeight(pdf_b, (1.0f - P_p) * pl) : misMixWeight(pdf_b, pl);
        }
        Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), Le), f_r), ac), pdf_b));
        hit = newHit;
        history = ez_mul(history, ez_divs(ez_scale(f_r, ac), pdf_b));
    }
    return Lo;
}

// The segment that ends at h is an interior one (a hit from inside on a triangle whose material record has a dielectric weight > 0),
// whatever its volume id
bool volInterior(const Scene& sc, const HitResult& h) {
    if (!h.isHit || !h.isInside) return false;
    const Material m = getMaterial(sc, h.triangle);
    return ez_trans_weight(m.transmission, m.metallic, m.IOR) > 0.0f;
}

// An interior segment draws no free flight; the grid's shadow streams still count it as one of the path's segments (gridFlightHook's
// bookkeeping, tests/oracle_medium_grid.cpp), so that they stay keyed on the bounce
void volSkipFlight(const PixelCtx& px) {
    if (!g_render_grid) return;
    if (t_path.gen != g_render_gen || t_path.px != px.px || t_path.py != px.py || t_path.frame != px.frameCounter) {
        t_path.gen = g_render_gen; t_path.px = px.px; t_path.py = px.py; t_path.frame = px.frameCounter;
        t_path.bounce = 0;
    } else {
        t_path.bounce++;
    }
}

// The medium loop of tests/oracle_light_tree.cpp and tests/oracle_emission_maps.cpp (the triangle light chosen by the tree tr or by the
// table) with the transmission mixture at surfaces, for EZRT_PARAM_VOLUMES with EZRT_PARAM_MEDIUM: an interior segment draws no free
// flight (the glass displaces the medium) and is absorbed at its hit before that hit is shaded; every other segment draws its flight as
// sections 14 and 20 define it (through the grid set by oracle_grid_render_set, else the homogeneous medium).  Light samples are
// TRANS's at surfaces and the phase function's at medium vertices, times their shadow ray's transmittance.  The weights of a path
// segment take |cos|.  bsdfOnly: no light samples, every emission and environment hit weighs 1; mutateFlight: interior segments draw
// their flight too (a mutation).
vec3 shadePixelVolMedium(const Scene& sc, const Tables& tb, const TexSet& ts, const MapSet& ms, const PunctSet& pt, const EmitSet& es, const TreeSet& tr,
                         bool treeOn, const ez_medium& med, const VolSet& vs, const ezrt_render_params& p, const ez_lens* lens, uint32_t ipx,
                         uint32_t ipy, uint32_t frameCounter, Counters& cn, First* first, bool bsdfOnly, bool mutateFlight) {
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
        const bool below = cosine < 0.0f;   // the previous BSDF sample went below its surface: no light strategy reaches it
        const float ac = ez_abs(cosine);
        float t_s;
        const float t_end = h.isHit ? h.distance : ez_u2f(0x7f800000u);
        bool scatter = false;
        if (volInterior(sc, h) && !mutateFlight) volSkipFlight(px);
        else scatter = gridFlightHook(&med, ray.startPoint, ray.direction, t_end, &px.rng.seed, &t_s) != 0;
        if (!scatter && !h.isHit) {
            if (bounce == 0) return hdrColor(sc, ray.direction, cn);
            float w = 1.0f;
            if (P_env > 0.0f && !below && !bsdfOnly) {
                const float pe = P_env * ez_env_pdf(tb.env.pdf.data(), tb.env.W, tb.env.H, ray.direction);
                w = (P_p > 0.0f) ? misMixWeight(pdf, (1.0f - P_p) * pe) : misMixWeight(pdf, pe);
            }
            Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), hdrColor(sc, ray.direction, cn)), f_r), ac), pdf));
            break;
        }
        if (!scatter) {
            vec3 T_vol;
            const bool absorbed = volAbsorb(sc, vs, h, &T_vol);
            if (absorbed) history = ez_mul(history, T_vol);
            bool mapped;
            const vec3 E = emitAt(sc, ts, es, h.triangle, h.hitPoint, &mapped);
            if (bounce == 0) {
                Le = absorbed ? ez_mul(E, T_vol) : E;
            } else {
                float w = 1.0f, pl;
                if (!below && !bsdfOnly &&
                    (treeOn ? treeHitPdf(sc, tr, h.triangle, ray.startPoint, h.distance, ray.direction, &pl)
                            : emitHitPdf(sc, es, tb.lt, h.triangle, h.distance, ray.direction, &pl))) {
                    if (envOn) pl = (1.0f - P_env) * pl;
                    w = (P_p > 0.0f) ? misMixWeight(pdf, (1.0f - P_p) * pl) : misMixWeight(pdf, pl);
                }
                Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), E), f_r), ac), pdf));
                history = ez_mul(history, ez_divs(ez_scale(f_r, ac), pdf));
            }
        } else {
            if (bounce > 0) history = ez_mul(history, ez_divs(ez_scale(f_r, ac), pdf));
            history = ez_mul(history, med.albedo);
        }
        if (bounce >= p.max_bounce) break;
        const vec3 P = scatter ? ez_add(ray.startPoint, ez_scale(ray.direction, t_s)) : h.hitPoint;
        const vec3 d = ray.direction;
        const vec3 Vv = ez_neg(h.viewDir);
        vec3 N = h.normal;
        Material material = scatter ? Material() : getMaterial(sc, h.triangle);
        if (!scatter) mapMaterial(sc, ts, ms, h.triangle, h.hitPoint, Vv, h.isInside, &material, &N);
        const TransLobe tl = scatter ? TransLobe() : transLobe(material, h.isInside);
        const float r_sel = px.rng.rand();
        const float r_1 = px.rng.rand();
        const float r_2 = px.rng.rand();
        float r_p = 0.0f, r_env;
        const bool punct = punctPick(P_p, r_sel, &r_p, &r_env);
        const bool envPick = !punct && ((P_env == 1.0f) || (P_env == 0.5f && r_env < 0.5f));
        const float r_tri = (P_env == 0.5f) ? (r_env - 0.5f) * 2.0f : r_env;
        // a lit light sample's value at P: the phase function's at a medium vertex, the mixture's at a surface
        const auto contrib = [&](vec3 Ll, vec3 E, float pdf_light) {
            return scatter ? mediumLightContrib(history, true, d, Vv, N, Ll, material, med.g, E, pdf_light)
                           : lightContrib(history, Vv, N, Ll, material, tl, E, pdf_light);
        };
        if (bsdfOnly) {
        } else if (punct) {
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
                        float pdf_unused;
                        f = (tl.t == 0.0f) ? BRDF_Evaluate(Vv, N, Ll, splat(0), splat(0), material, false) : BSDF_Evaluate(Vv, N, Ll, material, tl, &pdf_unused);
                        cl = ez_dot(N, Ll);
                    }
                    const vec3 c = ez_punct_contrib(history, f, cl, ez_v3(rec[8], rec[9], rec[10]), s);
                    Lo = ez_add(Lo, ez_scale(c, gridTransmittanceHook(&med, P, Ll, ez_medium_light_dist(tmax, rec[3] == 2.0f))));
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
                    const vec3 c = contrib(Ld, hdrColor(sc, Ld, cn), pl);
                    Lo = ez_add(Lo, ez_scale(c, gridTransmittanceHook(&med, P, Ld, ez_medium_light_dist(EZ_INF, 1))));
                }
            }
        } else if (K > 0) {
            float p_sel = 0.0f;
            const int k = treeOn ? ez_ltree_descend(tr.nodes, P, r_tri, &p_sel) : ez_light_select(tb.lt.cdf.data(), K, r_tri);
            const int tk = tb.lt.tri[k < 0 ? 0 : k];
            const Triangle T = getTriangle(sc, tk);
            const vec3 E = emitLight(sc, ts, es, tk, r_1, r_2);
            const vec3 D = ez_sub(ez_triangle_point(T.p1, T.p2, T.p3, r_1, r_2), P);
            const float dist = EZ_SQRT(ez_dot(D, D));
            const vec3 Ll = ez_normalize(D);
            const float cos_l = ez_abs(ez_dot(geoNormal(T), Ll));
            if (k >= 0 && (scatter || (tk != h.triangle && ez_dot(N, Ll) > 0.0f)) && cos_l != 0.0f && dist != 0.0f && !emitBlack(E)) {
                Ray sray;
                sray.startPoint = P;
                sray.direction = Ll;
                const float tmax = ez_light_tmax(dist);
                if (!occludedBounded(sc, sray, tmax, cn)) {
                    float pdf_light = treeOn ? ez_ltree_pdf(p_sel, ez_triangle_area(T.p1, T.p2, T.p3), dist, cos_l) : emitSamplePdf(sc, es, tb.lt, k, dist, Ll);
                    if (envOn) pdf_light = pdf_light * (1.0f - P_env);
                    if (P_p > 0.0f) pdf_light = pdf_light * (1.0f - P_p);
                    Lo = ez_add(Lo, ez_scale(contrib(Ll, E, pdf_light), gridTransmittanceHook(&med, P, Ll, ez_medium_light_dist(tmax, 0))));
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
            if (tl.t == 0.0f) {   // mode 4's sample
                cosine = ez_dot(N, L);
                if (cosine <= 0.0f) break;
                f_r = BRDF_Evaluate(Vv, N, L, splat(0), splat(0), material, false);
                pdf = BRDF_Pdf(Vv, N, L, material);
            } else {
                const float r_t = px.rng.rand();
                if (!SampleBSDF(xi_1, xi_2, xi_3, r_t, Vv, N, material, tl, &L, &f_r, &pdf, &cosine)) break;
            }
        }
        ray.startPoint = P;
        ray.direction = L;
    }
    return ez_add(Le, Lo);
}

// one sample of a render: with EZRT_PARAM_VOLUMES the transmission loop with the absorption (the camera ray's hit absorbed first: its
// history and its emission), or with the medium (sigma_t > 0) the medium loop above; the light tree's restatement otherwise
vec3 shadePixelVol(const Scene& sc, const Tables& tb, const TexSet& ts, const MapSet& ms, const PunctSet& pt, const EmitSet& es, const TreeSet& tr,
                   bool treeOn, const ez_medium& med, const VolSet& vs, const ezrt_render_params& p, const ez_lens* lens, uint32_t ipx, uint32_t ipy,
                   uint32_t frameCounter, Counters& cn, First* first, int testFlags) {
    if (!(p.reserved[0] & EZRT_PARAM_VOLUMES))
        return treeOn ? shadePixelTree(sc, tb, ts, ms, pt, es, tr, med, p, lens, ipx, ipy, frameCounter, cn, first)
                      : shadePixelEmit(sc, tb, ts, ms, pt, es, med, p, lens, ipx, ipy, frameCounter, cn, first);
    if ((p.reserved[0] & EZRT_PARAM_MEDIUM) && med.sigma_t > 0.0f)
        return shadePixelVolMedium(sc, tb, ts, ms, pt, es, tr, treeOn, med, vs, p, lens, ipx, ipy, frameCounter, cn, first, (testFlags & 1) != 0,
                                   (testFlags & 4) != 0);
    PixelCtx px;
    px.px = ipx; px.py = ipy; px.frameCounter = frameCounter;
    const Ray ray = cameraRay(p, lens, px);
    const HitResult firstHit = hitBVH(sc, ray, cn, 0);
    firstOf(sc, ts, ms, firstHit, first);
    if (!firstHit.isHit) return hdrColor(sc, ray.direction, cn);
    vec3 history = splat(1);
    bool mapped;
    vec3 Le = emitAt(sc, ts, es, firstHit.triangle, firstHit.hitPoint, &mapped);
    vec3 T_vol;
    if (volAbsorb(sc, vs, firstHit, &T_vol)) {
        history = ez_mul(history, T_vol);
        Le = ez_mul(Le, T_vol);
    }
    return ez_add(Le, pathTracingTransVol(sc, ts, ms, pt, es, tr, treeOn, tb.lt, tb.env, vs, firstHit, history, p.max_bounce, px, cn, (testFlags & 1) != 0,
                                             (testFlags & 2) != 0));
}

// The checks and tables every entry point shares; -2 where the library returns EZRT_ERR_INVALID
struct VolRender {
    Setup su;
    ez_lens lens;
    bool lensOn = false;
    Scene sc;
    Tables tb;
    EmitSet es;
    TreeSet tr;
    bool treeOn = false;
    VolSet vs;
};

int volRenderOf(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache, int hdrW, int hdrH,
                int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, int nTex, const ezrt_texture* tex, const float* uv, const int32_t* id,
                const int32_t* mr, const int32_t* nm, int nLights, const ezrt_punctual_light* lights, const int32_t* emit_id, const float* tree_nodes,
                const uint32_t* tree_paths, float mis_scale, int n_vol, const float* vol_sigma, const int32_t* vol_id, int x0, int y0, int x1, int y1,
                VolRender* r) {
    if (!p || !tris) return -1;
    // the medium beside transmission is rendered with the volumes only; punctSetup (the restatements without them) rejects it
    ezrt_render_params ps = *p;
    if ((p->reserved[0] & EZRT_PARAM_VOLUMES) && (p->reserved[0] & EZRT_PARAM_MEDIUM)) ps.reserved[0] &= ~EZRT_PARAM_TRANSMISSION;
    int rc = punctSetup(&ps, m, nTex, tex, uv, id, mr, nm, tris, nTriangles, nLights, lights, &r->su);
    if (rc) return rc;
    if ((p->reserved[0] & EZRT_PARAM_VOLUMES) && !(p->reserved[0] & EZRT_PARAM_TRANSMISSION)) return -2;
    if ((p->reserved[0] & EZRT_PARAM_EMISSION_MAPS) && (!(p->reserved[0] & EZRT_PARAM_TEXTURES) || !emit_id)) return -2;
    if (emit_id)
        for (int i = 0; i < nTriangles; i++)
            if (emit_id[i] < -1 || emit_id[i] >= nTex) return -2;
    if (n_vol > 0) {
        if (!vol_sigma || !vol_id) return -1;
        for (int i = 0; i < nTriangles; i++)
            if (vol_id[i] < -1 || vol_id[i] >= n_vol) return -2;
        r->vs.on = true;
        r->vs.sigma = vol_sigma;
        r->vs.id = vol_id;
    }
    rc = checkRender(tris, nTriangles, nodes, nNodes, hdr, hdrCache, p, x0, y0, x1, y1, &r->lens, &r->lensOn);
    if (rc) return rc;
    r->sc = makeScene(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p->env_color, p->mode, p->traverse);
    r->tb = makeTables(r->sc, *p, hdr, hdrW, hdrH);
    emitSetOf(r->sc, r->su.ts, (p->reserved[0] & EZRT_PARAM_EMISSION_MAPS) ? emit_id : r->su.none.data(), nullptr, &r->es);
    if (p->reserved[0] & EZRT_PARAM_EMISSION_MAPS) r->tb.lt = r->es.lt;
    r->treeOn = (p->reserved[0] & EZRT_PARAM_LIGHT_TREE) && !r->tb.lt.tri.empty();
    if (r->treeOn && (!tree_nodes || !tree_paths)) return -1;
    treeSetOf(r->sc, r->tb.lt, tree_nodes, tree_paths, mis_scale, &r->tr);
    return 0;
}

}  // namespace

extern "C" {

// ez_volume_sigma_a of n (colour channel, distance) pairs
void oracle_volume_sigma_a(int n, const float* c, const float* d, float* out) {
    for (int i = 0; i < n; i++) out[i] = ez_volume_sigma_a(c[i], d[i]);
}

// The window [x0,x1) x [y0,y1) as oracle_render_light_tree, with EZRT_PARAM_VOLUMES rendered by the n_vol volumes' sigma_a (vol_sigma,
// 3 floats each) and the triangles' ids vol_id (n_vol 0: no volumes).  test_flags: the restatement's switches (1: the independent
// estimator, 2: the mutation)
int oracle_render_volumes(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache, int hdrW,
                          int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, int nTex, const ezrt_texture* tex,
                          const float* uv, const int32_t* id, const int32_t* mr, const int32_t* nm, int nLights, const ezrt_punctual_light* lights,
                          const int32_t* emit_id, const float* tree_nodes, const uint32_t* tree_paths, float mis_scale, int n_vol,
                          const float* vol_sigma, const int32_t* vol_id, int test_flags, int x0, int y0, int x1, int y1, float* framebuffer,
                          float* aov, float* luma2, uint64_t* counters_out, int n_threads) {
    VolRender r;
    int rc = volRenderOf(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p, m, nTex, tex, uv, id, mr, nm, nLights, lights,
                         emit_id, tree_nodes, tree_paths, mis_scale, n_vol, vol_sigma, vol_id, x0, y0, x1, y1, &r);
    if (rc) return rc;
    if (!framebuffer || !luma2) return -1;
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
                    const vec3 color = shadePixelVol(r.sc, r.tb, r.su.ts, r.su.ms, r.su.pt, r.es, r.tr, r.treeOn, r.su.med, r.vs, *p, r.lensOn ? &r.lens : nullptr,
                                                     (uint32_t)pxl, (uint32_t)py, frame, cn, &f, test_flags);
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

// The adaptive form (tests/oracle_light_tree.cpp's loop with this file's sample function)
int oracle_render_volumes_adaptive(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache,
                                   int hdrW, int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, int nTex,
                                   const ezrt_texture* tex, const float* uv, const int32_t* id, const int32_t* mr, const int32_t* nm, int nLights,
                                   const ezrt_punctual_light* lights, const int32_t* emit_id, const float* tree_nodes, const uint32_t* tree_paths,
                                   float mis_scale, int n_vol, const float* vol_sigma, const int32_t* vol_id, const ezrt_adaptive_params* ap, int x0,
                                   int y0, int x1, int y1, float* framebuffer, int32_t* spp_out, float* luma2_out, uint64_t* counters_out, int n_threads) {
    VolRender r;
    int rc = volRenderOf(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p, m, nTex, tex, uv, id, mr, nm, nLights, lights,
                         emit_id, tree_nodes, tree_paths, mis_scale, n_vol, vol_sigma, vol_id, x0, y0, x1, y1, &r);
    if (rc) return rc;
    if (!ap || !framebuffer || !spp_out || !luma2_out) return -1;
    if (p->first_frame != 0 || ap->min_spp < 2 || ap->check_interval < 1 || !(ap->threshold > 0.0f)) return -1;
    if (x0 % EZRT_TILE_SIZE || y0 % EZRT_TILE_SIZE || (x1 % EZRT_TILE_SIZE && x1 != p->width) || (y1 % EZRT_TILE_SIZE && y1 != p->height)) return -1;
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
                        const vec3 color = shadePixelVol(r.sc, r.tb, r.su.ts, r.su.ms, r.su.pt, r.es, r.tr, r.treeOn, r.su.med, r.vs, *p,
                                                         r.lensOn ? &r.lens : nullptr, px, py, (uint32_t)f, cn, nullptr, 0);
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
