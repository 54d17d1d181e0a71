// oracle_light_tree.cpp -- CPU restatement of the light tree (EZRT_PARAM_LIGHT_TREE in EZRT_MODE_DISNEY_LIGHTS, ezrt_math.h, DESIGN.md
// section 19) over the emission maps' restatement (tests/oracle_emission_maps.cpp, included unchanged).  Its two loops -- the homogeneous
// medium's (mode 4's when there is no medium) and the transmission mixture's -- are restated with the triangle light chosen by the tree's
// descent from the shading point and with both pdfs ez_ltree_pdf, the emission hit's P_sel walked from the path's previous vertex, with
// every other option.  The tree is not built here: it is ezrt_light_tree_build's output, passed in.  Plain/window, feature-buffer and
// adaptive forms.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT, like the oracle it compiles in (build/libezrt_oracle_light_tree.so, tests/oracle_light_tree.py).
//
// A render without EZRT_PARAM_LIGHT_TREE, or whose table has no light, is the emission maps' restatement's, bit for bit.
#include "oracle_emission_maps.cpp"

namespace {

// The tree of a render: the node and path records, each triangle's light index in the render's table (-1: none), and the test-only
// factor of the emission hits' P_sel
struct TreeSet {
    const float* nodes = nullptr;
    const uint32_t* paths = nullptr;
    std::vector<int> light;
    float misScale = 1.0f;
};

void treeSetOf(const Scene& sc, const LightTable& lt, const float* nodes, const uint32_t* paths, float misScale, TreeSet* tr) {
    tr->nodes = nodes;
    tr->paths = paths;
    tr->misScale = misScale;
    tr->light.assign((size_t)sc.nTriangles, -1);
    for (size_t k = 0; k < lt.tri.size(); k++) tr->light[lt.tri[k]] = (int)k;
}

// A BSDF sample from Pprev whose emission hit is at distance t along d on triangle tri: false when tri is not a light of the table, else
// the tree's pdf of the hit point
bool treeHitPdf(const Scene& sc, const TreeSet& tr, int tri, vec3 Pprev, float t, vec3 d, float* pdf) {
    const int k = tr.light[tri];
    if (k < 0) return false;
    const uint32_t* pa = tr.paths + 4 * (size_t)k;
    const float q = ez_ltree_prob(tr.nodes, Pprev, ((uint64_t)pa[1] << 32) | pa[0], (int)pa[2]) * tr.misScale;
    *pdf = ez_ltree_pdf(q, ez_u2f(pa[3]), t, ez_abs(ez_dot(geoNormal(getTriangle(sc, tri)), d)));
    return true;
}

// shadePixelEmitMedium (tests/oracle_emission_maps.cpp) with the tree tr choosing the triangle light and giving both pdfs
vec3 shadePixelTreeMedium(const Scene& sc, const Tables& tb, const TexSet& ts, const MapSet& ms, const PunctSet& pt, const EmitSet& es, const TreeSet& tr,
                           const ez_medium& med,
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
                if (treeHitPdf(sc, tr, h.triangle, ray.startPoint, h.distance, ray.direction, &pl)) {
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
            float p_sel = 0.0f;
            const int k = ez_ltree_descend(tr.nodes, P, r_tri, &p_sel);
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
                    float pdf_light = ez_ltree_pdf(p_sel, ez_triangle_area(T.p1, T.p2, T.p3), dist, cos_l);
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

// pathTracingTransEmit (tests/oracle_emission_maps.cpp) with the tree tr
vec3 pathTracingTransTree(const Scene& sc, const TexSet& ts, const MapSet& ms, const PunctSet& pt, const EmitSet& es, const TreeSet& tr, const LightTable& lt,
                           const EnvTable& env,
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
            float p_sel = 0.0f;
            const int k = ez_ltree_descend(tr.nodes, hit.hitPoint, r_tri, &p_sel);
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
                    float pdf_light = ez_ltree_pdf(p_sel, ez_triangle_area(T.p1, T.p2, T.p3), dist, cos_l) * (1.0f - P_env);
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
        if (!below && treeHitPdf(sc, tr, newHit.triangle, hit.hitPoint, newHit.distance, L, &pl)) {
            pl = (1.0f - P_env) * pl;
            w = (P_p > 0.0f) ? misMixWeight(pdf_b, (1.0f - P_p) * pl) : misMixWeight(pdf_b, pl);
        }
        Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), Le), f_r), ac), pdf_b));
        hit = newHit;
        history = ez_mul(history, ez_divs(ez_scale(f_r, ac), pdf_b));
    }
    return Lo;
}

// one sample of a light-tree render: the transmission loop with EZRT_PARAM_TRANSMISSION, the medium loop otherwise
vec3 shadePixelTree(const Scene& sc, const Tables& tb, const TexSet& ts, const MapSet& ms, const PunctSet& pt, const EmitSet& es, const TreeSet& tr,
                    const ez_medium& med,
                    const ezrt_render_params& p, const ez_lens* lens, uint32_t ipx, uint32_t ipy, uint32_t frameCounter, Counters& cn, First* first) {
    if (!(p.reserved[0] & EZRT_PARAM_TRANSMISSION)) return shadePixelTreeMedium(sc, tb, ts, ms, pt, es, tr, med, p, lens, ipx, ipy, frameCounter, cn, first);
    PixelCtx px;
    px.px = ipx; px.py = ipy; px.frameCounter = frameCounter;
    const Ray ray = cameraRay(p, lens, px);
    const HitResult firstHit = hitBVH(sc, ray, cn, 0);
    firstOf(sc, ts, ms, firstHit, first);
    if (!firstHit.isHit) return hdrColor(sc, ray.direction, cn);
    bool mapped;
    return ez_add(emitAt(sc, ts, es, firstHit.triangle, firstHit.hitPoint, &mapped),
                  pathTracingTransTree(sc, ts, ms, pt, es, tr, tb.lt, tb.env, firstHit, p.max_bounce, px, cn));
}


}  // namespace

extern "C" {

// The inputs of ezrt_light_tree_build for the render's table: mode 4's (emit_id null) or the emission table of emit_id over the textures
// (tex, uv).  Returns K, writing min(K, cap) lights' vertices (9 floats) into verts_out and table weights into w_out; -2 where
// ezrt_scene_set_emission_maps returns EZRT_ERR_INVALID
int oracle_light_tree_table(const float* tris, int nTriangles, const float* nodes, int nNodes, int nTex, const ezrt_texture* tex, const float* uv,
                            const int32_t* emit_id, int cap, float* verts_out, float* w_out) {
    std::vector<int32_t> none((size_t)nTriangles, -1);
    TexSet ts;
    if (emit_id) {
        if (!texSetOf(nTex, tex, uv, none.data(), nTriangles, &ts)) return -2;
        for (int i = 0; i < nTriangles; i++)
            if (emit_id[i] < -1 || emit_id[i] >= nTex) return -2;
    }
    const Scene sc = makeScene(tris, nTriangles, nodes, nNodes, nullptr, nullptr, 0, 0, 0, nullptr, EZRT_MODE_DISNEY_LIGHTS, EZRT_TRAVERSE_ACCEL);
    EmitSet es;
    emitSetOf(sc, ts, emit_id ? emit_id : none.data(), nullptr, &es);
    const int K = (int)es.lt.tri.size();
    for (int k = 0; k < K && k < cap; k++) {
        const int t = es.lt.tri[k];
        const Triangle T = getTriangle(sc, t);
        const vec3 v[3] = {T.p1, T.p2, T.p3};
        for (int j = 0; j < 3; j++) {
            verts_out[9 * (size_t)k + 3 * j] = v[j].x; verts_out[9 * (size_t)k + 3 * j + 1] = v[j].y; verts_out[9 * (size_t)k + 3 * j + 2] = v[j].z;
        }
        w_out[k] = emitMapped(sc, es, t) ? ez_triangle_area(T.p1, T.p2, T.p3) * es.lumEff[t] : ez_light_weight(T.p1, T.p2, T.p3, getMaterial(sc, t).emissive);
    }
    return K;
}

// ezrt_math.h's descent (which 0: (P, r) -> (light, P_sel), -1 and 0 for no sample) and hit-side walk (which 1: (P, light) -> P_sel) over
// the tree records on n inputs
void oracle_light_tree_eval(const float* nodes, const uint32_t* paths, int which, int n, const float* P, const float* r, const int32_t* light_in,
                            int32_t* light_out, float* p_out) {
    for (int i = 0; i < n; i++) {
        const vec3 Pi = ez_v3(P[3 * (size_t)i], P[3 * (size_t)i + 1], P[3 * (size_t)i + 2]);
        if (which == 0) {
            float q = 0.0f;
            light_out[i] = ez_ltree_descend(nodes, Pi, r[i], &q);
            p_out[i] = q;
        } else {
            const uint32_t* pa = paths + 4 * (size_t)light_in[i];
            p_out[i] = ez_ltree_prob(nodes, Pi, ((uint64_t)pa[1] << 32) | pa[0], (int)pa[2]);
        }
    }
}

// The window [x0,x1) x [y0,y1) as oracle_render_emission_maps, with EZRT_PARAM_LIGHT_TREE rendered by the tree (tree_nodes, tree_paths:
// ezrt_light_tree_build's output over the render's table, oracle_light_tree_table; unused without the flag or lights).  Test-only
// input: mis_scale (1: none) scales the P_sel of the emission hits' MIS pdfs only
int oracle_render_light_tree(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache, int hdrW,
                           int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, int nTex, const ezrt_texture* tex,
                           const float* uv, const int32_t* id, const int32_t* mr, const int32_t* nm, int nLights, const ezrt_punctual_light* lights,
                           const int32_t* emit_id, const float* tree_nodes, const uint32_t* tree_paths, float mis_scale, int x0, int y0, int x1, int y1, float* framebuffer,
                             float* aov, float* luma2, uint64_t* counters_out, int n_threads) {
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
    emitSetOf(sc, su.ts, (p->reserved[0] & EZRT_PARAM_EMISSION_MAPS) ? emit_id : su.none.data(), nullptr, &es);
    if (p->reserved[0] & EZRT_PARAM_EMISSION_MAPS) tb.lt = es.lt;
    const bool treeOn = (p->reserved[0] & EZRT_PARAM_LIGHT_TREE) && !tb.lt.tri.empty();
    if (treeOn && (!tree_nodes || !tree_paths)) return -1;
    TreeSet tr;
    treeSetOf(sc, tb.lt, tree_nodes, tree_paths, mis_scale, &tr);
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
                    const vec3 color = treeOn ? shadePixelTree(sc, tb, su.ts, su.ms, su.pt, es, tr, su.med, *p, on ? &lens : nullptr, (uint32_t)pxl, (uint32_t)py,
                                                                      frame, cn, &f)
                                               : shadePixelEmit(sc, tb, su.ts, su.ms, su.pt, es, su.med, *p, on ? &lens : nullptr, (uint32_t)pxl, (uint32_t)py, frame,
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
int oracle_render_light_tree_adaptive(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache,
                                    int hdrW, int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, int nTex,
                                    const ezrt_texture* tex, const float* uv, const int32_t* id, const int32_t* mr, const int32_t* nm, int nLights,
                                    const ezrt_punctual_light* lights, const int32_t* emit_id, const float* tree_nodes, const uint32_t* tree_paths, float mis_scale,
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
    emitSetOf(sc, su.ts, (p->reserved[0] & EZRT_PARAM_EMISSION_MAPS) ? emit_id : su.none.data(), nullptr, &es);
    if (p->reserved[0] & EZRT_PARAM_EMISSION_MAPS) tb.lt = es.lt;
    const bool treeOn = (p->reserved[0] & EZRT_PARAM_LIGHT_TREE) && !tb.lt.tri.empty();
    if (treeOn && (!tree_nodes || !tree_paths)) return -1;
    TreeSet tr;
    treeSetOf(sc, tb.lt, tree_nodes, tree_paths, mis_scale, &tr);
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
                        const vec3 color = treeOn ? shadePixelTree(sc, tb, su.ts, su.ms, su.pt, es, tr, su.med, *p, on ? &lens : nullptr, px, py, (uint32_t)f, cn, nullptr)
                                                   : shadePixelEmit(sc, tb, su.ts, su.ms, su.pt, es, su.med, *p, on ? &lens : nullptr, px, py, (uint32_t)f, cn, nullptr);
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
