// oracle_material_maps.cpp -- CPU restatement of the material maps (EZRT_PARAM_MATERIAL_MAPS with EZRT_PARAM_TEXTURES in
// EZRT_MODE_DISNEY_LIGHTS, ezrt_math.h, DESIGN.md section 16): the metallic-roughness map and the tangent-space normal map at every
// surface hit but the last vertex, over the base-colour textures' restatement (tests/oracle_textures.cpp, included unchanged).  Two
// loops: the homogeneous medium's (mode 4's when there is no medium) and the transmission mixture's (tests/oracle_transmission.cpp's
// pathTracingTrans), each with the mapped material and normal, the environment light and the thin lens.  Plain/window,
// feature-buffer and adaptive forms; and the definition's functions (the table, the tangent frame, the mapped normal, the maps'
// filter) for the CPU tests.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT, like the oracle it compiles in (build/libezrt_oracle_material_maps.so,
// tests/oracle_material_maps.py).
#include "oracle_textures.cpp"

namespace {

struct MapSet {
    const int32_t* mr = nullptr;       // per triangle: the metallic-roughness map's texture id, -1: none
    const int32_t* normal = nullptr;   // ... the normal map's
};

bool mapSetOf(const int32_t* mr, const int32_t* nm, int nTex, int nTriangles, MapSet* out) {
    if (!mr || !nm) return false;
    for (int i = 0; i < nTriangles; i++)
        if (mr[i] < -1 || mr[i] >= nTex || mr[i] >= 65535 || nm[i] < -1 || nm[i] >= nTex || nm[i] >= 65535) return false;
    out->mr = mr;
    out->normal = nm;
    return true;
}

// The lookup of a hit on triangle tri at P with shading normal *N (hit from `inside`, viewed from V): the textured base colour, the
// metallic-roughness map's roughness and metallic, the normal map's normal -- tex_material's order
void mapMaterial(const Scene& sc, const TexSet& ts, const MapSet& ms, int tri, vec3 P, vec3 V, bool inside, Material* m, vec3* N,
                 float* uv_out = nullptr) {
    const Triangle T = getTriangle(sc, tri);
    const float* uv6 = ts.uv + 6 * (size_t)tri;
    float w1, w2, w3, u, v;
    ez_tri_bary(P, T.p1, T.p2, T.p3, geoNormal(T), &w1, &w2, &w3);
    ez_tex_uv(w1, w2, w3, uv6, &u, &v);
    if (uv_out) { uv_out[0] = u; uv_out[1] = v; }
    const int k = ts.id[tri];
    if (k >= 0) m->baseColor = ez_mul(m->baseColor, ez_tex_sample(ts.texels.data() + ts.off[k], ts.W[k], ts.H[k], u, v, ez_srgb_table));
    const int a = ms.mr[tri], b = ms.normal[tri];
    if (a >= 0) ez_mr_apply(ez_tex_sample(ts.texels.data() + ts.off[a], ts.W[a], ts.H[a], u, v, ez_unorm8_table), &m->roughness, &m->metallic);
    if (b >= 0) {
        const vec3 f = ez_tex_sample(ts.texels.data() + ts.off[b], ts.W[b], ts.H[b], u, v, ez_unorm8_table);
        *N = ez_normal_map(T.p1, T.p2, T.p3, uv6, u, v, f, *N, inside ? 1 : 0, V);
    }
}

// the first hit's feature record: the mapped albedo and normal
struct First {
    HitResult h;
    vec3 albedo, normal;
};

void firstOf(const Scene& sc, const TexSet& ts, const MapSet& ms, const HitResult& h, First* first) {
    if (!first) return;
    first->h = h;
    if (!h.isHit) return;
    Material m = getMaterial(sc, h.triangle);
    vec3 N = h.normal;
    mapMaterial(sc, ts, ms, h.triangle, h.hitPoint, ez_neg(h.viewDir), h.isInside, &m, &N);
    first->albedo = m.baseColor;
    first->normal = N;
}

// shadePixelTex (tests/oracle_textures.cpp) with the mapped material and normal at every surface vertex
vec3 shadePixelMapsMedium(const Scene& sc, const Tables& tb, const TexSet& ts, const MapSet& ms, const ez_medium& med, const ezrt_render_params& p,
                          const ez_lens* lens, uint32_t ipx, uint32_t ipy, uint32_t frameCounter, Counters& cn, First* first) {
    PixelCtx px;
    px.px = ipx; px.py = ipy; px.frameCounter = frameCounter;
    Ray ray = cameraRay(p, lens, px);
    const bool envOn = (p.reserved[0] & EZRT_PARAM_ENV_LIGHT) && tb.env.ok;
    const int K = (int)tb.lt.tri.size();
    const float P_env = envOn ? (K > 0 ? 0.5f : 1.0f) : 0.0f;
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
            const float w = (P_env > 0.0f) ? misMixWeight(pdf, P_env * ez_env_pdf(tb.env.pdf.data(), tb.env.W, tb.env.H, ray.direction)) : 1.0f;
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
                        const float pl = ez_light_pdf(lum, tb.lt.total_f, h.distance, ez_abs(ez_dot(geoNormal(T), ray.direction)));
                        w = envOn ? misMixWeight(pdf, (1.0f - P_env) * pl) : misMixWeight(pdf, pl);
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
        const bool envPick = (P_env == 1.0f) || (P_env == 0.5f && r_sel < 0.5f);
        const float r_tri = (P_env == 0.5f) ? (r_sel - 0.5f) * 2.0f : r_sel;
        if (envPick) {
            int texel;
            const vec3 Ld = ez_env_sample(tb.env.row.data(), tb.env.col.data(), tb.env.W, tb.env.H, r_1, r_2, &texel);
            const float pdf_env = P_env * ez_env_pdf(tb.env.pdf.data(), tb.env.W, tb.env.H, Ld);
            if (ez_finite(pdf_env) && pdf_env > 0.0f && (scatter || ez_dot(N, Ld) > 0.0f)) {
                Ray sray;
                sray.startPoint = P;
                sray.direction = Ld;
                if (!occludedBounded(sc, sray, EZ_INF, cn)) {
                    const vec3 c = mediumLightContrib(history, scatter, d, Vv, N, Ld, material, med.g, hdrColor(sc, Ld, cn), pdf_env);
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

// pathTracingTrans (tests/oracle_transmission.cpp) with the mapped material and normal at every vertex it shades
vec3 pathTracingTransMaps(const Scene& sc, const TexSet& ts, const MapSet& ms, const LightTable& lt, const EnvTable& env, HitResult hit,
                          int maxBounce, PixelCtx& px, Counters& cn) {
    vec3 Lo = splat(0);
    vec3 history = splat(1);
    const int K = (int)lt.tri.size();
    const float P_env = env.ok ? (K > 0 ? 0.5f : 1.0f) : 0.0f;
    for (int bounce = 0; bounce < maxBounce; bounce++) {
        vec3 Vv = ez_neg(hit.viewDir);
        vec3 N = hit.normal;
        Material material = getMaterial(sc, hit.triangle);
        mapMaterial(sc, ts, ms, hit.triangle, hit.hitPoint, Vv, hit.isInside, &material, &N);
        const TransLobe tl = transLobe(material, hit.isInside);

        const float r_sel = px.rng.rand();
        const float r_1 = px.rng.rand();
        const float r_2 = px.rng.rand();
        const bool envPick = (P_env == 1.0f) || (P_env == 0.5f && r_sel < 0.5f);
        const float r_tri = (P_env == 0.5f) ? (r_sel - 0.5f) * 2.0f : r_sel;
        if (envPick) {
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
            const float w = (P_env > 0.0f && !below) ? misMixWeight(pdf_b, P_env * ez_env_pdf(env.pdf.data(), env.W, env.H, L)) : 1.0f;
            Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), hdrColor(sc, L, cn)), f_r), ac), pdf_b));
            break;
        }
        const vec3 Le = getMaterial(sc, newHit.triangle).emissive;
        float w = 1.0f;
        const float lum = ez_luminance(Le);
        if (lum > 0.0f && !below) {
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

// one sample of a maps render: the transmission loop with EZRT_PARAM_TRANSMISSION, the medium loop otherwise
vec3 shadePixelMaps(const Scene& sc, const Tables& tb, const TexSet& ts, const MapSet& ms, const ez_medium& med, const ezrt_render_params& p,
                    const ez_lens* lens, uint32_t ipx, uint32_t ipy, uint32_t frameCounter, Counters& cn, First* first) {
    if (!(p.reserved[0] & EZRT_PARAM_TRANSMISSION)) return shadePixelMapsMedium(sc, tb, ts, ms, med, p, lens, ipx, ipy, frameCounter, cn, first);
    PixelCtx px;
    px.px = ipx; px.py = ipy; px.frameCounter = frameCounter;
    const Ray ray = cameraRay(p, lens, px);
    const HitResult firstHit = hitBVH(sc, ray, cn, 0);
    firstOf(sc, ts, ms, firstHit, first);
    if (!firstHit.isHit) return hdrColor(sc, ray.direction, cn);
    return ez_add(getMaterial(sc, firstHit.triangle).emissive, pathTracingTransMaps(sc, ts, ms, tb.lt, tb.env, firstHit, p.max_bounce, px, cn));
}

// the validated set-up shared by both forms: -2 where the library returns EZRT_ERR_INVALID
int mapsSetup(const ezrt_render_params* p, const ezrt_medium* m, int nTex, const ezrt_texture* tex, const float* uv, const int32_t* id,
              const int32_t* mr, const int32_t* nm, int nTriangles, ez_medium* med, TexSet* ts, MapSet* ms) {
    if (!(p->reserved[0] & EZRT_PARAM_MATERIAL_MAPS)) return -1;
    if (!(p->reserved[0] & EZRT_PARAM_TEXTURES)) return -2;
    if (p->mode != EZRT_MODE_DISNEY_LIGHTS || p->pipeline == EZRT_PIPELINE_MEGAKERNEL || !texSetOf(nTex, tex, uv, id, nTriangles, ts)) return -2;
    if (!mapSetOf(mr, nm, nTex, nTriangles, ms)) return -2;
    memset(med, 0, sizeof(*med));
    if (p->reserved[0] & EZRT_PARAM_MEDIUM) {
        if (p->reserved[0] & EZRT_PARAM_TRANSMISSION) return -2;
        if (!mediumOf(m, med)) return -2;
    }
    return 0;
}

}  // namespace

extern "C" {

void oracle_unorm8_table(float* out) { memcpy(out, ez_unorm8_table, sizeof(ez_unorm8_table)); }

// ez_tex_sample of the W x H RGBA8 texture with ez_unorm8_table at n (u, v) -> rgb (3 per row)
void oracle_unorm_sample(const uint8_t* rgba, int W, int H, int n, const float* uv, float* rgb) {
    std::vector<uint32_t> t((size_t)W * H);
    memcpy(t.data(), rgba, 4 * t.size());
    for (int i = 0; i < n; i++) {
        const vec3 c = ez_tex_sample(t.data(), W, H, uv[2 * i], uv[2 * i + 1], ez_unorm8_table);
        rgb[3 * i] = c.x; rgb[3 * i + 1] = c.y; rgb[3 * i + 2] = c.z;
    }
}

// ez_mr_apply of n filtered colours f (3 per row) to rm (roughness, metallic per row), in place
void oracle_mr_apply(int n, const float* f, float* rm) {
    for (int i = 0; i < n; i++) ez_mr_apply(ez_v3(f[3 * i], f[3 * i + 1], f[3 * i + 2]), &rm[2 * i], &rm[2 * i + 1]);
}

// ez_tangent_frame of n rows: p (9 floats: p1, p2, p3), uv6 (6), No (3) -> TB (6: T', B) and ok (1 or 0)
void oracle_tangent_frame(int n, const float* p, const float* uv6, const float* No, float* TB, int32_t* ok) {
    for (int i = 0; i < n; i++) {
        const float* q = p + 9 * i;
        vec3 T = splat(0), B = splat(0);
        ok[i] = ez_tangent_frame(ez_v3(q[0], q[1], q[2]), ez_v3(q[3], q[4], q[5]), ez_v3(q[6], q[7], q[8]), uv6 + 6 * i,
                                 ez_v3(No[3 * i], No[3 * i + 1], No[3 * i + 2]), &T, &B);
        float* o = TB + 6 * i;
        o[0] = T.x; o[1] = T.y; o[2] = T.z; o[3] = B.x; o[4] = B.y; o[5] = B.z;
    }
}

// ez_normal_map of n rows: p (9), uv6 (6), uv (2), f (3), N (3), inside (1), V (3) -> n (3)
void oracle_normal_map(int n, const float* p, const float* uv6, const float* uv, const float* f, const float* N, const int32_t* inside,
                       const float* V, float* out) {
    auto v3 = [](const float* a, int i) { return ez_v3(a[3 * i], a[3 * i + 1], a[3 * i + 2]); };
    for (int i = 0; i < n; i++) {
        const float* q = p + 9 * i;
        const vec3 r = ez_normal_map(ez_v3(q[0], q[1], q[2]), ez_v3(q[3], q[4], q[5]), ez_v3(q[6], q[7], q[8]), uv6 + 6 * i, uv[2 * i],
                                     uv[2 * i + 1], v3(f, i), v3(N, i), inside[i], v3(V, i));
        out[3 * i] = r.x; out[3 * i + 1] = r.y; out[3 * i + 2] = r.z;
    }
}

// The window [x0,x1) x [y0,y1) as oracle_render_textures, with EZRT_PARAM_MATERIAL_MAPS (required) and the maps' ids of
// ezrt_scene_set_material_maps; aov (8 floats per pixel): the mapped albedo and normal of the first hit
int oracle_render_material_maps(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache,
                                int hdrW, int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, int nTex,
                                const ezrt_texture* tex, const float* uv, const int32_t* id, const int32_t* mr, const int32_t* nm, int x0, int y0,
                                int x1, int y1, float* framebuffer, float* aov, float* luma2, uint64_t* counters_out, int n_threads) {
    if (!p) return -1;
    ez_medium med;
    TexSet ts;
    MapSet ms;
    int rc = mapsSetup(p, m, nTex, tex, uv, id, mr, nm, nTriangles, &med, &ts, &ms);
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
                    const vec3 color = shadePixelMaps(sc, tb, ts, ms, med, *p, on ? &lens : nullptr, (uint32_t)pxl, (uint32_t)py, frame, cn, &f);
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

// The adaptive form (tests/oracle_textures.cpp's loop with this file's sample function)
int oracle_render_material_maps_adaptive(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache,
                                         int hdrW, int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, int nTex,
                                         const ezrt_texture* tex, const float* uv, const int32_t* id, const int32_t* mr, const int32_t* nm,
                                         const ezrt_adaptive_params* ap, int x0, int y0, int x1, int y1, float* framebuffer, int32_t* spp_out,
                                         float* luma2_out, uint64_t* counters_out, int n_threads) {
    if (!p) return -1;
    ez_medium med;
    TexSet ts;
    MapSet ms;
    int rc = mapsSetup(p, m, nTex, tex, uv, id, mr, nm, nTriangles, &med, &ts, &ms);
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
                        const vec3 color = shadePixelMaps(sc, tb, ts, ms, med, *p, on ? &lens : nullptr, px, py, (uint32_t)f, cn, nullptr);
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
