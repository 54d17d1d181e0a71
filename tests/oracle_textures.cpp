// oracle_textures.cpp -- CPU restatement of base-colour textures (EZRT_PARAM_TEXTURES in EZRT_MODE_DISNEY_LIGHTS, ezrt_math.h,
// DESIGN.md section 15): mode 4 and the homogeneous medium's loop with the textured base colour at every surface hit, with and without
// EZRT_PARAM_ENV_LIGHT and the thin lens, over the medium restatement (tests/oracle_medium.cpp, included unchanged).  Plain/window,
// feature-buffer and adaptive forms; and the definition's two functions, ez_tri_bary and ez_tex_sample, for the CPU tests.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT, like the oracle it compiles in (build/libezrt_oracle_textures.so, tests/oracle_textures.py).
//
// A render without EZRT_PARAM_MEDIUM runs the medium loop with sigma_t = 0, which draws nothing and is mode 4's (tests/test_medium_oracle.py).
// EZRT_PARAM_TRANSMISSION is not restated here (-3): its textured renders are held to the constant-texture invariances.
#include "oracle_medium.cpp"

namespace {

struct TexSet {
    std::vector<int> off, W, H;
    std::vector<uint32_t> texels;
    const float* uv = nullptr;      // 6 floats per triangle
    const int32_t* id = nullptr;    // per triangle
};

bool texSetOf(int n, const ezrt_texture* t, const float* uv, const int32_t* id, int nTriangles, TexSet* out) {
    if (n < 1 || !t || !uv || !id) return false;
    size_t total = 0;
    for (int k = 0; k < n; k++) {
        if (t[k].width < 1 || t[k].width > 16384 || t[k].height < 1 || t[k].height > 16384 || !t[k].rgba || t[k].reserved != 0) return false;
        out->off.push_back((int)total);
        out->W.push_back(t[k].width);
        out->H.push_back(t[k].height);
        total += (size_t)t[k].width * t[k].height;
    }
    for (int i = 0; i < nTriangles; i++)
        if (id[i] < -1 || id[i] >= n) return false;
    out->texels.resize(total);
    for (int k = 0; k < n; k++) memcpy(out->texels.data() + out->off[k], t[k].rgba, 4 * (size_t)t[k].width * t[k].height);
    out->uv = uv;
    out->id = id;
    return true;
}

// the base colour `base` of the hit at P on triangle tri, textured
vec3 texturedBase(const Scene& sc, const TexSet& ts, int tri, vec3 P, vec3 base) {
    const Triangle T = getTriangle(sc, tri);
    float w1, w2, w3, u, v;
    ez_tri_bary(P, T.p1, T.p2, T.p3, geoNormal(T), &w1, &w2, &w3);
    ez_tex_uv(w1, w2, w3, ts.uv + 6 * (size_t)tri, &u, &v);
    const int k = ts.id[tri];
    if (k < 0) return base;
    return ez_mul(base, ez_tex_sample(ts.texels.data() + ts.off[k], ts.W[k], ts.H[k], u, v, ez_srgb_table));
}

// shadePixelMedium (tests/oracle_medium.cpp) with the textured material at every surface vertex; *albedo = the first hit's
vec3 shadePixelTex(const Scene& sc, const Tables& tb, const TexSet& ts, const ez_medium& med, const ezrt_render_params& p, const ez_lens* lens,
                   uint32_t ipx, uint32_t ipy, uint32_t frameCounter, Counters& cn, HitResult* first, vec3* albedo) {
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
        if (bounce == 0 && first) *first = h;
        if (bounce == 0 && albedo && h.isHit) *albedo = texturedBase(sc, ts, h.triangle, h.hitPoint, getMaterial(sc, h.triangle).baseColor);
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
        const vec3 Vv = ez_neg(h.viewDir), N = h.normal;
        Material material = scatter ? Material() : getMaterial(sc, h.triangle);
        if (!scatter) material.baseColor = texturedBase(sc, ts, h.triangle, h.hitPoint, material.baseColor);
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

// the validated set-up shared by both forms: -2 where the library returns EZRT_ERR_INVALID, -3 for what is not restated
int texSetup(const ezrt_render_params* p, const ezrt_medium* m, int nTex, const ezrt_texture* tex, const float* uv, const int32_t* id,
             int nTriangles, ez_medium* med, TexSet* ts) {
    if (!(p->reserved[0] & EZRT_PARAM_TEXTURES)) return -1;
    if (p->mode != EZRT_MODE_DISNEY_LIGHTS || p->pipeline == EZRT_PIPELINE_MEGAKERNEL || !texSetOf(nTex, tex, uv, id, nTriangles, ts)) return -2;
    if (p->reserved[0] & EZRT_PARAM_TRANSMISSION) return -3;
    memset(med, 0, sizeof(*med));
    if (p->reserved[0] & EZRT_PARAM_MEDIUM)
        if (!mediumOf(m, med)) return -2;
    return 0;
}

}  // namespace

extern "C" {

// ez_tri_bary of n points: P, p1, p2, p3, Ng (3 floats each per row) -> w (3 per row)
void oracle_tri_bary(int n, const float* P, const float* p1, const float* p2, const float* p3, const float* Ng, float* w) {
    auto v = [](const float* a, int i) { return ez_v3(a[3 * i], a[3 * i + 1], a[3 * i + 2]); };
    for (int i = 0; i < n; i++) ez_tri_bary(v(P, i), v(p1, i), v(p2, i), v(p3, i), v(Ng, i), w + 3 * i, w + 3 * i + 1, w + 3 * i + 2);
}

// ez_tex_sample of the W x H RGBA8 texture at n (u, v) -> rgb (3 per row); and the table
void oracle_tex_sample(const uint8_t* rgba, int W, int H, int n, const float* uv, float* rgb) {
    std::vector<uint32_t> t((size_t)W * H);
    memcpy(t.data(), rgba, 4 * t.size());
    for (int i = 0; i < n; i++) {
        const vec3 c = ez_tex_sample(t.data(), W, H, uv[2 * i], uv[2 * i + 1], ez_srgb_table);
        rgb[3 * i] = c.x; rgb[3 * i + 1] = c.y; rgb[3 * i + 2] = c.z;
    }
}
void oracle_srgb_table(float* out) { memcpy(out, ez_srgb_table, sizeof(ez_srgb_table)); }

// The window [x0,x1) x [y0,y1) as oracle_render_medium, with EZRT_PARAM_TEXTURES (required) and the textures of
// ezrt_scene_set_textures; m: the medium when EZRT_PARAM_MEDIUM is set.
int oracle_render_textures(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache, int hdrW,
                           int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, int nTex, const ezrt_texture* tex,
                           const float* uv, const int32_t* id, int x0, int y0, int x1, int y1, float* framebuffer, float* aov, float* luma2,
                           uint64_t* counters_out, int n_threads) {
    if (!p) return -1;
    ez_medium med;
    TexSet ts;
    int rc = texSetup(p, m, nTex, tex, uv, id, nTriangles, &med, &ts);
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
                    HitResult h;
                    vec3 albedo = splat(0);
                    const vec3 color = shadePixelTex(sc, tb, ts, med, *p, on ? &lens : nullptr, (uint32_t)pxl, (uint32_t)py, frame, cn, &h, &albedo);
                    const float a = EZ_DIV(1.0f, ez_u32_to_float(frame + 1u));
                    acc = ez_vmix(acc, color, a);
                    const float y = ez_luminance(color);
                    m2 = ez_mix(m2, y * y, a);
                    if (feat) {
                        float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                        if (h.isHit) {
                            v[0] = albedo.x; v[1] = albedo.y; v[2] = albedo.z; v[3] = 1.0f;
                            v[4] = h.normal.x; v[5] = h.normal.y; v[6] = h.normal.z; v[7] = h.distance;
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

// The adaptive form (tests/oracle_medium.cpp's loop with this file's sample function)
int oracle_render_textures_adaptive(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache,
                                    int hdrW, int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, int nTex,
                                    const ezrt_texture* tex, const float* uv, const int32_t* id, const ezrt_adaptive_params* ap, int x0, int y0,
                                    int x1, int y1, float* framebuffer, int32_t* spp_out, float* luma2_out, uint64_t* counters_out, int n_threads) {
    if (!p) return -1;
    ez_medium med;
    TexSet ts;
    int rc = texSetup(p, m, nTex, tex, uv, id, nTriangles, &med, &ts);
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
                        const vec3 color = shadePixelTex(sc, tb, ts, med, *p, on ? &lens : nullptr, px, py, (uint32_t)f, cn, nullptr, nullptr);
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
