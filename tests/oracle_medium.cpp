// oracle_medium.cpp -- CPU restatement of the homogeneous medium (EZRT_PARAM_MEDIUM in EZRT_MODE_DISNEY_LIGHTS, ezrt_math.h,
// DESIGN.md section 14): free flight on every segment, medium vertices with the Henyey-Greenstein phase function, and the light
// samples' transmittance, with and without EZRT_PARAM_ENV_LIGHT and the thin lens, over the lens restatement (tests/oracle_lens.cpp,
// included unchanged) and the oracle's functions.  Plain/window, feature-buffer and adaptive forms.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT, like the oracle it compiles in (build/libezrt_oracle_medium.so, tests/oracle_medium.py).
//
// phase_only (a switch of the restatement only): no light samples, and every emission and environment hit weighs 1 -- an
// independent estimator of the same integral, for the unbiasedness tests.
#include "oracle_lens.cpp"

namespace {

// the medium of the C ABI's struct, validated as ezrt_scene_set_medium validates it
bool mediumOf(const ezrt_medium* m, ez_medium* out) {
    if (!m) return false;
    if (!(ez_finite(m->sigma_t) && m->sigma_t >= 0.0f)) return false;
    for (int k = 0; k < 3; k++) {
        if (!(m->albedo[k] >= 0.0f && m->albedo[k] <= 1.0f)) return false;
        if (!(ez_finite(m->box_min[k]) && ez_finite(m->box_max[k]))) return false;
        if (m->box_min[k] > m->box_max[k]) return false;
    }
    if (!(m->g > -1.0f && m->g < 1.0f) || m->reserved != 0) return false;
    out->sigma_t = m->sigma_t;
    out->albedo = ez_v3(m->albedo[0], m->albedo[1], m->albedo[2]);
    out->g = m->g;
    out->bmin = ez_v3(m->box_min[0], m->box_min[1], m->box_min[2]);
    out->bmax = ez_v3(m->box_max[0], m->box_max[1], m->box_max[2]);
    return true;
}

// a lit light sample's contribution at a surface (mode 4's) or a medium vertex (the phase function), before the transmittance
vec3 mediumLightContrib(vec3 history, bool atMedium, vec3 d, vec3 Vv, vec3 N, vec3 Ll, const Material& m, float g, vec3 E, float pdf_light) {
    if (atMedium) {
        const float p = ez_hg_pdf(d, Ll, g);
        const float w = misMixWeight(pdf_light, p);
        return ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), E), splat(p)), 1.0f), pdf_light);
    }
    const vec3 f_r = BRDF_Evaluate(Vv, N, Ll, splat(0), splat(0), m, false);
    const float pdf_brdf = BRDF_Pdf(Vv, N, Ll, m);
    const float w = misMixWeight(pdf_light, pdf_brdf);
    return ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), E), f_r), ez_dot(N, Ll)), pdf_light);
}

// one sample, segment by segment as the wavefront kernels run it: *first = the camera ray's hit (the feature buffers)
vec3 shadePixelMedium(const Scene& sc, const Tables& tb, const ez_medium& med, const ezrt_render_params& p, const ez_lens* lens, uint32_t ipx,
                      uint32_t ipy, uint32_t frameCounter, Counters& cn, HitResult* first, bool phaseOnly) {
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
        if (bounce > 0 && pdf <= 0.0f) break;
        float t_s;
        const float t_end = h.isHit ? h.distance : ez_u2f(0x7f800000u);
        const bool scatter = ez_medium_flight(&med, ray.startPoint, ray.direction, t_end, &px.rng.seed, &t_s) != 0;
        if (!scatter && !h.isHit) {
            if (bounce == 0) return hdrColor(sc, ray.direction, cn);
            const float w = (P_env > 0.0f && !phaseOnly) ? misMixWeight(pdf, P_env * ez_env_pdf(tb.env.pdf.data(), tb.env.W, tb.env.H, ray.direction)) : 1.0f;
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
                if (lum > 0.0f && !phaseOnly) {
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
        // the vertex: P, and for a surface its frame and material
        const vec3 P = scatter ? ez_add(ray.startPoint, ez_scale(ray.direction, t_s)) : h.hitPoint;
        const vec3 d = ray.direction;
        const vec3 Vv = ez_neg(h.viewDir), N = h.normal;
        const Material material = scatter ? Material() : getMaterial(sc, h.triangle);
        const float r_sel = px.rng.rand();
        const float r_1 = px.rng.rand();
        const float r_2 = px.rng.rand();
        const bool envPick = (P_env == 1.0f) || (P_env == 0.5f && r_sel < 0.5f);
        const float r_tri = (P_env == 0.5f) ? (r_sel - 0.5f) * 2.0f : r_sel;
        if (phaseOnly) {
        } else if (envPick) {
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

}  // namespace

extern "C" {

// ez_hg_sample of n (d[3 i..], g[i], h[2 i], h[2 i + 1]) -> L (n x 3) and pdf = ez_hg_pdf(d, L, g) (n)
void oracle_hg_sample(int n, const float* d, const float* g, const float* h, float* L_out, float* pdf_out) {
    for (int i = 0; i < n; i++) {
        const vec3 dv = ez_v3(d[3 * i], d[3 * i + 1], d[3 * i + 2]);
        const vec3 L = ez_hg_sample(dv, g[i], h[2 * i], h[2 * i + 1]);
        L_out[3 * i] = L.x; L_out[3 * i + 1] = L.y; L_out[3 * i + 2] = L.z;
        if (pdf_out) pdf_out[i] = ez_hg_pdf(dv, L, g[i]);
    }
}

// ez_hg_pdf of n (d, L, g) triples
void oracle_hg_pdf(int n, const float* d, const float* L, const float* g, float* out) {
    for (int i = 0; i < n; i++)
        out[i] = ez_hg_pdf(ez_v3(d[3 * i], d[3 * i + 1], d[3 * i + 2]), ez_v3(L[3 * i], L[3 * i + 1], L[3 * i + 2]), g[i]);
}

// ez_box_overlap of n segments (o, d, t_end) with the box [bmin, bmax]: ok[i], t01[2 i..]
void oracle_box_overlap(int n, const float* o, const float* d, const float* t_end, const float* bmin, const float* bmax, int32_t* ok, float* t01) {
    for (int i = 0; i < n; i++) {
        float t0 = 0.0f, t1 = 0.0f;
        ok[i] = ez_box_overlap(ez_v3(o[3 * i], o[3 * i + 1], o[3 * i + 2]), ez_v3(d[3 * i], d[3 * i + 1], d[3 * i + 2]), ez_v3(bmin[0], bmin[1], bmin[2]),
                               ez_v3(bmax[0], bmax[1], bmax[2]), t_end[i], &t0, &t1);
        t01[2 * i] = t0; t01[2 * i + 1] = t1;
    }
}

// ez_medium_transmittance of n shadow rays (o, d, L) through the medium m; -2 for an invalid medium
int oracle_transmittance(const ezrt_medium* m, int n, const float* o, const float* d, const float* L, float* out) {
    ez_medium med;
    if (!mediumOf(m, &med)) return -2;
    for (int i = 0; i < n; i++)
        out[i] = ez_medium_transmittance(&med, ez_v3(o[3 * i], o[3 * i + 1], o[3 * i + 2]), ez_v3(d[3 * i], d[3 * i + 1], d[3 * i + 2]), L[i]);
    return 0;
}

// ez_free_flight of n draws
void oracle_free_flight(int n, const float* r, float sigma_t, float* out) {
    for (int i = 0; i < n; i++) out[i] = ez_free_flight(r[i], sigma_t);
}

// The window [x0,x1) x [y0,y1) as oracle_render_lens, with EZRT_PARAM_MEDIUM read from p->reserved[0] and the medium m (NULL: none).
// Without the flag: oracle_render_lens.  Returns -2 where the library returns EZRT_ERR_INVALID (no or an invalid medium, a mode
// other than 4, the megakernel, EZRT_PARAM_TRANSMISSION, an invalid lens).
int oracle_render_medium(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache, int hdrW,
                         int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, int x0, int y0, int x1, int y1, float* framebuffer,
                         float* aov, float* luma2, uint64_t* counters_out, int n_threads, int phase_only) {
    if (!p) return -1;
    if (!(p->reserved[0] & EZRT_PARAM_MEDIUM))
        return oracle_render_lens(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p, x0, y0, x1, y1, framebuffer, aov, luma2,
                                  counters_out, n_threads);
    ez_medium med;
    if (p->mode != EZRT_MODE_DISNEY_LIGHTS || p->pipeline == EZRT_PIPELINE_MEGAKERNEL || (p->reserved[0] & EZRT_PARAM_TRANSMISSION) || !mediumOf(m, &med))
        return -2;
    ez_lens lens;
    bool on;
    int rc = checkRender(tris, nTriangles, nodes, nNodes, hdr, hdrCache, p, x0, y0, x1, y1, &lens, &on);
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
                    const vec3 color = shadePixelMedium(sc, tb, med, *p, on ? &lens : nullptr, (uint32_t)pxl, (uint32_t)py, frame, cn, &h, phase_only != 0);
                    const float a = EZ_DIV(1.0f, ez_u32_to_float(frame + 1u));
                    acc = ez_vmix(acc, color, a);
                    const float y = ez_luminance(color);
                    m2 = ez_mix(m2, y * y, a);
                    if (feat) {
                        float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                        if (h.isHit) {
                            const vec3 albedo = getMaterial(sc, h.triangle).baseColor;
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

// The adaptive form (tests/oracle_lens.cpp's loop with this file's sample function): the tiles of the window (x0, y0 multiples of 16;
// x1, y1 multiples of 16 or the image edge) into framebuffer, spp_out, luma2_out.  counters_out: samples = sum of spp_out.  Returns -2
// as oracle_render_medium does; the flag is required.
int oracle_render_medium_adaptive(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache,
                                  int hdrW, int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_medium* m, const ezrt_adaptive_params* ap,
                                  int x0, int y0, int x1, int y1, float* framebuffer, int32_t* spp_out, float* luma2_out, uint64_t* counters_out,
                                  int n_threads) {
    if (!p || !(p->reserved[0] & EZRT_PARAM_MEDIUM)) return -1;
    ez_medium med;
    if (p->mode != EZRT_MODE_DISNEY_LIGHTS || p->pipeline == EZRT_PIPELINE_MEGAKERNEL || (p->reserved[0] & EZRT_PARAM_TRANSMISSION) || !mediumOf(m, &med))
        return -2;
    ez_lens lens;
    bool on;
    int rc = checkRender(tris, nTriangles, nodes, nNodes, hdr, hdrCache, p, x0, y0, x1, y1, &lens, &on);
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
                        const vec3 color = shadePixelMedium(sc, tb, med, *p, on ? &lens : nullptr, px, py, (uint32_t)f, cn, nullptr, false);
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
