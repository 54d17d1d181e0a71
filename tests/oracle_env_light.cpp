// oracle_env_light.cpp -- CPU restatement of the environment map as a light (EZRT_PARAM_ENV_LIGHT in EZRT_MODE_DISNEY_LIGHTS,
// ezrt_math.h, DESIGN.md section 11): the environment table, its sampler and density, and the flagged per-pixel integrator, over
// the light sampling mode's restatement (tests/oracle_lights.cpp, included unchanged) and the oracle's functions.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT, like the oracle it compiles in (build/libezrt_oracle_env_light.so,
// tests/oracle_env_light.py).
#include "oracle_lights.cpp"

namespace {

struct EnvTable {
    std::vector<float> row, col, pdf;   // H, H x W, H x W
    int W = 0, H = 0;
    double total = 0.0;
    bool ok = false;                    // false: no table (no map, or no texel of positive weight)
};

// the table of ezrt_math.h: weights in fp32, sums and quotients in float64, cast to float
EnvTable buildEnv(const float* hdr, int W, int H) {
    EnvTable t;
    if (!hdr || W <= 0 || H <= 0) return t;
    const size_t n = (size_t)W * H;
    std::vector<float> w(n);
    for (size_t k = 0; k < n; k++) w[k] = ez_env_weight(ez_v3(hdr[3 * k], hdr[3 * k + 1], hdr[3 * k + 2]), (int)(k / W), H);
    std::vector<double> R(H, 0.0);
    for (int i = 0; i < H; i++)
        for (int j = 0; j < W; j++) R[i] += (double)w[(size_t)i * W + j];
    double T = 0.0;
    for (int i = 0; i < H; i++) T += R[i];
    if (!(std::isfinite(T) && T > 0.0)) return t;
    t.W = W; t.H = H; t.total = T; t.ok = true;
    t.row.resize(H); t.col.resize(n); t.pdf.resize(n);
    double S = 0.0;
    for (int i = 0; i < H; i++) {
        S += R[i];
        t.row[i] = (float)(S / T);
        double c = 0.0;
        for (int j = 0; j < W; j++) {
            const size_t k = (size_t)i * W + j;
            c += (double)w[k];
            t.col[k] = (R[i] > 0.0) ? (float)(c / R[i]) : 0.0f;
            t.pdf[k] = (float)((double)w[k] / T);
        }
        if (R[i] > 0.0) t.col[(size_t)i * W + W - 1] = 1.0f;
    }
    t.row[H - 1] = 1.0f;
    return t;
}

// pathTracingLights (tests/oracle_lights.cpp) with the map as one more light, selected with probability P_env
vec3 pathTracingEnvLights(const Scene& sc, const LightTable& lt, const EnvTable& env, HitResult hit, int maxBounce, PixelCtx& px,
                          Counters& cn) {
    vec3 Lo = splat(0);
    vec3 history = splat(1);
    const int K = (int)lt.tri.size();
    const float P_env = env.ok ? (K > 0 ? 0.5f : 1.0f) : 0.0f;
    for (int bounce = 0; bounce < maxBounce; bounce++) {
        vec3 Vv = ez_neg(hit.viewDir);
        vec3 N = hit.normal;
        Material material = getMaterial(sc, hit.triangle);

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
                if (!occludedBounded(sc, sray, EZ_INF, cn)) {
                    const vec3 E = hdrColor(sc, Le, cn);
                    const vec3 f_r = BRDF_Evaluate(Vv, N, Le, splat(0), splat(0), material, false);
                    const float pdf_brdf = BRDF_Pdf(Vv, N, Le, material);
                    const float mis_weight = misMixWeight(pdf_env, pdf_brdf);
                    Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, mis_weight), E), f_r), ez_dot(N, Le)), pdf_env));
                }
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
                    const vec3 f_r = BRDF_Evaluate(Vv, N, Ll, splat(0), splat(0), material, false);
                    const float pdf_brdf = BRDF_Pdf(Vv, N, Ll, material);
                    const float mis_weight = misMixWeight(pdf_light, pdf_brdf);
                    Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, mis_weight), E), f_r), ez_dot(N, Ll)), pdf_light));
                }
            }
        }

        float xi_1, xi_2;
        sobolVec2(px.frameCounter + 1u, (uint32_t)bounce, &xi_1, &xi_2);
        CranleyPattersonRotation(&xi_1, &xi_2, px.px, px.py);
        float xi_3 = px.rng.rand();
        vec3 L = SampleBRDF(xi_1, xi_2, xi_3, Vv, N, material);
        float NdotL = ez_dot(N, L);
        if (NdotL <= 0.0f) break;

        Ray randomRay;
        randomRay.startPoint = hit.hitPoint;
        randomRay.direction = L;
        HitResult newHit = hitBVH(sc, randomRay, cn, 1);
        vec3 f_r = BRDF_Evaluate(Vv, N, L, splat(0), splat(0), material, false);
        float pdf_brdf = BRDF_Pdf(Vv, N, L, material);
        if (pdf_brdf <= 0.0f) break;
        if (!newHit.isHit) {   // the environment: MIS against the map's density (weight 1 without a table)
            const float w = (P_env > 0.0f) ? misMixWeight(pdf_brdf, P_env * ez_env_pdf(env.pdf.data(), env.W, env.H, L)) : 1.0f;
            Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), hdrColor(sc, L, cn)), f_r), NdotL), pdf_brdf));
            break;
        }
        const vec3 Le = getMaterial(sc, newHit.triangle).emissive;
        float w = 1.0f;
        const float lum = ez_luminance(Le);
        if (lum > 0.0f) {
            const Triangle T = getTriangle(sc, newHit.triangle);
            if (ez_is_light(ez_light_weight(T.p1, T.p2, T.p3, Le)))
                w = misMixWeight(pdf_brdf, (1.0f - P_env) * ez_light_pdf(lum, lt.total_f, newHit.distance, ez_abs(ez_dot(geoNormal(T), L))));
        }
        Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), Le), f_r), NdotL), pdf_brdf));
        hit = newHit;
        history = ez_mul(history, ez_divs(ez_scale(f_r, NdotL), pdf_brdf));
    }
    return Lo;
}

// shadePixelLights with pathTracingEnvLights
vec3 shadePixelEnvLights(const Scene& sc, const LightTable& lt, const EnvTable& env, const ezrt_render_params& p, uint32_t ipx, uint32_t ipy,
                         uint32_t frameCounter, Counters& cn) {
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
    if (!firstHit.isHit) return hdrColor(sc, ray.direction, cn);   // camera rays that leave the scene weigh 1
    return ez_add(getMaterial(sc, firstHit.triangle).emissive, pathTracingEnvLights(sc, lt, env, firstHit, p.max_bounce, px, cn));
}

}  // namespace

extern "C" {

// The environment table of a W x H map: returns 1 (table) or 0 (none); outputs as ezrt_scene_env_light's, any may be NULL.
int oracle_env_table(const float* hdr, int W, int H, float* row_cdf, float* col_cdf, float* texel_pdf, double* total) {
    const EnvTable t = buildEnv(hdr, W, H);
    if (total) *total = t.total;
    if (!t.ok) return 0;
    if (row_cdf) std::copy(t.row.begin(), t.row.end(), row_cdf);
    if (col_cdf) std::copy(t.col.begin(), t.col.end(), col_cdf);
    if (texel_pdf) std::copy(t.pdf.begin(), t.pdf.end(), texel_pdf);
    return 1;
}

// n samples of ez_env_sample for (r_1, r_2) pairs on the map's table: direction, the texel drawn, the texel the oracle's
// toSphericalCoord + nearest lookup finds in that direction, and ez_env_pdf of the direction.  Returns -1 without a table.
int oracle_env_samples(const float* hdr, int W, int H, int n, const float* r, float* dir_out, int32_t* texel_out, int32_t* lookup_out,
                       float* pdf_out) {
    const EnvTable t = buildEnv(hdr, W, H);
    if (!t.ok) return -1;
    for (int k = 0; k < n; k++) {
        int texel;
        const vec3 L = ez_env_sample(t.row.data(), t.col.data(), W, H, r[2 * k], r[2 * k + 1], &texel);
        float u, v;
        toSphericalCoord(ez_normalize(L), &u, &v);
        dir_out[3 * k] = L.x; dir_out[3 * k + 1] = L.y; dir_out[3 * k + 2] = L.z;
        texel_out[k] = texel;
        lookup_out[k] = ez_env_texel(u, v, W, H);
        pdf_out[k] = ez_env_pdf(t.pdf.data(), W, H, L);
    }
    return 0;
}

// ez_env_pdf of n directions on the map's table (0 everywhere without a table)
int oracle_env_pdf(const float* hdr, int W, int H, int n, const float* dirs, float* out) {
    const EnvTable t = buildEnv(hdr, W, H);
    for (int k = 0; k < n; k++)
        out[k] = t.ok ? ez_env_pdf(t.pdf.data(), W, H, ez_v3(dirs[3 * k], dirs[3 * k + 1], dirs[3 * k + 2])) : 0.0f;
    return t.ok ? 1 : 0;
}

// oracle_render_lights (tests/oracle_lights.cpp) with EZRT_PARAM_ENV_LIGHT read from p->reserved[0]: mode 4 with the flag runs the
// flagged integrator, anything else what oracle_render_lights runs.
int oracle_render_env_light(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache, int hdrW,
                            int hdrH, int hdrLinear, const ezrt_render_params* p, int x0, int y0, int x1, int y1, float* framebuffer,
                            float* luma2, uint64_t* counters_out, int n_threads) {
    const bool flagged = p && p->mode == EZRT_MODE_DISNEY_LIGHTS && (p->reserved[0] & EZRT_PARAM_ENV_LIGHT);
    if (!flagged)
        return oracle_render_lights(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p, x0, y0, x1, y1, framebuffer, luma2,
                                    counters_out, n_threads);
    if (!tris || !nodes || !framebuffer || !luma2 || nTriangles <= 0 || nNodes < 2) return -1;
    if (x0 < 0 || y0 < 0 || x1 > p->width || y1 > p->height || x1 <= x0 || y1 <= y0) return -1;
    Scene sc = makeScene(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p->env_color, p->mode, p->traverse);
    const LightTable lt = buildLights(sc);
    const EnvTable env = buildEnv(hdr, hdrW, hdrH);
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
                    const vec3 color = shadePixelEnvLights(sc, lt, env, *p, (uint32_t)pxl, (uint32_t)py, frame, cn);
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
