// oracle_lights.cpp -- CPU restatement of the light sampling mode (EZRT_MODE_DISNEY_LIGHTS, ezrt_math.h, DESIGN.md section 10):
// the light table, the bounded occlusion query of its shadow rays, and the per-pixel integrator, over the oracle's hitBVH,
// BRDF, sampling and misMixWeight.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT, like the oracle it compiles in (build/libezrt_oracle_lights.so, tests/oracle_lights.py).
//
// The oracle itself is unchanged.  The bounded query is its hitBVH walk restated with the best distance starting at tmax
// (shadow rays only need isHit, so the closest-hit walk gives the any-hit answer); it counts as a shadow ray.
#include "../oracle/ezrt_oracle.cpp"

namespace {

struct LightTable {
    std::vector<int32_t> tri;
    std::vector<float> cdf;
    double total = 0.0;
    float total_f = 0.0f;
};

inline vec3 geoNormal(const Triangle& t) { return ez_normalize(ez_cross(ez_sub(t.p2, t.p1), ez_sub(t.p3, t.p1))); }

LightTable buildLights(const Scene& sc) {
    LightTable lt;
    std::vector<float> w;
    for (int i = 0; i < sc.nTriangles; i++) {
        const Triangle t = getTriangle(sc, i);
        const float wi = ez_light_weight(t.p1, t.p2, t.p3, getMaterial(sc, i).emissive);
        if (!ez_is_light(wi)) continue;
        lt.tri.push_back(i);
        w.push_back(wi);
    }
    for (float x : w) lt.total += (double)x;
    double S = 0.0;
    for (float x : w) {
        S += (double)x;
        lt.cdf.push_back((float)(S / lt.total));
    }
    if (!lt.cdf.empty()) lt.cdf.back() = 1.0f;
    lt.total_f = (float)lt.total;
    return lt;
}

// hitBVH (P5/fsh:254-306) with the best distance starting at tmax: isHit iff a triangle the walk tests is accepted with t < tmax
bool occludedBounded(const Scene& sc, const Ray& ray, float tmax, Counters& cn) {
    cn.rays[2]++;
    float best = tmax;
    const bool prune = (sc.traverse != EZRT_TRAVERSE_REFERENCE);
    const float slack = prune ? pruneSlack(sc, ray) : 0.0f;
    int stack[256];
    float stackT0[256];
    int sp = 0;
    stackT0[sp] = -1.0f;
    stack[sp++] = 1;
    bool hit = false;
    while (sp > 0) {
        const int top = stack[--sp];
        if (prune && pruned(stackT0[sp], best, slack)) continue;
        const BVHNode node = getBVHNode(sc, top);
        if (node.n > 0) {
            const HitResult r = hitArray(sc, ray, node.index, node.index + node.n - 1, cn);
            if (r.isHit && r.distance < best) { best = r.distance; hit = true; }
            continue;
        }
        float d1 = EZ_INF, d2 = EZ_INF, e1 = -1.0f, e2 = -1.0f;
        if (node.left > 0) { const BVHNode l = getBVHNode(sc, node.left); d1 = hitAABB(ray, l.AA, l.BB, &e1); }
        if (node.right > 0) { const BVHNode r = getBVHNode(sc, node.right); d2 = hitAABB(ray, r.AA, r.BB, &e2); }
        bool h1 = d1 > 0, h2 = d2 > 0;
        if (prune) {
            if (h1 && pruned(e1, best, slack)) h1 = false;
            if (h2 && pruned(e2, best, slack)) h2 = false;
        }
        if (h1 && h2) {
            if (d1 < d2) { stackT0[sp] = e2; stack[sp++] = node.right; stackT0[sp] = e1; stack[sp++] = node.left; }
            else         { stackT0[sp] = e1; stack[sp++] = node.left;  stackT0[sp] = e2; stack[sp++] = node.right; }
        } else if (h1) { stackT0[sp] = e1; stack[sp++] = node.left; }
        else if (h2)   { stackT0[sp] = e2; stack[sp++] = node.right; }
    }
    return hit;
}

// pathTracingImportanceSampling (P5/fsh:810-890) with the environment sample replaced by one light sample on the emissive
// triangles, and the BRDF samples' emission hits on lights weighted by MIS
vec3 pathTracingLights(const Scene& sc, const LightTable& lt, HitResult hit, int maxBounce, PixelCtx& px, Counters& cn) {
    vec3 Lo = splat(0);
    vec3 history = splat(1);
    const int K = (int)lt.tri.size();
    for (int bounce = 0; bounce < maxBounce; bounce++) {
        vec3 Vv = ez_neg(hit.viewDir);
        vec3 N = hit.normal;
        Material material = getMaterial(sc, hit.triangle);

        const float r_sel = px.rng.rand();
        const float r_1 = px.rng.rand();
        const float r_2 = px.rng.rand();
        if (K > 0) {
            const int k = ez_light_select(lt.cdf.data(), K, r_sel);
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
                    const float pdf_light = ez_light_pdf(ez_luminance(E), lt.total_f, dist, cos_l);
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
        if (!newHit.isHit) {   // the environment: BRDF samples only, weight 1
            Lo = ez_add(Lo, contrib(history, hdrColor(sc, L, cn), f_r, NdotL, pdf_brdf));
            break;
        }
        const vec3 Le = getMaterial(sc, newHit.triangle).emissive;
        float w = 1.0f;
        const float lum = ez_luminance(Le);
        if (lum > 0.0f) {
            const Triangle T = getTriangle(sc, newHit.triangle);
            if (ez_is_light(ez_light_weight(T.p1, T.p2, T.p3, Le)))
                w = misMixWeight(pdf_brdf, ez_light_pdf(lum, lt.total_f, newHit.distance, ez_abs(ez_dot(geoNormal(T), L))));
        }
        Lo = ez_add(Lo, ez_divs(ez_scale(ez_mul(ez_mul(ez_scale(history, w), Le), f_r), NdotL), pdf_brdf));
        hit = newHit;
        history = ez_mul(history, ez_divs(ez_scale(f_r, NdotL), pdf_brdf));
    }
    return Lo;
}

// shadePixel (main(), P5/fsh:894-949) with pathTracingLights
vec3 shadePixelLights(const Scene& sc, const LightTable& lt, const ezrt_render_params& p, uint32_t ipx, uint32_t ipy, uint32_t frameCounter,
                      Counters& cn) {
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
    return ez_add(getMaterial(sc, firstHit.triangle).emissive, pathTracingLights(sc, lt, firstHit, p.max_bounce, px, cn));
}

}  // namespace

extern "C" {

// The light table: returns K, writes min(K, cap) triangle indices / cdf entries and *total = W (float64).
int oracle_light_table(const float* tris, int nTriangles, int cap, int32_t* tri_out, float* cdf_out, double* total_out) {
    if (!tris || nTriangles <= 0 || cap < 0) return -1;
    Scene sc = makeScene(tris, nTriangles, nullptr, 0, nullptr, nullptr, 0, 0, 0, nullptr, EZRT_MODE_DISNEY_LIGHTS, EZRT_TRAVERSE_REFERENCE);
    const LightTable lt = buildLights(sc);
    const int K = (int)lt.tri.size();
    for (int k = 0; k < K && k < cap; k++) {
        if (tri_out) tri_out[k] = lt.tri[k];
        if (cdf_out) cdf_out[k] = lt.cdf[k];
    }
    if (total_out) *total_out = lt.total;
    return K;
}

// Bounded occlusion of n rays as ezrt_occluded_rays: out_lit[i] = 1 iff nothing is accepted strictly before tmax[i]; when every
// tmax is +inf the rays are unbounded (best starts at the shader's INF, as mode 3's shadow rays).
int oracle_occluded(const float* tris, int nTriangles, const float* nodes, int nNodes, int n, const float* origins, const float* dirs,
                    const float* tmax, int traverse, int32_t* out_lit) {
    if (!tris || !nodes || n < 0 || !origins || !dirs || !tmax || !out_lit) return -1;
    Scene sc = makeScene(tris, nTriangles, nodes, nNodes, nullptr, nullptr, 0, 0, 0, nullptr, EZRT_MODE_DISNEY_LIGHTS, traverse);
    bool bounded = false;
    for (int i = 0; i < n; i++) bounded = bounded || !(std::isinf(tmax[i]) && tmax[i] > 0.0f);
    Counters cn;
    memset(&cn, 0, sizeof(cn));
    for (int i = 0; i < n; i++) {
        Ray ray;
        ray.startPoint = ez_v3(origins[3 * i], origins[3 * i + 1], origins[3 * i + 2]);
        ray.direction = ez_v3(dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2]);
        out_lit[i] = occludedBounded(sc, ray, bounded ? tmax[i] : EZ_INF, cn) ? 0 : 1;
    }
    return 0;
}

// n samples of ez_triangle_point (the light sampler) for (r_1, r_2) pairs
void oracle_triangle_points(const float* p /* 9 */, int n, const float* r, float* out) {
    const vec3 p1 = ez_v3(p[0], p[1], p[2]), p2 = ez_v3(p[3], p[4], p[5]), p3 = ez_v3(p[6], p[7], p[8]);
    for (int i = 0; i < n; i++) {
        const vec3 q = ez_triangle_point(p1, p2, p3, r[2 * i], r[2 * i + 1]);
        out[3 * i] = q.x; out[3 * i + 1] = q.y; out[3 * i + 2] = q.z;
    }
}

// The window [x0,x1) x [y0,y1) of the p->width x p->height grid, as oracle_render_window, in mode p->mode (4: the light sampling
// mode; others: the oracle's shadePixel), plus luma2 = the running mean of the squared sample luminance (in/out like the
// framebuffer when first_frame > 0).  counters_out as oracle_render_window's.
int oracle_render_lights(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache, int hdrW,
                         int hdrH, int hdrLinear, const ezrt_render_params* p, int x0, int y0, int x1, int y1, float* framebuffer, float* luma2,
                         uint64_t* counters_out, int n_threads) {
    if (!tris || !nodes || !p || !framebuffer || !luma2 || nTriangles <= 0 || nNodes < 2) return -1;
    if (x0 < 0 || y0 < 0 || x1 > p->width || y1 > p->height || x1 <= x0 || y1 <= y0) return -1;
    if (p->mode == EZRT_MODE_DISNEY_IS_MIS_P5 && (!hdr || !hdrCache)) return -1;
    Scene sc = makeScene(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p->env_color, p->mode, p->traverse);
    const LightTable lt = buildLights(sc);
    const bool lights = (p->mode == EZRT_MODE_DISNEY_LIGHTS);
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
                    const vec3 color = lights ? shadePixelLights(sc, lt, *p, (uint32_t)pxl, (uint32_t)py, frame, cn)
                                              : shadePixel(sc, *p, (uint32_t)pxl, (uint32_t)py, frame, cn);
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
