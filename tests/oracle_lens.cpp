// oracle_lens.cpp -- CPU restatement of the thin-lens camera (EZRT_PARAM_THIN_LENS, ezrt_math.h, DESIGN.md section 13): the camera
// ray, then every mode's existing path function from the first hit (the oracle's pathTracing / pathTracingImportanceSampling, the
// light sampling mode's, the environment light's and the transmission restatement's, tests/oracle_transmission.cpp, included
// unchanged), in plain, window, feature-buffer and adaptive forms.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT, like the oracle it compiles in (build/libezrt_oracle_lens.so, tests/oracle_lens.py).
//
// Without the flag the sample function is the pinhole's, so every render here equals the oracle's and the restatements' bit for bit.
#include "oracle_transmission.cpp"

#define EZRT_TILE_SIZE 16   // the 16x16 tiles of adaptive sampling (include/ezrt.h)

namespace {

// the lens of the render's parameters; false without the flag or when ez_lens_setup rejects them
bool lensOf(const ezrt_render_params& p, ez_lens* L) {
    if (!(p.reserved[0] & EZRT_PARAM_THIN_LENS)) return false;
    float R, f;
    memcpy(&R, &p.reserved[1], sizeof(float));
    memcpy(&f, &p.reserved[2], sizeof(float));
    return ez_lens_setup(p.eye, p.camera_rotate, R, f, L) != 0;
}

// main(), P5/fsh:915-925: the pinhole direction before normalisation; px.rng leaves with the two jitter draws taken
vec3 pinholeDir(const ezrt_render_params& p, PixelCtx& px) {
    px.rng.seed = (px.px * 1973u + px.py * 9277u + px.frameCounter * 26699u) | 1u;
    float pixx = EZ_DIV((float)px.px + 0.5f, (float)p.width) * 2.0f - 1.0f;
    float pixy = EZ_DIV((float)px.py + 0.5f, (float)p.height) * 2.0f - 1.0f;
    float aax = EZ_DIV(px.rng.rand() - 0.5f, (float)p.width);
    float aay = EZ_DIV(px.rng.rand() - 0.5f, (float)p.height);
    float vx = pixx + aax, vy = pixy + aay, vz = -1.5f, vw = 0.0f;
    const float* m = p.camera_rotate;
    return ez_v3(((m[0] * vx + m[4] * vy) + m[8] * vz) + m[12] * vw,
                 ((m[1] * vx + m[5] * vy) + m[9] * vz) + m[13] * vw,
                 ((m[2] * vx + m[6] * vy) + m[10] * vz) + m[14] * vw);
}

// the camera ray of the sample px (lens null: the pinhole's)
Ray cameraRay(const ezrt_render_params& p, const ez_lens* lens, PixelCtx& px) {
    const vec3 dir = pinholeDir(p, px);
    Ray ray;
    if (!lens) {
        ray.startPoint = ez_v3(p.eye[0], p.eye[1], p.eye[2]);
        ray.direction = ez_normalize(dir);
        return ray;
    }
    float r_a, r_b;
    ez_lens_draws(px.px, px.py, px.frameCounter, &r_a, &r_b);
    ez_lens_ray(lens, dir, r_a, r_b, &ray.startPoint, &ray.direction);
    return ray;
}

struct Tables {
    LightTable lt;
    EnvTable env;   // ok only with EZRT_PARAM_ENV_LIGHT and a map of positive weight
};

// one sample: the camera ray, its first hit (*first), then the mode's path function; the draws after the jitter are the pinhole's
vec3 shadePixelLens(const Scene& sc, const Tables& tb, const ezrt_render_params& p, const ez_lens* lens, uint32_t ipx, uint32_t ipy,
                    uint32_t frameCounter, Counters& cn, HitResult* first) {
    PixelCtx px;
    px.px = ipx; px.py = ipy; px.frameCounter = frameCounter;
    const Ray ray = cameraRay(p, lens, px);
    const HitResult firstHit = hitBVH(sc, ray, cn, 0);
    if (first) *first = firstHit;
    if (!firstHit.isHit) return hdrColor(sc, ray.direction, cn);
    vec3 Li;
    if (p.mode == EZRT_MODE_DISNEY_LIGHTS) {
        if (p.reserved[0] & EZRT_PARAM_TRANSMISSION) Li = pathTracingTrans(sc, tb.lt, tb.env, firstHit, p.max_bounce, px, cn, false);
        else if (p.reserved[0] & EZRT_PARAM_ENV_LIGHT) Li = pathTracingEnvLights(sc, tb.lt, tb.env, firstHit, p.max_bounce, px, cn);
        else Li = pathTracingLights(sc, tb.lt, firstHit, p.max_bounce, px, cn);
    } else if (p.mode == EZRT_MODE_DISNEY_IS_MIS_P5) {
        Li = pathTracingImportanceSampling(sc, firstHit, p.max_bounce, px, cn);
    } else {
        Li = pathTracing(sc, firstHit, p.max_bounce, px, cn);
    }
    return ez_add(getMaterial(sc, firstHit.triangle).emissive, Li);
}

int checkRender(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache,
                const ezrt_render_params* p, int x0, int y0, int x1, int y1, ez_lens* lens, bool* lensOn) {
    if (!tris || !nodes || !p || nTriangles <= 0 || nNodes < 2) return -1;
    if (x0 < 0 || y0 < 0 || x1 > p->width || y1 > p->height || x1 <= x0 || y1 <= y0) return -1;
    if (p->mode == EZRT_MODE_DISNEY_IS_MIS_P5 && (!hdr || !hdrCache)) return -1;
    *lensOn = lensOf(*p, lens);
    if ((p->reserved[0] & EZRT_PARAM_THIN_LENS) && !*lensOn) return -2;   // the library's EZRT_ERR_INVALID
    return 0;
}

Tables makeTables(const Scene& sc, const ezrt_render_params& p, const float* hdr, int hdrW, int hdrH) {
    Tables tb;
    if (p.mode == EZRT_MODE_DISNEY_LIGHTS) {
        tb.lt = buildLights(sc);
        if (p.reserved[0] & EZRT_PARAM_ENV_LIGHT) tb.env = buildEnv(hdr, hdrW, hdrH);
    }
    return tb;
}

void addCounters(Counters& total, const Counters& cn) {
    for (int k = 0; k < 3; k++) total.rays[k] += cn.rays[k];
    total.nodes += cn.nodes; total.tris += cn.tris; total.hits += cn.hits;
    total.hdr_lookups += cn.hdr_lookups;
    if (cn.max_stack > total.max_stack) total.max_stack = cn.max_stack;
}

void writeCounters(uint64_t* out, const Counters& total, uint64_t samples) {
    if (!out) return;
    out[0] = total.rays[0]; out[1] = total.rays[1]; out[2] = total.rays[2];
    out[3] = total.nodes; out[4] = total.tris; out[5] = total.hits;
    out[6] = total.hdr_lookups; out[7] = samples; out[8] = total.max_stack;
}

}  // namespace

extern "C" {

// ez_lens_setup: returns 1 and out[11] = eye, u0, u1, k, R, or 0 for invalid parameters
int oracle_lens_setup(const float* eye, const float* cam, float R, float f, float* out) {
    ez_lens L;
    if (!ez_lens_setup(eye, cam, R, f, &L)) return 0;
    const float v[11] = {L.eye.x, L.eye.y, L.eye.z, L.u0.x, L.u0.y, L.u0.z, L.u1.x, L.u1.y, L.u1.z, L.k, L.R};
    memcpy(out, v, sizeof(v));
    return 1;
}

// ez_concentric_disk of n pairs (u[2 i], u[2 i + 1]) -> xy[2 i], xy[2 i + 1]
void oracle_concentric_disk(int n, const float* u, float* xy) {
    for (int i = 0; i < n; i++) ez_concentric_disk(u[2 * i], u[2 * i + 1], &xy[2 * i], &xy[2 * i + 1]);
}

// The camera rays of n samples (px[i], py[i], frame[i]) under p (pinhole without the flag): origins, dirs (n x 3), and per sample
// the pinhole direction dir_pin (n x 3), the lens draws (n x 2, 0 without the flag) and the seed the path starts with.
// Returns -2 if the flag's parameters are invalid.
int oracle_camera_rays(const ezrt_render_params* p, int n, const uint32_t* px, const uint32_t* py, const uint32_t* frame, float* o_out,
                       float* d_out, float* dir_pin_out, float* draws_out, uint32_t* seed_out) {
    ez_lens lens;
    const bool on = lensOf(*p, &lens);
    if ((p->reserved[0] & EZRT_PARAM_THIN_LENS) && !on) return -2;
    for (int i = 0; i < n; i++) {
        PixelCtx c;
        c.px = px[i]; c.py = py[i]; c.frameCounter = frame[i];
        PixelCtx c2 = c;
        const vec3 dp = pinholeDir(*p, c2);
        const Ray r = cameraRay(*p, on ? &lens : nullptr, c);
        float ra = 0.0f, rb = 0.0f;
        if (on) ez_lens_draws(c.px, c.py, c.frameCounter, &ra, &rb);
        o_out[3 * i] = r.startPoint.x; o_out[3 * i + 1] = r.startPoint.y; o_out[3 * i + 2] = r.startPoint.z;
        d_out[3 * i] = r.direction.x; d_out[3 * i + 1] = r.direction.y; d_out[3 * i + 2] = r.direction.z;
        if (dir_pin_out) { dir_pin_out[3 * i] = dp.x; dir_pin_out[3 * i + 1] = dp.y; dir_pin_out[3 * i + 2] = dp.z; }
        if (draws_out) { draws_out[2 * i] = ra; draws_out[2 * i + 1] = rb; }
        if (seed_out) seed_out[i] = c.rng.seed;
    }
    return 0;
}

// The window [x0,x1) x [y0,y1) of the p->width x p->height grid into row-major window buffers: framebuffer (out_channels floats
// per pixel), luma2 (running mean of the squared sample luminance) and, when aov is not null, the feature buffers (8 floats:
// albedo.rgb, coverage, normal.xyz, depth) of ezrt_render_aov.  In/out when p->first_frame > 0.  counters_out as
// oracle_render_window's.  Returns -2 if the flag's parameters are invalid.
int oracle_render_lens(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache, int hdrW,
                       int hdrH, int hdrLinear, const ezrt_render_params* p, int x0, int y0, int x1, int y1, float* framebuffer, float* aov,
                       float* luma2, uint64_t* counters_out, int n_threads) {
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
                    const vec3 color = shadePixelLens(sc, tb, *p, on ? &lens : nullptr, (uint32_t)pxl, (uint32_t)py, frame, cn, &h);
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

// The adaptive form (tests/oracle_adaptive.cpp's loop with this file's sample function): the tiles of the window (x0, y0 multiples
// of 16; x1, y1 multiples of 16 or the image edge) into framebuffer, spp_out, luma2_out.  counters_out: samples = sum of spp_out.
int oracle_render_lens_adaptive(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache,
                                int hdrW, int hdrH, int hdrLinear, const ezrt_render_params* p, const ezrt_adaptive_params* ap, int x0, int y0,
                                int x1, int y1, float* framebuffer, int32_t* spp_out, float* luma2_out, uint64_t* counters_out, int n_threads) {
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
                        const vec3 color = shadePixelLens(sc, tb, *p, on ? &lens : nullptr, px, py, (uint32_t)f, cn, nullptr);
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
