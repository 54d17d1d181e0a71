// oracle_aov.cpp -- CPU restatement of the feature-buffer render (ezrt_render_aov) and of the a-trous denoiser (ezrt_denoise),
// include/ezrt.h; the arithmetic shared with the kernels is ezrt_math.h's.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT, like the oracle it compiles in (build/libezrt_oracle_aov.so, tests/oracle_aov.py).
//
// The render is the oracle's per-pixel loop with its sample function shadePixel.  The first hit of each sample is found by
// re-tracing the sample's camera ray (the same seed, jitter and direction as shadePixel's, main() P5/fsh:915-925) with the
// oracle's hitBVH into a scratch counter set, so the oracle itself is unchanged and the ray counts stay shadePixel's.
// The denoiser is a plain scalar loop over the pixels in the order ezrt_math.h states.
#include "../oracle/ezrt_oracle.cpp"

namespace {

// the first hit of the camera ray of (px, py, frame): exactly the ray shadePixel traces first
HitResult firstHit(const Scene& sc, const ezrt_render_params& p, uint32_t ipx, uint32_t ipy, uint32_t frameCounter) {
    Rng rng;
    rng.seed = (ipx * 1973u + ipy * 9277u + frameCounter * 26699u) | 1u;
    float pixx = EZ_DIV((float)ipx + 0.5f, (float)p.width) * 2.0f - 1.0f;
    float pixy = EZ_DIV((float)ipy + 0.5f, (float)p.height) * 2.0f - 1.0f;
    Ray ray;
    ray.startPoint = ez_v3(p.eye[0], p.eye[1], p.eye[2]);
    float aax = EZ_DIV(rng.rand() - 0.5f, (float)p.width);
    float aay = EZ_DIV(rng.rand() - 0.5f, (float)p.height);
    float vx = pixx + aax, vy = pixy + aay, vz = -1.5f, vw = 0.0f;
    const float* m = p.camera_rotate;
    vec3 dir = ez_v3(((m[0] * vx + m[4] * vy) + m[8] * vz) + m[12] * vw,
                     ((m[1] * vx + m[5] * vy) + m[9] * vz) + m[13] * vw,
                     ((m[2] * vx + m[6] * vy) + m[10] * vz) + m[14] * vw);
    ray.direction = ez_normalize(dir);
    Counters scratch;
    memset(&scratch, 0, sizeof(scratch));
    return hitBVH(sc, ray, scratch, 0);
}

}  // namespace

extern "C" {

// The window [x0,x1) x [y0,y1) of the p->width x p->height grid into row-major window buffers: framebuffer (out_channels
// floats per pixel), aov (8 floats: albedo.rgb, coverage, normal.xyz, depth), luma2 (running mean of the squared sample
// luminance).  All three are in/out when p->first_frame > 0.  counters_out as oracle_render_window's.
int oracle_render_aov(const float* tris, int nTriangles, const float* nodes, int nNodes, const float* hdr, const float* hdrCache, int hdrW,
                      int hdrH, int hdrLinear, const ezrt_render_params* p, int x0, int y0, int x1, int y1, float* framebuffer, float* aov,
                      float* luma2, uint64_t* counters_out, int n_threads) {
    if (!tris || !nodes || !p || !framebuffer || !aov || !luma2 || nTriangles <= 0 || nNodes < 2) return -1;
    if (x0 < 0 || y0 < 0 || x1 > p->width || y1 > p->height || x1 <= x0 || y1 <= y0) return -1;
    if (p->mode == EZRT_MODE_DISNEY_IS_MIS_P5 && (!hdr || !hdrCache)) return -1;
    Scene sc = makeScene(tris, nTriangles, nodes, nNodes, hdr, hdrCache, hdrW, hdrH, hdrLinear, p->env_color, p->mode, p->traverse);
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
                float* feat = aov + k * 8;
                vec3 acc = ez_v3(dst[0], dst[1], dst[2]);
                float m2 = luma2[k];
                if (p->first_frame == 0) {
                    acc = ez_v3(0, 0, 0);
                    m2 = 0.0f;
                    for (int c = 0; c < 8; c++) feat[c] = 0.0f;
                }
                for (int s = 0; s < p->spp; s++) {
                    const uint32_t frame = p->first_frame + (uint32_t)s;
                    const vec3 color = shadePixel(sc, *p, (uint32_t)pxl, (uint32_t)py, frame, cn);
                    const HitResult h = firstHit(sc, *p, (uint32_t)pxl, (uint32_t)py, frame);
                    float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                    if (h.isHit) {
                        const vec3 albedo = getMaterial(sc, h.triangle).baseColor;
                        v[0] = albedo.x; v[1] = albedo.y; v[2] = albedo.z; v[3] = 1.0f;
                        v[4] = h.normal.x; v[5] = h.normal.y; v[6] = h.normal.z; v[7] = h.distance;
                    }
                    const float a = EZ_DIV(1.0f, ez_u32_to_float(frame + 1u));
                    acc = ez_vmix(acc, color, a);
                    const float y = ez_luminance(color);
                    m2 = ez_mix(m2, y * y, a);
                    for (int c = 0; c < 8; c++) feat[c] = ez_mix(feat[c], v[c], a);
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

// ezrt_denoise over a full width x height image: color (channels floats per pixel), aov (8), luma2 (1) after n_frames frames
// -> out (channels floats per pixel; alpha copied; may be color).
int oracle_denoise(const ezrt_denoise_params* dp, const float* color, int channels, const float* aov, const float* luma2, int width,
                   int height, int n_frames, float* out) {
    if (!dp || !color || !aov || !luma2 || !out || width <= 0 || height <= 0 || n_frames < 1) return -1;
    if ((channels != 3 && channels != 4) || dp->iterations < 1 || dp->iterations > 10) return -1;
    const size_t n = (size_t)width * height;
    std::vector<float> cv(4 * n), nx(4 * n);
    for (size_t i = 0; i < n; i++) {
        const vec3 c = ez_v3(color[i * channels], color[i * channels + 1], color[i * channels + 2]);
        cv[4 * i] = c.x; cv[4 * i + 1] = c.y; cv[4 * i + 2] = c.z;
        cv[4 * i + 3] = ez_denoise_var0(luma2[i], c, n_frames);
    }
    for (int k = 0; k < dp->iterations; k++) {
        const int step = 1 << k;
        for (int y = 0; y < height; y++) {
            for (int x = 0; x < width; x++) {
                const size_t p = (size_t)y * width + x;
                const float* fp = aov + 8 * p;
                float* dst = &nx[4 * p];
                if (fp[3] == 0.0f) {   // coverage 0: passed through
                    for (int c = 0; c < 4; c++) dst[c] = cv[4 * p + c];
                    continue;
                }
                const vec3 a_p = ez_v3(fp[0], fp[1], fp[2]), n_p = ez_v3(fp[4], fp[5], fp[6]);
                const float z_p = fp[7];
                const float Y_p = ez_luminance(ez_v3(cv[4 * p], cv[4 * p + 1], cv[4 * p + 2]));
                const float sd_p = EZ_SQRT(cv[4 * p + 3]);
                float sw = 0.0f, sr = 0.0f, sg = 0.0f, sb = 0.0f, sv = 0.0f;
                for (int j = -2; j <= 2; j++) {
                    for (int i = -2; i <= 2; i++) {
                        const int qx = x + step * i, qy = y + step * j;
                        if (qx < 0 || qx >= width || qy < 0 || qy >= height) continue;
                        const size_t q = (size_t)qy * width + qx;
                        const float* cq = &cv[4 * q];
                        const float* fq = aov + 8 * q;
                        const float h = ez_b3(i) * ez_b3(j);
                        float w;
                        if (i == 0 && j == 0) {
                            w = h;
                        } else {
                            if (fq[3] == 0.0f || !ez_finite(cq[0]) || !ez_finite(cq[1]) || !ez_finite(cq[2]) || !ez_finite(cq[3])) continue;
                            const int ai = i < 0 ? -i : i, aj = j < 0 ? -j : j;
                            const int d = ai > aj ? ai : aj;
                            w = ez_atrous_weight(h, (float)(step * d), n_p, ez_v3(fq[4], fq[5], fq[6]), z_p, fq[7], Y_p,
                                                 ez_luminance(ez_v3(cq[0], cq[1], cq[2])), sd_p, a_p, ez_v3(fq[0], fq[1], fq[2]), dp->sigma_l,
                                                 dp->sigma_n, dp->sigma_z, dp->sigma_a);
                        }
                        sw = sw + w;
                        sr = sr + cq[0] * w; sg = sg + cq[1] * w; sb = sb + cq[2] * w;
                        sv = sv + (w * w) * cq[3];
                    }
                }
                dst[0] = EZ_DIV(sr, sw); dst[1] = EZ_DIV(sg, sw); dst[2] = EZ_DIV(sb, sw);
                dst[3] = EZ_DIV(sv, sw * sw);
            }
        }
        cv.swap(nx);
    }
    for (size_t i = 0; i < n; i++)
        for (int c = 0; c < 3; c++) out[i * channels + c] = cv[4 * i + c];
    if (channels == 4)
        for (size_t i = 0; i < n; i++) out[i * 4 + 3] = color[i * 4 + 3];
    return 0;
}

}  // extern "C"
