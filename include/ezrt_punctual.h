/*
 * ezrt_punctual.h -- the punctual lights' table of EZRT_PARAM_PUNCTUAL_LIGHTS (ezrt_math.h, DESIGN.md section 17), built on the
 * host in float64.  Host C++ only: the library (ezrt_scene_set_punctual_lights) and the CPU restatement build it from the same code.
 */
#ifndef EZRT_PUNCTUAL_H
#define EZRT_PUNCTUAL_H

#include <math.h>

#include <vector>

#include "ezrt.h"
#include "ezrt_math.h"

struct EzPunctTable {
    std::vector<int32_t> index;   // J: each light's index among the caller's lights
    std::vector<float> rec;       // 16 J floats (ezrt_math.h)
    std::vector<float> cdf, q;    // J each
    double W = 0.0;
};

/* r: half the diagonal of the box [bmin, bmax] of the triangles' fp32 vertices, in float64 */
static inline double ez_punct_radius(const float bmin[3], const float bmax[3]) {
    const double dx = (double)bmax[0] - bmin[0], dy = (double)bmax[1] - bmin[1], dz = (double)bmax[2] - bmin[2];
    return 0.5 * sqrt(dx * dx + dy * dy + dz * dz);
}

/* Light k's weight, with lum = ez_luminance(color) (fp32):
 *   point 4 pi I lum;  spot 2 pi I lum (1 - cos_i + (cos_i - cos_o) / 3);  directional pi r^2 E lum */
static inline double ez_punct_weight(const ezrt_punctual_light& l, double r) {
    const double lum = (double)ez_luminance(ez_v3(l.color[0], l.color[1], l.color[2]));
    const double I = (double)l.intensity;
    if (l.type == EZRT_PUNCTUAL_POINT) return 4.0 * M_PI * I * lum;
    if (l.type == EZRT_PUNCTUAL_SPOT) {
        const double ci = cos((double)l.inner_cone), co = cos((double)l.outer_cone);
        return 2.0 * M_PI * I * lum * (1.0 - ci + (ci - co) / 3.0);
    }
    return M_PI * r * r * I * lum;
}

/* Validates n lights and builds their table; the box is the scene's vertex box.  Returns -1 on success, or the index of the first
 * invalid light (n for a sum of weights that is not finite) with *why set; *out is written only on success. */
static inline int ez_punct_build(int n, const ezrt_punctual_light* L, const float bmin[3], const float bmax[3], EzPunctTable* out,
                                 const char** why) {
    const double r = ez_punct_radius(bmin, bmax);
    std::vector<double> w((size_t)n);
    for (int k = 0; k < n; k++) {
        const ezrt_punctual_light& l = L[k];
        const float f[13] = {l.position[0], l.position[1], l.position[2], l.direction[0], l.direction[1], l.direction[2], l.color[0],
                             l.color[1], l.color[2], l.intensity, l.inner_cone, l.outer_cone, 0.0f};
        *why = "an unknown type";
        if (l.type < EZRT_PUNCTUAL_POINT || l.type > EZRT_PUNCTUAL_DIRECTIONAL) return k;
        *why = "a non-finite field";
        for (int c = 0; c < 12; c++)
            if (!ez_finite(f[c])) return k;
        *why = "reserved != 0";
        if (l.reserved != 0) return k;
        *why = "a negative colour channel or intensity";
        if (!(l.color[0] >= 0.0f && l.color[1] >= 0.0f && l.color[2] >= 0.0f && l.intensity >= 0.0f)) return k;
        const double d2 = (double)l.direction[0] * l.direction[0] + (double)l.direction[1] * l.direction[1] + (double)l.direction[2] * l.direction[2];
        *why = "a zero-length direction";
        if (l.type != EZRT_PUNCTUAL_POINT && !(d2 > 0.0)) return k;
        *why = "spot cones outside 0 <= inner < outer <= pi/2";
        if (l.type == EZRT_PUNCTUAL_SPOT && !(l.inner_cone >= 0.0f && l.inner_cone < l.outer_cone && l.outer_cone <= (float)(M_PI / 2))) return k;
        w[k] = ez_punct_weight(l, r);
        *why = "a weight that is not finite";
        if (!isfinite(w[k])) return k;
    }
    EzPunctTable t;
    for (int k = 0; k < n; k++)
        if (w[k] > 0.0) t.W += w[k];
    *why = "a sum of weights that is not finite";
    if (!isfinite(t.W)) return n;
    double S = 0.0;
    for (int k = 0; k < n; k++) {
        if (!(w[k] > 0.0)) continue;
        const ezrt_punctual_light& l = L[k];
        S += w[k];
        t.index.push_back(k);
        t.cdf.push_back((float)(S / t.W));
        t.q.push_back((float)(w[k] / t.W));
        const double d2 = (double)l.direction[0] * l.direction[0] + (double)l.direction[1] * l.direction[1] + (double)l.direction[2] * l.direction[2];
        const double dn = (d2 > 0.0) ? sqrt(d2) : 1.0;
        const float rec[16] = {l.position[0], l.position[1], l.position[2], (float)l.type,
                               (float)(l.direction[0] / dn), (float)(l.direction[1] / dn), (float)(l.direction[2] / dn),
                               (float)cos((double)l.outer_cone),
                               l.intensity * l.color[0], l.intensity * l.color[1], l.intensity * l.color[2],
                               (float)cos((double)l.inner_cone), t.q.back(), 0.0f, 0.0f, 0.0f};
        t.rec.insert(t.rec.end(), rec, rec + 16);
    }
    if (!t.cdf.empty()) t.cdf.back() = 1.0f;
    *out = t;
    return -1;
}

#endif /* EZRT_PUNCTUAL_H */
