// oracle_medium_grid.cpp -- CPU restatement of the heterogeneous medium (EZRT_PARAM_MEDIUM_GRID in EZRT_MODE_DISNEY_LIGHTS, ezrt_math.h,
// DESIGN.md section 20).
//   Renders: the light tree's restatement (tests/oracle_light_tree.cpp, and through it the emission maps', punctual lights', ..., and
//   the homogeneous medium's, tests/oracle_medium.cpp) is included unchanged, with only its two medium functions replaced:
//   ez_medium_flight by ez_grid_flight and ez_medium_transmittance by ez_grid_transmittance through the grid set by
//   oracle_grid_render_set, its draws from the shadow stream of the sample's (pixel, frame, bounce).  The bounce is the count of the
//   path's free flights so far (each loop draws its flight once per segment, before that vertex's light sample); the pixel and frame
//   are the PixelCtx that holds the path's seed.  Without a grid set both are the homogeneous medium's, bit for bit.
//   Definition: the brick maxima, the lookup, and the brick walk's tracking restated with counters -- every tentative collision's
//   sigma against its majorant m (the definition's, which must never exceed m, and the lookup's without the brick clamp).
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT (build/libezrt_oracle_medium_grid.so, tests/oracle_medium_grid.py).
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <vector>

#include "ezrt_math.h"

int gridFlightHook(const ez_medium* m, ez_vec3 o, ez_vec3 d, float t_end, uint32_t* seed, float* t_s);
float gridTransmittanceHook(const ez_medium* m, ez_vec3 o, ez_vec3 d, float L);
#define ez_medium_flight gridFlightHook
#define ez_medium_transmittance gridTransmittanceHook
#include "oracle_light_tree.cpp"
#undef ez_medium_flight
#undef ez_medium_transmittance

namespace {

struct GridStats {
    unsigned long long collisions = 0;   // tentative collisions evaluated
    unsigned long long violations = 0;   // sigma > m with the definition's lookup (must stay 0)
    unsigned long long outside = 0;      // sigma > m with the lookup clamped to the lattice only (the brick clamp absorbed these)
    unsigned long long clamped = 0;      // lookups whose brick clamp moved the lattice coordinate
};

struct GridSet {
    ez_medium med;
    ez_grid g;
    std::vector<float> brick;
};

void gridSetOf(const float* med7, int nx, int ny, int nz, const float* rho, GridSet* gs) {
    gs->med = ez_medium{};
    gs->med.sigma_t = med7[0];
    gs->med.bmin = ez_v3(med7[1], med7[2], med7[3]);
    gs->med.bmax = ez_v3(med7[4], med7[5], med7[6]);
    gs->g = ez_grid{};
    gs->g.rho = rho;
    gs->g.n[0] = nx; gs->g.n[1] = ny; gs->g.n[2] = nz;
    for (int a = 0; a < 3; a++) gs->g.b[a] = ez_grid_bricks(gs->g.n[a]);
    gs->brick.assign((size_t)gs->g.b[0] * gs->g.b[1] * gs->g.b[2], 0.0f);
    for (int k = 0; k < gs->g.b[2]; k++)
        for (int j = 0; j < gs->g.b[1]; j++)
            for (int i = 0; i < gs->g.b[0]; i++) gs->brick[((size_t)k * gs->g.b[1] + j) * gs->g.b[0] + i] = ez_grid_brick_max(&gs->g, i, j, k);
    gs->g.brick = gs->brick.data();
}

// sigma at o + t d for the walk's brick b, with the counters
float gridSigmaAt(const GridSet& gs, ez_vec3 o, ez_vec3 d, float t, const int* b, float m, GridStats* st) {
    const ez_vec3 x = ez_add(o, ez_scale(d, t));
    int cl = 0;
    const float s = gs.med.sigma_t * ez_grid_rho(&gs.g, gs.med.bmin, gs.med.bmax, x, b, &cl);
    const float su = gs.med.sigma_t * ez_grid_rho(&gs.g, gs.med.bmin, gs.med.bmax, x, nullptr, nullptr);
    st->collisions++;
    st->violations += (s > m);
    st->outside += (su > m);
    st->clamped += (unsigned long long)cl;
    return s;
}

// ez_grid_flight and ez_grid_transmittance (which 1 / 2), restated with the counters
int gridTrack(const GridSet& gs, int which, ez_vec3 o, ez_vec3 d, float L, uint32_t* seed, float* out, GridStats* st) {
    const ez_medium& m = gs.med;
    float t0, t1;
    *out = (which == 2) ? 1.0f : 0.0f;
    if (!(m.sigma_t > 0.0f) || !ez_box_overlap(o, d, m.bmin, m.bmax, L, &t0, &t1)) return 0;
    ez_grid_walk w;
    ez_grid_walk_begin(&gs.g, o, d, m.bmin, m.bmax, t0, t1, &w);
    float T = 1.0f, tb;
    while (ez_grid_walk_interval(&w, &tb)) {
        const float mj = ez_grid_majorant(&gs.g, m.sigma_t, w.b);
        if (mj > 0.0f && w.ta < tb) {
            float t = w.ta;
            for (;;) {
                t = ez_grid_advance(t, ez_free_flight(ez_rand01(seed), mj));
                if (!(t < tb)) break;
                if (which == 1) {
                    const float r2 = ez_rand01(seed);
                    if (r2 * mj < gridSigmaAt(gs, o, d, t, w.b, mj, st)) {
                        *out = t;
                        return 1;
                    }
                } else {
                    T = T * EZ_DIV(mj - gridSigmaAt(gs, o, d, t, w.b, mj, st), mj);
                    if (!(T > 0.0f)) { *out = 0.0f; return 0; }
                    if (T < 0.0625f) {
                        if (!(ez_rand01(seed) < 0.25f)) { *out = 0.0f; return 0; }
                        T = T * 4.0f;
                    }
                }
            }
        }
        ez_grid_walk_next(&gs.g, o, d, m.bmin, m.bmax, &w, tb);
    }
    if (which == 2) *out = T;
    return 0;
}

// the grid of the flagged renders (oracle_grid_render_set; null: the homogeneous medium), and each thread's path: the PixelCtx of its
// seed and the count of its free flights, restarted when the pixel, frame or render changes
GridSet* g_render_grid = nullptr;
uint64_t g_render_gen = 0;
struct PathKey {
    uint64_t gen = ~0ull;
    uint32_t px = 0, py = 0, frame = 0;
    int bounce = 0;
};
thread_local PathKey t_path;

}  // namespace

int gridFlightHook(const ez_medium* m, ez_vec3 o, ez_vec3 d, float t_end, uint32_t* seed, float* t_s) {
    if (!g_render_grid) return ez_medium_flight(m, o, d, t_end, seed, t_s);
    const PixelCtx* px = (const PixelCtx*)((const char*)seed - offsetof(Rng, seed) - offsetof(PixelCtx, rng));
    if (t_path.gen != g_render_gen || t_path.px != px->px || t_path.py != px->py || t_path.frame != px->frameCounter) {
        t_path.gen = g_render_gen; t_path.px = px->px; t_path.py = px->py; t_path.frame = px->frameCounter;
        t_path.bounce = 0;
    } else {
        t_path.bounce++;
    }
    return ez_grid_flight(m, &g_render_grid->g, o, d, t_end, seed, t_s);
}

float gridTransmittanceHook(const ez_medium* m, ez_vec3 o, ez_vec3 d, float L) {
    if (!g_render_grid) return ez_medium_transmittance(m, o, d, L);
    uint32_t s = ez_grid_shadow_seed(t_path.px, t_path.py, t_path.frame, (uint32_t)t_path.bounce);
    return ez_grid_transmittance(m, &g_render_grid->g, o, d, L, &s);
}

extern "C" {

// the grid of the renders that follow (rho null: none, the homogeneous medium's renders); brick_scale scales its brick maxima
// (test-only, 1 for the definition's)
void oracle_grid_render_set(int nx, int ny, int nz, const float* rho, float brick_scale) {
    static GridSet gs;
    static std::vector<float> copy;
    g_render_gen++;
    if (!rho) {
        g_render_grid = nullptr;
        return;
    }
    copy.assign(rho, rho + (size_t)nx * ny * nz);
    const float med7[7] = {1, 0, 0, 0, 1, 1, 1};
    gridSetOf(med7, nx, ny, nz, copy.data(), &gs);
    for (float& b : gs.brick) b = b * brick_scale;
    g_render_grid = &gs;
}

// the brick maxima of the grid (bricks x fastest; cap >= the count, or null): returns the brick count; dims_out[3]: bricks per axis
int oracle_grid_bricks(int nx, int ny, int nz, const float* rho, int cap, float* out, int32_t* dims_out) {
    const float med7[7] = {1, 0, 0, 0, 1, 1, 1};
    GridSet gs;
    gridSetOf(med7, nx, ny, nz, rho, &gs);
    const int B = (int)gs.brick.size();
    if (out && cap >= B) memcpy(out, gs.brick.data(), sizeof(float) * B);
    if (dims_out)
        for (int a = 0; a < 3; a++) dims_out[a] = gs.g.b[a];
    return B;
}

// med7 = (sigma_t, box min, box max).  which 0: sigma at the points o -> out (lattice clamp only, as ezrt_scene_medium_eval);
// which 1: the free flight (o, d, t_end = L) from seed -> flag, t_s (out), the advanced seed (seed_out); which 2: the ratio-tracked
// transmittance (o, d, L) from seed -> out.  twin: the header's own ez_grid_flight / ez_grid_transmittance into flag2 / out2 /
// seed_out2 (null: skipped), for the restatement's agreement with them.  stats[4]: the counters (GridStats).  brick_scale scales the
// brick maxima (test-only, 1 for the definition's).
void oracle_grid_eval(const float* med7, int nx, int ny, int nz, const float* rho, int which, int n, const float* o, const float* d,
                      const float* L, const uint32_t* seed, int32_t* flag, float* out, uint32_t* seed_out, int32_t* flag2, float* out2,
                      uint32_t* seed_out2, unsigned long long* stats, float brick_scale) {
    GridSet gs;
    gridSetOf(med7, nx, ny, nz, rho, &gs);
    for (float& b : gs.brick) b = b * brick_scale;
    GridStats st;
#ifdef _OPENMP
#pragma omp parallel
#endif
    {
        GridStats my;
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 1024)
#endif
        for (int i = 0; i < n; i++) {
            const ez_vec3 oi = ez_v3(o[3 * i], o[3 * i + 1], o[3 * i + 2]);
            if (which == 0) {
                out[i] = gs.med.sigma_t * ez_grid_rho(&gs.g, gs.med.bmin, gs.med.bmax, oi, nullptr, nullptr);
                continue;
            }
            const ez_vec3 di = ez_v3(d[3 * i], d[3 * i + 1], d[3 * i + 2]);
            uint32_t s = seed[i];
            const int f = gridTrack(gs, which, oi, di, L[i], &s, &out[i], &my);
            if (flag) flag[i] = f;
            if (seed_out) seed_out[i] = s;
            if (out2) {
                uint32_t s2 = seed[i];
                if (which == 1) {
                    float t_s = 0.0f;
                    const int f2 = ez_grid_flight(&gs.med, &gs.g, oi, di, L[i], &s2, &t_s);
                    out2[i] = f2 ? t_s : 0.0f;
                    if (flag2) flag2[i] = f2;
                } else {
                    out2[i] = ez_grid_transmittance(&gs.med, &gs.g, oi, di, L[i], &s2);
                }
                if (seed_out2) seed_out2[i] = s2;
            }
        }
#ifdef _OPENMP
#pragma omp critical
#endif
        {
            st.collisions += my.collisions; st.violations += my.violations; st.outside += my.outside; st.clamped += my.clamped;
        }
    }
    if (stats) { stats[0] = st.collisions; stats[1] = st.violations; stats[2] = st.outside; stats[3] = st.clamped; }
}

// the shadow stream's seeds of n (pixel, frame, bounce) tuples
void oracle_grid_shadow_seed(int n, const uint32_t* px, const uint32_t* py, const uint32_t* frame, const uint32_t* bounce, uint32_t* out) {
    for (int i = 0; i < n; i++) out[i] = ez_grid_shadow_seed(px[i], py[i], frame[i], bounce[i]);
}

}  // extern "C"
