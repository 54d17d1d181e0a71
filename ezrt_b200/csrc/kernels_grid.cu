// kernels_grid.cu -- the density-grid instantiations (EZRT_PARAM_MEDIUM_GRID, DESIGN.md section 20): k_shade<4, LIST, .., MEDIUM = true, ..,
// LTREE = false, GRID = true> and k_nee<4, .., MEDIUM = true, .., GRID = true> for every combination of the light sampling mode's options
// that has the medium, launched by launch_shade and launch_nee through launch_shade_grid and launch_nee_grid, and the kernel of
// ezrt_scene_medium_eval.  kernels_grid_ltree.cu compiles this file's k_shade launcher with LTREE = true.  kernels.cu compiled with
// EZRT_KERNELS_GRID keeps only k_shade, k_nee and their helpers, so the translation units compile side by side.
#ifndef EZRT_GRID_LTREE
#define EZRT_KERNELS_GRID
#define EZRT_GRID_LTREE false
#define EZRT_GRID_LAUNCH launch_shade_grid
#endif
#include "kernels.cu"

template <bool LIST>
static void launch_shade_grid_t(int blocks, const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, int bounce, uint32_t batch_first_frame,
                                PathQueue qin, const uint32_t* in_count, PathQueue qout, uint32_t* out_count, ShadowQueue sq, uint32_t* s_count,
                                float4* Lo, float4* Le, uint32_t n_fused, uint32_t n_frames, const uint32_t* list, const float2* side_hit,
                                float4* aov_rec, const LightOptions& o, cudaStream_t st) {
    with_bools([&](auto A, auto E, auto TX, auto MP, auto P, auto EM) {
        // the medium without transmission; the maps with the textures
        if constexpr ((TX || !MP) && (TX || !EM))
            k_shade<EZRT_MODE_DISNEY_LIGHTS, LIST, A, E, false, true, TX, MP, P, EM, EZRT_GRID_LTREE, true><<<blocks, 128, 0, st>>>(
                sc, rd, tiles, bounce, batch_first_frame, qin, in_count, qout, out_count, sq, s_count, Lo, Le, n_fused, n_frames, list, side_hit, aov_rec,
                o.lights, o.env, o.med, o.tex, o.maps, o.punct, o.emit, o.tree, o.grid, o.vol);
    }, aov_rec != nullptr, o.env_on, o.tex_on, o.maps_on, o.punct_on, o.emap_on);
}

void EZRT_GRID_LAUNCH(bool list, int blocks, const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, int bounce, uint32_t batch_first_frame,
                      PathQueue qin, const uint32_t* in_count, PathQueue qout, uint32_t* out_count, ShadowQueue sq, uint32_t* s_count, float4* Lo,
                      float4* Le, uint32_t n_fused, uint32_t n_frames, const uint32_t* list_idx, const float2* side_hit, float4* aov_rec,
                      const LightOptions& o, cudaStream_t st) {
    if (list)
        launch_shade_grid_t<true>(blocks, sc, rd, tiles, bounce, batch_first_frame, qin, in_count, qout, out_count, sq, s_count, Lo, Le, n_fused, n_frames,
                                  list_idx, side_hit, aov_rec, o, st);
    else
        launch_shade_grid_t<false>(blocks, sc, rd, tiles, bounce, batch_first_frame, qin, in_count, qout, out_count, sq, s_count, Lo, Le, n_fused, n_frames,
                                   list_idx, side_hit, aov_rec, o, st);
}

#if !EZRT_GRID_LTREE
void launch_nee_grid(int blocks, const SceneDev& sc, const RenderDev& rd, ShadowQueue sq, const uint32_t* s_count, float4* Lo, const LightOptions& o,
                     const TileDev* tiles, int bounce, uint32_t batch_first_frame, cudaStream_t st) {
    with_bools([&](auto E, auto TX, auto MP, auto P, auto EM) {
        if constexpr ((TX || !MP) && (TX || !EM))
            k_nee<EZRT_MODE_DISNEY_LIGHTS, E, false, true, TX, MP, P, EM, true><<<blocks, 128, 0, st>>>(sc, rd, sq, s_count, Lo, o.med, o.tex, o.maps,
                                                                                                     o.punct, o.emit, o.grid, tiles, bounce,
                                                                                                     batch_first_frame);
    }, o.env_on, o.tex_on, o.maps_on, o.punct_on, o.emap_on);
}

__global__ void __launch_bounds__(128) k_medium_eval(MediumDev med, GridDev grid, int which, int n, const float* __restrict__ o,
                                                     const float* __restrict__ d, const float* __restrict__ L, const uint32_t* __restrict__ seed,
                                                     int32_t* __restrict__ out_i, float* __restrict__ out0, uint32_t* __restrict__ seed_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const vec3 oi = ez_v3(o[3 * i], o[3 * i + 1], o[3 * i + 2]);
    if (which == 0) {
        out0[i] = med.sigma_t * ez_grid_rho(&grid, med.bmin, med.bmax, oi, nullptr, nullptr);
        return;
    }
    const vec3 di = ez_v3(d[3 * i], d[3 * i + 1], d[3 * i + 2]);
    uint32_t s = seed[i];
    if (which == 1) {
        float t_s = 0.0f;
        out_i[i] = ez_grid_flight(&med, &grid, oi, di, L[i], &s, &t_s);
        out0[i] = t_s;
        seed_out[i] = s;
    } else {
        out0[i] = ez_grid_transmittance(&med, &grid, oi, di, L[i], &s);
    }
}

void launch_medium_eval(const MediumDev& med, const GridDev& grid, int which, int n, const float* o, const float* d, const float* L,
                        const uint32_t* seed, int32_t* out_i, float* out0, uint32_t* seed_out, cudaStream_t st) {
    if (n > 0) k_medium_eval<<<div_up(n, 128), 128, 0, st>>>(med, grid, which, n, o, d, L, seed, out_i, out0, seed_out);
}
#endif
