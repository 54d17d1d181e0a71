// kernels_vol.cu -- the volume instantiations (EZRT_PARAM_VOLUMES, DESIGN.md section 21): k_shade<4, LIST, .., TRANS = true, MEDIUM = false,
// .., LTREE = false, GRID = false, VOL = true> for every combination of the light sampling mode's options that has transmission and no
// medium, launched by launch_shade through launch_shade_vol.  kernels_vol_ltree.cu compiles this file's launcher with LTREE = true.
// kernels_vol_medium.cu and kernels_vol_medium_ltree.cu compile it with EZRT_VOL_MEDIUM: k_shade<.., TRANS = true, MEDIUM = true, ..,
// GRID, VOL = true>, the glass inside the homogeneous medium or the density grid, and (kernels_vol_medium.cu) the k_nee<.., TRANS = true,
// MEDIUM = true, .., GRID> of launch_nee_vol_medium.  kernels.cu compiled with EZRT_KERNELS_VOL keeps only k_shade, k_nee and their
// helpers, so the translation units compile side by side.
#ifndef EZRT_VOL_LAUNCH
#define EZRT_VOL_LTREE false
#define EZRT_VOL_MEDIUM false
#define EZRT_VOL_LAUNCH launch_shade_vol
#endif
#define EZRT_KERNELS_VOL
#include "kernels.cu"

template <bool LIST>
static void launch_shade_vol_t(int blocks, const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, int bounce, uint32_t batch_first_frame,
                               PathQueue qin, const uint32_t* in_count, PathQueue qout, uint32_t* out_count, ShadowQueue sq, uint32_t* s_count,
                               float4* Lo, float4* Le, uint32_t n_fused, uint32_t n_frames, const uint32_t* list, const float2* side_hit,
                               float4* aov_rec, const LightOptions& o, cudaStream_t st) {
#if EZRT_VOL_MEDIUM
    with_bools([&](auto A, auto E, auto G, auto TX, auto MP, auto P, auto EM) {
        // the maps with the textures
        if constexpr ((TX || !MP) && (TX || !EM))
            k_shade<EZRT_MODE_DISNEY_LIGHTS, LIST, A, E, true, true, TX, MP, P, EM, EZRT_VOL_LTREE, G, true><<<blocks, 128, 0, st>>>(
                sc, rd, tiles, bounce, batch_first_frame, qin, in_count, qout, out_count, sq, s_count, Lo, Le, n_fused, n_frames, list, side_hit, aov_rec,
                o.lights, o.env, o.med, o.tex, o.maps, o.punct, o.emit, o.tree, o.grid, o.vol);
    }, aov_rec != nullptr, o.env_on, o.grid_on, o.tex_on, o.maps_on, o.punct_on, o.emap_on);
#else
    with_bools([&](auto A, auto E, auto TX, auto MP, auto P, auto EM) {
        // the maps with the textures
        if constexpr ((TX || !MP) && (TX || !EM))
            k_shade<EZRT_MODE_DISNEY_LIGHTS, LIST, A, E, true, false, TX, MP, P, EM, EZRT_VOL_LTREE, false, true><<<blocks, 128, 0, st>>>(
                sc, rd, tiles, bounce, batch_first_frame, qin, in_count, qout, out_count, sq, s_count, Lo, Le, n_fused, n_frames, list, side_hit, aov_rec,
                o.lights, o.env, o.med, o.tex, o.maps, o.punct, o.emit, o.tree, o.grid, o.vol);
    }, aov_rec != nullptr, o.env_on, o.tex_on, o.maps_on, o.punct_on, o.emap_on);
#endif
}

void EZRT_VOL_LAUNCH(bool list, int blocks, const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, int bounce, uint32_t batch_first_frame,
                     PathQueue qin, const uint32_t* in_count, PathQueue qout, uint32_t* out_count, ShadowQueue sq, uint32_t* s_count, float4* Lo,
                     float4* Le, uint32_t n_fused, uint32_t n_frames, const uint32_t* list_idx, const float2* side_hit, float4* aov_rec,
                     const LightOptions& o, cudaStream_t st) {
    if (list)
        launch_shade_vol_t<true>(blocks, sc, rd, tiles, bounce, batch_first_frame, qin, in_count, qout, out_count, sq, s_count, Lo, Le, n_fused, n_frames,
                                 list_idx, side_hit, aov_rec, o, st);
    else
        launch_shade_vol_t<false>(blocks, sc, rd, tiles, bounce, batch_first_frame, qin, in_count, qout, out_count, sq, s_count, Lo, Le, n_fused, n_frames,
                                  list_idx, side_hit, aov_rec, o, st);
}

#if EZRT_VOL_MEDIUM && !EZRT_VOL_LTREE
void launch_nee_vol_medium(int blocks, const SceneDev& sc, const RenderDev& rd, ShadowQueue sq, const uint32_t* s_count, float4* Lo, const LightOptions& o,
                           const TileDev* tiles, int bounce, uint32_t batch_first_frame, cudaStream_t st) {
    with_bools([&](auto E, auto G, auto TX, auto MP, auto P, auto EM) {
        if constexpr ((TX || !MP) && (TX || !EM))
            k_nee<EZRT_MODE_DISNEY_LIGHTS, E, true, true, TX, MP, P, EM, G><<<blocks, 128, 0, st>>>(sc, rd, sq, s_count, Lo, o.med, o.tex, o.maps, o.punct,
                                                                                               o.emit, o.grid, tiles, bounce, batch_first_frame);
    }, o.env_on, o.grid_on, o.tex_on, o.maps_on, o.punct_on, o.emap_on);
}
#endif
