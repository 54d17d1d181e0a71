// kernels_ltree.cu -- the light-tree instantiations of k_shade (EZRT_PARAM_LIGHT_TREE, DESIGN.md section 19): k_shade<4, LIST, ..,
// LTREE = true> for every combination of the light sampling mode's options, launched by launch_shade through launch_shade_ltree.
// kernels.cu compiled with EZRT_KERNELS_LTREE keeps only what k_shade needs, so the two translation units compile side by side.
#define EZRT_KERNELS_LTREE
#include "kernels.cu"

template <bool LIST>
static void launch_shade_ltree_t(int blocks, const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, int bounce, uint32_t batch_first_frame,
                                 PathQueue qin, const uint32_t* in_count, PathQueue qout, uint32_t* out_count, ShadowQueue sq, uint32_t* s_count,
                                 float4* Lo, float4* Le, uint32_t n_fused, uint32_t n_frames, const uint32_t* list, const float2* side_hit,
                                 float4* aov_rec, const LightOptions& o, cudaStream_t st) {
    with_bools([&](auto A, auto E, auto T, auto X, auto TX, auto MP, auto P, auto EM) {
        // the medium without transmission; the maps with the textures
        if constexpr (!(T && X) && (TX || !MP) && (TX || !EM))
            k_shade<EZRT_MODE_DISNEY_LIGHTS, LIST, A, E, T, X, TX, MP, P, EM, true><<<blocks, 128, 0, st>>>(
                sc, rd, tiles, bounce, batch_first_frame, qin, in_count, qout, out_count, sq, s_count, Lo, Le, n_fused, n_frames, list, side_hit, aov_rec,
                o.lights, o.env, o.med, o.tex, o.maps, o.punct, o.emit, o.tree, o.grid, o.vol);
    }, aov_rec != nullptr, o.env_on, o.trans_on, o.medium_on, o.tex_on, o.maps_on, o.punct_on, o.emap_on);
}

void launch_shade_ltree(bool list, int blocks, const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, int bounce, uint32_t batch_first_frame,
                        PathQueue qin, const uint32_t* in_count, PathQueue qout, uint32_t* out_count, ShadowQueue sq, uint32_t* s_count, float4* Lo,
                        float4* Le, uint32_t n_fused, uint32_t n_frames, const uint32_t* list_idx, const float2* side_hit, float4* aov_rec,
                        const LightOptions& o, cudaStream_t st) {
    if (list)
        launch_shade_ltree_t<true>(blocks, sc, rd, tiles, bounce, batch_first_frame, qin, in_count, qout, out_count, sq, s_count, Lo, Le, n_fused, n_frames,
                                   list_idx, side_hit, aov_rec, o, st);
    else
        launch_shade_ltree_t<false>(blocks, sc, rd, tiles, bounce, batch_first_frame, qin, in_count, qout, out_count, sq, s_count, Lo, Le, n_fused, n_frames,
                                    list_idx, side_hit, aov_rec, o, st);
}
