// kernels.h -- launchers of kernels.cu (internal to libezrt_b200.so)
#ifndef EZRT_KERNELS_H
#define EZRT_KERNELS_H

#include <algorithm>

#include "device_scene.h"

// extend/shadow kernels: persistent blocks; the register cap of 64 lets 1024 threads reside per SM
#ifndef EZRT_EXTEND_MAX_THREADS
#define EZRT_EXTEND_MAX_THREADS 1024
#endif
#define EZRT_EXTEND_THREADS EZRT_EXTEND_MAX_THREADS
#ifndef EZRT_EXTEND_LB_BLOCKS
#define EZRT_EXTEND_LB_BLOCKS 1
#endif
#define EZRT_EXTEND_BLOCKS_PER_SM 1

// The light sampling mode's options of a render (capi.cu light_options), passed as one value to launch_shade, launch_deferred_lane
// and launch_nee, which pick the k_shade / k_nee instantiation from them:
//   env_on    EZRT_PARAM_ENV_LIGHT and the scene has an environment table: the map is one more light (<.., ENV>)
//   trans_on  EZRT_PARAM_TRANSMISSION: materials with a dielectric lobe (<.., TRANS>)
//   medium_on EZRT_PARAM_MEDIUM with sigma_t > 0: the homogeneous medium med (<.., MEDIUM>); never with trans_on
//   tex_on    EZRT_PARAM_TEXTURES: the scene's base-colour textures tex (<.., TEX>)
//   maps_on   EZRT_PARAM_MATERIAL_MAPS (with tex_on): the material maps of tex (<.., TEX, MAPS>)
// All off outside the light sampling mode; the tables are zero where unused, as the kernels' parameters.
struct LightOptions {
    LightsDev lights{};   // the light table (light sampling mode)
    EnvDev env{};         // the environment table (env_on)
    MediumDev med{};      // the medium (medium_on)
    TexDev tex{};         // the textures and the shadow slots' base colours (tex_on)
    MapsDev maps{};       // the maps' table and the shadow slots' metallic (maps_on)
    bool env_on = false, trans_on = false, medium_on = false, tex_on = false, maps_on = false;
};

// lens (EZRT_PARAM_THIN_LENS): the thin-lens camera rays (k_generate<true>); null: the pinhole's
void launch_generate(const RenderDev& rd, const TileDev* tiles, uint32_t n_slots, uint32_t batch_first_frame, PathQueue q,
                     uint32_t* q_count, int n_sms, cudaStream_t st, const LensDev* lens = nullptr);
void launch_extend(const SceneDev& sc, bool prune, bool anyhit, PathQueue q, const uint32_t* q_count, uint32_t* work,
                   const uint32_t* perm, int to_accel, uint32_t n_max, int n_sms, cudaStream_t st, float2* side_hit = nullptr, int gate = 0);
// counts (params.profile = 2): [0] 128-byte node visits, [1] triangle tests, [2] quantised node visits, then the W8 kernels' phase
// cycles (extend_w8: refill, node steps, triangle steps, ray ends) and their step, visit and test counts (node steps, triangle
// steps, node visits, triangle tests), EZRT_W8_PASS_WORDS from [EZRT_W8_PHASES_EXTEND] (bounce) and from [EZRT_W8_PHASES_SHADOW]
#define EZRT_W8_PASS_WORDS 8
#define EZRT_W8_PHASES_EXTEND 3
#define EZRT_W8_PHASES_SHADOW (EZRT_W8_PHASES_EXTEND + EZRT_W8_PASS_WORDS)
#define EZRT_TOTALS 24   // the render's 64-bit totals: rays, samples, deferred rays, then counts at [5]
// exact_gate: the exact pass over the deferred rays that follows the accel kernel -- 0: always (in line); 2: only when more than
// EZRT_SIDE_CAP rays were deferred (the caller runs launch_deferred_lane on a side stream for the usual handful)
void launch_extend_accel(const SceneDev& sc, PathQueue q, const uint32_t* q_count, uint32_t* work, uint32_t* defer_list,
                         uint32_t* defer_count, uint32_t* defer_work, uint32_t n_max, int n_sms, unsigned long long* counts, const uint32_t* perm,
                         cudaStream_t st, int exact_gate = 0);
void launch_ray_sort(const SceneDev& sc, PathQueue q, const uint32_t* q_count, uint32_t* keys, uint32_t* bins, uint32_t* perm,
                     uint32_t n_max, int n_sms, cudaStream_t st);
void launch_shadow(const SceneDev& sc, bool prune, ShadowQueue sq, const uint32_t* s_count, uint32_t* work, float4* Lo,
                   const uint32_t* perm, uint32_t n_max, int n_sms, cudaStream_t st, bool bounded = false);
// bounded (light sampling mode): shadow ray j looks for occluders strictly before sq.nrm[j].w only
void launch_shadow_accel(const SceneDev& sc, ShadowQueue sq, const uint32_t* s_count, uint32_t* work, float4* Lo, uint32_t* defer_list,
                         uint32_t* defer_count, uint32_t* defer_work, uint32_t n_max, int n_sms, unsigned long long* counts, cudaStream_t st,
                         bool bounded = false);
void launch_shade(const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, int bounce, uint32_t batch_first_frame,
                  PathQueue qin, const uint32_t* in_count, PathQueue qout, uint32_t* out_count, ShadowQueue sq,
                  uint32_t* s_count, float4* Lo, float4* Le, uint32_t n_max, uint32_t n_fused, uint32_t n_frames, int n_sms, cudaStream_t st,
                  float4* aov_rec,   // feature-buffer render, bounce 0 writes the first-hit records (k_shade<.., AOV>); else null
                  const LightOptions& o);
void launch_extend_camera(const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, uint32_t batch_first_frame, uint32_t n_slots, uint32_t n_frames, PathQueue q,
                          uint32_t* work, uint32_t* defer_list, uint32_t* defer_count, uint32_t* defer_work, int n_sms, unsigned long long* counts,
                          cudaStream_t st, int exact_gate = 0);
void launch_deferred_lane(const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, int bounce, uint32_t batch_first_frame, PathQueue qin,
                          const uint32_t* defer_list, const uint32_t* defer_count, uint32_t* defer_work, float2* side_hit, PathQueue qout,
                          uint32_t* out_count, ShadowQueue sq, uint32_t* s_count, float4* Lo, float4* Le, uint32_t n_fused, uint32_t n_frames,
                          int n_sms, cudaStream_t st, float4* aov_rec, const LightOptions& o);
// after a shadow pass (accel or exact, including the exact pass over deferred shadow rays): contributions of the unoccluded light samples
void launch_nee(const SceneDev& sc, const RenderDev& rd, ShadowQueue sq, const uint32_t* s_count, float4* Lo, uint32_t n_max, int n_sms, cudaStream_t st,
                const LightOptions& o);
// light table of the light sampling mode: every triangle's weight (w: n_triangles floats) -> the lights in triangle order
// (idx_out, w_out: n floats each; *count = K) -> their 64-byte records (rec: 4 K float4)
void launch_light_weights(const SceneDev& sc, float* w, cudaStream_t st);
// environment table: the weight of every texel of the scene's map (w: hdr_w * hdr_h floats, row-major)
void launch_env_weights(const SceneDev& sc, float* w, cudaStream_t st);
void launch_light_compact(const float* w, int n, int32_t* idx_out, float* w_out, int32_t* count, cudaStream_t st);
void launch_light_records(const SceneDev& sc, const int32_t* idx, int n, float4* rec, cudaStream_t st);
// running mean of the batch's frames into fb (k_blend).  Adaptive sampling (luma2, spp_map): k_blend<true> also keeps the running mean of
// the squared sample luminance and the per-pixel frame count; the feature-buffer render (luma2, aov_rec, aov; spp_map null):
// k_blend<true, true> also blends the first-hit records of aov_rec into aov (8 floats per pixel).  Null pointers: the plain blend.
void launch_blend(const RenderDev& rd, const TileDev* tiles, int nf, uint32_t batch_first_frame, const float4* Lo, const float4* Le,
                  float* fb, float* luma2, int32_t* spp_map, const float4* aov_rec, float* aov, cudaStream_t st);
// convergence test of the rd.n_tiles tiles of tiles_in after n_frames frames: the surviving tiles -> tiles_out (input order),
// counts[0] = surviving tiles, counts[1] = their in-image pixels; keep holds rd.n_tiles bytes, *blocks_done must be 0 (left 0)
void launch_adaptive_check(const RenderDev& rd, const TileDev* tiles_in, int n_frames, float threshold, const float* fb, const float* luma2,
                           unsigned char* keep, unsigned int* blocks_done, TileDev* tiles_out, int32_t* counts, cudaStream_t st);
void launch_tally(const uint32_t* q_counts, const uint32_t* s_counts, const uint32_t* d_ext, const uint32_t* d_sh, int n_stages,
                  unsigned long long* totals, uint32_t n_primary, cudaStream_t st);
void launch_megakernel(const SceneDev& sc, const RenderDev& rd, const TileDev* tiles, bool prune, int spp, float* fb,
                       unsigned long long* totals, cudaStream_t st, const LensDev* lens = nullptr);
// ezrt_camera_rays: n camera rays (device arrays) -> origins, dirs (n x 3 floats each); lens null: the pinhole's
void launch_camera_rays(const RenderDev& rd, const LensDev* lens, int n, const uint32_t* px, const uint32_t* py, const uint32_t* frame,
                        float* o, float* d, cudaStream_t st);
void launch_trace_finish(const SceneDev& sc, int n, PathQueue q, int p3fudge, int accel_space, int* hit, float* dist, int* tri, int* inside,
                         float* point, float* normal, cudaStream_t st);
void launch_eval_brdf(int which, int n, const float* V, const float* N, const float* L, const float* xi, const float* materials,
                      float* out, cudaStream_t st);
// the transmission mixture for ezrt_eval_bsdf (8 floats out per tuple)
void launch_eval_bsdf(int which, int n, const float* V, const float* N, const float* L, const float* xi, const int* inside,
                      const float* materials, float* out, cudaStream_t st);
// the texcoord records of the accel order: acc_rec[a] = rec[acc_tri_ref[a]] (2 float4 each, n triangles)
void launch_tex_gather(const float4* rec, const uint32_t* acc_tri_ref, int n, float4* acc_rec, cudaStream_t st);
// ezrt_scene_sample_textures: n (reference triangle, point) pairs -> uv (2 floats) and the textured base colour (3 floats) each
void launch_sample_textures(const SceneDev& sc, const TexDev& tex, int n, const int32_t* tri, const float* points, float* uv, float* rgb,
                            cudaStream_t st);
// ezrt_scene_sample_materials: n hits (reference triangle, o, d, t as 7 floats) -> 10 floats each (uv, base colour, roughness,
// metallic, shading normal)
void launch_sample_materials(const SceneDev& sc, const TexDev& tex, const MapsDev& maps, int n, const int32_t* tri, const float* odt, float* out, cudaStream_t st);
// the maps' words (n, reference order) into the fourth word of rec[2 i + 1] and, with acc_tri_ref, of acc_rec[2 a + 1]
void launch_maps_set(const uint32_t* words, const uint32_t* acc_tri_ref, int n, float4* rec, float4* acc_rec, cudaStream_t st);
void launch_eval_math(int which, int n, const float* a, const float* b, float* out, cudaStream_t st);
void launch_tonemap(const float* in, int channels, float* out, long long n, float limit, cudaStream_t st);
void launch_partition_scatter(const float* compact, float* full, const TileDev* tiles, int n_tiles, int width, int channels,
                              cudaStream_t st);
// the a-trous denoiser over a full width x height image: colour (channels 3 or 4) + aov (8 floats, 16-byte aligned) + luma2 after
// n_frames frames -> out (may be color); cv0, cv1: width * height float4 each (ping-pong)
void launch_denoise(const float* color, int channels, const float* aov, const float* luma2, int n_frames, int width, int height, int iterations,
                    float sigma_l, float sigma_n, float sigma_z, float sigma_a, float4* cv0, float4* cv1, float* out, cudaStream_t st);

#endif
