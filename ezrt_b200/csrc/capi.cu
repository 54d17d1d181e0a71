// capi.cu -- device half of the C ABI (include/ezrt.h): scene upload/repack, render
// orchestration (wavefront + megakernel), image partition helpers and the single-function
// test entry points.  Host-side scene building lives in host_scene.cpp.
#include <cuda_runtime.h>

#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <array>
#include <map>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "device_scene.h"
#include "ezrt.h"
#include "ezrt_internal.h"
#include "ezrt_math.h"
#include "kernels.h"
#include "w8_node.h"

#define CU_CHECK(call)                                                                                  \
    do {                                                                                                \
        cudaError_t e__ = (call);                                                                       \
        if (e__ != cudaSuccess)                                                                         \
            return ezrt_set_error(EZRT_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), \
                                  __FILE__, __LINE__);                                                  \
    } while (0)

namespace {

struct DeviceBuffer {
    void* p = nullptr;
    size_t bytes = 0;
    int ensure(size_t need) {
        if (need <= bytes) return EZRT_OK;
        if (p) cudaFree(p);
        p = nullptr;
        bytes = 0;
        cudaError_t e = cudaMalloc(&p, need);
        if (e != cudaSuccess) return ezrt_set_error(EZRT_ERR_NOMEM, "cudaMalloc(%zu) failed: %s", need, cudaGetErrorString(e));
        bytes = need;
        return EZRT_OK;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        bytes = 0;
    }
};

// tiles of part `rank` of `count` (ezrt_internal.h): row-major tile order, (tx+ty)%count == rank
std::vector<TileDev> partition_tiles(int width, int height, int rank, int count) {
    std::vector<TileDev> tiles;
    int tx_n = (width + EZRT_TILE - 1) / EZRT_TILE, ty_n = (height + EZRT_TILE - 1) / EZRT_TILE;
    int offset = 0;
    for (int ty = 0; ty < ty_n; ty++)
        for (int tx = 0; tx < tx_n; tx++) {
            if ((tx + ty) % count != rank) continue;
            TileDev t;
            t.x0 = tx * EZRT_TILE;
            t.y0 = ty * EZRT_TILE;
            t.w = std::min(EZRT_TILE, width - t.x0);
            t.h = std::min(EZRT_TILE, height - t.y0);
            t.pixel_offset = offset;
            offset += t.w * t.h;
            tiles.push_back(t);
        }
    return tiles;
}

}  // namespace

struct ezrt_scene {
    int device = 0;
    int n_sms = 148;
    SceneDev dev{};
    DeviceBuffer nodes, tri_geo, tri_shade, materials, hdr, hdr_cache;
    DeviceBuffer acc_hot, acc_tri_ref, tri_leaf, leaf_box, defer_buf, acc_tri_leaf, ref_to_acc, acc_wide, acc_wide_q16;   // acc_hot = W8 nodes | geometry (| vertices) | shading records of the accel order
    int acc_depth = 0;
    int n_materials = 0;
    int tree_depth = 0;
    // render state (lazily sized)
    DeviceBuffer tiles_buf, queue_buf[2], shadow_buf, lo_buf, le_buf, counters_buf, totals_buf, fb_buf, sort_buf;
    // adaptive sampling: two surviving-tile lists (ping-pong), per-tile verdicts, the test's counters; the host entry point's spp map + luma2
    DeviceBuffer adapt_buf, adapt_maps_buf;
    // feature-buffer renders: the first-hit records of a batch (32 B per sample slot); the host entry point's aov + luma2.
    // The denoiser: its ping-pong (colour, variance) images; the host entry point's device copies of its inputs
    DeviceBuffer aov_rec_buf, aov_maps_buf, denoise_buf, denoise_io_buf;
    // the light table of the light sampling mode (build_lights, at its first use): records | cdf
    DeviceBuffer lights_buf;
    bool lights_built = false;
    LightsDev lights{};
    std::vector<int32_t> light_tri;   // the lights' triangles (caller's order)
    std::vector<float> light_cdf;
    double light_total = 0.0;         // W, the float64 sum of the weights
    // the environment map's light table (build_env, at the first render with EZRT_PARAM_ENV_LIGHT): row cdf | column cdf | texel pdf
    DeviceBuffer env_buf;
    bool env_built = false;
    EnvDev env{};                     // row_cdf null: the scene has no table (no map, or no texel of positive weight)
    double env_total = 0.0;           // T, the float64 sum of the texel weights
    // the homogeneous medium of EZRT_PARAM_MEDIUM (ezrt_scene_set_medium), copied into the kernels' parameters at every render
    bool has_medium = false;
    MediumDev medium{};
    // the base-colour textures of EZRT_PARAM_TEXTURES (ezrt_scene_set_textures): sRGB table | texture table | texels, and the texcoord
    // records in reference | accel order; tex.sh_base is set per render
    DeviceBuffer tex_buf, tex_rec_buf;
    bool has_textures = false;
    // the material maps of EZRT_PARAM_MATERIAL_MAPS (ezrt_scene_set_material_maps): their ids live in the texcoord records' fourth word
    bool has_maps = false;
    int n_textures = 0;
    TexDev tex{};
    MapsDev maps{};   // maps.sh_metal is set per render
    void* hot_base = nullptr;   // accel nodes | geometry (| vertices) | shading records (L2 persisting window)
    size_t hot_bytes = 0;
    size_t l2_persist_bytes = 0;
    size_t max_window_bytes = 0;  // persisting L2 set-aside granted by the device (0 = feature off)
    bool regular_tree = true;  // false: only the literal REFERENCE traversal is valid for the caller's tree
    bool have_accel = true;    // false: no acceleration tree (irregular caller tree, or a degenerate one too deep for the stacks): ACCEL runs as PRUNED
    int camera_pixel_major = 1;  // camera pass: a warp traces the samples of one pixel (env EZRT_CAMERA_ORDER=frame: an 8x4 block of one frame)
    int sort_rays = 0;  // env EZRT_SORT_RAYS=1 enables the bounce-ray sort (measured: no gain with per-lane refill)
    int tiles_key[4] = {-1, -1, -1, -1};
    std::vector<TileDev> tiles;
    size_t n_pixels = 0;       // pixels of the owned tiles
    size_t fmax = 0, fmax_key[2] = {0, 0};   // frames per batch that fit the free memory, for (slots per frame, bytes per slot)
    cudaStream_t own_stream = nullptr, copy_stream = nullptr;
    // the accel policy's deferred lane: exact traversal + shading of the few deferred rays beside the main k_shade (DESIGN.md)
    cudaStream_t side_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    DeviceBuffer side_hit_buf;
    int deferred_lane = 1;   // env EZRT_DEFERRED_LANE=0: the exact pass in line, as in round 1
    cudaEvent_t fb_event = nullptr, fb_wait = nullptr;   // ezrt_render: the H2D of lastFrame runs beside the tracing kernels
    cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
    bool have_timing = false;
    unsigned long long launches = 0;
    // params.profile: one event pair per launch, summed per kernel class by ezrt_get_kernel_times
    std::vector<cudaEvent_t> ev_pool;
    struct Span { int cls; int e0, e1; };
    std::vector<Span> spans;
    size_t ev_used = 0;
    bool profiling = false;
    int span_begin(int cls, cudaStream_t st) {
        if (!profiling) return -1;
        while (ev_pool.size() < ev_used + 2) {
            cudaEvent_t e;
            if (cudaEventCreate(&e) != cudaSuccess) return -1;
            ev_pool.push_back(e);
        }
        Span sp{cls, (int)ev_used, (int)ev_used + 1};
        ev_used += 2;
        cudaEventRecord(ev_pool[sp.e0], st);
        spans.push_back(sp);
        return (int)spans.size() - 1;
    }
    void span_end(int id, cudaStream_t st) {
        if (id >= 0) cudaEventRecord(ev_pool[spans[id].e1], st);
    }
};

namespace {

int carve_queue(DeviceBuffer& buf, size_t capacity, PathQueue& q) {
    size_t per = sizeof(float4) * 4 + sizeof(float2);
    int rc = buf.ensure(per * capacity + 256);
    if (rc) return rc;
    char* p = (char*)buf.p;
    q.ray_o = (float4*)p; p += sizeof(float4) * capacity;
    q.ray_d = (float4*)p; p += sizeof(float4) * capacity;
    q.hist = (float4*)p;  p += sizeof(float4) * capacity;
    q.fr = (float4*)p;    p += sizeof(float4) * capacity;
    q.hit = (float2*)p;
    return EZRT_OK;
}
int carve_shadow(DeviceBuffer& buf, size_t capacity, ShadowQueue& q) {
    int rc = buf.ensure((size_t)EZRT_SHADOW_SLOT_BYTES * capacity + 256);
    if (rc) return rc;
    char* p = (char*)buf.p;
    q.ray_o = (float4*)p; p += sizeof(float4) * capacity;
    q.ray_d = (float4*)p; p += sizeof(float4) * capacity;
    q.nrm = (float4*)p;   p += sizeof(float4) * capacity;
    q.view = (float4*)p;  p += sizeof(float4) * capacity;
    q.hist = (float4*)p;  p += sizeof(float4) * capacity;
    q.lit = (unsigned char*)p;
    return EZRT_OK;
}

// EZRT_PARAM_THIN_LENS: true with the lens in *lens when the flag is set and its parameters are valid (ez_lens_setup)
bool thin_lens(const ezrt_render_params* p, LensDev* lens) {
    if (!(p->reserved[0] & EZRT_PARAM_THIN_LENS)) return false;
    float R, f;
    memcpy(&R, &p->reserved[1], sizeof(float));
    memcpy(&f, &p->reserved[2], sizeof(float));
    return ez_lens_setup(p->eye, p->camera_rotate, R, f, lens) != 0;
}

int validate_params(const ezrt_scene* scene, const ezrt_render_params* p) {
    if (!scene || !p) return ezrt_set_error(EZRT_ERR_INVALID, "render: null argument");
    if (p->width <= 0 || p->height <= 0 || p->spp < 0) return ezrt_set_error(EZRT_ERR_INVALID, "render: bad image size/spp");
    if (p->mode < 0 || p->mode > EZRT_MODE_DISNEY_LIGHTS) return ezrt_set_error(EZRT_ERR_INVALID, "render: unknown mode %d", p->mode);
    if (p->mode == EZRT_MODE_DISNEY_LIGHTS && p->pipeline == EZRT_PIPELINE_MEGAKERNEL)
        return ezrt_set_error(EZRT_ERR_INVALID, "render: the light sampling mode runs on the wavefront pipeline only");
    if ((p->reserved[0] & EZRT_PARAM_ENV_LIGHT) && p->mode != EZRT_MODE_DISNEY_LIGHTS)
        return ezrt_set_error(EZRT_ERR_INVALID, "render: EZRT_PARAM_ENV_LIGHT needs the light sampling mode (got mode %d)", p->mode);
    if ((p->reserved[0] & EZRT_PARAM_TRANSMISSION) && p->mode != EZRT_MODE_DISNEY_LIGHTS)
        return ezrt_set_error(EZRT_ERR_INVALID, "render: EZRT_PARAM_TRANSMISSION needs the light sampling mode (got mode %d)", p->mode);
    LensDev lens;
    if (!thin_lens(p, &lens) && (p->reserved[0] & EZRT_PARAM_THIN_LENS))
        return ezrt_set_error(EZRT_ERR_INVALID, "render: EZRT_PARAM_THIN_LENS needs a finite lens radius and focus distance > 0 and columns 0-2 "
                                                "of camera_rotate of finite, non-zero length");
    if (p->reserved[0] & EZRT_PARAM_MEDIUM) {
        if (p->mode != EZRT_MODE_DISNEY_LIGHTS)
            return ezrt_set_error(EZRT_ERR_INVALID, "render: EZRT_PARAM_MEDIUM needs the light sampling mode (got mode %d)", p->mode);
        if (p->reserved[0] & EZRT_PARAM_TRANSMISSION)
            return ezrt_set_error(EZRT_ERR_INVALID, "render: EZRT_PARAM_MEDIUM is not rendered with EZRT_PARAM_TRANSMISSION (glass is defined with vacuum outside)");
        if (!scene->has_medium) return ezrt_set_error(EZRT_ERR_INVALID, "render: EZRT_PARAM_MEDIUM needs a medium (ezrt_scene_set_medium)");
    }
    if (p->reserved[0] & EZRT_PARAM_TEXTURES) {
        if (p->mode != EZRT_MODE_DISNEY_LIGHTS)
            return ezrt_set_error(EZRT_ERR_INVALID, "render: EZRT_PARAM_TEXTURES needs the light sampling mode (got mode %d)", p->mode);
        if (!scene->has_textures) return ezrt_set_error(EZRT_ERR_INVALID, "render: EZRT_PARAM_TEXTURES needs textures (ezrt_scene_set_textures)");
    }
    if (p->reserved[0] & EZRT_PARAM_MATERIAL_MAPS) {
        if (!(p->reserved[0] & EZRT_PARAM_TEXTURES))
            return ezrt_set_error(EZRT_ERR_INVALID, "render: EZRT_PARAM_MATERIAL_MAPS needs EZRT_PARAM_TEXTURES");
        if (!scene->has_maps) return ezrt_set_error(EZRT_ERR_INVALID, "render: EZRT_PARAM_MATERIAL_MAPS needs maps (ezrt_scene_set_material_maps)");
    }
    if (p->max_bounce < 0 || p->max_bounce > 64) return ezrt_set_error(EZRT_ERR_INVALID, "render: max_bounce out of range");
    if (p->out_channels != 3 && p->out_channels != 4) return ezrt_set_error(EZRT_ERR_INVALID, "render: out_channels must be 3 or 4");
    if (p->part_count < 1 || p->part_rank < 0 || p->part_rank >= p->part_count)
        return ezrt_set_error(EZRT_ERR_INVALID, "render: bad partition %d/%d", p->part_rank, p->part_count);
    if (p->mode == EZRT_MODE_DISNEY_IS_MIS_P5 && (!scene->dev.hdr || !scene->dev.hdr_cache))
        return ezrt_set_error(EZRT_ERR_INVALID, "render: IS/MIS mode needs an HDR map and its cache");
    return EZRT_OK;
}

int prepare_tiles(ezrt_scene* s, const ezrt_render_params* p, cudaStream_t st) {
    int key[4] = {p->width, p->height, p->part_rank, p->part_count};
    if (memcmp(key, s->tiles_key, sizeof(key)) == 0) return EZRT_OK;
    s->tiles = partition_tiles(p->width, p->height, p->part_rank, p->part_count);
    size_t bytes = sizeof(TileDev) * std::max<size_t>(1, s->tiles.size());
    int rc = s->tiles_buf.ensure(bytes);
    if (rc) return rc;
    if (!s->tiles.empty()) CU_CHECK(cudaMemcpyAsync(s->tiles_buf.p, s->tiles.data(), sizeof(TileDev) * s->tiles.size(), cudaMemcpyHostToDevice, st));
    CU_CHECK(cudaStreamSynchronize(st));  // s->tiles is pageable host memory
    memcpy(s->tiles_key, key, sizeof(key));
    s->n_pixels = 0;
    for (const TileDev& t : s->tiles) s->n_pixels += (size_t)t.w * t.h;
    return EZRT_OK;
}

struct ScatterEntry { TileDev* d_tiles; int n; };
std::map<std::array<int, 5>, ScatterEntry>& scatter_cache() {
    static std::map<std::array<int, 5>, ScatterEntry> cache;
    return cache;
}
std::mutex& scatter_mutex() {
    static std::mutex mu;
    return mu;
}

int validate_adaptive(const ezrt_render_params* p, const ezrt_adaptive_params* a) {
    if (!a) return ezrt_set_error(EZRT_ERR_INVALID, "render_adaptive: null adaptive params");
    if (!std::isfinite(a->threshold) || !(a->threshold > 0.0f))
        return ezrt_set_error(EZRT_ERR_INVALID, "render_adaptive: threshold must be finite and > 0 (got %g)", (double)a->threshold);
    if (a->min_spp < 2) return ezrt_set_error(EZRT_ERR_INVALID, "render_adaptive: min_spp must be >= 2 (got %d)", a->min_spp);
    if (a->check_interval < 1) return ezrt_set_error(EZRT_ERR_INVALID, "render_adaptive: check_interval must be >= 1 (got %d)", a->check_interval);
    if (a->reserved != 0) return ezrt_set_error(EZRT_ERR_INVALID, "render_adaptive: reserved field must be 0");
    if (p->first_frame != 0) return ezrt_set_error(EZRT_ERR_INVALID, "render_adaptive: first_frame must be 0 (an adaptive render cannot be resumed)");
    if (p->pipeline != EZRT_PIPELINE_WAVEFRONT) return ezrt_set_error(EZRT_ERR_INVALID, "render_adaptive: only the wavefront pipeline samples adaptively");
    return EZRT_OK;
}

// what the wavefront loop needs beyond a plain render: the criterion and the per-pixel outputs (device)
struct AdaptiveRun {
    float threshold;
    int min_spp, check_interval;
    int32_t* d_spp;
    float* d_luma2;
};

int validate_aov(const ezrt_render_params* p) {
    if (p->pipeline != EZRT_PIPELINE_WAVEFRONT) return ezrt_set_error(EZRT_ERR_INVALID, "render_aov: only the wavefront pipeline writes feature buffers");
    return EZRT_OK;
}

// the feature-buffer render's per-pixel outputs (device): 8 floats of first-hit features, the running mean of the squared luminance
struct AovRun {
    float* d_aov;
    float* d_luma2;
};

// The light table of the light sampling mode (ezrt_math.h, DESIGN.md section 10), built once per scene on stream st from the
// scene's own records: every triangle's weight, the lights kept in triangle order, their weights summed in float64 on the host,
// the cdf and the 64-byte records uploaded.  Synchronises st.
int build_lights(ezrt_scene* s, cudaStream_t st) {
    if (s->lights_built) return EZRT_OK;
    const int n = s->dev.n_triangles;
    struct TmpBuffer : DeviceBuffer { ~TmpBuffer() { release(); } } tmp;
    int rc = tmp.ensure(sizeof(float) * 2 * (size_t)n + sizeof(int32_t) * ((size_t)n + 4));
    if (rc) return rc;
    float* d_w = (float*)tmp.p;
    float* d_wk = d_w + n;
    int32_t* d_idx = (int32_t*)(d_wk + n);
    int32_t* d_count = d_idx + n;
    launch_light_weights(s->dev, d_w, st);
    launch_light_compact(d_w, n, d_idx, d_wk, d_count, st);
    int32_t K = 0;
    CU_CHECK(cudaMemcpyAsync(&K, d_count, sizeof(K), cudaMemcpyDeviceToHost, st));
    CU_CHECK(cudaStreamSynchronize(st));
    std::vector<float> w(K);
    std::vector<int32_t> idx(K);
    if (K > 0) {
        CU_CHECK(cudaMemcpyAsync(w.data(), d_wk, sizeof(float) * K, cudaMemcpyDeviceToHost, st));
        CU_CHECK(cudaMemcpyAsync(idx.data(), d_idx, sizeof(int32_t) * K, cudaMemcpyDeviceToHost, st));
        CU_CHECK(cudaStreamSynchronize(st));
    }
    double W = 0.0;
    for (int k = 0; k < K; k++) W += (double)w[k];
    std::vector<float> cdf(K);
    double S = 0.0;
    for (int k = 0; k < K; k++) {
        S += (double)w[k];
        cdf[k] = (float)(S / W);
    }
    if (K > 0) cdf[K - 1] = 1.0f;
    LightsDev lt{};
    if (K > 0) {
        const size_t rec_bytes = sizeof(float4) * 4 * (size_t)K;
        if ((rc = s->lights_buf.ensure(rec_bytes + sizeof(float) * (size_t)K))) return rc;
        lt.rec = (const float4*)s->lights_buf.p;
        lt.cdf = (const float*)((char*)s->lights_buf.p + rec_bytes);
        launch_light_records(s->dev, d_idx, K, (float4*)lt.rec, st);
        CU_CHECK(cudaMemcpyAsync((void*)lt.cdf, cdf.data(), sizeof(float) * K, cudaMemcpyHostToDevice, st));
        CU_CHECK(cudaStreamSynchronize(st));   // cdf is pageable host memory; tmp is freed below
    }
    CU_CHECK(cudaGetLastError());
    lt.n = K;
    lt.w_total = (float)W;
    s->lights = lt;
    s->light_tri = idx;
    s->light_cdf = cdf;
    s->light_total = W;
    s->lights_built = true;
    return EZRT_OK;
}

// The environment map's light table (ezrt_math.h, DESIGN.md section 11), built once per scene on stream st from the scene's copy
// of the map: every texel's weight on the device, the sums and cdfs in float64 on the host, the three arrays uploaded.
// Synchronises st.  A scene without a map, or whose texels all weigh 0, has no table.
int build_env(ezrt_scene* s, cudaStream_t st) {
    if (s->env_built) return EZRT_OK;
    const int W = s->dev.hdr_w, H = s->dev.hdr_h;
    EnvDev env{};
    double T = 0.0;
    if (s->dev.hdr && W > 0 && H > 0) {
        const size_t n = (size_t)W * H;
        struct TmpBuffer : DeviceBuffer { ~TmpBuffer() { release(); } } tmp;
        int rc = tmp.ensure(sizeof(float) * n);
        if (rc) return rc;
        launch_env_weights(s->dev, (float*)tmp.p, st);
        std::vector<float> w(n);
        CU_CHECK(cudaMemcpyAsync(w.data(), tmp.p, sizeof(float) * n, cudaMemcpyDeviceToHost, st));
        CU_CHECK(cudaStreamSynchronize(st));
        std::vector<double> R(H, 0.0);
        for (int i = 0; i < H; i++) {
            double r = 0.0;
            for (int j = 0; j < W; j++) r += (double)w[(size_t)i * W + j];
            R[i] = r;
        }
        for (int i = 0; i < H; i++) T += R[i];
        if (std::isfinite(T) && T > 0.0) {
            // one host array in the device layout: row cdf (H) | column cdf (H x W) | texel pdf (H x W)
            std::vector<float> tab((size_t)H + 2 * n);
            float* row_cdf = tab.data();
            float* col_cdf = row_cdf + H;
            float* texel_pdf = col_cdf + n;
            double S = 0.0;
            for (int i = 0; i < H; i++) {
                S += R[i];
                row_cdf[i] = (float)(S / T);
                double c = 0.0;
                for (int j = 0; j < W; j++) {
                    const size_t k = (size_t)i * W + j;
                    c += (double)w[k];
                    col_cdf[k] = (R[i] > 0.0) ? (float)(c / R[i]) : 0.0f;
                    texel_pdf[k] = (float)((double)w[k] / T);
                }
                if (R[i] > 0.0) col_cdf[(size_t)i * W + W - 1] = 1.0f;
            }
            row_cdf[H - 1] = 1.0f;
            if ((rc = s->env_buf.ensure(sizeof(float) * tab.size()))) return rc;
            CU_CHECK(cudaMemcpyAsync(s->env_buf.p, tab.data(), sizeof(float) * tab.size(), cudaMemcpyHostToDevice, st));
            CU_CHECK(cudaStreamSynchronize(st));   // tab is pageable host memory
            env.row_cdf = (const float*)s->env_buf.p;
            env.col_cdf = env.row_cdf + H;
            env.texel_pdf = env.col_cdf + n;
            env.w = W;
            env.h = H;
        } else {
            T = 0.0;
        }
    }
    CU_CHECK(cudaGetLastError());
    s->env = env;
    s->env_total = T;
    s->env_built = true;
    return EZRT_OK;
}

RenderDev make_render_dev(const ezrt_scene* s, const ezrt_render_params* p) {
    RenderDev rd;
    rd.width = p->width; rd.height = p->height;
    rd.mode = p->mode; rd.max_bounce = p->max_bounce; rd.traverse = p->traverse;
    memcpy(rd.eye, p->eye, sizeof(rd.eye));
    memcpy(rd.cam, p->camera_rotate, sizeof(rd.cam));
    memcpy(rd.env, p->env_color, sizeof(rd.env));
    rd.first_frame = p->first_frame;
    rd.out_channels = p->out_channels;
    rd.compact_out = (p->part_count > 1) ? 1 : 0;
    rd.n_tiles = (int)s->tiles.size();
    rd.accel_space = (s->regular_tree && s->have_accel && p->traverse == EZRT_TRAVERSE_ACCEL && p->pipeline == EZRT_PIPELINE_WAVEFRONT) ? 1 : 0;
    return rd;
}

}  // namespace

extern "C" {

// ------------------------------------------------------------------------------------------
// scene upload + repack (replaces the TBO / texture uploads P5/main.cpp:878-906)
// ------------------------------------------------------------------------------------------
int ezrt_scene_create(int device, const float* tris, int n_triangles, const float* nodes, int n_nodes, const float* hdr,
                      const float* hdr_cache, int hdr_w, int hdr_h, int hdr_filter_linear, ezrt_scene** out_scene) {
    if (!tris || !nodes || !out_scene || n_triangles <= 0 || n_nodes < 2)
        return ezrt_set_error(EZRT_ERR_INVALID, "scene_create: need triangles and at least the dummy + root node");
    if ((hdr || hdr_cache) && (hdr_w <= 0 || hdr_h <= 0)) return ezrt_set_error(EZRT_ERR_INVALID, "scene_create: bad HDR size");
    if (n_triangles >= (1 << 24)) return ezrt_set_error(EZRT_ERR_INVALID, "scene_create: more than 2^24 triangles (ints-as-floats limit)");
    int n_dev = 0;
    CU_CHECK(cudaGetDeviceCount(&n_dev));
    if (device < 0 || device >= n_dev) return ezrt_set_error(EZRT_ERR_CUDA, "scene_create: no CUDA device %d (have %d)", device, n_dev);
    CU_CHECK(cudaSetDevice(device));
    // env EZRT_VERBOSE=1: wall-clock of the stages on stderr (all host work except the uploads)
    const bool verbose = getenv("EZRT_VERBOSE") && atoi(getenv("EZRT_VERBOSE")) != 0;
    auto t_last = std::chrono::steady_clock::now();
    auto lap = [&](const char* what) {
        if (!verbose) return;
        const auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[ezrt_scene_create] %-44s %8.1f ms\n", what, std::chrono::duration<double, std::milli>(now - t_last).count());
        t_last = now;
    };

    // ---- decode + validate the tree (getBVHNode, P5/fsh:138-155) ----
    // Host work on the caller's tree only: runs on its own thread while this one feeds the GPU (triangle upload, records,
    // acceleration-tree build).  Errors are carried back as (code, message): ezrt_set_error is per thread.
    struct HNode { int left, right, n, index; };
    std::vector<HNode> hn(n_nodes);
    std::vector<int> inner_id(n_nodes, -1);
    int n_inner = 0, max_depth = 0, n_top = 0, root_ref = 0;
    bool regular_tree = true;
    std::vector<float4> gnodes, leaf_box;
    std::vector<int> tri_leaf(n_triangles, 0);
    std::string ref_msg;
    auto ref_fail = [&](int code, const char* fmt, int a = 0, int b = 0, int c = 0) {
        char buf[256];
        snprintf(buf, sizeof(buf), fmt, a, b, c);
        ref_msg = buf;
        return code;
    };
    auto ref_stage = [&]() -> int {
    for (int i = 0; i < n_nodes; i++) {
        const float* s = nodes + (size_t)i * EZRT_BVHNODE_FLOATS;
        hn[i].left = (int)s[0]; hn[i].right = (int)s[1]; hn[i].n = (int)s[3]; hn[i].index = (int)s[4];
    }
    std::vector<char> seen(n_nodes, 0);
    {
        std::vector<std::pair<int, int>> stk;
        stk.push_back({1, 1});
        while (!stk.empty()) {
            auto [i, depth] = stk.back();
            stk.pop_back();
            if (i < 1 || i >= n_nodes) return ref_fail(EZRT_ERR_BAD_TREE, "scene_create: child index %d out of range", i);
            if (seen[i]) return ref_fail(EZRT_ERR_BAD_TREE, "scene_create: node %d reachable twice", i);
            seen[i] = 1;
            max_depth = std::max(max_depth, depth);
            const HNode& nd = hn[i];
            if (nd.n > 0) {
                if (nd.n > EZRT_LEAF_MAX_N) return ref_fail(EZRT_ERR_BAD_TREE, "scene_create: leaf %d holds %d > %d triangles", i, nd.n, EZRT_LEAF_MAX_N);
                if (nd.index < 0 || nd.index + nd.n > n_triangles) return ref_fail(EZRT_ERR_BAD_TREE, "scene_create: leaf %d range out of bounds", i);
            } else {
                // the shader would read the dummy node 0 for a missing child (P5/fsh:278-302); not supported
                if (nd.left <= 0 || nd.right <= 0) return ref_fail(EZRT_ERR_BAD_TREE, "scene_create: inner node %d lacks a child", i);
                stk.push_back({nd.right, depth + 1});
                stk.push_back({nd.left, depth + 1});
            }
        }
    }
    if (max_depth + 1 > EZRT_MAX_STACK) return ref_fail(EZRT_ERR_BAD_TREE, "scene_create: tree depth %d exceeds %d", max_depth, EZRT_MAX_STACK - 1);
    // The ACCEL and PRUNED policies rely on what buildBVH* guarantees: every triangle in exactly one leaf,
    // leaf boxes bounding their triangles, child boxes inside their parent's.  A caller-supplied tree that
    // breaks any of these is only ever walked literally (REFERENCE policy), whatever the params ask for.
    {
        std::vector<unsigned char> cover(n_triangles, 0);
        for (int i = 1; i < n_nodes && regular_tree; i++) {
            if (!seen[i]) continue;
            const float* B = nodes + (size_t)i * EZRT_BVHNODE_FLOATS;
            if (hn[i].n > 0) {
                for (int k = 0; k < hn[i].n && regular_tree; k++) {
                    const int t = hn[i].index + k;
                    if (cover[t]++) regular_tree = false;
                    const float* v = tris + (size_t)t * EZRT_TRIANGLE_FLOATS;
                    for (int c = 0; c < 9; c++)
                        if (!(v[c] >= B[6 + c % 3] && v[c] <= B[9 + c % 3])) regular_tree = false;
                }
            } else {
                for (int c : {hn[i].left, hn[i].right}) {
                    const float* C = nodes + (size_t)c * EZRT_BVHNODE_FLOATS;
                    for (int a = 0; a < 3; a++)
                        if (!(C[6 + a] >= B[6 + a] && C[9 + a] <= B[9 + a])) regular_tree = false;
                }
            }
        }
        for (int t = 0; t < n_triangles && regular_tree; t++)
            if (cover[t] != 1) regular_tree = false;
    }
    // Record numbering: the top of the tree level by level (these records are staged in shared memory
    // by the traversal kernels: 61% of all inner-node visits hit depth <= 9 on the 1M-triangle scene),
    // whole levels while they fit EZRT_TOP_NODES_MAX; everything below in the builder's pre-order.
    {
        std::vector<int> level, next;
        if (hn[1].n <= 0) level.push_back(1);
        while (!level.empty() && n_top + (int)level.size() <= EZRT_TOP_NODES_MAX) {
            next.clear();
            for (int i : level) {
                inner_id[i] = n_top++;
                if (hn[hn[i].left].n <= 0) next.push_back(hn[i].left);
                if (hn[hn[i].right].n <= 0) next.push_back(hn[i].right);
            }
            level.swap(next);
        }
    }
    n_inner = n_top;
    for (int i = 1; i < n_nodes; i++)
        if (seen[i] && hn[i].n <= 0 && inner_id[i] < 0) inner_id[i] = n_inner++;

    auto child_ref = [&](int c) -> int {
        if (hn[c].n > 0) return (int)(EZRT_LEAF_FLAG | ((uint32_t)hn[c].index << 7) | (uint32_t)hn[c].n);
        return inner_id[c];
    };
    auto pack_node = [](float4* g, const float* LA, const float* LB, const float* RA, const float* RB, int rl, int rr) {
        float fl, fr;
        memcpy(&fl, &rl, 4);
        memcpy(&fr, &rr, 4);
        g[0] = make_float4(LA[0], LA[1], LB[0], LB[1]);  // left : AA.x AA.y | BB.x BB.y
        g[1] = make_float4(RA[0], RA[1], RB[0], RB[1]);  // right: AA.x AA.y | BB.x BB.y
        g[2] = make_float4(LA[2], LB[2], RA[2], RB[2]);  // left AA.z BB.z  | right AA.z BB.z
        g[3] = make_float4(fl, fr, 0.0f, 0.0f);          // child references
    };
    gnodes.assign((size_t)std::max(1, n_inner) * 4, make_float4(0.0f, 0.0f, 0.0f, 0.0f));
    for (int i = 1; i < n_nodes; i++) {
        if (inner_id[i] < 0) continue;
        const float* L = nodes + (size_t)hn[i].left * EZRT_BVHNODE_FLOATS;
        const float* R = nodes + (size_t)hn[i].right * EZRT_BVHNODE_FLOATS;
        pack_node(&gnodes[(size_t)inner_id[i] * 4], L + 6, L + 9, R + 6, R + 9, child_ref(hn[i].left), child_ref(hn[i].right));
    }
    // reference leaf of every triangle + leaf boxes (accel policy: "does the shader reach this leaf?")
    for (int i = 1; i < n_nodes; i++) {
        if (!seen[i] || hn[i].n <= 0) continue;
        const float* B = nodes + (size_t)i * EZRT_BVHNODE_FLOATS;
        int slot = (int)(leaf_box.size() / 2);
        leaf_box.push_back(make_float4(B[6], B[7], B[8], 0.0f));
        leaf_box.push_back(make_float4(B[9], B[10], B[11], 0.0f));
        for (int k = 0; k < hn[i].n; k++) tri_leaf[hn[i].index + k] = slot;
    }

    root_ref = child_ref(1);
    return EZRT_OK;
    };   // ref_stage
    // ---- the scene object, the worker for the caller's tree, and the clean-up of every early return ----
    ezrt_scene* sc = new (std::nothrow) ezrt_scene();
    if (!sc) return ezrt_set_error(EZRT_ERR_NOMEM, "scene_create: out of host memory");
    sc->device = device;
    int ref_rc = EZRT_OK;
    double ref_ms = 0.0;
    struct Cleanup {   // declared after everything the worker touches: joined first, then those locals go
        ezrt_scene* sc = nullptr;
        std::thread worker;
        DeviceBuffer raw;
        ~Cleanup() {
            if (worker.joinable()) worker.join();
            raw.release();
            if (sc) ezrt_scene_destroy(sc);
        }
    } guard;
    guard.sc = sc;
    auto ref_timed = [&]() {
        const auto t0 = std::chrono::steady_clock::now();
        ref_rc = ref_stage();
        ref_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    };
    try {
        guard.worker = std::thread(ref_timed);
    } catch (...) {
        ref_timed();   // no thread to be had: in line
    }
    // ---- triangles: upload the caller's array once; geometry records, shading records, material runs and the scene
    // bounds are made from it on the device (scene_prep.cu) ----
    DeviceBuffer& raw = guard.raw;
    {
        int r = raw.ensure((size_t)n_triangles * EZRT_TRIANGLE_FLOATS * sizeof(float));
        if (r) return r;
        if (cudaMemcpy(raw.p, tris, (size_t)n_triangles * EZRT_TRIANGLE_FLOATS * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess)
            return ezrt_set_error(EZRT_ERR_CUDA, "scene_create: upload failed: %s", cudaGetErrorString(cudaGetLastError()));
    }
    lap("triangles: upload");
    EzrtPrepInfo prep;
    {
        int r = sc->tri_geo.ensure((size_t)n_triangles * 4 * sizeof(float4));
        if (!r) r = sc->tri_shade.ensure((size_t)n_triangles * 3 * sizeof(float4));
        if (!r) r = ezrt_prep_records((const float*)raw.p, n_triangles, sc->tri_geo.p, sc->tri_shade.p, prep);
        if (r) return r;
    }
    std::vector<float4> mats;
    for (int m = 0; m < prep.n_materials; m++) {
        const float* v = &prep.materials[(size_t)m * EZRT_MATERIAL_FLOATS];
        mats.push_back(make_float4(v[0], v[1], v[2], v[3]));
        mats.push_back(make_float4(v[4], v[5], v[6], v[7]));
        mats.push_back(make_float4(v[8], v[9], v[10], v[11]));
        mats.push_back(make_float4(v[12], v[13], v[14], v[15]));
        mats.push_back(make_float4(v[16], v[17], 0.0f, 0.0f));
    }
    const float max_abs = prep.max_abs;
    float bmin[3], bmax[3];
    for (int k = 0; k < 3; k++) { bmin[k] = prep.bmin[k]; bmax[k] = prep.bmax[k]; }
    lap("triangles: geometry / shading records, materials (device)");
    // ---- acceleration tree: sentinel-free SAH over the same triangles (DESIGN.md "accel"), collapsed to 8-wide
    // quantised nodes (accel_w8.cpp, w8_node.h).  A tree too deep for the traversal stacks (degenerate input) is
    // dropped: the scene then renders with the PRUNED policy on the caller's tree, as for an irregular tree.
    const float prune_delta = max_abs * 1.52587890625e-05f;  // 2^-16 * scene extent
    EzrtW4Tree w4;
    EzrtRawArray<float>& acc_wide = w4.nodes;
    EzrtRawArray<uint32_t>& acc_wide_q = w4.q16;
    std::vector<uint32_t> w8_words;
    int acc_wide_root = 0;
    std::vector<uint32_t> acc_order;
    int acc_depth = 0, w8_depth = 0, w8_near_bit[3] = {0, 1, 2};
    bool have_accel = true;
    {
        // Which form of the tree the accel kernels walk, chosen by scene size (env EZRT_ACCEL=4 / 8 forces one):
        //   8: 8-wide nodes with 8-bit quantised boxes in octant order (k_extend_w8): 96-byte records, fewer L1 wavefronts per
        //      ray, more instructions.  On an H100 SXM it measured 2258 vs 1773 Mrays/s on C3 and 1956 vs 1546 on C4 (1 M
        //      triangles) against the 4-wide form (bench.py, 700 W)
        //   4: 4-wide nodes with exact fp32 boxes, children sorted by entry distance (k_extend_accel): 10841-10883 vs
        //      10476-10513 Mrays/s on C2 (5,300 triangles, whose tree stays in L1; bench.py, 400 W)
        // The threshold lies between the two measured sizes.  A scene of at most W8_MAX_LEAF_TRIS triangles is one leaf of the
        // 4-wide form's binary tree, which the 4-wide builder does not take: the W8 builder handles it.
        int accel_form = (n_triangles >= (1 << 16)) ? 8 : 4;
        if (const char* we = getenv("EZRT_ACCEL")) {
            const int v = atoi(we);
            if (v == 4 || v == 8) accel_form = v;
        }
        if (n_triangles <= W8_MAX_LEAF_TRIS) accel_form = 8;
        // the binary tree's leaves: the 4-wide form keeps ranges of <= 4 triangles as leaves; the W8 form builds down to
        // W8_BINARY_LEAF_TRIS and leaves the choice of its leaves to the collapse (w8_node.h)
        const int leaf_n = (accel_form == 8) ? W8_BINARY_LEAF_TRIS : W8_MAX_LEAF_TRIS;
        std::vector<EzrtAccelNode> an;
        std::vector<uint32_t> order_bin;
        // on the GPU (accel_build.cu; the same tree node for node); env EZRT_BUILD=host: the host builder (host_scene.cpp)
        const char* be = getenv("EZRT_BUILD");
        if (be && !strcmp(be, "host")) {
            ezrt_build_accel(tris, n_triangles, leaf_n, an, order_bin);
            lap("acceleration tree: binary SAH build (host)");
        } else {
            const int brc = ezrt_build_accel_device((const float*)raw.p, n_triangles, leaf_n, an, order_bin, nullptr);
            if (brc < 0) return brc;
            lap("acceleration tree: binary SAH build (device)");
        }
        // boxes inflated by 2*delta: a hit hitTriangle accepts lies within delta of its triangle's box, so
        // the inflated boxes of the whole ancestor chain are entered no later than the hit distance
        const float pad = 2.0f * prune_delta;
        EzrtW8Tree w8;
        ezrt_w8_axis_bits(bmin, bmax, w8_near_bit);
        if (accel_form == 8) {
            const int wrc = ezrt_build_w8(an, order_bin, pad, max_abs, w8_near_bit, W8_COST_TRI, ezrt_host_threads(), w8);
            if (wrc != 0 || w8.depth > EZRT_W8_SMEM_STACK + W8_LOCAL_STACK) {
                have_accel = false;
            } else {
                acc_order = w8.tri_order;
                w8_words.swap(w8.nodes);
                w8_depth = w8.depth;
            }
        } else {
            // 4-wide collapse: SAH-optimal choice of each node's children (EzrtCollapse; env EZRT_W4_COLLAPSE=greedy: round 1's
            // "replace the largest inner child" rule); leaves = sub-trees of <= 4 consecutive triangles; packed by accel_w8.cpp
            const char* ce = getenv("EZRT_W4_COLLAPSE");
            const bool greedy = ce && !strcmp(ce, "greedy");
            const char* qe = getenv("EZRT_ACCEL_Q16");
            const bool want_q16 = !(qe && atoi(qe) == 0);
            if (ezrt_build_w4(an, pad, max_abs, greedy, want_q16, ezrt_host_threads(), w4) != 0) {
                have_accel = false;
            } else {
                acc_order = order_bin;
                acc_wide_root = w4.root;
                acc_depth = w4.depth;
                if (3 * w4.depth + 2 > EZRT_ACCEL_STACK) { w4.nodes.clear(); have_accel = false; }  // too deep for the traversal stack
                if (!have_accel) w4.q16.clear();
            }
        }
        if (!have_accel) {
            acc_order.resize(n_triangles);
            for (int i = 0; i < n_triangles; i++) acc_order[i] = (uint32_t)i;
        }
        raw.release();
    }
    lap("acceleration tree: collapse, pack");
    // ---- the caller's tree is needed from here on ----
    if (guard.worker.joinable()) guard.worker.join();
    if (verbose) fprintf(stderr, "[ezrt_scene_create] %-44s %8.1f ms (worker thread, overlapped)\n", "reference tree: decode, validate, repack", ref_ms);
    if (ref_rc) return ezrt_set_error(ref_rc, "%s", ref_msg.c_str());
    lap("wait for the reference-tree worker");
    cudaDeviceProp prop;   // cudaGetDeviceProperties takes milliseconds: once per device and process
    {
        static std::mutex mu;
        static std::map<int, cudaDeviceProp> cache;
        std::lock_guard<std::mutex> lock(mu);
        auto it = cache.find(device);
        if (it == cache.end()) {
            memset(&prop, 0, sizeof(prop));
            if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) cudaGetLastError();
            else cache[device] = prop;
        } else {
            prop = it->second;
        }
    }
    if (prop.multiProcessorCount > 0) {
        sc->n_sms = prop.multiProcessorCount;
        sc->max_window_bytes = (size_t)prop.accessPolicyMaxWindowSize;
    }
    int rc = EZRT_OK;
    auto upload = [&](DeviceBuffer& b, const void* src, size_t bytes) -> int {
        int r = b.ensure(std::max<size_t>(bytes, 16));
        if (r) return r;
        if (bytes && cudaMemcpy(b.p, src, bytes, cudaMemcpyHostToDevice) != cudaSuccess)
            return ezrt_set_error(EZRT_ERR_CUDA, "scene_create: upload failed: %s", cudaGetErrorString(cudaGetLastError()));
        return EZRT_OK;
    };
    EzrtLap sub("ezrt_scene_create uploads");
    if (!rc) rc = upload(sc->nodes, gnodes.data(), gnodes.size() * sizeof(float4));
    if (!rc) rc = upload(sc->materials, mats.data(), mats.size() * sizeof(float4));
    sub("reference-tree nodes, materials");
    // acceleration tree nodes | triangle geometry | shading records in ONE allocation: the window the
    // L2 persisting-access policy is set on while a render runs (the data every ray touches at random)
    const size_t acc_nodes_bytes = ((std::max<size_t>(w8_words.size(), 4) * sizeof(uint32_t) + 255) / 256) * 256;
    size_t acc_geo_bytes = (((size_t)n_triangles * 4 * sizeof(float4) + 255) / 256) * 256;   // flat; the indexed layout below shrinks it
    const size_t acc_shade_bytes = (((size_t)n_triangles * 3 * sizeof(float4) + 255) / 256) * 256;
    if (!rc) rc = sc->acc_hot.ensure(acc_nodes_bytes + acc_geo_bytes + acc_shade_bytes);
    if (!rc) {
        char* base = (char*)sc->acc_hot.p;
        cudaError_t e = w8_words.empty() ? cudaSuccess : cudaMemcpy(base, w8_words.data(), w8_words.size() * sizeof(uint32_t), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) rc = ezrt_set_error(EZRT_ERR_CUDA, "scene_create: upload failed: %s", cudaGetErrorString(e));
        sc->hot_base = base;
        sc->hot_bytes = acc_nodes_bytes + acc_geo_bytes + acc_shade_bytes;
    }
    sub("hot allocation");
    if (!rc) rc = upload(sc->acc_tri_ref, acc_order.data(), acc_order.size() * sizeof(uint32_t));
    if (!rc && !acc_wide.empty()) rc = upload(sc->acc_wide, acc_wide.data(), acc_wide.size() * sizeof(float));
    if (!rc && !acc_wide_q.empty()) rc = upload(sc->acc_wide_q16, acc_wide_q.data(), acc_wide_q.size() * sizeof(uint32_t));
    if (!rc) rc = upload(sc->tri_leaf, tri_leaf.data(), tri_leaf.size() * sizeof(int));
    if (!rc) rc = upload(sc->leaf_box, leaf_box.data(), leaf_box.size() * sizeof(float4));
    sub("order, wide nodes, leaf map, leaf boxes");
    // geometry, shading records and the reference-leaf map in the acceleration tree's order, and the inverse permutation:
    // gathered on the device
    if (!rc) rc = sc->acc_tri_leaf.ensure((size_t)n_triangles * sizeof(int));
    if (!rc) rc = sc->ref_to_acc.ensure((size_t)n_triangles * sizeof(uint32_t));
    if (!rc)
        rc = ezrt_prep_gather(sc->tri_geo.p, sc->tri_shade.p, (const int*)sc->tri_leaf.p, (const uint32_t*)sc->acc_tri_ref.p, n_triangles,
                              (char*)sc->acc_hot.p + acc_nodes_bytes, (char*)sc->acc_hot.p + acc_nodes_bytes + acc_geo_bytes,
                              (int*)sc->acc_tri_leaf.p, (uint32_t*)sc->ref_to_acc.p);
    sub("gather");
    // The W8 form's triangle records, indexed where that is smaller (32 T + 16 V < 64 T): 32 B per triangle, (N, d0) (i1, i2, i3, 0),
    // plus 16 B per distinct vertex position, numbered by first use in the tree's order, instead of 64 B per triangle.  A scene that
    // shares its vertices (a mesh: about one vertex per two triangles) then keeps its triangle records in H100's 50 MB L2 up to
    // about 1.2 M triangles instead of 0.8 M (DESIGN.md section 4); a triangle soup keeps the flat records.  The 4-wide form and the
    // reference-order tri_geo are always flat.
    size_t acc_vert_bytes = 0;
    int n_vert = 0;
    bool tri_indexed = false;
    if (!rc && !w8_words.empty()) {
        DeviceBuffer ids, hot;
        rc = ids.ensure((size_t)n_triangles * 6 * sizeof(uint32_t));
        uint32_t* vid = (uint32_t*)ids.p;
        uint32_t* vert_src = vid + (size_t)n_triangles * 3;
        if (!rc) rc = ezrt_prep_vertex_ids((const char*)sc->acc_hot.p + acc_nodes_bytes, n_triangles, vid, vert_src, n_vert);
        if (!rc && 32 * (size_t)n_triangles + 16 * (size_t)n_vert < 64 * (size_t)n_triangles) {
            const size_t rec_bytes = (((size_t)n_triangles * 2 * sizeof(float4) + 255) / 256) * 256;
            const size_t vert_bytes = (((size_t)n_vert * sizeof(float4) + 255) / 256) * 256;
            rc = hot.ensure(acc_nodes_bytes + rec_bytes + vert_bytes + acc_shade_bytes);
            const char* old_base = (const char*)sc->acc_hot.p;
            char* base = (char*)hot.p;
            if (!rc && (cudaMemcpy(base, old_base, acc_nodes_bytes, cudaMemcpyDeviceToDevice) != cudaSuccess ||
                        cudaMemcpy(base + acc_nodes_bytes + rec_bytes + vert_bytes, old_base + acc_nodes_bytes + acc_geo_bytes, acc_shade_bytes,
                                   cudaMemcpyDeviceToDevice) != cudaSuccess))
                rc = ezrt_set_error(EZRT_ERR_CUDA, "scene_create: copy failed: %s", cudaGetErrorString(cudaGetLastError()));
            if (!rc) rc = ezrt_prep_indexed(old_base + acc_nodes_bytes, n_triangles, vid, vert_src, n_vert, base + acc_nodes_bytes, base + acc_nodes_bytes + rec_bytes);
            if (!rc) {
                std::swap(sc->acc_hot, hot);
                acc_geo_bytes = rec_bytes;
                acc_vert_bytes = vert_bytes;
                tri_indexed = true;
                sc->hot_base = sc->acc_hot.p;
                sc->hot_bytes = acc_nodes_bytes + acc_geo_bytes + acc_vert_bytes + acc_shade_bytes;
            }
        }
        hot.release();
        ids.release();
    }
    if (verbose && !rc && !w8_words.empty())
        fprintf(stderr, "[ezrt_scene_create] triangle records: %s (%d triangles, %d distinct vertices)\n", tri_indexed ? "indexed" : "flat", n_triangles, n_vert);
    sub("indexed triangle records");
    if (!rc && hdr) rc = upload(sc->hdr, hdr, sizeof(float) * 3 * (size_t)hdr_w * hdr_h);
    if (!rc && hdr_cache) rc = upload(sc->hdr_cache, hdr_cache, sizeof(float) * 3 * (size_t)hdr_w * hdr_h);
    sub("environment map, cache");
    if (!rc && cudaStreamCreateWithFlags(&sc->own_stream, cudaStreamNonBlocking) != cudaSuccess) rc = ezrt_set_error(EZRT_ERR_CUDA, "scene_create: stream");
    if (!rc && (cudaEventCreate(&sc->ev_start) != cudaSuccess || cudaEventCreate(&sc->ev_stop) != cudaSuccess)) rc = ezrt_set_error(EZRT_ERR_CUDA, "scene_create: events");
    sub("stream, events");
    if (rc) return rc;
    lap("uploads, records in the tree's order (device)");
    guard.sc = nullptr;   // from here on the scene is the caller's
    sc->n_materials = prep.n_materials;
    sc->regular_tree = regular_tree;
    sc->have_accel = have_accel;
    sc->tree_depth = max_depth;
    SceneDev& d = sc->dev;
    d.nodes = (const float4*)sc->nodes.p;
    d.tri_geo = (const float4*)sc->tri_geo.p;
    d.tri_shade = (const float4*)sc->tri_shade.p;
    d.materials = (const float4*)sc->materials.p;
    d.hdr = hdr ? (const float*)sc->hdr.p : nullptr;
    d.hdr_cache = hdr_cache ? (const float*)sc->hdr_cache.p : nullptr;
    d.hdr_w = hdr_w; d.hdr_h = hdr_h; d.hdr_linear = hdr_filter_linear ? 1 : 0;
    d.root_ref = root_ref;
    d.w8_nodes = w8_words.empty() ? nullptr : (const uint4*)sc->acc_hot.p;
    for (int k = 0; k < 3; k++) d.w8_near_bit[k] = w8_near_bit[k];
    d.w8_stack_entries = std::max(1, std::min(w8_depth, EZRT_W8_SMEM_STACK));
    d.w8_origin_limit = W8_ORIGIN_LIMIT_REL * max_abs;
    // decode range of the quantised form in use (W8, else Q16) with its decode bias: 2^15 for W8, 2^23 for Q16 (device_functions.cuh)
    d.quant_inv_limit = !w8_words.empty() ? ezrt_quant_inv_limit(ezrt_w8_max_scale(w8_words.data(), w8_words.size() / W8_NODE_WORDS), W8_DECODE_BIAS, max_abs)
                      : !acc_wide_q.empty() ? ezrt_quant_inv_limit(ezrt_q16_max_scale(acc_wide_q.data(), acc_wide_q.size() / 24), 8388608.0, max_abs)
                                            : W8_INV_LIMIT;
    d.w8_decode_bits = W8_DECODE_BITS;
    d.w8_tri_weight = 1;   // cooperative triangle step: 1 over 2 is +1 % on C3 and C4 (H100, DESIGN.md section 6)
    if (const char* e = getenv("EZRT_TRI_W")) d.w8_tri_weight = std::max(1, std::min(64, atoi(e)));
    d.acc_tri_geo = (const float4*)((const char*)sc->acc_hot.p + acc_nodes_bytes);
    d.acc_tri_vert = tri_indexed ? (const float4*)((const char*)sc->acc_hot.p + acc_nodes_bytes + acc_geo_bytes) : nullptr;
    d.acc_tri_indexed = tri_indexed ? 1 : 0;
    d.acc_tri_ref = (const uint32_t*)sc->acc_tri_ref.p;
    d.acc_wide_nodes = acc_wide.empty() ? nullptr : (const float4*)sc->acc_wide.p;
    d.acc_wide_root_ref = acc_wide_root;
    d.acc_wide_q16 = acc_wide_q.empty() ? nullptr : (const uint4*)sc->acc_wide_q16.p;
    d.q16_decode_bits = 0x4B000000u;
    d.tri_l1_bypass = ((size_t)n_triangles * 64 > ((size_t)4 << 20)) ? 1 : 0;  // > 4 MB of triangle records: stream them past L1
    if (const char* e = getenv("EZRT_TRI_L1_BYPASS")) d.tri_l1_bypass = atoi(e) != 0;
    d.acc_tri_shade = (const float4*)((const char*)sc->acc_hot.p + acc_nodes_bytes + acc_geo_bytes + acc_vert_bytes);
    d.acc_tri_leaf = (const int*)sc->acc_tri_leaf.p;
    d.ref_to_acc = (const uint32_t*)sc->ref_to_acc.p;
    d.tri_leaf = (const int*)sc->tri_leaf.p;
    d.leaf_box = (const float4*)sc->leaf_box.p;
    sc->acc_depth = acc_depth;
    d.n_triangles = n_triangles;
    d.n_inner = n_inner;
    d.top_nodes = n_top;
    if (const char* e = getenv("EZRT_TOP_NODES")) {
        d.top_nodes = std::max(0, std::min(n_top, atoi(e)));
    }
    d.prune_delta = prune_delta;  // 2^-16 * scene extent (DESIGN.md "pruning")
    for (int k = 0; k < 3; k++) {
        d.bmin[k] = bmin[k];
        float ext = bmax[k] - bmin[k];
        d.cell_scale[k] = (ext > 0.0f) ? 32.0f / ext : 0.0f;
    }
    if (const char* e = getenv("EZRT_SORT_RAYS")) sc->sort_rays = atoi(e);
    if (const char* e = getenv("EZRT_DEFERRED_LANE")) sc->deferred_lane = atoi(e) != 0;
    if (const char* e = getenv("EZRT_CAMERA_ORDER")) sc->camera_pixel_major = strcmp(e, "frame") != 0;
    {   // optional L2 persistence for the randomly-accessed tree data (env EZRT_L2_PERSIST=1)
        // measured on C3: -8 % (the set-aside shrinks the L2 left for the streaming queue traffic) -> off by default
        const char* e = getenv("EZRT_L2_PERSIST");
        if (e && atoi(e) != 0 && prop.persistingL2CacheMaxSize > 0) {
            size_t want = std::min<size_t>(sc->hot_bytes, (size_t)prop.persistingL2CacheMaxSize);
            if (cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want) == cudaSuccess) sc->l2_persist_bytes = want;
            cudaGetLastError();
        }
    }
    d.refill_thresh = 24;
    d.refill_thresh_camera = 0;
    if (const char* e = getenv("EZRT_REFILL_CAM")) d.refill_thresh_camera = std::max(0, std::min(32, atoi(e)));
    d.inner_thresh = 16;
    d.leaf_thresh = 16;   // tuned with the cheaper leaf passes on S-1M (16 over 12)
    d.work_chunk = 32;
    d.work_chunk_camera = 64;
    if (const char* e = getenv("EZRT_CHUNK_CAM")) d.work_chunk_camera = std::max(32, std::min(65536, atoi(e)));
    if (const char* e = getenv("EZRT_CHUNK")) d.work_chunk = std::max(32, std::min(65536, atoi(e)));
    if (const char* e = getenv("EZRT_LEAF_T")) d.leaf_thresh = std::max(1, std::min(33, atoi(e)));
    if (const char* e = getenv("EZRT_REFILL_T")) d.refill_thresh = std::max(1, std::min(32, atoi(e)));
    if (const char* e = getenv("EZRT_INNER_T")) d.inner_thresh = std::max(1, std::min(32, atoi(e)));
    *out_scene = sc;
    return EZRT_OK;
}

int ezrt_scene_set_medium(ezrt_scene* s, const ezrt_medium* m) {
    if (!s) return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_medium: null scene");
    if (!m) {
        s->has_medium = false;
        s->medium = MediumDev{};
        return EZRT_OK;
    }
    if (!(ez_finite(m->sigma_t) && m->sigma_t >= 0.0f)) return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_medium: sigma_t must be finite and >= 0");
    for (int k = 0; k < 3; k++) {
        if (!(m->albedo[k] >= 0.0f && m->albedo[k] <= 1.0f)) return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_medium: albedo must lie in [0, 1]");
        if (!(ez_finite(m->box_min[k]) && ez_finite(m->box_max[k]))) return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_medium: the box must be finite");
        if (m->box_min[k] > m->box_max[k]) return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_medium: box_min > box_max on axis %d", k);
    }
    if (!(m->g > -1.0f && m->g < 1.0f)) return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_medium: g must lie in (-1, 1)");
    if (m->reserved != 0) return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_medium: reserved must be 0");
    MediumDev d;
    d.sigma_t = m->sigma_t;
    d.albedo = ez_v3(m->albedo[0], m->albedo[1], m->albedo[2]);
    d.g = m->g;
    d.bmin = ez_v3(m->box_min[0], m->box_min[1], m->box_min[2]);
    d.bmax = ez_v3(m->box_max[0], m->box_max[1], m->box_max[2]);
    s->medium = d;
    s->has_medium = true;
    return EZRT_OK;
}

int ezrt_scene_set_textures(ezrt_scene* s, int n_textures, const ezrt_texture* textures, const float* texcoords, const int32_t* texture_id) {
    if (!s) return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_textures: null scene");
    CU_CHECK(cudaSetDevice(s->device));
    if (!textures) {
        CU_CHECK(cudaDeviceSynchronize());   // renders already enqueued still read the buffers
        s->tex_buf.release(); s->tex_rec_buf.release();
        s->has_textures = false;
        s->has_maps = false;
        s->n_textures = 0;
        s->tex = TexDev{};
        s->maps = MapsDev{};
        return EZRT_OK;
    }
    const int n_tri = s->dev.n_triangles;
    if (n_textures < 1 || !texcoords || !texture_id) return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_textures: bad argument");
    size_t n_texels = 0;
    for (int k = 0; k < n_textures; k++) {
        const ezrt_texture& t = textures[k];
        if (t.width < 1 || t.width > 16384 || t.height < 1 || t.height > 16384)
            return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_textures: texture %d is %dx%d (each side 1 to 16384)", k, t.width, t.height);
        if (!t.rgba || t.reserved != 0) return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_textures: texture %d has no texels or reserved != 0", k);
        n_texels += (size_t)t.width * t.height;
    }
    for (int i = 0; i < n_tri; i++)
        if (texture_id[i] < -1 || texture_id[i] >= n_textures)
            return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_textures: triangle %d has texture id %d (valid: -1 to %d)", i, texture_id[i], n_textures - 1);
    // host staging: sRGB table | texture table | texels; reference-order records.  The new buffers are filled before the previous
    // ones are released, so that a failure leaves the scene's textures as they were.
    const size_t lut_bytes = 2 * 256 * sizeof(float), table_bytes = ((sizeof(int4) * (size_t)n_textures + 255) / 256) * 256;
    if (n_texels > (size_t)INT32_MAX) return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_textures: more than 2^31 texels");
    std::vector<unsigned char> host;
    std::vector<float4> rec;
    try {
        host.resize(lut_bytes + table_bytes + 4 * n_texels);
        rec.resize(2 * (size_t)n_tri);
    } catch (const std::bad_alloc&) {
        return ezrt_set_error(EZRT_ERR_NOMEM, "scene_set_textures: host staging of %zu texels", n_texels);
    }
    memcpy(host.data(), ez_srgb_table, sizeof(ez_srgb_table));   // then ez_unorm8_table, for the material maps
    memcpy(host.data() + sizeof(ez_srgb_table), ez_unorm8_table, sizeof(ez_unorm8_table));
    int4* table = (int4*)(host.data() + lut_bytes);
    size_t off = 0;
    for (int k = 0; k < n_textures; k++) {
        const size_t n = (size_t)textures[k].width * textures[k].height;
        table[k] = make_int4((int)off, textures[k].width, textures[k].height, 0);
        memcpy(host.data() + lut_bytes + table_bytes + 4 * off, textures[k].rgba, 4 * n);
        off += n;
    }
    for (int i = 0; i < n_tri; i++) {
        const float* c = texcoords + 6 * (size_t)i;
        int32_t id = texture_id[i];
        float idf;
        memcpy(&idf, &id, 4);
        rec[2 * (size_t)i] = make_float4(c[0], c[1], c[2], c[3]);
        rec[2 * (size_t)i + 1] = make_float4(c[4], c[5], idf, 0.0f);
    }
    DeviceBuffer nbuf, nrec;
    int rc = nbuf.ensure(host.size());
    if (!rc) rc = nrec.ensure(2 * sizeof(float4) * 2 * (size_t)std::max(n_tri, 1));
    if (rc) { nbuf.release(); nrec.release(); return rc; }
    float4* d_rec = (float4*)nrec.p;
    float4* d_acc = d_rec + 2 * (size_t)n_tri;
    cudaError_t e = cudaMemcpy(nbuf.p, host.data(), host.size(), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_rec, rec.data(), sizeof(float4) * rec.size(), cudaMemcpyHostToDevice);
    if (e == cudaSuccess && s->dev.acc_tri_ref && n_tri > 0) {
        launch_tex_gather(d_rec, s->dev.acc_tri_ref, n_tri, d_acc, 0);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();   // also: renders already enqueued still read the previous buffers
    if (e != cudaSuccess) {
        nbuf.release(); nrec.release();
        return ezrt_set_error(EZRT_ERR_CUDA, "scene_set_textures: %s", cudaGetErrorString(e));
    }
    s->tex_buf.release(); s->tex_rec_buf.release();
    s->tex_buf = nbuf; s->tex_rec_buf = nrec;   // DeviceBuffer frees only on release(): the pointers move to the scene
    TexDev t{};
    t.rec = d_rec;
    t.acc_rec = d_acc;
    t.lut = (const float*)s->tex_buf.p;
    s->maps.unorm = t.lut + 256;
    t.table = (const int4*)((const char*)s->tex_buf.p + lut_bytes);
    t.texels = (const uint32_t*)((const char*)s->tex_buf.p + lut_bytes + table_bytes);
    s->tex = t;
    s->has_textures = true;
    s->n_textures = n_textures;
    s->has_maps = false;   // the new records' fourth words are 0: the maps' ids referred to the previous textures
    return EZRT_OK;
}

int ezrt_scene_set_material_maps(ezrt_scene* s, const int32_t* metal_rough_id, const int32_t* normal_id) {
    if (!s) return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_material_maps: null scene");
    if (!s->has_textures) return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_material_maps: no textures (ezrt_scene_set_textures)");
    if ((metal_rough_id == nullptr) != (normal_id == nullptr)) return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_material_maps: bad argument");
    const int n_tri = s->dev.n_triangles;
    const int n_tex = s->n_textures;
    std::vector<uint32_t> words;
    try {
        words.assign((size_t)n_tri, 0u);
    } catch (const std::bad_alloc&) {
        return ezrt_set_error(EZRT_ERR_NOMEM, "scene_set_material_maps: host staging");
    }
    if (metal_rough_id) {
        for (int i = 0; i < n_tri; i++) {
            const int32_t a = metal_rough_id[i], b = normal_id[i];
            if (a < -1 || a >= n_tex || a >= 65535 || b < -1 || b >= n_tex || b >= 65535)
                return ezrt_set_error(EZRT_ERR_INVALID, "scene_set_material_maps: triangle %d has map ids (%d, %d) (valid: -1 to %d)", i, a, b,
                                      std::min(n_tex, 65535) - 1);
            words[i] = (uint32_t)(a + 1) | ((uint32_t)(b + 1) << 16);
        }
    }
    CU_CHECK(cudaSetDevice(s->device));
    if (n_tri > 0) {
        DeviceBuffer buf;
        int rc = buf.ensure(sizeof(uint32_t) * (size_t)n_tri);
        if (rc) return rc;
        cudaError_t e = cudaDeviceSynchronize();   // renders already enqueued still read the records
        if (e == cudaSuccess) e = cudaMemcpy(buf.p, words.data(), sizeof(uint32_t) * (size_t)n_tri, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) {
            launch_maps_set((const uint32_t*)buf.p, s->dev.acc_tri_ref, n_tri, (float4*)s->tex.rec, (float4*)s->tex.acc_rec, 0);
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
        buf.release();
        if (e != cudaSuccess) return ezrt_set_error(EZRT_ERR_CUDA, "scene_set_material_maps: %s", cudaGetErrorString(e));
    }
    s->has_maps = metal_rough_id != nullptr;
    return EZRT_OK;
}

int ezrt_scene_sample_materials(ezrt_scene* s, int n, const int32_t* tri, const float* hits, float* out) {
    if (!s || n < 0 || (n > 0 && (!tri || !hits || !out))) return ezrt_set_error(EZRT_ERR_INVALID, "scene_sample_materials: bad argument");
    if (!s->has_textures) return ezrt_set_error(EZRT_ERR_INVALID, "scene_sample_materials: no textures (ezrt_scene_set_textures)");
    for (int i = 0; i < n; i++)
        if (tri[i] < 0 || tri[i] >= s->dev.n_triangles) return ezrt_set_error(EZRT_ERR_INVALID, "scene_sample_materials: triangle %d out of range", tri[i]);
    if (n == 0) return EZRT_OK;
    CU_CHECK(cudaSetDevice(s->device));
    DeviceBuffer buf;
    int rc = buf.ensure(sizeof(float) * 18 * (size_t)n + 256);
    if (rc) return rc;
    int32_t* d_tri = (int32_t*)buf.p;
    float* d_h = (float*)(d_tri + n);
    float* d_out = d_h + 7 * (size_t)n;
    cudaError_t e = cudaMemcpy(d_tri, tri, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_h, hits, sizeof(float) * 7 * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        launch_sample_materials(s->dev, s->tex, s->maps, n, d_tri, d_h, d_out, 0);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, d_out, sizeof(float) * 10 * (size_t)n, cudaMemcpyDeviceToHost);
    buf.release();
    if (e != cudaSuccess) return ezrt_set_error(EZRT_ERR_CUDA, "scene_sample_materials: %s", cudaGetErrorString(e));
    return EZRT_OK;
}

int ezrt_scene_sample_textures(ezrt_scene* s, int n, const int32_t* tri, const float* points, float* uv_out, float* rgb_out) {
    if (!s || n < 0 || (n > 0 && (!tri || !points || !uv_out || !rgb_out))) return ezrt_set_error(EZRT_ERR_INVALID, "scene_sample_textures: bad argument");
    if (!s->has_textures) return ezrt_set_error(EZRT_ERR_INVALID, "scene_sample_textures: no textures (ezrt_scene_set_textures)");
    for (int i = 0; i < n; i++)
        if (tri[i] < 0 || tri[i] >= s->dev.n_triangles) return ezrt_set_error(EZRT_ERR_INVALID, "scene_sample_textures: triangle %d out of range", tri[i]);
    if (n == 0) return EZRT_OK;
    CU_CHECK(cudaSetDevice(s->device));
    DeviceBuffer buf;
    int rc = buf.ensure(sizeof(float) * 9 * (size_t)n + 256);
    if (rc) return rc;
    int32_t* d_tri = (int32_t*)buf.p;
    float* d_p = (float*)(d_tri + n);
    float* d_uv = d_p + 3 * (size_t)n;
    float* d_rgb = d_uv + 2 * (size_t)n;
    cudaError_t e = cudaMemcpy(d_tri, tri, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_p, points, sizeof(float) * 3 * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        launch_sample_textures(s->dev, s->tex, n, d_tri, d_p, d_uv, d_rgb, 0);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(uv_out, d_uv, sizeof(float) * 2 * (size_t)n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(rgb_out, d_rgb, sizeof(float) * 3 * (size_t)n, cudaMemcpyDeviceToHost);
    buf.release();
    if (e != cudaSuccess) return ezrt_set_error(EZRT_ERR_CUDA, "scene_sample_textures: %s", cudaGetErrorString(e));
    return EZRT_OK;
}

int ezrt_scene_destroy(ezrt_scene* s) {
    if (!s) return EZRT_OK;
    cudaSetDevice(s->device);
    s->nodes.release(); s->tri_geo.release(); s->tri_shade.release(); s->materials.release();
    s->hdr.release(); s->hdr_cache.release(); s->tiles_buf.release();
    s->acc_hot.release(); s->acc_tri_ref.release(); s->tri_leaf.release(); s->leaf_box.release(); s->defer_buf.release();
    s->acc_tri_leaf.release(); s->ref_to_acc.release(); s->acc_wide.release(); s->acc_wide_q16.release();
    s->queue_buf[0].release(); s->queue_buf[1].release(); s->shadow_buf.release();
    s->lo_buf.release(); s->le_buf.release(); s->counters_buf.release(); s->totals_buf.release(); s->fb_buf.release(); s->sort_buf.release();
    s->adapt_buf.release(); s->adapt_maps_buf.release();
    s->aov_rec_buf.release(); s->aov_maps_buf.release(); s->denoise_buf.release(); s->denoise_io_buf.release();
    s->lights_buf.release(); s->env_buf.release(); s->tex_buf.release(); s->tex_rec_buf.release();
    if (s->own_stream) cudaStreamDestroy(s->own_stream);
    if (s->copy_stream) cudaStreamDestroy(s->copy_stream);
    if (s->side_stream) cudaStreamDestroy(s->side_stream);
    if (s->ev_fork) cudaEventDestroy(s->ev_fork);
    if (s->ev_join) cudaEventDestroy(s->ev_join);
    s->side_hit_buf.release();
    if (s->fb_event) cudaEventDestroy(s->fb_event);
    if (s->ev_start) cudaEventDestroy(s->ev_start);
    if (s->ev_stop) cudaEventDestroy(s->ev_stop);
    for (cudaEvent_t e : s->ev_pool) cudaEventDestroy(e);
    delete s;
    return EZRT_OK;
}

// ------------------------------------------------------------------------------------------
// render
// ------------------------------------------------------------------------------------------
// The light sampling mode's options of a render (LightOptions, kernels.h) from the validated params: builds the light table, and the
// environment table when the map is a light, at the first render that needs them.
static int light_options(ezrt_scene* s, const ezrt_render_params* p, cudaStream_t st, LightOptions& o) {
    o = LightOptions{};
    if (p->mode != EZRT_MODE_DISNEY_LIGHTS) return EZRT_OK;
    int rc = build_lights(s, st);
    if (rc) return rc;
    o.lights = s->lights;
    // EZRT_PARAM_ENV_LIGHT: the map is one more light when the scene has a table (P_env = 1/2 beside triangle lights, 1 without);
    // without a table the render is mode 4's, and mode 4's kernels run
    if (p->reserved[0] & EZRT_PARAM_ENV_LIGHT) {
        if ((rc = build_env(s, st))) return rc;
        if (s->env.row_cdf) {
            o.env = s->env;
            o.env.p_env = (o.lights.n > 0) ? 0.5f : 1.0f;
            o.env_on = true;
        }
    }
    o.trans_on = (p->reserved[0] & EZRT_PARAM_TRANSMISSION) != 0;
    // EZRT_PARAM_MEDIUM (validated: a medium is set, no transmission); sigma_t == 0 is mode 4 and runs its kernels
    if ((p->reserved[0] & EZRT_PARAM_MEDIUM) && s->medium.sigma_t > 0.0f) {
        o.med = s->medium;
        o.medium_on = true;
    }
    // EZRT_PARAM_TEXTURES (validated: textures are set); tex.sh_base is carved with the shadow queue
    if (p->reserved[0] & EZRT_PARAM_TEXTURES) {
        o.tex = s->tex;
        o.tex_on = true;
        o.maps = s->maps;
        o.maps_on = (p->reserved[0] & EZRT_PARAM_MATERIAL_MAPS) != 0;   // validated: with the textures, and maps are set
    }
    return EZRT_OK;
}

// The render of ezrt_render_device (ad == av == nullptr), ezrt_render_adaptive_device (ad) and ezrt_render_aov_device (av): the
// arguments are validated.
static int render_device_impl(ezrt_scene* s, const ezrt_render_params* p, float* d_fb, cudaStream_t st, const AdaptiveRun* ad,
                              const AovRun* av = nullptr) {
    CU_CHECK(cudaSetDevice(s->device));
    int rc = prepare_tiles(s, p, st);
    if (rc) return rc;
    rc = s->totals_buf.ensure(sizeof(unsigned long long) * EZRT_TOTALS);
    if (rc) return rc;
    unsigned long long* totals = (unsigned long long*)s->totals_buf.p;
    // EZRT_PARAM_ACCUMULATE: counters, kernel spans and the device-time bracket continue from the previous render
    // (a benchmark reads them once after K renders instead of synchronising after every one)
    const bool accumulate = (p->reserved[0] & EZRT_PARAM_ACCUMULATE) != 0 && s->have_timing;
    if (!accumulate) {
        CU_CHECK(cudaEventRecord(s->ev_start, st));
        CU_CHECK(cudaMemsetAsync(totals, 0, sizeof(unsigned long long) * EZRT_TOTALS, st));
        s->launches = 0;
        s->spans.clear();
        s->ev_used = 0;
    }
    s->have_timing = false;   // set again once ev_stop is recorded (an early error return must not leave a dangling bracket)
    s->profiling = (p->profile == 1);
    RenderDev rd = make_render_dev(s, p);
    const TileDev* d_tiles = (const TileDev*)s->tiles_buf.p;
    const bool prune = s->regular_tree && (p->traverse != EZRT_TRAVERSE_REFERENCE);
    const bool accel = s->regular_tree && s->have_accel && (p->traverse == EZRT_TRAVERSE_ACCEL);
    LensDev lens_v;
    const LensDev* lens = thin_lens(p, &lens_v) ? &lens_v : nullptr;   // EZRT_PARAM_THIN_LENS (validated)
    if (rd.n_tiles == 0 || p->spp == 0) {
        CU_CHECK(cudaEventRecord(s->ev_stop, st));
        s->have_timing = true;
        return EZRT_OK;
    }

    if (p->pipeline == EZRT_PIPELINE_MEGAKERNEL) {
        if (s->fb_wait) {
            CU_CHECK(cudaStreamWaitEvent(st, s->fb_wait, 0));
            s->fb_wait = nullptr;
        }
        int sp = s->span_begin(0, st);
        launch_megakernel(s->dev, rd, d_tiles, prune, p->spp, d_fb, totals, st, lens);
        s->span_end(sp, st);
        s->launches++;
        CU_CHECK(cudaGetLastError());
        CU_CHECK(cudaEventRecord(s->ev_stop, st));
        s->have_timing = true;
        return EZRT_OK;
    }

    const size_t per_frame = (size_t)rd.n_tiles * EZRT_TILE_PIXELS;
    // the modes with a shadow pass: mode 3's environment samples, the light sampling mode's bounded light samples
    const bool lights_mode = (p->mode == EZRT_MODE_DISNEY_LIGHTS);
    const bool is_mode = (p->mode == EZRT_MODE_DISNEY_IS_MIS_P5) || lights_mode;
    LightOptions lopt;
    if ((rc = light_options(s, p, st, lopt))) return rc;
    int F = p->frames_per_batch;
    if (F <= 0) F = (int)std::max<size_t>(1, ((size_t)32 << 20) / per_frame);  // ~32 M sample slots per batch (~7.5 GB of state):
                                                                              // long queues amortise the persistent kernels' ramp-up and tail
    F = std::min(F, p->spp);
    {   // bound the batch by the memory that is actually there (scratch already held by this scene counts as available);
        // asked once per (slots per frame, integrator): cudaMemGetInfo is a driver round trip, the render path is launch-only
        const size_t per_slot = 2 * (sizeof(float4) * 4 + sizeof(float2)) + 2 * sizeof(float4) + sizeof(uint32_t) +
                                (is_mode ? (size_t)EZRT_SHADOW_SLOT_BYTES : 0) + (lopt.tex_on ? sizeof(float4) : 0) + (lopt.maps_on ? sizeof(float) : 0) + (s->sort_rays ? 2 * sizeof(uint32_t) : 0) +
                                (av ? 2 * sizeof(float4) : 0);
        if (s->fmax_key[0] != per_frame || s->fmax_key[1] != per_slot) {
            size_t free_b = 0, total_b = 0;
            s->fmax = (size_t)1 << 30;
            if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) {
                const size_t held = s->queue_buf[0].bytes + s->queue_buf[1].bytes + s->shadow_buf.bytes + s->lo_buf.bytes + s->le_buf.bytes +
                                    s->defer_buf.bytes + s->sort_buf.bytes + s->aov_rec_buf.bytes;
                const size_t avail = (size_t)((double)(free_b + held) * 0.9);
                s->fmax = avail / per_slot / per_frame;
                if (s->fmax < 1) return ezrt_set_error(EZRT_ERR_NOMEM, "render: %zu MB free, one frame of wavefront state needs %zu MB", free_b >> 20, (per_slot * per_frame) >> 20);
            }
            s->fmax_key[0] = per_frame;
            s->fmax_key[1] = per_slot;
        }
        F = (int)std::min<size_t>((size_t)F, s->fmax);
    }
    const size_t capacity = per_frame * (size_t)F;
    if (capacity >= ((size_t)1 << 31)) return ezrt_set_error(EZRT_ERR_INVALID, "render: batch too large");
    PathQueue q[2];
    ShadowQueue sq{};
    if ((rc = carve_queue(s->queue_buf[0], capacity, q[0]))) return rc;
    if ((rc = carve_queue(s->queue_buf[1], capacity, q[1]))) return rc;
    if ((rc = carve_shadow(s->shadow_buf, is_mode ? capacity : 1, sq))) return rc;
    if ((rc = s->lo_buf.ensure(sizeof(float4) * capacity))) return rc;
    if ((rc = s->le_buf.ensure(sizeof(float4) * capacity))) return rc;
    if (lopt.tex_on) {   // the shadow slots' textured base colours, after the 81-byte slots (the plain renders' slots stay as they are)
        if ((rc = s->shadow_buf.ensure(((size_t)EZRT_SHADOW_SLOT_BYTES + sizeof(float4)) * capacity + 512))) return rc;
        if ((rc = carve_shadow(s->shadow_buf, capacity, sq))) return rc;
        lopt.tex.sh_base = (float4*)((((uintptr_t)sq.lit + capacity) + 255) & ~(uintptr_t)255);
    }
    if (lopt.maps_on) {   // ... and their mapped metallic after those (the roughness rides in sh_base's fourth word)
        if ((rc = s->shadow_buf.ensure(((size_t)EZRT_SHADOW_SLOT_BYTES + sizeof(float4) + sizeof(float)) * capacity + 768))) return rc;
        if ((rc = carve_shadow(s->shadow_buf, capacity, sq))) return rc;
        lopt.tex.sh_base = (float4*)((((uintptr_t)sq.lit + capacity) + 255) & ~(uintptr_t)255);
        lopt.maps.sh_metal = (float*)((((uintptr_t)(lopt.tex.sh_base + capacity)) + 255) & ~(uintptr_t)255);
    }
    float4* aov_rec = nullptr;   // feature-buffer render only: the first-hit record of every sample slot
    if (av) {
        if ((rc = s->aov_rec_buf.ensure(2 * sizeof(float4) * capacity))) return rc;
        aov_rec = (float4*)s->aov_rec_buf.p;
    }
    const int n_stages = p->max_bounce + 2;
    // counters: [0,n) queue sizes, [n,2n) shadow sizes, [2n,3n) extend work, [3n,4n) shadow work,
    // [4n,6n) deferred-ray counts of the accel passes (extend, shadow), [6n,8n) work counters of their exact passes
    const int n_counters = 8 * n_stages;
    if ((rc = s->counters_buf.ensure(sizeof(uint32_t) * n_counters))) return rc;
    uint32_t* cnt = (uint32_t*)s->counters_buf.p;
    uint32_t *q_count = cnt, *s_count = cnt + n_stages, *w_ext = cnt + 2 * n_stages, *w_sh = cnt + 3 * n_stages;
    uint32_t *d_ext = cnt + 4 * n_stages, *d_sh = cnt + 5 * n_stages, *dw_ext = cnt + 6 * n_stages, *dw_sh = cnt + 7 * n_stages;
    if ((rc = s->defer_buf.ensure(sizeof(uint32_t) * (capacity + 64)))) return rc;
    uint32_t* defer_list = (uint32_t*)s->defer_buf.p;
    float4* Lo = (float4*)s->lo_buf.p;
    float4* Le = (float4*)s->le_buf.p;
    uint32_t *sort_keys = nullptr, *sort_perm = nullptr, *sort_bins = nullptr;
    if (s->sort_rays) {   // the optional bounce-ray sort (exact policies only)
        if ((rc = s->sort_buf.ensure(sizeof(uint32_t) * (2 * capacity + EZRT_SORT_BINS + 64)))) return rc;
        sort_keys = (uint32_t*)s->sort_buf.p;
        sort_perm = sort_keys + capacity;
        sort_bins = sort_perm + capacity;
    }

    unsigned long long* const count_ptr = (p->profile == 2) ? totals + 5 : nullptr;  // node visits, triangle tests of the W8 kernels
    // the deferred lane needs a second stream (highest priority: its small blocks go first when an SM has room), two events and
    // the hit records of up to EZRT_SIDE_CAP deferred rays
    const bool lane = accel && s->deferred_lane;
    float2* side_hit = nullptr;
    if (lane) {
        if (!s->side_stream) {
            int lo_pri = 0, hi_pri = 0;
            cudaDeviceGetStreamPriorityRange(&lo_pri, &hi_pri);
            if (cudaStreamCreateWithPriority(&s->side_stream, cudaStreamNonBlocking, hi_pri) != cudaSuccess) return ezrt_set_error(EZRT_ERR_CUDA, "render: side stream");
            if (cudaEventCreateWithFlags(&s->ev_fork, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&s->ev_join, cudaEventDisableTiming) != cudaSuccess)
                return ezrt_set_error(EZRT_ERR_CUDA, "render: events");
        }
        if ((rc = s->side_hit_buf.ensure(sizeof(float2) * (size_t)EZRT_SIDE_CAP))) return rc;
        side_hit = (float2*)s->side_hit_buf.p;
    }
    const bool l2_window = accel && s->l2_persist_bytes > 0 && s->hot_bytes > 0;
    if (l2_window) {
        cudaStreamAttrValue attr;
        memset(&attr, 0, sizeof(attr));
        attr.accessPolicyWindow.base_ptr = s->hot_base;
        attr.accessPolicyWindow.num_bytes = std::min<size_t>(s->hot_bytes, (size_t)s->max_window_bytes);
        attr.accessPolicyWindow.hitRatio = (float)std::min(1.0, (double)s->l2_persist_bytes / (double)attr.accessPolicyWindow.num_bytes);
        attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
        attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
        cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &attr);
        cudaGetLastError();
    }
    // Adaptive sampling: batches end on the test points; after each test the next batches run over the surviving tiles only
    // (rd.n_tiles, d_tiles), and with an automatic batch size they take more frames, up to the capacity sized above.
    TileDev *tiles_a = nullptr, *tiles_b = nullptr;
    unsigned char* keep = nullptr;
    unsigned int* blocks_done = nullptr;
    int32_t* test_counts = nullptr;
    if (ad) {
        const size_t list_bytes = ((sizeof(TileDev) * (size_t)rd.n_tiles + 255) / 256) * 256;
        const size_t keep_bytes = (((size_t)rd.n_tiles + 255) / 256) * 256;
        if ((rc = s->adapt_buf.ensure(2 * list_bytes + keep_bytes + 16))) return rc;
        char* base = (char*)s->adapt_buf.p;
        tiles_a = (TileDev*)base;
        tiles_b = (TileDev*)(base + list_bytes);
        keep = (unsigned char*)(base + 2 * list_bytes);
        blocks_done = (unsigned int*)(base + 2 * list_bytes + keep_bytes);
        test_counts = (int32_t*)(blocks_done + 1);
        CU_CHECK(cudaMemsetAsync(blocks_done, 0, sizeof(unsigned int), st));
    }
    size_t active_pixels = s->n_pixels;
    int next_test = ad ? ad->min_spp : p->spp;
    for (int done = 0; done < p->spp && rd.n_tiles > 0;) {
        const int nf = std::min(F, std::min(p->spp, next_test) - done);
        const uint32_t n_slots = (uint32_t)((size_t)rd.n_tiles * EZRT_TILE_PIXELS * (size_t)nf);
        const uint32_t batch_first = p->first_frame + (uint32_t)done;
        CU_CHECK(cudaMemsetAsync(cnt, 0, sizeof(uint32_t) * n_counters, st));
        // accel policy: camera rays are generated inside the first extend kernel.  Thin-lens camera rays do not share an origin:
        // k_generate<true> queues them and bounce 0 takes the unfused form under every policy (the accel policy's per-ray kernels,
        // k_shade reading the rays back from queue 0)
        const bool fused_camera = accel && !lens;
        int sp = -1;
        if (!fused_camera) {
            sp = s->span_begin(3, st);
            launch_generate(rd, d_tiles, n_slots, batch_first, q[0], &q_count[0], s->n_sms, st, lens);
            s->span_end(sp, st);
            s->launches++;
        }
        for (int b = 0; b <= p->max_bounce; b++) {
            PathQueue& qin = q[b & 1];
            PathQueue& qout = q[(b + 1) & 1];
            const uint32_t* perm = nullptr;
            if (b > 0 && s->sort_rays) {  // optional experiment
                sp = s->span_begin(3, st);
                launch_ray_sort(s->dev, qin, &q_count[b], sort_keys, sort_bins, sort_perm, n_slots, s->n_sms, st);
                s->span_end(sp, st);
                s->launches += 3;
                perm = sort_perm;
            }
            sp = s->span_begin(0, st);
            const int exact_gate = lane ? 2 : 0;   // lane: only an overflowing list of deferred rays is traced in line
            if (accel && fused_camera && b == 0) {
                launch_extend_camera(s->dev, rd, d_tiles, batch_first, n_slots, s->camera_pixel_major ? (uint32_t)nf : 0u, qin, &w_ext[b], defer_list, &d_ext[b], &dw_ext[b],
                                     s->n_sms, count_ptr, st, exact_gate);
                s->launches++;
            } else if (accel) {
                launch_extend_accel(s->dev, qin, &q_count[b], &w_ext[b], defer_list, &d_ext[b], &dw_ext[b], n_slots, s->n_sms, count_ptr, perm, st, exact_gate);
                s->launches++;
            } else {
                launch_extend(s->dev, prune, false, qin, &q_count[b], &w_ext[b], perm, 0, n_slots, s->n_sms, st);
            }
            s->span_end(sp, st);
            const uint32_t n_fused = (fused_camera && b == 0) ? n_slots : 0u;
            if (lane) {   // fork: the deferred rays of this bounce are traced exactly and shaded on the side stream ...
                CU_CHECK(cudaEventRecord(s->ev_fork, st));
                CU_CHECK(cudaStreamWaitEvent(s->side_stream, s->ev_fork, 0));
                launch_deferred_lane(s->dev, rd, d_tiles, b, batch_first, qin, defer_list, &d_ext[b], &dw_ext[b], side_hit, qout, &q_count[b + 1], sq, &s_count[b],
                                     Lo, Le, n_fused, (uint32_t)nf, s->n_sms, s->side_stream, b == 0 ? aov_rec : nullptr, lopt);
                CU_CHECK(cudaEventRecord(s->ev_join, s->side_stream));
                s->launches += 2;
            }
            sp = s->span_begin(1, st);
            launch_shade(s->dev, rd, d_tiles, b, batch_first, qin, &q_count[b], qout, &q_count[b + 1], sq, &s_count[b], Lo, Le,
                         n_slots, n_fused, (uint32_t)nf, s->n_sms, st, b == 0 ? aov_rec : nullptr, lopt);
            if (lane) CU_CHECK(cudaStreamWaitEvent(st, s->ev_join, 0));   // ... while this k_shade shades all the others; join
            s->span_end(sp, st);
            s->launches += 2;
            if (is_mode && b < p->max_bounce) {
                sp = s->span_begin(2, st);
                if (accel) {
                    launch_shadow_accel(s->dev, sq, &s_count[b], &w_sh[b], Lo, defer_list, &d_sh[b], &dw_sh[b], n_slots, s->n_sms, count_ptr, st, lights_mode);
                    s->launches++;
                } else {
                    launch_shadow(s->dev, prune, sq, &s_count[b], &w_sh[b], Lo, nullptr, n_slots, s->n_sms, st, lights_mode);
                }
                s->span_end(sp, st);
                sp = s->span_begin(1, st);   // shading work: counted with k_shade
                launch_nee(s->dev, rd, sq, &s_count[b], Lo, n_slots, s->n_sms, st, lopt);
                s->span_end(sp, st);
                s->launches += 2;
            }
        }
        sp = s->span_begin(3, st);
        if (s->fb_wait) {   // ezrt_render: lastFrame arrives on the copy stream
            CU_CHECK(cudaStreamWaitEvent(st, s->fb_wait, 0));
            s->fb_wait = nullptr;
        }
        launch_blend(rd, d_tiles, nf, batch_first, Lo, Le, d_fb, av ? av->d_luma2 : ad ? ad->d_luma2 : nullptr, ad ? ad->d_spp : nullptr, aov_rec,
                     av ? av->d_aov : nullptr, st);
        launch_tally(q_count, s_count, d_ext, d_sh, p->max_bounce + 1, totals, fused_camera ? (uint32_t)(active_pixels * (size_t)nf) : 0u, st);
        s->span_end(sp, st);
        s->launches += 2;
        done += nf;
        if (ad && done == next_test && done < p->spp) {
            TileDev* survivors = (d_tiles == tiles_a) ? tiles_b : tiles_a;
            sp = s->span_begin(3, st);
            launch_adaptive_check(rd, d_tiles, done, ad->threshold, d_fb, ad->d_luma2, keep, blocks_done, survivors, test_counts, st);
            s->span_end(sp, st);
            s->launches++;
            CU_CHECK(cudaGetLastError());
            int32_t left[2] = {0, 0};   // surviving tiles, their pixels: the one synchronisation of a test
            CU_CHECK(cudaMemcpyAsync(left, test_counts, sizeof(left), cudaMemcpyDeviceToHost, st));
            CU_CHECK(cudaStreamSynchronize(st));
            d_tiles = survivors;
            rd.n_tiles = left[0];
            active_pixels = (size_t)left[1];
            if (p->frames_per_batch <= 0 && rd.n_tiles > 0)
                F = (int)std::min<size_t>(capacity / ((size_t)rd.n_tiles * EZRT_TILE_PIXELS), (size_t)p->spp);
            next_test += ad->check_interval;
        }
    }
    if (l2_window) {  // leave the caller's stream as it was
        cudaStreamAttrValue attr;
        memset(&attr, 0, sizeof(attr));
        attr.accessPolicyWindow.num_bytes = 0;
        cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &attr);
        cudaGetLastError();
    }
    CU_CHECK(cudaGetLastError());
    CU_CHECK(cudaEventRecord(s->ev_stop, st));
    s->have_timing = true;
    return EZRT_OK;
}

int ezrt_render_device(ezrt_scene* s, const ezrt_render_params* p, float* d_fb, void* cuda_stream) {
    int rc = validate_params(s, p);
    if (rc) return rc;
    if (!d_fb) return ezrt_set_error(EZRT_ERR_INVALID, "render: null framebuffer");
    return render_device_impl(s, p, d_fb, (cudaStream_t)cuda_stream, nullptr);
}

int ezrt_render_adaptive_device(ezrt_scene* s, const ezrt_render_params* p, const ezrt_adaptive_params* a, float* d_fb, int32_t* d_spp,
                                float* d_luma2, void* cuda_stream) {
    int rc = validate_params(s, p);
    if (!rc) rc = validate_adaptive(p, a);
    if (rc) return rc;
    if (!d_fb || !d_spp || !d_luma2) return ezrt_set_error(EZRT_ERR_INVALID, "render_adaptive: null output buffer");
    const AdaptiveRun ad{a->threshold, a->min_spp, a->check_interval, d_spp, d_luma2};
    return render_device_impl(s, p, d_fb, (cudaStream_t)cuda_stream, &ad);
}

int ezrt_render_adaptive(ezrt_scene* s, const ezrt_render_params* p, const ezrt_adaptive_params* a, float* framebuffer, int32_t* spp,
                         float* luma2) {
    int rc = validate_params(s, p);
    if (!rc) rc = validate_adaptive(p, a);
    if (rc) return rc;
    if (!framebuffer || !spp || !luma2) return ezrt_set_error(EZRT_ERR_INVALID, "render_adaptive: null output buffer");
    CU_CHECK(cudaSetDevice(s->device));
    const size_t npix = (size_t)ezrt_partition_pixels(p->width, p->height, p->part_rank, p->part_count);
    const size_t fb_bytes = sizeof(float) * npix * p->out_channels;
    const size_t map_bytes = ((sizeof(float) * npix + 255) / 256) * 256;
    if ((rc = s->fb_buf.ensure(std::max<size_t>(fb_bytes, 16)))) return rc;
    if ((rc = s->adapt_maps_buf.ensure(2 * map_bytes + 16))) return rc;
    int32_t* d_spp = (int32_t*)s->adapt_maps_buf.p;
    float* d_luma2 = (float*)((char*)s->adapt_maps_buf.p + map_bytes);
    cudaStream_t st = s->own_stream;
    s->fb_wait = nullptr;
    const AdaptiveRun ad{a->threshold, a->min_spp, a->check_interval, d_spp, d_luma2};
    if ((rc = render_device_impl(s, p, (float*)s->fb_buf.p, st, &ad))) return rc;
    CU_CHECK(cudaMemcpyAsync(framebuffer, s->fb_buf.p, fb_bytes, cudaMemcpyDeviceToHost, st));
    CU_CHECK(cudaMemcpyAsync(spp, d_spp, sizeof(int32_t) * npix, cudaMemcpyDeviceToHost, st));
    CU_CHECK(cudaMemcpyAsync(luma2, d_luma2, sizeof(float) * npix, cudaMemcpyDeviceToHost, st));
    CU_CHECK(cudaStreamSynchronize(st));
    return EZRT_OK;
}

int ezrt_render(ezrt_scene* s, const ezrt_render_params* p, float* framebuffer) {
    int rc = validate_params(s, p);
    if (rc) return rc;
    if (!framebuffer) return ezrt_set_error(EZRT_ERR_INVALID, "render: null framebuffer");
    CU_CHECK(cudaSetDevice(s->device));
    int64_t npix = ezrt_partition_pixels(p->width, p->height, p->part_rank, p->part_count);
    size_t bytes = sizeof(float) * (size_t)npix * p->out_channels;
    rc = s->fb_buf.ensure(std::max<size_t>(bytes, 16));
    if (rc) return rc;
    cudaStream_t st = s->own_stream;
    // lastFrame is only needed by the first k_blend: its upload runs on a second stream, under the tracing kernels
    s->fb_wait = nullptr;
    static const bool overlap_upload = []() { const char* e = getenv("EZRT_RENDER_OVERLAP"); return !(e && atoi(e) == 0); }();
    if (p->first_frame > 0 && !overlap_upload) {
        CU_CHECK(cudaMemcpyAsync(s->fb_buf.p, framebuffer, bytes, cudaMemcpyHostToDevice, st));
    } else if (p->first_frame > 0) {
        if (!s->copy_stream && cudaStreamCreateWithFlags(&s->copy_stream, cudaStreamNonBlocking) != cudaSuccess) return ezrt_set_error(EZRT_ERR_CUDA, "render: stream");
        if (!s->fb_event && cudaEventCreateWithFlags(&s->fb_event, cudaEventDisableTiming) != cudaSuccess) return ezrt_set_error(EZRT_ERR_CUDA, "render: event");
        CU_CHECK(cudaMemcpyAsync(s->fb_buf.p, framebuffer, bytes, cudaMemcpyHostToDevice, s->copy_stream));
        CU_CHECK(cudaEventRecord(s->fb_event, s->copy_stream));
        s->fb_wait = s->fb_event;
    }
    rc = ezrt_render_device(s, p, (float*)s->fb_buf.p, st);
    if (s->fb_wait) {  // the render returned before its first blend (error, empty part): do not leave the copy behind
        cudaStreamWaitEvent(st, s->fb_wait, 0);
        s->fb_wait = nullptr;
    }
    if (rc) return rc;
    CU_CHECK(cudaMemcpyAsync(framebuffer, s->fb_buf.p, bytes, cudaMemcpyDeviceToHost, st));
    CU_CHECK(cudaStreamSynchronize(st));
    return EZRT_OK;
}

int ezrt_render_aov_device(ezrt_scene* s, const ezrt_render_params* p, float* d_fb, float* d_aov, float* d_luma2, void* cuda_stream) {
    int rc = validate_params(s, p);
    if (!rc) rc = validate_aov(p);
    if (rc) return rc;
    if (!d_fb || !d_aov || !d_luma2) return ezrt_set_error(EZRT_ERR_INVALID, "render_aov: null output buffer");
    if ((uintptr_t)d_aov % 16) return ezrt_set_error(EZRT_ERR_INVALID, "render_aov: the aov buffer must be 16-byte aligned");
    const AovRun av{d_aov, d_luma2};
    return render_device_impl(s, p, d_fb, (cudaStream_t)cuda_stream, nullptr, &av);
}

int ezrt_render_aov(ezrt_scene* s, const ezrt_render_params* p, float* framebuffer, float* aov, float* luma2) {
    int rc = validate_params(s, p);
    if (!rc) rc = validate_aov(p);
    if (rc) return rc;
    if (!framebuffer || !aov || !luma2) return ezrt_set_error(EZRT_ERR_INVALID, "render_aov: null output buffer");
    CU_CHECK(cudaSetDevice(s->device));
    const size_t npix = (size_t)ezrt_partition_pixels(p->width, p->height, p->part_rank, p->part_count);
    const size_t fb_bytes = sizeof(float) * npix * p->out_channels;
    const size_t aov_bytes = ((sizeof(float) * 8 * npix + 255) / 256) * 256;
    if ((rc = s->fb_buf.ensure(std::max<size_t>(fb_bytes, 16)))) return rc;
    if ((rc = s->aov_maps_buf.ensure(aov_bytes + sizeof(float) * npix + 16))) return rc;
    float* d_aov = (float*)s->aov_maps_buf.p;
    float* d_luma2 = (float*)((char*)s->aov_maps_buf.p + aov_bytes);
    cudaStream_t st = s->own_stream;
    s->fb_wait = nullptr;
    if (p->first_frame > 0) {   // all three are in/out: the render goes on from where they stand
        CU_CHECK(cudaMemcpyAsync(s->fb_buf.p, framebuffer, fb_bytes, cudaMemcpyHostToDevice, st));
        CU_CHECK(cudaMemcpyAsync(d_aov, aov, sizeof(float) * 8 * npix, cudaMemcpyHostToDevice, st));
        CU_CHECK(cudaMemcpyAsync(d_luma2, luma2, sizeof(float) * npix, cudaMemcpyHostToDevice, st));
    }
    const AovRun av{d_aov, d_luma2};
    if ((rc = render_device_impl(s, p, (float*)s->fb_buf.p, st, nullptr, &av))) return rc;
    CU_CHECK(cudaMemcpyAsync(framebuffer, s->fb_buf.p, fb_bytes, cudaMemcpyDeviceToHost, st));
    CU_CHECK(cudaMemcpyAsync(aov, d_aov, sizeof(float) * 8 * npix, cudaMemcpyDeviceToHost, st));
    CU_CHECK(cudaMemcpyAsync(luma2, d_luma2, sizeof(float) * npix, cudaMemcpyDeviceToHost, st));
    CU_CHECK(cudaStreamSynchronize(st));
    return EZRT_OK;
}

static int validate_denoise(const ezrt_scene* s, const ezrt_denoise_params* dp, int channels, int width, int height, int n_frames) {
    if (!s || !dp) return ezrt_set_error(EZRT_ERR_INVALID, "denoise: null argument");
    if (dp->iterations < 1 || dp->iterations > 10) return ezrt_set_error(EZRT_ERR_INVALID, "denoise: iterations must be in 1..10 (got %d)", dp->iterations);
    const float sg[4] = {dp->sigma_l, dp->sigma_n, dp->sigma_z, dp->sigma_a};
    for (float v : sg)
        if (!std::isfinite(v) || !(v > 0.0f)) return ezrt_set_error(EZRT_ERR_INVALID, "denoise: every sigma must be finite and > 0 (got %g)", (double)v);
    if (dp->reserved != 0) return ezrt_set_error(EZRT_ERR_INVALID, "denoise: reserved field must be 0");
    if (channels != 3 && channels != 4) return ezrt_set_error(EZRT_ERR_INVALID, "denoise: channels must be 3 or 4");
    if (width <= 0 || height <= 0) return ezrt_set_error(EZRT_ERR_INVALID, "denoise: bad image size");
    if (n_frames < 1) return ezrt_set_error(EZRT_ERR_INVALID, "denoise: n_frames must be >= 1 (got %d)", n_frames);
    return EZRT_OK;
}

static int denoise_impl(ezrt_scene* s, const ezrt_denoise_params* dp, const float* d_color, int channels, const float* d_aov, const float* d_luma2,
                        int width, int height, int n_frames, float* d_out, cudaStream_t st) {
    const size_t npix = (size_t)width * height;
    const size_t half = ((sizeof(float4) * npix + 255) / 256) * 256;
    int rc = s->denoise_buf.ensure(2 * half);
    if (rc) return rc;
    float4* cv0 = (float4*)s->denoise_buf.p;
    float4* cv1 = (float4*)((char*)s->denoise_buf.p + half);
    launch_denoise(d_color, channels, d_aov, d_luma2, n_frames, width, height, dp->iterations, dp->sigma_l, dp->sigma_n, dp->sigma_z,
                   dp->sigma_a, cv0, cv1, d_out, st);
    CU_CHECK(cudaGetLastError());
    return EZRT_OK;
}

int ezrt_denoise_device(ezrt_scene* s, const ezrt_denoise_params* dp, const float* d_color, int channels, const float* d_aov,
                        const float* d_luma2, int width, int height, int n_frames, float* d_out, void* cuda_stream) {
    int rc = validate_denoise(s, dp, channels, width, height, n_frames);
    if (rc) return rc;
    if (!d_color || !d_aov || !d_luma2 || !d_out) return ezrt_set_error(EZRT_ERR_INVALID, "denoise: null buffer");
    if ((uintptr_t)d_aov % 16) return ezrt_set_error(EZRT_ERR_INVALID, "denoise: the aov buffer must be 16-byte aligned");
    CU_CHECK(cudaSetDevice(s->device));
    return denoise_impl(s, dp, d_color, channels, d_aov, d_luma2, width, height, n_frames, d_out, (cudaStream_t)cuda_stream);
}

int ezrt_denoise(ezrt_scene* s, const ezrt_denoise_params* dp, const float* color, int channels, const float* aov, const float* luma2,
                 int width, int height, int n_frames, float* out) {
    int rc = validate_denoise(s, dp, channels, width, height, n_frames);
    if (rc) return rc;
    if (!color || !aov || !luma2 || !out) return ezrt_set_error(EZRT_ERR_INVALID, "denoise: null buffer");
    CU_CHECK(cudaSetDevice(s->device));
    const size_t npix = (size_t)width * height;
    const size_t aov_bytes = ((sizeof(float) * 8 * npix + 255) / 256) * 256;
    const size_t color_bytes = ((sizeof(float) * channels * npix + 255) / 256) * 256;
    if ((rc = s->denoise_io_buf.ensure(aov_bytes + color_bytes + sizeof(float) * npix))) return rc;
    float* d_aov = (float*)s->denoise_io_buf.p;
    float* d_color = (float*)((char*)s->denoise_io_buf.p + aov_bytes);
    float* d_luma2 = (float*)((char*)s->denoise_io_buf.p + aov_bytes + color_bytes);
    cudaStream_t st = s->own_stream;
    CU_CHECK(cudaMemcpyAsync(d_aov, aov, sizeof(float) * 8 * npix, cudaMemcpyHostToDevice, st));
    CU_CHECK(cudaMemcpyAsync(d_color, color, sizeof(float) * channels * npix, cudaMemcpyHostToDevice, st));
    CU_CHECK(cudaMemcpyAsync(d_luma2, luma2, sizeof(float) * npix, cudaMemcpyHostToDevice, st));
    if ((rc = denoise_impl(s, dp, d_color, channels, d_aov, d_luma2, width, height, n_frames, d_color, st))) return rc;
    CU_CHECK(cudaMemcpyAsync(out, d_color, sizeof(float) * channels * npix, cudaMemcpyDeviceToHost, st));
    CU_CHECK(cudaStreamSynchronize(st));
    return EZRT_OK;
}

int ezrt_get_counters(ezrt_scene* s, ezrt_counters* out) {
    if (!s || !out) return ezrt_set_error(EZRT_ERR_INVALID, "get_counters: null argument");
    memset(out, 0, sizeof(*out));
    if (!s->have_timing) return EZRT_OK;
    CU_CHECK(cudaSetDevice(s->device));
    CU_CHECK(cudaEventSynchronize(s->ev_stop));
    unsigned long long t[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    CU_CHECK(cudaMemcpy(t, s->totals_buf.p, sizeof(t), cudaMemcpyDeviceToHost));
    out->deferred_rays = t[4];
    out->node_visits = t[5] + t[7];          // t[5]: visits of 128-byte exact nodes, t[7]: of quantised nodes (Q16 form 96 B, W8 80 B)
    out->tri_tests = t[6];
    out->node_bytes = t[5] * 128ull + t[7] * 96ull;
    out->tri_bytes = t[6] * 64ull;
    out->node_visits_96 = t[7];
    float ms = 0.0f;
    CU_CHECK(cudaEventElapsedTime(&ms, s->ev_start, s->ev_stop));
    out->primary_rays = t[0]; out->bounce_rays = t[1]; out->shadow_rays = t[2];
    out->rays = t[0] + t[1] + t[2];
    out->samples = t[3];
    out->kernel_launches = s->launches;
    out->device_ms = ms;
    return EZRT_OK;
}

// words [first, first + 4) of the bounce and the shadow pass's blocks of the totals (kernels.h) -> out[0..3], out[4..7]
static int w8_pass_words(ezrt_scene* s, int first, uint64_t* out) {
    for (int k = 0; k < 8; k++) out[k] = 0;
    if (!s->have_timing) return EZRT_OK;
    CU_CHECK(cudaSetDevice(s->device));
    CU_CHECK(cudaEventSynchronize(s->ev_stop));
    static_assert(5 + EZRT_W8_PHASES_SHADOW + EZRT_W8_PASS_WORDS <= EZRT_TOTALS, "totals layout");
    unsigned long long t[EZRT_TOTALS];
    CU_CHECK(cudaMemcpy(t, s->totals_buf.p, sizeof(t), cudaMemcpyDeviceToHost));
    for (int k = 0; k < 4; k++) {
        out[k] = t[5 + EZRT_W8_PHASES_EXTEND + first + k];
        out[4 + k] = t[5 + EZRT_W8_PHASES_SHADOW + first + k];
    }
    return EZRT_OK;
}

int ezrt_get_w8_phase_cycles(ezrt_scene* s, uint64_t* out) {
    if (!s || !out) return ezrt_set_error(EZRT_ERR_INVALID, "get_w8_phase_cycles: null argument");
    return w8_pass_words(s, 0, out);
}

int ezrt_get_w8_step_counts(ezrt_scene* s, uint64_t* out) {
    if (!s || !out) return ezrt_set_error(EZRT_ERR_INVALID, "get_w8_step_counts: null argument");
    return w8_pass_words(s, 4, out);
}

int ezrt_get_kernel_times(ezrt_scene* s, double* ms, uint64_t* launches) {
    if (!s || !ms || !launches) return ezrt_set_error(EZRT_ERR_INVALID, "get_kernel_times: null argument");
    for (int k = 0; k < 4; k++) { ms[k] = 0.0; launches[k] = 0; }
    if (!s->have_timing || s->spans.empty()) return EZRT_OK;
    CU_CHECK(cudaSetDevice(s->device));
    CU_CHECK(cudaEventSynchronize(s->ev_stop));
    for (const auto& sp : s->spans) {
        float t = 0.0f;
        CU_CHECK(cudaEventElapsedTime(&t, s->ev_pool[sp.e0], s->ev_pool[sp.e1]));
        ms[sp.cls] += t;
        launches[sp.cls] += 1;
    }
    return EZRT_OK;
}

// ------------------------------------------------------------------------------------------
// image partition
// ------------------------------------------------------------------------------------------
int64_t ezrt_partition_pixels(int width, int height, int rank, int count) {
    if (width <= 0 || height <= 0 || count < 1 || rank < 0 || rank >= count) return EZRT_ERR_INVALID;
    int64_t n = 0;
    for (const TileDev& t : partition_tiles(width, height, rank, count)) n += (int64_t)t.w * t.h;
    return n;
}

int ezrt_partition_scatter(const float* d_compact, float* d_full, int width, int height, int channels, int rank, int count,
                           void* cuda_stream) {
    if (!d_compact || !d_full || channels < 1) return ezrt_set_error(EZRT_ERR_INVALID, "partition_scatter: bad argument");
    if (width <= 0 || height <= 0 || count < 1 || rank < 0 || rank >= count) return ezrt_set_error(EZRT_ERR_INVALID, "partition_scatter: bad partition");
    // device tile lists are cached per (device, image, part): the gather runs once per render
    auto& cache = scatter_cache();
    std::mutex& mu = scatter_mutex();
    int device = 0;
    CU_CHECK(cudaGetDevice(&device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    ScatterEntry ent;
    {
        std::lock_guard<std::mutex> lock(mu);
        std::array<int, 5> key = {device, width, height, rank, count};
        auto it = cache.find(key);
        if (it == cache.end()) {
            std::vector<TileDev> tiles = partition_tiles(width, height, rank, count);
            ScatterEntry e{nullptr, (int)tiles.size()};
            if (!tiles.empty()) {
                CU_CHECK(cudaMalloc(&e.d_tiles, sizeof(TileDev) * tiles.size()));
                CU_CHECK(cudaMemcpy(e.d_tiles, tiles.data(), sizeof(TileDev) * tiles.size(), cudaMemcpyHostToDevice));
            }
            it = cache.emplace(key, e).first;
        }
        ent = it->second;
    }
    if (ent.n == 0) return EZRT_OK;
    launch_partition_scatter(d_compact, d_full, ent.d_tiles, ent.n, width, channels, st);
    CU_CHECK(cudaGetLastError());
    return EZRT_OK;
}

int ezrt_partition_cache_clear(int device) {
    std::lock_guard<std::mutex> lock(scatter_mutex());
    auto& cache = scatter_cache();
    int prev = 0;
    cudaGetDevice(&prev);
    for (auto it = cache.begin(); it != cache.end();) {
        if (device < 0 || it->first[0] == device) {
            if (it->second.d_tiles) {
                cudaSetDevice(it->first[0]);
                cudaFree(it->second.d_tiles);
            }
            it = cache.erase(it);
        } else {
            ++it;
        }
    }
    cudaSetDevice(prev);
    cudaGetLastError();
    return EZRT_OK;
}

int ezrt_partition_scatter_host(const float* compact, float* full, int width, int height, int channels, int rank, int count) {
    if (!compact || !full || channels < 1) return ezrt_set_error(EZRT_ERR_INVALID, "partition_scatter_host: bad argument");
    for (const TileDev& t : partition_tiles(width, height, rank, count))
        for (int iy = 0; iy < t.h; iy++)
            for (int ix = 0; ix < t.w; ix++) {
                size_t src = ((size_t)t.pixel_offset + (size_t)iy * t.w + ix) * channels;
                size_t dst = ((size_t)(t.y0 + iy) * width + (t.x0 + ix)) * channels;
                for (int c = 0; c < channels; c++) full[dst + c] = compact[src + c];
            }
    return EZRT_OK;
}

// ------------------------------------------------------------------------------------------
// post pass
// ------------------------------------------------------------------------------------------
int ezrt_post_tonemap(const float* d_in, int channels, float* d_out, int64_t n_pixels, float limit, void* cuda_stream) {
    if (!d_in || !d_out || (channels != 3 && channels != 4) || n_pixels < 0) return ezrt_set_error(EZRT_ERR_INVALID, "post_tonemap: bad argument");
    launch_tonemap(d_in, channels, d_out, (long long)n_pixels, limit, (cudaStream_t)cuda_stream);
    CU_CHECK(cudaGetLastError());
    return EZRT_OK;
}

// ------------------------------------------------------------------------------------------
// single-function entry points (parity tests)
// ------------------------------------------------------------------------------------------
int ezrt_trace_rays(ezrt_scene* s, int n, const float* origins, const float* dirs, int traverse, int any_hit, int p3_normal_fudge,
                    int32_t* out_hit, float* out_distance, int32_t* out_triangle, int32_t* out_inside, float* out_point,
                    float* out_normal) {
    if (!s || n < 0 || !origins || !dirs || !out_hit || !out_distance || !out_triangle || !out_inside || !out_point || !out_normal)
        return ezrt_set_error(EZRT_ERR_INVALID, "trace_rays: null argument");
    if (n == 0) return EZRT_OK;
    CU_CHECK(cudaSetDevice(s->device));
    // the rays go through the production path: a ray queue traced by the persistent extend kernels
    std::vector<float4> ho(n), hd(n);
    for (int i = 0; i < n; i++) {
        ho[i] = make_float4(origins[3 * i], origins[3 * i + 1], origins[3 * i + 2], 0.0f);
        hd[i] = make_float4(dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2], 0.0f);
    }
    DeviceBuffer buf;
    const size_t N = (size_t)n;
    int rc = buf.ensure(sizeof(float4) * 2 * N + sizeof(float2) * N + sizeof(float) * 7 * N + sizeof(int) * 4 * N + 1024);
    if (rc) return rc;
    char* p = (char*)buf.p;
    PathQueue q{};
    q.ray_o = (float4*)p; p += sizeof(float4) * N;
    q.ray_d = (float4*)p; p += sizeof(float4) * N;
    q.hit = (float2*)p; p += sizeof(float2) * N;
    float* d_point = (float*)p; p += sizeof(float) * 3 * N;
    float* d_normal = (float*)p; p += sizeof(float) * 3 * N;
    float* d_dist = (float*)p; p += sizeof(float) * N;
    int* d_hit = (int*)p; p += sizeof(int) * N;
    int* d_tri = (int*)p; p += sizeof(int) * N;
    int* d_inside = (int*)p; p += sizeof(int) * N;
    uint32_t* d_defer = (uint32_t*)p; p += sizeof(uint32_t) * N;
    uint32_t* d_cnt = (uint32_t*)p;  // [0] n, [1] work, [2] deferred, [3] deferred work
    if (!s->regular_tree) traverse = EZRT_TRAVERSE_REFERENCE;
    else if (traverse == EZRT_TRAVERSE_ACCEL && (!s->have_accel || any_hit)) traverse = EZRT_TRAVERSE_PRUNED;  // any-hit probes take the exact kernel
    cudaStream_t st = s->own_stream;
    const uint32_t counters[4] = {(uint32_t)n, 0u, 0u, 0u};
    cudaError_t e = cudaMemcpyAsync(q.ray_o, ho.data(), sizeof(float4) * N, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(q.ray_d, hd.data(), sizeof(float4) * N, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_cnt, counters, sizeof(counters), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        if (traverse == EZRT_TRAVERSE_ACCEL)
            launch_extend_accel(s->dev, q, d_cnt, d_cnt + 1, d_defer, d_cnt + 2, d_cnt + 3, (uint32_t)n, s->n_sms, nullptr, nullptr, st);
        else
            launch_extend(s->dev, traverse != EZRT_TRAVERSE_REFERENCE, any_hit != 0, q, d_cnt, d_cnt + 1, nullptr, 0, (uint32_t)n, s->n_sms, st);
        launch_trace_finish(s->dev, n, q, p3_normal_fudge, traverse == EZRT_TRAVERSE_ACCEL, d_hit, d_dist, d_tri, d_inside, d_point, d_normal, st);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(out_hit, d_hit, sizeof(int) * N, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out_distance, d_dist, sizeof(float) * N, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out_triangle, d_tri, sizeof(int) * N, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out_inside, d_inside, sizeof(int) * N, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out_point, d_point, sizeof(float) * 3 * N, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out_normal, d_normal, sizeof(float) * 3 * N, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    buf.release();
    if (e != cudaSuccess) return ezrt_set_error(EZRT_ERR_CUDA, "trace_rays: %s", cudaGetErrorString(e));
    return EZRT_OK;
}

int ezrt_scene_lights(ezrt_scene* s, int cap, int32_t* tri_out, float* cdf_out, double* total_out) {
    if (!s || cap < 0) return ezrt_set_error(EZRT_ERR_INVALID, "scene_lights: bad argument");
    CU_CHECK(cudaSetDevice(s->device));
    int rc = build_lights(s, s->own_stream);
    if (rc) return rc;
    const int K = (int)s->light_tri.size();
    const int m = std::min(K, cap);
    if (tri_out) std::copy(s->light_tri.begin(), s->light_tri.begin() + m, tri_out);
    if (cdf_out) std::copy(s->light_cdf.begin(), s->light_cdf.begin() + m, cdf_out);
    if (total_out) *total_out = s->light_total;
    return K;
}

int ezrt_scene_env_light(ezrt_scene* s, float* row_cdf, float* col_cdf, float* texel_pdf, double* total) {
    if (!s) return ezrt_set_error(EZRT_ERR_INVALID, "scene_env_light: null scene");
    CU_CHECK(cudaSetDevice(s->device));
    int rc = build_env(s, s->own_stream);
    if (rc) return rc;
    if (total) *total = s->env_total;
    if (!s->env.row_cdf) return 0;
    const size_t H = (size_t)s->env.h, n = (size_t)s->env.w * s->env.h;
    cudaStream_t st = s->own_stream;
    if (row_cdf) CU_CHECK(cudaMemcpyAsync(row_cdf, s->env.row_cdf, sizeof(float) * H, cudaMemcpyDeviceToHost, st));
    if (col_cdf) CU_CHECK(cudaMemcpyAsync(col_cdf, s->env.col_cdf, sizeof(float) * n, cudaMemcpyDeviceToHost, st));
    if (texel_pdf) CU_CHECK(cudaMemcpyAsync(texel_pdf, s->env.texel_pdf, sizeof(float) * n, cudaMemcpyDeviceToHost, st));
    CU_CHECK(cudaStreamSynchronize(st));
    return 1;
}

int ezrt_occluded_rays(ezrt_scene* s, int n, const float* origins, const float* dirs, const float* tmax, int traverse, int32_t* out_lit) {
    if (!s || n < 0 || !origins || !dirs || !tmax || !out_lit) return ezrt_set_error(EZRT_ERR_INVALID, "occluded_rays: null argument");
    if (traverse < EZRT_TRAVERSE_ACCEL || traverse > EZRT_TRAVERSE_PRUNED) return ezrt_set_error(EZRT_ERR_INVALID, "occluded_rays: bad traverse");
    if (n == 0) return EZRT_OK;
    CU_CHECK(cudaSetDevice(s->device));
    // the render's shadow pass over a shadow queue of n rays (only ray_o, ray_d, nrm.w and lit are read / written)
    const size_t N = (size_t)n;
    std::vector<float4> ho(N), hd(N), hn(N);
    bool bounded = false;
    for (size_t i = 0; i < N; i++) {
        ho[i] = make_float4(origins[3 * i], origins[3 * i + 1], origins[3 * i + 2], 0.0f);
        hd[i] = make_float4(dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2], 0.0f);
        hn[i] = make_float4(0.0f, 0.0f, 0.0f, tmax[i]);
        bounded = bounded || !(std::isinf(tmax[i]) && tmax[i] > 0.0f);
    }
    struct TmpBuffer : DeviceBuffer { ~TmpBuffer() { release(); } } qbuf, buf;
    ShadowQueue sq{};
    int rc = carve_shadow(qbuf, N, sq);
    if (rc) return rc;
    if ((rc = buf.ensure(sizeof(uint32_t) * (N + 8)))) return rc;
    uint32_t* d_defer = (uint32_t*)buf.p;
    uint32_t* d_cnt = d_defer + N;   // [0] n, [1] work, [2] deferred, [3] deferred work
    const bool prune = s->regular_tree && traverse != EZRT_TRAVERSE_REFERENCE;
    const bool accel = s->regular_tree && s->have_accel && traverse == EZRT_TRAVERSE_ACCEL;
    cudaStream_t st = s->own_stream;
    const uint32_t counters[4] = {(uint32_t)n, 0u, 0u, 0u};
    std::vector<unsigned char> lit(N);
    CU_CHECK(cudaMemcpyAsync(sq.ray_o, ho.data(), sizeof(float4) * N, cudaMemcpyHostToDevice, st));
    CU_CHECK(cudaMemcpyAsync(sq.ray_d, hd.data(), sizeof(float4) * N, cudaMemcpyHostToDevice, st));
    CU_CHECK(cudaMemcpyAsync(sq.nrm, hn.data(), sizeof(float4) * N, cudaMemcpyHostToDevice, st));
    CU_CHECK(cudaMemcpyAsync(d_cnt, counters, sizeof(counters), cudaMemcpyHostToDevice, st));
    if (accel) launch_shadow_accel(s->dev, sq, d_cnt, d_cnt + 1, nullptr, d_defer, d_cnt + 2, d_cnt + 3, (uint32_t)n, s->n_sms, nullptr, st, bounded);
    else launch_shadow(s->dev, prune, sq, d_cnt, d_cnt + 1, nullptr, nullptr, (uint32_t)n, s->n_sms, st, bounded);
    CU_CHECK(cudaGetLastError());
    CU_CHECK(cudaMemcpyAsync(lit.data(), sq.lit, N, cudaMemcpyDeviceToHost, st));
    CU_CHECK(cudaStreamSynchronize(st));
    for (size_t i = 0; i < N; i++) out_lit[i] = lit[i] ? 1 : 0;
    return EZRT_OK;
}

int ezrt_eval_brdf(int device, int which, int n, const float* V, const float* N, const float* L, const float* xi,
                   const float* materials, float* out) {
    if (n < 0 || !V || !N || !materials || !out || which < 0 || which > 3) return ezrt_set_error(EZRT_ERR_INVALID, "eval_brdf: bad argument");
    if (which != 3 && !L) return ezrt_set_error(EZRT_ERR_INVALID, "eval_brdf: L required");
    if (which == 3 && !xi) return ezrt_set_error(EZRT_ERR_INVALID, "eval_brdf: xi required");
    if (n == 0) return EZRT_OK;
    CU_CHECK(cudaSetDevice(device));
    DeviceBuffer buf;
    size_t f3 = sizeof(float) * 3 * (size_t)n;
    int rc = buf.ensure(f3 * 5 + sizeof(float) * 18 * (size_t)n + 256);
    if (rc) return rc;
    float* dV = (float*)buf.p;
    float* dN = dV + 3 * (size_t)n;
    float* dL = dN + 3 * (size_t)n;
    float* dXi = dL + 3 * (size_t)n;
    float* dOut = dXi + 3 * (size_t)n;
    float* dM = dOut + 3 * (size_t)n;
    cudaError_t e = cudaMemcpy(dV, V, f3, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dN, N, f3, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && L) e = cudaMemcpy(dL, L, f3, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && xi) e = cudaMemcpy(dXi, xi, f3, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dM, materials, sizeof(float) * 18 * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        launch_eval_brdf(which, n, dV, dN, L ? dL : nullptr, xi ? dXi : nullptr, dM, dOut, 0);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, dOut, f3, cudaMemcpyDeviceToHost);
    buf.release();
    if (e != cudaSuccess) return ezrt_set_error(EZRT_ERR_CUDA, "eval_brdf: %s", cudaGetErrorString(e));
    return EZRT_OK;
}

int ezrt_camera_rays(ezrt_scene* s, const ezrt_render_params* p, int n, const uint32_t* px, const uint32_t* py, const uint32_t* frame,
                     float* origins_out, float* dirs_out) {
    int rc = validate_params(s, p);
    if (rc) return rc;
    if (n < 0 || !px || !py || !frame || !origins_out || !dirs_out) return ezrt_set_error(EZRT_ERR_INVALID, "camera_rays: bad argument");
    if (n == 0) return EZRT_OK;
    CU_CHECK(cudaSetDevice(s->device));
    RenderDev rd{};
    rd.width = p->width; rd.height = p->height;
    memcpy(rd.eye, p->eye, sizeof(rd.eye));
    memcpy(rd.cam, p->camera_rotate, sizeof(rd.cam));
    LensDev lens_v;
    const LensDev* lens = thin_lens(p, &lens_v) ? &lens_v : nullptr;
    DeviceBuffer buf;
    const size_t u1 = sizeof(uint32_t) * (size_t)n, f3 = sizeof(float) * 3 * (size_t)n;
    if ((rc = buf.ensure(3 * u1 + 2 * f3 + 256))) return rc;
    uint32_t* dPx = (uint32_t*)buf.p;
    uint32_t* dPy = dPx + n;
    uint32_t* dFr = dPy + n;
    float* dO = (float*)(dFr + n);
    float* dD = dO + 3 * (size_t)n;
    cudaError_t e = cudaMemcpy(dPx, px, u1, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dPy, py, u1, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dFr, frame, u1, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        launch_camera_rays(rd, lens, n, dPx, dPy, dFr, dO, dD, 0);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(origins_out, dO, f3, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(dirs_out, dD, f3, cudaMemcpyDeviceToHost);
    buf.release();
    if (e != cudaSuccess) return ezrt_set_error(EZRT_ERR_CUDA, "camera_rays: %s", cudaGetErrorString(e));
    return EZRT_OK;
}

int ezrt_eval_bsdf(int device, int which, int n, const float* V, const float* N, const float* L, const float* xi, const int32_t* inside,
                   const float* materials, float* out) {
    if (n < 0 || !V || !N || !inside || !materials || !out || which < 0 || which > 2) return ezrt_set_error(EZRT_ERR_INVALID, "eval_bsdf: bad argument");
    if (which != 2 && !L) return ezrt_set_error(EZRT_ERR_INVALID, "eval_bsdf: L required");
    if (which == 2 && !xi) return ezrt_set_error(EZRT_ERR_INVALID, "eval_bsdf: xi required");
    if (n == 0) return EZRT_OK;
    CU_CHECK(cudaSetDevice(device));
    DeviceBuffer buf;
    const size_t f3 = sizeof(float) * 3 * (size_t)n;
    int rc = buf.ensure(f3 * 3 + sizeof(float) * (4 + 8 + 18) * (size_t)n + sizeof(int32_t) * (size_t)n + 256);
    if (rc) return rc;
    float* dV = (float*)buf.p;
    float* dN = dV + 3 * (size_t)n;
    float* dL = dN + 3 * (size_t)n;
    float* dXi = dL + 3 * (size_t)n;
    float* dOut = dXi + 4 * (size_t)n;
    float* dM = dOut + 8 * (size_t)n;
    int32_t* dIn = (int32_t*)(dM + 18 * (size_t)n);
    cudaError_t e = cudaMemcpy(dV, V, f3, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dN, N, f3, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && L) e = cudaMemcpy(dL, L, f3, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && xi) e = cudaMemcpy(dXi, xi, sizeof(float) * 4 * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dM, materials, sizeof(float) * 18 * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dIn, inside, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        launch_eval_bsdf(which, n, dV, dN, L ? dL : nullptr, xi ? dXi : nullptr, dIn, dM, dOut, 0);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, dOut, sizeof(float) * 8 * (size_t)n, cudaMemcpyDeviceToHost);
    buf.release();
    if (e != cudaSuccess) return ezrt_set_error(EZRT_ERR_CUDA, "eval_bsdf: %s", cudaGetErrorString(e));
    return EZRT_OK;
}

int ezrt_accel_build(int device, const float* tris, int n_triangles, int leaf_n, int where, int32_t* links_out, float* boxes_out,
                     int nodes_cap, uint32_t* order_out, double* ms) {
    if (!tris || n_triangles <= 0 || leaf_n < 1) return ezrt_set_error(EZRT_ERR_INVALID, "accel_build: bad argument");
    std::vector<EzrtAccelNode> an;
    std::vector<uint32_t> order;
    const auto t0 = std::chrono::steady_clock::now();
    int n_nodes = 0;
    if (where == 1) {
        n_nodes = ezrt_build_accel(tris, n_triangles, leaf_n, an, order);
    } else {
        int n_dev = 0;
        CU_CHECK(cudaGetDeviceCount(&n_dev));
        if (device < 0 || device >= n_dev) return ezrt_set_error(EZRT_ERR_CUDA, "accel_build: no CUDA device %d (have %d)", device, n_dev);
        CU_CHECK(cudaSetDevice(device));
        DeviceBuffer raw;
        int rc = raw.ensure((size_t)n_triangles * EZRT_TRIANGLE_FLOATS * sizeof(float));
        if (rc) return rc;
        if (cudaMemcpy(raw.p, tris, (size_t)n_triangles * EZRT_TRIANGLE_FLOATS * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
            raw.release();
            return ezrt_set_error(EZRT_ERR_CUDA, "accel_build: upload failed: %s", cudaGetErrorString(cudaGetLastError()));
        }
        n_nodes = ezrt_build_accel_device((const float*)raw.p, n_triangles, leaf_n, an, order, nullptr);
        raw.release();
    }
    if (n_nodes < 0) return n_nodes;
    if (ms) *ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if ((links_out || boxes_out) && nodes_cap < n_nodes) return ezrt_set_error(EZRT_ERR_INVALID, "accel_build: %d nodes, room for %d", n_nodes, nodes_cap);
    for (int i = 0; i < n_nodes; i++) {
        if (links_out) { links_out[4 * i] = an[i].left; links_out[4 * i + 1] = an[i].right; links_out[4 * i + 2] = an[i].n; links_out[4 * i + 3] = an[i].index; }
        if (boxes_out)
            for (int k = 0; k < 3; k++) { boxes_out[6 * i + k] = an[i].AA[k]; boxes_out[6 * i + 3 + k] = an[i].BB[k]; }
    }
    if (order_out) memcpy(order_out, order.data(), sizeof(uint32_t) * (size_t)n_triangles);
    return n_nodes;
}

int ezrt_eval_math(int device, int which, int n, const float* a, const float* b, float* out) {
    if (n < 0 || !a || !out || which < 0 || which > 7) return ezrt_set_error(EZRT_ERR_INVALID, "eval_math: bad argument");
    if (n == 0) return EZRT_OK;
    CU_CHECK(cudaSetDevice(device));
    DeviceBuffer buf;
    size_t fN = sizeof(float) * (size_t)n;
    int rc = buf.ensure(fN * 3 + 256);
    if (rc) return rc;
    float* dA = (float*)buf.p;
    float* dB = dA + n;
    float* dO = dB + n;
    cudaError_t e = cudaMemcpy(dA, a, fN, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && b) e = cudaMemcpy(dB, b, fN, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        launch_eval_math(which, n, dA, b ? dB : nullptr, dO, 0);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, dO, fN, cudaMemcpyDeviceToHost);
    buf.release();
    if (e != cudaSuccess) return ezrt_set_error(EZRT_ERR_CUDA, "eval_math: %s", cudaGetErrorString(e));
    return EZRT_OK;
}

}  // extern "C"
