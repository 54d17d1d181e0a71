// gather_bench.cu -- measured ceiling for the traversal kernels' access pattern (development tool, not product):
// every lane reads its own randomly chosen record (64 / 96 / 128 bytes, 32-byte pieces as pairs of 128-bit loads
// through L1 exactly as k_extend_* do) from a table that is L2-resident (16 MB) or not (1 GB).  The result -- GB/s of
// RECORD bytes delivered to the lanes -- is a ceiling for the extend kernels, next to the plain-copy HBM peak.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/_bin/gather_bench tools/gather_bench.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

__device__ __forceinline__ uint32_t mix(uint32_t s) {
    s = (s ^ 61u) ^ (s >> 16); s *= 9u; s ^= s >> 4; s *= 0x27d4eb2du; s ^= s >> 15;
    return s;
}
__device__ __forceinline__ void ldg256(const void* p, uint4& a, uint4& b) {
    const char* c = static_cast<const char*>(p);
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w) : "l"(c));
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w) : "l"(c + 16));
}
// NL = 32-byte pieces per record, DEP = the next record index depends on the loaded data (a traversal step)
template <int NL, bool DEP>
__global__ void __launch_bounds__(1024, 1) k_gather(const char* table, uint32_t n_rec, uint32_t rec_bytes, int iters, uint32_t* sink) {
    uint32_t s = mix(blockIdx.x * blockDim.x + threadIdx.x + 12345u);
    uint32_t acc = 0;
    for (int it = 0; it < iters; it++) {
        const char* p = table + (size_t)(s % n_rec) * rec_bytes;
        uint32_t x = 0;
#pragma unroll
        for (int l = 0; l < NL; l++) {
            uint4 a, b;
            ldg256(p + 32 * l, a, b);
            x ^= a.x ^ a.w ^ b.y ^ b.w;
        }
        acc ^= x;
        s = DEP ? mix(s ^ x) : mix(s);
    }
    if (acc == 0x12345678u) sink[0] = acc;
}
__device__ __forceinline__ void ldg128(const void* p, uint4& a) {
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w) : "l"(p));
}
// the same with NL 128-bit loads per record (records only 16-byte aligned)
template <int NL>
__global__ void __launch_bounds__(1024, 1) k_gather128(const char* table, uint32_t n_rec, uint32_t rec_bytes, int iters, uint32_t* sink) {
    uint32_t s = mix(blockIdx.x * blockDim.x + threadIdx.x + 12345u);
    uint32_t acc = 0;
    for (int it = 0; it < iters; it++) {
        const char* p = table + (size_t)(s % n_rec) * rec_bytes;
        uint32_t x = 0;
#pragma unroll
        for (int l = 0; l < NL; l++) {
            uint4 a;
            ldg128(p + 16 * l, a);
            x ^= a.x ^ a.w;
        }
        acc ^= x;
        s = mix(s ^ x);
    }
    if (acc == 0x12345678u) sink[0] = acc;
}
// shared-memory variant: a lane reads NL x 16 bytes of a random record of a 64 KB table held in shared memory
template <int NL>
__global__ void __launch_bounds__(1024, 1) k_gather_smem(int iters, uint32_t* sink) {
    extern __shared__ uint4 tab[];
    const int n16 = 64 * 1024 / 16;
    for (int i = threadIdx.x; i < n16; i += blockDim.x) tab[i] = make_uint4(i, i * 3, i * 5, i * 7);
    __syncthreads();
    const uint32_t n_rec = n16 / NL;
    uint32_t s = mix(blockIdx.x * blockDim.x + threadIdx.x + 777u), acc = 0;
    for (int it = 0; it < iters; it++) {
        const uint4* p = tab + (s % n_rec) * NL;
        uint32_t x = 0;
#pragma unroll
        for (int l = 0; l < NL; l++) { uint4 a = p[l]; x ^= a.x ^ a.w; }
        acc ^= x;
        s = mix(s ^ x);
    }
    if (acc == 0x12345678u) sink[0] = acc;
}

template <class F>
static float time_ms(F launch) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    launch();  // warm-up
    cudaDeviceSynchronize();
    float best = 1e30f;
    for (int r = 0; r < 5; r++) {
        cudaEventRecord(e0);
        launch();
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) best = ms;
    }
    return best;
}

int main() {
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    const int sms = prop.multiProcessorCount;
    uint32_t* sink;
    cudaMalloc(&sink, 4);
    const size_t sizes[2] = {(size_t)16 << 20, (size_t)1 << 30};
    const char* names[2] = {"l2_resident_16MB", "hbm_1GB"};
    const int iters = 512;
    printf("{\"gpu\": \"%s\", \"sms\": %d, \"block\": 1024, \"results\": [\n", prop.name, sms);
    bool first = true;
    for (int si = 0; si < 2; si++) {
        char* table;
        if (cudaMalloc(&table, sizes[si]) != cudaSuccess) continue;
        cudaMemset(table, 1, sizes[si]);
        for (int rec = 64; rec <= 128; rec += 32) {
            const uint32_t n_rec = (uint32_t)(sizes[si] / rec);
            for (int dep = 0; dep < 2; dep++) {
                auto launch = [&]() {
#define GB(NL) (dep ? k_gather<NL, true><<<sms, 1024>>>(table, n_rec, rec, iters, sink) : k_gather<NL, false><<<sms, 1024>>>(table, n_rec, rec, iters, sink))
                    if (rec == 64) GB(2); else if (rec == 96) GB(3); else GB(4);
#undef GB
                };
                const float ms = time_ms(launch);
                const double bytes = (double)sms * 1024 * iters * rec;
                printf("%s  {\"table\": \"%s\", \"record_bytes\": %d, \"dependent\": %d, \"ms\": %.4f, \"gbs\": %.1f, \"grecords_per_s\": %.2f}", first ? "" : ",\n",
                       names[si], rec, dep, ms, bytes / ms / 1e6, bytes / rec / ms / 1e6);
                first = false;
            }
        }
        cudaFree(table);
    }
    {   // 128-bit loads, record sizes 32..128 in steps of 16, tables of 2 / 6 / 16 / 48 MB
        const size_t tsz[4] = {(size_t)2 << 20, (size_t)6 << 20, (size_t)16 << 20, (size_t)48 << 20};
        for (int si = 0; si < 4; si++) {
            char* table;
            if (cudaMalloc(&table, tsz[si]) != cudaSuccess) continue;
            cudaMemset(table, 1, tsz[si]);
            for (int nl = 2; nl <= 8; nl++) {
                const int rec = nl * 16;
                const uint32_t n_rec = (uint32_t)(tsz[si] / rec);
                auto launch = [&]() {
                    switch (nl) {
                        case 2: k_gather128<2><<<sms, 1024>>>(table, n_rec, rec, iters, sink); break;
                        case 3: k_gather128<3><<<sms, 1024>>>(table, n_rec, rec, iters, sink); break;
                        case 4: k_gather128<4><<<sms, 1024>>>(table, n_rec, rec, iters, sink); break;
                        case 5: k_gather128<5><<<sms, 1024>>>(table, n_rec, rec, iters, sink); break;
                        case 6: k_gather128<6><<<sms, 1024>>>(table, n_rec, rec, iters, sink); break;
                        case 7: k_gather128<7><<<sms, 1024>>>(table, n_rec, rec, iters, sink); break;
                        default: k_gather128<8><<<sms, 1024>>>(table, n_rec, rec, iters, sink); break;
                    }
                };
                const float ms = time_ms(launch);
                const double bytes = (double)sms * 1024 * iters * rec;
                printf(",\n  {\"table\": \"global_%zuMB_ld128\", \"record_bytes\": %d, \"dependent\": 1, \"ms\": %.4f, \"gbs\": %.1f, \"grecords_per_s\": %.2f}", tsz[si] >> 20, rec, ms,
                       bytes / ms / 1e6, bytes / rec / ms / 1e6);
            }
            // 256-bit loads on the same tables (32-byte multiples)
            for (int rec = 32; rec <= 128; rec += 32) {
                const uint32_t n_rec = (uint32_t)(tsz[si] / rec);
                auto launch = [&]() {
                    if (rec == 32) k_gather<1, true><<<sms, 1024>>>(table, n_rec, rec, iters, sink);
                    else if (rec == 64) k_gather<2, true><<<sms, 1024>>>(table, n_rec, rec, iters, sink);
                    else if (rec == 96) k_gather<3, true><<<sms, 1024>>>(table, n_rec, rec, iters, sink);
                    else k_gather<4, true><<<sms, 1024>>>(table, n_rec, rec, iters, sink);
                };
                const float ms = time_ms(launch);
                const double bytes = (double)sms * 1024 * iters * rec;
                printf(",\n  {\"table\": \"global_%zuMB_ld256\", \"record_bytes\": %d, \"dependent\": 1, \"ms\": %.4f, \"gbs\": %.1f, \"grecords_per_s\": %.2f}", tsz[si] >> 20, rec, ms,
                       bytes / ms / 1e6, bytes / rec / ms / 1e6);
            }
            cudaFree(table);
        }
    }
    {   // the L2 cliff: 32-, 48- and 64-byte records (128-bit loads, dependent) from tables of 16 to 128 MB, around H100's
        // 50 MB L2 -- where the W8 triangle records of a 1 M-triangle scene lie (64 MB flat, 32 MB indexed + the vertices)
        const int tmb[6] = {16, 32, 48, 64, 96, 128};
        for (int si = 0; si < 6; si++) {
            const size_t bytes_t = (size_t)tmb[si] << 20;
            char* table;
            if (cudaMalloc(&table, bytes_t) != cudaSuccess) continue;
            cudaMemset(table, 1, bytes_t);
            for (int nl = 2; nl <= 4; nl++) {
                const int rec = nl * 16;
                const uint32_t n_rec = (uint32_t)(bytes_t / rec);
                auto launch = [&]() {
                    if (nl == 2) k_gather128<2><<<sms, 1024>>>(table, n_rec, rec, iters, sink);
                    else if (nl == 3) k_gather128<3><<<sms, 1024>>>(table, n_rec, rec, iters, sink);
                    else k_gather128<4><<<sms, 1024>>>(table, n_rec, rec, iters, sink);
                };
                const float ms = time_ms(launch);
                const double bytes = (double)sms * 1024 * iters * rec;
                printf(",\n  {\"table\": \"cliff_%dMB_ld128\", \"record_bytes\": %d, \"dependent\": 1, \"ms\": %.4f, \"gbs\": %.1f, \"grecords_per_s\": %.2f}", tmb[si], rec, ms,
                       bytes / ms / 1e6, bytes / rec / ms / 1e6);
            }
            cudaFree(table);
        }
    }
    for (int nl = 2; nl <= 8; nl *= 2) {
        auto launch = [&]() {
            if (nl == 2) { cudaFuncSetAttribute(k_gather_smem<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536); k_gather_smem<2><<<sms, 1024, 65536>>>(4096, sink); }
            else if (nl == 4) { cudaFuncSetAttribute(k_gather_smem<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536); k_gather_smem<4><<<sms, 1024, 65536>>>(4096, sink); }
            else { cudaFuncSetAttribute(k_gather_smem<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536); k_gather_smem<8><<<sms, 1024, 65536>>>(4096, sink); }
        };
        const float ms = time_ms(launch);
        const double bytes = (double)sms * 1024 * 4096 * nl * 16;
        printf(",\n  {\"table\": \"shared_64KB\", \"record_bytes\": %d, \"dependent\": 1, \"ms\": %.4f, \"gbs\": %.1f, \"grecords_per_s\": %.2f}", nl * 16, ms, bytes / ms / 1e6,
               bytes / (nl * 16) / ms / 1e6);
    }
    printf("\n]}\n");
    return 0;
}
