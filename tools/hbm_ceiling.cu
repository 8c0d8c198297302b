// hbm_ceiling.cu -- what this card's HBM delivers to a pure read stream and to a read+write copy, as a function of the bytes in flight per SM.
//
// Standalone (CUDA runtime only, not part of libppq_b200); built and driven by tools/hbm_ceiling.py.  Prints one JSON object per
// configuration on stdout.  Every kernel streams one of several rotating buffers that together exceed the L2 many times over, so no
// launch finds its input in L2.
//   read_ldg   min/max reduction, LDG.128 (ld.global.nc.L1::no_allocate), U loads in flight per thread, warp-contiguous segments
//   read_bulk  min/max reduction fed by a producer warp that issues 1-D cp.async.bulk global->shared copies into a ring of stages
//              (full/empty mbarriers); 8 consumer warps reduce from shared memory
//   copy_ldg   y = x with LDG.128 / STG.128, U loads in flight per thread (8 bytes of traffic per element)
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>
#include <algorithm>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

__device__ __forceinline__ float4 ld_stream4(const float4 *p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
struct MM {
    float lo, hi;
    __device__ MM() : lo(INFINITY), hi(-INFINITY) {}
    __device__ void add(float4 v) { lo = fminf(lo, fminf(fminf(v.x, v.y), fminf(v.z, v.w))); hi = fmaxf(hi, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w))); }
    __device__ void store(float *out) {
        for (int o = 16; o > 0; o >>= 1) { lo = fminf(lo, __shfl_xor_sync(~0u, lo, o)); hi = fmaxf(hi, __shfl_xor_sync(~0u, hi, o)); }
        if ((threadIdx.x & 31) == 0) { out[0] = lo; out[1] = hi; }     // racy on purpose: only keeps the reduction alive
    }
};

template <int U>
__global__ void read_ldg(const float4 *__restrict__ x, int64_t n4, float *out) {
    MM mm;
    const int64_t lane = threadIdx.x & 31, warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t base = warp * 32 * U; base < n4; base += warps * 32 * U) {
        float4 v[U];
#pragma unroll
        for (int j = 0; j < U; j++) if (base + j * 32 + lane < n4) v[j] = ld_stream4(x + base + j * 32 + lane);
#pragma unroll
        for (int j = 0; j < U; j++) if (base + j * 32 + lane < n4) mm.add(v[j]);
    }
    mm.store(out);
}

template <int U>
__global__ void copy_ldg(const float4 *__restrict__ x, float4 *__restrict__ y, int64_t n4) {
    const int64_t lane = threadIdx.x & 31, warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t base = warp * 32 * U; base < n4; base += warps * 32 * U) {
        float4 v[U];
#pragma unroll
        for (int j = 0; j < U; j++) if (base + j * 32 + lane < n4) v[j] = ld_stream4(x + base + j * 32 + lane);
#pragma unroll
        for (int j = 0; j < U; j++) if (base + j * 32 + lane < n4) y[base + j * 32 + lane] = v[j];
    }
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile("{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D_%=;\nbra W_%=;\nD_%=:\n}\n"
                 ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

constexpr int kBulkConsumers = 256;
// tile_bytes a multiple of 16; dynamic shared memory = stages x tile_bytes, then 2 x stages mbarriers
__global__ void __launch_bounds__(kBulkConsumers + 32) read_bulk(const float4 *__restrict__ x, int64_t n4, int stages, int tile_bytes, float *out) {
    extern __shared__ __align__(128) unsigned char smem[];
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + (size_t)stages * tile_bytes), *empty = full + stages;
    const int tv = tile_bytes / 16;
    const int64_t tiles = (n4 + tv - 1) / tv;
    const int64_t mine = blockIdx.x < tiles ? (tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; s++) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(full + s)));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(empty + s)), "r"(kBulkConsumers / 32));
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x >= kBulkConsumers) {
        if (threadIdx.x == kBulkConsumers) {
            for (int64_t k = 0; k < mine; k++) {
                const int s = (int)(k % stages);
                if (k >= stages) mbar_wait(empty + s, (uint32_t)(((k / stages) - 1) & 1));
                const int64_t t = blockIdx.x + k * gridDim.x;
                const int64_t v = n4 - t * tv;
                const uint32_t bytes = (uint32_t)((v < tv ? v : tv) * 16);
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(full + s)), "r"(bytes) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(smem_u32(smem + (size_t)s * tile_bytes)), "l"(x + t * tv), "r"(bytes), "r"(smem_u32(full + s)) : "memory");
            }
        }
        return;
    }
    MM mm;
    for (int64_t k = 0; k < mine; k++) {
        const int s = (int)(k % stages);
        mbar_wait(full + s, (uint32_t)((k / stages) & 1));
        const int64_t t = blockIdx.x + k * gridDim.x;
        const int64_t v = n4 - t * tv;
        const int nv = (int)(v < tv ? v : tv);
        const float4 *tile = reinterpret_cast<const float4 *>(smem + (size_t)s * tile_bytes);
        for (int i = threadIdx.x; i < nv; i += kBulkConsumers) mm.add(tile[i]);
        __syncwarp();
        if ((threadIdx.x & 31) == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(empty + s)) : "memory");
    }
    mm.store(out);
}

int main(int argc, char **argv) {
    const size_t buf_bytes = (argc > 1 ? strtoull(argv[1], nullptr, 10) : 384ull) << 20;    // MiB per buffer
    const int nbuf = argc > 2 ? atoi(argv[2]) : 4;
    const int reps = argc > 3 ? atoi(argv[3]) : 40;
    int dev = 0, sms = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, dev));
    const int64_t n4 = (int64_t)(buf_bytes / 16);
    std::vector<float4 *> bufs(nbuf + 1);
    for (auto &b : bufs) { CK(cudaMalloc(&b, buf_bytes)); CK(cudaMemset(b, 0, buf_bytes)); }
    float *out;
    CK(cudaMalloc(&out, 1 << 20));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    printf("{\"device\": \"%s\", \"sms\": %d, \"l2_mb\": %.1f, \"buffers\": %d, \"buffer_mib\": %zu}\n", prop.name, sms,
           prop.l2CacheSize / 1048576.0, nbuf, buf_bytes >> 20);

    // Time `reps` launches rotating over the buffers (after one warm-up round); the best of three such windows.
    auto time_it = [&](auto launch, double bytes_per_launch) {
        for (int i = 0; i < nbuf; i++) launch(i);
        CK(cudaDeviceSynchronize());
        double best = 0;
        for (int w = 0; w < 3; w++) {
            CK(cudaEventRecord(e0));
            for (int i = 0; i < reps; i++) launch(i % nbuf);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            CK(cudaGetLastError());
            float ms;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            best = std::max(best, bytes_per_launch * reps / (ms * 1e-3) / 1e9);
        }
        return best;
    };
    auto report = [&](const char *kind, const char *how, int threads, int resident, double depth_bytes, double gbs) {
        printf("{\"kind\": \"%s\", \"config\": \"%s\", \"threads\": %d, \"ctas_per_sm\": %d, \"depth_kb_per_sm\": %.0f, \"gbs\": %.1f}\n",
               kind, how, threads, resident, depth_bytes / 1024.0, gbs);
        fflush(stdout);
    };

    // ---- LDG.128 read stream: bytes in flight per SM = resident threads x U x 16
    auto ldg = [&](auto kern, int U, int threads) {
        int resident = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kern, threads, 0));
        const int grid = sms * resident;
        const double gbs = time_it([&](int i) { kern<<<grid, threads>>>(bufs[i], n4, out); }, (double)buf_bytes);
        char how[64]; snprintf(how, sizeof how, "U=%d", U);
        report("read_ldg", how, threads, resident, (double)resident * threads * U * 16, gbs);
    };
    ldg(read_ldg<1>, 1, 1024);
    ldg(read_ldg<2>, 2, 1024);
    ldg(read_ldg<4>, 4, 1024);
    ldg(read_ldg<4>, 4, 512);
    ldg(read_ldg<8>, 8, 512);
    ldg(read_ldg<8>, 8, 256);
    ldg(read_ldg<16>, 16, 256);

    // ---- cp.async.bulk ring: bytes in flight per SM = resident CTAs x stages x tile
    CK(cudaFuncSetAttribute(read_bulk, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    const int cfg[][3] = {{8192, 2, 2}, {8192, 4, 2}, {16384, 4, 2}, {16384, 4, 3}, {16384, 8, 2}, {32768, 4, 2}, {16384, 6, 2}};
    for (auto &c : cfg) {
        const int tile = c[0], stages = c[1], want = c[2];
        const int smem = stages * tile + 2 * stages * 8;
        int resident = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, read_bulk, kBulkConsumers + 32, smem));
        resident = std::min(resident, want);
        const int grid = sms * resident;
        const double gbs = time_it([&](int i) { read_bulk<<<grid, kBulkConsumers + 32, smem>>>(bufs[i], n4, stages, tile, out); }, (double)buf_bytes);
        char how[64]; snprintf(how, sizeof how, "tile=%dKB stages=%d", tile / 1024, stages);
        report("read_bulk", how, kBulkConsumers + 32, resident, (double)resident * stages * tile, gbs);
    }

    // ---- read+write copy (8 bytes of traffic per element), destination rotates too
    auto cp = [&](auto kern, int U, int threads) {
        int resident = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kern, threads, 0));
        const int grid = sms * resident;
        const double gbs = time_it([&](int i) { kern<<<grid, threads>>>(bufs[i], bufs[(i + 1) % (nbuf + 1)], n4); }, 2.0 * buf_bytes);
        char how[64]; snprintf(how, sizeof how, "U=%d", U);
        report("copy_ldg", how, threads, resident, (double)resident * threads * U * 16, gbs);
    };
    cp(copy_ldg<2>, 2, 1024);
    cp(copy_ldg<4>, 4, 512);
    cp(copy_ldg<8>, 8, 256);
    for (auto b : bufs) CK(cudaFree(b));
    CK(cudaFree(out));
    return 0;
}
