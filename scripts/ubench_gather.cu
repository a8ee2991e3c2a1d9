// Micro-benchmarks that bound the triple scorer (K1) at the 15K / 100K shapes on sm_90a — the questions left open by
// DESIGN.md §4 "where the scorer's time goes":
//   1. rows/s of independent 400-B row gathers (4 lanes × 16 B … one warp per row, 128-bit loads) from a table that is
//      L2-resident (12 MB) or not (320 MB), as a function of the rows each warp has in flight (1, 2, 4, 8);
//   2. latency of ONE dependent chain per warp: index → row → index taken from that row (what a positive's
//      triple → candidate list → entity row → hash probe chain looks like), L2-resident and DRAM;
//   3. red.global.add.v4.f32 throughput into an L2-resident gradient table: distinct rows vs 64 hot rows (hubs);
//   4. cost of one cooperative grid barrier at one CTA per SM and at full occupancy;
//   5. the same independent gathers as 1-D bulk async copies (cp.async.bulk = TMA's linear mode, one elected lane per
//      row, completion on an mbarrier) into shared memory — does TMA staging beat 25 lanes × ld.global.v4 for 400-B rows?
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -rdc=false -o scripts/ubench_gather.bin scripts/ubench_gather.cu
// Run on the GPU box: scripts/ubench_gather.bin > gpurun_out/ubench_gather.txt
#include <cooperative_groups.h>
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

constexpr int PITCH = 100;            // floats per row (400 B)

__device__ __forceinline__ uint32_t pcg(uint32_t x) {
    x = x * 747796405u + 2891336453u;
    const uint32_t w = ((x >> ((x >> 28) + 4u)) ^ x) * 277803737u;
    return (w >> 22) ^ w;
}

// 1. independent gathers, INFLIGHT rows per warp issued before the first use
template <int INFLIGHT>
__global__ void __launch_bounds__(256) k_gather(const float* __restrict__ tab, uint32_t rows, int per_warp, float* out) {
    const int lane = threadIdx.x & 31, warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    float acc = 0.f;
    for (int it = 0; it < per_warp; it += INFLIGHT) {
        float4 v[INFLIGHT];
#pragma unroll
        for (int j = 0; j < INFLIGHT; ++j) {
            const uint32_t r = pcg(warp * 9781u + (it + j) * 31u) % rows;
            v[j] = lane < PITCH / 4 ? __ldg(reinterpret_cast<const float4*>(tab + (size_t)r * PITCH) + lane) : make_float4(0, 0, 0, 0);
        }
#pragma unroll
        for (int j = 0; j < INFLIGHT; ++j) acc += v[j].x + v[j].y + v[j].z + v[j].w;
    }
    if (acc == 1234.5f) out[0] = acc;
}

// 5. independent gathers through the bulk-copy engine: lane 0 of each warp arms its mbarrier with INFLIGHT × 400 B and
// issues INFLIGHT bulk copies; the warp waits on the barrier's phase and reads the rows from shared memory.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

template <int INFLIGHT>
__global__ void __launch_bounds__(256) k_gather_bulk(const float* __restrict__ tab, uint32_t rows, int per_warp, float* out) {
    __shared__ __align__(128) float stage[8][INFLIGHT][128];      // 512-B slots, one set per warp
    __shared__ __align__(8) unsigned long long bar[8];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t b = smem_u32(&bar[w]);
    if (lane == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(b), "r"(1));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    float acc = 0.f;
    uint32_t phase = 0;
    for (int it = 0; it < per_warp; it += INFLIGHT) {
        if (lane == 0) {
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(b), "r"(INFLIGHT * PITCH * 4) : "memory");
#pragma unroll
            for (int j = 0; j < INFLIGHT; ++j) {
                const uint32_t r = pcg(warp * 9781u + (it + j) * 31u) % rows;
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             :: "r"(smem_u32(&stage[w][j][0])), "l"(tab + (size_t)r * PITCH), "r"(PITCH * 4), "r"(b) : "memory");
            }
        }
        asm volatile("{\n .reg .pred p;\n WAIT_%=:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @!p bra WAIT_%=;\n}"
                     :: "r"(b), "r"(phase) : "memory");
        phase ^= 1u;
#pragma unroll
        for (int j = 0; j < INFLIGHT; ++j)
            if (lane < PITCH / 4) { const float4 v = reinterpret_cast<const float4*>(&stage[w][j][0])[lane]; acc += v.x + v.y + v.z + v.w; }
        __syncwarp();                                            // all lanes have read the slots before they are refilled
    }
    if (acc == 1234.5f) out[0] = acc;
}

// 2. one dependent chain per warp: the next row index is read out of the current row
__global__ void __launch_bounds__(256) k_chain(const float* __restrict__ tab, uint32_t rows, int hops, float* out) {
    const int lane = threadIdx.x & 31, warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    uint32_t r = pcg(warp * 7919u) % rows;
    float acc = 0.f;
    for (int h = 0; h < hops; ++h) {
        const float4 v = lane < PITCH / 4 ? __ldg(reinterpret_cast<const float4*>(tab + (size_t)r * PITCH) + lane) : make_float4(0, 0, 0, 0);
        acc += v.y;
        r = __shfl_sync(0xffffffffu, __float_as_uint(v.x), 0) % rows;      // column 0 holds a random next index
    }
    if (acc == 1234.5f) out[0] = acc;
}

// 3. vector reductions into a gradient table
__global__ void __launch_bounds__(256) k_red(float* __restrict__ grad, uint32_t rows, int per_warp, int hot) {
    const int lane = threadIdx.x & 31, warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    for (int it = 0; it < per_warp; ++it) {
        uint32_t r = pcg(warp * 9781u + it * 31u) % rows;
        if (hot) r %= 64u;
        if (lane < PITCH / 4) {
            float* p = grad + (size_t)r * PITCH + 4 * lane;
            asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};" :: "l"(p), "f"(1.f), "f"(1.f), "f"(1.f), "f"(1.f) : "memory");
        }
    }
}

// 4. grid barriers
__global__ void __launch_bounds__(256) k_gridsync(int n, float* out) {
    cooperative_groups::grid_group g = cooperative_groups::this_grid();
    float acc = 0.f;
    for (int i = 0; i < n; ++i) { acc += 1.f; g.sync(); }
    if (acc == 1234.5f) out[0] = acc;
}

template <typename F>
static float time_ms(F launch, int reps = 5) {
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    float best = 1e30f;
    for (int r = 0; r < reps; ++r) {
        CK(cudaEventRecord(e0)); launch(); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
        if (r && ms < best) best = ms;          // first repetition = warm-up
    }
    return best;
}

int main() {
    int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    float* out; CK(cudaMalloc(&out, 1024));
    const uint32_t row_counts[2] = {30000u, 800000u};        // 12 MB (L2-resident) and 320 MB
    for (uint32_t rows : row_counts) {
        std::vector<float> host((size_t)rows * PITCH);
        for (size_t r = 0; r < rows; ++r) {
            uint32_t nxt = (uint32_t)((r * 2654435761ull + 12345ull) % rows);
            for (int c = 0; c < PITCH; ++c) host[r * PITCH + c] = 0.001f * c;
            memcpy(&host[r * PITCH], &nxt, 4);               // column 0: bit pattern of the next row index
        }
        float* tab; CK(cudaMalloc(&tab, host.size() * 4));
        CK(cudaMemcpy(tab, host.data(), host.size() * 4, cudaMemcpyHostToDevice));
        const int grid = sms * 8, per_warp = 256;
        const double n_rows = (double)grid * 8 * per_warp;
        printf("== table of %u rows x 400 B (%.0f MB)\n", rows, rows * 400.0 / 1e6);
        float ms;
        ms = time_ms([&] { k_gather<1><<<grid, 256>>>(tab, rows, per_warp, out); });
        printf("gather, 1 row in flight per warp : %.3f ms  %.2f Grows/s  %.0f GB/s\n", ms, n_rows / ms * 1e-6, n_rows * 400 / ms * 1e-6);
        ms = time_ms([&] { k_gather<2><<<grid, 256>>>(tab, rows, per_warp, out); });
        printf("gather, 2 rows in flight per warp: %.3f ms  %.2f Grows/s  %.0f GB/s\n", ms, n_rows / ms * 1e-6, n_rows * 400 / ms * 1e-6);
        ms = time_ms([&] { k_gather<4><<<grid, 256>>>(tab, rows, per_warp, out); });
        printf("gather, 4 rows in flight per warp: %.3f ms  %.2f Grows/s  %.0f GB/s\n", ms, n_rows / ms * 1e-6, n_rows * 400 / ms * 1e-6);
        ms = time_ms([&] { k_gather<8><<<grid, 256>>>(tab, rows, per_warp, out); });
        printf("gather, 8 rows in flight per warp: %.3f ms  %.2f Grows/s  %.0f GB/s\n", ms, n_rows / ms * 1e-6, n_rows * 400 / ms * 1e-6);
        ms = time_ms([&] { k_gather_bulk<4><<<grid, 256>>>(tab, rows, per_warp, out); });
        printf("bulk-copy gather (cp.async.bulk + mbarrier), 4 rows in flight per warp: %.3f ms  %.2f Grows/s  %.0f GB/s\n", ms, n_rows / ms * 1e-6, n_rows * 400 / ms * 1e-6);
        ms = time_ms([&] { k_gather_bulk<8><<<grid, 256>>>(tab, rows, per_warp, out); });
        printf("bulk-copy gather (cp.async.bulk + mbarrier), 8 rows in flight per warp: %.3f ms  %.2f Grows/s  %.0f GB/s\n", ms, n_rows / ms * 1e-6, n_rows * 400 / ms * 1e-6);
        for (int g : {1, sms, sms * 8}) {
            const int hops = 2000;
            ms = time_ms([&] { k_chain<<<g, 256>>>(tab, rows, hops, out); });
            printf("dependent chain, %5d CTAs: %.1f ns per hop\n", g, ms * 1e6 / hops);
        }
        float* grad; CK(cudaMalloc(&grad, host.size() * 4)); CK(cudaMemset(grad, 0, host.size() * 4));
        for (int hot = 0; hot < 2; ++hot) {
            ms = time_ms([&] { k_red<<<grid, 256>>>(grad, rows, per_warp, hot); });
            printf("red.v4 row reductions, %s: %.3f ms  %.2f Grows/s  %.0f GB/s\n", hot ? "64 hot rows    " : "distinct rows  ", ms,
                   n_rows / ms * 1e-6, n_rows * 400 / ms * 1e-6);
        }
        CK(cudaFree(grad)); CK(cudaFree(tab));
    }
    for (int per_sm : {1, 8}) {
        int n = 200, grid = sms * per_sm;
        void* args[] = {&n, &out};
        float ms = time_ms([&] { CK(cudaLaunchCooperativeKernel((void*)k_gridsync, dim3(grid), dim3(256), args, 0, 0)); });
        printf("cooperative grid barrier, %d CTA(s) per SM: %.2f us per barrier\n", per_sm, ms * 1e3 / n);
    }
    return 0;
}
