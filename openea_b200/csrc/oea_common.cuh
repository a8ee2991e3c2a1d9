// oea_common.cuh — device helpers shared by the liboea kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/oea.h"

#define OEA_WARP 32
#define OEA_FULL 0xffffffffu

#define OEA_CUDA_TRY(expr)                                   \
    do {                                                     \
        cudaError_t _e = (expr);                             \
        if (_e != cudaSuccess) return -(int)_e;              \
    } while (0)

// OEA_LAUNCH(kernel, grid, block, dynamic smem bytes, stream, args…): `kernel<<<grid, block, smem, stream>>>(args…)`,
// or — under tests/emu — the same kernel function run block by block on the CPU warp emulator (whole grid: not every
// kernel is grid-stride).  A template-id with commas must be bound to a local `auto kernel = …` first.
#ifdef OEA_HOST_EMU
#define OEA_LAUNCH(KERNEL, GRID, BLOCK, SMEM, STREAM, ...) emu::launch(dim3(GRID), dim3(BLOCK), [&] { KERNEL(__VA_ARGS__); })
#else
#define OEA_LAUNCH(KERNEL, GRID, BLOCK, SMEM, STREAM, ...) KERNEL<<<(GRID), (BLOCK), (SMEM), (STREAM)>>>(__VA_ARGS__)
#endif

// OEA_LAUNCH of a grid-stride kernel (one that covers its work whatever the grid).  Under tests/emu it runs on at most
// two blocks, which keeps the emulated thread count small.
#ifdef OEA_HOST_EMU
#define OEA_LAUNCH_STRIDED(KERNEL, GRID, BLOCK, SMEM, STREAM, ...) \
    OEA_LAUNCH(KERNEL, ((GRID) < 2 ? (GRID) : 2), BLOCK, SMEM, STREAM, __VA_ARGS__)
#else
#define OEA_LAUNCH_STRIDED OEA_LAUNCH
#endif

// Cooperative launch (the kernel uses cooperative_groups::this_grid().sync()); the arguments must be lvalues of exactly
// the kernel's parameter types.  Under tests/emu the grid is ONE block (every kernel launched this way walks its work
// with grid-stride loops) and the grid barrier is that block's barrier.
#ifdef OEA_HOST_EMU
#define OEA_LAUNCH_COOPERATIVE(KERNEL, GRID, BLOCK, STREAM, ...) \
    (emu::launch(dim3(1), dim3(BLOCK), [&] { KERNEL(__VA_ARGS__); }), cudaSuccess)
#else
template <typename Kernel, typename... Args>
static inline cudaError_t oea_launch_cooperative(Kernel kernel, int grid, int block, cudaStream_t stream, Args&... args) {
    void* argv[] = {(void*)&args...};
    return cudaLaunchCooperativeKernel((void*)kernel, dim3(grid), dim3(block), argv, 0, stream);
}
#define OEA_LAUNCH_COOPERATIVE(KERNEL, GRID, BLOCK, STREAM, ...) oea_launch_cooperative(KERNEL, GRID, BLOCK, STREAM, __VA_ARGS__)
#endif

// The dynamically sized shared-memory array of a kernel (under tests/emu: a static one of the largest size used).
#ifdef OEA_HOST_EMU
#define OEA_DYNAMIC_SMEM(NAME) static float NAME[57344]
#define OEA_DYNAMIC_SMEM_ALIGNED16(NAME) alignas(16) static float NAME[57344]
#else
#define OEA_DYNAMIC_SMEM(NAME) extern __shared__ float NAME[]
#define OEA_DYNAMIC_SMEM_ALIGNED16(NAME) extern __shared__ __align__(16) float NAME[]
#endif

#ifdef OEA_HOST_EMU   // tests/emu: the kernels run on the CPU's warp emulator; there is no launch to check
#define OEA_LAUNCH_CHECK() do { } while (0)
#else
#define OEA_LAUNCH_CHECK()                                   \
    do {                                                     \
        cudaError_t _e = cudaPeekAtLastError();              \
        if (_e != cudaSuccess) { cudaGetLastError(); return -(int)_e; } \
    } while (0)
#endif

namespace oea {

__host__ __device__ __forceinline__ bool aligned16(const void* p) {
    return (reinterpret_cast<uintptr_t>(p) & 15u) == 0;
}

// ---- fp32 pair arithmetic ----------------------------------------------------------------------
// Two independent IEEE fp32 lanes (fma.rn / add.rn / mul.rn each); Hopper has no packed fp32x2 instructions, so these are
// two scalar operations.
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 lo2(float4 a) { return make_float2(a.x, a.y); }
__device__ __forceinline__ float2 hi2(float4 a) { return make_float2(a.z, a.w); }
__device__ __forceinline__ float4 cat4(float2 lo, float2 hi) { return make_float4(lo.x, lo.y, hi.x, hi.y); }

// ---- float4 arithmetic -------------------------------------------------------------------------
__device__ __forceinline__ float4 f4(float a) { return make_float4(a, a, a, a); }
__device__ __forceinline__ float4 operator+(float4 a, float4 b) { return cat4(add2(lo2(a), lo2(b)), add2(hi2(a), hi2(b))); }
// a − b as fma(b, −1, a): one rounding, identical to the subtraction
__device__ __forceinline__ float4 operator-(float4 a, float4 b) { const float2 m = make_float2(-1.f, -1.f); return cat4(fma2(lo2(b), m, lo2(a)), fma2(hi2(b), m, hi2(a))); }
__device__ __forceinline__ float4 operator*(float4 a, float s) { const float2 ss = make_float2(s, s); return cat4(mul2(lo2(a), ss), mul2(hi2(a), ss)); }
__device__ __forceinline__ float4 neg(float4 a) { return make_float4(-a.x, -a.y, -a.z, -a.w); }
__device__ __forceinline__ float dot4(float4 a, float4 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w))); }
__device__ __forceinline__ float4 fma4(float4 a, float s, float4 c) { const float2 ss = make_float2(s, s); return cat4(fma2(lo2(a), ss, lo2(c)), fma2(hi2(a), ss, hi2(c))); }
// acc.x + acc.y accumulates <a, b> over calls: two independent fma chains, summed by the caller at the end
__device__ __forceinline__ void dot4_acc2(float2& acc, float4 a, float4 b) { acc = fma2(lo2(a), lo2(b), acc); acc = fma2(hi2(a), hi2(b), acc); }
__device__ __forceinline__ float sgn(float x) { return (float)(x > 0.f) - (float)(x < 0.f); }  // TF sign(0) = 0
__device__ __forceinline__ float4 sgn4(float4 a) { return make_float4(sgn(a.x), sgn(a.y), sgn(a.z), sgn(a.w)); }
__device__ __forceinline__ float abs_sum4(float4 a) { return fabsf(a.x) + fabsf(a.y) + fabsf(a.z) + fabsf(a.w); }

// ---- memory ------------------------------------------------------------------------------------
__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// 128-bit vector reduction to global memory (sm_90+: red.global.add.v4.f32), no return value.
__device__ __forceinline__ void red_add4(float* p, float4 v) {
#ifdef OEA_HOST_EMU
    atomicAdd(p, v.x); atomicAdd(p + 1, v.y); atomicAdd(p + 2, v.z); atomicAdd(p + 3, v.w);   // warps may run concurrently
#else
    asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};"
                 :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
#endif
}

// L2 prefetch of the 128-B lines a row of `bytes` bytes starting at p touches (p is 16-B aligned)
#ifdef OEA_HOST_EMU
__device__ __forceinline__ void prefetch_l2(const void*) {}
#else
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" :: "l"(p)); }
#endif
__device__ __forceinline__ void prefetch_row_l2(const float* row, int pitch_floats) {
    const char* b = reinterpret_cast<const char*>(row);
    const int bytes = pitch_floats * 4;
    for (int o = 0; o < bytes; o += 128) prefetch_l2(b + o);
}

// ---- warp reductions ---------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(OEA_FULL, v, o);
    return v;
}
__device__ __forceinline__ void warp_sum2(float& a, float& b) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(OEA_FULL, a, o);
        b += __shfl_xor_sync(OEA_FULL, b, o);
    }
}
__device__ __forceinline__ void warp_sum3(float& a, float& b, float& c) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(OEA_FULL, a, o);
        b += __shfl_xor_sync(OEA_FULL, b, o);
        c += __shfl_xor_sync(OEA_FULL, c, o);
    }
}

// ---- hashing / counter RNG ---------------------------------------------------------------------
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {  // splitmix64 finaliser
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ uint32_t mix32(uint32_t x) {  // lowbias32
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}
// Unbiased-enough bounded draw: high 32 bits of a 64-bit hash, multiply-shift into [0, n).
__host__ __device__ __forceinline__ uint32_t bounded(uint64_t r, uint32_t n) {
    return (uint32_t)(((r >> 32) * (uint64_t)n) >> 32);
}

// Pseudo-random permutation of [0, n) by a 4-round balanced Feistel network + cycle walking.
// Replaces random.shuffle(triples_list) of models/basic_model.py:234-235: a bijection per epoch key.
__host__ __device__ __forceinline__ uint32_t feistel_perm(uint32_t i, uint32_t n, uint64_t key) {
    if (n <= 1) return 0;
    uint32_t bits = 32 - (uint32_t)
#ifdef __CUDA_ARCH__
        __clz(n - 1);
#else
        __builtin_clz(n - 1);
#endif
    uint32_t hb = (bits + 1) >> 1;
    if (hb == 0) hb = 1;
    const uint32_t hmask = (1u << hb) - 1u;
    uint32_t x = i;
    do {
        uint32_t l = x >> hb, r = x & hmask;
#pragma unroll
        for (int round = 0; round < 4; ++round) {
            uint32_t f = mix32(r ^ (uint32_t)(key >> (16 * round)) ^ (0x9E3779B9u * (round + 1))) & hmask;
            uint32_t nl = r;
            r = l ^ f;
            l = nl;
        }
        x = (l << hb) | r;
    } while (x >= n);
    return x;
}

// 32-bit counter RNG for the sampler: one PCG-style output permutation per draw (≈6 integer instructions).
__host__ __device__ __forceinline__ uint32_t pcg32(uint32_t x) {
    x = x * 747796405u + 2891336453u;
    const uint32_t w = ((x >> ((x >> 28) + 4u)) ^ x) * 277803737u;
    return (w >> 22) ^ w;
}
// uniform integer in [0, n) from 32 random bits (multiply-high)
__device__ __forceinline__ uint32_t bounded32(uint32_t r, uint32_t n) { return __umulhi(r, n); }
// slot hash of a packed 64-bit triple key
__host__ __device__ __forceinline__ uint32_t key_hash(uint64_t key) {
    return pcg32((uint32_t)key ^ pcg32((uint32_t)(key >> 32) + 0x9E3779B9u));
}

// ---- triple membership set ---------------------------------------------------------------------
__host__ __device__ __forceinline__ uint64_t triple_key(uint32_t h, uint32_t r, uint32_t t, uint32_t ent_bits, uint32_t rel_bits) {
    return ((uint64_t)h << (ent_bits + rel_bits)) | ((uint64_t)r << ent_bits) | (uint64_t)t;
}
// Blocked Bloom filter in front of the slots: a key sets four bits of ONE 64-bit word.  The word comes from a hash
// independent of key_hash (high and low halves swap roles), so a key's slot and its filter word are uncorrelated; the
// four bit positions are four 6-bit fields of one further mix of that hash.  engine.tripleset_filter restates both in
// torch.  At ≥ 16 bits per key the filter rejects ≈ 99 % of absent keys with one load from a table 8× smaller than the
// slots (2 MB at the 100K shape), which stays in L2 where the slots do not.
__host__ __device__ __forceinline__ uint32_t tset_filter_hash(uint64_t key) {
    return pcg32((uint32_t)(key >> 32) ^ pcg32((uint32_t)key ^ 0x2545F491u));
}
__host__ __device__ __forceinline__ uint64_t tset_filter_bits(uint32_t fh) {
    const uint32_t b = pcg32(fh ^ 0x68E31DA4u);
    return (1ull << (b & 63u)) | (1ull << ((b >> 6) & 63u)) | (1ull << ((b >> 12) & 63u)) | (1ull << ((b >> 18) & 63u));
}
__device__ __forceinline__ bool tset_contains(const oea_tripleset& s, uint64_t key) {
    if (s.filter != nullptr) {
        const uint32_t fh = tset_filter_hash(key);
        const uint64_t bits = tset_filter_bits(fh);
        if ((__ldg(s.filter + (fh & (s.filter_words - 1u))) & bits) != bits) return false;
    }
    const uint32_t mask = s.capacity - 1u;
    uint32_t slot = key_hash(key) & mask;
    while (true) {
        uint64_t v = __ldg(s.slots + slot);
        if (v == key) return true;
        if (v == 0xFFFFFFFFFFFFFFFFull) return false;
        slot = (slot + 1u) & mask;
    }
}

// softplus(x) = log(1 + e^x), overflow-safe (losses.py:70-71 use the naive form; identical in range)
__device__ __forceinline__ float softplus(float x) { return fmaxf(x, 0.f) + log1pf(__expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + __expf(-x)); }

}  // namespace oea
