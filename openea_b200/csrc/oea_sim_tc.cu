// oea_sim_tc.cu — path (iii), K3 on the Hopper tensor cores: S = E1·E2ᵀ in 3×TF32 (wgmma.mma_async m64n128k8 .tf32, fp32
// accumulators in registers), stored (optionally as the CSLS matrix 2·S − r_i − c_j) for the streaming CSLS passes.  sm_90a.
//
// Reference maths: modules/finding/similarity.py:11-54 (`sim`: np.matmul for inner / normalised cosine) and :57-77 (CSLS).
// The FP32 FFMA tile kernel of oea_sim.cu is the default and the bit-level reference; this kernel is the opt-in fast path
// (OEA_SIM_TC=1) for the materialised evaluation and the dense GEMM-NT of the GNN layers.  3×TF32: every operand x is split
// as x = hi + lo with hi = tf32(x) and lo = x − hi; a·b ≈ lo_a·hi_b + hi_a·lo_b + hi_a·hi_b accumulated in fp32 — the
// dropped lo·lo term is 2⁻²² relative, below fp32 rounding, so values agree with the FFMA kernel to fp32 round-off
// (summation order differs).
//
// One CTA (two warpgroups, 256 threads) per 128 × 128 output tile, persistent over tiles, two CTAs per SM so that one CTA's
// loads and epilogue overlap the other's MMAs.  Per 16-wide K chunk:
//   load      every thread reads its share of the chunk's 128 E1 rows and 128 E2 rows (128-bit global loads) one chunk
//             ahead, while the previous chunk's MMAs run; splits hi / lo in registers and stores both into the K-major,
//             no-swizzle wgmma layout (8-row × 16-B core matrices: byte = (r/8)·512 + (k/4)·128 + (r%8)·16 + (k%4)·4);
//             two shared-memory buffers alternate between chunks;
//   mma       warpgroup g issues 2 k-steps × 3 wgmma (M = 64 rows 64g … 64g+63, N = 128, K = 8) from shared-memory
//             descriptors and keeps at most one chunk's group in flight (wgmma.wait_group 1) before the buffer it read is
//             refilled;
//   epilogue  the m64n128 fragment: thread (warp w, lane l) of warpgroup g holds rows 64g + 16(w%4) + l/4 (+8), columns
//             8j + 2(l%4) (+1) — a quad of lanes writes 32 contiguous bytes of a row, every sector fully used.
#include <stdlib.h>
#include "oea_rowmath.cuh"

namespace oea {

constexpr int TCM = 128, TCN = 128, TCK = 16;             // tile rows of E1, rows of E2, K chunk (fp32 elements)
constexpr int TC_THREADS = 256;                           // two warpgroups: rows 0-63 and 64-127 of the tile
constexpr int TC_A_BYTES = TCM * TCK * 4, TC_B_BYTES = TCN * TCK * 4;
constexpr int TC_STAGE_BYTES = 2 * TC_A_BYTES + 2 * TC_B_BYTES;     // A hi/lo, B hi/lo: 32 KB
constexpr int TC_SMEM_BYTES = 2 * TC_STAGE_BYTES;                    // two stages: 64 KB, two CTAs per SM
constexpr int TC_GROUP_BYTES = 8 * 16 * (TCK / 4);                   // one 8-row group of core matrices across the chunk

struct TcParams {
    const float* e1; const float* e2;
    const float* row_off; const float* col_off;
    float* out; long long ld_out;
    int n1, n2, pitch1, pitch2, kdim;
    int tiles_m, tiles_n;
};

#ifndef OEA_HOST_EMU
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// K-major, no-swizzle shared-memory matrix descriptor of wgmma: start address, leading byte offset (between the two 16-B
// K halves of one K = 8 step) and stride byte offset (between 8-row groups), all >> 4; base offset 0, layout type 0.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32);
}

// D[64 × 128] (+)= A[64 × 8] · B[128 × 8]ᵀ in TF32, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// round-to-nearest split on the magnitude: hi keeps tf32's 10 mantissa bits, lo = x − hi is exact (the MMA reads lo's
// top 11 bits).  Integer ops: cvt.rna.tf32 runs on the quarter-rate conversion pipe.
__device__ __forceinline__ void split_store(float4 v, char* hi, char* lo, int off) {
    float4 h, l;
    h.x = __uint_as_float((__float_as_uint(v.x) + 0x1000u) & 0xFFFFE000u); h.y = __uint_as_float((__float_as_uint(v.y) + 0x1000u) & 0xFFFFE000u);
    h.z = __uint_as_float((__float_as_uint(v.z) + 0x1000u) & 0xFFFFE000u); h.w = __uint_as_float((__float_as_uint(v.w) + 0x1000u) & 0xFFFFE000u);
    l.x = v.x - h.x; l.y = v.y - h.y; l.z = v.z - h.z; l.w = v.w - h.w;
    *reinterpret_cast<float4*>(hi + off) = h;
    *reinterpret_cast<float4*>(lo + off) = l;
}

// One operand's share of a [128 × 16] chunk: thread t covers rows (t % 8) + 8·(t / 32) + 64p and the 16-B column
// (t / 8) % 4, so the 8 threads of a shared-memory phase write 8 different rows of one core matrix (conflict-free) and a
// warp's loads use whole 32-B sectors.
struct ChunkRegs { float4 a[2], b[2]; };

__device__ __forceinline__ void load_chunk(const TcParams& P, int row0, int col0, int k0, int tid, ChunkRegs& c) {
    const int r_in = (tid & 7) + 8 * (tid >> 5), kc = (tid >> 3) & 3, k = k0 + 4 * kc;
#pragma unroll
    for (int p = 0; p < 2; ++p) {
        const int r = r_in + 64 * p;
        c.a[p] = c.b[p] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < P.kdim) {                                  // kdim % 4 == 0: a 16-B column is all in or all out
            if (row0 + r < P.n1) c.a[p] = __ldg(reinterpret_cast<const float4*>(P.e1 + (size_t)(row0 + r) * P.pitch1 + k));
            if (col0 + r < P.n2) c.b[p] = __ldg(reinterpret_cast<const float4*>(P.e2 + (size_t)(col0 + r) * P.pitch2 + k));
        }
    }
}

__device__ __forceinline__ void store_chunk(const ChunkRegs& c, char* stage, int tid) {
    const int r_in = (tid & 7) + 8 * (tid >> 5), kc = (tid >> 3) & 3;
#pragma unroll
    for (int p = 0; p < 2; ++p) {
        const int r = r_in + 64 * p;
        const int off = (r >> 3) * TC_GROUP_BYTES + kc * 128 + (r & 7) * 16;
        split_store(c.a[p], stage, stage + TC_A_BYTES, off);
        split_store(c.b[p], stage + 2 * TC_A_BYTES, stage + 2 * TC_A_BYTES + TC_B_BYTES, off);
    }
}

__global__ void __launch_bounds__(TC_THREADS, 2)
k_sim_store_tc(TcParams P) {
    extern __shared__ __align__(128) char smem[];
    const int tid = threadIdx.x, wg = tid >> 7, warp4 = (tid >> 5) & 3, lane = tid & 31;
    const int n_chunks = (P.kdim + TCK - 1) / TCK;
    const long long n_tiles = (long long)P.tiles_m * P.tiles_n;
    const bool use_csls = P.row_off != nullptr;

    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int row0 = (int)(tile / P.tiles_n) * TCM, col0 = (int)(tile % P.tiles_n) * TCN;
        float d[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) d[i] = 0.f;
        ChunkRegs regs;
        load_chunk(P, row0, col0, 0, tid, regs);
        for (int ch = 0; ch < n_chunks; ++ch) {
            char* stage = smem + (ch & 1) * TC_STAGE_BYTES;
            __syncthreads();                  // both warpgroups have retired the MMAs of chunk ch − 2, which read this stage
            store_chunk(regs, stage, tid);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy stores → visible to wgmma
            __syncthreads();
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
            const uint32_t ah = smem_u32(stage) + wg * (64 / 8) * TC_GROUP_BYTES, al = ah + TC_A_BYTES;
            const uint32_t bh = smem_u32(stage + 2 * TC_A_BYTES), bl = bh + TC_B_BYTES;
#pragma unroll
            for (int s = 0; s < TCK / 8; ++s) {                      // one K = 8 step = two 16-B core-matrix columns
                const uint32_t o = (uint32_t)s * 256u;
                wgmma_tf32(d, gmma_desc(al + o, 128, TC_GROUP_BYTES), gmma_desc(bh + o, 128, TC_GROUP_BYTES), (ch | s) != 0 ? 1u : 0u);
                wgmma_tf32(d, gmma_desc(ah + o, 128, TC_GROUP_BYTES), gmma_desc(bl + o, 128, TC_GROUP_BYTES), 1u);   // small terms first
                wgmma_tf32(d, gmma_desc(ah + o, 128, TC_GROUP_BYTES), gmma_desc(bh + o, 128, TC_GROUP_BYTES), 1u);
            }
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            if (ch + 1 < n_chunks) load_chunk(P, row0, col0, (ch + 1) * TCK, tid, regs);   // in flight behind the MMAs
            asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
        }
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");

        // ---- epilogue: straight from the accumulator fragment ----
        const int rbase = row0 + 64 * wg + 16 * warp4 + (lane >> 2);
        float roff[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = rbase + 8 * h;
            roff[h] = (use_csls && r < P.n1) ? __ldg(P.row_off + r) : 0.f;
        }
#pragma unroll
        for (int j = 0; j < TCN / 8; ++j) {
            const int c = col0 + 8 * j + 2 * (lane & 3);
            const float c0f = (use_csls && c < P.n2) ? __ldg(P.col_off + c) : 0.f;
            const float c1f = (use_csls && c + 1 < P.n2) ? __ldg(P.col_off + c + 1) : 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = rbase + 8 * h;
                float2 o2 = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
                if (use_csls) { o2.x = (2.f * o2.x - roff[h]) - c0f; o2.y = (2.f * o2.y - roff[h]) - c1f; }
                if (r < P.n1 && c < P.n2) {
                    float* orow = P.out + (size_t)r * P.ld_out;
                    if (c + 1 < P.ld_out) *reinterpret_cast<float2*>(orow + c) = o2;   // ld_out % 4 == 0, c even: 8-B aligned
                    else orow[c] = o2.x;
                }
            }
        }
    }
}
#endif  // OEA_HOST_EMU

}  // namespace oea

using namespace oea;

extern "C" int oea_sim_matrix_tc(const oea_sim_cfg* c, const float* e1, const float* e2, const float* row_off, const float* col_off,
                                 float* out, int64_t ld_out, void* stream) {
    if (!c || !e1 || !e2 || !out) return OEA_ERR_NULL;
    if (c->metric != OEA_METRIC_INNER) return OEA_ERR_KIND;           // inner product (cosine = inner of normalised rows)
    if (c->n1 < 1 || c->n2 < 1 || c->dim < 1) return OEA_ERR_SHAPE;
    if (c->pitch1 < c->dim || c->pitch2 < c->dim || (c->pitch1 & 3) || (c->pitch2 & 3) || c->pitch1 > 2048 || c->pitch2 > 2048) return OEA_ERR_DIM;
    if (!aligned16(e1) || !aligned16(e2) || !aligned16(out) || (ld_out & 3) != 0 || ld_out < c->n2) return OEA_ERR_ALIGN;
    if ((row_off == nullptr) != (col_off == nullptr)) return OEA_ERR_NULL;
#ifndef OEA_HOST_EMU
    TcParams P;
    P.e1 = e1; P.e2 = e2; P.row_off = row_off; P.col_off = col_off; P.out = out; P.ld_out = ld_out;
    P.n1 = c->n1; P.n2 = c->n2; P.pitch1 = c->pitch1; P.pitch2 = c->pitch2;
    P.kdim = c->pitch1 < c->pitch2 ? c->pitch1 : c->pitch2;          // padding columns are zero on both sides
    P.tiles_m = (c->n1 + TCM - 1) / TCM; P.tiles_n = (c->n2 + TCN - 1) / TCN;
    static bool attr_set = false;
    if (!attr_set) {
        OEA_CUDA_TRY(cudaFuncSetAttribute(k_sim_store_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES));
        attr_set = true;
    }
    const long long tiles = (long long)P.tiles_m * P.tiles_n;
    const long long cap = 2ll * sm_count_cached();
    const int grid = (int)(tiles < cap ? tiles : cap);
    k_sim_store_tc<<<grid, TC_THREADS, TC_SMEM_BYTES, (cudaStream_t)stream>>>(P);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
#else
    return OEA_ERR_KIND;
#endif
}
