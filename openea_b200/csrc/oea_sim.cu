// oea_sim.cu — path (iii): all-pairs similarity, CSLS, per-row top-k, rank-of-gold (K3).  sm_90a.
//
// Restates (no code shared):
//   modules/finding/similarity.py:11-83   sim(): inner / cosine / euclidean / manhattan, csls_sim()
//   modules/finding/alignment.py:146-168  calculate_rank(): argmax + rank of the gold column
//   modules/bootstrapping/alignment_finder.py:54-76  threshold filter ∧ per-row top-k
//   modules/train/batch.py:157-165        find_neighbours(): per-row k largest (large k)
//
// The n1×n2 matrix is never materialised for top-k / rank: a 128×128 FP32 register-tiled kernel
// (FP32 FFMA so that alignment indices match float32 BLAS; manhattan is not a contraction) walks the
// column tiles of one row block and folds each finished tile into a per-row top-k list (smem) or a
// per-thread argmax + rank counter (registers).
#include <float.h>
#include <stdlib.h>
#include "oea_common.cuh"

namespace oea {

enum { EPI_TOPK = 0, EPI_RANK = 1, EPI_STORE = 2 };

constexpr int TM = 128, TN = 128, BK = 16;
constexpr int SIM_THREADS = 256;
constexpr int STAGES = 3;          // cp.async pipeline depth of the operand tiles

#ifdef OEA_HOST_EMU   // tests/emu: the copy is synchronous, groups are empty
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) { memcpy(smem_dst, gmem_src, 16); }
__device__ __forceinline__ void cp_async_commit() {}
template <int N>
__device__ __forceinline__ void cp_async_wait() {}
#else
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N)); }
#endif
constexpr int KMAX = 32;  // per-row top-k list lives in one warp's lanes
constexpr int TS_LD = TN + 4;  // tile staging row stride: 16-B aligned rows, conflict-free 128-bit stores

// similarity value from the accumulated contraction (similarity.py:36-51)
template <int METRIC>
__device__ __forceinline__ float sim_value(float acc) {
    if (METRIC == OEA_METRIC_INNER) return acc;
    if (METRIC == OEA_METRIC_L1) return 1.f - acc;       // 1 − cityblock
    return 1.f - sqrtf(fmaxf(acc, 0.f));                 // 1 − euclidean
}
template <int METRIC>
__device__ __forceinline__ float sim_accum(float a, float b, float acc) {
    if (METRIC == OEA_METRIC_INNER) return fmaf(a, b, acc);
    if (METRIC == OEA_METRIC_L1) return acc + fabsf(a - b);
    const float dlt = a - b;
    return fmaf(dlt, dlt, acc);
}
// CSLS: 2·S − r_i − c_j (similarity.py:73-77)
__device__ __forceinline__ float csls_value(float s, float r, float c) { return (2.f * s - r) - c; }

struct SimParams {
    const float* e1; const float* e2;
    const float* e1t; const float* e2t;    // k-major copies [kpad, ldt] (zero padded): tiles stream in with 16-B cp.async
    long long ld1t, ld2t;
    int n1, n2, pitch1, pitch2, kdim;      // kdim = min(pitch1, pitch2) rounded: contraction length
    const float* row_off; const float* col_off;  // CSLS r_i / c_j or nullptr
    int col_tiles_per_split;
    // top-k
    int k, kcap; float* part_val; int* part_idx; int splits;
    // rank
    const int* gold; const float* gold_val; unsigned long long* best; int* rank;
    // store
    float* out; long long ld_out;
};

template <int METRIC, int EPI>
__global__ void __launch_bounds__(SIM_THREADS, 2)
k_sim_tile(SimParams P) {
    OEA_DYNAMIC_SMEM_ALIGNED16(smem);
    float (*As)[BK][TM] = reinterpret_cast<float (*)[BK][TM]>(smem);                      // [STAGES][BK][TM]
    float (*Bs)[BK][TN] = reinterpret_cast<float (*)[BK][TN]>(smem + STAGES * BK * TM);   // [STAGES][BK][TN]
    float* Ts = smem + STAGES * BK * TM + STAGES * BK * TN;                                    // [TM][TS_LD] (TOPK only)
    float* Lv = Ts + (TM / 2) * TS_LD;                                            // [TM][kcap]
    int* Li = reinterpret_cast<int*>(Lv + TM * P.kcap);                              // [TM][kcap]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tx = tid & 15, ty = tid >> 4;
    const int row0 = blockIdx.x * TM;
    const int n_col_tiles = (P.n2 + TN - 1) / TN;
    const int ct0 = blockIdx.y * P.col_tiles_per_split;
    const int ct1 = min(n_col_tiles, ct0 + P.col_tiles_per_split);

    const float* At = P.e1t + row0;      // this row block's columns of the k-major copy
    const int ld_kk = tid >> 5, ld_c4 = (tid & 31) * 4;   // loader mapping: 2 × (k = tid/32 + 8i, 4 consecutive rows)

    if (EPI == EPI_TOPK) {
        for (int i = tid; i < TM * P.kcap; i += SIM_THREADS) { Lv[i] = -FLT_MAX; Li[i] = -1; }
    }
    // per-thread rank state (EPI_RANK): counters + running arg-max; gold value/column are re-read per tile
    float bestv[8]; int besti[8], cnt[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { bestv[i] = -FLT_MAX; besti[i] = 0x7fffffff; cnt[i] = 0; }
    const int nk = (P.kdim + BK - 1) / BK;

    for (int ct = ct0; ct < ct1; ++ct) {
        const int col0 = ct * TN;
        const float* Bt = P.e2t + col0;
        float acc[8][8];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

        auto issue = [&](int kc, int stage) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int kk = ld_kk + 8 * i;
                cp_async16(&As[stage][kk][ld_c4], At + (size_t)(kc * BK + kk) * P.ld1t + ld_c4);
                cp_async16(&Bs[stage][kk][ld_c4], Bt + (size_t)(kc * BK + kk) * P.ld2t + ld_c4);
            }
        };
        __syncthreads();   // previous tile's compute / epilogue readers are done with every stage
#pragma unroll
        for (int st = 0; st < STAGES - 1; ++st) {
            if (st < nk) issue(st, st);
            cp_async_commit();
        }
        for (int kc = 0; kc < nk; ++kc) {
            cp_async_wait<STAGES - 2>();   // chunk kc has landed (for this thread) …
            __syncthreads();               // … for every thread; and everyone finished chunk kc−1 (its stage is refilled next)
            if (kc + STAGES - 1 < nk) issue(kc + STAGES - 1, (kc + STAGES - 1) % STAGES);
            cp_async_commit();
            const int buf = kc % STAGES;
            const int kk_end = min(BK, P.kdim - kc * BK);   // kdim % 4 == 0: the tail chunk runs 4, 8 or 12 steps
#pragma unroll 4
            for (int kk = 0; kk < kk_end; ++kk) {
                const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
                const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
                const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
                const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
                const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[i][j] = sim_accum<METRIC>(a[i], b[j], acc[i][j]);
            }
        }

        // ---- epilogue ----
        float coff[8], roff[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = col0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + j - 4);
            coff[j] = (P.col_off && c < P.n2) ? __ldg(P.col_off + c) : 0.f;
            const int r = row0 + (j < 4 ? ty * 4 + j : 64 + ty * 4 + j - 4);
            roff[j] = (P.row_off && r < P.n1) ? __ldg(P.row_off + r) : 0.f;
        }
        const bool use_csls = P.row_off != nullptr;
        if (EPI == EPI_TOPK) {
            // two halves of 64 rows (thread rows i = 0..3, then 4..7) through a 64-row staging buffer
            const int k = P.k;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                if (half == 1) __syncthreads();   // scan of half 0 finished before Ts is overwritten
#pragma unroll
                for (int ii = 0; ii < 4; ++ii) {
                    const int i = half * 4 + ii;
                    const int rl = ty * 4 + ii;   // row inside the half
#pragma unroll
                    for (int jj = 0; jj < 2; ++jj) {
                        const int cl = jj == 0 ? tx * 4 : 64 + tx * 4;
                        float v[4];
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            v[j] = sim_value<METRIC>(acc[i][jj * 4 + j]);
                            if (use_csls) v[j] = csls_value(v[j], roff[i], coff[jj * 4 + j]);
                            if (col0 + cl + j >= P.n2) v[j] = -FLT_MAX;
                        }
                        *reinterpret_cast<float4*>(&Ts[rl * TS_LD + cl]) = make_float4(v[0], v[1], v[2], v[3]);
                    }
                }
                __syncthreads();
                for (int rh = warp; rh < TM / 2; rh += SIM_THREADS / 32) {
                    const int rl = half * 64 + rh;   // row inside the tile
                    float lv = lane < P.kcap ? Lv[rl * P.kcap + lane] : -FLT_MAX;
                    int li = lane < P.kcap ? Li[rl * P.kcap + lane] : -1;
                    float tau = __shfl_sync(OEA_FULL, lv, k - 1);
                    bool changed = false;
#pragma unroll
                    for (int m = 0; m < TN / 32; ++m) {
                        const float c = Ts[rh * TS_LD + lane + 32 * m];
                        unsigned pass = __ballot_sync(OEA_FULL, c > tau);
                        while (pass) {
                            const int src = __ffs(pass) - 1;
                            pass &= pass - 1;
                            const float cv = __shfl_sync(OEA_FULL, c, src);
                            if (!(cv > tau)) continue;   // tau rose since the ballot
                            const int ci = col0 + src + 32 * m;
                            // entries with value >= cv keep their place (they have lower column indices)
                            const int pos = __popc(__ballot_sync(OEA_FULL, lane < k && lv >= cv));
                            const float up_v = __shfl_up_sync(OEA_FULL, lv, 1);
                            const int up_i = __shfl_up_sync(OEA_FULL, li, 1);
                            if (lane > pos) { lv = up_v; li = up_i; }
                            else if (lane == pos) { lv = cv; li = ci; }
                            tau = __shfl_sync(OEA_FULL, lv, k - 1);
                            changed = true;
                        }
                    }
                    if (changed && lane < P.kcap) { Lv[rl * P.kcap + lane] = lv; Li[rl * P.kcap + lane] = li; }
                }
            }
            // the next tile's first __syncthreads orders these smem reads before Ts is rewritten
        } else if (EPI == EPI_RANK) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int r = row0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
                const bool ok = r < P.n1;
                const float gval = ok ? __ldg(P.gold_val + r) : FLT_MAX;
                const int goldc = ok ? __ldg(P.gold + r) : -1;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = col0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + j - 4);
                    float v = sim_value<METRIC>(acc[i][j]);
                    if (use_csls) v = csls_value(v, roff[i], coff[j]);
                    if (c < P.n2) {
                        // rank of gold = #{better} + #{equal with a lower index} ("lower index wins")
                        cnt[i] += (v > gval) || (v == gval && c < goldc);
                        if (v > bestv[i]) { bestv[i] = v; besti[i] = c; }   // columns ascend per thread
                    }
                }
            }
        } else {  // EPI_STORE
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int r = row0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
                if (r >= P.n1) continue;
#pragma unroll
                for (int jj = 0; jj < 2; ++jj) {
                    const int c = col0 + (jj == 0 ? tx * 4 : 64 + tx * 4);
                    float v[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        v[j] = sim_value<METRIC>(acc[i][jj * 4 + j]);
                        if (use_csls) v[j] = csls_value(v[j], roff[i], coff[jj * 4 + j]);
                    }
                    float* o = P.out + (size_t)r * P.ld_out + c;
                    if (c + 3 < P.n2 && (P.ld_out & 3) == 0) *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
                    else {
#pragma unroll
                        for (int j = 0; j < 4; ++j) if (c + j < P.n2) o[j] = v[j];
                    }
                }
            }
        }
    }

    if (EPI == EPI_TOPK) {
        __syncthreads();
        for (int rl = warp; rl < TM; rl += SIM_THREADS / 32) {
            const int r = row0 + rl;
            if (r < P.n1 && lane < P.k) {
                const size_t o = ((size_t)r * P.splits + blockIdx.y) * P.k + lane;
                P.part_val[o] = Lv[rl * P.kcap + lane];
                P.part_idx[o] = Li[rl * P.kcap + lane];
            }
        }
    } else if (EPI == EPI_RANK) {
        // reduce across the 16 threads (tx) that share a row: they sit in one half-warp
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            int c = cnt[i]; float bv = bestv[i]; int bi = besti[i];
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) {
                c += __shfl_xor_sync(OEA_FULL, c, o);
                const float ov = __shfl_xor_sync(OEA_FULL, bv, o);
                const int oi = __shfl_xor_sync(OEA_FULL, bi, o);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            const int r = row0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
            if (tx == 0 && r < P.n1) {
                if (c) atomicAdd(P.rank + r, c);
                // order-preserving float → uint, high word; low word = ~index so the lowest index wins ties
                unsigned u = __float_as_uint(bv);
                u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
                const unsigned long long packed = ((unsigned long long)u << 32) | (unsigned)(0x7fffffff - bi);
                atomicMax(P.best + r, packed);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Short-contraction store kernel (kdim ≤ 104, i.e. the d = 75 / 100 embeddings of MTransE / BootEA): the A panel of the
// row block ([kdim][128], ≤ 53 KB) is loaded ONCE and stays in shared memory for every column tile; a B tile arrives as
// two half-K stages ([KH][128] each), so a tile costs 2 block barriers instead of 7 and every load has half a tile of
// FFMA work to land behind.  Same 8×8 register tile, same ascending-k accumulation as k_sim_tile, hence
// bit-identical values.  2 CTAs per SM (2 × (2·KH + 2·KH)·128·4 B ≤ 213 KB).
// ------------------------------------------------------------------------------------------------
constexpr int SHORTK_MAX = 104;

template <int METRIC>
__global__ void __launch_bounds__(SIM_THREADS, 2)
k_sim_store_shortk(SimParams P, int KH) {
    OEA_DYNAMIC_SMEM_ALIGNED16(smem);
    float* Ares = smem;                       // [2·KH][TM]
    float* Bbuf0 = Ares + 2 * KH * TM;        // [KH][TN]  k in [0, KH)
    float* Bbuf1 = Bbuf0 + KH * TN;           // [KH][TN]  k in [KH, 2·KH)

    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int row0 = blockIdx.x * TM;
    const int n_col_tiles = (P.n2 + TN - 1) / TN;
    const int ct0 = blockIdx.y * P.col_tiles_per_split;
    const int ct1 = min(n_col_tiles, ct0 + P.col_tiles_per_split);
    if (ct0 >= ct1) return;
    const int ld_kk = tid >> 5, ld_c4 = (tid & 31) * 4;
    const float* At = P.e1t + row0;

    auto issue_b = [&](int ct, int half) {
        const float* Bt = P.e2t + (size_t)ct * TN + (size_t)(half * KH) * P.ld2t;
        float* dst = half ? Bbuf1 : Bbuf0;
        for (int kk = ld_kk; kk < KH; kk += 8) cp_async16(dst + kk * TN + ld_c4, Bt + (size_t)kk * P.ld2t + ld_c4);
    };
    for (int kk = ld_kk; kk < 2 * KH; kk += 8) cp_async16(Ares + kk * TM + ld_c4, At + (size_t)kk * P.ld1t + ld_c4);
    issue_b(ct0, 0);
    cp_async_commit();

    const bool use_csls = P.row_off != nullptr;
    float roff[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int r = row0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
        roff[i] = (use_csls && r < P.n1) ? __ldg(P.row_off + r) : 0.f;
    }
    const int k_half1 = P.kdim - KH;          // k-steps of the second half that carry data (multiple of 4, ≥ 0)

    for (int ct = ct0; ct < ct1; ++ct) {
        const int col0 = ct * TN;
        float acc[8][8];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

#pragma unroll
        for (int half = 0; half < 2; ++half) {
            cp_async_wait<0>();
            __syncthreads();      // this half has landed for everyone; everyone is done with the other buffer
            if (half == 0) issue_b(ct, 1);                       // second half of this tile → Bbuf1
            else if (ct + 1 < ct1) issue_b(ct + 1, 0);           // first half of the next tile → Bbuf0
            cp_async_commit();
            const float* Ab = Ares + half * KH * TM;
            const float* Bb = half ? Bbuf1 : Bbuf0;
            const int kk_end = half ? k_half1 : min(KH, P.kdim);
#pragma unroll 4
            for (int kk = 0; kk < kk_end; ++kk) {
                const float4 a0 = *reinterpret_cast<const float4*>(Ab + kk * TM + ty * 4);
                const float4 a1 = *reinterpret_cast<const float4*>(Ab + kk * TM + 64 + ty * 4);
                const float4 b0 = *reinterpret_cast<const float4*>(Bb + kk * TN + tx * 4);
                const float4 b1 = *reinterpret_cast<const float4*>(Bb + kk * TN + 64 + tx * 4);
                const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[i][j] = sim_accum<METRIC>(a[i], b[j], acc[i][j]);
            }
        }

        float coff[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = col0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + j - 4);
            coff[j] = (use_csls && c < P.n2) ? __ldg(P.col_off + c) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = row0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
            if (r >= P.n1) continue;
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
                const int c = col0 + (jj == 0 ? tx * 4 : 64 + tx * 4);
                float v[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    v[j] = sim_value<METRIC>(acc[i][jj * 4 + j]);
                    if (use_csls) v[j] = csls_value(v[j], roff[i], coff[jj * 4 + j]);
                }
                float* o = P.out + (size_t)r * P.ld_out + c;
                if (c + 3 < P.n2 && (P.ld_out & 3) == 0) *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
                else {
#pragma unroll
                    for (int j = 0; j < 4; ++j) if (c + j < P.n2) o[j] = v[j];
                }
            }
        }
    }
    cp_async_wait<0>();
}

// Merge the per-split sorted lists of a row (splits ascend in column index, so ties keep the lower index).
__global__ void __launch_bounds__(256)
k_topk_merge(const float* __restrict__ part_val, const int* __restrict__ part_idx, int n1, int splits, int k,
             float* __restrict__ out_val, int* __restrict__ out_idx, float* __restrict__ out_mean) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n1) return;
    float lv = -FLT_MAX; int li = -1;
    const size_t base = (size_t)row * splits * k;
    if (lane < k) { lv = part_val[base + lane]; li = part_idx[base + lane]; }
    for (int s = 1; s < splits; ++s) {
        float tau = __shfl_sync(OEA_FULL, lv, k - 1);
        for (int m = 0; m < k; ++m) {
            const float cv = part_val[base + (size_t)s * k + m];
            const int ci = part_idx[base + (size_t)s * k + m];
            if (!(cv > tau)) break;  // lists are sorted descending
            const int pos = __popc(__ballot_sync(OEA_FULL, lane < k && lv >= cv));
            const float up_v = __shfl_up_sync(OEA_FULL, lv, 1);
            const int up_i = __shfl_up_sync(OEA_FULL, li, 1);
            if (lane > pos) { lv = up_v; li = up_i; }
            else if (lane == pos) { lv = cv; li = ci; }
            tau = __shfl_sync(OEA_FULL, lv, k - 1);
        }
    }
    if (lane < k) {
        if (out_val) out_val[(size_t)row * k + lane] = lv;
        if (out_idx) out_idx[(size_t)row * k + lane] = li;
    }
    if (out_mean) {  // np.mean over the k nearest values (similarity.py:80-83)
        float s = lane < k ? lv : 0.f;
        s = warp_sum(s);
        if (lane == 0) out_mean[row] = s / (float)k;
    }
}

// Similarity of row i with its gold column, bit-identical to the tile kernel's accumulation order.
template <int METRIC>
__global__ void k_sim_gold(const float* __restrict__ e1, const float* __restrict__ e2, int n1, int pitch1, int pitch2,
                           int kdim, const int* __restrict__ gold, const float* __restrict__ row_off,
                           const float* __restrict__ col_off, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n1) return;
    const int g = gold[i];
    const float* a = e1 + (size_t)i * pitch1;
    const float* b = e2 + (size_t)g * pitch2;
    float acc = 0.f;
    for (int k = 0; k < kdim; ++k) acc = sim_accum<METRIC>(__ldg(a + k), __ldg(b + k), acc);
    float v = sim_value<METRIC>(acc);
    if (row_off) v = csls_value(v, row_off[i], col_off[g]);
    out[i] = v;
}

__global__ void k_rank_finish(const unsigned long long* __restrict__ best, int n1, int* __restrict__ top1) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n1) top1[i] = 0x7fffffff - (int)(best[i] & 0xffffffffu);
}

// sklearn.preprocessing.normalize(x) (similarity.py:30-32): x / ||x||₂, zero rows stay zero.
__global__ void __launch_bounds__(256)
k_rows_normalize(const float* __restrict__ in, int in_pitch, int n, int dim, float* __restrict__ out, int out_pitch) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n) return;
    const float* src = in + (size_t)row * in_pitch;
    float ss = 0.f;
    for (int c = lane; c < dim; c += 32) { const float x = src[c]; ss = fmaf(x, x, ss); }
    ss = warp_sum(ss);
    const float inv = ss > 0.f ? 1.f / sqrtf(ss) : 0.f;
    float* dst = out + (size_t)row * out_pitch;
    for (int c = lane; c < out_pitch; c += 32) dst[c] = c < dim ? src[c] * inv : 0.f;
}

// k-major copy of an operand: out[k][r] = in[r][k] for r < n, k < pitch; zero elsewhere ([kpad, ld] with
// kpad = ceil16(pitch), ld = ceil128(n)), so the tile loader needs no bounds checks.  32×32 smem tiles.
__global__ void __launch_bounds__(256)
k_sim_transpose(const float* __restrict__ in, int pitch, int n, float* __restrict__ out, long long ld, int kpad) {
    __shared__ float t[32][33];
    const int r0 = blockIdx.x * 32, k0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 8 rows of 32 threads
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = r0 + ty + 8 * i, k = k0 + tx;
        t[ty + 8 * i][tx] = (r < n && k < pitch) ? __ldg(in + (size_t)r * pitch + k) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int k = k0 + ty + 8 * i, r = r0 + tx;
        if (k < kpad && r < ld) out[(size_t)k * ld + r] = t[tx][ty + 8 * i];
    }
}

static size_t sim_smem_bytes(int epi, int kcap) {
    size_t f = STAGES * BK * TM + STAGES * BK * TN;
    if (epi == EPI_TOPK) f += (TM / 2) * TS_LD + 2 * TM * kcap;
    return f * sizeof(float);
}

static int check_sim(const oea_sim_cfg* c, const float* e1, const float* e2) {
    if (!c || !e1 || !e2) return OEA_ERR_NULL;
    if (c->n1 <= 0 || c->n2 <= 0 || c->dim <= 0) return OEA_ERR_DIM;
    if (c->pitch1 < c->dim || c->pitch2 < c->dim || (c->pitch1 & 3) || (c->pitch2 & 3)) return OEA_ERR_DIM;
    if (!aligned16(e1) || !aligned16(e2)) return OEA_ERR_ALIGN;
    if (c->metric < OEA_METRIC_INNER || c->metric > OEA_METRIC_L2) return OEA_ERR_KIND;
    if (!c->e1_t || !c->e2_t) return OEA_ERR_NULL;                       // k-major copies from oea_sim_transpose
    const int64_t np1 = ((int64_t)c->n1 + TM - 1) / TM * TM, np2 = ((int64_t)c->n2 + TN - 1) / TN * TN;
    if (c->ld1_t < np1 || c->ld2_t < np2 || (c->ld1_t & 3) || (c->ld2_t & 3)) return OEA_ERR_SHAPE;
    if (!aligned16(c->e1_t) || !aligned16(c->e2_t)) return OEA_ERR_ALIGN;
    return OEA_OK;
}

// OEA_SIM_NO_SHORTK=1 keeps the 3-stage streaming tile kernel for every shape (A/B measurements, tests of both paths)
static bool sim_no_shortk() {
    const char* v = getenv("OEA_SIM_NO_SHORTK");
    return v != nullptr && v[0] == '1';
}

static int sm_count() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) sms = 132;
    }
    return sms;
}

template <int EPI>
static int launch_sim(const oea_sim_cfg* c, SimParams& P, int splits, cudaStream_t st) {
    const dim3 grid((c->n1 + TM - 1) / TM, splits);
    const size_t smem = sim_smem_bytes(EPI, P.kcap);
#define OEA_SIM_LAUNCH(M)                                                                                     \
    do {                                                                                                      \
        OEA_CUDA_TRY(cudaFuncSetAttribute(k_sim_tile<M, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        OEA_LAUNCH((k_sim_tile<M, EPI>), grid, SIM_THREADS, smem, st, P);                                               \
    } while (0)
    switch (c->metric) {
        case OEA_METRIC_INNER: OEA_SIM_LAUNCH(OEA_METRIC_INNER); break;
        case OEA_METRIC_L1: OEA_SIM_LAUNCH(OEA_METRIC_L1); break;
        default: OEA_SIM_LAUNCH(OEA_METRIC_L2); break;
    }
#undef OEA_SIM_LAUNCH
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

// Column splits per row block: the split count that wastes the least of the last wave.  A CTA's time is
// proportional to its number of column tiles, so with `slots` resident CTAs the kernel takes
// ceil(row_blocks·splits / slots) · ceil(col_tiles / splits) tile-times: a partial wave costs a whole one.
static int pick_splits(int n1, int n2) {
    const int row_blocks = (n1 + TM - 1) / TM, col_tiles = (n2 + TN - 1) / TN;
    const long long slots = 2LL * sm_count();              // 2 CTAs per SM (registers and shared memory both allow 2)
    int best = 1;
    long long best_cost = -1;
    const int max_splits = col_tiles < 64 ? col_tiles : 64;
    for (int sp = 1; sp <= max_splits; ++sp) {
        const long long per = (col_tiles + sp - 1) / sp;
        const long long eff_splits = (col_tiles + per - 1) / per;
        const long long waves = (row_blocks * eff_splits + slots - 1) / slots;
        const long long cost = waves * per * 64 + eff_splits;   // tile-times first, then fewer partial lists to merge
        if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = sp; }
    }
    return best;
}

static void fill_common(SimParams& P, const oea_sim_cfg* c, const float* e1, const float* e2,
                        const float* row_off, const float* col_off, int splits) {
    P.e1 = e1; P.e2 = e2; P.e1t = c->e1_t; P.e2t = c->e2_t; P.ld1t = c->ld1_t; P.ld2t = c->ld2_t; P.n1 = c->n1; P.n2 = c->n2; P.pitch1 = c->pitch1; P.pitch2 = c->pitch2;
    P.kdim = c->pitch1 < c->pitch2 ? c->pitch1 : c->pitch2;   // padding columns are zero on both sides
    P.row_off = row_off; P.col_off = col_off;
    const int col_tiles = (c->n2 + TN - 1) / TN;
    P.col_tiles_per_split = (col_tiles + splits - 1) / splits;
    P.splits = splits;
}

}  // namespace oea

using namespace oea;

extern "C" int64_t oea_sim_transpose_ld(int32_t n) { return n > 0 ? ((int64_t)n + TM - 1) / TM * TM : 0; }
extern "C" size_t oea_sim_transpose_bytes(int32_t n, int32_t pitch) {
    if (n <= 0 || pitch <= 0) return 0;
    return (size_t)((pitch + BK - 1) / BK * BK) * (size_t)oea_sim_transpose_ld(n) * sizeof(float);
}
extern "C" int oea_sim_transpose(const float* in, int32_t pitch, int32_t n, float* out, void* stream) {
    if (!in || !out) return OEA_ERR_NULL;
    if (n <= 0 || pitch <= 0 || (pitch & 3)) return OEA_ERR_DIM;
    const long long ld = oea_sim_transpose_ld(n);
    const int kpad = (pitch + BK - 1) / BK * BK;
    const dim3 grid((unsigned)((ld + 31) / 32), (unsigned)((kpad + 31) / 32));
    OEA_LAUNCH(k_sim_transpose, grid, 256, 0, (cudaStream_t)stream, in, pitch, n, out, ld, kpad);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" size_t oea_sim_topk_workspace_bytes(const oea_sim_cfg* c, int32_t k) {
    if (!c || k < 1 || k > KMAX) return 0;
    const int splits = pick_splits(c->n1, c->n2);
    return (size_t)c->n1 * splits * k * (sizeof(float) + sizeof(int));
}

extern "C" int oea_sim_topk(const oea_sim_cfg* c, const float* e1, const float* e2,
                            const float* row_off, const float* col_off, int32_t k,
                            float* out_val, int32_t* out_idx, float* out_mean,
                            void* workspace, size_t workspace_bytes, void* stream) {
    int rc = check_sim(c, e1, e2); if (rc) return rc;
    if (k < 1 || k > KMAX || k > c->n2) return OEA_ERR_RANGE;
    if ((row_off == nullptr) != (col_off == nullptr)) return OEA_ERR_NULL;
    if (!out_val && !out_idx && !out_mean) return OEA_ERR_NULL;
    const int splits = pick_splits(c->n1, c->n2);
    const size_t need = (size_t)c->n1 * splits * k * (sizeof(float) + sizeof(int));
    if (!workspace || workspace_bytes < need) return OEA_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    SimParams P{};
    fill_common(P, c, e1, e2, row_off, col_off, splits);
    // splits that start past the last column tile would leave garbage: recompute the effective count
    const int col_tiles = (c->n2 + TN - 1) / TN;
    const int eff_splits = (col_tiles + P.col_tiles_per_split - 1) / P.col_tiles_per_split;
    P.splits = eff_splits;
    P.k = k;
    P.kcap = k <= 8 ? 8 : (k <= 16 ? 16 : 32);
    P.part_val = (float*)workspace;
    P.part_idx = (int*)((char*)workspace + (size_t)c->n1 * splits * k * sizeof(float));
    rc = launch_sim<EPI_TOPK>(c, P, eff_splits, st); if (rc) return rc;
    OEA_LAUNCH(k_topk_merge, (c->n1 + 7) / 8, 256, 0, st, P.part_val, P.part_idx, c->n1, eff_splits, k, out_val, out_idx, out_mean);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" size_t oea_sim_rank_workspace_bytes(const oea_sim_cfg* c) {
    if (!c) return 0;
    return (size_t)c->n1 * (sizeof(unsigned long long) + sizeof(float));
}

extern "C" int oea_sim_rank(const oea_sim_cfg* c, const float* e1, const float* e2,
                            const float* row_off, const float* col_off, const int32_t* gold,
                            int32_t* out_top1, int32_t* out_rank,
                            void* workspace, size_t workspace_bytes, void* stream) {
    int rc = check_sim(c, e1, e2); if (rc) return rc;
    if (!gold || !out_top1 || !out_rank) return OEA_ERR_NULL;
    if ((row_off == nullptr) != (col_off == nullptr)) return OEA_ERR_NULL;
    const size_t need = oea_sim_rank_workspace_bytes(c);
    if (!workspace || workspace_bytes < need) return OEA_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    unsigned long long* best = (unsigned long long*)workspace;
    float* gold_val = (float*)((char*)workspace + (size_t)c->n1 * sizeof(unsigned long long));
    OEA_CUDA_TRY(cudaMemsetAsync(best, 0, (size_t)c->n1 * sizeof(unsigned long long), st));
    OEA_CUDA_TRY(cudaMemsetAsync(out_rank, 0, (size_t)c->n1 * sizeof(int), st));
    const int splits = pick_splits(c->n1, c->n2);
    SimParams P{};
    fill_common(P, c, e1, e2, row_off, col_off, splits);
    const int col_tiles = (c->n2 + TN - 1) / TN;
    const int eff_splits = (col_tiles + P.col_tiles_per_split - 1) / P.col_tiles_per_split;
    P.splits = eff_splits;
    const int gb = (c->n1 + 127) / 128;
    switch (c->metric) {
        case OEA_METRIC_INNER: OEA_LAUNCH(k_sim_gold<OEA_METRIC_INNER>, gb, 128, 0, st, e1, e2, c->n1, c->pitch1, c->pitch2, P.kdim, gold, row_off, col_off, gold_val); break;
        case OEA_METRIC_L1: OEA_LAUNCH(k_sim_gold<OEA_METRIC_L1>, gb, 128, 0, st, e1, e2, c->n1, c->pitch1, c->pitch2, P.kdim, gold, row_off, col_off, gold_val); break;
        default: OEA_LAUNCH(k_sim_gold<OEA_METRIC_L2>, gb, 128, 0, st, e1, e2, c->n1, c->pitch1, c->pitch2, P.kdim, gold, row_off, col_off, gold_val); break;
    }
    OEA_LAUNCH_CHECK();
    P.gold = gold; P.gold_val = gold_val; P.best = best; P.rank = out_rank;
    rc = launch_sim<EPI_RANK>(c, P, eff_splits, st); if (rc) return rc;
    OEA_LAUNCH(k_rank_finish, gb, 128, 0, st, best, c->n1, out_top1);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_sim_matrix(const oea_sim_cfg* c, const float* e1, const float* e2,
                              const float* row_off, const float* col_off, float* out, int64_t ld_out, void* stream) {
    int rc = check_sim(c, e1, e2); if (rc) return rc;
    if (!out) return OEA_ERR_NULL;
    if (ld_out < c->n2) return OEA_ERR_SHAPE;
    if ((row_off == nullptr) != (col_off == nullptr)) return OEA_ERR_NULL;
    SimParams P{};
    const int col_tiles = (c->n2 + TN - 1) / TN;
    int splits = pick_splits(c->n1, c->n2);
    fill_common(P, c, e1, e2, row_off, col_off, splits);
    const int eff_splits = (col_tiles + P.col_tiles_per_split - 1) / P.col_tiles_per_split;
    P.out = out; P.ld_out = ld_out;
    if (P.kdim <= SHORTK_MAX && !sim_no_shortk()) {
        const int KH = ((P.kdim + 1) / 2 + 3) / 4 * 4;        // k-steps per half stage; 2·KH ≤ the k-major copies' padded rows
        const size_t smem = (size_t)(2 * KH * TM + 2 * KH * TN) * sizeof(float);
        const dim3 grid((c->n1 + TM - 1) / TM, eff_splits);
        cudaStream_t st = (cudaStream_t)stream;
#define OEA_SHORTK_LAUNCH(M)                                                                                              \
    do {                                                                                                                  \
        OEA_CUDA_TRY(cudaFuncSetAttribute(k_sim_store_shortk<M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        OEA_LAUNCH(k_sim_store_shortk<M>, grid, SIM_THREADS, smem, st, P, KH);                                                    \
    } while (0)
        switch (c->metric) {
            case OEA_METRIC_INNER: OEA_SHORTK_LAUNCH(OEA_METRIC_INNER); break;
            case OEA_METRIC_L1: OEA_SHORTK_LAUNCH(OEA_METRIC_L1); break;
            default: OEA_SHORTK_LAUNCH(OEA_METRIC_L2); break;
        }
#undef OEA_SHORTK_LAUNCH
        OEA_LAUNCH_CHECK();
        return OEA_OK;
    }
    return launch_sim<EPI_STORE>(c, P, eff_splits, (cudaStream_t)stream);
}

extern "C" int oea_rows_normalize(const float* in, int32_t in_pitch, int32_t n, int32_t dim, float* out, int32_t out_pitch,
                                  void* stream) {
    if (!in || !out) return OEA_ERR_NULL;
    if (n < 0 || dim <= 0 || in_pitch < dim || out_pitch < dim) return OEA_ERR_DIM;
    if (n == 0) return OEA_OK;
    OEA_LAUNCH(k_rows_normalize, (n + 7) / 8, 256, 0, (cudaStream_t)stream, in, in_pitch, n, dim, out, out_pitch);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

// ------------------------------------------------------------------------------------------------
// Large-k per-row selection (ε-truncated neighbour search): 3-pass MSB radix select (11+11+10 bits)
// on the order-preserving integer image of the floats, then one compaction pass.  One CTA per row;
// passes 2-4 re-read the row from L2.
// ------------------------------------------------------------------------------------------------
namespace oea {

__device__ __forceinline__ unsigned fkey(float f) {
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

constexpr int SEL_THREADS = 512;
constexpr int SEL_BINS = 2048;

__global__ void __launch_bounds__(SEL_THREADS)
k_rows_select(const float* __restrict__ mat, long long ld, int n_rows, int n_cols, int k,
              const int32_t* __restrict__ col_ids, int32_t* __restrict__ out) {
    __shared__ unsigned hist[SEL_BINS];
    __shared__ unsigned s_chunk[32];
    __shared__ unsigned s_prefix, s_mask, s_remaining, s_gt, s_eq;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int row = blockIdx.x; row < n_rows; row += gridDim.x) {
        const float* src = mat + (size_t)row * ld;
        if (tid == 0) { s_prefix = 0u; s_mask = 0u; s_remaining = (unsigned)k; s_gt = 0u; s_eq = 0u; }
        __syncthreads();
#pragma unroll 1
        for (int pass = 0; pass < 3; ++pass) {
            const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
            const int nb = pass == 2 ? 1024 : 2048;
            for (int i = tid; i < SEL_BINS; i += SEL_THREADS) hist[i] = 0u;
            __syncthreads();
            const unsigned prefix = s_prefix, mask = s_mask;
            for (int j = tid; j < n_cols; j += SEL_THREADS) {
                const unsigned u = fkey(__ldg(src + j));
                if ((u & mask) == prefix) atomicAdd(&hist[(u >> shift) & (unsigned)(nb - 1)], 1u);
            }
            __syncthreads();
            // suffix search from the top bin: find digit D with count(> D) < remaining <= count(>= D)
            if (warp == 0) {
                const int per = nb / 32;
                // read before the __syncwarp below: the lane that owns the digit rewrites s_remaining, and no lane may
                // still be about to read it then (independent thread scheduling gives no convergence guarantee)
                const unsigned remaining = s_remaining;
                unsigned csum = 0;
                for (int b = 0; b < per; ++b) csum += hist[lane * per + b];
                s_chunk[lane] = csum;
                __syncwarp();
                unsigned above = 0;  // elements in chunks above this lane's chunk
                for (int l = lane + 1; l < 32; ++l) above += s_chunk[l];
                const bool mine = above < remaining && above + csum >= remaining;
                if (mine) {
                    unsigned acc = above;
                    for (int b = per - 1; b >= 0; --b) {
                        const unsigned h = hist[lane * per + b];
                        if (acc + h >= remaining) {
                            s_prefix = prefix | ((unsigned)(lane * per + b) << shift);
                            s_mask = mask | ((unsigned)(nb - 1) << shift);
                            s_remaining = remaining - acc;
                            break;
                        }
                        acc += h;
                    }
                }
            }
            __syncthreads();
        }
        const unsigned T = s_prefix, take_eq = s_remaining;
        const unsigned n_gt = (unsigned)k - take_eq;
        int32_t* dst = out + (size_t)row * k;
        for (int j = tid; j < n_cols; j += SEL_THREADS) {
            const unsigned u = fkey(__ldg(src + j));
            if (u > T) {
                const unsigned p = atomicAdd(&s_gt, 1u);
                dst[p] = col_ids ? __ldg(col_ids + j) : j;
            } else if (u == T) {
                const unsigned e = atomicAdd(&s_eq, 1u);
                if (e < take_eq) dst[n_gt + e] = col_ids ? __ldg(col_ids + j) : j;
            }
        }
        __syncthreads();
    }
}

}  // namespace oea

extern "C" int oea_rows_select_topk(const float* mat, int64_t ld, int32_t n_rows, int32_t n_cols, int32_t k,
                                    const int32_t* col_ids, int32_t* out_idx, void* stream) {
    if (!mat || !out_idx) return OEA_ERR_NULL;
    if (n_rows < 0 || n_cols <= 0 || ld < n_cols) return OEA_ERR_SHAPE;
    if (k < 1 || k > n_cols) return OEA_ERR_RANGE;
    if (n_rows == 0) return OEA_OK;
    const int grid = n_rows < 4 * sm_count() ? n_rows : 4 * sm_count();
    OEA_LAUNCH(k_rows_select, grid, SEL_THREADS, 0, (cudaStream_t)stream, mat, ld, n_rows, n_cols, k, col_ids, out_idx);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

// ================================================================================================
// CSLS evaluation on a MATERIALISED similarity matrix (one FP32 tile pass with the store epilogue, then three
// HBM-bound streaming passes) — used when n1·n2·4 B fits the budget: 1 contraction pass instead of 3.
//   k_mat_row_topk_mean : r_i  = mean of the k largest of row i            (warp per row, 128-bit streaming loads)
//   k_mat_col_topk_mean : c_j  = mean of the k largest of column j         (CTA per 128-column strip, smem transpose)
//   k_mat_rank          : arg-max and rank-of-gold of 2·S − r_i − c_j      (warp per row)
// The per-row list logic (ballot + shuffle insertion into a lane-resident sorted list) is the one of the tile kernel.
// ================================================================================================
namespace oea {

// insert candidate values (one per lane, `c`) into the lane-resident descending list `lv` (entries 0..k-1)
__device__ __forceinline__ void list_insert_vals(float c, float& lv, float& tau, int k, int lane) {
    unsigned pass = __ballot_sync(OEA_FULL, c > tau);
    while (pass) {
        const int src = __ffs(pass) - 1;
        pass &= pass - 1;
        const float cv = __shfl_sync(OEA_FULL, c, src);
        if (!(cv > tau)) continue;
        const int pos = __popc(__ballot_sync(OEA_FULL, lane < k && lv >= cv));
        const float up = __shfl_up_sync(OEA_FULL, lv, 1);
        if (lane > pos) lv = up; else if (lane == pos) lv = cv;
        tau = __shfl_sync(OEA_FULL, lv, k - 1);
    }
}

__global__ void __launch_bounds__(256)
k_mat_row_topk_mean(const float* __restrict__ mat, long long ld, int n_rows, int n_cols, int k, float* __restrict__ out_mean) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n_rows) return;                       // whole warps exit together (8 rows per CTA, one per warp)
    const float* src = mat + (size_t)row * ld;
    float lv = -FLT_MAX, tau = -FLT_MAX;
    const int n4 = n_cols >> 2;
    for (int base = 0; base < n4; base += 32) {      // warp-uniform trip count: the list helpers use full-mask shuffles
        const int q = base + lane;
        const float4 v = q < n4 ? ldg4(src + 4 * q) : make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX);
        // the insertion path is rare once tau has risen; the order inside a row is irrelevant for the mean
        if (__ballot_sync(OEA_FULL, v.x > tau || v.y > tau || v.z > tau || v.w > tau)) {
            list_insert_vals(v.x, lv, tau, k, lane); list_insert_vals(v.y, lv, tau, k, lane);
            list_insert_vals(v.z, lv, tau, k, lane); list_insert_vals(v.w, lv, tau, k, lane);
        }
    }
    {   // the last n_cols % 4 columns
        const int j = n4 * 4 + lane;
        list_insert_vals(j < n_cols ? __ldg(src + j) : -FLT_MAX, lv, tau, k, lane);
    }
    float s = lane < k ? lv : 0.f;
    s = warp_sum(s);
    if (lane == 0) out_mean[row] = s / (float)k;
}

// ---- column k-means: thread-owned columns, register-resident sorted lists, rows split over warps ----------------
// Lane l of a warp owns CPT consecutive columns (128-bit or 64-bit loads, a warp row is 32·CPT·4 contiguous bytes);
// each owned column keeps its KCAP largest values in a descending register list (insert = one FMNMX pair per
// slot, taken only when the value beats the list's tail).  The rows are cut into S = 8·gridDim.y splits (one per
// warp), every split writes its KCAP-list per column and k_col_partial_merge folds the S lists.  No shared memory,
// no block barrier; 8 row loads are in flight per thread.
constexpr int CP_WARPS = 8, CP_UNROLL = 8;

template <int KCAP>
__device__ __forceinline__ void reg_list_insert(float (&L)[KCAP], float x) {
#pragma unroll
    for (int i = 0; i < KCAP; ++i) {
        const float hi = fmaxf(L[i], x);
        x = fminf(L[i], x);
        L[i] = hi;
    }
}

template <int KCAP, int CPT>
__global__ void __launch_bounds__(CP_WARPS * 32)
k_mat_col_topk_partial(const float* __restrict__ mat, long long ld, int n_rows, int n_cols, int rows_per_split,
                       float* __restrict__ part, long long ldp) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int c0 = (blockIdx.x * 32 + lane) * CPT;
    const int split = blockIdx.y * CP_WARPS + warp;
    const int r0 = split * rows_per_split;
    const int r1 = min(n_rows, r0 + rows_per_split);
    float L[CPT][KCAP];
#pragma unroll
    for (int q = 0; q < CPT; ++q)
#pragma unroll
        for (int i = 0; i < KCAP; ++i) L[q][i] = -FLT_MAX;
    if (c0 < n_cols) {
        const float* src = mat + (size_t)r0 * ld + c0;
        for (int r = r0; r < r1; r += CP_UNROLL) {
            float v[CP_UNROLL][CPT];
#pragma unroll
            for (int u = 0; u < CP_UNROLL; ++u) {
                if (r + u < r1) {
                    if (CPT == 4) {
                        const float4 t = ldg4(src + (size_t)u * ld);
                        v[u][0] = t.x; v[u][1] = t.y; v[u][CPT - 2] = t.z; v[u][CPT - 1] = t.w;
                    } else {
                        const float2 t = __ldg(reinterpret_cast<const float2*>(src + (size_t)u * ld));
                        v[u][0] = t.x; v[u][CPT - 1] = t.y;
                    }
                } else {
#pragma unroll
                    for (int q = 0; q < CPT; ++q) v[u][q] = -FLT_MAX;
                }
            }
            src += (size_t)CP_UNROLL * ld;
#pragma unroll
            for (int u = 0; u < CP_UNROLL; ++u)
#pragma unroll
                for (int q = 0; q < CPT; ++q)
                    if (v[u][q] > L[q][KCAP - 1]) reg_list_insert<KCAP>(L[q], v[u][q]);
        }
    }
    // columns past n_cols inside the padded leading dimension hold whatever the store pass left: never written out
#pragma unroll
    for (int q = 0; q < CPT; ++q) {
        const int c = c0 + q;
        if (c < n_cols) {
#pragma unroll
            for (int i = 0; i < KCAP; ++i) part[((size_t)split * KCAP + i) * ldp + c] = L[q][i];
        }
    }
}

// Fold the S per-split lists of a column: 32 columns per CTA, 8 threads per column each folding every 8th split,
// then one of them folds the 8 intermediate lists (shared memory).  Reads are 128 contiguous bytes per warp.
template <int KCAP>
__global__ void __launch_bounds__(256)
k_col_partial_merge(const float* __restrict__ part, long long ldp, int n_cols, int n_splits, int k, float* __restrict__ out_mean) {
    __shared__ float s_lists[8][KCAP][32];
    const int cx = threadIdx.x & 31, sg = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + cx;
    float M[KCAP];
#pragma unroll
    for (int i = 0; i < KCAP; ++i) M[i] = -FLT_MAX;
    if (c < n_cols) {
        for (int sidx = sg; sidx < n_splits; sidx += 8) {
#pragma unroll
            for (int i = 0; i < KCAP; ++i) {
                const float x = __ldg(part + ((size_t)sidx * KCAP + i) * ldp + c);
                if (x > M[KCAP - 1]) reg_list_insert<KCAP>(M, x);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < KCAP; ++i) s_lists[sg][i][cx] = M[i];
    __syncthreads();
    if (sg != 0 || c >= n_cols) return;
    for (int g = 1; g < 8; ++g) {
#pragma unroll
        for (int i = 0; i < KCAP; ++i) {
            const float x = s_lists[g][i][cx];
            if (x > M[KCAP - 1]) reg_list_insert<KCAP>(M, x);
        }
    }
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < KCAP; ++i) if (i < k) sum += M[i];
    out_mean[c] = sum / (float)k;
}

static int col_kcap(int k) { return k <= 4 ? 4 : (k <= 8 ? 8 : (k <= 10 ? 10 : (k <= 16 ? 16 : 32))); }
static int col_cpt(int kcap) { return kcap <= 16 ? 4 : 2; }
// row splits: 8 per CTA row; enough CTAs for two per SM, but at least 64 rows per split
static int col_grid_y(int n_rows, int n_cols, int cpt) {
    const int groups = (n_cols + 32 * cpt - 1) / (32 * cpt);
    int gy = (2 * sm_count() + groups - 1) / groups;
    if (gy < 1) gy = 1;
    if (gy > 16) gy = 16;
    while (gy > 1 && (n_rows + gy * CP_WARPS - 1) / (gy * CP_WARPS) < 64) --gy;
    return gy;
}

// arg-max and rank of the gold column over one stored row (warp per row, 128-bit loads).  Rank rule of
// calculate_rank's argsort (alignment.py:146-168, "lower index wins"): #{v > gold} + #{v == gold, j < gold column};
// left of the gold column that is one ≥ test, right of it one > test, so only the group holding it takes the general
// rule.  The running maximum is updated through a per-group max first (updates are rare after the first groups).
__global__ void __launch_bounds__(256)
k_mat_rank(const float* __restrict__ mat, long long ld, int n_rows, int n_cols, const float* __restrict__ row_off,
           const float* __restrict__ col_off, const int* __restrict__ gold, int* __restrict__ out_top1, int* __restrict__ out_rank) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    const float* src = mat + (size_t)row * ld;
    const bool csls = row_off != nullptr;
    const float ro = csls ? __ldg(row_off + row) : 0.f;
    const int g = __ldg(gold + row);
    float gval = __ldg(src + g);
    if (csls) gval = csls_value(gval, ro, __ldg(col_off + g));
    int cnt = 0, besti = 0x7fffffff;
    float bestv = -FLT_MAX;
    const bool vec = (ld & 3) == 0 && aligned16(mat) && (!csls || aligned16(col_off));
    const int n4 = vec ? (n_cols >> 2) : 0;
    for (int j4 = lane; j4 < n4; j4 += 32) {
        const int j = 4 * j4;
        float4 v = ldg4(src + j);
        if (csls) {
            const float4 co = ldg4(col_off + j);
            v = fma4(v, 2.f, f4(-ro)) - co;          // (2·s − r) − c, the rounding of csls_value
        }
        if (j + 3 < g) cnt += (v.x >= gval) + (v.y >= gval) + (v.z >= gval) + (v.w >= gval);
        else if (j > g) cnt += (v.x > gval) + (v.y > gval) + (v.z > gval) + (v.w > gval);
        else {
            cnt += (v.x > gval) || (v.x == gval && j < g);
            cnt += (v.y > gval) || (v.y == gval && j + 1 < g);
            cnt += (v.z > gval) || (v.z == gval && j + 2 < g);
            cnt += (v.w > gval) || (v.w == gval && j + 3 < g);
        }
        if (fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)) > bestv) {      // columns ascend per lane: first maximum kept
            if (v.x > bestv) { bestv = v.x; besti = j; }
            if (v.y > bestv) { bestv = v.y; besti = j + 1; }
            if (v.z > bestv) { bestv = v.z; besti = j + 2; }
            if (v.w > bestv) { bestv = v.w; besti = j + 3; }
        }
    }
    for (int j = 4 * n4 + lane; j < n_cols; j += 32) {
        float v = __ldg(src + j);
        if (csls) v = csls_value(v, ro, __ldg(col_off + j));
        cnt += (v > gval) || (v == gval && j < g);
        if (v > bestv) { bestv = v; besti = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        cnt += __shfl_xor_sync(OEA_FULL, cnt, o);
        const float ov = __shfl_xor_sync(OEA_FULL, bestv, o);
        const int oi = __shfl_xor_sync(OEA_FULL, besti, o);
        if (ov > bestv || (ov == bestv && oi < besti)) { bestv = ov; besti = oi; }
    }
    if (lane == 0) { out_rank[row] = cnt; out_top1[row] = besti; }
}

// Hits@k counts, Σ(rank+1) and Σ1/(rank+1) of a rank vector in one launch (alignment.py:55-69 does this on the host).
// out[0..n_top) = #{rank < top_k[i]}, out[n_top] = Σ(rank+1), out[n_top+1] = Σ 1/(rank+1); fp64, zeroed by the caller.
constexpr int STATS_MAX_TOP = 8;
struct TopKs { int v[STATS_MAX_TOP]; };
__global__ void __launch_bounds__(256)
k_rank_stats(const int* __restrict__ rank, int n, TopKs tk, int n_top, double* __restrict__ out) {
    __shared__ double s_acc[8][STATS_MAX_TOP + 2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int hits[STATS_MAX_TOP];
#pragma unroll
    for (int i = 0; i < STATS_MAX_TOP; ++i) hits[i] = 0;
    double mr = 0.0, mrr = 0.0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int r = __ldg(rank + i);
#pragma unroll
        for (int t = 0; t < STATS_MAX_TOP; ++t) hits[t] += (t < n_top && r < tk.v[t]);
        mr += (double)(r + 1);
        mrr += 1.0 / (double)(r + 1);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int t = 0; t < STATS_MAX_TOP; ++t) hits[t] += __shfl_xor_sync(OEA_FULL, hits[t], o);
        mr += __shfl_xor_sync(OEA_FULL, mr, o);
        mrr += __shfl_xor_sync(OEA_FULL, mrr, o);
    }
    if (lane == 0) {
#pragma unroll
        for (int t = 0; t < STATS_MAX_TOP; ++t) s_acc[warp][t] = (double)hits[t];
        s_acc[warp][STATS_MAX_TOP] = mr; s_acc[warp][STATS_MAX_TOP + 1] = mrr;
    }
    __syncthreads();
    if (threadIdx.x < STATS_MAX_TOP + 2) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += s_acc[w][threadIdx.x];
        const int slot = threadIdx.x < STATS_MAX_TOP ? threadIdx.x : n_top + (threadIdx.x - STATS_MAX_TOP);
        if (threadIdx.x >= STATS_MAX_TOP || threadIdx.x < n_top) atomicAdd(out + slot, t);
    }
}

}  // namespace oea

extern "C" size_t oea_matrix_topk_mean_workspace_bytes(int32_t n_rows, int32_t n_cols, int32_t k, int32_t by_column) {
    if (!by_column || n_rows <= 0 || n_cols <= 0 || k < 1 || k > KMAX) return 0;
    const int kcap = col_kcap(k), cpt = col_cpt(kcap);
    const int gy = col_grid_y(n_rows, n_cols, cpt);
    const size_t ldp = ((size_t)n_cols + 3) / 4 * 4;
    return (size_t)gy * CP_WARPS * kcap * ldp * sizeof(float);
}

extern "C" int oea_matrix_topk_mean(const float* mat, int64_t ld, int32_t n_rows, int32_t n_cols, int32_t k,
                                    int32_t by_column, float* out_mean, void* workspace, size_t workspace_bytes,
                                    void* stream) {
    if (!mat || !out_mean) return OEA_ERR_NULL;
    if (n_rows <= 0 || n_cols <= 0 || ld < n_cols || (ld & 3) || !aligned16(mat)) return OEA_ERR_SHAPE;
    if (k < 1 || k > KMAX || k > (by_column ? n_rows : n_cols)) return OEA_ERR_RANGE;
    cudaStream_t st = (cudaStream_t)stream;
    if (!by_column) {
        OEA_LAUNCH(k_mat_row_topk_mean, (n_rows + 7) / 8, 256, 0, st, mat, ld, n_rows, n_cols, k, out_mean);
        OEA_LAUNCH_CHECK();
        return OEA_OK;
    }
    const size_t need = oea_matrix_topk_mean_workspace_bytes(n_rows, n_cols, k, 1);
    if (!workspace || workspace_bytes < need || !aligned16(workspace)) return OEA_ERR_WORKSPACE;
    const int kcap = col_kcap(k), cpt = col_cpt(kcap);
    const int gy = col_grid_y(n_rows, n_cols, cpt);
    const int n_splits = gy * CP_WARPS;
    const int rows_per_split = (n_rows + n_splits - 1) / n_splits;
    const long long ldp = ((long long)n_cols + 3) / 4 * 4;
    float* part = (float*)workspace;
    const dim3 grid((n_cols + 32 * cpt - 1) / (32 * cpt), gy);
#define OEA_COL_LAUNCH(KC, CP)                                                                                         \
    do {                                                                                                               \
        OEA_LAUNCH((k_mat_col_topk_partial<KC, CP>), grid, CP_WARPS * 32, 0, st, mat, ld, n_rows, n_cols, rows_per_split, part, ldp); \
        OEA_LAUNCH(k_col_partial_merge<KC>, (n_cols + 31) / 32, 256, 0, st, part, ldp, n_cols, n_splits, k, out_mean);        \
    } while (0)
    switch (kcap) {
        case 4: OEA_COL_LAUNCH(4, 4); break;
        case 8: OEA_COL_LAUNCH(8, 4); break;
        case 10: OEA_COL_LAUNCH(10, 4); break;
        case 16: OEA_COL_LAUNCH(16, 4); break;
        default: OEA_COL_LAUNCH(32, 2); break;
    }
#undef OEA_COL_LAUNCH
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_rank_stats(const int32_t* rank, int32_t n, const int32_t* top_k_host, int32_t n_top, double* out,
                              void* stream) {
    if (!rank || !out || (n_top > 0 && !top_k_host)) return OEA_ERR_NULL;
    if (n <= 0 || n_top < 0 || n_top > STATS_MAX_TOP) return OEA_ERR_RANGE;
    TopKs tk{};
    for (int i = 0; i < n_top; ++i) tk.v[i] = top_k_host[i];
    cudaStream_t st = (cudaStream_t)stream;
    OEA_CUDA_TRY(cudaMemsetAsync(out, 0, (size_t)(n_top + 2) * sizeof(double), st));
    int blocks = (n + 255) / 256;
    if (blocks > 2 * sm_count()) blocks = 2 * sm_count();
    OEA_LAUNCH(k_rank_stats, blocks, 256, 0, st, rank, n, tk, n_top, out);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_matrix_rank(const float* mat, int64_t ld, int32_t n_rows, int32_t n_cols, const float* row_off,
                               const float* col_off, const int32_t* gold, int32_t* out_top1, int32_t* out_rank, void* stream) {
    if (!mat || !gold || !out_top1 || !out_rank) return OEA_ERR_NULL;
    if ((row_off == nullptr) != (col_off == nullptr)) return OEA_ERR_NULL;
    if (n_rows <= 0 || n_cols <= 0 || ld < n_cols) return OEA_ERR_SHAPE;
    OEA_LAUNCH(k_mat_rank, (n_rows + 7) / 8, 256, 0, (cudaStream_t)stream, mat, ld, n_rows, n_cols, row_off, col_off, gold, out_top1, out_rank);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}
