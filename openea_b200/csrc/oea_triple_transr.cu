// oea_triple_transr.cu — path (i), TransR on the fed boundary: the triples of a step grouped by relation, so that every
// relation's d×d matrix is read once and its gradient reduced once per chunk of triples.  sm_90a.
//
// Maths restated from the reference (no code shared):
//   models/trans/transr.py:14-52   h' = l2_normalize(M_r·ĥ), t' = l2_normalize(M_r·t̂) (unconditionally), the loss of
//                                  get_loss_func on (h', r̂, t'); rel_matrix [R, d·d] is never normalised
//   modules/base/losses.py:15-73   margin / limited / logistic / positive losses (sums)
// ĥ, t̂ and r̂ go through tf.nn.l2_normalize when their table has l2_norm, as every other lookup of path (i).
//
// Layout: the matrix table is an ordinary oea_table of R·d rows of width d; row r·d + i is row i of M_r.  Its gradient
// rows are flagged like any other table's, so oea_rowopt_apply is TF's sparse update of the relation's d² entries.
//
// One call = a memset and seven kernels on `stream`, no allocation, no host synchronisation:
//   1. memset + k_transr_count   histogram of the n_pos + n_neg scored triples by relation, with an arrival ticket each
//   2. k_transr_plan             (one CTA) exclusive scan of the histogram; the work list of chunks (relation, first,
//                                count ≤ C): a relation with more than C triples in the step is split, as the hub segments
//                                of k_spmm_segments are.  The chunk count stays on the device.
//   3. k_transr_scatter          bucket by ticket, then k_transr_stable: each triple's rank among the ids of its bucket, so
//                                that a bucket lists its triples in input order (a stable counting sort) whatever order the
//                                tickets were drawn in.  That pass costs Σ_r count_r² comparisons (L1-resident reads).
//   4. k_transr_fwd<SCORE>       one CTA per chunk: M_r staged once in shared memory, the chunk's ĥ / t̂ gathered with
//                                128-bit loads, P = X·M_rᵀ as a register-tiled FP32 GEMM (no TF32), then per triple the
//                                projections' l2_normalize and the L1 / L2² score.  The raw projections go to the workspace:
//                                the backward reads them back instead of recomputing 4·d² FLOP per triple.
//   5. k_transr_loss             dL/dE of every triple once every score exists (a margin pair's two triples may sit in
//                                different chunks: a fed negative need not share its positive's relation).
//   6. k_transr_bwd<SCORE>       one CTA per chunk again: the score gradient through the projections' normalisation
//                                (G), dM_r = Σ_j G_jᵀ·X_j as the chunk's GEMM, pushed once per chunk into the d gradient rows
//                                of M_r with red.global.add.v4.f32; dX = G·M_r through the entity normalisation into
//                                ent.grad; the relation row's gradient summed over the chunk and pushed once.
//
// Shared memory rows have a stride of pitch + 1 floats (odd), so that a GEMM operand read along either axis by the 16
// threads of a half-warp hits 16 distinct banks.  Thread tile: 16 × 16 threads, 8 × 8 outputs each (rows m = ty + 16a,
// columns n = tx + 16b), which covers the 2·C = 128 rows of a chunk and the ≤ 128 columns of a row.
#include "oea_rowmath.cuh"

namespace oea {

constexpr int kTransrChunk = 64;                        // C: triples per chunk
constexpr int kTransrRows = 2 * kTransrChunk;           // rows of a tile: the chunk's ĥ then its t̂
constexpr int kTransrMaxPitch = 128;

struct TransrWs {
    size_t hist, offs, ticket, tmp, order, chunks, n_chunks, energy, dloss, proj, total;
};

// workspace sections, each 256-B aligned: per relation [hist | offs], per scored triple [ticket | tmp | order | E | dL/dE],
// the chunk list, and the raw projections M_r·ĥ (rows 0 … N−1, by sorted position) and M_r·t̂ (rows N … 2N−1)
static TransrWs transr_layout(int n_pos, int n_neg, int pitch, int n_rel) {
    const size_t n = (size_t)n_pos + (size_t)n_neg;
    const size_t max_chunks = (n + kTransrChunk - 1) / kTransrChunk + (n < (size_t)n_rel ? n : (size_t)n_rel);
    TransrWs w;
    size_t at = 0;
    auto take = [&](size_t bytes) { const size_t o = at; at += (bytes + 255) & ~(size_t)255; return o; };
    w.hist = take(4 * (size_t)n_rel);
    w.offs = take(4 * (size_t)n_rel);
    w.ticket = take(4 * n);
    w.tmp = take(4 * n);
    w.order = take(4 * n);
    w.chunks = take(16 * max_chunks);
    w.n_chunks = take(4);
    w.energy = take(4 * n);
    w.dloss = take(4 * n);
    w.proj = take(4 * 2 * n * (size_t)pitch);
    w.total = at;
    return w;
}

struct TransrBatch {
    const int32_t *ph, *pr, *pt, *nh, *nr, *nt;
    int n_pos, n_neg;
    __device__ __forceinline__ int rel(int i) const { return i < n_pos ? __ldg(pr + i) : __ldg(nr + i - n_pos); }
    __device__ __forceinline__ int head(int i) const { return i < n_pos ? __ldg(ph + i) : __ldg(nh + i - n_pos); }
    __device__ __forceinline__ int tail(int i) const { return i < n_pos ? __ldg(pt + i) : __ldg(nt + i - n_pos); }
};

// ---- bucketing -----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_transr_count(TransrBatch B, int32_t* __restrict__ hist, int32_t* __restrict__ ticket) {
    const int n = B.n_pos + B.n_neg;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        ticket[i] = atomicAdd(hist + B.rel(i), 1);
}

// one CTA: offsets and the chunk list.  (count, chunks) of a relation are scanned together as one 64-bit word.
__global__ void __launch_bounds__(kThreads)
k_transr_plan(const int32_t* __restrict__ hist, int n_rel, int32_t* __restrict__ offs, int4* __restrict__ chunks,
              int32_t* __restrict__ n_chunks) {
    __shared__ unsigned long long s_warp[kWarpsPerBlock];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long carry = 0;
    for (int base = 0; base < n_rel; base += kThreads) {
        const int r = base + threadIdx.x;
        const int c = r < n_rel ? hist[r] : 0;
        const int nch = (c + kTransrChunk - 1) / kTransrChunk;
        const unsigned long long mine = ((unsigned long long)nch << 32) | (unsigned)c;
        unsigned long long inc = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long v = __shfl_up_sync(OEA_FULL, inc, o);
            if (lane >= o) inc += v;
        }
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        unsigned long long before = carry, total = 0;
        for (int w = 0; w < kWarpsPerBlock; ++w) {
            if (w < warp) before += s_warp[w];
            total += s_warp[w];
        }
        const unsigned long long excl = before + inc - mine;
        if (r < n_rel) {
            const int off = (int)(excl & 0xffffffffu), ch0 = (int)(excl >> 32);
            offs[r] = off;
            for (int j = 0; j < nch; ++j) {
                const int first = j * kTransrChunk;
                chunks[ch0 + j] = make_int4(r, off + first, min(kTransrChunk, c - first), 0);
            }
        }
        carry += total;
        __syncthreads();                                  // s_warp is reused by the next tile
    }
    if (threadIdx.x == 0) *n_chunks = (int32_t)(carry >> 32);
}

__global__ void __launch_bounds__(kThreads)
k_transr_scatter(TransrBatch B, const int32_t* __restrict__ offs, const int32_t* __restrict__ ticket,
                 int32_t* __restrict__ tmp) {
    const int n = B.n_pos + B.n_neg;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        tmp[offs[B.rel(i)] + ticket[i]] = i;
}

// the bucket of relation r holds its triples in input order: position = offs[r] + #{ids of the bucket below mine}
__global__ void __launch_bounds__(kThreads)
k_transr_stable(TransrBatch B, const int32_t* __restrict__ hist, const int32_t* __restrict__ offs,
                const int32_t* __restrict__ tmp, int32_t* __restrict__ order) {
    const int n = B.n_pos + B.n_neg;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
        const int v = __ldg(tmp + p);
        const int r = B.rel(v);
        const int lo = __ldg(offs + r), hi = lo + __ldg(hist + r);
        int rank = 0;
        for (int q = lo; q < hi; ++q) rank += __ldg(tmp + q) < v;
        order[lo + rank] = v;
    }
}

// ---- the chunk's tiles in shared memory ----------------------------------------------------------------------------
// C[m][n] = Σ_{k<K} A(m, k)·B(k, n) for this thread's 8 × 8 outputs m = ty + 16a, n = tx + 16b.  A(m, k) = A[m·sam + k·sak],
// B(k, n) = B[k·sbk + n·sbn]: the 16 threads of a half-warp share ty (one broadcast address of A) and read 16 consecutive
// n of B, at stride 1 or pitch + 1 — conflict-free either way.  FP32 FFMA only.
__device__ __forceinline__ void tile_gemm(float (&acc)[8][8], const float* A, int sam, int sak, const float* Bm, int sbk,
                                          int sbn, int K, int ty, int tx) {
#pragma unroll
    for (int a = 0; a < 8; ++a)
#pragma unroll
        for (int b = 0; b < 8; ++b) acc[a][b] = 0.f;
    const float* pa = A + ty * sam;
    const float* pb = Bm + tx * sbn;
    for (int k = 0; k < K; ++k) {
        float av[8], bv[8];
#pragma unroll
        for (int a = 0; a < 8; ++a) av[a] = pa[16 * a * sam];
#pragma unroll
        for (int b = 0; b < 8; ++b) bv[b] = pb[16 * b * sbn];
#pragma unroll
        for (int a = 0; a < 8; ++a)
#pragma unroll
            for (int b = 0; b < 8; ++b) acc[a][b] = fmaf(av[a], bv[b], acc[a][b]);
        pa += sak;
        pb += sbk;
    }
}

// the valid outputs (m < m_n, n < n_n) of a tile_gemm into a shared tile of row stride ld
__device__ __forceinline__ void tile_store(const float (&acc)[8][8], float* S, int ld, int m_n, int n_n, int ty, int tx) {
#pragma unroll
    for (int a = 0; a < 8; ++a)
#pragma unroll
        for (int b = 0; b < 8; ++b) {
            const int m = ty + 16 * a, n = tx + 16 * b;
            if (m < m_n && n < n_n) S[m * ld + n] = acc[a][b];
        }
}

// a row of ≤ 128 columns between a warp's registers (Row<1>: lane l holds columns 4l … 4l+3) and a shared tile row;
// columns at or past `dim` read as 0
__device__ __forceinline__ void st_row(float* s, const Row<1>& x, int dim, int lane) {
    const int c = 4 * lane;
    if (c < dim) s[c] = x.v[0].x;
    if (c + 1 < dim) s[c + 1] = x.v[0].y;
    if (c + 2 < dim) s[c + 2] = x.v[0].z;
    if (c + 3 < dim) s[c + 3] = x.v[0].w;
}
__device__ __forceinline__ Row<1> ld_row(const float* s, int dim, int lane) {
    const int c = 4 * lane;
    Row<1> x;
    x.v[0] = make_float4(c < dim ? s[c] : 0.f, c + 1 < dim ? s[c + 1] : 0.f, c + 2 < dim ? s[c + 2] : 0.f,
                         c + 3 < dim ? s[c + 3] : 0.f);
    return x;
}

struct TransrDev {
    TableDev ent, rel, mat;
    int dim, pitch;
};

// M_r (rows r·d … r·d + d − 1 of the matrix table) into the shared tile Ms, row stride ld
__device__ __forceinline__ void stage_matrix(const TransrDev& T, int r, float* Ms, int ld) {
    const int p4 = T.pitch >> 2;
    const float* base = T.mat.w + (size_t)r * T.dim * T.pitch;
    for (int e = threadIdx.x; e < T.dim * p4; e += blockDim.x) {
        const int i = e / p4, q = e - i * p4;
        const float4 v = ldg4(base + (size_t)i * T.pitch + 4 * q);
        float* s = Ms + i * ld + 4 * q;
        s[0] = v.x; s[1] = v.y; s[2] = v.z; s[3] = v.w;
    }
}

// ---- forward: scores and raw projections ---------------------------------------------------------------------------
template <int SCORE>
__global__ void __launch_bounds__(kThreads)
k_transr_fwd(TransrDev T, TransrBatch B, const int4* __restrict__ chunks, const int32_t* __restrict__ n_chunks,
             const int32_t* __restrict__ order, float* __restrict__ energy, float* __restrict__ proj) {
    OEA_DYNAMIC_SMEM_ALIGNED16(smem);
    const int ld = T.pitch + 1, d = T.dim;
    float* Ms = smem;
    float* Xs = smem + kTransrRows * ld;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int n = B.n_pos + B.n_neg, nc = *n_chunks;
    for (int c = blockIdx.x; c < nc; c += gridDim.x) {
        const int4 ch = chunks[c];
        const int r = ch.x, first = ch.y, cnt = ch.z;
        __syncthreads();                                  // the previous chunk's readers of Ms / Xs are done
        stage_matrix(T, r, Ms, ld);
        for (int j = warp; j < cnt; j += kWarpsPerBlock) {
            const int id = __ldg(order + first + j);
            st_row(Xs + j * ld, lookup<1>(T.ent, B.head(id), lane).x, d, lane);
            st_row(Xs + (cnt + j) * ld, lookup<1>(T.ent, B.tail(id), lane).x, d, lane);
        }
        __syncthreads();
        float acc[8][8];
        tile_gemm(acc, Xs, ld, 1, Ms, 1, ld, d, ty, tx);          // P[j][i] = Σ_k X[j][k]·M[i][k]
        __syncthreads();                                  // every read of Xs is done: P replaces X
        tile_store(acc, Xs, ld, 2 * cnt, d, ty, tx);
        __syncthreads();
        const NRow<1> xr = lookup<1>(T.rel, r, lane);
        for (int j = warp; j < cnt; j += kWarpsPerBlock) {
            const int id = __ldg(order + first + j);
            const Row<1> ph = ld_row(Xs + j * ld, d, lane), pt = ld_row(Xs + (cnt + j) * ld, d, lane);
            if (4 * lane < T.pitch) {
                *reinterpret_cast<float4*>(proj + (size_t)(first + j) * T.pitch + 4 * lane) = ph.v[0];
                *reinterpret_cast<float4*>(proj + (size_t)(n + first + j) * T.pitch + 4 * lane) = pt.v[0];
            }
            const NRow<1> nh = normalised<1>(ph), nt = normalised<1>(pt);
            const Row<1> u = r_sub(r_add(nh.x, xr.x), nt.x);
            const float E = warp_sum(score_partial<SCORE, 1>(u));
            if (lane == 0) energy[id] = E;
        }
    }
}

// ---- loss: dL/dE per triple ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_transr_loss(const float* __restrict__ energy, float* __restrict__ dloss, int n_pos, int n_neg, oea_loss_cfg cfg,
              float scale, double* __restrict__ loss_out) {
    __shared__ double s_loss[kWarpsPerBlock];
    const bool margin = cfg.loss_kind == OEA_LOSS_MARGIN;
    const int items = margin ? n_pos : n_pos + n_neg;
    float acc = 0.f;
    for (int i0 = blockIdx.x * blockDim.x; i0 < items; i0 += gridDim.x * blockDim.x) {   // warp-uniform trip count
        const int i = i0 + threadIdx.x;
        if (i >= items) continue;
        if (margin) {                                     // relu(m + E⁺_i − E⁻_i), as k_model_margin
            const float v = cfg.margin + energy[i] - energy[n_pos + i];
            const float g = v > 0.f ? scale : 0.f;
            acc += fmaxf(v, 0.f) * scale;
            dloss[i] = g;
            dloss[n_pos + i] = -g;
        } else {
            float L, g;
            loss_of(cfg.loss_kind, i >= n_pos, energy[i], cfg, L, g);
            acc += L * scale;
            dloss[i] = g * scale;
        }
    }
    LossAcc lacc{s_loss};
    lacc.flush(warp_sum(acc), loss_out);
}

// ---- backward ----------------------------------------------------------------------------------------------------------
template <int SCORE>
__global__ void __launch_bounds__(kThreads)
k_transr_bwd(TransrDev T, TransrBatch B, const int4* __restrict__ chunks, const int32_t* __restrict__ n_chunks,
             const int32_t* __restrict__ order, const float* __restrict__ dloss, const float* __restrict__ proj) {
    OEA_DYNAMIC_SMEM_ALIGNED16(smem);
    __shared__ int s_any;
    const int ld = T.pitch + 1, d = T.dim;
    float* Ms = smem;
    float* Xs = Ms + kTransrRows * ld;
    float* Gs = Xs + kTransrRows * ld;
    float* s_gr = Gs + kTransrRows * ld;                  // [kWarpsPerBlock][kTransrMaxPitch]: the warps' relation gradients
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int n = B.n_pos + B.n_neg, nc = *n_chunks;
    for (int c = blockIdx.x; c < nc; c += gridDim.x) {
        const int4 ch = chunks[c];
        const int r = ch.x, first = ch.y, cnt = ch.z;
        __syncthreads();
        if (threadIdx.x == 0) s_any = 0;
        stage_matrix(T, r, Ms, ld);
        const NRow<1> xr = lookup<1>(T.rel, r, lane);
        Row<1> gr;
        gr.v[0] = f4(0.f);
        __syncthreads();
        // G: d loss / d (M_r·ĥ) and d loss / d (M_r·t̂) through the projections' l2_normalize; X: ĥ and t̂
        for (int j = warp; j < cnt; j += kWarpsPerBlock) {
            const int id = __ldg(order + first + j);
            const float g = __ldg(dloss + id);
            st_row(Xs + j * ld, lookup<1>(T.ent, B.head(id), lane).x, d, lane);
            st_row(Xs + (cnt + j) * ld, lookup<1>(T.ent, B.tail(id), lane).x, d, lane);
            Row<1> gh, gt;
            gh.v[0] = gt.v[0] = f4(0.f);
            if (g != 0.f) {
                const NRow<1> nh = normalised<1>(load_row<1>(proj, first + j, T.pitch, lane));
                const NRow<1> nt = normalised<1>(load_row<1>(proj, n + first + j, T.pitch, lane));
                const Row<1> du = r_scale(score_dir<SCORE, 1>(r_sub(r_add(nh.x, xr.x), nt.x)), g);
                gh = back_normalised<1>(du, nh);
                gt = back_normalised<1>(r_neg(du), nt);
                gr = r_add(gr, du);
                if (lane == 0) s_any = 1;
            }
            st_row(Gs + j * ld, gh, d, lane);
            st_row(Gs + (cnt + j) * ld, gt, d, lane);
        }
        st_row(s_gr + warp * kTransrMaxPitch, gr, T.pitch, lane);
        __syncthreads();
        if (!s_any) continue;                             // no active triple in the chunk: nothing to push (block-uniform)
        float acc[8][8];
        tile_gemm(acc, Gs, 1, ld, Xs, ld, 1, 2 * cnt, ty, tx);    // dM[i][k] = Σ_j G[j][i]·X[j][k]
        __syncthreads();                                  // X is read by nobody else: dM replaces it
        tile_store(acc, Xs, ld, d, d, ty, tx);
        tile_gemm(acc, Gs, ld, 1, Ms, ld, 1, d, ty, tx);          // dX[j][k] = Σ_i G[j][i]·M[i][k]
        __syncthreads();                                  // every read of Gs is done: dX replaces G
        tile_store(acc, Gs, ld, 2 * cnt, d, ty, tx);
        __syncthreads();
        // dM_r: one vector reduction per matrix row, once per chunk
        for (int i = warp; i < d; i += kWarpsPerBlock) {
            red_row<1>(T.mat.g, r * d + i, T.pitch, lane, ld_row(Xs + i * ld, d, lane));
            if (lane == 0) T.mat.touched[r * d + i] = 1;
        }
        // dĥ, dt̂ through the entity table's normalisation (the rows are gathered again for their norms)
        for (int j = warp; j < cnt; j += kWarpsPerBlock) {
            const int id = __ldg(order + first + j);
            if (__ldg(dloss + id) == 0.f) continue;
            const int h = B.head(id), t = B.tail(id);
            push<1>(T.ent, h, lane, ld_row(Gs + j * ld, d, lane), lookup<1>(T.ent, h, lane));
            push<1>(T.ent, t, lane, ld_row(Gs + (cnt + j) * ld, d, lane), lookup<1>(T.ent, t, lane));
        }
        // r̂: the chunk's sum through the relation table's normalisation
        if (warp == 0) {
            Row<1> sum;
            sum.v[0] = f4(0.f);
            for (int w = 0; w < kWarpsPerBlock; ++w) sum = r_add(sum, ld_row(s_gr + w * kTransrMaxPitch, T.pitch, lane));
            push<1>(T.rel, r, lane, sum, xr);
        }
    }
}

static int transr_smem_fwd(int pitch) { return 2 * kTransrRows * (pitch + 1) * (int)sizeof(float); }
static int transr_smem_bwd(int pitch) {
    return (3 * kTransrRows * (pitch + 1) + kWarpsPerBlock * kTransrMaxPitch) * (int)sizeof(float);
}

}  // namespace oea

using namespace oea;

extern "C" size_t oea_transr_workspace_bytes(int32_t n_pos, int32_t n_neg, int32_t dim, int32_t n_rel) {
    if (n_pos < 0 || n_neg < 0 || dim <= 0 || n_rel <= 0) return 0;
    return transr_layout(n_pos, n_neg, (dim + 3) / 4 * 4, n_rel).total;
}

extern "C" int oea_transr_score_fed(const oea_model* model,
                                    const int32_t* pos_h, const int32_t* pos_r, const int32_t* pos_t, int32_t n_pos,
                                    const int32_t* neg_h, const int32_t* neg_r, const int32_t* neg_t, int32_t n_neg,
                                    const oea_loss_cfg* loss, float loss_scale, void* workspace, size_t workspace_bytes,
                                    double* loss_out, void* stream) {
    if (model == nullptr) return OEA_ERR_NULL;
    if (model->kind != OEA_MODEL_TRANSR) return OEA_ERR_KIND;
    int rc = check_table(model->ent, true); if (rc) return rc;
    rc = check_table(model->rel, true); if (rc) return rc;
    rc = check_table(model->rel_aux, true); if (rc) return rc;
    const oea_table *ent = model->ent, *rel = model->rel, *mat = model->rel_aux;
    if (rel->dim != ent->dim || rel->pitch != ent->pitch || mat->pitch != ent->pitch) return OEA_ERR_DIM;
    if (ent->pitch > kTransrMaxPitch) return OEA_ERR_DIM;
    if (mat->dim != ent->dim || (int64_t)mat->rows != (int64_t)rel->rows * ent->dim) return OEA_ERR_SHAPE;
    if (!loss || !loss_out) return OEA_ERR_NULL;
    if (n_pos < 0 || n_neg < 0) return OEA_ERR_SHAPE;
    if (n_pos > 0 && (!pos_h || !pos_r || !pos_t)) return OEA_ERR_NULL;
    if (n_neg > 0 && (!neg_h || !neg_r || !neg_t)) return OEA_ERR_NULL;
    if (loss->loss_kind < OEA_LOSS_MARGIN || loss->loss_kind > OEA_LOSS_LOGSIGMOID) return OEA_ERR_KIND;
    if (loss->score_kind != OEA_SCORE_L1 && loss->score_kind != OEA_SCORE_L2SQ) return OEA_ERR_KIND;
    if (loss->loss_kind == OEA_LOSS_MARGIN && n_pos != n_neg) return OEA_ERR_SHAPE;
    const TransrWs w = transr_layout(n_pos, n_neg, ent->pitch, rel->rows);
    if (workspace == nullptr || workspace_bytes < w.total || !aligned16(workspace)) return OEA_ERR_WORKSPACE;
    const int n = n_pos + n_neg;
    if (n == 0) return OEA_OK;

    char* ws = static_cast<char*>(workspace);
    int32_t* hist = reinterpret_cast<int32_t*>(ws + w.hist);
    int32_t* offs = reinterpret_cast<int32_t*>(ws + w.offs);
    int32_t* ticket = reinterpret_cast<int32_t*>(ws + w.ticket);
    int32_t* tmp = reinterpret_cast<int32_t*>(ws + w.tmp);
    int32_t* order = reinterpret_cast<int32_t*>(ws + w.order);
    int4* chunks = reinterpret_cast<int4*>(ws + w.chunks);
    int32_t* n_chunks = reinterpret_cast<int32_t*>(ws + w.n_chunks);
    float* energy = reinterpret_cast<float*>(ws + w.energy);
    float* dloss = reinterpret_cast<float*>(ws + w.dloss);
    float* proj = reinterpret_cast<float*>(ws + w.proj);
    const TransrBatch B{pos_h, pos_r, pos_t, neg_h, neg_r, neg_t, n_pos, n_neg};
    TransrDev T;
    T.ent = table_dev(ent); T.rel = table_dev(rel); T.mat = table_dev(mat);
    T.mat.norm = false;                                   // rel_matrix is never normalised (transr.py:20-21)
    T.dim = ent->dim; T.pitch = ent->pitch;
    cudaStream_t st = (cudaStream_t)stream;
    const bool l1 = loss->score_kind == OEA_SCORE_L1;

    const int items_grid = grid_for((n + OEA_WARP - 1) / OEA_WARP);        // one thread per triple
    // ⌈n / C⌉ + min(R, n) chunks at most; the surplus CTAs see the device-side count and exit
    const int chunk_grid = (n + kTransrChunk - 1) / kTransrChunk + (n < rel->rows ? n : rel->rows);
    OEA_CUDA_TRY(cudaMemsetAsync(hist, 0, sizeof(int32_t) * (size_t)rel->rows, st));
    OEA_LAUNCH_STRIDED(k_transr_count, items_grid, kThreads, 0, st, B, hist, ticket);
    OEA_LAUNCH(k_transr_plan, 1, kThreads, 0, st, hist, rel->rows, offs, chunks, n_chunks);
    OEA_LAUNCH_STRIDED(k_transr_scatter, items_grid, kThreads, 0, st, B, offs, ticket, tmp);
    OEA_LAUNCH_STRIDED(k_transr_stable, items_grid, kThreads, 0, st, B, hist, offs, tmp, order);
    OEA_LAUNCH_CHECK();

    const int smem_f = transr_smem_fwd(T.pitch), smem_b = transr_smem_bwd(T.pitch);
    auto fwd = l1 ? k_transr_fwd<OEA_SCORE_L1> : k_transr_fwd<OEA_SCORE_L2SQ>;
    auto bwd = l1 ? k_transr_bwd<OEA_SCORE_L1> : k_transr_bwd<OEA_SCORE_L2SQ>;
    OEA_CUDA_TRY(cudaFuncSetAttribute(fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_f));
    OEA_CUDA_TRY(cudaFuncSetAttribute(bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_b));
    OEA_LAUNCH_STRIDED(fwd, chunk_grid, kThreads, smem_f, st, T, B, chunks, n_chunks, order, energy, proj);
    OEA_LAUNCH_STRIDED(k_transr_loss, items_grid, kThreads, 0, st, energy, dloss, n_pos, n_neg, *loss, loss_scale, loss_out);
    OEA_LAUNCH_STRIDED(bwd, chunk_grid, kThreads, smem_b, st, T, B, chunks, n_chunks, order, dloss, proj);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}
