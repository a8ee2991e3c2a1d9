// oea_spmm.cu — path (ii): sparse-adjacency × dense-embedding neighbour aggregation (K2) and the
// L1 margin alignment loss of the GNN approaches.  sm_90a.
//
// Restates (no code shared):
//   approaches/gcn_align.py:79-86,239-267   dot(sparse) = tf.sparse_tensor_dense_matmul ; GraphConvolution
//   approaches/gcn_align.py:298-320         align_loss (L1 margin over seed pairs, k negatives per side)
//   approaches/rdgcn.py:293-315             get_loss (same shape, k negatives per side)
//
// SpMM Y = A·X with A in CSR (int32 col, fp32 val): HBM/L2-bound gather of X rows.  Rows with at most
// LONG_ROW non-zeros are handled one warp per row (col/val fetched 32 at a time, coalesced, and
// broadcast by shuffle; the X row is read with 128-bit loads); hub rows (Zipf degree) get a whole CTA
// cut into 512-non-zero segments (one CTA each) whose partial rows are added in order — no atomics, deterministic.
#include <climits>

#include "oea_common.cuh"

namespace oea {

constexpr int SPMM_WARPS = 8;
constexpr int SPMM_THREADS = SPMM_WARPS * 32;
constexpr int LONG_ROW = 256;

template <int VEC>
struct Acc {
    float4 v[VEC];
};

template <int VEC>
__device__ __forceinline__ void acc_zero(Acc<VEC>& a) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) a.v[i] = f4(0.f);
}

// accumulate val·X[col, :] over the non-zeros [p0, p1) of one row into acc (lane owns float4 columns lane+32i).
// The non-zeros are taken U at a time: U independent row gathers are issued before the first FMA, so a row's
// latency is one round trip per U non-zeros instead of one per non-zero.
template <int VEC>
__device__ __forceinline__ void spmm_span(const int32_t* __restrict__ col, const float* __restrict__ val,
                                          int p0, int p1, const float* __restrict__ X, int ldx, int d4, int lane,
                                          Acc<VEC>& acc) {
    constexpr int U = VEC <= 1 ? 8 : (VEC == 2 ? 4 : 2);
    for (int base = p0; base < p1; base += 32) {
        const int p = base + lane;
        int c = 0; float w = 0.f;
        if (p < p1) { c = __ldg(col + p); w = __ldg(val + p); }   // lanes past the end contribute 0·X[0]
        const int cnt = min(32, p1 - base);
        for (int j0 = 0; j0 < cnt; j0 += U) {
            float4 x[U][VEC];
            float wj[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const bool on = j0 + u < cnt;                       // warp-uniform
                const int cj = __shfl_sync(OEA_FULL, c, (j0 + u) & 31);
                const float ws = __shfl_sync(OEA_FULL, w, (j0 + u) & 31);
                wj[u] = on ? ws : 0.f;
                const float* xr = X + (size_t)cj * ldx;
#pragma unroll
                for (int i = 0; i < VEC; ++i) {
                    const int q = lane + 32 * i;
                    x[u][i] = (on && q < d4) ? ldg4(xr + 4 * q) : f4(0.f);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u)
#pragma unroll
                for (int i = 0; i < VEC; ++i) acc.v[i] = fma4(x[u][i], wj[u], acc.v[i]);
        }
    }
}

struct SpmmEpi {
    int relu;                 // y = max(y, 0)
    const float* mask_src;    // y = mask_src[row, c] > 0 ? y : 0   (relu backward), same ld as Y
    float beta;               // y += beta · Y_old
};

template <int VEC>
__device__ __forceinline__ void spmm_store(const Acc<VEC>& acc, float* __restrict__ Y, int ldy, int row, int d4, int lane,
                                           const SpmmEpi& e) {
    float* yr = Y + (size_t)row * ldy;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        const int q = lane + 32 * i;
        if (q >= d4) continue;
        float4 v = acc.v[i];
        if (e.beta != 0.f) { const float4 o = *reinterpret_cast<const float4*>(yr + 4 * q); v = fma4(o, e.beta, v); }
        if (e.relu) v = make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
        if (e.mask_src) {
            const float4 m = ldg4(e.mask_src + (size_t)row * ldy + 4 * q);
            v = make_float4(m.x > 0.f ? v.x : 0.f, m.y > 0.f ? v.y : 0.f, m.z > 0.f ? v.z : 0.f, m.w > 0.f ? v.w : 0.f);
        }
        *reinterpret_cast<float4*>(yr + 4 * q) = v;
    }
}

template <int VEC>
__global__ void __launch_bounds__(SPMM_THREADS)
k_spmm_warp_rows(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col, const float* __restrict__ val,
                 int n_rows, int max_len, const float* __restrict__ X, int ldx, float* __restrict__ Y, int ldy, int d4,
                 SpmmEpi epi) {
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * SPMM_WARPS + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * SPMM_WARPS;
    for (int row = warp_global; row < n_rows; row += n_warps) {
        const int p0 = __ldg(rowptr + row), p1 = __ldg(rowptr + row + 1);
        if (p1 - p0 > max_len) continue;    // hub row: k_spmm_segments + k_spmm_finalize
        Acc<VEC> acc;
        acc_zero(acc);
        spmm_span<VEC>(col, val, p0, p1, X, ldx, d4, lane, acc);
        spmm_store<VEC>(acc, Y, ldy, row, d4, lane, epi);
    }
}

// Hub rows (> LONG_ROW non-zeros) are cut into segments of SEG_NNZ non-zeros; one CTA per segment (8 warps ×
// SEG_NNZ/8 non-zeros, smem reduction) writes a partial row into the workspace, then one warp per hub row adds its
// partials IN ORDER and applies the epilogue — no atomics, deterministic, and the longest row no longer sets the
// kernel's critical path.
constexpr int SEG_NNZ = 512;

template <int VEC>
__global__ void __launch_bounds__(SPMM_THREADS)
k_spmm_segments(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col, const float* __restrict__ val,
                const int32_t* __restrict__ long_rows, const int32_t* __restrict__ seg_row, const int32_t* __restrict__ seg_start,
                int n_seg, const float* __restrict__ X, int ldx, float* __restrict__ partial, int ldp, int d4) {
    OEA_DYNAMIC_SMEM_ALIGNED16(red);               // [SPMM_WARPS][VEC*32] float4
    float4* red4 = reinterpret_cast<float4*>(red);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int sgi = blockIdx.x; sgi < n_seg; sgi += gridDim.x) {
        const int row = __ldg(long_rows + __ldg(seg_row + sgi));
        const int p_end = __ldg(rowptr + row + 1);
        const int s0 = __ldg(seg_start + sgi), s1 = min(p_end, s0 + SEG_NNZ);
        const int per = SEG_NNZ / SPMM_WARPS;
        const int a = min(s1, s0 + warp * per), b = min(s1, a + per);
        Acc<VEC> acc;
        acc_zero(acc);
        spmm_span<VEC>(col, val, a, b, X, ldx, d4, lane, acc);
#pragma unroll
        for (int i = 0; i < VEC; ++i) red4[(warp * VEC + i) * 32 + lane] = acc.v[i];
        __syncthreads();
        if (warp == 0) {
            float* pr = partial + (size_t)sgi * ldp;
#pragma unroll
            for (int i = 0; i < VEC; ++i) {
                float4 sum = red4[i * 32 + lane];
                for (int w = 1; w < SPMM_WARPS; ++w) sum = sum + red4[(w * VEC + i) * 32 + lane];
                const int q = lane + 32 * i;
                if (q < d4) *reinterpret_cast<float4*>(pr + 4 * q) = sum;
            }
        }
        __syncthreads();
    }
}

template <int VEC>
__global__ void __launch_bounds__(SPMM_THREADS)
k_spmm_finalize(const int32_t* __restrict__ long_rows, const int32_t* __restrict__ seg_ptr, int n_long,
                const float* __restrict__ partial, int ldp, float* __restrict__ Y, int ldy, int d4, SpmmEpi epi) {
    const int lane = threadIdx.x & 31;
    const int li = blockIdx.x * SPMM_WARPS + (threadIdx.x >> 5);
    if (li >= n_long) return;
    Acc<VEC> acc;
    acc_zero(acc);
    for (int sgi = __ldg(seg_ptr + li); sgi < __ldg(seg_ptr + li + 1); ++sgi) {
        const float* pr = partial + (size_t)sgi * ldp;
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
            const int q = lane + 32 * i;
            if (q < d4) acc.v[i] = acc.v[i] + *reinterpret_cast<const float4*>(pr + 4 * q);
        }
    }
    spmm_store<VEC>(acc, Y, ldy, __ldg(long_rows + li), d4, lane, epi);
}

// ------------------------------------------------------------------------------------------------
// L1 margin alignment loss (gcn_align.py:298-320 / rdgcn.py:293-315):
//   A_i = ‖x[l_i] − x[r_i]‖₁ ; for each of the 2k negatives (nl, nr) of i: relu(A_i + γ − ‖x[nl] − x[nr]‖₁)
//   loss = Σ / (2·k·t).  One warp per seed pair; gradients scatter-add into grad [N, ld] (pre-zeroed).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_align_loss_l1(const float* __restrict__ x, int ld, int dim, const int32_t* __restrict__ left, const int32_t* __restrict__ right,
                int t, int k, const int32_t* __restrict__ neg_left, const int32_t* __restrict__ neg_right,
                const int32_t* __restrict__ neg2_left, const int32_t* __restrict__ neg2_right, float gamma, float scale,
                double* __restrict__ loss_out, float* __restrict__ grad) {
    __shared__ double s_part[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int warp_global = blockIdx.x * 8 + warp, n_warps = gridDim.x * 8;
    float wloss = 0.f;
    for (int i = warp_global; i < t; i += n_warps) {
        const int l = __ldg(left + i), r = __ldg(right + i);
        const float* xl = x + (size_t)l * ld; const float* xr = x + (size_t)r * ld;
        float a = 0.f;
        for (int c = lane; c < dim; c += 32) a += fabsf(__ldg(xl + c) - __ldg(xr + c));
        a = warp_sum(a);
        const float dplus = a + gamma;
        int active = 0;
        for (int j = 0; j < 2 * k; ++j) {
            const int idx = i * k + (j < k ? j : j - k);
            const int nl = j < k ? __ldg(neg_left + idx) : __ldg(neg2_left + idx);
            const int nr = j < k ? __ldg(neg_right + idx) : __ldg(neg2_right + idx);
            const float* yl = x + (size_t)nl * ld; const float* yr = x + (size_t)nr * ld;
            float b = 0.f;
            for (int c = lane; c < dim; c += 32) b += fabsf(__ldg(yl + c) - __ldg(yr + c));
            b = warp_sum(b);
            const float v = dplus - b;
            if (v > 0.f) {
                wloss += v;
                ++active;
                for (int c = lane; c < dim; c += 32) {
                    const float s = sgn(__ldg(yl + c) - __ldg(yr + c)) * scale;
                    if (s != 0.f) { atomicAdd(grad + (size_t)nl * ld + c, -s); atomicAdd(grad + (size_t)nr * ld + c, s); }
                }
            }
        }
        if (active) {
            for (int c = lane; c < dim; c += 32) {
                const float s = sgn(__ldg(xl + c) - __ldg(xr + c)) * scale * (float)active;
                if (s != 0.f) { atomicAdd(grad + (size_t)l * ld + c, s); atomicAdd(grad + (size_t)r * ld + c, -s); }
            }
        }
    }
    if (lane == 0) s_part[warp] = (double)wloss;
    __syncthreads();
    if (threadIdx.x == 0) { double s = 0.0; for (int w = 0; w < 8; ++w) s += s_part[w]; if (s != 0.0) atomicAdd(loss_out, s * (double)scale); }
}

static int spmm_sm_count() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) sms = 132;
    }
    return sms;
}

}  // namespace oea

using namespace oea;

extern "C" size_t oea_spmm_workspace_bytes(int32_t n_segments, int32_t d) {
    return n_segments > 0 && d > 0 ? (size_t)n_segments * (size_t)d * sizeof(float) : 0;
}

extern "C" int oea_spmm_csr(const oea_csr* A, const oea_spmm_hubs* hubs,
                            const float* X, int32_t ldx, float* Y, int32_t ldy, int32_t d,
                            int32_t relu, const float* mask_src, float beta,
                            void* workspace, size_t workspace_bytes, void* stream) {
    if (!A || !A->rowptr || !X || !Y) return OEA_ERR_NULL;
    if (A->nnz > 0 && (!A->col || !A->val)) return OEA_ERR_NULL;
    if (A->n_rows <= 0 || d <= 0 || (d & 3) || d > 512 || ldx < d || ldy < d || (ldx & 3) || (ldy & 3)) return OEA_ERR_DIM;
    if (!aligned16(X) || !aligned16(Y) || (mask_src && !aligned16(mask_src))) return OEA_ERR_ALIGN;
    const int n_long = hubs ? hubs->n_long : 0, n_seg = hubs ? hubs->n_seg : 0;
    if (n_long < 0 || n_seg < n_long) return OEA_ERR_RANGE;
    if (n_long > 0) {
        if (!hubs->long_rows || !hubs->seg_ptr || !hubs->seg_row || !hubs->seg_start) return OEA_ERR_NULL;
        if (!workspace || workspace_bytes < oea_spmm_workspace_bytes(n_seg, d) || !aligned16(workspace)) return OEA_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    SpmmEpi epi{relu, mask_src, beta};
    const int d4 = d >> 2;
    // with a hub plan the warp-per-row kernel leaves rows of more than LONG_ROW non-zeros to the segment kernels;
    // without one it takes every row, so no row is left unwritten
    const int max_len = n_long > 0 ? LONG_ROW : INT_MAX;
    const int blocks = (A->n_rows + SPMM_WARPS - 1) / SPMM_WARPS;
    const int grid = blocks < spmm_sm_count() * 8 ? blocks : spmm_sm_count() * 8;
    float* partial = (float*)workspace;
#define OEA_SPMM(V)                                                                                                          \
    do {                                                                                                                     \
        OEA_LAUNCH(k_spmm_warp_rows<V>, grid, SPMM_THREADS, 0, st, A->rowptr, A->col, A->val, A->n_rows, max_len,      \
                   X, ldx, Y, ldy, d4, epi);                                                                                 \
        if (n_long > 0) {                                                                                                    \
            OEA_LAUNCH(k_spmm_segments<V>, n_seg, SPMM_THREADS, SPMM_WARPS * V * 32 * sizeof(float4), st,                    \
                A->rowptr, A->col, A->val, hubs->long_rows, hubs->seg_row, hubs->seg_start, n_seg, X, ldx, partial, d, d4);  \
            OEA_LAUNCH(k_spmm_finalize<V>, (n_long + SPMM_WARPS - 1) / SPMM_WARPS, SPMM_THREADS, 0, st,                      \
                hubs->long_rows, hubs->seg_ptr, n_long, partial, d, Y, ldy, d4, epi);                                        \
        }                                                                                                                    \
    } while (0)
    if (d <= 128) OEA_SPMM(1); else if (d <= 256) OEA_SPMM(2); else if (d <= 384) OEA_SPMM(3); else OEA_SPMM(4);
#undef OEA_SPMM
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_spmm_segment_nnz(void) { return SEG_NNZ; }

extern "C" int oea_spmm_long_row_threshold(void) { return LONG_ROW; }

extern "C" int oea_align_loss_l1(const float* x, int32_t ld, int32_t dim, const int32_t* left, const int32_t* right, int32_t t,
                                 int32_t k, const int32_t* neg_left, const int32_t* neg_right,
                                 const int32_t* neg2_left, const int32_t* neg2_right, float gamma,
                                 double* loss_out, float* grad, void* stream) {
    if (!x || !left || !right || !neg_left || !neg_right || !neg2_left || !neg2_right || !loss_out || !grad) return OEA_ERR_NULL;
    if (t <= 0 || k <= 0 || dim <= 0 || ld < dim) return OEA_ERR_SHAPE;
    const float scale = 1.0f / (2.0f * (float)k * (float)t);
    const int blocks = (t + 7) / 8;
    OEA_LAUNCH(k_align_loss_l1, blocks, 256, 0, (cudaStream_t)stream, x, ld, dim, left, right, t, k, neg_left, neg_right,
               neg2_left, neg2_right, gamma, scale, loss_out, grad);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

// ================================================================================================
// Edge-softmax attention over a sparse neighbourhood (AliNet's AliNetGraphAttentionLayer, alinet.py:656-677;
// RDGCN's add_sparse_att_layer has the same softmax-over-edges shape, rdgcn.py:202-215):
//   logit_ij = leaky_relu(a_ij·(s1_i + s2_j)) over the non-zeros (i, j) of the adjacency, alpha = row softmax,
//   out_i = Σ_j alpha_ij · M_j.
// Forward  = k_edge_softmax_fwd (alpha per edge) + oea_spmm_csr with alpha as the values.
// Backward = k_sddmm (d alpha_ij = <dOut_i, M_j>) + k_edge_softmax_bwd (softmax / leaky-relu Jacobians,
//            d s1 by rows, d s2 scattered by column) + oea_spmm_csr on the transposed pattern for d M.
// ================================================================================================
namespace oea {

__device__ __forceinline__ float leaky(float x, float slope) { return x > 0.f ? x : slope * x; }

// one warp per row: alpha[e] = softmax_row(leaky(a_e·(s1_i + s2_col(e))))
__global__ void __launch_bounds__(256)
k_edge_softmax_fwd(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col, const float* __restrict__ aval,
                   int n_rows, const float* __restrict__ s1, const float* __restrict__ s2, float slope,
                   float* __restrict__ alpha) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    const int p0 = __ldg(rowptr + row), p1 = __ldg(rowptr + row + 1);
    const bool node_mode = s1 != nullptr;     // else: aval[e] IS the pre-activation logit of edge e
    const float si = node_mode ? __ldg(s1 + row) : 0.f;
    float mx = -3.0e38f;
    for (int p = p0 + lane; p < p1; p += 32) {
        const float pre = node_mode ? __ldg(aval + p) * (si + __ldg(s2 + __ldg(col + p))) : __ldg(aval + p);
        const float l = leaky(pre, slope);
        alpha[p] = l;
        mx = fmaxf(mx, l);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(OEA_FULL, mx, o));
    float sum = 0.f;
    for (int p = p0 + lane; p < p1; p += 32) { const float e = __expf(alpha[p] - mx); alpha[p] = e; sum += e; }
    sum = warp_sum(sum);
    const float inv = sum > 0.f ? 1.f / sum : 0.f;
    for (int p = p0 + lane; p < p1; p += 32) alpha[p] *= inv;
}

// sampled dense-dense product on the sparsity pattern: out[e] = <G[row(e), :], M[col(e), :]>; warp per row
__global__ void __launch_bounds__(256)
k_sddmm(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col, int n_rows,
        const float* __restrict__ G, int ldg_, const float* __restrict__ M, int ldm, int d4, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    const int p0 = __ldg(rowptr + row), p1 = __ldg(rowptr + row + 1);
    const float* g = G + (size_t)row * ldg_;
    for (int p = p0; p < p1; ++p) {
        const float* m = M + (size_t)__ldg(col + p) * ldm;
        float acc = 0.f;
        for (int q = lane; q < d4; q += 32) acc += dot4(ldg4(g + 4 * q), ldg4(m + 4 * q));
        acc = warp_sum(acc);
        if (lane == 0) out[p] = acc;
    }
}

// softmax + leaky-relu backward per row; d s1[i] = Σ_e a_e·dlogit_e ; d s2[col(e)] += a_e·dlogit_e (atomics)
__global__ void __launch_bounds__(256)
k_edge_softmax_bwd(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col, const float* __restrict__ aval,
                   int n_rows, const float* __restrict__ s1, const float* __restrict__ s2, float slope,
                   const float* __restrict__ alpha, const float* __restrict__ dalpha,
                   float* __restrict__ ds1, float* __restrict__ ds2) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    const int p0 = __ldg(rowptr + row), p1 = __ldg(rowptr + row + 1);
    float dotp = 0.f;
    for (int p = p0 + lane; p < p1; p += 32) dotp += __ldg(alpha + p) * __ldg(dalpha + p);
    dotp = warp_sum(dotp);
    if (s1 == nullptr) {   // edge-logit mode: ds1 is a per-EDGE output [nnz] = d loss / d aval[e]
        for (int p = p0 + lane; p < p1; p += 32) {
            const float pre = __ldg(aval + p);
            ds1[p] = __ldg(alpha + p) * (__ldg(dalpha + p) - dotp) * (pre > 0.f ? 1.f : slope);
        }
        return;
    }
    const float si = __ldg(s1 + row);
    float acc1 = 0.f;
    for (int p = p0 + lane; p < p1; p += 32) {
        const int c = __ldg(col + p);
        const float a = __ldg(aval + p);
        const float pre = a * (si + __ldg(s2 + c));
        const float dl = __ldg(alpha + p) * (__ldg(dalpha + p) - dotp) * (pre > 0.f ? 1.f : slope) * a;
        acc1 += dl;
        if (dl != 0.f) atomicAdd(ds2 + c, dl);
    }
    acc1 = warp_sum(acc1);
    if (lane == 0) ds1[row] = acc1;
}

}  // namespace oea

extern "C" int oea_edge_softmax_fwd(const oea_csr* A, const float* s1, const float* s2, float slope, float* alpha, void* stream) {
    if (!A || !A->rowptr || !alpha) return OEA_ERR_NULL;
    if ((s1 == nullptr) != (s2 == nullptr)) return OEA_ERR_NULL;     // both (node mode) or neither (edge-logit mode)
    if (A->nnz > 0 && (!A->col || !A->val)) return OEA_ERR_NULL;
    if (A->n_rows <= 0) return OEA_ERR_DIM;
    OEA_LAUNCH(k_edge_softmax_fwd, (A->n_rows + 7) / 8, 256, 0, (cudaStream_t)stream, A->rowptr, A->col, A->val, A->n_rows, s1, s2, slope, alpha);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_sddmm(const oea_csr* A, const float* G, int32_t ldg_, const float* M, int32_t ldm, int32_t d, float* out, void* stream) {
    if (!A || !A->rowptr || !G || !M || !out) return OEA_ERR_NULL;
    if (A->n_rows <= 0 || d <= 0 || (d & 3) || ldg_ < d || ldm < d || (ldg_ & 3) || (ldm & 3)) return OEA_ERR_DIM;
    if (!aligned16(G) || !aligned16(M)) return OEA_ERR_ALIGN;
    OEA_LAUNCH(k_sddmm, (A->n_rows + 7) / 8, 256, 0, (cudaStream_t)stream, A->rowptr, A->col, A->n_rows, G, ldg_, M, ldm, d >> 2, out);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_edge_softmax_bwd(const oea_csr* A, const float* s1, const float* s2, float slope, const float* alpha,
                                    const float* dalpha, float* ds1, float* ds2, void* stream) {
    if (!A || !A->rowptr || !alpha || !dalpha || !ds1) return OEA_ERR_NULL;
    if ((s1 == nullptr) != (s2 == nullptr) || (s1 != nullptr && !ds2)) return OEA_ERR_NULL;
    if (A->n_rows <= 0) return OEA_ERR_DIM;
    OEA_LAUNCH(k_edge_softmax_bwd, (A->n_rows + 7) / 8, 256, 0, (cudaStream_t)stream, A->rowptr, A->col, A->val, A->n_rows, s1, s2,
               slope, alpha, dalpha, ds1, ds2);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}
