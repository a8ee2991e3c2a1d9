// oea_rowmath.cuh — embedding-row arithmetic shared by the path-(i) kernels (oea_triple.cu, oea_triple_ext.cu):
// a row of `dim` floats held as VEC float4 per lane of one warp, TF's l2_normalize and its Jacobian, the score and
// loss functions of modules/base/losses.py, the per-block loss accumulator, and the host-side table checks / grid
// sizing.  sm_90a.
#pragma once
#include "oea_common.cuh"

namespace oea {

constexpr int kWarpsPerBlock = 8;
constexpr int kThreads = kWarpsPerBlock * OEA_WARP;
constexpr float kNormEps = 1e-12f;  // tf.nn.l2_normalize epsilon

template <int VEC>
struct Row {
    float4 v[VEC];
};

template <int VEC>
__device__ __forceinline__ Row<VEC> load_row(const float* __restrict__ base, int row, int pitch, int lane) {
    Row<VEC> r;
    const float* p = base + (size_t)row * pitch;
    const int p4 = pitch >> 2;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        const int c = lane + i * OEA_WARP;
        r.v[i] = (c < p4) ? ldg4(p + 4 * c) : f4(0.f);
    }
    return r;
}

template <int VEC>
__device__ __forceinline__ void red_row(float* __restrict__ base, int row, int pitch, int lane, const Row<VEC>& g) {
    float* p = base + (size_t)row * pitch;
    const int p4 = pitch >> 2;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        const int c = lane + i * OEA_WARP;
        if (c < p4) red_add4(p + 4 * c, g.v[i]);
    }
}

template <int VEC>
__device__ __forceinline__ float sumsq(const Row<VEC>& a) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) s += dot4(a.v[i], a.v[i]);
    return s;
}
template <int VEC>
__device__ __forceinline__ float dotr(const Row<VEC>& a, const Row<VEC>& b) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) s += dot4(a.v[i], b.v[i]);
    return s;
}

// inverse norm as tf.nn.l2_normalize: rsqrt(max(Σx², 1e-12)); 1 when the table is not normalised.
__device__ __forceinline__ float inv_norm(float ss, bool on) { return on ? rsqrtf(fmaxf(ss, kNormEps)) : 1.f; }

// Gradient w.r.t. the raw row given the gradient w.r.t. the normalised row (ghat), the normalised
// row xhat, <xhat, ghat> (dot) and 1/||x||.  When Σx² < eps TF's max() picks eps and the Jacobian
// is just the scale.
template <int VEC>
__device__ __forceinline__ Row<VEC> through_norm(const Row<VEC>& ghat, const Row<VEC>& xhat, float dot, float inv,
                                                 float ss, bool on) {
    Row<VEC> g;
    const float proj = (on && ss >= kNormEps) ? dot : 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) g.v[i] = fma4(xhat.v[i], -proj, ghat.v[i]) * inv;
    return g;
}

template <int SCORE, int VEC>
__device__ __forceinline__ float score_partial(const Row<VEC>& u) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) s += (SCORE == OEA_SCORE_L1) ? abs_sum4(u.v[i]) : dot4(u.v[i], u.v[i]);
    return s;
}
// d score / d u
template <int SCORE, int VEC>
__device__ __forceinline__ Row<VEC> score_dir(const Row<VEC>& u) {
    Row<VEC> d;
#pragma unroll
    for (int i = 0; i < VEC; ++i) d.v[i] = (SCORE == OEA_SCORE_L1) ? sgn4(u.v[i]) : u.v[i] * 2.f;
    return d;
}

// Per-triple loss value and d(loss)/d(score).  TF conventions: relu'(0) = 0.
__device__ __forceinline__ void loss_of(int loss_kind, bool is_neg, float s, const oea_loss_cfg& c, float& L, float& g) {
    switch (loss_kind) {
        case OEA_LOSS_LIMITED:
            if (!is_neg) { L = fmaxf(s - c.margin, 0.f); g = (s > c.margin) ? 1.f : 0.f; }
            else { L = c.balance * fmaxf(c.neg_margin - s, 0.f); g = (s < c.neg_margin) ? -c.balance : 0.f; }
            break;
        case OEA_LOSS_LOGISTIC:
            if (!is_neg) { L = softplus(s); g = 1.f / (1.f + expf(-s)); }
            else { L = softplus(-s); g = -1.f / (1.f + expf(s)); }
            break;
        case OEA_LOSS_LOGSIGMOID:  // −log σ(−s) = softplus(s)
            L = softplus(s); g = 1.f / (1.f + expf(-s));
            break;
        default:  // OEA_LOSS_POSITIVE
            L = s; g = 1.f;
            break;
    }
}

// Block-level loss accumulation: per-warp partials → one fp64 atomic per block.
struct LossAcc {
    double* smem;  // [kWarpsPerBlock]
    __device__ __forceinline__ void flush(float warp_loss, double* out, int n_warps_block = kWarpsPerBlock) {
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        if (lane == 0) smem[warp] = (double)warp_loss;
        __syncthreads();
        if (threadIdx.x == 0) {
            double t = 0.0;
            for (int i = 0; i < n_warps_block; ++i) t += smem[i];
            if (t != 0.0) atomicAdd(out, t);
        }
    }
};

struct TableDev {
    const float* w;
    float* g;
    int32_t* touched;
    int pitch;
    bool norm;
};

__host__ inline TableDev table_dev(const oea_table* t) {
    TableDev d;
    d.w = t->weight; d.g = t->grad; d.touched = t->touched; d.pitch = t->pitch; d.norm = t->l2_norm != 0;
    return d;
}

// ---- host-side validation + dispatch -----------------------------------------------------------
inline int check_table(const oea_table* t, bool need_grad) {
    if (t == nullptr || t->weight == nullptr) return OEA_ERR_NULL;
    if (need_grad && (t->grad == nullptr || t->touched == nullptr)) return OEA_ERR_NULL;
    if (t->rows <= 0 || t->dim <= 0 || t->pitch < t->dim || (t->pitch & 3) != 0) return OEA_ERR_DIM;
    if (t->pitch > 512) return OEA_ERR_DIM;
    if (!aligned16(t->weight) || (need_grad && !aligned16(t->grad))) return OEA_ERR_ALIGN;
    return OEA_OK;
}

inline int sm_count_cached() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) sms = 132;
    }
    return sms;
}

inline int grid_for(int n_warp_items) {
    const int blocks_needed = (n_warp_items + kWarpsPerBlock - 1) / kWarpsPerBlock;
    const int cap = sm_count_cached() * 8;  // 8 CTAs × 8 warps = 64 resident warps per SM
    return blocks_needed < 1 ? 1 : (blocks_needed < cap ? blocks_needed : cap);
}

// Exactly one resident wave for kernel `fn` (grid-stride loops do the rest): a partial last wave would run at a
// fraction of the machine for a whole block duration.
template <typename Fn>
static int grid_one_wave(Fn fn, int n_warp_items, int warps_per_block = kWarpsPerBlock) {
    static int occ = 0;   // one static per kernel instantiation
    if (occ == 0 && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, warps_per_block * OEA_WARP, 0) != cudaSuccess || occ < 1)) occ = 1;
    const int blocks_needed = (n_warp_items + warps_per_block - 1) / warps_per_block;
    const int cap = sm_count_cached() * occ;
    return blocks_needed < 1 ? 1 : (blocks_needed < cap ? blocks_needed : cap);
}

#define OEA_DISPATCH_VEC(pitch, CALL)                 \
    do {                                              \
        if ((pitch) <= 128) { CALL(1); }              \
        else if ((pitch) <= 256) { CALL(2); }         \
        else if ((pitch) <= 384) { CALL(3); }         \
        else { CALL(4); }                             \
    } while (0)

}  // namespace oea
