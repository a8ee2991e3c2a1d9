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

// c ? a : b, field by field.  `const TableDev& t = c ? a : b` on kernel parameters takes their addresses, which puts
// both structs in a local-memory stack frame; choosing each field keeps the choice in registers.
__device__ __forceinline__ TableDev pick_table(bool c, const TableDev& a, const TableDev& b) {
    TableDev t;
    t.w = c ? a.w : b.w; t.g = c ? a.g : b.g; t.touched = c ? a.touched : b.touched;
    t.pitch = c ? a.pitch : b.pitch; t.norm = c ? a.norm : b.norm;
    return t;
}

// ---- whole-row arithmetic (oea_triple_ext.cu, oea_triple_transr.cu) ------------------------------------------
__device__ __forceinline__ float4 mul4(float4 a, float4 b) { return cat4(mul2(lo2(a), lo2(b)), mul2(hi2(a), hi2(b))); }

template <int VEC>
__device__ __forceinline__ Row<VEC> r_scale(const Row<VEC>& a, float s) {
    Row<VEC> o;
#pragma unroll
    for (int i = 0; i < VEC; ++i) o.v[i] = a.v[i] * s;
    return o;
}
template <int VEC>
__device__ __forceinline__ Row<VEC> r_add(const Row<VEC>& a, const Row<VEC>& b) {
    Row<VEC> o;
#pragma unroll
    for (int i = 0; i < VEC; ++i) o.v[i] = a.v[i] + b.v[i];
    return o;
}
template <int VEC>
__device__ __forceinline__ Row<VEC> r_sub(const Row<VEC>& a, const Row<VEC>& b) {
    Row<VEC> o;
#pragma unroll
    for (int i = 0; i < VEC; ++i) o.v[i] = a.v[i] - b.v[i];
    return o;
}
template <int VEC>
__device__ __forceinline__ Row<VEC> r_neg(const Row<VEC>& a) {
    Row<VEC> o;
#pragma unroll
    for (int i = 0; i < VEC; ++i) o.v[i] = neg(a.v[i]);
    return o;
}
// a·s + c
template <int VEC>
__device__ __forceinline__ Row<VEC> r_fma(const Row<VEC>& a, float s, const Row<VEC>& c) {
    Row<VEC> o;
#pragma unroll
    for (int i = 0; i < VEC; ++i) o.v[i] = fma4(a.v[i], s, c.v[i]);
    return o;
}
// element-wise product
template <int VEC>
__device__ __forceinline__ Row<VEC> r_mul(const Row<VEC>& a, const Row<VEC>& b) {
    Row<VEC> o;
#pragma unroll
    for (int i = 0; i < VEC; ++i) o.v[i] = mul4(a.v[i], b.v[i]);
    return o;
}

// A normalised row together with what the backward through l2_normalize needs.
template <int VEC>
struct NRow {
    Row<VEC> x;   // x·rsqrt(max(Σx², eps)) (or x itself when the normalisation is off)
    float inv;    // the scale that was applied
    float ss;     // Σx² of the un-normalised row
};

// tf.nn.embedding_lookup(init_embeddings(..., is_l2_norm), row)
template <int VEC>
__device__ __forceinline__ NRow<VEC> lookup(const TableDev& T, int row, int lane) {
    NRow<VEC> r;
    r.x = load_row<VEC>(T.w, row, T.pitch, lane);
    r.ss = warp_sum(sumsq(r.x));
    r.inv = inv_norm(r.ss, T.norm);
    r.x = r_scale(r.x, r.inv);
    return r;
}
// tf.nn.l2_normalize of a computed row
template <int VEC>
__device__ __forceinline__ NRow<VEC> normalised(const Row<VEC>& v) {
    NRow<VEC> r;
    r.ss = warp_sum(sumsq(v));
    r.inv = inv_norm(r.ss, true);
    r.x = r_scale(v, r.inv);
    return r;
}
// gradient w.r.t. the argument of normalised() given the gradient w.r.t. its result
template <int VEC>
__device__ __forceinline__ Row<VEC> back_normalised(const Row<VEC>& ghat, const NRow<VEC>& n) {
    const float dot = warp_sum(dotr(n.x, ghat));
    return through_norm(ghat, n.x, dot, n.inv, n.ss, true);
}
// gradient of a lookup(): through the table's normalisation, then one vector reduction into its gradient row
template <int VEC>
__device__ __forceinline__ void push(const TableDev& T, int row, int lane, const Row<VEC>& ghat, const NRow<VEC>& n) {
    const float dot = warp_sum(dotr(n.x, ghat));
    const Row<VEC> g = through_norm(ghat, n.x, dot, n.inv, n.ss, T.norm);
    red_row<VEC>(T.g, row, T.pitch, lane, g);
    if (lane == 0) T.touched[row] = 1;
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

// Exactly one resident wave for kernel `K` (grid-stride loops do the rest): a partial last wave would run at a
// fraction of the machine for a whole block duration.  The kernel is a template argument, not a parameter, so every
// kernel has its own cached occupancy: kernels with the same parameter list but different launch bounds (the duo and
// octet sampled steps) must not share one, or a cooperative launch could ask for more CTAs than can be co-resident.
template <auto K>
static int grid_one_wave(int n_warp_items, int warps_per_block = kWarpsPerBlock) {
    static int occ = 0;   // one static per kernel
    if (occ == 0 && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, K, warps_per_block * OEA_WARP, 0) != cudaSuccess || occ < 1)) occ = 1;
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
