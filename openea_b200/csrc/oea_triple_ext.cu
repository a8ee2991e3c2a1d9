// oea_triple_ext.cu — path (i), SURVEY §8f-2: the other score functions of the reference's models/ on the
// fed boundary (index vectors in, gradients scattered into the tables), one warp per triple.  sm_90a.
//
// Maths restated from the reference (no code shared):
//   models/trans/transh.py:25-51        TransH   e⊥ = e − <e, n̂> n̂,  n̂ = l2_normalize(normal_vector[r])
//   approaches/bootea_transh.py:57-95   the same projection under the limited loss
//   models/trans/transd.py:26-65        TransD   e⊥ = l2_normalize(e + <e, e_p> r_p)
//   models/semantic/distmult.py:43-59   DistMult score Σ h∘r∘t, softplus(−label·score), reduce_mean
//   models/semantic/simple.py:50-86     SimplE   (Σ l2n(h_H∘r₁)∘t_T + Σ l2n(t_H∘r₂)∘h_T)/2, softplus(∓score)
//   modules/base/losses.py:15-73        margin / limited / logistic / positive losses (sums)
// Every table lookup goes through tf.nn.l2_normalize when the table was created with is_l2_norm
// (modules/base/initializers.py:26-50) and the gradient flows back through it into the raw variable.
//
// The similarity models are handled as energies E = −score so that the loss functions of oea_rowmath.cuh serve
// both families: logistic(E) = softplus(E⁺) + softplus(−E⁻) = softplus(−score⁺) + softplus(score⁻).
//
// Each triple is a Triple<MODEL> context: forward() gathers the 3–6 rows with 128-bit loads, normalises them and
// returns the energy; backward(g) pushes g·dE/d(row) through the projection and the normalisations and leaves
// through red.global.add.v4.f32 into the gradient tables.  tests/kernel_model_ext.py states the same arithmetic in
// NumPy and is checked against torch autograd on the CPU (tests/test_oracle_triple_ext.py).
#include "oea_rowmath.cuh"

namespace oea {

struct ModelDev {
    TableDev ent, rel, ent_aux, rel_aux;
};

// ---- whole-row arithmetic --------------------------------------------------------------------------------------
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

// ---- one triple of each model ------------------------------------------------------------------------------------
template <int MODEL, int SCORE, int VEC>
struct Triple;

// TransE (models/trans/transe.py:33-45): the family's base case; also cross-checks this file against oea_triple.cu
template <int SCORE, int VEC>
struct Triple<OEA_MODEL_TRANSE, SCORE, VEC> {
    int h, r, t;
    NRow<VEC> xh, xr, xt;
    Row<VEC> u;
    __device__ __forceinline__ float forward(const ModelDev& M, int h_, int r_, int t_, int lane) {
        h = h_; r = r_; t = t_;
        xh = lookup<VEC>(M.ent, h, lane);
        xr = lookup<VEC>(M.rel, r, lane);
        xt = lookup<VEC>(M.ent, t, lane);
        u = r_sub(r_add(xh.x, xr.x), xt.x);
        return warp_sum(score_partial<SCORE, VEC>(u));
    }
    __device__ __forceinline__ void backward(const ModelDev& M, float g, int lane) {
        const Row<VEC> du = r_scale(score_dir<SCORE, VEC>(u), g);
        push<VEC>(M.ent, h, lane, du, xh);
        push<VEC>(M.rel, r, lane, du, xr);
        push<VEC>(M.ent, t, lane, r_neg(du), xt);
    }
};

// TransH: u = ĥ + r̂ − t̂ − (a − b)·n̂ with a = <ĥ, n̂>, b = <t̂, n̂>; rel_aux = normal_vector
template <int SCORE, int VEC>
struct Triple<OEA_MODEL_TRANSH, SCORE, VEC> {
    int h, r, t;
    NRow<VEC> xh, xr, xt, n1, n2;   // n1 = the table's own normalisation, n2 = _calc's l2_normalize of it
    Row<VEC> u;
    float ab;
    __device__ __forceinline__ float forward(const ModelDev& M, int h_, int r_, int t_, int lane) {
        h = h_; r = r_; t = t_;
        xh = lookup<VEC>(M.ent, h, lane);
        xr = lookup<VEC>(M.rel, r, lane);
        xt = lookup<VEC>(M.ent, t, lane);
        n1 = lookup<VEC>(M.rel_aux, r, lane);
        n2 = normalised<VEC>(n1.x);
        float a = dotr(xh.x, n2.x), b = dotr(xt.x, n2.x);
        warp_sum2(a, b);
        ab = a - b;
        u = r_fma(n2.x, -ab, r_sub(r_add(xh.x, xr.x), xt.x));
        return warp_sum(score_partial<SCORE, VEC>(u));
    }
    __device__ __forceinline__ void backward(const ModelDev& M, float g, int lane) {
        const Row<VEC> du = r_scale(score_dir<SCORE, VEC>(u), g);
        const float c = warp_sum(dotr(du, n2.x));
        const Row<VEC> dh = r_fma(n2.x, -c, du);                                    // d/dĥ ; d/dt̂ = −dh
        const Row<VEC> dn2 = r_fma(r_sub(xh.x, xt.x), -c, r_scale(du, -ab));       // −(a−b)·du − c·(ĥ − t̂)
        const Row<VEC> dn1 = back_normalised<VEC>(dn2, n2);
        push<VEC>(M.ent, h, lane, dh, xh);
        push<VEC>(M.ent, t, lane, r_neg(dh), xt);
        push<VEC>(M.rel, r, lane, du, xr);
        push<VEC>(M.rel_aux, r, lane, dn1, n1);
    }
};

// TransD: e⊥ = l2_normalize(ê + <ê, ê_p>·r̂_p); ent_aux = ent_transfer, rel_aux = rel_transfer
template <int SCORE, int VEC>
struct Triple<OEA_MODEL_TRANSD, SCORE, VEC> {
    int h, r, t;
    NRow<VEC> xh, xt, ph, pt, xr, pr, vh, vt;
    Row<VEC> u;
    float a, b;
    __device__ __forceinline__ float forward(const ModelDev& M, int h_, int r_, int t_, int lane) {
        h = h_; r = r_; t = t_;
        xh = lookup<VEC>(M.ent, h, lane);
        xt = lookup<VEC>(M.ent, t, lane);
        ph = lookup<VEC>(M.ent_aux, h, lane);
        pt = lookup<VEC>(M.ent_aux, t, lane);
        xr = lookup<VEC>(M.rel, r, lane);
        pr = lookup<VEC>(M.rel_aux, r, lane);
        a = dotr(xh.x, ph.x); b = dotr(xt.x, pt.x);
        warp_sum2(a, b);
        vh = normalised<VEC>(r_fma(pr.x, a, xh.x));
        vt = normalised<VEC>(r_fma(pr.x, b, xt.x));
        u = r_sub(r_add(vh.x, xr.x), vt.x);
        return warp_sum(score_partial<SCORE, VEC>(u));
    }
    __device__ __forceinline__ void backward(const ModelDev& M, float g, int lane) {
        const Row<VEC> du = r_scale(score_dir<SCORE, VEC>(u), g);
        const Row<VEC> dvh = back_normalised<VEC>(du, vh);
        const Row<VEC> dvt = back_normalised<VEC>(r_neg(du), vt);
        float eh = dotr(dvh, pr.x), et = dotr(dvt, pr.x);
        warp_sum2(eh, et);
        push<VEC>(M.ent, h, lane, r_fma(ph.x, eh, dvh), xh);
        push<VEC>(M.ent, t, lane, r_fma(pt.x, et, dvt), xt);
        push<VEC>(M.ent_aux, h, lane, r_scale(xh.x, eh), ph);
        push<VEC>(M.ent_aux, t, lane, r_scale(xt.x, et), pt);
        push<VEC>(M.rel, r, lane, du, xr);
        push<VEC>(M.rel_aux, r, lane, r_fma(dvh, a, r_scale(dvt, b)), pr);
    }
};

// DistMult: E = −Σ ĥ∘r̂∘t̂ (SCORE unused)
template <int SCORE, int VEC>
struct Triple<OEA_MODEL_DISTMULT, SCORE, VEC> {
    int h, r, t;
    NRow<VEC> xh, xr, xt;
    __device__ __forceinline__ float forward(const ModelDev& M, int h_, int r_, int t_, int lane) {
        h = h_; r = r_; t = t_;
        xh = lookup<VEC>(M.ent, h, lane);
        xr = lookup<VEC>(M.rel, r, lane);
        xt = lookup<VEC>(M.ent, t, lane);
        return -warp_sum(dotr(r_mul(xh.x, xr.x), xt.x));
    }
    __device__ __forceinline__ void backward(const ModelDev& M, float g, int lane) {
        const float w = -g;   // d loss / d score
        push<VEC>(M.ent, h, lane, r_scale(r_mul(xr.x, xt.x), w), xh);
        push<VEC>(M.ent, t, lane, r_scale(r_mul(xh.x, xr.x), w), xt);
        push<VEC>(M.rel, r, lane, r_scale(r_mul(xh.x, xt.x), w), xr);
    }
};

// SimplE: ent = head_ent_embeds, ent_aux = tail_ent_embeds, rel = rel_embeds1, rel_aux = rel_embeds2
template <int SCORE, int VEC>
struct Triple<OEA_MODEL_SIMPLE, SCORE, VEC> {
    int h, r, t;
    NRow<VEC> Hh, Ht, Th, Tt, r1, r2, q1, q2;
    __device__ __forceinline__ float forward(const ModelDev& M, int h_, int r_, int t_, int lane) {
        h = h_; r = r_; t = t_;
        Hh = lookup<VEC>(M.ent, h, lane);
        Ht = lookup<VEC>(M.ent, t, lane);
        Th = lookup<VEC>(M.ent_aux, h, lane);
        Tt = lookup<VEC>(M.ent_aux, t, lane);
        r1 = lookup<VEC>(M.rel, r, lane);
        r2 = lookup<VEC>(M.rel_aux, r, lane);
        q1 = normalised<VEC>(r_mul(Hh.x, r1.x));
        q2 = normalised<VEC>(r_mul(Ht.x, r2.x));
        float s1 = dotr(q1.x, Tt.x), s2 = dotr(q2.x, Th.x);
        warp_sum2(s1, s2);
        return -0.5f * (s1 + s2);
    }
    __device__ __forceinline__ void backward(const ModelDev& M, float g, int lane) {
        const float w = -0.5f * g;   // d loss / d each direction's score
        const Row<VEC> dp1 = back_normalised<VEC>(r_scale(Tt.x, w), q1);
        const Row<VEC> dp2 = back_normalised<VEC>(r_scale(Th.x, w), q2);
        push<VEC>(M.ent, h, lane, r_mul(dp1, r1.x), Hh);
        push<VEC>(M.ent, t, lane, r_mul(dp2, r2.x), Ht);
        push<VEC>(M.ent_aux, t, lane, r_scale(q1.x, w), Tt);
        push<VEC>(M.ent_aux, h, lane, r_scale(q2.x, w), Th);
        push<VEC>(M.rel, r, lane, r_mul(dp1, Hh.x), r1);
        push<VEC>(M.rel_aux, r, lane, r_mul(dp2, Ht.x), r2);
    }
};

// ---- kernels -------------------------------------------------------------------------------------------------------
// Independent losses (limited / logistic / positive / logsigmoid), `scale` multiplies loss and gradient
// (DistMult's reduce_mean): one warp per triple, positives first.
template <int MODEL, int SCORE, int VEC>
__global__ void __launch_bounds__(kThreads)
k_model_fed(ModelDev M,
            const int32_t* __restrict__ ph, const int32_t* __restrict__ pr, const int32_t* __restrict__ pt, int n_pos,
            const int32_t* __restrict__ nh, const int32_t* __restrict__ nr, const int32_t* __restrict__ nt, int n_neg,
            oea_loss_cfg cfg, float scale, double* __restrict__ loss_out) {
    __shared__ double s_loss[kWarpsPerBlock];
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    const int total = n_pos + n_neg;
    float warp_loss = 0.f;
    for (int i = warp_global; i < total; i += n_warps) {
        const bool is_neg = i >= n_pos;
        const int j = is_neg ? i - n_pos : i;
        const int h = is_neg ? __ldg(nh + j) : __ldg(ph + j);
        const int r = is_neg ? __ldg(nr + j) : __ldg(pr + j);
        const int t = is_neg ? __ldg(nt + j) : __ldg(pt + j);
        Triple<MODEL, SCORE, VEC> T;
        const float E = T.forward(M, h, r, t, lane);
        float L, g;
        loss_of(cfg.loss_kind, is_neg, E, cfg, L, g);
        warp_loss += L * scale;
        g *= scale;
        if (g != 0.f) T.backward(M, g, lane);
    }
    LossAcc acc{s_loss};
    acc.flush(warp_loss, loss_out);
}

// Margin-based loss Σ relu(m + E⁺_i − E⁻_i) (losses.py:15-27, one negative per positive): one warp per pair.
template <int MODEL, int SCORE, int VEC>
__global__ void __launch_bounds__(kThreads)
k_model_margin(ModelDev M,
               const int32_t* __restrict__ ph, const int32_t* __restrict__ pr, const int32_t* __restrict__ pt,
               const int32_t* __restrict__ nh, const int32_t* __restrict__ nr, const int32_t* __restrict__ nt, int n,
               oea_loss_cfg cfg, float scale, double* __restrict__ loss_out) {
    __shared__ double s_loss[kWarpsPerBlock];
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    float warp_loss = 0.f;
    for (int i = warp_global; i < n; i += n_warps) {
        Triple<MODEL, SCORE, VEC> P, N;
        const float ep = P.forward(M, __ldg(ph + i), __ldg(pr + i), __ldg(pt + i), lane);
        const float en = N.forward(M, __ldg(nh + i), __ldg(nr + i), __ldg(nt + i), lane);
        const float v = cfg.margin + ep - en;
        warp_loss += fmaxf(v, 0.f) * scale;
        if (v > 0.f) {
            P.backward(M, scale, lane);
            N.backward(M, -scale, lane);
        }
    }
    LossAcc acc{s_loss};
    acc.flush(warp_loss, loss_out);
}

static int check_model(const oea_model* m, ModelDev* out) {
    if (m == nullptr) return OEA_ERR_NULL;
    if (m->kind < OEA_MODEL_TRANSE || m->kind > OEA_MODEL_SIMPLE) return OEA_ERR_KIND;
    const bool need_ent_aux = m->kind == OEA_MODEL_TRANSD || m->kind == OEA_MODEL_SIMPLE;
    const bool need_rel_aux = m->kind == OEA_MODEL_TRANSH || need_ent_aux;
    int rc = check_table(m->ent, true); if (rc) return rc;
    rc = check_table(m->rel, true); if (rc) return rc;
    if (need_ent_aux) { rc = check_table(m->ent_aux, true); if (rc) return rc; }
    if (need_rel_aux) { rc = check_table(m->rel_aux, true); if (rc) return rc; }
    const oea_table* all[4] = {m->ent, m->rel, need_ent_aux ? m->ent_aux : nullptr, need_rel_aux ? m->rel_aux : nullptr};
    for (const oea_table* t : all)
        if (t != nullptr && (t->pitch != m->ent->pitch || t->dim != m->ent->dim)) return OEA_ERR_DIM;
    if (m->ent->pitch > 256) return OEA_ERR_DIM;   // two float4 per lane
    if (need_ent_aux && m->ent_aux->rows != m->ent->rows) return OEA_ERR_SHAPE;
    if (need_rel_aux && m->rel_aux->rows != m->rel->rows) return OEA_ERR_SHAPE;
    out->ent = table_dev(m->ent);
    out->rel = table_dev(m->rel);
    out->ent_aux = need_ent_aux ? table_dev(m->ent_aux) : out->ent;
    out->rel_aux = need_rel_aux ? table_dev(m->rel_aux) : out->rel;
    return OEA_OK;
}

}  // namespace oea

using namespace oea;

extern "C" int oea_model_score_fed(const oea_model* model,
                                   const int32_t* pos_h, const int32_t* pos_r, const int32_t* pos_t, int32_t n_pos,
                                   const int32_t* neg_h, const int32_t* neg_r, const int32_t* neg_t, int32_t n_neg,
                                   const oea_loss_cfg* loss, float loss_scale, double* loss_out, void* stream) {
    ModelDev M;
    int rc = check_model(model, &M); if (rc) return rc;
    if (!loss || !loss_out) return OEA_ERR_NULL;
    if (n_pos < 0 || n_neg < 0) return OEA_ERR_SHAPE;
    if (n_pos > 0 && (!pos_h || !pos_r || !pos_t)) return OEA_ERR_NULL;
    if (n_neg > 0 && (!neg_h || !neg_r || !neg_t)) return OEA_ERR_NULL;
    if (loss->loss_kind < OEA_LOSS_MARGIN || loss->loss_kind > OEA_LOSS_LOGSIGMOID) return OEA_ERR_KIND;
    const bool bilinear = model->kind == OEA_MODEL_DISTMULT || model->kind == OEA_MODEL_SIMPLE;
    if (!bilinear && loss->score_kind != OEA_SCORE_L1 && loss->score_kind != OEA_SCORE_L2SQ) return OEA_ERR_KIND;
    const bool margin = loss->loss_kind == OEA_LOSS_MARGIN;
    if (margin && n_pos != n_neg) return OEA_ERR_SHAPE;
    if (n_pos + n_neg == 0) return OEA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const bool l1 = !bilinear && loss->score_kind == OEA_SCORE_L1;
    const int grid = grid_for(margin ? n_pos : n_pos + n_neg);

#ifdef OEA_HOST_EMU   // tests/emu: the same kernels on the CPU warp emulator (two blocks keep the thread count small)
#define OEA_RUN(KERNEL, ...) emu::launch(grid < 2 ? grid : 2, kThreads, [&] { KERNEL(__VA_ARGS__); })
#else
#define OEA_RUN(KERNEL, ...) KERNEL<<<grid, kThreads, 0, st>>>(__VA_ARGS__)
#endif
#define OEA_LAUNCH_MODEL(MODEL, SCORE, V)                                                                              \
    do {                                                                                                               \
        if (margin) { auto kernel = k_model_margin<MODEL, SCORE, V>;                                                   \
                      OEA_RUN(kernel, M, pos_h, pos_r, pos_t, neg_h, neg_r, neg_t, n_pos, *loss, loss_scale, loss_out); } \
        else { auto kernel = k_model_fed<MODEL, SCORE, V>;                                                             \
               OEA_RUN(kernel, M, pos_h, pos_r, pos_t, n_pos, neg_h, neg_r, neg_t, n_neg, *loss, loss_scale, loss_out); } \
    } while (0)
#define OEA_LAUNCH_VEC(MODEL, SCORE)                                                  \
    do {                                                                              \
        if (model->ent->pitch <= 128) OEA_LAUNCH_MODEL(MODEL, SCORE, 1);              \
        else OEA_LAUNCH_MODEL(MODEL, SCORE, 2);                                       \
    } while (0)
#define OEA_LAUNCH_SCORE(MODEL)                                                       \
    do {                                                                              \
        if (l1) OEA_LAUNCH_VEC(MODEL, OEA_SCORE_L1);                                  \
        else OEA_LAUNCH_VEC(MODEL, OEA_SCORE_L2SQ);                                   \
    } while (0)

    switch (model->kind) {
        case OEA_MODEL_TRANSE: OEA_LAUNCH_SCORE(OEA_MODEL_TRANSE); break;
        case OEA_MODEL_TRANSH: OEA_LAUNCH_SCORE(OEA_MODEL_TRANSH); break;
        case OEA_MODEL_TRANSD: OEA_LAUNCH_SCORE(OEA_MODEL_TRANSD); break;
        case OEA_MODEL_DISTMULT: OEA_LAUNCH_VEC(OEA_MODEL_DISTMULT, OEA_SCORE_L2SQ); break;
        default: OEA_LAUNCH_VEC(OEA_MODEL_SIMPLE, OEA_SCORE_L2SQ); break;
    }
#undef OEA_LAUNCH_SCORE
#undef OEA_LAUNCH_VEC
#undef OEA_LAUNCH_MODEL
#undef OEA_RUN
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}
