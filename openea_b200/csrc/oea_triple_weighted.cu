// oea_triple_weighted.cu — path (i) for the callers that weight every training pair (SURVEY §8f-2: "the remaining
// approaches on the same kernel"):
//
//   k_score_margin_weighted   scale · Σ_i w_i · relu(margin + s(pos_i) − s(neg_i)),  s = ‖ĥ + r̂ − t̂‖ (L1 or squared L2)
//       IPTransE's alignment loss on the triples of newly aligned entities, w_i = the pair's similarity
//       (approaches/iptranse.py:170-174,208-226), and its relation-path loss Σ (1/w_i)·relu(m + ‖r̂x + r̂y − r̂‖² −
//       ‖r̂x' + r̂y' − r̂'‖²) (iptranse.py:176-185): there all three rows of a "triple" are relation rows, so the
//       entity table and the relation table of the call are the same table — legal here, every gradient leaves
//       through red.global.add.
//   k_pair_distance           scale · Σ_i w_i · ‖ê_a(i) − ê_b(i)‖²
//       IMUSE's align loss over the entity pairs its string matcher found (approaches/imuse.py:303-306).
//
// k_score_margin_weighted scores a pair with the TransE triple of oea_transe.cuh; k_pair_distance uses the same row
// arithmetic and normalisation Jacobian (oea_rowmath.cuh).  One warp per pair, the six (two) rows of a pair in
// registers.  HBM / L2 bound: 6·4·d B gathered per pair, up to as much reduced.  sm_90a.
#include "oea_transe.cuh"

using namespace oea;

namespace {

template <int SCORE, int VEC>
__global__ void __launch_bounds__(kThreads)
k_score_margin_weighted(ModelDev M,
                        const int32_t* __restrict__ ph, const int32_t* __restrict__ pr, const int32_t* __restrict__ pt,
                        const int32_t* __restrict__ nh, const int32_t* __restrict__ nr, const int32_t* __restrict__ nt,
                        int n, const float* __restrict__ weights, int reciprocal, float scale, float margin,
                        double* __restrict__ loss_out) {
    __shared__ double s_loss[kWarpsPerBlock];
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    float warp_loss = 0.f;

    for (int i = warp_global; i < n; i += n_warps) {
        float w = weights != nullptr ? __ldg(weights + i) : 1.f;
        if (reciprocal) w = 1.f / w;                       // tf.cast(1 / weight, tf.float32), iptranse.py:179
        w *= scale;
        Triple<OEA_MODEL_TRANSE, SCORE, VEC> P, N;
        P.gather(M, __ldg(ph + i), __ldg(pr + i), __ldg(pt + i), lane);
        N.gather(M, __ldg(nh + i), __ldg(nr + i), __ldg(nt + i), lane);
        float sp = P.score(M), sn = N.score(M);
        warp_sum2(sp, sn);
        const float v = margin + sp - sn;
        warp_loss += w * fmaxf(v, 0.f);
        if (v > 0.f && w != 0.f) {                         // relu'(0) = 0 as TF; a zero-weight pair flags no row
            P.backward(M, w, lane);
            N.backward(M, -w, lane);
        }
    }
    LossAcc acc{s_loss};
    acc.flush(warp_loss, loss_out);
}

template <int VEC>
__global__ void __launch_bounds__(kThreads)
k_pair_distance(TableDev ent, const int32_t* __restrict__ ia, const int32_t* __restrict__ ib, int n,
                const float* __restrict__ weights, float scale, double* __restrict__ loss_out) {
    __shared__ double s_loss[kWarpsPerBlock];
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    float warp_loss = 0.f;

    for (int i = warp_global; i < n; i += n_warps) {
        const int a = __ldg(ia + i), b = __ldg(ib + i);
        const float w = scale * (weights != nullptr ? __ldg(weights + i) : 1.f);
        Row<VEC> xa = load_row<VEC>(ent.w, a, ent.pitch, lane);
        Row<VEC> xb = load_row<VEC>(ent.w, b, ent.pitch, lane);
        float ssa = sumsq(xa), ssb = sumsq(xb);
        warp_sum2(ssa, ssb);
        const float inva = inv_norm(ssa, ent.norm), invb = inv_norm(ssb, ent.norm);
        Row<VEC> du;
#pragma unroll
        for (int c = 0; c < VEC; ++c) {
            xa.v[c] = xa.v[c] * inva; xb.v[c] = xb.v[c] * invb;
            du.v[c] = xa.v[c] - xb.v[c];
        }
        float s = sumsq(du), da, db;
#pragma unroll
        for (int c = 0; c < VEC; ++c) du.v[c] = du.v[c] * (2.f * w);        // d(w·‖u‖²)/du
        da = dotr(xa, du); db = dotr(xb, du);
        warp_sum3(s, da, db);
        warp_loss += w * s;
        if (w != 0.f) {
            Row<VEC> ga = through_norm(du, xa, da, inva, ssa, ent.norm);
            Row<VEC> gb = through_norm(du, xb, db, invb, ssb, ent.norm);
#pragma unroll
            for (int c = 0; c < VEC; ++c) gb.v[c] = neg(gb.v[c]);
            red_row<VEC>(ent.g, a, ent.pitch, lane, ga);
            red_row<VEC>(ent.g, b, ent.pitch, lane, gb);
            if (lane == 0) { ent.touched[a] = 1; ent.touched[b] = 1; }
        }
    }
    LossAcc acc{s_loss};
    acc.flush(warp_loss, loss_out);
}

}  // namespace

extern "C" int oea_triple_score_margin_weighted(const oea_table* ent, const oea_table* rel,
                                                const int32_t* pos_h, const int32_t* pos_r, const int32_t* pos_t,
                                                const int32_t* neg_h, const int32_t* neg_r, const int32_t* neg_t, int32_t n,
                                                const float* weights, int32_t weight_mode, float scale,
                                                const oea_loss_cfg* loss, double* loss_out, void* stream) {
    int rc = check_table(ent, true); if (rc) return rc;
    rc = check_table(rel, true); if (rc) return rc;
    if (loss == nullptr || loss_out == nullptr) return OEA_ERR_NULL;
    if (n < 0) return OEA_ERR_SHAPE;
    if (n > 0 && (!pos_h || !pos_r || !pos_t || !neg_h || !neg_r || !neg_t)) return OEA_ERR_NULL;
    if (ent->pitch != rel->pitch || ent->dim != rel->dim) return OEA_ERR_DIM;
    if (loss->score_kind != OEA_SCORE_L1 && loss->score_kind != OEA_SCORE_L2SQ) return OEA_ERR_KIND;
    if (weight_mode != OEA_WEIGHT_DIRECT && weight_mode != OEA_WEIGHT_RECIPROCAL) return OEA_ERR_KIND;
    if (n == 0) return OEA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const TableDev e = table_dev(ent), r = table_dev(rel);
    const ModelDev M{e, r, e, r, ent->dim, 0.f, 0.f};
    const bool l1 = loss->score_kind == OEA_SCORE_L1;
    const int grid = grid_for(n);
    const int recip = weight_mode == OEA_WEIGHT_RECIPROCAL && weights != nullptr;
#define CALL(V)                                                                                                           \
    if (l1) OEA_LAUNCH((k_score_margin_weighted<OEA_SCORE_L1, V>), grid, kThreads, 0, st, M, pos_h, pos_r, pos_t, neg_h,    \
                       neg_r, neg_t, n, weights, recip, scale, loss->margin, loss_out);                                       \
    else OEA_LAUNCH((k_score_margin_weighted<OEA_SCORE_L2SQ, V>), grid, kThreads, 0, st, M, pos_h, pos_r, pos_t, neg_h,     \
                    neg_r, neg_t, n, weights, recip, scale, loss->margin, loss_out)
    OEA_DISPATCH_VEC(ent->pitch, CALL);
#undef CALL
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_pair_distance_loss(const oea_table* ent, const int32_t* ids_a, const int32_t* ids_b, int32_t n,
                                      const float* weights, float scale, double* loss_out, void* stream) {
    int rc = check_table(ent, true); if (rc) return rc;
    if (loss_out == nullptr) return OEA_ERR_NULL;
    if (n < 0) return OEA_ERR_SHAPE;
    if (n > 0 && (!ids_a || !ids_b)) return OEA_ERR_NULL;
    if (n == 0) return OEA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    TableDev e = table_dev(ent);
    const int grid = grid_for(n);
#define CALL(V) OEA_LAUNCH((k_pair_distance<V>), grid, kThreads, 0, st, e, ids_a, ids_b, n, weights, scale, loss_out)
    OEA_DISPATCH_VEC(ent->pitch, CALL);
#undef CALL
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}
