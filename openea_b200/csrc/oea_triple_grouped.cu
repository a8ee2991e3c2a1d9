// oea_triple_grouped.cu — the fed step of path (i) for batches in the reference's layout (modules/train/batch.py:36-45:
// the k negatives of positive p sit at p·k … p·k+k−1 and differ from it in ONE end), one warp per positive AND its
// negatives.  Same maths as k_score_fed / k_score_margin (models/basic_model.py:80-98, modules/base/losses.py:15-73);
// what changes is the traffic: the positive's three rows are loaded and normalised once, a negative that shares two of
// them loads one row, and the gradients of the shared rows are summed in registers (the Jacobian of l2_normalize is
// linear in the incoming gradient) and leave as three vector reductions per positive instead of three per triple:
// 3 + k row loads and 3 + k row reductions per positive instead of 3·(1 + k) each.  A negative that shares fewer than
// two rows with its positive (any fed batch is legal) takes the general path of k_score_fed for that triple.  sm_90a.
//
// Opt-in: oea_triple_step_fed_host uses it when OEA_FED_GROUPED=1 (until it has been timed on hardware);
// tests/test_emu_triple_grouped.py checks it on the CPU warp emulator against the C oracle.
#include <stdlib.h>
#include <cooperative_groups.h>

#include "oea_rowmath.cuh"
#include "oea_rowopt.cuh"
#include "oea_duo.cuh"

namespace oea {

template <int SCORE, int VEC>
__device__ __forceinline__ void
grouped_score_body(const TableDev& ent, const TableDev& rel,
                   const int32_t* __restrict__ ph, const int32_t* __restrict__ pr, const int32_t* __restrict__ pt, int n_pos,
                   const int32_t* __restrict__ nh, const int32_t* __restrict__ nr, const int32_t* __restrict__ nt, int k,
                   const oea_loss_cfg& cfg, double* __restrict__ loss_out, double* s_loss) {
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    const bool margin_mode = cfg.loss_kind == OEA_LOSS_MARGIN;       // Σ relu(m + s⁺ − s⁻), k == 1
    float warp_loss = 0.f;

    for (int p = warp_global; p < n_pos; p += n_warps) {
        const int h = __ldg(ph + p), r = __ldg(pr + p), t = __ldg(pt + p);
        Row<VEC> xh = load_row<VEC>(ent.w, h, ent.pitch, lane);
        Row<VEC> xr = load_row<VEC>(rel.w, r, rel.pitch, lane);
        Row<VEC> xt = load_row<VEC>(ent.w, t, ent.pitch, lane);
        float ssh = sumsq(xh), ssr = sumsq(xr), sst = sumsq(xt);
        warp_sum3(ssh, ssr, sst);
        const float ih = inv_norm(ssh, ent.norm), ir = inv_norm(ssr, rel.norm), it = inv_norm(sst, ent.norm);
        Row<VEC> hr, rt, u, Gh, Gr, Gt;      // hr = ĥ + r̂, rt = r̂ − t̂; G* = Σ d loss / d (normalised row)
#pragma unroll
        for (int c = 0; c < VEC; ++c) {
            xh.v[c] = xh.v[c] * ih; xr.v[c] = xr.v[c] * ir; xt.v[c] = xt.v[c] * it;
            hr.v[c] = xh.v[c] + xr.v[c];
            rt.v[c] = xr.v[c] - xt.v[c];
            u.v[c] = hr.v[c] - xt.v[c];
        }
        const float sp = warp_sum(score_partial<SCORE, VEC>(u));
        float L = 0.f, g = 0.f;
        if (!margin_mode) loss_of(cfg.loss_kind, false, sp, cfg, L, g);
        warp_loss += L;
        bool any_grad = g != 0.f;
        const Row<VEC> dir_pos = score_dir<SCORE, VEC>(u);
#pragma unroll
        for (int c = 0; c < VEC; ++c) { Gh.v[c] = dir_pos.v[c] * g; Gr.v[c] = Gh.v[c]; Gt.v[c] = neg(Gh.v[c]); }

        for (int j = 0; j < k; ++j) {
            const size_t q = (size_t)p * k + j;
            const int eh = __ldg(nh + q), er = __ldg(nr + q), et = __ldg(nt + q);
            const bool share_tail = er == r && et == t;          // head corrupted (or an exact copy of the positive)
            const bool share_head = er == r && eh == h;          // tail corrupted
            if (share_tail || share_head) {
                const bool head = share_tail;                    // the row that is new: the head (else the tail)
                const int e = head ? eh : et;
                Row<VEC> xe = load_row<VEC>(ent.w, e, ent.pitch, lane);
                const float sse = warp_sum(sumsq(xe));
                const float ie = inv_norm(sse, ent.norm);
#pragma unroll
                for (int c = 0; c < VEC; ++c) {
                    xe.v[c] = xe.v[c] * ie;
                    u.v[c] = head ? (xe.v[c] + rt.v[c]) : (hr.v[c] - xe.v[c]);
                }
                const Row<VEC> dir = score_dir<SCORE, VEC>(u);
                float sn = score_partial<SCORE, VEC>(u), de = dotr(xe, dir);
                warp_sum2(sn, de);
                if (margin_mode) {
                    const float v = cfg.margin + sp - sn;
                    L = fmaxf(v, 0.f);
                    g = v > 0.f ? -1.f : 0.f;
                    if (v > 0.f) {       // the positive's share of the active hinge
#pragma unroll
                        for (int c = 0; c < VEC; ++c) { Gh.v[c] = Gh.v[c] + dir_pos.v[c]; Gr.v[c] = Gr.v[c] + dir_pos.v[c]; Gt.v[c] = Gt.v[c] - dir_pos.v[c]; }
                        any_grad = true;
                    }
                } else {
                    loss_of(cfg.loss_kind, true, sn, cfg, L, g);
                }
                warp_loss += L;
                if (g != 0.f) {
                    any_grad = true;
                    const float ge = head ? g : -g;              // d/dê = ±g·dir
                    Row<VEC> Ge;
#pragma unroll
                    for (int c = 0; c < VEC; ++c) {
                        const float4 du = dir.v[c] * g;
                        Gr.v[c] = Gr.v[c] + du;
                        if (head) Gt.v[c] = Gt.v[c] - du; else Gh.v[c] = Gh.v[c] + du;
                        Ge.v[c] = dir.v[c] * ge;
                    }
                    const Row<VEC> out = through_norm(Ge, xe, ge * de, ie, sse, ent.norm);
                    red_row<VEC>(ent.g, e, ent.pitch, lane, out);
                    if (lane == 0) ent.touched[e] = 1;
                }
            } else {
                // general triple: nothing to share with the positive (k_score_fed's path)
                Row<VEC> yh = load_row<VEC>(ent.w, eh, ent.pitch, lane);
                Row<VEC> yr = load_row<VEC>(rel.w, er, rel.pitch, lane);
                Row<VEC> yt = load_row<VEC>(ent.w, et, ent.pitch, lane);
                float s1 = sumsq(yh), s2 = sumsq(yr), s3 = sumsq(yt);
                warp_sum3(s1, s2, s3);
                const float i1 = inv_norm(s1, ent.norm), i2 = inv_norm(s2, rel.norm), i3 = inv_norm(s3, ent.norm);
#pragma unroll
                for (int c = 0; c < VEC; ++c) {
                    yh.v[c] = yh.v[c] * i1; yr.v[c] = yr.v[c] * i2; yt.v[c] = yt.v[c] * i3;
                    u.v[c] = yh.v[c] + yr.v[c] - yt.v[c];
                }
                const float sn = warp_sum(score_partial<SCORE, VEC>(u));
                if (margin_mode) {
                    const float v = cfg.margin + sp - sn;
                    L = fmaxf(v, 0.f);
                    g = v > 0.f ? -1.f : 0.f;
                    if (v > 0.f) {
#pragma unroll
                        for (int c = 0; c < VEC; ++c) { Gh.v[c] = Gh.v[c] + dir_pos.v[c]; Gr.v[c] = Gr.v[c] + dir_pos.v[c]; Gt.v[c] = Gt.v[c] - dir_pos.v[c]; }
                        any_grad = true;
                    }
                } else {
                    loss_of(cfg.loss_kind, true, sn, cfg, L, g);
                }
                warp_loss += L;
                if (g != 0.f) {
                    Row<VEC> du = score_dir<SCORE, VEC>(u);
#pragma unroll
                    for (int c = 0; c < VEC; ++c) du.v[c] = du.v[c] * g;
                    float d1 = dotr(yh, du), d2 = dotr(yr, du), d3 = dotr(yt, du);
                    warp_sum3(d1, d2, d3);
                    const Row<VEC> g1 = through_norm(du, yh, d1, i1, s1, ent.norm);
                    const Row<VEC> g2 = through_norm(du, yr, d2, i2, s2, rel.norm);
                    Row<VEC> g3 = through_norm(du, yt, d3, i3, s3, ent.norm);
#pragma unroll
                    for (int c = 0; c < VEC; ++c) g3.v[c] = neg(g3.v[c]);
                    red_row<VEC>(ent.g, eh, ent.pitch, lane, g1);
                    red_row<VEC>(rel.g, er, rel.pitch, lane, g2);
                    red_row<VEC>(ent.g, et, ent.pitch, lane, g3);
                    if (lane == 0) { ent.touched[eh] = 1; rel.touched[er] = 1; ent.touched[et] = 1; }
                }
            }
        }

        if (any_grad) {
            float dh = dotr(xh, Gh), dr = dotr(xr, Gr), dt = dotr(xt, Gt);
            warp_sum3(dh, dr, dt);
            const Row<VEC> oh = through_norm(Gh, xh, dh, ih, ssh, ent.norm);
            const Row<VEC> orr = through_norm(Gr, xr, dr, ir, ssr, rel.norm);
            const Row<VEC> ot = through_norm(Gt, xt, dt, it, sst, ent.norm);
            red_row<VEC>(ent.g, h, ent.pitch, lane, oh);
            red_row<VEC>(rel.g, r, rel.pitch, lane, orr);
            red_row<VEC>(ent.g, t, ent.pitch, lane, ot);
            if (lane == 0) { ent.touched[h] = 1; rel.touched[r] = 1; ent.touched[t] = 1; }
        }
    }
    LossAcc acc{s_loss};
    acc.flush(warp_loss, loss_out);
}

template <int SCORE, int VEC>
__global__ void __launch_bounds__(kThreads)
k_score_fed_grouped(TableDev ent, TableDev rel,
                    const int32_t* __restrict__ ph, const int32_t* __restrict__ pr, const int32_t* __restrict__ pt, int n_pos,
                    const int32_t* __restrict__ nh, const int32_t* __restrict__ nr, const int32_t* __restrict__ nt, int k,
                    oea_loss_cfg cfg, double* __restrict__ loss_out) {
    __shared__ double s_loss[kWarpsPerBlock];
    grouped_score_body<SCORE, VEC>(ent, rel, ph, pr, pt, n_pos, nh, nr, nt, k, cfg, loss_out, s_loss);
}

// The whole fed training step as ONE cooperative launch: grouped scoring + gradients, grid barrier, octet row optimiser
// (the host-index step's two kernels and the launch ramp between them in one; same structure as k_step_sampled_oct).
template <int SCORE, int VEC, int KIND>
__global__ void __launch_bounds__(kThreads)
k_step_fed_grouped(TableDev ent, TableDev rel,
                   const int32_t* __restrict__ ph, const int32_t* __restrict__ pr, const int32_t* __restrict__ pt, int n_pos,
                   const int32_t* __restrict__ nh, const int32_t* __restrict__ nr, const int32_t* __restrict__ nt, int k,
                   oea_loss_cfg cfg, double* __restrict__ loss_out, OptTab A, OptTab B, float lr) {
    __shared__ double s_loss[kWarpsPerBlock];
    grouped_score_body<SCORE, VEC>(ent, rel, ph, pr, pt, n_pos, nh, nr, nt, k, cfg, loss_out, s_loss);
    cooperative_groups::this_grid().sync();
    rowopt_flagged_body<KIND>(A, B, ent.pitch, lr, blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5), gridDim.x * kWarpsPerBlock);
}

// The duo scorer (oea_duo.cuh) on a fed batch: two positives per warp, octet row layout, squared-L2 score, pitch <= 128,
// k <= 16.  Negatives that share fewer than two rows with their positive take the general-triple path inside the body.
__global__ void __launch_bounds__(kDuoThreads, OEA_DUO_MINB)
k_score_fed_duo(TableDev ent, TableDev rel, FedBatch F, oea_loss_cfg cfg, double* __restrict__ loss_out) {
    __shared__ double s_loss[kDuoWarps];
    __shared__ DuoStage s_stage[kDuoWarps];
    SampledParams none;
    duo_score_body<true>(ent, rel, none, F, cfg, loss_out, nullptr, s_loss, s_stage);
}

template <int KIND>
__global__ void __launch_bounds__(kDuoThreads, OEA_DUO_MINB)
k_step_fed_duo(TableDev ent, TableDev rel, FedBatch F, oea_loss_cfg cfg, double* __restrict__ loss_out, OptTab A, OptTab B, float lr) {
    __shared__ double s_loss[kDuoWarps];
    __shared__ DuoStage s_stage[kDuoWarps];
    SampledParams none;
    duo_score_body<true>(ent, rel, none, F, cfg, loss_out, nullptr, s_loss, s_stage);
    cooperative_groups::this_grid().sync();
    rowopt_flagged_body<KIND>(A, B, ent.pitch, lr, blockIdx.x * kDuoWarps + (threadIdx.x >> 5), gridDim.x * kDuoWarps);
}

}  // namespace oea

using namespace oea;

extern "C" int oea_triple_score_fed_grouped(const oea_table* ent, const oea_table* rel,
                                            const int32_t* pos_h, const int32_t* pos_r, const int32_t* pos_t, int32_t n_pos,
                                            const int32_t* neg_h, const int32_t* neg_r, const int32_t* neg_t, int32_t n_neg,
                                            const oea_loss_cfg* loss, double* loss_out, void* stream) {
    int rc = check_table(ent, true); if (rc) return rc;
    rc = check_table(rel, true); if (rc) return rc;
    if (!loss || !loss_out) return OEA_ERR_NULL;
    if (ent->pitch != rel->pitch || ent->dim != rel->dim) return OEA_ERR_DIM;
    if (n_pos <= 0 || n_neg < 0 || n_neg % n_pos != 0) return OEA_ERR_SHAPE;      // k negatives per positive, grouped
    if (!pos_h || !pos_r || !pos_t || (n_neg > 0 && (!neg_h || !neg_r || !neg_t))) return OEA_ERR_NULL;
    if (loss->loss_kind < OEA_LOSS_MARGIN || loss->loss_kind > OEA_LOSS_LOGSIGMOID) return OEA_ERR_KIND;
    if (loss->score_kind != OEA_SCORE_L1 && loss->score_kind != OEA_SCORE_L2SQ) return OEA_ERR_KIND;
    const int k = n_neg / n_pos;
    if (loss->loss_kind == OEA_LOSS_MARGIN && k != 1) return OEA_ERR_SHAPE;
    if ((loss->loss_kind == OEA_LOSS_POSITIVE || loss->loss_kind == OEA_LOSS_LOGSIGMOID) && k != 0) return OEA_ERR_SHAPE;
    TableDev e = table_dev(ent), r = table_dev(rel);
    const bool l1 = loss->score_kind == OEA_SCORE_L1;
    if (!l1 && ent->pitch <= 128 && oea_use_duo(k)) {
        FedBatch F{pos_h, pos_r, pos_t, neg_h, neg_r, neg_t, n_pos, k};
        const int grid = grid_one_wave<k_score_fed_duo>((n_pos + 1) / 2, kDuoWarps);
        OEA_LAUNCH(k_score_fed_duo, grid, kDuoThreads, 0, (cudaStream_t)stream, e, r, F, *loss, loss_out);
        OEA_LAUNCH_CHECK();
        return OEA_OK;
    }
    const int grid = grid_for(n_pos);
#define OEA_RUN_GROUPED(S, V) \
    OEA_LAUNCH((k_score_fed_grouped<S, V>), grid, kThreads, 0, (cudaStream_t)stream, e, r, pos_h, pos_r, pos_t, n_pos, neg_h, neg_r, neg_t, k, *loss, loss_out)
#define CALL(V) do { if (l1) OEA_RUN_GROUPED(OEA_SCORE_L1, V); else OEA_RUN_GROUPED(OEA_SCORE_L2SQ, V); } while (0)
    OEA_DISPATCH_VEC(ent->pitch, CALL);
#undef CALL
#undef OEA_RUN_GROUPED
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

// One cooperative launch for the whole fed step (grouped scorer + row optimiser).  Same contract as
// oea_triple_score_fed_grouped followed by oea_rowopt_apply_pair; squared-L2 score, pitch <= 256, Adagrad / SGD —
// OEA_ERR_KIND otherwise (the caller then takes the two-launch path).
extern "C" int oea_triple_step_fed_grouped(const oea_table* ent, const oea_table* rel,
                                           const int32_t* pos_h, const int32_t* pos_r, const int32_t* pos_t, int32_t n_pos,
                                           const int32_t* neg_h, const int32_t* neg_r, const int32_t* neg_t, int32_t n_neg,
                                           const oea_loss_cfg* loss, const oea_opt_cfg* opt, double* loss_out, void* stream) {
    int rc = check_table(ent, true); if (rc) return rc;
    rc = check_table(rel, true); if (rc) return rc;
    if (!loss || !loss_out || !opt) return OEA_ERR_NULL;
    if (ent->pitch != rel->pitch || ent->dim != rel->dim) return OEA_ERR_DIM;
    if (n_pos <= 0 || n_neg < 0 || n_neg % n_pos != 0) return OEA_ERR_SHAPE;
    if (!pos_h || !pos_r || !pos_t || (n_neg > 0 && (!neg_h || !neg_r || !neg_t))) return OEA_ERR_NULL;
    if (loss->loss_kind < OEA_LOSS_MARGIN || loss->loss_kind > OEA_LOSS_LOGSIGMOID) return OEA_ERR_KIND;
    if (loss->score_kind != OEA_SCORE_L2SQ || ent->pitch > 256) return OEA_ERR_KIND;
    if (opt->kind != OEA_OPT_ADAGRAD && opt->kind != OEA_OPT_SGD) return OEA_ERR_KIND;
    if (opt->kind == OEA_OPT_ADAGRAD && (!ent->state1 || !rel->state1)) return OEA_ERR_NULL;
    int k = n_neg / n_pos;
    if (loss->loss_kind == OEA_LOSS_MARGIN && k != 1) return OEA_ERR_SHAPE;
    if ((loss->loss_kind == OEA_LOSS_POSITIVE || loss->loss_kind == OEA_LOSS_LOGSIGMOID) && k != 0) return OEA_ERR_SHAPE;
    cudaStream_t st = (cudaStream_t)stream;
    TableDev e = table_dev(ent), r = table_dev(rel);
    OptTab A{ent->weight, ent->grad, ent->state1, ent->touched, ent->rows}, B{rel->weight, rel->grad, rel->state1, rel->touched, rel->rows};
    oea_loss_cfg cfg = *loss;
    float lr = opt->lr;
    int np = n_pos;
    if (ent->pitch <= 128 && oea_use_duo(k)) {
        FedBatch F{pos_h, pos_r, pos_t, neg_h, neg_r, neg_t, n_pos, k};
        if (opt->kind == OEA_OPT_ADAGRAD) {
            const int grid = grid_one_wave<k_step_fed_duo<OEA_OPT_ADAGRAD>>((n_pos + 1) / 2, kDuoWarps);
            OEA_CUDA_TRY(OEA_LAUNCH_COOPERATIVE(k_step_fed_duo<OEA_OPT_ADAGRAD>, grid, kDuoThreads, st, e, r, F, cfg, loss_out, A, B, lr));
        } else {
            const int grid = grid_one_wave<k_step_fed_duo<OEA_OPT_SGD>>((n_pos + 1) / 2, kDuoWarps);
            OEA_CUDA_TRY(OEA_LAUNCH_COOPERATIVE(k_step_fed_duo<OEA_OPT_SGD>, grid, kDuoThreads, st, e, r, F, cfg, loss_out, A, B, lr));
        }
        return OEA_OK;
    }
#define OEA_RUN_STEP(V, KIND)                                                                                            \
    do { const int grid = grid_one_wave<k_step_fed_grouped<OEA_SCORE_L2SQ, V, KIND>>(n_pos);                             \
         OEA_CUDA_TRY(OEA_LAUNCH_COOPERATIVE((k_step_fed_grouped<OEA_SCORE_L2SQ, V, KIND>), grid, kThreads, st, e, r, pos_h, pos_r, \
                                             pos_t, np, neg_h, neg_r, neg_t, k, cfg, loss_out, A, B, lr)); } while (0)
    if (ent->pitch <= 128) { if (opt->kind == OEA_OPT_ADAGRAD) OEA_RUN_STEP(1, OEA_OPT_ADAGRAD); else OEA_RUN_STEP(1, OEA_OPT_SGD); }
    else { if (opt->kind == OEA_OPT_ADAGRAD) OEA_RUN_STEP(2, OEA_OPT_ADAGRAD); else OEA_RUN_STEP(2, OEA_OPT_SGD); }
#undef OEA_RUN_STEP
    return OEA_OK;
}
