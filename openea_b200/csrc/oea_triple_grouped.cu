// oea_triple_grouped.cu — the fed step of path (i) for batches in the reference's layout (modules/train/batch.py:36-45:
// the k negatives of positive p sit at p·k … p·k+k−1 and differ from it in ONE end), one warp per positive AND its
// negatives: the per-positive body of oea_transe.cuh on a fed batch, and the duo scorer (oea_duo.cuh) for the
// squared-L2 score at pitch <= 128.  Same maths as oea_triple_score_fed (models/basic_model.py:80-98,
// modules/base/losses.py:15-73); what changes is the traffic: 3 + k row loads and 3 + k row reductions per positive
// instead of 3·(1 + k) each.  sm_90a.
//
// Opt-in: oea_triple_step_fed_host uses it when OEA_FED_GROUPED=1 (until it has been timed on hardware);
// tests/test_emu_triple_grouped.py checks it on the CPU warp emulator against the C oracle.
#include <cooperative_groups.h>

#include "oea_rowmath.cuh"
#include "oea_rowopt.cuh"
#include "oea_duo.cuh"
#include "oea_transe.cuh"

namespace oea {

// The per-positive body (oea_transe.cuh) on a fed batch, one warp per positive and its negatives.  The index vectors
// arrive as __restrict__ parameters: passed as a FedBatch, the VEC = 4 instantiation spills more.
template <int SCORE, int VEC>
__global__ void __launch_bounds__(kThreads)
k_score_fed_grouped(TableDev ent, TableDev rel,
                    const int32_t* __restrict__ ph, const int32_t* __restrict__ pr, const int32_t* __restrict__ pt, int n_pos,
                    const int32_t* __restrict__ nh, const int32_t* __restrict__ nr, const int32_t* __restrict__ nt, int k,
                    oea_loss_cfg cfg, double* __restrict__ loss_out) {
    __shared__ double s_loss[kWarpsPerBlock];
    const FedBatch F{ph, pr, pt, nh, nr, nt, n_pos, k};
    const SampledParams none{};
    positive_score_body<SCORE, VEC, true>(ent, rel, none, F, cfg, loss_out, nullptr, s_loss);
}

// The whole fed step as ONE cooperative launch: the per-positive body, grid barrier, octet row optimiser
// (the host-index step's two kernels and the launch ramp between them in one; same structure as k_step_sampled_oct).
template <int SCORE, int VEC, int KIND>
__global__ void __launch_bounds__(kThreads)
k_step_fed_grouped(TableDev ent, TableDev rel, FedBatch F, oea_loss_cfg cfg, double* __restrict__ loss_out, OptTab A, OptTab B,
                   float lr) {
    __shared__ double s_loss[kWarpsPerBlock];
    const SampledParams none{};
    positive_score_body<SCORE, VEC, true>(ent, rel, none, F, cfg, loss_out, nullptr, s_loss);
    cooperative_groups::this_grid().sync();
    rowopt_flagged_body<KIND>(A, B, ent.pitch, lr, blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5), gridDim.x * kWarpsPerBlock);
}

// The duo scorer (oea_duo.cuh) on a fed batch: two positives per warp, octet row layout, squared-L2 score, pitch <= 128,
// k <= 16.  Negatives that share fewer than two rows with their positive take the general-triple path inside the body.
__global__ void __launch_bounds__(kDuoThreads, kDuoMinB)
k_score_fed_duo(TableDev ent, TableDev rel, FedBatch F, oea_loss_cfg cfg, double* __restrict__ loss_out) {
    __shared__ double s_loss[kDuoWarps];
    __shared__ DuoStage s_stage[kDuoWarps];
    const SampledParams none{};
    duo_score_body<true>(ent, rel, none, F, cfg, loss_out, nullptr, s_loss, s_stage);
}

template <int KIND>
__global__ void __launch_bounds__(kDuoThreads, kDuoMinB)
k_step_fed_duo(TableDev ent, TableDev rel, FedBatch F, oea_loss_cfg cfg, double* __restrict__ loss_out, OptTab A, OptTab B, float lr) {
    __shared__ double s_loss[kDuoWarps];
    __shared__ DuoStage s_stage[kDuoWarps];
    const SampledParams none{};
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
    const FedBatch F{pos_h, pos_r, pos_t, neg_h, neg_r, neg_t, n_pos, k};
    if (!l1 && ent->pitch <= 128 && k <= kDuoMaxK) {
        const int grid = grid_one_wave<k_score_fed_duo>((n_pos + 1) / 2, kDuoWarps);
        OEA_LAUNCH(k_score_fed_duo, grid, kDuoThreads, 0, (cudaStream_t)stream, e, r, F, *loss, loss_out);
        OEA_LAUNCH_CHECK();
        return OEA_OK;
    }
    const int grid = grid_for(n_pos);
#define CALL(V)                                                                                                           \
    if (l1) OEA_LAUNCH((k_score_fed_grouped<OEA_SCORE_L1, V>), grid, kThreads, 0, (cudaStream_t)stream, e, r, pos_h, pos_r, \
                       pos_t, n_pos, neg_h, neg_r, neg_t, k, *loss, loss_out);                                             \
    else OEA_LAUNCH((k_score_fed_grouped<OEA_SCORE_L2SQ, V>), grid, kThreads, 0, (cudaStream_t)stream, e, r, pos_h, pos_r, \
                    pos_t, n_pos, neg_h, neg_r, neg_t, k, *loss, loss_out)
    OEA_DISPATCH_VEC(ent->pitch, CALL);
#undef CALL
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
    FedBatch F{pos_h, pos_r, pos_t, neg_h, neg_r, neg_t, n_pos, k};
    if (ent->pitch <= 128 && k <= kDuoMaxK) {
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
         OEA_CUDA_TRY(OEA_LAUNCH_COOPERATIVE((k_step_fed_grouped<OEA_SCORE_L2SQ, V, KIND>), grid, kThreads, st, e, r, F, cfg, loss_out, A, B, lr)); \
    } while (0)
    if (ent->pitch <= 128) { if (opt->kind == OEA_OPT_ADAGRAD) OEA_RUN_STEP(1, OEA_OPT_ADAGRAD); else OEA_RUN_STEP(1, OEA_OPT_SGD); }
    else { if (opt->kind == OEA_OPT_ADAGRAD) OEA_RUN_STEP(2, OEA_OPT_ADAGRAD); else OEA_RUN_STEP(2, OEA_OPT_SGD); }
#undef OEA_RUN_STEP
    return OEA_OK;
}
