// oea_pipeline.cu — the fed step with HOST index buffers as a depth-2 pipeline: the host→device copy of step i+1
// overlaps the kernels of step i, and the host reads step i's loss while step i+1 runs.  Same kernels and the same
// strictly sequential table updates as oea_triple_step_fed_host (the session.run(feed_dict) boundary of
// models/basic_model.py:222-232); only the copies and the host wait move off the critical path.  sm_90a.
//
// Two slots, each with its own device index buffer, device loss scalar and pinned host loss scalar:
//   submit(slot):   copy stream   wait computed[slot]  (the slot's previous user has finished reading the buffers)
//                                 H2D pos / neg index vectors → idx[slot] ; record copied[slot]
//                   compute stream wait copied[slot] ; loss[slot] = 0 ; score ; row optimiser ; D2H loss[slot] ;
//                                 record computed[slot]
//   collect(slot):  host waits computed[slot], returns the loss
// The caller owns streams, events and buffers (no allocation here) and keeps a submitted step's pinned host index
// buffers untouched until that step's `copied` event has fired — with two host buffers used alternately that is
// guaranteed by collect(slot) of the step two submissions earlier.
#include <stdlib.h>

#include "oea_rowmath.cuh"

using namespace oea;

extern "C" int oea_triple_step_fed_host_submit(const oea_table* ent, const oea_table* rel, const oea_fed_pipeline* pipe,
                                               int32_t slot, const int32_t* pos_hrt_host, int32_t n_pos,
                                               const int32_t* neg_hrt_host, int32_t n_neg,
                                               const oea_loss_cfg* loss, const oea_opt_cfg* opt) {
    if (!pipe || !opt || !loss) return OEA_ERR_NULL;
    if (slot != 0 && slot != 1) return OEA_ERR_RANGE;
    if (!pipe->dev_idx[slot] || !pipe->dev_loss[slot] || !pipe->host_loss[slot] || !pipe->ev_copied[slot] ||
        !pipe->ev_computed[slot])
        return OEA_ERR_NULL;
    if (n_pos < 0 || n_neg < 0) return OEA_ERR_SHAPE;
    if ((n_pos > 0 && !pos_hrt_host) || (n_neg > 0 && !neg_hrt_host)) return OEA_ERR_NULL;
    cudaStream_t copy = (cudaStream_t)pipe->copy_stream, comp = (cudaStream_t)pipe->compute_stream;
    cudaEvent_t copied = (cudaEvent_t)pipe->ev_copied[slot], computed = (cudaEvent_t)pipe->ev_computed[slot];
    int32_t* dpos = pipe->dev_idx[slot];
    int32_t* dneg = dpos + 3 * (size_t)n_pos;
    OEA_CUDA_TRY(cudaStreamWaitEvent(copy, computed, 0));        // a never-recorded event is complete: the first use passes
    if (n_pos) OEA_CUDA_TRY(cudaMemcpyAsync(dpos, pos_hrt_host, 3 * (size_t)n_pos * sizeof(int32_t), cudaMemcpyHostToDevice, copy));
    if (n_neg) OEA_CUDA_TRY(cudaMemcpyAsync(dneg, neg_hrt_host, 3 * (size_t)n_neg * sizeof(int32_t), cudaMemcpyHostToDevice, copy));
    OEA_CUDA_TRY(cudaEventRecord(copied, copy));
    OEA_CUDA_TRY(cudaStreamWaitEvent(comp, copied, 0));
    OEA_CUDA_TRY(cudaMemsetAsync(pipe->dev_loss[slot], 0, sizeof(double), comp));
    // OEA_FED_GROUPED=1: same opt-in as oea_triple_step_fed_host (a positive scored together with its negatives)
    const char* grouped_env = getenv("OEA_FED_GROUPED");
    const bool grouped = grouped_env && grouped_env[0] == '1' && n_pos > 0 && n_neg % n_pos == 0;
    const char* fused_env = getenv("OEA_FED_FUSED");     // one cooperative launch (oea_triple_step_fed_grouped) where it applies
    int rc = OEA_ERR_KIND;
    if (fused_env && fused_env[0] == '1' && n_pos > 0 && n_neg % n_pos == 0)
        rc = oea_triple_step_fed_grouped(ent, rel, dpos, dpos + n_pos, dpos + 2 * (size_t)n_pos, n_pos,
                                         dneg, dneg + n_neg, dneg + 2 * (size_t)n_neg, n_neg, loss, opt, pipe->dev_loss[slot], comp);
    if (rc == OEA_ERR_KIND) {
        rc = grouped
            ? oea_triple_score_fed_grouped(ent, rel, dpos, dpos + n_pos, dpos + 2 * (size_t)n_pos, n_pos,
                                           dneg, dneg + n_neg, dneg + 2 * (size_t)n_neg, n_neg, loss, pipe->dev_loss[slot], comp)
            : oea_triple_score_fed(ent, rel, dpos, dpos + n_pos, dpos + 2 * (size_t)n_pos, n_pos,
                                   dneg, dneg + n_neg, dneg + 2 * (size_t)n_neg, n_neg, loss, pipe->dev_loss[slot], comp);
        if (rc) return rc;
        rc = oea_rowopt_apply_pair(ent, rel, opt, comp);
    }
    if (rc) return rc;
    OEA_CUDA_TRY(cudaMemcpyAsync(pipe->host_loss[slot], pipe->dev_loss[slot], sizeof(double), cudaMemcpyDeviceToHost, comp));
    OEA_CUDA_TRY(cudaEventRecord(computed, comp));
    return OEA_OK;
}

extern "C" int oea_triple_step_fed_host_collect(const oea_fed_pipeline* pipe, int32_t slot, float* loss_host) {
    if (!pipe || !loss_host) return OEA_ERR_NULL;
    if (slot != 0 && slot != 1) return OEA_ERR_RANGE;
    if (!pipe->ev_computed[slot] || !pipe->host_loss[slot]) return OEA_ERR_NULL;
    OEA_CUDA_TRY(cudaEventSynchronize((cudaEvent_t)pipe->ev_computed[slot]));
    *loss_host = (float)(*pipe->host_loss[slot]);
    return OEA_OK;
}
