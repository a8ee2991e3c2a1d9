// oea_pipeline.cu — the fed step with HOST index buffers (the session.run(feed_dict) boundary of
// models/basic_model.py:222-232): the synchronous oea_triple_step_fed_host, and the same step as a depth-2 pipeline in
// which the host→device copy of step i+1 overlaps the kernels of step i and the host reads step i's loss while step
// i+1 runs.  Both run the same kernels (fed_step_kernels) and the same strictly sequential table updates; the pipeline
// only moves the copies and the host wait off the critical path.  sm_90a.
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

static bool env_is_1(const char* name) {
    const char* v = getenv(name);   // read per call: bench.py and the tests flip it inside one process
    return v != nullptr && v[0] == '1';
}

// The kernels of one fed step on device index vectors dpos = [3, n_pos] h|r|t and dneg = [3, n_neg], on `stream`:
//   OEA_FED_FUSED=1:   grouped scoring and the row optimiser as one cooperative launch (oea_triple_step_fed_grouped)
//                      where that kernel applies, otherwise as below;
//   OEA_FED_GROUPED=1: a positive scored together with its negatives (oea_triple_score_fed_grouped), else one warp per
//                      triple (oea_triple_score_fed); then oea_rowopt_apply_pair.
// Both switches need the reference's layout (n_neg a multiple of n_pos).
static int fed_step_kernels(const oea_table* ent, const oea_table* rel, const int32_t* dpos, int32_t n_pos,
                            const int32_t* dneg, int32_t n_neg, const oea_loss_cfg* loss, const oea_opt_cfg* opt,
                            double* dev_loss, void* stream) {
    const bool layout = n_pos > 0 && n_neg % n_pos == 0;
    const int32_t *ph = dpos, *pr = dpos + n_pos, *pt = dpos + 2 * (size_t)n_pos;
    const int32_t *nh = dneg, *nr = dneg + n_neg, *nt = dneg + 2 * (size_t)n_neg;
    int rc = OEA_ERR_KIND;
    if (layout && env_is_1("OEA_FED_FUSED"))
        rc = oea_triple_step_fed_grouped(ent, rel, ph, pr, pt, n_pos, nh, nr, nt, n_neg, loss, opt, dev_loss, stream);
    if (rc != OEA_ERR_KIND) return rc;
    rc = layout && env_is_1("OEA_FED_GROUPED")
        ? oea_triple_score_fed_grouped(ent, rel, ph, pr, pt, n_pos, nh, nr, nt, n_neg, loss, dev_loss, stream)
        : oea_triple_score_fed(ent, rel, ph, pr, pt, n_pos, nh, nr, nt, n_neg, loss, dev_loss, stream);
    if (rc) return rc;
    return oea_rowopt_apply_pair(ent, rel, opt, stream);
}

extern "C" int oea_triple_step_fed_host(const oea_table* ent, const oea_table* rel,
                                        const int32_t* pos_hrt_host, int32_t n_pos,
                                        const int32_t* neg_hrt_host, int32_t n_neg,
                                        const oea_loss_cfg* loss, const oea_opt_cfg* opt,
                                        int32_t* dev_idx_ws, double* dev_loss_ws, double* loss_pinned_host,
                                        float* loss_host, void* stream) {
    if (!dev_idx_ws || !dev_loss_ws || !loss_pinned_host || !loss_host || !opt) return OEA_ERR_NULL;
    if (n_pos < 0 || n_neg < 0) return OEA_ERR_SHAPE;
    if ((n_pos > 0 && !pos_hrt_host) || (n_neg > 0 && !neg_hrt_host)) return OEA_ERR_NULL;
    cudaStream_t st = (cudaStream_t)stream;
    int32_t* dpos = dev_idx_ws;
    int32_t* dneg = dev_idx_ws + 3 * (size_t)n_pos;
    if (n_pos) OEA_CUDA_TRY(cudaMemcpyAsync(dpos, pos_hrt_host, 3 * (size_t)n_pos * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    if (n_neg) OEA_CUDA_TRY(cudaMemcpyAsync(dneg, neg_hrt_host, 3 * (size_t)n_neg * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OEA_CUDA_TRY(cudaMemsetAsync(dev_loss_ws, 0, sizeof(double), st));
    const int rc = fed_step_kernels(ent, rel, dpos, n_pos, dneg, n_neg, loss, opt, dev_loss_ws, stream);
    if (rc) return rc;
    OEA_CUDA_TRY(cudaMemcpyAsync(loss_pinned_host, dev_loss_ws, sizeof(double), cudaMemcpyDeviceToHost, st));
    OEA_CUDA_TRY(cudaStreamSynchronize(st));
    *loss_host = (float)(*loss_pinned_host);
    return OEA_OK;
}

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
    const int rc = fed_step_kernels(ent, rel, dpos, n_pos, dneg, n_neg, loss, opt, pipe->dev_loss[slot], comp);
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
