// oea_transe.cuh — path (i)'s warp-per-row TransE (models/trans/transe.py:33-45, modules/base/losses.py:15-73,
// initializers.py:26): the one-triple context Triple<OEA_MODEL_TRANSE> and the per-positive body that scores a positive
// together with its k negatives, for both sources of a batch (fed index vectors, or the on-device sampler).  A row of
// `dim` floats is held as VEC float4 per lane (dim <= 128·VEC); row reductions are warp shuffles; gradients leave
// through red.global.add.v4.f32 into the gradient tables.  sm_90a.
#pragma once
#include "oea_rowmath.cuh"
#include "oea_sampler.cuh"

namespace oea {

// The tables of one model of the score-function family (oea_triple_ext.cu); TransE reads ent and rel only.
struct ModelDev {
    TableDev ent, rel, ent_aux, rel_aux;
    int dim;                 // columns that carry data (HolE's correlation wraps modulo dim)
    float gamma, phase;      // RotatE: γ and the phase scale π/ρ (oea_model.gamma / .phase); unused by the other kinds
};

// One triple of a model: forward() gathers and normalises its rows and returns the energy; backward(g) pushes
// g·dE/d(row) through the normalisations into the gradient tables and flags the rows.
template <int MODEL, int SCORE, int VEC>
struct Triple;

// TransE: E = ‖ĥ + r̂ − t̂‖ (L1) or its square (L2).  Also the general triple of the per-positive body below, and the
// triple of the weighted margin loss, where ent and rel may be the same table.  forward() = gather() + score() + the
// warp reduction: a kernel that scores a positive and a negative together issues both gathers first, so that six row
// loads are in flight before the first reduction, and reduces both scores in one pass.
template <int SCORE, int VEC>
struct Triple<OEA_MODEL_TRANSE, SCORE, VEC> {
    int h, r, t;
    NRow<VEC> xh, xr, xt;
    Row<VEC> u;
    __device__ __forceinline__ void gather(const ModelDev& M, int h_, int r_, int t_, int lane) {
        h = h_; r = r_; t = t_;
        xh.x = load_row<VEC>(M.ent.w, h, M.ent.pitch, lane);
        xr.x = load_row<VEC>(M.rel.w, r, M.rel.pitch, lane);
        xt.x = load_row<VEC>(M.ent.w, t, M.ent.pitch, lane);
    }
    __device__ __forceinline__ float score(const ModelDev& M) {
        xh.ss = sumsq(xh.x); xr.ss = sumsq(xr.x); xt.ss = sumsq(xt.x);
        warp_sum3(xh.ss, xr.ss, xt.ss);
        xh.inv = inv_norm(xh.ss, M.ent.norm); xr.inv = inv_norm(xr.ss, M.rel.norm); xt.inv = inv_norm(xt.ss, M.ent.norm);
        xh.x = r_scale(xh.x, xh.inv); xr.x = r_scale(xr.x, xr.inv); xt.x = r_scale(xt.x, xt.inv);
        u = r_sub(r_add(xh.x, xr.x), xt.x);
        return score_partial<SCORE, VEC>(u);          // this lane's share: the caller reduces
    }
    __device__ __forceinline__ float forward(const ModelDev& M, int h_, int r_, int t_, int lane) {
        gather(M, h_, r_, t_, lane);
        return warp_sum(score(M));
    }
    __device__ __forceinline__ void backward(const ModelDev& M, float g, int lane) {
        const Row<VEC> du = r_scale(score_dir<SCORE, VEC>(u), g);
        push<VEC>(M.ent, h, lane, du, xh);
        push<VEC>(M.rel, r, lane, du, xr);
        push<VEC>(M.ent, t, lane, r_neg(du), xt);
    }
};

// index vectors of a fed batch (device pointers) in the reference's layout: the k negatives of positive p at
// p·k … p·k+k−1 (modules/train/batch.py:36-45)
struct FedBatch {
    const int32_t* ph; const int32_t* pr; const int32_t* pt;
    const int32_t* nh; const int32_t* nr; const int32_t* nt;
    int n_pos, k;
};

// One warp per positive AND its k negatives.  The positive's three rows are loaded and normalised once, a negative that
// shares two of them loads one row, and the gradients of the shared rows are summed in registers (the Jacobian of
// l2_normalize is linear in the incoming gradient) and leave as three vector reductions per positive: 3 + k row loads
// and 3 + k row reductions per positive instead of 3·(1 + k) each.
//   SAMPLED (FED = false): the positive is drawn by the Feistel permutation of the step's slice and its negatives by
//     sample_negatives<32> (oea_sampler.cuh, modules/train/batch.py:89-119); `dbg` (optional) receives the draws.
//   FED: positive p and negatives p·k + j from F.  A negative that shares fewer than two rows with its positive (any
//     fed batch is legal) is scored as a general triple.
template <int SCORE, int VEC, bool FED>
__device__ __forceinline__ void positive_score_body(const TableDev& ent, const TableDev& rel, const SampledParams& P,
                                                    const FedBatch& F, const oea_loss_cfg& cfg, double* __restrict__ loss_out,
                                                    int32_t* __restrict__ dbg, double* s_loss) {
    uint64_t seed = 0;
    if (!FED) seed = P.dev_seed != nullptr ? P.seed ^ __ldg(reinterpret_cast<const unsigned long long*>(P.dev_seed)) : P.seed;
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    const int n_pos = FED ? F.n_pos : P.n_slice[0] + P.n_slice[1];
    const int k = FED ? F.k : P.k;
    const int sw = FED ? 1 : P.shard_world, sr = FED ? 0 : P.shard_rank;
    const bool margin_mode = cfg.loss_kind == OEA_LOSS_MARGIN;       // Σ relu(m + s⁺ − s⁻), k == 1
    const ModelDev M{ent, rel, ent, rel, 0, 0.f, 0.f};
    float warp_loss = 0.f;

    for (int p = warp_global * sw + sr; p < n_pos; p += n_warps * sw) {
        int h, r, t;
        int neg_e = 0;
        unsigned head_mask = 0u;
        if (FED) {
            h = __ldg(F.ph + p); r = __ldg(F.pr + p); t = __ldg(F.pt + p);
        } else {
            const SampledPositive s = draw_positive<32>(P, seed, p, lane, false, &ent, &rel);
            h = s.h; r = s.r; t = s.t;
            // lane j < k owns negative j
            bool neg_head = false;
            sample_negatives<32>(P, seed, P.kg[s.q], true, p, h, r, t, k, lane, neg_e, neg_head);
            head_mask = __ballot_sync(OEA_FULL, neg_head);
            if (dbg != nullptr) dump_draws<32>(dbg, p, k, s, head_mask, lane, neg_e);
        }

        // ---- positive triple ----
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

        // loss L and d loss / d s⁻ (g) of a negative of score sn; an active hinge also adds the positive's share to G*
        auto negative_loss = [&](float sn) {
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
        };

        // ---- negatives: only the corrupted row is new ----
        for (int j = 0; j < k; ++j) {
            int e, eh = 0, er = 0, et = 0;
            bool head, shared = true;
            if (FED) {
                const size_t q = (size_t)p * k + j;
                eh = __ldg(F.nh + q); er = __ldg(F.nr + q); et = __ldg(F.nt + q);
                const bool share_tail = er == r && et == t;          // head corrupted (or an exact copy of the positive)
                const bool share_head = er == r && eh == h;          // tail corrupted
                shared = share_tail || share_head;
                head = share_tail;                                   // the row that is new: the head (else the tail)
                e = head ? eh : et;
            } else {
                e = __shfl_sync(OEA_FULL, neg_e, j);
                head = (head_mask >> j) & 1u;
            }
            if (shared) {
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
                negative_loss(sn);
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
                Triple<OEA_MODEL_TRANSE, SCORE, VEC> N;              // nothing to share with the positive
                negative_loss(N.forward(M, eh, er, et, lane));
                if (g != 0.f) N.backward(M, g, lane);
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

}  // namespace oea
