// oea_triple.cu — path (i): negative-sampled triple scoring forward+backward (K1), the row
// optimiser, the fused on-device sampler, and the table lookup.  sm_90a.
//
// Maths restated from the reference (no code shared):
//   modules/base/losses.py:15-73      score + losses (sums, squared L2)
//   modules/base/initializers.py:26   l2_normalize wrapper around every lookup
//   modules/base/optimizers.py:10-20  TF1 Adagrad / Adam / SGD
//   modules/train/batch.py:36-119     batch slicing + corrupt-head/tail negative sampling
//   approaches/bootea.py:197          alignment loss
//
// Work decomposition: one warp per triple (fed path) or per positive + its k negatives (sampled
// path).  A row of `dim` floats is held as VEC float4 per lane (dim <= 128·VEC), loaded with
// 128-bit coalesced reads; row reductions are warp shuffles; gradients leave through 128-bit
// vector reductions (red.global.add.v4.f32) into the L2-resident gradient table.
#include <stdlib.h>
#include "oea_rowmath.cuh"
#include "oea_rowopt.cuh"
#include "oea_sampler.cuh"
#include "oea_duo.cuh"
#include <cooperative_groups.h>

namespace oea {

// ------------------------------------------------------------------------------------------------
// Fed path, independent losses (limited / logistic / positive / logsigmoid): one warp per triple.
// ------------------------------------------------------------------------------------------------
template <int SCORE, int VEC>
__global__ void __launch_bounds__(kThreads)
k_score_fed(TableDev ent, TableDev rel,
            const int32_t* __restrict__ ph, const int32_t* __restrict__ pr, const int32_t* __restrict__ pt, int n_pos,
            const int32_t* __restrict__ nh, const int32_t* __restrict__ nr, const int32_t* __restrict__ nt, int n_neg,
            oea_loss_cfg cfg, double* __restrict__ loss_out) {
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
        Row<VEC> xh = load_row<VEC>(ent.w, h, ent.pitch, lane);
        Row<VEC> xr = load_row<VEC>(rel.w, r, rel.pitch, lane);
        Row<VEC> xt = load_row<VEC>(ent.w, t, ent.pitch, lane);
        float ssh = sumsq(xh), ssr = sumsq(xr), sst = sumsq(xt);
        warp_sum3(ssh, ssr, sst);
        const float ih = inv_norm(ssh, ent.norm), ir = inv_norm(ssr, rel.norm), it = inv_norm(sst, ent.norm);
        Row<VEC> u;
#pragma unroll
        for (int c = 0; c < VEC; ++c) {
            xh.v[c] = xh.v[c] * ih; xr.v[c] = xr.v[c] * ir; xt.v[c] = xt.v[c] * it;
            u.v[c] = xh.v[c] + xr.v[c] - xt.v[c];
        }
        const float s = warp_sum(score_partial<SCORE, VEC>(u));
        float L, g;
        loss_of(cfg.loss_kind, is_neg, s, cfg, L, g);
        warp_loss += L;
        if (g != 0.f) {
            Row<VEC> du = score_dir<SCORE, VEC>(u);
#pragma unroll
            for (int c = 0; c < VEC; ++c) du.v[c] = du.v[c] * g;
            float dh = dotr(xh, du), dr = dotr(xr, du), dt = dotr(xt, du);
            warp_sum3(dh, dr, dt);
            Row<VEC> gh = through_norm(du, xh, dh, ih, ssh, ent.norm);
            Row<VEC> gr = through_norm(du, xr, dr, ir, ssr, rel.norm);
            Row<VEC> gt = through_norm(du, xt, dt, it, sst, ent.norm);
#pragma unroll
            for (int c = 0; c < VEC; ++c) gt.v[c] = neg(gt.v[c]);
            red_row<VEC>(ent.g, h, ent.pitch, lane, gh);
            red_row<VEC>(rel.g, r, rel.pitch, lane, gr);
            red_row<VEC>(ent.g, t, ent.pitch, lane, gt);
            if (lane == 0) { ent.touched[h] = 1; rel.touched[r] = 1; ent.touched[t] = 1; }
        }
    }
    LossAcc acc{s_loss};
    acc.flush(warp_loss, loss_out);
}

// ------------------------------------------------------------------------------------------------
// Fed path, margin-based loss Σ relu(m + s⁺_i − s⁻_i) (losses.py:15-27; k = 1): warp per pair.
// ------------------------------------------------------------------------------------------------
template <int SCORE, int VEC>
__global__ void __launch_bounds__(kThreads)
k_score_margin(TableDev ent, TableDev rel,
               const int32_t* __restrict__ ph, const int32_t* __restrict__ pr, const int32_t* __restrict__ pt,
               const int32_t* __restrict__ nh, const int32_t* __restrict__ nr, const int32_t* __restrict__ nt, int n,
               oea_loss_cfg cfg, double* __restrict__ loss_out) {
    __shared__ double s_loss[kWarpsPerBlock];
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    float warp_loss = 0.f;

    for (int i = warp_global; i < n; i += n_warps) {
        int idx[2][3] = {{__ldg(ph + i), __ldg(pr + i), __ldg(pt + i)}, {__ldg(nh + i), __ldg(nr + i), __ldg(nt + i)}};
        Row<VEC> xh[2], xr[2], xt[2], u[2];
        float ih[2], ir[2], it[2], ssh[2], ssr[2], sst[2], s[2];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            xh[q] = load_row<VEC>(ent.w, idx[q][0], ent.pitch, lane);
            xr[q] = load_row<VEC>(rel.w, idx[q][1], rel.pitch, lane);
            xt[q] = load_row<VEC>(ent.w, idx[q][2], ent.pitch, lane);
        }
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            ssh[q] = sumsq(xh[q]); ssr[q] = sumsq(xr[q]); sst[q] = sumsq(xt[q]);
            warp_sum3(ssh[q], ssr[q], sst[q]);
            ih[q] = inv_norm(ssh[q], ent.norm); ir[q] = inv_norm(ssr[q], rel.norm); it[q] = inv_norm(sst[q], ent.norm);
#pragma unroll
            for (int c = 0; c < VEC; ++c) {
                xh[q].v[c] = xh[q].v[c] * ih[q]; xr[q].v[c] = xr[q].v[c] * ir[q]; xt[q].v[c] = xt[q].v[c] * it[q];
                u[q].v[c] = xh[q].v[c] + xr[q].v[c] - xt[q].v[c];
            }
            s[q] = score_partial<SCORE, VEC>(u[q]);
        }
        warp_sum2(s[0], s[1]);
        const float v = cfg.margin + s[0] - s[1];
        warp_loss += fmaxf(v, 0.f);
        if (v > 0.f) {
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const float g = q == 0 ? 1.f : -1.f;
                Row<VEC> du = score_dir<SCORE, VEC>(u[q]);
#pragma unroll
                for (int c = 0; c < VEC; ++c) du.v[c] = du.v[c] * g;
                float dh = dotr(xh[q], du), dr = dotr(xr[q], du), dt = dotr(xt[q], du);
                warp_sum3(dh, dr, dt);
                Row<VEC> gh = through_norm(du, xh[q], dh, ih[q], ssh[q], ent.norm);
                Row<VEC> gr = through_norm(du, xr[q], dr, ir[q], ssr[q], rel.norm);
                Row<VEC> gt = through_norm(du, xt[q], dt, it[q], sst[q], ent.norm);
#pragma unroll
                for (int c = 0; c < VEC; ++c) gt.v[c] = neg(gt.v[c]);
                red_row<VEC>(ent.g, idx[q][0], ent.pitch, lane, gh);
                red_row<VEC>(rel.g, idx[q][1], rel.pitch, lane, gr);
                red_row<VEC>(ent.g, idx[q][2], ent.pitch, lane, gt);
                if (lane == 0) { ent.touched[idx[q][0]] = 1; rel.touched[idx[q][1]] = 1; ent.touched[idx[q][2]] = 1; }
            }
        }
    }
    LossAcc acc{s_loss};
    acc.flush(warp_loss, loss_out);
}

// ------------------------------------------------------------------------------------------------
// Fused sampled step: warp per positive; samples its k negatives on device, loads 3 + k rows,
// keeps the gradients of the three shared rows in registers, and issues 3 + k row reductions.
// ------------------------------------------------------------------------------------------------
template <int SCORE, int VEC>
__global__ void __launch_bounds__(kThreads)
k_score_sampled(TableDev ent, TableDev rel, SampledParams P, oea_loss_cfg cfg,
                double* __restrict__ loss_out, int32_t* __restrict__ dbg) {
    __shared__ double s_loss[kWarpsPerBlock];
    if (P.dev_seed != nullptr) P.seed ^= __ldg(reinterpret_cast<const unsigned long long*>(P.dev_seed));
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    const int n_pos = P.n_slice[0] + P.n_slice[1];
    const int k = P.k;
    float warp_loss = 0.f;

    for (int p = warp_global * P.shard_world + P.shard_rank; p < n_pos; p += n_warps * P.shard_world) {
        const int q = p < P.n_slice[0] ? 0 : 1;
        const oea_kg_view& kg = P.kg[q];
        const int local = q == 0 ? p : p - P.n_slice[0];
        const uint32_t tri = feistel_perm((uint32_t)(P.start[q] + local), (uint32_t)kg.n_triples,
                                          P.seed ^ (q ? 0xA5A5A5A5DEADBEEFull : 0x0123456789ABCDEFull));
        int hrt = 0;
        if (lane < 3) hrt = __ldg(kg.triples + 3 * (size_t)tri + lane);
        const int h = __shfl_sync(OEA_FULL, hrt, 0);
        const int r = __shfl_sync(OEA_FULL, hrt, 1);
        const int t = __shfl_sync(OEA_FULL, hrt, 2);
        if (lane < 3) {   // overlap the three shared rows' fetch with the sampling chain
            const float* rowp = lane == 1 ? rel.w + (size_t)r * rel.pitch : ent.w + (size_t)(lane == 0 ? h : t) * ent.pitch;
            prefetch_row_l2(rowp, ent.pitch);
        }

        // ---- negative sampling (batch.py:89-119), lane j < k owns negative j ----
        int neg_e = 0;
        bool neg_head = false;
        warp_sample_negatives(P, P.seed, kg, p, h, r, t, k, lane, ent.w, ent.pitch, neg_e, neg_head);
        const unsigned head_mask = __ballot_sync(OEA_FULL, neg_head);
        if (dbg != nullptr) {
            int32_t* row = dbg + (size_t)p * (2 + k);
            if (lane == 0) { row[0] = (int32_t)tri + (q ? (1 << 30) : 0); row[1] = (int32_t)head_mask; }
            if (lane < k) row[2 + lane] = neg_e;
        }

        // ---- positive triple ----
        Row<VEC> xh = load_row<VEC>(ent.w, h, ent.pitch, lane);
        Row<VEC> xr = load_row<VEC>(rel.w, r, rel.pitch, lane);
        Row<VEC> xt = load_row<VEC>(ent.w, t, ent.pitch, lane);
        float ssh = sumsq(xh), ssr = sumsq(xr), sst = sumsq(xt);
        warp_sum3(ssh, ssr, sst);
        const float ih = inv_norm(ssh, ent.norm), ir = inv_norm(ssr, rel.norm), it = inv_norm(sst, ent.norm);
        Row<VEC> hr, rt, u, Gh, Gr, Gt;  // hr = ĥ + r̂, rt = r̂ − t̂
#pragma unroll
        for (int c = 0; c < VEC; ++c) {
            xh.v[c] = xh.v[c] * ih; xr.v[c] = xr.v[c] * ir; xt.v[c] = xt.v[c] * it;
            hr.v[c] = xh.v[c] + xr.v[c];
            rt.v[c] = xr.v[c] - xt.v[c];
            u.v[c] = hr.v[c] - xt.v[c];
        }
        const float sp = warp_sum(score_partial<SCORE, VEC>(u));
        const bool margin_mode = cfg.loss_kind == OEA_LOSS_MARGIN;   // Σ relu(m + s⁺ − s⁻), k == 1
        float L = 0.f, g = 0.f;
        if (!margin_mode) loss_of(cfg.loss_kind, false, sp, cfg, L, g);
        warp_loss += L;
        bool any_grad = g != 0.f;
        const Row<VEC> dir_pos = score_dir<SCORE, VEC>(u);
#pragma unroll
        for (int c = 0; c < VEC; ++c) { Gh.v[c] = dir_pos.v[c] * g; Gr.v[c] = Gh.v[c]; Gt.v[c] = neg(Gh.v[c]); }

        // ---- negatives: only the corrupted row is new ----
        for (int j = 0; j < k; ++j) {
            const int e = __shfl_sync(OEA_FULL, neg_e, j);
            const bool head = (head_mask >> j) & 1u;
            Row<VEC> xe = load_row<VEC>(ent.w, e, ent.pitch, lane);
            const float sse = warp_sum(sumsq(xe));
            const float ie = inv_norm(sse, ent.norm);
#pragma unroll
            for (int c = 0; c < VEC; ++c) {
                xe.v[c] = xe.v[c] * ie;
                u.v[c] = head ? (xe.v[c] + rt.v[c]) : (hr.v[c] - xe.v[c]);
            }
            Row<VEC> dir = score_dir<SCORE, VEC>(u);
            float sn = score_partial<SCORE, VEC>(u), de = dotr(xe, dir);
            warp_sum2(sn, de);
            if (margin_mode) {
                const float v = cfg.margin + sp - sn;
                L = fmaxf(v, 0.f);
                g = v > 0.f ? -1.f : 0.f;
                if (v > 0.f) {   // the positive's share of the active hinge
#pragma unroll
                    for (int c = 0; c < VEC; ++c) { Gh.v[c] = Gh.v[c] + dir_pos.v[c]; Gr.v[c] = Gr.v[c] + dir_pos.v[c]; Gt.v[c] = Gt.v[c] - dir_pos.v[c]; }
                }
            } else {
                loss_of(cfg.loss_kind, true, sn, cfg, L, g);
            }
            warp_loss += L;
            if (g != 0.f) {
                any_grad = true;
                const float ge = head ? g : -g;  // d/dê = ±g·dir
                Row<VEC> Ge;
#pragma unroll
                for (int c = 0; c < VEC; ++c) {
                    const float4 du = dir.v[c] * g;
                    Gr.v[c] = Gr.v[c] + du;
                    if (head) Gt.v[c] = Gt.v[c] - du; else Gh.v[c] = Gh.v[c] + du;
                    Ge.v[c] = dir.v[c] * ge;
                }
                Row<VEC> out = through_norm(Ge, xe, ge * de, ie, sse, ent.norm);
                red_row<VEC>(ent.g, e, ent.pitch, lane, out);
                if (lane == 0) ent.touched[e] = 1;
            }
        }

        if (any_grad) {
            float dh = dotr(xh, Gh), dr = dotr(xr, Gr), dt = dotr(xt, Gt);
            warp_sum3(dh, dr, dt);
            Row<VEC> oh = through_norm(Gh, xh, dh, ih, ssh, ent.norm);
            Row<VEC> orr = through_norm(Gr, xr, dr, ir, ssr, rel.norm);
            Row<VEC> ot = through_norm(Gt, xt, dt, it, sst, ent.norm);
            red_row<VEC>(ent.g, h, ent.pitch, lane, oh);
            red_row<VEC>(rel.g, r, rel.pitch, lane, orr);
            red_row<VEC>(ent.g, t, ent.pitch, lane, ot);
            if (lane == 0) { ent.touched[h] = 1; rel.touched[r] = 1; ent.touched[t] = 1; }
        }
    }
    LossAcc acc{s_loss};
    acc.flush(warp_loss, loss_out);
}


// ------------------------------------------------------------------------------------------------
// Fused sampled step, v2 ("octet" layout) for the squared-L2 score and pitch <= 128 floats:
// 8 lanes hold one row (4 float4 per lane), so a warp works on 4 rows at once — the three reductions of
// a row are 3 shuffle steps shared by 4 rows instead of 5 steps per row, and 4 row gathers are in flight
// per warp.  Because the score is quadratic, the gradients of the three shared rows are affine in the
// negatives: only Σ g_j·ê_j (per corrupted side) and Σ g_j are accumulated per octet, merged across the
// 4 octets once, and octets 0/1/2 finish rows h / r / t.
// ------------------------------------------------------------------------------------------------
#ifndef OEA_OCT_WARPS
#define OEA_OCT_WARPS 4
#endif
#ifndef OEA_OCT_MINB
#define OEA_OCT_MINB 6       // 6 CTAs × 4 warps: at most 80 registers per thread
#endif
#ifndef OEA_OCT_E_SMEM
#define OEA_OCT_E_SMEM 1
#endif
constexpr int kOctWarps = OEA_OCT_WARPS;      // warps per CTA of the octet kernel
constexpr int kOctThreads = kOctWarps * OEA_WARP;

// Per-warp staging in shared memory.  The kernel is issue-latency bound (≈2 000 warp instructions per positive on
// a chain of 5 dependent memory hops), so what matters is resident warps per scheduler: keeping ĥ+r̂ / r̂−t̂ (read-only
// in phase 2, one copy per warp, broadcast to the 4 octets) and the per-octet Σ g·ê accumulators out of the register
// file takes the kernel from 128 to ≤ 64 registers, i.e. from 16 to 32 resident warps per SM.
struct OctStage {
    float4 hr[4][8];     // ĥ + r̂   (slot q = l + 8·i)
    float4 rt[4][8];     // r̂ − t̂
#if OEA_OCT_E_SMEM
    float4 Eh[4][32];    // Σ g_j·ê_j over this lane's octet, head-corrupted negatives
    float4 Et[4][32];    //                                  tail-corrupted
#endif
};

__device__ __forceinline__ void oct_score_body(const TableDev& ent, const TableDev& rel, const SampledParams& P,
                                               const oea_loss_cfg& cfg, double* __restrict__ loss_out,
                                               int32_t* __restrict__ dbg, double* s_loss, OctStage* s_stage) {
    // P stays in the constant bank (P.kg[q] is indexed there, no local copy); the per-replay seed is a register
    const uint64_t seed = P.dev_seed != nullptr ? P.seed ^ __ldg(reinterpret_cast<const unsigned long long*>(P.dev_seed))
                                                : P.seed;
    const int lane = threadIdx.x & 31, oct = lane >> 3, l = lane & 7;
    OctStage& S = s_stage[threadIdx.x >> 5];
    const int warp_global = blockIdx.x * kOctWarps + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kOctWarps;
    const int n_pos = P.n_slice[0] + P.n_slice[1];
    const int k = P.k;
    const int p4 = ent.pitch >> 2;
    const bool margin_mode = cfg.loss_kind == OEA_LOSS_MARGIN;
    float lane_loss = 0.f;

    for (int p = warp_global * P.shard_world + P.shard_rank; p < n_pos; p += n_warps * P.shard_world) {
        const int q = p < P.n_slice[0] ? 0 : 1;
        const oea_kg_view& kg = P.kg[q];
        const int local = q == 0 ? p : p - P.n_slice[0];
        const uint32_t tri = (P.diag & 8) ? (uint32_t)(P.start[q] + local)
                                          : feistel_perm((uint32_t)(P.start[q] + local), (uint32_t)kg.n_triples,
                                                         seed ^ (q ? 0xA5A5A5A5DEADBEEFull : 0x0123456789ABCDEFull));
        int hrt = 0;
        if (lane < 3) hrt = __ldg(kg.triples + 3 * (size_t)tri + lane);
        const int h = __shfl_sync(OEA_FULL, hrt, 0);
        const int r = __shfl_sync(OEA_FULL, hrt, 1);
        const int t = __shfl_sync(OEA_FULL, hrt, 2);
        if (lane < 3) {   // overlap the three shared rows' fetch with the sampling chain
            const float* rowp = lane == 1 ? rel.w + (size_t)r * rel.pitch : ent.w + (size_t)(lane == 0 ? h : t) * ent.pitch;
            prefetch_row_l2(rowp, ent.pitch);
        }

        int neg_e = 0;
        bool neg_head = false;
        if (P.diag & 1) { neg_e = __ldg(kg.entities + (uint32_t)(p * 31 + lane * 977) % (uint32_t)kg.n_entities); neg_head = (p + lane) & 1; }
        else warp_sample_negatives(P, seed, kg, p, h, r, t, k, lane, ent.w, ent.pitch, neg_e, neg_head);
        const unsigned head_mask = __ballot_sync(OEA_FULL, neg_head);
        if (dbg != nullptr) {
            int32_t* row = dbg + (size_t)p * (2 + k);
            if (lane == 0) { row[0] = (int32_t)tri + (q ? (1 << 30) : 0); row[1] = (int32_t)head_mask; }
            if (lane < k) row[2 + lane] = neg_e;
        }

        // ---- phase 1: the three shared rows (every octet computes the same copy; octet 0 stages it) ----
        float ih, ir, it, ssh, ssr, sst, sp;
        __syncwarp();   // the previous positive's phase 3 has finished reading the stage
        {
            const R4 xh = load_oct(ent.w, h, ent.pitch, l, p4);
            const R4 xr = load_oct(rel.w, r, rel.pitch, l, p4);
            const R4 xt = load_oct(ent.w, t, ent.pitch, l, p4);
            {
                float2 ah = make_float2(0.f, 0.f), ar = ah, at = ah;
#pragma unroll
                for (int i = 0; i < 4; ++i) { dot4_acc2(ah, xh.v[i], xh.v[i]); dot4_acc2(ar, xr.v[i], xr.v[i]); dot4_acc2(at, xt.v[i], xt.v[i]); }
                ssh = oct_sum(ah.x + ah.y); ssr = oct_sum(ar.x + ar.y); sst = oct_sum(at.x + at.y);
            }
            ih = inv_norm(ssh, ent.norm); ir = inv_norm(ssr, rel.norm); it = inv_norm(sst, ent.norm);
            float2 sp_part = make_float2(0.f, 0.f);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float4 a = xh.v[i] * ih, b = xr.v[i] * ir, c = xt.v[i] * it;
                const float4 hr = a + b, rt = b - c;
                if (oct == 0) { S.hr[i][l] = hr; S.rt[i][l] = rt; }
                const float4 up = hr - c;
                dot4_acc2(sp_part, up, up);
#if OEA_OCT_E_SMEM
                S.Eh[i][lane] = f4(0.f);
                S.Et[i][lane] = f4(0.f);
#endif
            }
            sp = oct_sum(sp_part.x + sp_part.y);
        }
        __syncwarp();
        float Lp = 0.f, gp = 0.f;
        if (!margin_mode) loss_of(cfg.loss_kind, false, sp, cfg, Lp, gp);
        if (lane == 0) lane_loss += Lp;

        // ---- phase 2: negatives, four at a time (octet o takes negative 4·round + o) ----
#if !OEA_OCT_E_SMEM
        R4 Eh, Et;   // Σ g_j·ê_j over head- / tail-corrupted negatives of this octet
#pragma unroll
        for (int i = 0; i < 4; ++i) { Eh.v[i] = f4(0.f); Et.v[i] = f4(0.f); }
#endif
        float Gh_s = 0.f, Gt_s = 0.f;
        const int rounds = (P.diag & 4) ? 0 : (k + 3) >> 2;
        for (int round = 0; round < rounds; ++round) {
            const int j = 4 * round + oct;
            const bool valid = j < k;
            const int e_id = __shfl_sync(OEA_FULL, neg_e, valid ? j : 0);
            const bool head = (head_mask >> (valid ? j : 0)) & 1u;
            R4 e = load_oct(ent.w, valid ? e_id : h, ent.pitch, l, p4);
            float2 sse2 = make_float2(0.f, 0.f);
#pragma unroll
            for (int i = 0; i < 4; ++i) dot4_acc2(sse2, e.v[i], e.v[i]);
            const float sse = oct_sum(sse2.x + sse2.y);
            const float ie = inv_norm(sse, ent.norm);
            // u = ê + (r̂ − t̂) for a corrupted head, (ĥ + r̂) − ê for a corrupted tail
            const float4* base = head ? &S.rt[0][0] : &S.hr[0][0];
            const float sgn = head ? 1.f : -1.f;
            R4 u;
            float2 s_part = make_float2(0.f, 0.f), d_part = s_part;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                e.v[i] = e.v[i] * ie;
                u.v[i] = fma4(e.v[i], sgn, base[i * 8 + l]);
                dot4_acc2(s_part, u.v[i], u.v[i]);
                dot4_acc2(d_part, e.v[i], u.v[i]);
            }
            const float sn = oct_sum(s_part.x + s_part.y);
            const float de = oct_sum(d_part.x + d_part.y);
            float L = 0.f, g = 0.f;
            if (margin_mode) {
                const float v = cfg.margin + sp - sn;
                L = fmaxf(v, 0.f);
                g = v > 0.f ? -1.f : 0.f;
                if (valid && v > 0.f) gp = 1.f;   // k == 1: only octet 0 is valid; broadcast below
            } else {
                loss_of(cfg.loss_kind, true, sn, cfg, L, g);
            }
            if (!valid) { L = 0.f; g = 0.f; }
            if (l == 0) lane_loss += L;
            if (g != 0.f) {
                // d s/d ê = ±2u ; through the normaliser: (ĝ − ê<ê,ĝ>)/‖x‖
                const float c = 2.f * sgn * g * ie;
                const float proj = (ent.norm && sse >= kNormEps) ? de : 0.f;
#if OEA_OCT_E_SMEM
                float4* acc = head ? &S.Eh[0][0] : &S.Et[0][0];
#endif
                float* grow = ent.g + (size_t)e_id * ent.pitch;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
#if OEA_OCT_E_SMEM
                    acc[i * 32 + lane] = fma4(e.v[i], g, acc[i * 32 + lane]);
#else
                    if (head) Eh.v[i] = fma4(e.v[i], g, Eh.v[i]); else Et.v[i] = fma4(e.v[i], g, Et.v[i]);
#endif
                    if (!(P.diag & 2) && l + 8 * i < p4) red_add4(grow + 4 * (l + 8 * i), fma4(e.v[i], -proj, u.v[i]) * c);
                }
                if (head) Gh_s += g; else Gt_s += g;
                if (!(P.diag & 2) && l == 0) ent.touched[e_id] = 1;
            }
        }
        if (margin_mode) gp = __shfl_sync(OEA_FULL, gp, 0);

        // ---- phase 3: merge the octets, finish rows h (octet 0), r (octet 1), t (octet 2) ----
        Gh_s = cross_oct_sum(Gh_s);
        Gt_s = cross_oct_sum(Gt_s);
        __syncwarp();   // the accumulators of all four octets are visible
        if (gp != 0.f || Gh_s != 0.f || Gt_s != 0.f) {
            // all four octets run the same arithmetic on their own row (full-mask shuffles inside); octet 3
            // mirrors octet 2 and writes nothing.  Ĝ = α·P + β·A + γ·B with per-role scalars:
            //   h: P + A      r: P + A + B      t: −P − B      (P = 2g⁺u⁺, A = 2(G_t·hr − E_t), B = 2(G_h·rt + E_h))
            const int role = oct < 3 ? oct : 2;
            const int row = role == 0 ? h : (role == 1 ? r : t);
            const TableDev& tab = role == 1 ? rel : ent;
            const R4 xo = load_oct(tab.w, row, tab.pitch, l, p4);                    // L1 hit
            const float io = role == 0 ? ih : (role == 1 ? ir : it);
            const float so = role == 0 ? ssh : (role == 1 ? ssr : sst);
            const float alpha = role == 2 ? -2.f * gp : 2.f * gp;
            const float beta = role == 2 ? 0.f : 2.f, gamma = role == 0 ? 0.f : (role == 1 ? 2.f : -2.f);
            // u⁺ = hr − t̂ and t̂ = r̂ − rt... kept affine in the staged rows: α·u⁺ = α·hr − α·t̂, t̂ reloaded (L1 hit)
            const R4 xt = load_oct(ent.w, t, ent.pitch, l, p4);
            const float c_hr = alpha + beta * Gt_s, c_rt = gamma * Gh_s, c_t = -alpha * it;
            R4 G;
            float2 dpart2 = make_float2(0.f, 0.f);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
#if OEA_OCT_E_SMEM
                const float4 eh = (S.Eh[i][l] + S.Eh[i][8 + l]) + (S.Eh[i][16 + l] + S.Eh[i][24 + l]);
                const float4 et = (S.Et[i][l] + S.Et[i][8 + l]) + (S.Et[i][16 + l] + S.Et[i][24 + l]);
#else
                float4 eh = Eh.v[i], et = Et.v[i];
                eh.x = cross_oct_sum(eh.x); eh.y = cross_oct_sum(eh.y); eh.z = cross_oct_sum(eh.z); eh.w = cross_oct_sum(eh.w);
                et.x = cross_oct_sum(et.x); et.y = cross_oct_sum(et.y); et.z = cross_oct_sum(et.z); et.w = cross_oct_sum(et.w);
#endif
                // α(hr − t̂) + β(G_t·hr − E_t) + γ(G_h·rt + E_h)
                float4 g4 = S.hr[i][l] * c_hr;
                g4 = fma4(S.rt[i][l], c_rt, g4);
                g4 = fma4(xt.v[i], c_t, g4);
                g4 = fma4(et, -beta, g4);
                g4 = fma4(eh, gamma, g4);
                G.v[i] = g4;
                dot4_acc2(dpart2, xo.v[i], g4);
            }
            const float dot = oct_sum((dpart2.x + dpart2.y) * io);
            const float proj = (tab.norm && so >= kNormEps) ? dot : 0.f;
            if (oct < 3 && !(P.diag & 2)) {
                R4 out;
#pragma unroll
                for (int i = 0; i < 4; ++i) out.v[i] = fma4(xo.v[i] * io, -proj, G.v[i]) * io;
                red_oct(tab.g, row, tab.pitch, l, p4, out);
                if (l == 0) tab.touched[row] = 1;
            }
        }
    }
    const float warp_loss = warp_sum(lane_loss);
    LossAcc acc{s_loss};
    acc.flush(warp_loss, loss_out, kOctWarps);
}

__global__ void __launch_bounds__(kOctThreads, OEA_OCT_MINB)
k_score_sampled_oct(TableDev ent, TableDev rel, const __grid_constant__ SampledParams P, oea_loss_cfg cfg,
                    double* __restrict__ loss_out, int32_t* __restrict__ dbg) {
    __shared__ double s_loss[kOctWarps];
    __shared__ OctStage s_stage[kOctWarps];
    oct_score_body(ent, rel, P, cfg, loss_out, dbg, s_loss, s_stage);
}

// The whole sampled training step as ONE cooperative launch: score + gradients, grid barrier, row optimiser.
// Saves the second launch and its ramp; the grid is one resident wave by
// construction (grid_one_wave), which is what a cooperative launch requires.
template <int KIND>
__global__ void __launch_bounds__(kOctThreads, OEA_OCT_MINB)
k_step_sampled_oct(TableDev ent, TableDev rel, const __grid_constant__ SampledParams P, oea_loss_cfg cfg,
                   double* __restrict__ loss_out, OptTab A, OptTab B, float lr) {
    __shared__ double s_loss[kOctWarps];
    __shared__ OctStage s_stage[kOctWarps];
    oct_score_body(ent, rel, P, cfg, loss_out, nullptr, s_loss, s_stage);
    cooperative_groups::this_grid().sync();
    oct_rowopt_body<KIND>(A, B, ent.pitch, lr, blockIdx.x * kOctWarps + (threadIdx.x >> 5), gridDim.x * kOctWarps);
}

// The duo scorer (oea_duo.cuh): two positives per warp, sampled source.
__global__ void __launch_bounds__(kDuoThreads, OEA_DUO_MINB)
k_score_sampled_duo(TableDev ent, TableDev rel, const __grid_constant__ SampledParams P, oea_loss_cfg cfg,
                    double* __restrict__ loss_out, int32_t* __restrict__ dbg) {
    __shared__ double s_loss[kDuoWarps];
    __shared__ DuoStage s_stage[kDuoWarps];
    FedBatch none{};
    duo_score_body<false>(ent, rel, P, none, cfg, loss_out, dbg, s_loss, s_stage);
}

// The whole sampled training step as ONE cooperative launch, duo scorer: score + gradients, grid barrier, row optimiser.
template <int KIND>
__global__ void __launch_bounds__(kDuoThreads, OEA_DUO_MINB)
k_step_sampled_duo(TableDev ent, TableDev rel, const __grid_constant__ SampledParams P, oea_loss_cfg cfg,
                   double* __restrict__ loss_out, OptTab A, OptTab B, float lr) {
    __shared__ double s_loss[kDuoWarps];
    __shared__ DuoStage s_stage[kDuoWarps];
    FedBatch none{};
    duo_score_body<false>(ent, rel, P, none, cfg, loss_out, nullptr, s_loss, s_stage);
    cooperative_groups::this_grid().sync();
    oct_rowopt_body<KIND>(A, B, ent.pitch, lr, blockIdx.x * kDuoWarps + (threadIdx.x >> 5), gridDim.x * kDuoWarps);
}

// ------------------------------------------------------------------------------------------------
// Row optimiser: one warp per row, flagged rows only (Adagrad / SGD) or all rows (Adam).
// TF1 semantics (optimizers.py:10-20): Adagrad acc += g², x −= lr·g/√acc (no ε, acc0 = 0.1 set by
// the caller); Adam lr_t = lr·√(1−β2^t)/(1−β1^t), x −= lr_t·m/(√v + ε).
// ------------------------------------------------------------------------------------------------
template <int KIND>
__global__ void __launch_bounds__(kThreads)
k_rowopt(float* __restrict__ w, float* __restrict__ grad, float* __restrict__ s1, float* __restrict__ s2,
         int32_t* __restrict__ touched, int rows, int pitch, float lr, float beta1, float beta2, float eps,
         float lr_t) {
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    const int p4 = pitch >> 2;
    for (int row = warp_global; row < rows; row += n_warps) {
        if (KIND != OEA_OPT_ADAM) {
            if (touched[row] == 0) continue;
        }
        const size_t base = (size_t)row * pitch;
        for (int c = lane; c < p4; c += OEA_WARP) {
            const size_t o = base + 4 * (size_t)c;
            float4 g = *reinterpret_cast<float4*>(grad + o);
            float4 x = *reinterpret_cast<float4*>(w + o);
            if (KIND == OEA_OPT_ADAGRAD) {
                float4 a = *reinterpret_cast<float4*>(s1 + o);
                a.x = fmaf(g.x, g.x, a.x); a.y = fmaf(g.y, g.y, a.y); a.z = fmaf(g.z, g.z, a.z); a.w = fmaf(g.w, g.w, a.w);
                x.x -= lr * g.x * rsqrtf(a.x); x.y -= lr * g.y * rsqrtf(a.y);
                x.z -= lr * g.z * rsqrtf(a.z); x.w -= lr * g.w * rsqrtf(a.w);
                *reinterpret_cast<float4*>(s1 + o) = a;
            } else if (KIND == OEA_OPT_SGD) {
                x.x -= lr * g.x; x.y -= lr * g.y; x.z -= lr * g.z; x.w -= lr * g.w;
            } else {
                float4 m = *reinterpret_cast<float4*>(s1 + o);
                float4 v = *reinterpret_cast<float4*>(s2 + o);
                m.x = beta1 * m.x + (1.f - beta1) * g.x; m.y = beta1 * m.y + (1.f - beta1) * g.y;
                m.z = beta1 * m.z + (1.f - beta1) * g.z; m.w = beta1 * m.w + (1.f - beta1) * g.w;
                v.x = beta2 * v.x + (1.f - beta2) * g.x * g.x; v.y = beta2 * v.y + (1.f - beta2) * g.y * g.y;
                v.z = beta2 * v.z + (1.f - beta2) * g.z * g.z; v.w = beta2 * v.w + (1.f - beta2) * g.w * g.w;
                x.x -= lr_t * m.x / (sqrtf(v.x) + eps); x.y -= lr_t * m.y / (sqrtf(v.y) + eps);
                x.z -= lr_t * m.z / (sqrtf(v.z) + eps); x.w -= lr_t * m.w / (sqrtf(v.w) + eps);
                *reinterpret_cast<float4*>(s1 + o) = m;
                *reinterpret_cast<float4*>(s2 + o) = v;
            }
            *reinterpret_cast<float4*>(w + o) = x;
            *reinterpret_cast<float4*>(grad + o) = f4(0.f);
        }
        __syncwarp();      // every lane has read the flag (above) before lane 0 clears it: no reliance on convergence
        if (lane == 0) touched[row] = 0;
    }
}

// Normalised lookup: out[i] = normalise(weight[ids[i]]) (basic_model.py:106-121 `.eval()` reads).
__global__ void __launch_bounds__(kThreads)
k_lookup(const float* __restrict__ w, int pitch, int dim, bool norm, const int32_t* __restrict__ ids, int n,
         float* __restrict__ out, int out_pitch) {
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    for (int i = warp_global; i < n; i += n_warps) {
        const int row = ids ? __ldg(ids + i) : i;
        const float* src = w + (size_t)row * pitch;
        float ss = 0.f;
        for (int c = lane; c < dim; c += OEA_WARP) { const float x = __ldg(src + c); ss = fmaf(x, x, ss); }
        ss = warp_sum(ss);
        const float inv = inv_norm(ss, norm);
        float* dst = out + (size_t)i * out_pitch;
        for (int c = lane; c < out_pitch; c += OEA_WARP) dst[c] = c < dim ? __ldg(src + c) * inv : 0.f;
    }
}



}  // namespace oea

using namespace oea;

extern "C" int oea_abi_version(void) { return OEA_ABI_VERSION; }

extern "C" const char* oea_error_string(int code) {
    if (code < 0) return cudaGetErrorString((cudaError_t)(-code));
    switch (code) {
        case OEA_OK: return "ok";
        case OEA_ERR_NULL: return "required pointer is NULL";
        case OEA_ERR_DIM: return "rows/dim/pitch out of range (pitch % 4 == 0, dim <= pitch <= 512)";
        case OEA_ERR_ALIGN: return "pointer not 16-byte aligned";
        case OEA_ERR_KIND: return "unknown score/loss/optimiser/metric kind";
        case OEA_ERR_SHAPE: return "inconsistent batch shapes";
        case OEA_ERR_RANGE: return "parameter out of range";
        case OEA_ERR_WORKSPACE: return "workspace too small";
        default: return "unknown error";
    }
}

extern "C" int oea_triple_score_fed(const oea_table* ent, const oea_table* rel,
                                    const int32_t* pos_h, const int32_t* pos_r, const int32_t* pos_t, int32_t n_pos,
                                    const int32_t* neg_h, const int32_t* neg_r, const int32_t* neg_t, int32_t n_neg,
                                    const oea_loss_cfg* loss, double* loss_out, void* stream) {
    int rc = check_table(ent, true); if (rc) return rc;
    rc = check_table(rel, true); if (rc) return rc;
    if (loss == nullptr || loss_out == nullptr) return OEA_ERR_NULL;
    if (n_pos < 0 || n_neg < 0) return OEA_ERR_SHAPE;
    if (n_pos > 0 && (!pos_h || !pos_r || !pos_t)) return OEA_ERR_NULL;
    if (n_neg > 0 && (!neg_h || !neg_r || !neg_t)) return OEA_ERR_NULL;
    if (ent->pitch != rel->pitch || ent->dim != rel->dim) return OEA_ERR_DIM;
    if (loss->score_kind != OEA_SCORE_L1 && loss->score_kind != OEA_SCORE_L2SQ) return OEA_ERR_KIND;
    if (loss->loss_kind < OEA_LOSS_MARGIN || loss->loss_kind > OEA_LOSS_LOGSIGMOID) return OEA_ERR_KIND;
    if (loss->loss_kind == OEA_LOSS_MARGIN && n_neg != n_pos) return OEA_ERR_SHAPE;  // args_hander.py:19-21
    if ((loss->loss_kind == OEA_LOSS_POSITIVE || loss->loss_kind == OEA_LOSS_LOGSIGMOID) && n_neg != 0) return OEA_ERR_SHAPE;
    if (n_pos + n_neg == 0) return OEA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    TableDev e = table_dev(ent), r = table_dev(rel);
    const bool l1 = loss->score_kind == OEA_SCORE_L1;
    if (loss->loss_kind == OEA_LOSS_MARGIN) {
        const int grid = grid_for(n_pos);
#define CALL(V)                                                                                                         \
        if (l1) OEA_LAUNCH((k_score_margin<OEA_SCORE_L1, V>), grid, kThreads, 0, st, e, r, pos_h, pos_r, pos_t, neg_h, neg_r, neg_t, n_pos, *loss, loss_out); \
        else OEA_LAUNCH((k_score_margin<OEA_SCORE_L2SQ, V>), grid, kThreads, 0, st, e, r, pos_h, pos_r, pos_t, neg_h, neg_r, neg_t, n_pos, *loss, loss_out)
        OEA_DISPATCH_VEC(ent->pitch, CALL);
#undef CALL
    } else {
#define CALL(V)                                                                                                         \
        if (l1) { const int grid = grid_one_wave(k_score_fed<OEA_SCORE_L1, V>, n_pos + n_neg);                              \
                  OEA_LAUNCH((k_score_fed<OEA_SCORE_L1, V>), grid, kThreads, 0, st, e, r, pos_h, pos_r, pos_t, n_pos, neg_h, neg_r, neg_t, n_neg, *loss, loss_out); } \
        else { const int grid = grid_one_wave(k_score_fed<OEA_SCORE_L2SQ, V>, n_pos + n_neg);                               \
               OEA_LAUNCH((k_score_fed<OEA_SCORE_L2SQ, V>), grid, kThreads, 0, st, e, r, pos_h, pos_r, pos_t, n_pos, neg_h, neg_r, neg_t, n_neg, *loss, loss_out); }
        OEA_DISPATCH_VEC(ent->pitch, CALL);
#undef CALL
    }
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_rowopt_apply(const oea_table* t, const oea_opt_cfg* opt, void* stream) {
    int rc = check_table(t, true); if (rc) return rc;
    if (opt == nullptr) return OEA_ERR_NULL;
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = grid_for(t->rows);
    switch (opt->kind) {
        case OEA_OPT_ADAGRAD:
            if (!t->state1) return OEA_ERR_NULL;
            OEA_LAUNCH(k_rowopt<OEA_OPT_ADAGRAD>, grid, kThreads, 0, st, t->weight, t->grad, t->state1, nullptr, t->touched, t->rows, t->pitch, opt->lr, 0.f, 0.f, 0.f, 0.f);
            break;
        case OEA_OPT_SGD:
            OEA_LAUNCH(k_rowopt<OEA_OPT_SGD>, grid, kThreads, 0, st, t->weight, t->grad, nullptr, nullptr, t->touched, t->rows, t->pitch, opt->lr, 0.f, 0.f, 0.f, 0.f);
            break;
        case OEA_OPT_ADADELTA:
            return oea_rowopt_adadelta(t, opt, stream);   // oea_optim_ext.cu
        case OEA_OPT_ADAM: {
            if (!t->state1 || !t->state2) return OEA_ERR_NULL;
            if (opt->t < 1) return OEA_ERR_RANGE;
            const double b1t = 1.0 - pow((double)opt->beta1, (double)opt->t);
            const double b2t = 1.0 - pow((double)opt->beta2, (double)opt->t);
            const float lr_t = (float)((double)opt->lr * sqrt(b2t) / b1t);
            OEA_LAUNCH(k_rowopt<OEA_OPT_ADAM>, grid, kThreads, 0, st, t->weight, t->grad, t->state1, t->state2, t->touched, t->rows, t->pitch, opt->lr, opt->beta1, opt->beta2, opt->eps, lr_t);
            break;
        }
        default:
            return OEA_ERR_KIND;
    }
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

// OEA_SCORE_V1=1 selects the warp-per-row kernel for every shape (A/B measurements, tests of both paths).
static bool oea_force_v1() {
    const char* v = getenv("OEA_SCORE_V1");   // read per call: tests flip it inside one process
    return v != nullptr && v[0] == '1';
}

// OEA_NO_FUSE=1 keeps the sampled step as two launches (score, optimiser): A/B of the cooperative fused launch.
static bool oea_no_fuse() {
    const char* v = getenv("OEA_NO_FUSE");
    return v != nullptr && v[0] == '1';
}

// Argument checks + step parameters shared by the score-only and the fused-step entry points.
static int sampled_prepare(const oea_table* ent, const oea_table* rel, const oea_kg_view* kg1, const oea_kg_view* kg2,
                           const oea_tripleset* tset, const oea_sample_cfg* smp, const oea_loss_cfg* loss,
                           const double* loss_out, oea::SampledParams* Pout, int* n_pos_out_host) {
    using namespace oea;
    int rc = check_table(ent, true); if (rc) return rc;
    rc = check_table(rel, true); if (rc) return rc;
    if (!smp || !loss || !loss_out) return OEA_ERR_NULL;
    if (ent->pitch != rel->pitch || ent->dim != rel->dim) return OEA_ERR_DIM;
    if (loss->loss_kind < OEA_LOSS_MARGIN || loss->loss_kind > OEA_LOSS_LOGSIGMOID) return OEA_ERR_KIND;
    if (loss->loss_kind == OEA_LOSS_MARGIN && smp->neg_per_pos != 1) return OEA_ERR_SHAPE;   // args_hander.py:19-21
    if ((loss->loss_kind == OEA_LOSS_POSITIVE || loss->loss_kind == OEA_LOSS_LOGSIGMOID) && smp->neg_per_pos != 0) return OEA_ERR_SHAPE;
    if ((loss->loss_kind == OEA_LOSS_LIMITED || loss->loss_kind == OEA_LOSS_LOGISTIC) && smp->neg_per_pos < 1) return OEA_ERR_SHAPE;
    if (loss->score_kind != OEA_SCORE_L1 && loss->score_kind != OEA_SCORE_L2SQ) return OEA_ERR_KIND;
    return sampler_prepare(kg1, kg2, tset, smp, Pout, n_pos_out_host);
}

extern "C" int oea_triple_score_sampled(const oea_table* ent, const oea_table* rel,
                                        const oea_kg_view* kg1, const oea_kg_view* kg2, const oea_tripleset* tset,
                                        const oea_sample_cfg* smp, const oea_loss_cfg* loss,
                                        double* loss_out, int32_t* n_pos_out, int32_t* dbg_neg, void* stream) {
    SampledParams P;
    int n_pos_prepared = 0;
    int rc = sampled_prepare(ent, rel, kg1, kg2, tset, smp, loss, loss_out, &P, &n_pos_prepared); if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int n_pos = P.n_slice[0] + P.n_slice[1];
    if (n_pos_out) OEA_CUDA_TRY(cudaMemcpyAsync(n_pos_out, &n_pos, sizeof(int), cudaMemcpyHostToDevice, st));
    if (n_pos == 0) return OEA_OK;
    TableDev e = table_dev(ent), r = table_dev(rel);
    const bool l1 = loss->score_kind == OEA_SCORE_L1;
    if (!l1 && ent->pitch <= 128 && !oea_force_v1() && oea_use_duo(P.k)) {
        const int pairs = ((n_pos + P.shard_world - 1) / P.shard_world + 1) / 2;
        const int grid = grid_one_wave(k_score_sampled_duo, pairs, kDuoWarps);
        OEA_LAUNCH(k_score_sampled_duo, grid, kDuoThreads, 0, st, e, r, P, *loss, loss_out, dbg_neg);
    } else if (!l1 && ent->pitch <= 128 && !oea_force_v1()) {
        const int grid = grid_one_wave(k_score_sampled_oct, (n_pos + P.shard_world - 1) / P.shard_world, kOctWarps);
        OEA_LAUNCH(k_score_sampled_oct, grid, kOctThreads, 0, st, e, r, P, *loss, loss_out, dbg_neg);
    } else {
#define CALL(V)                                                                                              \
    if (l1) { const int grid = grid_one_wave(k_score_sampled<OEA_SCORE_L1, V>, (n_pos + P.shard_world - 1) / P.shard_world);                     \
              OEA_LAUNCH((k_score_sampled<OEA_SCORE_L1, V>), grid, kThreads, 0, st, e, r, P, *loss, loss_out, dbg_neg); } \
    else { const int grid = grid_one_wave(k_score_sampled<OEA_SCORE_L2SQ, V>, (n_pos + P.shard_world - 1) / P.shard_world);                      \
           OEA_LAUNCH((k_score_sampled<OEA_SCORE_L2SQ, V>), grid, kThreads, 0, st, e, r, P, *loss, loss_out, dbg_neg); }
        OEA_DISPATCH_VEC(ent->pitch, CALL);
#undef CALL
    }
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_rowopt_apply_pair(const oea_table* a, const oea_table* b, const oea_opt_cfg* opt, void* stream);

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
    // OEA_FED_GROUPED=1: score a positive together with its negatives when the batch has the reference's layout
    // (oea_triple_grouped.cu; opt-in until it has been timed on hardware)
    const char* grouped_env = getenv("OEA_FED_GROUPED");
    const bool grouped = grouped_env && grouped_env[0] == '1' && n_pos > 0 && n_neg % n_pos == 0;
    // OEA_FED_FUSED=1: grouped scoring and the row optimiser as one cooperative launch where that kernel applies
    const char* fused_env = getenv("OEA_FED_FUSED");
    int rc = OEA_ERR_KIND;
    if (fused_env && fused_env[0] == '1' && n_pos > 0 && n_neg % n_pos == 0)
        rc = oea_triple_step_fed_grouped(ent, rel, dpos, dpos + n_pos, dpos + 2 * (size_t)n_pos, n_pos,
                                         dneg, dneg + n_neg, dneg + 2 * (size_t)n_neg, n_neg, loss, opt, dev_loss_ws, stream);
    if (rc == OEA_ERR_KIND) {
        rc = grouped
            ? oea_triple_score_fed_grouped(ent, rel, dpos, dpos + n_pos, dpos + 2 * (size_t)n_pos, n_pos,
                                           dneg, dneg + n_neg, dneg + 2 * (size_t)n_neg, n_neg, loss, dev_loss_ws, stream)
            : oea_triple_score_fed(ent, rel, dpos, dpos + n_pos, dpos + 2 * (size_t)n_pos, n_pos,
                                   dneg, dneg + n_neg, dneg + 2 * (size_t)n_neg, n_neg, loss, dev_loss_ws, stream);
        if (rc) return rc;
        rc = oea_rowopt_apply_pair(ent, rel, opt, stream);
    }
    if (rc) return rc;
    OEA_CUDA_TRY(cudaMemcpyAsync(loss_pinned_host, dev_loss_ws, sizeof(double), cudaMemcpyDeviceToHost, st));
    OEA_CUDA_TRY(cudaStreamSynchronize(st));
    *loss_host = (float)(*loss_pinned_host);
    return OEA_OK;
}

extern "C" int oea_table_lookup(const oea_table* t, const int32_t* ids, int32_t n, float* out, int32_t out_pitch,
                                void* stream) {
    int rc = check_table(t, false); if (rc) return rc;
    if (out == nullptr) return OEA_ERR_NULL;
    if (n < 0 || out_pitch < t->dim) return OEA_ERR_SHAPE;
    if (n == 0) return OEA_OK;
    OEA_LAUNCH(k_lookup, grid_for(n), kThreads, 0, (cudaStream_t)stream, t->weight, t->pitch, t->dim, t->l2_norm != 0, ids, n, out, out_pitch);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

namespace oea {
__global__ void k_tripleset_build(const int32_t* __restrict__ triples, int n, unsigned long long* slots, uint32_t capacity,
                                  uint32_t ent_bits, uint32_t rel_bits) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t key = triple_key(triples[3 * (size_t)i], triples[3 * (size_t)i + 1], triples[3 * (size_t)i + 2], ent_bits, rel_bits);
    const uint32_t mask = capacity - 1u;
    uint32_t slot = key_hash(key) & mask;
    while (true) {
        const unsigned long long prev = atomicCAS(slots + slot, 0xFFFFFFFFFFFFFFFFull, (unsigned long long)key);
        if (prev == 0xFFFFFFFFFFFFFFFFull || prev == key) return;
        slot = (slot + 1u) & mask;
    }
}
}  // namespace oea

extern "C" int oea_tripleset_build(const int32_t* triples, int32_t n, uint64_t* slots, uint32_t capacity,
                                   uint32_t ent_bits, uint32_t rel_bits, void* stream) {
    if (!slots || (n > 0 && !triples)) return OEA_ERR_NULL;
    if (n < 0 || capacity == 0 || (capacity & (capacity - 1)) != 0 || (uint64_t)capacity < 2ull * (uint64_t)n) return OEA_ERR_RANGE;
    if (2 * ent_bits + rel_bits > 63) return OEA_ERR_RANGE;
    cudaStream_t st = (cudaStream_t)stream;
    OEA_CUDA_TRY(cudaMemsetAsync(slots, 0xFF, (size_t)capacity * sizeof(uint64_t), st));
    if (n == 0) return OEA_OK;
    OEA_LAUNCH(k_tripleset_build, (n + 255) / 256, 256, 0, st, triples, n, (unsigned long long*)slots, capacity, ent_bits, rel_bits);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

// ================================================================================================
// Generic pieces for graphs that are not the fused triple step: gradient scatter through the
// normalised lookup, the losses of modules/base/losses.py on already-gathered rows, and the
// MTransE mapping loss (losses.py:76-80).
// ================================================================================================
namespace oea {

// backward of `normalise(weight[ids[i]])`: grad_rows [n, gpitch] are d/d(normalised row)
__global__ void __launch_bounds__(kThreads)
k_table_scatter(const float* __restrict__ w, float* __restrict__ grad, int32_t* __restrict__ touched, int pitch,
                int dim, bool norm, const int32_t* __restrict__ ids, int n, const float* __restrict__ g_rows, int gpitch) {
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    for (int i = warp_global; i < n; i += n_warps) {
        const int row = __ldg(ids + i);
        const float* x = w + (size_t)row * pitch;
        const float* g = g_rows + (size_t)i * gpitch;
        float ss = 0.f, dot = 0.f;
        for (int c = lane; c < dim; c += 32) { const float xv = __ldg(x + c); ss = fmaf(xv, xv, ss); dot = fmaf(xv, __ldg(g + c), dot); }
        warp_sum2(ss, dot);
        const float inv = inv_norm(ss, norm);
        // x̂ = x·inv ; <x̂, g> = dot·inv ; dx = (g − x̂·<x̂,g>)·inv
        const float proj = (norm && ss >= kNormEps) ? dot * inv * inv : 0.f;
        float* o = grad + (size_t)row * pitch;
        for (int c = lane; c < dim; c += 32) atomicAdd(o + c, (__ldg(g + c) - __ldg(x + c) * proj) * inv);
        if (lane == 0) touched[row] = 1;
    }
}

// losses.py on gathered rows: warp per triple (or per pos/neg pair for the margin loss)
template <int SCORE>
__global__ void __launch_bounds__(kThreads)
k_loss_rows(const float* __restrict__ ph, const float* __restrict__ pr, const float* __restrict__ pt, int n_pos,
            const float* __restrict__ nh, const float* __restrict__ nr, const float* __restrict__ nt, int n_neg,
            int dim, int pitch, oea_loss_cfg cfg, double* __restrict__ loss_out,
            float* __restrict__ gph, float* __restrict__ gpr, float* __restrict__ gpt,
            float* __restrict__ gnh, float* __restrict__ gnr, float* __restrict__ gnt) {
    __shared__ double s_loss[kWarpsPerBlock];
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    const bool margin = cfg.loss_kind == OEA_LOSS_MARGIN;
    const int total = margin ? n_pos : n_pos + n_neg;
    float warp_loss = 0.f;
    for (int i = warp_global; i < total; i += n_warps) {
        const bool is_neg = !margin && i >= n_pos;
        const size_t o = (size_t)(is_neg ? i - n_pos : i) * pitch;
        const float* h = (is_neg ? nh : ph) + o; const float* r = (is_neg ? nr : pr) + o; const float* t = (is_neg ? nt : pt) + o;
        float s = 0.f, s2 = 0.f;
        for (int c = lane; c < dim; c += 32) {
            const float u = h[c] + r[c] - t[c];
            s += SCORE == OEA_SCORE_L1 ? fabsf(u) : u * u;
            if (margin) { const float v = nh[o + c] + nr[o + c] - nt[o + c]; s2 += SCORE == OEA_SCORE_L1 ? fabsf(v) : v * v; }
        }
        warp_sum2(s, s2);
        float L, g, g2 = 0.f;
        if (margin) { const float v = cfg.margin + s - s2; L = fmaxf(v, 0.f); g = v > 0.f ? 1.f : 0.f; g2 = -g; }
        else loss_of(cfg.loss_kind, is_neg, s, cfg, L, g);
        warp_loss += L;
        float* gh = (is_neg ? gnh : gph) + o; float* gr = (is_neg ? gnr : gpr) + o; float* gt = (is_neg ? gnt : gpt) + o;
        for (int c = lane; c < dim; c += 32) {
            const float u = h[c] + r[c] - t[c];
            const float du = g * (SCORE == OEA_SCORE_L1 ? sgn(u) : 2.f * u);
            gh[c] = du; gr[c] = du; gt[c] = -du;
            if (margin) {
                const float v = nh[o + c] + nr[o + c] - nt[o + c];
                const float dv = g2 * (SCORE == OEA_SCORE_L1 ? sgn(v) : 2.f * v);
                gnh[o + c] = dv; gnr[o + c] = dv; gnt[o + c] = -dv;
            }
        }
    }
    LossAcc acc{s_loss};
    acc.flush(warp_loss, loss_out);
}

// Mapping loss part 1 (losses.py:77-78): per pair r = e2 − e1·M ; loss += ‖r‖² ; g2 = 2r ; g1 = −2·r·Mᵀ ;
// gM += −2·e1ᵀ r.  One CTA per 8 pairs; the CTA's partial gM goes out with one atomic per element.
constexpr int MAP_PAIRS = 8;
__global__ void __launch_bounds__(256)
k_mapping_pairs(const float* __restrict__ e1, const float* __restrict__ e2, int n, int dim, int pitch,
                const float* __restrict__ M, int mpitch, float alpha, double* __restrict__ loss_out,
                float* __restrict__ g1, float* __restrict__ g2, float* __restrict__ gM) {
    OEA_DYNAMIC_SMEM(sm);
    float* a = sm;                       // [MAP_PAIRS][dim]  e1 rows
    float* r = sm + MAP_PAIRS * dim;     // [MAP_PAIRS][dim]  residuals
    __shared__ double s_part[8];
    const int tid = threadIdx.x, p0 = blockIdx.x * MAP_PAIRS;
    const int np = min(MAP_PAIRS, n - p0);
    for (int i = tid; i < MAP_PAIRS * dim; i += 256) {
        const int p = i / dim, c = i % dim;
        a[i] = p < np ? e1[(size_t)(p0 + p) * pitch + c] : 0.f;
    }
    __syncthreads();
    float local = 0.f;
    for (int i = tid; i < MAP_PAIRS * dim; i += 256) {          // y = e1·M, column c of pair p
        const int p = i / dim, c = i % dim;
        float y = 0.f;
        for (int k = 0; k < dim; ++k) y = fmaf(a[p * dim + k], __ldg(M + (size_t)k * mpitch + c), y);
        const float res = p < np ? e2[(size_t)(p0 + p) * pitch + c] - y : 0.f;
        r[i] = res;
        local += res * res;
        if (p < np) g2[(size_t)(p0 + p) * pitch + c] = 2.f * alpha * res;
    }
    __syncthreads();
    for (int i = tid; i < MAP_PAIRS * dim; i += 256) {          // g1 = −2·r·Mᵀ
        const int p = i / dim, k = i % dim;
        if (p >= np) continue;
        float acc = 0.f;
        for (int c = 0; c < dim; ++c) acc = fmaf(r[p * dim + c], __ldg(M + (size_t)k * mpitch + c), acc);
        g1[(size_t)(p0 + p) * pitch + k] = -2.f * alpha * acc;
    }
    for (int i = tid; i < dim * dim; i += 256) {                // gM[k][c] += −2·Σ_p e1[p][k]·r[p][c]
        const int k = i / dim, c = i % dim;
        float acc = 0.f;
#pragma unroll
        for (int p = 0; p < MAP_PAIRS; ++p) acc = fmaf(a[p * dim + k], r[p * dim + c], acc);
        if (acc != 0.f) atomicAdd(gM + (size_t)k * mpitch + c, -2.f * alpha * acc);
    }
    local = warp_sum(local);
    if ((tid & 31) == 0) s_part[tid >> 5] = (double)local;
    __syncthreads();
    if (tid == 0) { double t = 0.0; for (int i = 0; i < 8; ++i) t += s_part[i]; atomicAdd(loss_out, (double)alpha * t); }
}

// Mapping loss part 2 (losses.py:79): G = M·Mᵀ − I ; loss += ΣG² ; gM += 4·G·M.  Grid of row blocks of G.
__global__ void __launch_bounds__(256)
k_mapping_orth(const float* __restrict__ M, int dim, int mpitch, float alpha, double* __restrict__ loss_out,
               float* __restrict__ gM, float* __restrict__ Gws) {
    // pass A (blockIdx.y == 0): G rows ; pass B is a second launch reading Gws
    const int row = blockIdx.x;
    __shared__ double s_part[8];
    float local = 0.f;
    for (int j = threadIdx.x; j < dim; j += 256) {
        float acc = 0.f;
        for (int k = 0; k < dim; ++k) acc = fmaf(__ldg(M + (size_t)row * mpitch + k), __ldg(M + (size_t)j * mpitch + k), acc);
        const float g = acc - (row == j ? 1.f : 0.f);
        Gws[(size_t)row * dim + j] = g;
        local += g * g;
    }
    local = warp_sum(local);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = (double)local;
    __syncthreads();
    if (threadIdx.x == 0) { double t = 0.0; for (int i = 0; i < 8; ++i) t += s_part[i]; atomicAdd(loss_out, (double)alpha * t); }
}
__global__ void __launch_bounds__(256)
k_mapping_orth_grad(const float* __restrict__ M, int dim, int mpitch, float alpha, const float* __restrict__ Gws, float* __restrict__ gM) {
    const int row = blockIdx.x;
    for (int c = threadIdx.x; c < dim; c += 256) {
        float acc = 0.f;
        for (int j = 0; j < dim; ++j) acc = fmaf(Gws[(size_t)row * dim + j], __ldg(M + (size_t)j * mpitch + c), acc);
        atomicAdd(gM + (size_t)row * mpitch + c, 4.f * alpha * acc);
    }
}

}  // namespace oea

extern "C" int oea_table_scatter_grad(const oea_table* t, const int32_t* ids, int32_t n, const float* grad_rows,
                                      int32_t grad_pitch, void* stream) {
    int rc = check_table(t, true); if (rc) return rc;
    if (n < 0 || grad_pitch < t->dim) return OEA_ERR_SHAPE;
    if (n == 0) return OEA_OK;
    if (!ids || !grad_rows) return OEA_ERR_NULL;
    OEA_LAUNCH(k_table_scatter, grid_for(n), kThreads, 0, (cudaStream_t)stream, t->weight, t->grad, t->touched, t->pitch, t->dim,
                                                                        t->l2_norm != 0, ids, n, grad_rows, grad_pitch);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_loss_rows(const float* ph, const float* pr, const float* pt, int32_t n_pos,
                             const float* nh, const float* nr, const float* nt, int32_t n_neg,
                             int32_t dim, int32_t pitch, const oea_loss_cfg* loss, double* loss_out,
                             float* g_ph, float* g_pr, float* g_pt, float* g_nh, float* g_nr, float* g_nt, void* stream) {
    if (!loss || !loss_out) return OEA_ERR_NULL;
    if (n_pos < 0 || n_neg < 0 || dim <= 0 || pitch < dim) return OEA_ERR_SHAPE;
    if (n_pos > 0 && (!ph || !pr || !pt || !g_ph || !g_pr || !g_pt)) return OEA_ERR_NULL;
    if (n_neg > 0 && (!nh || !nr || !nt || !g_nh || !g_nr || !g_nt)) return OEA_ERR_NULL;
    if (loss->loss_kind < OEA_LOSS_MARGIN || loss->loss_kind > OEA_LOSS_LOGSIGMOID) return OEA_ERR_KIND;
    if (loss->loss_kind == OEA_LOSS_MARGIN && n_neg != n_pos) return OEA_ERR_SHAPE;
    if ((loss->loss_kind == OEA_LOSS_POSITIVE || loss->loss_kind == OEA_LOSS_LOGSIGMOID) && n_neg != 0) return OEA_ERR_SHAPE;
    if (n_pos + n_neg == 0) return OEA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = grid_for(n_pos + n_neg);
    if (loss->score_kind == OEA_SCORE_L1)
        OEA_LAUNCH(k_loss_rows<OEA_SCORE_L1>, grid, kThreads, 0, st, ph, pr, pt, n_pos, nh, nr, nt, n_neg, dim, pitch, *loss, loss_out, g_ph, g_pr, g_pt, g_nh, g_nr, g_nt);
    else if (loss->score_kind == OEA_SCORE_L2SQ)
        OEA_LAUNCH(k_loss_rows<OEA_SCORE_L2SQ>, grid, kThreads, 0, st, ph, pr, pt, n_pos, nh, nr, nt, n_neg, dim, pitch, *loss, loss_out, g_ph, g_pr, g_pt, g_nh, g_nr, g_nt);
    else return OEA_ERR_KIND;
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" size_t oea_mapping_workspace_bytes(int32_t dim) { return dim > 0 ? (size_t)dim * dim * sizeof(float) : 0; }

extern "C" int oea_mapping_fwd_bwd(const float* e1, const float* e2, int32_t n, int32_t dim, int32_t pitch,
                                   const float* M, int32_t mpitch, float alpha, double* loss_out,
                                   float* g_e1, float* g_e2, float* g_M, void* workspace, size_t workspace_bytes,
                                   void* stream) {
    if (!M || !loss_out || !g_M || !workspace) return OEA_ERR_NULL;
    if (n < 0 || dim <= 0 || dim > 512 || pitch < dim || mpitch < dim) return OEA_ERR_DIM;
    if (n > 0 && (!e1 || !e2 || !g_e1 || !g_e2)) return OEA_ERR_NULL;
    if (workspace_bytes < oea_mapping_workspace_bytes(dim)) return OEA_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    if (n > 0) {
        const size_t smem = 2 * (size_t)MAP_PAIRS * dim * sizeof(float);
        OEA_LAUNCH(k_mapping_pairs, (n + MAP_PAIRS - 1) / MAP_PAIRS, 256, smem, st, e1, e2, n, dim, pitch, M, mpitch, alpha, loss_out, g_e1, g_e2, g_M);
        OEA_LAUNCH_CHECK();
    }
    OEA_LAUNCH(k_mapping_orth, dim, 256, 0, st, M, dim, mpitch, alpha, loss_out, g_M, (float*)workspace);
    OEA_LAUNCH_CHECK();
    OEA_LAUNCH(k_mapping_orth_grad, dim, 256, 0, st, M, dim, mpitch, alpha, (const float*)workspace, g_M);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

// ================================================================================================
// One call per training step: fused sampler+scorer, then ONE row-optimiser launch over both tables.
// ================================================================================================
namespace oea {


// Adagrad / SGD over the concatenated row space [ent rows | rel rows] (same pitch), flagged rows only.
template <int KIND>
__global__ void __launch_bounds__(kThreads)
k_rowopt_pair(OptTab A, OptTab B, int pitch, float lr) {
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    const int p4 = pitch >> 2;
    const int total = A.rows + B.rows;
    for (int r = warp_global; r < total; r += n_warps) {
        const bool first = r < A.rows;
        const OptTab& T = first ? A : B;
        const int row = first ? r : r - A.rows;
        if (T.touched[row] == 0) continue;
        const size_t base = (size_t)row * pitch;
        for (int c = lane; c < p4; c += OEA_WARP) {
            const size_t o = base + 4 * (size_t)c;
            const float4 g = *reinterpret_cast<const float4*>(T.g + o);
            float4 x = *reinterpret_cast<float4*>(T.w + o);
            if (KIND == OEA_OPT_ADAGRAD) {
                float4 a = *reinterpret_cast<float4*>(T.s1 + o);
                a.x = fmaf(g.x, g.x, a.x); a.y = fmaf(g.y, g.y, a.y); a.z = fmaf(g.z, g.z, a.z); a.w = fmaf(g.w, g.w, a.w);
                x.x -= lr * g.x * rsqrtf(a.x); x.y -= lr * g.y * rsqrtf(a.y);
                x.z -= lr * g.z * rsqrtf(a.z); x.w -= lr * g.w * rsqrtf(a.w);
                *reinterpret_cast<float4*>(T.s1 + o) = a;
            } else {
                x.x -= lr * g.x; x.y -= lr * g.y; x.z -= lr * g.z; x.w -= lr * g.w;
            }
            *reinterpret_cast<float4*>(T.w + o) = x;
            *reinterpret_cast<float4*>(T.g + o) = f4(0.f);
        }
        __syncwarp();      // as in k_rowopt: all lanes have read the flag before it is cleared
        if (lane == 0) T.touched[row] = 0;
    }
}

}  // namespace oea

extern "C" int oea_rowopt_apply_pair(const oea_table* a, const oea_table* b, const oea_opt_cfg* opt, void* stream) {
    int rc = check_table(a, true); if (rc) return rc;
    rc = check_table(b, true); if (rc) return rc;
    if (!opt) return OEA_ERR_NULL;
    if (opt->kind == OEA_OPT_ADAM || opt->kind == OEA_OPT_ADADELTA || a->pitch != b->pitch) {   // dense rules / mismatched pitch: two launches
        rc = oea_rowopt_apply(a, opt, stream); if (rc) return rc;
        return oea_rowopt_apply(b, opt, stream);
    }
    if (opt->kind == OEA_OPT_ADAGRAD && (!a->state1 || !b->state1)) return OEA_ERR_NULL;
    OptTab A{a->weight, a->grad, a->state1, a->touched, a->rows}, B{b->weight, b->grad, b->state1, b->touched, b->rows};
    const int grid = grid_for(a->rows + b->rows);
    cudaStream_t st = (cudaStream_t)stream;
    if (opt->kind == OEA_OPT_ADAGRAD) OEA_LAUNCH(k_rowopt_pair<OEA_OPT_ADAGRAD>, grid, kThreads, 0, st, A, B, a->pitch, opt->lr);
    else if (opt->kind == OEA_OPT_SGD) OEA_LAUNCH(k_rowopt_pair<OEA_OPT_SGD>, grid, kThreads, 0, st, A, B, a->pitch, opt->lr);
    else return OEA_ERR_KIND;
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_triple_step_sampled(const oea_table* ent, const oea_table* rel,
                                       const oea_kg_view* kg1, const oea_kg_view* kg2, const oea_tripleset* tset,
                                       const oea_sample_cfg* smp, const oea_loss_cfg* loss, const oea_opt_cfg* opt,
                                       double* loss_out, int32_t* n_pos_out, void* stream) {
    if (!opt) return OEA_ERR_NULL;
    if (smp && smp->shard_world > 1) return OEA_ERR_RANGE;   // sharded batches: score_sampled → gradient exchange → rowopt
    // One cooperative launch when the octet kernel applies and the optimiser is row-sparse (Adagrad / SGD)
    const bool fuse = loss && ent && rel && loss->score_kind == OEA_SCORE_L2SQ && ent->pitch <= 128 && !oea_force_v1() &&
                      (opt->kind == OEA_OPT_ADAGRAD || opt->kind == OEA_OPT_SGD) && !oea_no_fuse();
    if (!fuse) {
        int rc = oea_triple_score_sampled(ent, rel, kg1, kg2, tset, smp, loss, loss_out, n_pos_out, nullptr, stream);
        if (rc) return rc;
        return oea_rowopt_apply_pair(ent, rel, opt, stream);
    }
    SampledParams P;
    int n_pos = 0;
    int rc = sampled_prepare(ent, rel, kg1, kg2, tset, smp, loss, loss_out, &P, &n_pos); if (rc) return rc;
    if (P.shard_world != 1) return OEA_ERR_RANGE;      // a sharded batch needs the gradient exchange between score and optimiser
    if (opt->kind == OEA_OPT_ADAGRAD && (!ent->state1 || !rel->state1)) return OEA_ERR_NULL;
    cudaStream_t st = (cudaStream_t)stream;
    if (n_pos_out) OEA_CUDA_TRY(cudaMemcpyAsync(n_pos_out, &n_pos, sizeof(int), cudaMemcpyHostToDevice, st));
    if (n_pos == 0) return OEA_OK;
    TableDev e = table_dev(ent), r = table_dev(rel);
    OptTab A{ent->weight, ent->grad, ent->state1, ent->touched, ent->rows}, B{rel->weight, rel->grad, rel->state1, rel->touched, rel->rows};
    oea_loss_cfg cfg = *loss;
    float lr = opt->lr;
    if (oea_use_duo(P.k)) {
        const int pairs = (n_pos + 1) / 2;
        if (opt->kind == OEA_OPT_ADAGRAD) {
            const int grid = grid_one_wave(k_step_sampled_duo<OEA_OPT_ADAGRAD>, pairs, kDuoWarps);
            OEA_CUDA_TRY(OEA_LAUNCH_COOPERATIVE(k_step_sampled_duo<OEA_OPT_ADAGRAD>, grid, kDuoThreads, st, e, r, P, cfg, loss_out, A, B, lr));
        } else {
            const int grid = grid_one_wave(k_step_sampled_duo<OEA_OPT_SGD>, pairs, kDuoWarps);
            OEA_CUDA_TRY(OEA_LAUNCH_COOPERATIVE(k_step_sampled_duo<OEA_OPT_SGD>, grid, kDuoThreads, st, e, r, P, cfg, loss_out, A, B, lr));
        }
        return OEA_OK;
    }
    if (opt->kind == OEA_OPT_ADAGRAD) {
        const int grid = grid_one_wave(k_step_sampled_oct<OEA_OPT_ADAGRAD>, n_pos, kOctWarps);
        OEA_CUDA_TRY(OEA_LAUNCH_COOPERATIVE(k_step_sampled_oct<OEA_OPT_ADAGRAD>, grid, kOctThreads, st, e, r, P, cfg, loss_out, A, B, lr));
    } else {
        const int grid = grid_one_wave(k_step_sampled_oct<OEA_OPT_SGD>, n_pos, kOctWarps);
        OEA_CUDA_TRY(OEA_LAUNCH_COOPERATIVE(k_step_sampled_oct<OEA_OPT_SGD>, grid, kOctThreads, st, e, r, P, cfg, loss_out, A, B, lr));
    }
    return OEA_OK;
}
