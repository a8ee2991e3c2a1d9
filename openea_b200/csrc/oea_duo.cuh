// oea_duo.cuh — the octet row layout of path (i) and the "duo" scorer: one warp scores TWO positives at once.  sm_90a.
//
// Octet layout (squared-L2 score, pitch <= 128 floats): 8 lanes hold one embedding row, 4 float4 per lane, so the three
// reductions of a row are 3 shuffle steps and a warp has 4 rows in flight.
//
// Duo scorer: lanes 0-15 work on positive A, lanes 16-31 on positive B of a pair; each half-warp is two octets.  Per
// positive the negatives are taken two at a time (k = 10: five full rounds instead of three rounds of four with two
// idle octets), the sampling chain / phase 1 instructions serve two positives, and two independent dependent-load
// chains are in flight per warp — the kernel is latency/issue bound (dependent gathers per positive over L2-resident
// tables), not bandwidth bound.  A step of B positives needs B/2 warp tasks, so the
// 5 000-positive step of the 15K shape fits one resident wave without the 2-tasks-vs-1 tail of the octet kernel.
// Same maths as the octet kernel and — for the sampled source — the same draws as every sampled scorer
// (modules/base/losses.py:15-73, modules/train/batch.py:36-119, initializers.py:26); requires k <= 16.
//
// Two sources of (positive, negatives): SAMPLED (fused on-device sampler, oea_sampler.cuh) and FED (index vectors in the
// reference's batch layout: the k negatives of positive p at p·k … p·k+k−1, batch.py:36-45).  A fed negative that does
// not share two rows with its positive (any fed batch is legal) is scored as a general triple by the whole warp.
#pragma once
#include "oea_rowmath.cuh"
#include "oea_rowopt.cuh"
#include "oea_sampler.cuh"
#include "oea_transe.cuh"

namespace oea {

struct R4 {
    float4 v[4];
};
__device__ __forceinline__ R4 load_oct(const float* __restrict__ base, int row, int pitch, int l, int p4) {
    R4 r;
    const float* p = base + (size_t)row * pitch;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int q = l + 8 * i;
        r.v[i] = q < p4 ? ldg4(p + 4 * q) : f4(0.f);
    }
    return r;
}
__device__ __forceinline__ void red_oct(float* __restrict__ base, int row, int pitch, int l, int p4, const R4& g) {
    float* p = base + (size_t)row * pitch;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int q = l + 8 * i;
        if (q < p4) red_add4(p + 4 * q, g.v[i]);
    }
}
__device__ __forceinline__ float oct_sum(float v) {
    v += __shfl_xor_sync(OEA_FULL, v, 1);
    v += __shfl_xor_sync(OEA_FULL, v, 2);
    v += __shfl_xor_sync(OEA_FULL, v, 4);
    return v;
}
__device__ __forceinline__ float cross_oct_sum(float v) {
    v += __shfl_xor_sync(OEA_FULL, v, 8);
    v += __shfl_xor_sync(OEA_FULL, v, 16);
    return v;
}

constexpr int kDuoWarps = 4;
constexpr int kDuoMinB = 5;      // 5 CTAs x 4 warps: at most 96 registers per thread, no spills
constexpr int kDuoThreads = kDuoWarps * OEA_WARP;
constexpr int kDuoMaxK = 16;

// Per-warp staging: ĥ+r̂ and r̂−t̂ of both positives (read-only in phase 2, broadcast to the half's two octets) and the
// per-lane Σ g·ê accumulators (kept out of the register file, as in the octet kernel).
struct DuoStage {
    float4 hr[2][4][8];
    float4 rt[2][4][8];
    float4 Eh[4][32];
    float4 Et[4][32];
};

template <bool FED>
__device__ __forceinline__ void duo_score_body(const TableDev& ent, const TableDev& rel, const SampledParams& P, const FedBatch& F,
                                               const oea_loss_cfg& cfg, double* __restrict__ loss_out,
                                               int32_t* __restrict__ dbg, double* s_loss, DuoStage* s_stage) {
    uint64_t seed = 0;
    if (!FED) seed = P.dev_seed != nullptr ? P.seed ^ __ldg(reinterpret_cast<const unsigned long long*>(P.dev_seed)) : P.seed;
    const int lane = threadIdx.x & 31, half = lane >> 4, hl = lane & 15, o2 = (lane >> 3) & 1, l = lane & 7;
    const int hbase = lane & 16;                  // first lane of this lane's half
    DuoStage& S = s_stage[threadIdx.x >> 5];
    const int warp_global = blockIdx.x * kDuoWarps + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kDuoWarps;
    const int n_pos = FED ? F.n_pos : P.n_slice[0] + P.n_slice[1];
    const int k = FED ? F.k : P.k;
    const int sw = FED ? 1 : P.shard_world, sr = FED ? 0 : P.shard_rank;
    const int n_mine = n_pos > sr ? (n_pos - sr + sw - 1) / sw : 0;     // this launch's positives: p = sr + sw·m
    const int p4 = ent.pitch >> 2;
    const bool margin_mode = cfg.loss_kind == OEA_LOSS_MARGIN;
    float lane_loss = 0.f;

    for (int pair = warp_global; 2 * pair < n_mine; pair += n_warps) {
        const int m = 2 * pair + half;
        const bool live = m < n_mine;                // an odd tail leaves half B idle: it mirrors A and writes nothing
        const int p = sr + sw * (live ? m : 2 * pair);
        int h, r, t;
        int neg_e = 0;
        bool neg_head = false, neg_general = false;
        int g_h = 0, g_r = 0, g_t = 0;               // FED: this lane's negative as fed (general-triple path)
        if (FED) {
            h = __ldg(F.ph + p); r = __ldg(F.pr + p); t = __ldg(F.pt + p);
            if (hl < k) {
                const size_t q = (size_t)p * k + hl;
                g_h = __ldg(F.nh + q); g_r = __ldg(F.nr + q); g_t = __ldg(F.nt + q);
                const bool share_tail = g_r == r && g_t == t;       // head corrupted (or a copy of the positive)
                const bool share_head = g_r == r && g_h == h;       // tail corrupted
                neg_head = share_tail;
                neg_e = share_tail ? g_h : g_t;
                neg_general = live && !(share_tail || share_head);
            }
        } else {
            const SampledPositive s = draw_positive<16>(P, seed, p, lane, P.diag & 8, &ent, &rel);
            const oea_kg_view& kg = P.kg[s.q];
            h = s.h; r = s.r; t = s.t;
            if (P.diag & 1) { neg_e = __ldg(kg.entities + (uint32_t)(p * 31 + hl * 977) % (uint32_t)kg.n_entities); neg_head = (p + hl) & 1; }
            else sample_negatives<16>(P, seed, kg, live, p, h, r, t, k, lane, neg_e, neg_head);
            const unsigned hm_all = __ballot_sync(OEA_FULL, neg_head);
            if (dbg != nullptr && live) dump_draws<16>(dbg, p, k, s, hm_all, lane, neg_e);
        }
        const unsigned head_mask = __ballot_sync(OEA_FULL, neg_head);
        const unsigned general_mask = FED ? __ballot_sync(OEA_FULL, neg_general) : 0u;

        // ---- phase 1: the three shared rows of each half's positive (both octets compute the same copy; octet 0 stages it)
        float ih, ir, it, ssh, ssr, sst, sp;
        __syncwarp();   // the previous pair's phase 3 has finished reading the stage
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
                if (o2 == 0) { S.hr[half][i][l] = hr; S.rt[half][i][l] = rt; }
                const float4 up = hr - c;
                dot4_acc2(sp_part, up, up);
                S.Eh[i][lane] = f4(0.f);
                S.Et[i][lane] = f4(0.f);
            }
            sp = oct_sum(sp_part.x + sp_part.y);
        }
        __syncwarp();
        float Lp = 0.f, gp = 0.f;
        if (!margin_mode) loss_of(cfg.loss_kind, false, sp, cfg, Lp, gp);
        if (hl == 0 && live) lane_loss += Lp;

        // ---- phase 2: negatives, two at a time per positive (octet o2 of a half takes negative 2·round + o2) ----
        float Gh_s = 0.f, Gt_s = 0.f;
        const int rounds = (!FED && (P.diag & 4)) ? 0 : (k + 1) >> 1;
        for (int round = 0; round < rounds; ++round) {
            const int j = 2 * round + o2;
            const int src = hbase + (j < k ? j : 0);
            const bool valid = live && j < k && !((general_mask >> src) & 1u);
            const int e_id = __shfl_sync(OEA_FULL, neg_e, src);
            const bool head = (head_mask >> src) & 1u;
            R4 e = load_oct(ent.w, valid ? e_id : h, ent.pitch, l, p4);
            float2 sse2 = make_float2(0.f, 0.f);
#pragma unroll
            for (int i = 0; i < 4; ++i) dot4_acc2(sse2, e.v[i], e.v[i]);
            const float sse = oct_sum(sse2.x + sse2.y);
            const float ie = inv_norm(sse, ent.norm);
            // u = ê + (r̂ − t̂) for a corrupted head, (ĥ + r̂) − ê for a corrupted tail
            const float4* base = head ? &S.rt[half][0][0] : &S.hr[half][0][0];
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
                if (valid && v > 0.f) gp = 1.f;   // k == 1: only octet 0 of a half is valid; broadcast below
            } else {
                loss_of(cfg.loss_kind, true, sn, cfg, L, g);
            }
            if (!valid) { L = 0.f; g = 0.f; }
            if (l == 0) lane_loss += L;
            if (g != 0.f) {
                // d s/d ê = ±2u ; through the normaliser: (ĝ − ê<ê,ĝ>)/‖x‖
                const float c = 2.f * sgn * g * ie;
                const float proj = (ent.norm && sse >= kNormEps) ? de : 0.f;
                float4* acc = head ? &S.Eh[0][0] : &S.Et[0][0];
                float* grow = ent.g + (size_t)e_id * ent.pitch;
                const bool out = FED || !(P.diag & 2);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    acc[i * 32 + lane] = fma4(e.v[i], g, acc[i * 32 + lane]);
                    if (out && l + 8 * i < p4) red_add4(grow + 4 * (l + 8 * i), fma4(e.v[i], -proj, u.v[i]) * c);
                }
                if (head) Gh_s += g; else Gt_s += g;
                if (out && l == 0) ent.touched[e_id] = 1;
            }
        }
        if (margin_mode) gp = __shfl_sync(OEA_FULL, gp, hbase);

        // ---- FED only: negatives that share fewer than two rows with their positive, one at a time by the whole warp
        // (octet 0 / 1 / 2 holds row h / r / t of the general triple, octet 3 mirrors t and writes nothing) ----
        if (FED) {
            unsigned gm = general_mask;
            while (gm != 0u) {
                const int b = __ffs((int)gm) - 1;
                gm &= gm - 1u;
                const int eh = __shfl_sync(OEA_FULL, g_h, b), er = __shfl_sync(OEA_FULL, g_r, b), et = __shfl_sync(OEA_FULL, g_t, b);
                const float sp_b = __shfl_sync(OEA_FULL, sp, b);
                const int oct = lane >> 3;
                const int role = oct < 3 ? oct : 2;
                const TableDev tab = pick_table(role == 1, rel, ent);
                const int row = role == 0 ? eh : (role == 1 ? er : et);
                R4 x = load_oct(tab.w, row, tab.pitch, l, p4);
                float2 ss2 = make_float2(0.f, 0.f);
#pragma unroll
                for (int i = 0; i < 4; ++i) dot4_acc2(ss2, x.v[i], x.v[i]);
                const float ss = oct_sum(ss2.x + ss2.y);
                const float inv = inv_norm(ss, tab.norm);
                R4 u;
                float2 s2 = make_float2(0.f, 0.f);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    x.v[i] = x.v[i] * inv;
                    float4 a, bb, c;       // x̂_h, x̂_r, x̂_t slots (l + 8i) from octets 0, 1, 2
                    a.x = __shfl_sync(OEA_FULL, x.v[i].x, l); a.y = __shfl_sync(OEA_FULL, x.v[i].y, l);
                    a.z = __shfl_sync(OEA_FULL, x.v[i].z, l); a.w = __shfl_sync(OEA_FULL, x.v[i].w, l);
                    bb.x = __shfl_sync(OEA_FULL, x.v[i].x, 8 + l); bb.y = __shfl_sync(OEA_FULL, x.v[i].y, 8 + l);
                    bb.z = __shfl_sync(OEA_FULL, x.v[i].z, 8 + l); bb.w = __shfl_sync(OEA_FULL, x.v[i].w, 8 + l);
                    c.x = __shfl_sync(OEA_FULL, x.v[i].x, 16 + l); c.y = __shfl_sync(OEA_FULL, x.v[i].y, 16 + l);
                    c.z = __shfl_sync(OEA_FULL, x.v[i].z, 16 + l); c.w = __shfl_sync(OEA_FULL, x.v[i].w, 16 + l);
                    u.v[i] = (a + bb) - c;
                    dot4_acc2(s2, u.v[i], u.v[i]);
                }
                const float sn = oct_sum(s2.x + s2.y);
                float L = 0.f, g = 0.f;
                if (margin_mode) {
                    const float v = cfg.margin + sp_b - sn;
                    L = fmaxf(v, 0.f);
                    g = v > 0.f ? -1.f : 0.f;
                    if (v > 0.f && hbase == (b & 16)) gp = 1.f;
                } else {
                    loss_of(cfg.loss_kind, true, sn, cfg, L, g);
                }
                if (lane == 0) lane_loss += L;
                if (g != 0.f) {
                    float2 d2 = make_float2(0.f, 0.f);
#pragma unroll
                    for (int i = 0; i < 4; ++i) dot4_acc2(d2, x.v[i], u.v[i]);
                    const float sg = role == 2 ? -2.f * g : 2.f * g;           // d/dx̂ = ±2g·u
                    const float d = oct_sum(d2.x + d2.y);
                    const float proj = (tab.norm && ss >= kNormEps) ? d : 0.f;
                    if (oct < 3) {
                        R4 out;
#pragma unroll
                        for (int i = 0; i < 4; ++i) out.v[i] = fma4(x.v[i], -proj, u.v[i]) * (sg * inv);
                        red_oct(tab.g, row, tab.pitch, l, p4, out);
                        if (l == 0) tab.touched[row] = 1;
                    }
                }
            }
        }

        // ---- phase 3: merge each half's two octets, finish rows h and r (pass 0), then t (pass 1) ----
        Gh_s += __shfl_xor_sync(OEA_FULL, Gh_s, 8);
        Gt_s += __shfl_xor_sync(OEA_FULL, Gt_s, 8);
        __syncwarp();   // the accumulators of both octets of a half are visible
        const bool any = live && (gp != 0.f || Gh_s != 0.f || Gt_s != 0.f);
        if (__ballot_sync(OEA_FULL, any) != 0u) {
            // Ĝ = α·P + β·A + γ·B with per-role scalars:
            //   h: P + A      r: P + A + B      t: −P − B      (P = 2g⁺u⁺, A = 2(G_t·hr − E_t), B = 2(G_h·rt + E_h))
            const R4 xt = load_oct(ent.w, t, ent.pitch, l, p4);                          // L1 hit
#pragma unroll 1
            for (int pass = 0; pass < 2; ++pass) {
                const int role = pass == 0 ? o2 : 2;
                const int row = role == 0 ? h : (role == 1 ? r : t);
                const TableDev tab = pick_table(role == 1, rel, ent);
                const R4 xo = load_oct(tab.w, row, tab.pitch, l, p4);                    // L1 hit
                const float io = role == 0 ? ih : (role == 1 ? ir : it);
                const float so = role == 0 ? ssh : (role == 1 ? ssr : sst);
                const float alpha = role == 2 ? -2.f * gp : 2.f * gp;
                const float beta = role == 2 ? 0.f : 2.f, gamma = role == 0 ? 0.f : (role == 1 ? 2.f : -2.f);
                const float c_hr = alpha + beta * Gt_s, c_rt = gamma * Gh_s, c_t = -alpha * it;
                R4 G;
                float2 dpart2 = make_float2(0.f, 0.f);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float4 eh = S.Eh[i][hbase + l] + S.Eh[i][hbase + 8 + l];
                    const float4 et = S.Et[i][hbase + l] + S.Et[i][hbase + 8 + l];
                    // α(hr − t̂) + β(G_t·hr − E_t) + γ(G_h·rt + E_h)
                    float4 g4 = S.hr[half][i][l] * c_hr;
                    g4 = fma4(S.rt[half][i][l], c_rt, g4);
                    g4 = fma4(xt.v[i], c_t, g4);
                    g4 = fma4(et, -beta, g4);
                    g4 = fma4(eh, gamma, g4);
                    G.v[i] = g4;
                    dot4_acc2(dpart2, xo.v[i], g4);
                }
                const float dot = oct_sum((dpart2.x + dpart2.y) * io);
                const float proj = (tab.norm && so >= kNormEps) ? dot : 0.f;
                const bool out = FED || !(P.diag & 2);
                if (any && out && !(pass == 1 && o2 == 1)) {
                    R4 o;
#pragma unroll
                    for (int i = 0; i < 4; ++i) o.v[i] = fma4(xo.v[i] * io, -proj, G.v[i]) * io;
                    red_oct(tab.g, row, tab.pitch, l, p4, o);
                    if (l == 0) tab.touched[row] = 1;
                }
            }
        }
    }
    const float warp_loss = warp_sum(lane_loss);
    LossAcc acc{s_loss};
    acc.flush(warp_loss, loss_out, kDuoWarps);
}

}  // namespace oea
