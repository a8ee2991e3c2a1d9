// oea_triple_ext.cu — path (i), SURVEY §8f-2: the score functions of the reference's models/ on the fed boundary
// (index vectors in, gradients scattered into the tables), one warp per triple.  sm_90a.
//
// Maths restated from the reference (no code shared):
//   models/trans/transe.py:33-45       TransE   ĥ + r̂ − t̂ (oea_transe.cuh; also oea_triple_score_fed, pitch <= 512)
//   models/trans/transh.py:25-51       TransH   e⊥ = e − <e, n̂> n̂,  n̂ = l2_normalize(normal_vector[r])
//   approaches/bootea_transh.py:57-95   the same projection under the limited loss
//   models/trans/transd.py:26-65        TransD   e⊥ = l2_normalize(e + <e, e_p> r_p)
//   models/semantic/distmult.py:43-59   DistMult score Σ h∘r∘t, softplus(−label·score), reduce_mean
//   models/semantic/simple.py:50-86     SimplE   (Σ l2n(h_H∘r₁)∘t_T + Σ l2n(t_H∘r₂)∘h_T)/2, softplus(∓score)
//   models/semantic/rotate.py:52-110    RotatE   E = Σ_i |ĥ_i·e^{iθ_i} − t̂_i| − γ, θ = r̂·π/ρ, ρ = (γ + 2)/dim
//   approaches/bootea_rotate.py:48-108,149-160  the same energy; log-sigmoid losses, alignment loss = positives only
//   models/semantic/hole.py:41-86       HolE     E = −σ(<l2n(r̂), ccorr(ĥ, t̂)>), Σ relu(m + E⁺ − mean_k E⁻)
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
//
// RotatE and HolE (tests/semantic_ext_oracle.py states both graphs in float64 torch autograd):
//   * fp32 storage and arithmetic.  The reference creates RotatE's variables as float64; every table, optimiser and
//     similarity kernel of this engine is fp32, so RotatE trains in fp32.  cos/sin come from the accurate sincosf
//     (not __sinf/__cosf: θ reaches π·dim/(γ+2) ≈ 23 at the shipped γ = 12, d = 100, where the fast forms lose digits).
//   * The gradient of the modulus √(a² + b²) at a zero coordinate is taken as 0.  TF's gradient of tf.norm there is
//     NaN (0/0), the likely source of the NaN losses rotate.py:11-17 warns about; the engine stays finite instead.
//   * HolE computes the circular correlation directly, O(d²) per triple: ĥ and t̂ are staged twice over (indices
//     0 … 2d−1, so that i + k never needs a modulo) in this warp's shared memory, and lane l owns the output
//     coordinates k = l, l + 32, …  The index wraps modulo dim, never pitch.  HolE trains with the margin loss over the
//     reference batch layout (negatives of positive p at p·k … p·k+k−1, their energies averaged): k_hole_margin.
#include "oea_transe.cuh"

namespace oea {

// ---- one triple of each model (TransE, the base case, is in oea_transe.cuh) ----------------------------------------
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

__device__ __forceinline__ float comp(const float4& v, int j) { return j == 0 ? v.x : j == 1 ? v.y : j == 2 ? v.z : v.w; }
__device__ __forceinline__ float& comp(float4& v, int j) { return j == 0 ? v.x : j == 1 ? v.y : j == 2 ? v.z : v.w; }

// RotatE (rotate.py:61-93): ent = re_ent_embeds, ent_aux = im_ent_embeds, rel = rel_embeds (phases); SCORE unused.
// Per coordinate a = ĥ_re·cos θ − ĥ_im·sin θ − t̂_re, b = ĥ_re·sin θ + ĥ_im·cos θ − t̂_im, E = Σ √(a² + b²) − γ.
// Padding columns are zero in every table: θ = 0, a = b = 0, no contribution and (modulus gradient 0) no gradient.
template <int SCORE, int VEC>
struct Triple<OEA_MODEL_ROTATE, SCORE, VEC> {
    int h, r, t;
    NRow<VEC> hre, him, tre, tim, xr;
    Row<VEC> a, b, c, s;     // the two residuals and cos θ, sin θ of every coordinate
    __device__ __forceinline__ float forward(const ModelDev& M, int h_, int r_, int t_, int lane) {
        h = h_; r = r_; t = t_;
        hre = lookup<VEC>(M.ent, h, lane);
        him = lookup<VEC>(M.ent_aux, h, lane);
        tre = lookup<VEC>(M.ent, t, lane);
        tim = lookup<VEC>(M.ent_aux, t, lane);
        xr = lookup<VEC>(M.rel, r, lane);
        float dist = 0.f;
#pragma unroll
        for (int i = 0; i < VEC; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float sn, cs;
                sincosf(comp(xr.x.v[i], j) * M.phase, &sn, &cs);
                const float hr = comp(hre.x.v[i], j), hi = comp(him.x.v[i], j);
                const float av = fmaf(hr, cs, fmaf(-hi, sn, -comp(tre.x.v[i], j)));
                const float bv = fmaf(hr, sn, fmaf(hi, cs, -comp(tim.x.v[i], j)));
                comp(a.v[i], j) = av; comp(b.v[i], j) = bv;
                comp(c.v[i], j) = cs; comp(s.v[i], j) = sn;
                dist += sqrtf(fmaf(av, av, bv * bv));
            }
        return warp_sum(dist) - M.gamma;
    }
    __device__ __forceinline__ void backward(const ModelDev& M, float g, int lane) {
        Row<VEC> dhre, dhim, dtre, dtim, dr;
#pragma unroll
        for (int i = 0; i < VEC; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float av = comp(a.v[i], j), bv = comp(b.v[i], j), cs = comp(c.v[i], j), sn = comp(s.v[i], j);
                const float m = sqrtf(fmaf(av, av, bv * bv));
                const float w = m > 0.f ? g / m : 0.f;            // d|·|/d(a, b) = (a, b)/|·|, taken as 0 at 0
                const float da = av * w, db = bv * w;
                const float hr = comp(hre.x.v[i], j), hi = comp(him.x.v[i], j);
                comp(dhre.v[i], j) = fmaf(da, cs, db * sn);
                comp(dhim.v[i], j) = fmaf(db, cs, -da * sn);
                comp(dtre.v[i], j) = -da;
                comp(dtim.v[i], j) = -db;
                // dθ = da·(−ĥ_re·sin θ − ĥ_im·cos θ) + db·(ĥ_re·cos θ − ĥ_im·sin θ)
                const float dth = fmaf(da, -fmaf(hr, sn, hi * cs), db * fmaf(hr, cs, -hi * sn));
                comp(dr.v[i], j) = dth * M.phase;
            }
        push<VEC>(M.ent, h, lane, dhre, hre);
        push<VEC>(M.ent_aux, h, lane, dhim, him);
        push<VEC>(M.ent, t, lane, dtre, tre);
        push<VEC>(M.ent_aux, t, lane, dtim, tim);
        push<VEC>(M.rel, r, lane, dr, xr);
    }
};

// HolE (hole.py:48-60): ent, rel; s = <l2n(r̂), ccorr(ĥ, t̂)>, ccorr_k = Σ_i ĥ_i·t̂_{(i+k) mod dim}, E = −σ(s).
// `sm` is this warp's staging area of kHoleSmem floats: ĥ twice over [0, 2·256), t̂ twice over [512, 1024), the
// normalised relation [1024, 1280).  The context keeps its rows in registers and re-stages them whenever it uses the
// area, so several contexts of one warp may share it.
constexpr int kHoleMaxDim = 256;
constexpr int kHoleSmem = 5 * kHoleMaxDim;

template <int SCORE, int VEC>
struct Triple<OEA_MODEL_HOLE, SCORE, VEC> {
    static constexpr int MK = 4 * VEC;       // output coordinates per lane: k = lane + 32·m, m < MK
    int h, r, t;
    float* sm;
    NRow<VEC> xh, xt, xr, xn;                // xn = _calc's l2_normalize of the looked-up relation (hole.py:57)
    float sig;                               // σ(s)
    __device__ __forceinline__ void stage(int dim, int lane) {
        float* hh = sm;
        float* tt = sm + 2 * kHoleMaxDim;
        float* nn = sm + 4 * kHoleMaxDim;
        __syncwarp();                        // earlier readers of the area are done
#pragma unroll
        for (int i = 0; i < VEC; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int c = 4 * (lane + i * OEA_WARP) + j;
                if (c < dim) {
                    hh[c] = hh[c + dim] = comp(xh.x.v[i], j);
                    tt[c] = tt[c + dim] = comp(xt.x.v[i], j);
                    nn[c] = comp(xn.x.v[i], j);
                }
            }
        __syncwarp();
    }
    __device__ __forceinline__ float forward(const ModelDev& M, int h_, int r_, int t_, int lane) {
        h = h_; r = r_; t = t_;
        xh = lookup<VEC>(M.ent, h, lane);
        xt = lookup<VEC>(M.ent, t, lane);
        xr = lookup<VEC>(M.rel, r, lane);
        xn = normalised<VEC>(xr.x);
        const int dim = M.dim, mk = (dim + OEA_WARP - 1) / OEA_WARP;
        stage(dim, lane);
        const float* hh = sm;
        const float* tt = sm + 2 * kHoleMaxDim;
        const float* nn = sm + 4 * kHoleMaxDim;
        float cc[MK];
#pragma unroll
        for (int m = 0; m < MK; ++m) cc[m] = 0.f;
        for (int i = 0; i < dim; ++i) {
            const float hv = hh[i];
#pragma unroll
            for (int m = 0; m < MK; ++m)
                if (m < mk) cc[m] = fmaf(hv, tt[i + lane + m * OEA_WARP], cc[m]);
        }
        float sv = 0.f;
#pragma unroll
        for (int m = 0; m < MK; ++m) {
            const int k = lane + m * OEA_WARP;
            if (k < dim) sv = fmaf(nn[k], cc[m], sv);
        }
        sv = warp_sum(sv);
        sig = 1.f / (1.f + expf(-sv));
        return -sig;
    }
    __device__ __forceinline__ void backward(const ModelDev& M, float g, int lane) {
        const int dim = M.dim, mk = (dim + OEA_WARP - 1) / OEA_WARP, p4 = M.ent.pitch >> 2;
        const float gs = -g * sig * (1.f - sig);                 // d loss / d s
        stage(dim, lane);
        float* hh = sm;
        float* tt = sm + 2 * kHoleMaxDim;
        float* nn = sm + 4 * kHoleMaxDim;
        float cc[MK], dh[MK], dt[MK];
#pragma unroll
        for (int m = 0; m < MK; ++m) cc[m] = dh[m] = dt[m] = 0.f;
        // ∂s/∂n_k = ccorr_k,  ∂s/∂ĥ_i = Σ_k n_k·t̂_{i+k},  ∂s/∂t̂_j = Σ_k n_k·ĥ_{j−k}  (all indices mod dim)
        for (int q = 0; q < dim; ++q) {
            const float hv = hh[q], nv = nn[q];
#pragma unroll
            for (int m = 0; m < MK; ++m) {
                if (m < mk) {
                    const int o = lane + m * OEA_WARP;
                    cc[m] = fmaf(hv, tt[q + o], cc[m]);
                    dh[m] = fmaf(nv, tt[q + o], dh[m]);
                    dt[m] = fmaf(nv, hh[o - q + dim], dt[m]);
                }
            }
        }
        __syncwarp();                                            // every lane has read the staged rows
#pragma unroll
        for (int m = 0; m < MK; ++m) {
            const int o = lane + m * OEA_WARP;
            if (o < 4 * p4) {                                    // padding columns of the results are zero
                const bool in = o < dim;
                hh[o] = in ? gs * dh[m] : 0.f;
                tt[o] = in ? gs * dt[m] : 0.f;
                nn[o] = in ? gs * cc[m] : 0.f;
            }
        }
        __syncwarp();
        Row<VEC> gh, gt, gn;
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
            const int c = lane + i * OEA_WARP;
            const bool in = c < p4;
            gh.v[i] = in ? make_float4(hh[4 * c], hh[4 * c + 1], hh[4 * c + 2], hh[4 * c + 3]) : f4(0.f);
            gt.v[i] = in ? make_float4(tt[4 * c], tt[4 * c + 1], tt[4 * c + 2], tt[4 * c + 3]) : f4(0.f);
            gn.v[i] = in ? make_float4(nn[4 * c], nn[4 * c + 1], nn[4 * c + 2], nn[4 * c + 3]) : f4(0.f);
        }
        push<VEC>(M.ent, h, lane, gh, xh);
        push<VEC>(M.ent, t, lane, gt, xt);
        push<VEC>(M.rel, r, lane, back_normalised<VEC>(gn, xn), xr);
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
        float ep, en;
        if constexpr (MODEL == OEA_MODEL_TRANSE) {      // six row loads in flight before the first reduction
            P.gather(M, __ldg(ph + i), __ldg(pr + i), __ldg(pt + i), lane);
            N.gather(M, __ldg(nh + i), __ldg(nr + i), __ldg(nt + i), lane);
            ep = P.score(M);
            en = N.score(M);
            warp_sum2(ep, en);
        } else {
            ep = P.forward(M, __ldg(ph + i), __ldg(pr + i), __ldg(pt + i), lane);
            en = N.forward(M, __ldg(nh + i), __ldg(nr + i), __ldg(nt + i), lane);
        }
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

// HolE's margin loss over the reference batch layout (hole.py:78-84): Σ_p relu(m + E⁺_p − (1/k)·Σ_j E⁻_{p·k+j}).
// One warp per positive and its k negatives; at k = 1 this is k_model_margin's pairing.  The negatives' contexts are
// not kept (k is a run-time value): an active pair recomputes each negative's forward before its backward.
template <int VEC>
__global__ void __launch_bounds__(kThreads)
k_hole_margin(ModelDev M,
              const int32_t* __restrict__ ph, const int32_t* __restrict__ pr, const int32_t* __restrict__ pt,
              const int32_t* __restrict__ nh, const int32_t* __restrict__ nr, const int32_t* __restrict__ nt, int n_pos,
              int k, oea_loss_cfg cfg, float scale, double* __restrict__ loss_out) {
    using HolE = Triple<OEA_MODEL_HOLE, OEA_SCORE_L2SQ, VEC>;
    __shared__ float s_stage[kWarpsPerBlock][kHoleSmem];
    __shared__ double s_loss[kWarpsPerBlock];
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    float* sm = s_stage[threadIdx.x >> 5];
    const float inv_k = 1.f / (float)k;
    float warp_loss = 0.f;
    for (int i = warp_global; i < n_pos; i += n_warps) {
        HolE P;
        P.sm = sm;
        const float ep = P.forward(M, __ldg(ph + i), __ldg(pr + i), __ldg(pt + i), lane);
        float en = 0.f;
        for (int j = 0; j < k; ++j) {
            const int q = i * k + j;
            HolE N;
            N.sm = sm;
            en += N.forward(M, __ldg(nh + q), __ldg(nr + q), __ldg(nt + q), lane);
        }
        const float v = cfg.margin + ep - en * inv_k;
        warp_loss += fmaxf(v, 0.f) * scale;
        if (v > 0.f) {
            P.backward(M, scale, lane);
            for (int j = 0; j < k; ++j) {
                const int q = i * k + j;
                HolE N;
                N.sm = sm;
                N.forward(M, __ldg(nh + q), __ldg(nr + q), __ldg(nt + q), lane);
                N.backward(M, -scale * inv_k, lane);
            }
        }
    }
    LossAcc acc{s_loss};
    acc.flush(warp_loss, loss_out);
}

static int check_model(const oea_model* m, ModelDev* out) {
    if (m == nullptr) return OEA_ERR_NULL;
    if (m->kind < OEA_MODEL_TRANSE || m->kind > OEA_MODEL_HOLE) return OEA_ERR_KIND;
    const bool need_ent_aux = m->kind == OEA_MODEL_TRANSD || m->kind == OEA_MODEL_SIMPLE || m->kind == OEA_MODEL_ROTATE;
    const bool need_rel_aux = m->kind == OEA_MODEL_TRANSH || m->kind == OEA_MODEL_TRANSD || m->kind == OEA_MODEL_SIMPLE;
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
    out->dim = m->ent->dim;
    out->gamma = m->kind == OEA_MODEL_ROTATE ? m->gamma : 0.f;
    out->phase = m->kind == OEA_MODEL_ROTATE ? m->phase : 0.f;
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
    const bool margin = loss->loss_kind == OEA_LOSS_MARGIN;
    cudaStream_t st = (cudaStream_t)stream;

#ifdef OEA_HOST_EMU   // tests/emu: the same kernels on the CPU warp emulator (two blocks keep the thread count small)
#define OEA_RUN(KERNEL, ...) emu::launch(grid < 2 ? grid : 2, kThreads, [&] { KERNEL(__VA_ARGS__); })
#else
#define OEA_RUN(KERNEL, ...) KERNEL<<<grid, kThreads, 0, st>>>(__VA_ARGS__)
#endif

    // RotatE: the independent losses only (its own log-sigmoid pair is OEA_LOSS_LOGISTIC); score_kind is not read
    if (model->kind == OEA_MODEL_ROTATE) {
        if (margin) return OEA_ERR_KIND;
        if (n_pos + n_neg == 0) return OEA_OK;
        const int grid = grid_for(n_pos + n_neg);
        if (model->ent->pitch <= 128) {
            auto kernel = k_model_fed<OEA_MODEL_ROTATE, OEA_SCORE_L2SQ, 1>;
            OEA_RUN(kernel, M, pos_h, pos_r, pos_t, n_pos, neg_h, neg_r, neg_t, n_neg, *loss, loss_scale, loss_out);
        } else {
            auto kernel = k_model_fed<OEA_MODEL_ROTATE, OEA_SCORE_L2SQ, 2>;
            OEA_RUN(kernel, M, pos_h, pos_r, pos_t, n_pos, neg_h, neg_r, neg_t, n_neg, *loss, loss_scale, loss_out);
        }
        OEA_LAUNCH_CHECK();
        return OEA_OK;
    }
    // HolE: the margin loss with n_neg / n_pos negatives per positive (reference layout); score_kind is not read
    if (model->kind == OEA_MODEL_HOLE) {
        if (!margin) return OEA_ERR_KIND;
        if (n_pos + n_neg == 0) return OEA_OK;
        if (n_pos == 0 || n_neg % n_pos != 0 || n_neg == 0) return OEA_ERR_SHAPE;
        const int k = n_neg / n_pos;
        const int grid = grid_for(n_pos);
        if (model->ent->pitch <= 128) {
            auto kernel = k_hole_margin<1>;
            OEA_RUN(kernel, M, pos_h, pos_r, pos_t, neg_h, neg_r, neg_t, n_pos, k, *loss, loss_scale, loss_out);
        } else {
            auto kernel = k_hole_margin<2>;
            OEA_RUN(kernel, M, pos_h, pos_r, pos_t, neg_h, neg_r, neg_t, n_pos, k, *loss, loss_scale, loss_out);
        }
        OEA_LAUNCH_CHECK();
        return OEA_OK;
    }

    const bool bilinear = model->kind == OEA_MODEL_DISTMULT || model->kind == OEA_MODEL_SIMPLE;
    if (!bilinear && loss->score_kind != OEA_SCORE_L1 && loss->score_kind != OEA_SCORE_L2SQ) return OEA_ERR_KIND;
    if (margin && n_pos != n_neg) return OEA_ERR_SHAPE;
    if (n_pos + n_neg == 0) return OEA_OK;
    const bool l1 = !bilinear && loss->score_kind == OEA_SCORE_L1;
    const int grid = grid_for(margin ? n_pos : n_pos + n_neg);
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
        default: OEA_LAUNCH_VEC(OEA_MODEL_SIMPLE, OEA_SCORE_L2SQ); break;   // SIMPLE (ROTATE / HOLE returned above)
    }
#undef OEA_LAUNCH_SCORE
#undef OEA_LAUNCH_VEC
#undef OEA_LAUNCH_MODEL
#undef OEA_RUN
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

// TransE with the tables of the call (path (i)'s fed scorer): the kernels above at every pitch up to 512.
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
    const TableDev e = table_dev(ent), r = table_dev(rel);
    const ModelDev M{e, r, e, r, ent->dim, 0.f, 0.f};
    const bool l1 = loss->score_kind == OEA_SCORE_L1;
    if (loss->loss_kind == OEA_LOSS_MARGIN) {
        const int grid = grid_for(n_pos);
#define CALL(V)                                                                                                         \
        if (l1) OEA_LAUNCH((k_model_margin<OEA_MODEL_TRANSE, OEA_SCORE_L1, V>), grid, kThreads, 0, st, M, pos_h, pos_r, pos_t, neg_h, neg_r, neg_t, n_pos, *loss, 1.f, loss_out); \
        else OEA_LAUNCH((k_model_margin<OEA_MODEL_TRANSE, OEA_SCORE_L2SQ, V>), grid, kThreads, 0, st, M, pos_h, pos_r, pos_t, neg_h, neg_r, neg_t, n_pos, *loss, 1.f, loss_out)
        OEA_DISPATCH_VEC(ent->pitch, CALL);
#undef CALL
    } else {
#define CALL(V)                                                                                                         \
        if (l1) { const int grid = grid_one_wave<k_model_fed<OEA_MODEL_TRANSE, OEA_SCORE_L1, V>>(n_pos + n_neg);        \
                  OEA_LAUNCH((k_model_fed<OEA_MODEL_TRANSE, OEA_SCORE_L1, V>), grid, kThreads, 0, st, M, pos_h, pos_r, pos_t, n_pos, neg_h, neg_r, neg_t, n_neg, *loss, 1.f, loss_out); } \
        else { const int grid = grid_one_wave<k_model_fed<OEA_MODEL_TRANSE, OEA_SCORE_L2SQ, V>>(n_pos + n_neg);         \
               OEA_LAUNCH((k_model_fed<OEA_MODEL_TRANSE, OEA_SCORE_L2SQ, V>), grid, kThreads, 0, st, M, pos_h, pos_r, pos_t, n_pos, neg_h, neg_r, neg_t, n_neg, *loss, 1.f, loss_out); }
        OEA_DISPATCH_VEC(ent->pitch, CALL);
#undef CALL
    }
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}
