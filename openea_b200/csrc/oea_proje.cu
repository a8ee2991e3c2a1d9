// oea_proje.cu — path (i), ProjE: TF's unique log-uniform candidate sampler on the device and the step of
// models/neural/proje.py:46-74 (a projection layer with three training-mode batch norms, then tf.nn.nce_loss over one
// sampled set of classes the whole batch shares).  The same sampler and NCE head also make the general sampled-NCE step
// of approaches/attr2vec.py:113-124 (oea_nce_score_fed) and its per-step pair draw (oea_pairs_draw).
// sm_90a, FP32 FFMA only.
//
// Maths restated from the reference and from TF 1.x (no code shared):
//   models/neural/proje.py:51-62   x_h = ê[h], x_r = r̂[r]; y_h = BN(x_h), y_r = BN(x_r) with ONE shared beta and each its
//                                  own batch moments; z = y_h·w + y_r·w + b (the same mlp_w twice, AUTO_REUSE); X = BN_out(z)
//                                  BN: contrib.layers.batch_norm defaults — training mode, biased batch variance,
//                                  ε = 1e-3, center (beta), no scale
//   models/neural/proje.py:64-72   Σ_b nce_loss(entity_w, entity_b, t_b, X_b, num_sampled = S, num_classes = E):
//                                  logits x·w_c + b_c − log q(c), sigmoid cross-entropy (true class → 1, sampled → 0),
//                                  accidental hits kept
//   LogUniformSampler              P(c) = log((c+2)/(c+1)) / log(E+1); draw = ⌊exp(u·log(E+1))⌋ − 1 mod E; unique: the
//                                  first S distinct draws, num_tries = draws taken; expected count
//                                  q(c) = −expm1(num_tries·log1p(−P(c))), or P(c)·S when num_tries == S (fp32, as TF)
//
// oea_logu_sample_unique: one CTA.  Draw j is a pure function of (seed, j).  Rounds of kRound draws: every draw
// atomicMin's its index into first[class], so after the round's barrier draw j is new iff first[class] == j (a class
// drawn in an earlier round, or earlier in this round, holds a smaller index).  A block scan over the new draws in draw
// order gives their positions; the draw that takes position S − 1 writes num_tries.  Exactly the sequential loop's result.
//
// oea_proje_score_fed: a memset and nine kernels on `stream`, no allocation, no host synchronisation:
//   1. k_proje_gather       one warp per positive: ê[h], r̂[r] into the workspace
//   2. k_proje_columns_fwd  one CTA per column: both input BNs, the shared-weight combination, the output BN → X
//   3. k_nce_logq           log q(c) of the sampled set, once
//      k_nce_logits         128 × 128 tiles of X·W_Sᵀ (W_S = entity_w rows of the sampled set): the sampled logits'
//                           loss, G = σ(logit) into the workspace, Σ_b G into entity_b's gradient
//   4. k_nce_dx             dX = G·W_S, split over the sampled set so that a batch of 500 still fills the machine
//   5. k_nce_dw             dW_S = Gᵀ·X, split over the batch, pushed with red.global.add.v4.f32 (a sampled row may also
//                           be a label row)
//   6. k_nce_true           one warp per positive, scale 1 over the raw entity_w: the true logit, its loss, g = σ(t) − 1
//                           into dX, entity_w and entity_b
//   7. k_proje_columns_bwd  one CTA per column: back through the three BNs and the combination; the gradients of mlp_w,
//                           mlp_bias and both betas are this CTA's column sums
//   8. k_proje_push         one warp per positive: dx_h, dx_r through the tables' normalisation into ent.grad, rel.grad
//
// oea_nce_score_fed: loss_scale · Σ_b nce_loss(ŵ, b, label_b, x̂[input_b]) with each table normalised or raw by its own
// flag.  A memset and nine kernels, the head's three GEMMs shared with ProjE through the W_S addressing policy:
//   1. k_nce_stage          one warp per sampled class: ŵ_s and its 1/‖w_s‖, Σw² into the workspace ([S, pitch],
//                           contiguous), dŴ_s zeroed
//   2. k_nce_gather         one warp per row of the batch: x̂[input_b] into the workspace
//   3. k_nce_logq, k_nce_logits<StagedW>, k_nce_dx<StagedW>, k_nce_dw<StagedW>: the head over the staged block; G
//                           carries the scale, dŴ_S accumulates in the workspace
//   4. k_nce_true           one warp per row: ŵ_label normalised in registers, the true logit, its loss, dX, and its
//                           part of the label row's gradient pushed through the normalisation itself
//   5. k_nce_w_push         one warp per sampled class: dŴ_s through the normalisation into cls_w.grad (red: a sampled
//                           class can also be a label; the Jacobian is linear, so the two parts are pushed separately)
//   6. k_nce_in_push        one warp per row: dX through the input table's normalisation into its gradient
//
// oea_conve_score_fed (models/neural/conve.py:42-79): two memsets and thirteen kernels, ProjE's head among them unchanged:
//   1. k_conve_conv_fwd     one CTA per positive: the stacked image, its batch norm and dropout (kept in img), the 3×3
//                           convolution, the per-filter batch norm, ReLU and dropout → A [n, 2Fd]
//   2. k_nce_dx<StagedW>    Z = A·W: the head's dX kernel with G := A, S := 2Fd and W_S := fc_w, split over the 2Fd
//                           inputs; k_conve_fc_out: bias, ReLU and the output batch norm → X
//   3. the head: k_nce_logq, k_nce_logits / k_nce_dx / k_nce_dw <GatheredW>, k_nce_true
//   4. k_conve_fc_out_bwd   dX → dz; k_nce_dw<StagedW>: dW = Aᵀ·dz (the head's dW kernel, G := A, X := dz);
//                           k_conve_fc_dx: dA = dz·Wᵀ through the ReLU and dropout, written over A
//   5. k_conve_conv_dw      the convolution's and its batch norm's gradients per filter; k_conve_conv_dx: one CTA per
//                           positive back to the image, through its dropout and batch norm, and into ent.grad, rel.grad
//
// oea_pairs_draw: B distinct rows of an [n, 2] pair array, row i = feistel_perm(i, n, key(seed, epoch, step)) for i < B.
#include "oea_rowmath.cuh"

namespace oea {

constexpr int kProjeMaxPitch = 128;
constexpr float kBnEps = 1e-3f;                   // tf.contrib.layers.batch_norm epsilon
constexpr int kDrawsPerThread = 16;
constexpr int kRound = kThreads * kDrawsPerThread;
constexpr int kTile = 128;                        // GEMM tile: 128 × 128 outputs, 16 × 16 threads of 8 × 8
constexpr int kTk = 16;                           // reduction slice staged per iteration
constexpr int kTld = kTile + 4;                   // shared row stride of a staged slice

// a row width in floats rounded up to whole float4s: table pitches, and the row strides of G and ConvE's A
constexpr int round4(int v) { return (v + 3) / 4 * 4; }

// a workspace cut into sections in the order they are taken, each 256-B aligned; `at` ends as the total
struct WsCarver {
    size_t at = 0;
    size_t take(size_t bytes) { const size_t o = at; at += (bytes + 255) & ~(size_t)255; return o; }
};

struct ProjeWs {
    size_t first, xh, xr, z, x, dx, dxh, dxr, stats, lq, g, total;
    int ldg;                                      // row stride of G: S rounded up to 4
};

// workspace sections: the sampler's first-draw index per class, then per positive six rows of `pitch` floats, eight
// rows of column statistics, log q of every sampled class, and G [n_pos, ldg]
static ProjeWs proje_layout(int n_pos, int num_sampled, int pitch, int n_classes) {
    ProjeWs w;
    WsCarver c;
    const size_t row = 4 * (size_t)n_pos * pitch;
    w.ldg = round4(num_sampled);
    w.first = c.take(4 * (size_t)n_classes);
    w.xh = c.take(row);
    w.xr = c.take(row);
    w.z = c.take(row);
    w.x = c.take(row);
    w.dx = c.take(row);
    w.dxh = c.take(row);
    w.dxr = c.take(row);
    w.stats = c.take(4 * 8 * (size_t)pitch);
    w.lq = c.take(4 * (size_t)num_sampled);
    w.g = c.take(4 * (size_t)n_pos * w.ldg);
    w.total = c.at;
    return w;
}

// ---- the sampler ---------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ int logu_draw(uint64_t seed, long long j, double log_range, int n_classes) {
    const uint64_t r = mix64(seed ^ mix64((uint64_t)j));
    const double u = (double)(r >> 11) * 0x1.0p-53;
    const long long v = (long long)exp(u * log_range) - 1;
    return (int)(v % n_classes);
}

// block-wide exclusive scan of one int per thread; *total gets the sum.  s has kWarpsPerBlock ints.
__device__ __forceinline__ int block_excl_scan(int v, int* s, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(OEA_FULL, inc, o);
        if (lane >= o) inc += u;
    }
    if (lane == 31) s[warp] = inc;
    __syncthreads();
    int before = 0, all = 0;
    for (int w = 0; w < kWarpsPerBlock; ++w) {
        if (w < warp) before += s[w];
        all += s[w];
    }
    *total = all;
    __syncthreads();                                      // s is reused by the next scan
    return before + inc - v;
}

__global__ void __launch_bounds__(kThreads)
k_logu_sample(int n_classes, int num_sampled, uint64_t seed, int32_t* __restrict__ first, int32_t* __restrict__ sampled,
              int32_t* __restrict__ num_tries) {
    __shared__ int s_scan[kWarpsPerBlock];
    const double log_range = log1p((double)n_classes);
    for (int c = threadIdx.x; c < n_classes; c += blockDim.x) first[c] = INT_MAX;
    __syncthreads();
    int picked = 0;                                       // block-uniform
    for (long long base = 0; picked < num_sampled; base += kRound) {
        int cls[kDrawsPerThread];
        const long long j0 = base + (long long)threadIdx.x * kDrawsPerThread;
#pragma unroll
        for (int k = 0; k < kDrawsPerThread; ++k) {
            cls[k] = logu_draw(seed, j0 + k, log_range, n_classes);
            atomicMin(first + cls[k], (int)(j0 + k));
        }
        __syncthreads();
        unsigned fresh = 0;
#pragma unroll
        for (int k = 0; k < kDrawsPerThread; ++k)
            if (__ldcg(first + cls[k]) == (int)(j0 + k)) fresh |= 1u << k;
        int total;
        int at = picked + block_excl_scan(__popc(fresh), s_scan, &total);
#pragma unroll
        for (int k = 0; k < kDrawsPerThread; ++k) {
            if (!((fresh >> k) & 1u)) continue;
            if (at < num_sampled) sampled[at] = cls[k];
            if (at == num_sampled - 1) *num_tries = (int32_t)(j0 + k + 1);
            ++at;
        }
        picked += total;
    }
}

// q(c) of TF's RangeSampler for the log-uniform distribution, in fp32
__device__ __forceinline__ float log_expected_count(int c, int n_classes, int num_sampled, int num_tries) {
    const float p = (float)(log((c + 2.0) / (c + 1.0)) / log1p((double)n_classes));
    const float q = num_tries == num_sampled ? p * (float)num_sampled : -expm1f((float)num_tries * log1pf(-p));
    return logf(q);
}

// log q(c) of every sampled class, once per call: the logits' epilogue reads it for each row tile
__global__ void __launch_bounds__(kThreads)
k_nce_logq(const int32_t* __restrict__ sampled, const int32_t* __restrict__ num_tries, int n_classes, int num_sampled,
           float* __restrict__ lq) {
    const int tries = *num_tries;
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < num_sampled; s += gridDim.x * blockDim.x)
        lq[s] = log_expected_count(__ldg(sampled + s), n_classes, num_sampled, tries);
}

__device__ __forceinline__ float sigmoid_acc(float x) { return 1.f / (1.f + expf(-x)); }

// num_sampled and ldg are the columns of G and its row stride: the sampled set's size S and round4(S) in the head, and
// 2Fd and A's row stride when ConvE's dense layer runs on k_nce_dx / k_nce_dw with G := A
struct ProjeDev {
    TableDev ent, rel, w, b, prm;
    int dim, pitch, n_classes, num_sampled, ldg;
};

// How the NCE head addresses the sampled classes' rows W_S and scales its loss (the last kernel argument).  The row of
// sampled slot s is asked for with `id` = sampled + s, written as the kernel always wrote it (ProjE's SASS depends on
// that address arithmetic), and with s itself.  ProjE: entity_w rows gathered by class id, dW_S reduced straight into
// entity_w's gradient, the loss summed.
struct GatheredW {
    __device__ __forceinline__ const float* w_row(const ProjeDev& T, const int32_t* id, int) const {
        return T.w.w + (size_t)__ldg(id) * T.pitch;
    }
    __device__ __forceinline__ float* dw_row(const ProjeDev& T, const int32_t* id, int) const {
        return T.w.g + (size_t)__ldg(id) * T.pitch;
    }
    __device__ __forceinline__ float scaled(float v) const { return v; }
};
// oea_nce_score_fed: ŵ_S staged contiguously by k_nce_stage, dŴ_S accumulated in the workspace (k_nce_w_push takes it
// through the normalisation), loss and every gradient times `scale`.  ConvE's dense layer: fc_w and its gradient.
struct StagedW {
    const float* w;
    float* dw;
    float scale;
    __device__ __forceinline__ const float* w_row(const ProjeDev& T, const int32_t*, int s) const {
        return w + (size_t)s * T.pitch;
    }
    __device__ __forceinline__ float* dw_row(const ProjeDev& T, const int32_t*, int s) const { return dw + (size_t)s * T.pitch; }
    __device__ __forceinline__ float scaled(float v) const { return v * scale; }
};

// ---- projection layer ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_proje_gather(ProjeDev T, const int32_t* __restrict__ ph, const int32_t* __restrict__ pr, int n,
               float* __restrict__ xh, float* __restrict__ xr) {
    const int lane = threadIdx.x & 31;
    for (int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < n; b += (gridDim.x * blockDim.x) >> 5) {
        const Row<1> h = lookup<1>(T.ent, __ldg(ph + b), lane).x, r = lookup<1>(T.rel, __ldg(pr + b), lane).x;
        if (4 * lane < T.pitch) {
            *reinterpret_cast<float4*>(xh + (size_t)b * T.pitch + 4 * lane) = h.v[0];
            *reinterpret_cast<float4*>(xr + (size_t)b * T.pitch + 4 * lane) = r.v[0];
        }
    }
}

// the sums of a and b over the block, returned to every thread
__device__ __forceinline__ void block_sum2(float& a, float& b, float* s) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    a = warp_sum(a);
    b = warp_sum(b);
    if (lane == 0) { s[2 * warp] = a; s[2 * warp + 1] = b; }
    __syncthreads();
    a = b = 0.f;
    for (int w = 0; w < kWarpsPerBlock; ++w) { a += s[2 * w]; b += s[2 * w + 1]; }
    __syncthreads();
}

// stats rows: 0 μ_h, 1 rstd_h, 2 μ_r, 3 rstd_r, 4 μ_z, 5 rstd_z.  params rows: 0 mlp_w, 1 mlp_bias, 2 β_in, 3 β_out.
__global__ void __launch_bounds__(kThreads)
k_proje_columns_fwd(ProjeDev T, int n, const float* __restrict__ xh, const float* __restrict__ xr, float* __restrict__ z,
                    float* __restrict__ x, float* __restrict__ stats) {
    __shared__ float s_red[2 * kWarpsPerBlock];
    const int P = T.pitch;
    const float inv_n = 1.f / (float)n;
    for (int c = blockIdx.x; c < P; c += gridDim.x) {
        if (c >= T.dim) {                                 // padding columns of X stay zero for the head's float4 loads
            for (int b = threadIdx.x; b < n; b += blockDim.x) x[(size_t)b * P + c] = 0.f;
            continue;
        }
        float sh = 0.f, sr = 0.f;
        for (int b = threadIdx.x; b < n; b += blockDim.x) { sh += xh[(size_t)b * P + c]; sr += xr[(size_t)b * P + c]; }
        block_sum2(sh, sr, s_red);
        const float mh = sh * inv_n, mr = sr * inv_n;
        float vh = 0.f, vr = 0.f;
        for (int b = threadIdx.x; b < n; b += blockDim.x) {
            const float a = xh[(size_t)b * P + c] - mh, e = xr[(size_t)b * P + c] - mr;
            vh = fmaf(a, a, vh);
            vr = fmaf(e, e, vr);
        }
        block_sum2(vh, vr, s_red);
        const float rh = rsqrtf(vh * inv_n + kBnEps), rr = rsqrtf(vr * inv_n + kBnEps);
        const float w = T.prm.w[c], bias = T.prm.w[P + c], beta_in = T.prm.w[2 * P + c], beta_out = T.prm.w[3 * P + c];
        float sz = 0.f, unused = 0.f;
        for (int b = threadIdx.x; b < n; b += blockDim.x) {
            const float yh = fmaf(xh[(size_t)b * P + c] - mh, rh, beta_in), yr = fmaf(xr[(size_t)b * P + c] - mr, rr, beta_in);
            const float v = yh * w + yr * w + bias;
            z[(size_t)b * P + c] = v;
            sz += v;
        }
        block_sum2(sz, unused, s_red);
        const float mz = sz * inv_n;
        float vz = 0.f;
        unused = 0.f;
        for (int b = threadIdx.x; b < n; b += blockDim.x) {
            const float a = z[(size_t)b * P + c] - mz;
            vz = fmaf(a, a, vz);
        }
        block_sum2(vz, unused, s_red);
        const float rz = rsqrtf(vz * inv_n + kBnEps);
        for (int b = threadIdx.x; b < n; b += blockDim.x) x[(size_t)b * P + c] = fmaf(z[(size_t)b * P + c] - mz, rz, beta_out);
        if (threadIdx.x == 0) {
            stats[c] = mh; stats[P + c] = rh; stats[2 * P + c] = mr; stats[3 * P + c] = rr;
            stats[4 * P + c] = mz; stats[5 * P + c] = rz;
        }
    }
}

__global__ void __launch_bounds__(kThreads)
k_proje_columns_bwd(ProjeDev T, int n, const float* __restrict__ xh, const float* __restrict__ xr,
                    const float* __restrict__ z, float* __restrict__ dx, const float* __restrict__ stats,
                    float* __restrict__ dxh, float* __restrict__ dxr) {
    __shared__ float s_red[2 * kWarpsPerBlock];
    const int P = T.pitch;
    const float inv_n = 1.f / (float)n;
    for (int c = blockIdx.x; c < P; c += gridDim.x) {
        if (c >= T.dim) {                                 // padding columns: the push reads whole rows
            for (int b = threadIdx.x; b < n; b += blockDim.x) dxh[(size_t)b * P + c] = dxr[(size_t)b * P + c] = 0.f;
            continue;
        }
        const float mh = stats[c], rh = stats[P + c], mr = stats[2 * P + c], rr = stats[3 * P + c];
        const float mz = stats[4 * P + c], rz = stats[5 * P + c];
        const float w = T.prm.w[c], beta_in = T.prm.w[2 * P + c];
        // output BN: dβ_out = Σ dX, dz = rstd·(dX − mean dX − ẑ·mean(dX·ẑ))
        float s1 = 0.f, s2 = 0.f;
        for (int b = threadIdx.x; b < n; b += blockDim.x) {
            const float g = dx[(size_t)b * P + c];
            s1 += g;
            s2 = fmaf(g, (z[(size_t)b * P + c] - mz) * rz, s2);
        }
        block_sum2(s1, s2, s_red);
        const float m1 = s1 * inv_n, m2 = s2 * inv_n;
        // dz (stored over dX), and the sums the combination and the input BNs need
        float sdz = 0.f, sdw = 0.f, sh = 0.f, sr = 0.f;
        for (int b = threadIdx.x; b < n; b += blockDim.x) {
            const size_t i = (size_t)b * P + c;
            const float zh = (z[i] - mz) * rz;
            const float dz = rz * (dx[i] - m1 - zh * m2);
            dx[i] = dz;
            const float nh = (xh[i] - mh) * rh, nr = (xr[i] - mr) * rr;
            sdz += dz;
            sdw = fmaf(dz, nh + beta_in + nr + beta_in, sdw);
            sh = fmaf(dz, nh, sh);
            sr = fmaf(dz, nr, sr);
        }
        block_sum2(sdz, sdw, s_red);
        block_sum2(sh, sr, s_red);
        // input BNs: dy = w·dz for both; dx̂ = rstd·(dy − mean dy − x̂·mean(dy·x̂))
        const float md = w * sdz * inv_n, mdh = w * sh * inv_n, mdr = w * sr * inv_n;
        for (int b = threadIdx.x; b < n; b += blockDim.x) {
            const size_t i = (size_t)b * P + c;
            const float dy = w * dx[i];
            dxh[i] = rh * (dy - md - (xh[i] - mh) * rh * mdh);
            dxr[i] = rr * (dy - md - (xr[i] - mr) * rr * mdr);
        }
        if (threadIdx.x == 0) {
            T.prm.g[c] += sdw;
            T.prm.g[P + c] += sdz;
            T.prm.g[2 * P + c] += 2.f * w * sdz;
            T.prm.g[3 * P + c] += s1;
            if (c == 0)
                for (int r = 0; r < 4; ++r) T.prm.touched[r] = 1;
        }
    }
}

__global__ void __launch_bounds__(kThreads)
k_proje_push(ProjeDev T, const int32_t* __restrict__ ph, const int32_t* __restrict__ pr, int n,
             const float* __restrict__ dxh, const float* __restrict__ dxr) {
    const int lane = threadIdx.x & 31;
    for (int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < n; b += (gridDim.x * blockDim.x) >> 5) {
        const int h = __ldg(ph + b), r = __ldg(pr + b);
        push<1>(T.ent, h, lane, load_row<1>(dxh, b, T.pitch, lane), lookup<1>(T.ent, h, lane));
        push<1>(T.rel, r, lane, load_row<1>(dxr, b, T.pitch, lane), lookup<1>(T.rel, r, lane));
    }
}

// ---- the NCE head: 128 × 128 FP32 register tiles -------------------------------------------------------------------
// C[m][n] += Σ_{k<kTk} As[k][m]·Bs[k][n] for this thread's 8 × 8 outputs m = ty + 16a, n = tx + 16b.  The 16 threads of
// a half-warp share ty (one broadcast address of As) and read 16 consecutive n of Bs: conflict-free.
__device__ __forceinline__ void tile_mma(float (&acc)[8][8], const float* As, const float* Bs, int ty, int tx) {
#pragma unroll
    for (int k = 0; k < kTk; ++k) {
        float av[8], bv[8];
#pragma unroll
        for (int a = 0; a < 8; ++a) av[a] = As[k * kTld + ty + 16 * a];
#pragma unroll
        for (int b = 0; b < 8; ++b) bv[b] = Bs[k * kTld + tx + 16 * b];
#pragma unroll
        for (int a = 0; a < 8; ++a)
#pragma unroll
            for (int b = 0; b < 8; ++b) acc[a][b] = fmaf(av[a], bv[b], acc[a][b]);
    }
}

// S[k][i] = src(row i, column k0 + k) for i < 128, k < kTk, from rows contiguous along k (row pointer rp(i), or nullptr
// for a row outside the operand); columns at or past kn read as 0.  kn and k0 are multiples of 4.
template <class RowPtr>
__device__ __forceinline__ void stage_rows_t(float* S, RowPtr rp, int k0, int kn) {
    for (int e = threadIdx.x; e < kTile * (kTk / 4); e += blockDim.x) {
        const int i = e >> 2, q = e & 3, k = k0 + 4 * q;
        const float* p = rp(i);
        const float4 v = (p != nullptr && k < kn) ? ldg4(p + k) : f4(0.f);
        S[(4 * q) * kTld + i] = v.x; S[(4 * q + 1) * kTld + i] = v.y;
        S[(4 * q + 2) * kTld + i] = v.z; S[(4 * q + 3) * kTld + i] = v.w;
    }
}

// S[k][i] = src(row k, column i) for k < kTk, i < 128, from rows contiguous along i (row pointer rp(k), or nullptr);
// columns at or past cn read as 0.  cn is a multiple of 4.
template <class RowPtr>
__device__ __forceinline__ void stage_rows_n(float* S, RowPtr rp, int cn) {
    for (int e = threadIdx.x; e < kTk * (kTile / 4); e += blockDim.x) {
        const int k = e >> 5, i = 4 * (e & 31);
        const float* p = rp(k);
        const float4 v = (p != nullptr && i < cn) ? ldg4(p + i) : f4(0.f);
        *reinterpret_cast<float4*>(S + k * kTld + i) = v;
    }
}

__device__ __forceinline__ void zero_acc(float (&acc)[8][8]) {
#pragma unroll
    for (int a = 0; a < 8; ++a)
#pragma unroll
        for (int b = 0; b < 8; ++b) acc[a][b] = 0.f;
}

// logits of the sampled classes: tile (bt, st) of [n × S]; G = σ(logit) for the backward, Σ_b G into entity_b's gradient
template <class H>
__global__ void __launch_bounds__(kThreads)
k_nce_logits(ProjeDev T, int n, const float* __restrict__ x, const int32_t* __restrict__ sampled,
             const float* __restrict__ lqs, float* __restrict__ G, double* __restrict__ loss_out, H h) {
    __shared__ __align__(16) float As[kTk * kTld];
    __shared__ __align__(16) float Bs[kTk * kTld];
    __shared__ float s_db[kTile];
    __shared__ double s_loss[kWarpsPerBlock];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int S = T.num_sampled;
    const int mt = (n + kTile - 1) / kTile, nt = (T.ldg + kTile - 1) / kTile;
    float lsum = 0.f;
    for (int t = blockIdx.x; t < mt * nt; t += gridDim.x) {
        const int m0 = (t % mt) * kTile, n0 = (t / mt) * kTile;
        float acc[8][8];
        zero_acc(acc);
        for (int k0 = 0; k0 < T.pitch; k0 += kTk) {
            __syncthreads();
            stage_rows_t(As, [&](int i) { return m0 + i < n ? x + (size_t)(m0 + i) * T.pitch : nullptr; }, k0, T.pitch);
            stage_rows_t(Bs, [&](int i) { return n0 + i < S ? h.w_row(T, sampled + n0 + i, n0 + i) : nullptr; }, k0, T.pitch);
            __syncthreads();
            tile_mma(acc, As, Bs, ty, tx);
        }
        if (threadIdx.x < kTile) s_db[threadIdx.x] = 0.f;
        __syncthreads();
#pragma unroll
        for (int b = 0; b < 8; ++b) {
            const int s = n0 + tx + 16 * b;
            float bias = 0.f, lq = 0.f;
            if (s < S) {
                const int c = __ldg(sampled + s);
                bias = T.b.w[(size_t)c * T.b.pitch];
                lq = __ldg(lqs + s);
            }
            float col = 0.f;
#pragma unroll
            for (int a = 0; a < 8; ++a) {
                const int m = m0 + ty + 16 * a;
                if (m >= n || s >= T.ldg) continue;
                float g = 0.f;
                if (s < S) {
                    const float logit = acc[a][b] + bias - lq;
                    lsum += softplus(logit);
                    g = h.scaled(sigmoid_acc(logit));
                    col += g;
                }
                G[(size_t)m * T.ldg + s] = g;
            }
            if (s < S) atomicAdd(s_db + tx + 16 * b, col);
        }
        __syncthreads();
        if (threadIdx.x < kTile && n0 + (int)threadIdx.x < S) {
            const int c = __ldg(sampled + n0 + threadIdx.x);
            atomicAdd(T.b.g + (size_t)c * T.b.pitch, s_db[threadIdx.x]);
            if (m0 == 0) { T.b.touched[c] = 1; T.w.touched[c] = 1; }
        }
    }
    LossAcc lacc{s_loss};
    lacc.flush(h.scaled(warp_sum(lsum)), loss_out);
}

// dX[b][:] += Σ_{s in split} G[b][s]·W_S[s][:]; tile t = (b tile, split of the sampled set)
template <class H>
__global__ void __launch_bounds__(kThreads)
k_nce_dx(ProjeDev T, int n, const float* __restrict__ G, const int32_t* __restrict__ sampled, int split,
         float* __restrict__ dx, H h) {
    __shared__ __align__(16) float As[kTk * kTld];
    __shared__ __align__(16) float Bs[kTk * kTld];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int S = T.num_sampled;
    const int mt = (n + kTile - 1) / kTile, st = (S + split - 1) / split;
    for (int t = blockIdx.x; t < mt * st; t += gridDim.x) {
        const int m0 = (t % mt) * kTile, s0 = (t / mt) * split, s1 = min(S, s0 + split);
        float acc[8][8];
        zero_acc(acc);
        for (int k0 = s0; k0 < s1; k0 += kTk) {
            __syncthreads();
            // A(b, s) = G[b][s]: rows along s.  A split ends on a multiple of kTk or at S, and G's columns S … ldg − 1
            // are zero, so the slice needs no clipping inside a float4
            stage_rows_t(As, [&](int i) { return m0 + i < n ? G + (size_t)(m0 + i) * T.ldg : nullptr; }, k0,
                         (s1 + 3) / 4 * 4);
            stage_rows_n(Bs, [&](int k) { return k0 + k < s1 ? h.w_row(T, sampled + k0 + k, k0 + k) : nullptr; }, T.pitch);
            __syncthreads();
            tile_mma(acc, As, Bs, ty, tx);
        }
#pragma unroll
        for (int a = 0; a < 8; ++a) {
            const int m = m0 + ty + 16 * a;
            if (m >= n) continue;
#pragma unroll
            for (int b = 0; b < 8; ++b) {
                const int c = tx + 16 * b;
                if (c < T.dim) atomicAdd(dx + (size_t)m * T.pitch + c, acc[a][b]);
            }
        }
    }
}

// dW_S[s][:] += Σ_{b in split} G[b][s]·X[b][:]; tile t = (sampled tile, split of the batch)
template <class H>
__global__ void __launch_bounds__(kThreads)
k_nce_dw(ProjeDev T, int n, const float* __restrict__ G, const float* __restrict__ x, const int32_t* __restrict__ sampled,
         int split, H h) {
    __shared__ __align__(16) float As[kTk * kTld];
    __shared__ __align__(16) float Bs[kTk * kTld];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int S = T.num_sampled;
    const int mt = (S + kTile - 1) / kTile, bt = (n + split - 1) / split;
    for (int t = blockIdx.x; t < mt * bt; t += gridDim.x) {
        const int m0 = (t % mt) * kTile, b0 = (t / mt) * split, b1 = min(n, b0 + split);
        float acc[8][8];
        zero_acc(acc);
        for (int k0 = b0; k0 < b1; k0 += kTk) {
            __syncthreads();
            // A(s, b) = G[b][s]: G's rows run along s, so the slice is staged without a transpose
            stage_rows_n(As, [&](int k) { return k0 + k < b1 ? G + (size_t)(k0 + k) * T.ldg + m0 : nullptr; },
                         min(kTile, T.ldg - m0));
            stage_rows_n(Bs, [&](int k) { return k0 + k < b1 ? x + (size_t)(k0 + k) * T.pitch : nullptr; }, T.pitch);
            __syncthreads();
            tile_mma(acc, As, Bs, ty, tx);
        }
        // rows of 128 floats in registers are 8 strided columns per thread: go through shared memory for float4 reds
        __syncthreads();
        float* Cs = As;                                   // 16 rows at a time
#pragma unroll
        for (int a = 0; a < 8; ++a) {
#pragma unroll
            for (int b = 0; b < 8; ++b) Cs[ty * kTld + tx + 16 * b] = acc[a][b];
            __syncthreads();
            for (int e = threadIdx.x; e < 16 * (kTile / 4); e += blockDim.x) {
                const int r = e >> 5, c = 4 * (e & 31), s = m0 + r + 16 * a;
                if (s < S && c < T.pitch)
                    red_add4(h.dw_row(T, sampled + s, s) + c, *reinterpret_cast<const float4*>(Cs + r * kTld + c));
            }
            __syncthreads();
        }
    }
}

// ---- the general sampled-NCE step (oea_nce_score_fed) ---------------------------------------------------------------
struct NceWs {
    size_t first, x, dx, w, dw, winv, wss, lq, g, total;
    int ldg;
};

// workspace sections: the sampler's first-draw index per class, x̂ and dX̂ [n, pitch], ŵ_S and dŴ_S [S, pitch],
// 1/‖w_s‖ and Σw_s² [S], log q [S], G [n, ldg]
static NceWs nce_layout(int n, int num_sampled, int pitch, int n_classes) {
    NceWs w;
    WsCarver c;
    w.ldg = round4(num_sampled);
    w.first = c.take(4 * (size_t)n_classes);
    w.x = c.take(4 * (size_t)n * pitch);
    w.dx = c.take(4 * (size_t)n * pitch);
    w.w = c.take(4 * (size_t)num_sampled * pitch);
    w.dw = c.take(4 * (size_t)num_sampled * pitch);
    w.winv = c.take(4 * (size_t)num_sampled);
    w.wss = c.take(4 * (size_t)num_sampled);
    w.lq = c.take(4 * (size_t)num_sampled);
    w.g = c.take(4 * (size_t)n * w.ldg);
    w.total = c.at;
    return w;
}

__global__ void __launch_bounds__(kThreads)
k_nce_stage(ProjeDev T, const int32_t* __restrict__ sampled, float* __restrict__ ws_w, float* __restrict__ ws_dw,
            float* __restrict__ winv, float* __restrict__ wss) {
    const int lane = threadIdx.x & 31;
    for (int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; s < T.num_sampled; s += (gridDim.x * blockDim.x) >> 5) {
        const NRow<1> w = lookup<1>(T.w, __ldg(sampled + s), lane);
        if (4 * lane < T.pitch) {
            *reinterpret_cast<float4*>(ws_w + (size_t)s * T.pitch + 4 * lane) = w.x.v[0];
            *reinterpret_cast<float4*>(ws_dw + (size_t)s * T.pitch + 4 * lane) = f4(0.f);
        }
        if (lane == 0) { winv[s] = w.inv; wss[s] = w.ss; }
    }
}

__global__ void __launch_bounds__(kThreads)
k_nce_gather(ProjeDev T, const int32_t* __restrict__ ids, int n, float* __restrict__ x) {
    const int lane = threadIdx.x & 31;
    for (int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < n; b += (gridDim.x * blockDim.x) >> 5) {
        const Row<1> v = lookup<1>(T.ent, __ldg(ids + b), lane).x;
        if (4 * lane < T.pitch) *reinterpret_cast<float4*>(x + (size_t)b * T.pitch + 4 * lane) = v.v[0];
    }
}

// the true class of every row: ŵ_label normalised here, the logit, the loss, dX, and the label row's part of its
// gradient through the normalisation.  ProjE and ConvE run it at scale 1 over their raw entity_w, where lookup and push
// scale by exactly 1.
__global__ void __launch_bounds__(kThreads)
k_nce_true(ProjeDev T, const int32_t* __restrict__ labels, int n, const float* __restrict__ x,
           const int32_t* __restrict__ num_tries, float scale, float* __restrict__ dx, double* __restrict__ loss_out) {
    __shared__ double s_loss[kWarpsPerBlock];
    const int lane = threadIdx.x & 31;
    const int tries = *num_tries;
    float lsum = 0.f;
    for (int b0 = (blockIdx.x * blockDim.x) >> 5; b0 < n; b0 += (gridDim.x * blockDim.x) >> 5) {   // warp-uniform
        const int b = b0 + (threadIdx.x >> 5);
        if (b >= n) continue;
        const int c = __ldg(labels + b);
        const Row<1> xb = load_row<1>(x, b, T.pitch, lane);
        const NRow<1> wc = lookup<1>(T.w, c, lane);
        const float logit = warp_sum(dotr(xb, wc.x)) + T.b.w[(size_t)c * T.b.pitch] -
                            log_expected_count(c, T.n_classes, T.num_sampled, tries);
        const float g = -sigmoid_acc(-logit) * scale;     // scale·(σ(t) − 1)
        if (lane == 0) {
            lsum += softplus(-logit);
            atomicAdd(T.b.g + (size_t)c * T.b.pitch, g);
            T.b.touched[c] = 1;
        }
        if (4 * lane < T.pitch) {
            float4* d = reinterpret_cast<float4*>(dx + (size_t)b * T.pitch + 4 * lane);
            *d = fma4(wc.x.v[0], g, *d);
        }
        push<1>(T.w, c, lane, r_scale(xb, g), wc);
    }
    LossAcc lacc{s_loss};
    lacc.flush(warp_sum(lsum) * scale, loss_out);
}

__global__ void __launch_bounds__(kThreads)
k_nce_w_push(ProjeDev T, const int32_t* __restrict__ sampled, const float* __restrict__ ws_w,
             const float* __restrict__ ws_dw, const float* __restrict__ winv, const float* __restrict__ wss) {
    const int lane = threadIdx.x & 31;
    for (int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; s < T.num_sampled; s += (gridDim.x * blockDim.x) >> 5) {
        NRow<1> w;
        w.x = load_row<1>(ws_w, s, T.pitch, lane);
        w.inv = winv[s];
        w.ss = wss[s];
        push<1>(T.w, __ldg(sampled + s), lane, load_row<1>(ws_dw, s, T.pitch, lane), w);
    }
}

__global__ void __launch_bounds__(kThreads)
k_nce_in_push(ProjeDev T, const int32_t* __restrict__ ids, int n, const float* __restrict__ dx) {
    const int lane = threadIdx.x & 31;
    for (int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < n; b += (gridDim.x * blockDim.x) >> 5) {
        const int i = __ldg(ids + b);
        push<1>(T.ent, i, lane, load_row<1>(dx, b, T.pitch, lane), lookup<1>(T.ent, i, lane));
    }
}

// ---- the per-step pair draw (oea_pairs_draw) ------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint64_t pairs_key(uint64_t seed, int epoch, int step) {
    return mix64(seed ^ mix64(((uint64_t)(uint32_t)epoch << 32) | (uint32_t)step));
}

__global__ void __launch_bounds__(kThreads)
k_pairs_draw(const int32_t* __restrict__ pairs, uint32_t n, int batch, uint64_t key, int32_t* __restrict__ first,
             int32_t* __restrict__ second) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < batch; i += gridDim.x * blockDim.x) {
        const size_t row = feistel_perm((uint32_t)i, n, key);
        first[i] = __ldg(pairs + 2 * row);
        second[i] = __ldg(pairs + 2 * row + 1);
    }
}

// grids of the head's kernels for a batch of n and S sampled classes.  ConvE's dense layer takes its own for (n, 2Fd,
// lda): its forward and dW run on k_nce_dx and k_nce_dw, and its dA kernel tiles [n, lda] as the logits tile [n, ldg].
struct HeadGrids {
    int rows, lg, dx, dw, split_s, split_b;
};

// `len` cut into about `parts` pieces, each a multiple of kTk
static int split_of(int len, int parts) { const int s = (len + parts - 1) / parts; return (s + kTk - 1) / kTk * kTk; }

static HeadGrids head_grids(int n, int S, int ldg) {
    HeadGrids h;
#ifdef OEA_HOST_EMU   // tests/emu: grid-stride kernels on two blocks keep the emulated thread count small
    h.rows = h.lg = h.dx = h.dw = 2;
    h.split_s = h.split_b = 2 * kTk;                      // several splits even on small cases
#else
    const int mt_b = (n + kTile - 1) / kTile, mt_s = (S + kTile - 1) / kTile;
    h.rows = grid_for(n);
    h.lg = mt_b * ((ldg + kTile - 1) / kTile);
    // split each reduction so that about two CTAs per SM run: a batch of 500 is only four row tiles, and S = 4096
    // only 32 column tiles
    const int want = 2 * sm_count_cached();
    h.split_s = split_of(S, (want + mt_b - 1) / mt_b);
    h.split_b = split_of(n, (want + mt_s - 1) / mt_s);
    h.dx = mt_b * ((S + h.split_s - 1) / h.split_s);
    h.dw = mt_s * ((n + h.split_b - 1) / h.split_b);
#endif
    return h;
}

// ---- ConvE's tower (oea_conve_score_fed) ----------------------------------------------------------------------------
// An inference-mode batch norm at its initial moving moments (mean 0, variance 1) scales by γ/√(1 + ε) and shifts by β.
constexpr float kBnInfer = 0.99950037468777f;     // 1/√(1 + 1e-3)
constexpr int kConvCols = 12;                      // conv table row f: 9 taps (dy·3 + dx), bias, γ₂, β₂

struct ConveDev {
    TableDev conv, bn_in, fc_w, fc_out;            // [F, 12]; [2, y] γ₁, β₁; [2Fd, d]; [3, d] bias, γ₃, β₃
    int x, y, F, K, lda;                           // image rows per vector, columns; filters; 2Fd and A's row stride
    float keep;
    uint64_t seed;
};

// tf.nn.dropout's mask as a pure function of (seed, site, flat index): element i of site s is kept iff
// u = (pcg32(key_s ^ i) >> 8)·2⁻²⁴ < keep, key_s = pcg32(lo(seed) ^ pcg32(hi(seed) + s·0x9E3779B9)).  keep = 1 keeps all.
__host__ __device__ __forceinline__ uint32_t dropout_key(uint64_t seed, uint32_t site) {
    return pcg32((uint32_t)seed ^ pcg32((uint32_t)(seed >> 32) + site * 0x9E3779B9u));
}
__host__ __device__ __forceinline__ bool dropout_kept(uint32_t key, uint32_t i, float keep) {
    return (float)(pcg32(key ^ i) >> 8) * 0x1.0p-24f < keep;
}

// one CTA per positive: ê[h], r̂[r] stacked into the [2x, y] image, the input BN (per column) and dropout into img
// [n, 2d]; the 3×3 'same' cross-correlation, the per-filter BN, ReLU and dropout into A [n, lda] (index f·2d + i·y + j)
__global__ void __launch_bounds__(kThreads)
k_conve_conv_fwd(ProjeDev T, ConveDev C, const int32_t* __restrict__ ph, const int32_t* __restrict__ pr, int n,
                 float* __restrict__ img, float* __restrict__ A) {
    __shared__ __align__(16) float s_raw[2][kProjeMaxPitch];
    __shared__ float s_img[2 * kProjeMaxPitch];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int d = T.dim, D2 = 2 * d, y = C.y, H = 2 * C.x;
    const uint32_t key0 = dropout_key(C.seed, 0), key1 = dropout_key(C.seed, 1);
    for (int b = blockIdx.x; b < n; b += gridDim.x) {
        if (warp < 2) {
            const Row<1> v = lookup<1>(pick_table(warp == 0, T.ent, T.rel), __ldg((warp == 0 ? ph : pr) + b), lane).x;
            if (4 * lane < T.pitch) *reinterpret_cast<float4*>(&s_raw[warp][4 * lane]) = v.v[0];
        }
        __syncthreads();
        for (int e = threadIdx.x; e < D2; e += blockDim.x) {
            const int j = e % y, half = e >= d;
            const float u = fmaf(s_raw[half][e - half * d], C.bn_in.w[j] * kBnInfer, C.bn_in.w[C.bn_in.pitch + j]);
            const float v = dropout_kept(key0, (uint32_t)(b * D2 + e), C.keep) ? u / C.keep : 0.f;
            s_img[e] = v;
            img[(size_t)b * D2 + e] = v;
        }
        __syncthreads();
        for (int o = threadIdx.x; o < C.lda; o += blockDim.x) {
            float v = 0.f;
            if (o < C.K) {
                const int f = o / D2, pos = o - f * D2, i = pos / y, j = pos - i * y;
                const float* k = C.conv.w + (size_t)f * C.conv.pitch;
                float q = k[9];
#pragma unroll
                for (int dy = 0; dy < 3; ++dy) {
                    const int ii = i + dy - 1;
                    if (ii < 0 || ii >= H) continue;
#pragma unroll
                    for (int dx = 0; dx < 3; ++dx) {
                        const int jj = j + dx - 1;
                        if (jj >= 0 && jj < y) q = fmaf(k[3 * dy + dx], s_img[ii * y + jj], q);
                    }
                }
                const float p = fmaf(q, k[10] * kBnInfer, k[11]);
                if (p > 0.f && dropout_kept(key1, (uint32_t)b * (uint32_t)C.K + (uint32_t)o, C.keep)) v = p / C.keep;
            }
            A[(size_t)b * C.lda + o] = v;                 // columns K … lda − 1 stay zero for the GEMMs' float4 loads
        }
        __syncthreads();
    }
}

// the dense layer's bias and ReLU and the output BN: z += bias (kept for the backward), X = γ₃·relu(z)/√(1+ε) + β₃
__global__ void __launch_bounds__(kThreads)
k_conve_fc_out(ProjeDev T, ConveDev C, int n, float* __restrict__ z, float* __restrict__ x) {
    const int P = T.pitch;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)n * P; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % P);
        if (c >= T.dim) { x[i] = 0.f; continue; }           // padding columns of X stay zero for the head's float4 loads
        const float v = z[i] + C.fc_out.w[c];
        z[i] = v;
        x[i] = fmaf(v > 0.f ? v : 0.f, C.fc_out.w[P + c] * kBnInfer, C.fc_out.w[2 * P + c]);
    }
}

// back through the output BN and the dense ReLU: dX → dz in place; the column sums are the gradients of the dense bias,
// γ₃ and β₃.  Thread column c = threadIdx.x % 128, two rows per block step.  Flags every row of the tower's tables.
__global__ void __launch_bounds__(kThreads)
k_conve_fc_out_bwd(ProjeDev T, ConveDev C, int n, const float* __restrict__ z, float* __restrict__ dx) {
    __shared__ float s_sum[3][kThreads];
    const int P = T.pitch, c = threadIdx.x & (kProjeMaxPitch - 1), r0 = threadIdx.x / kProjeMaxPitch;
    float sb = 0.f, sg = 0.f, sbeta = 0.f;
    if (c < P) {
        const float g3 = c < T.dim ? C.fc_out.w[P + c] * kBnInfer : 0.f;
        for (int b = 2 * blockIdx.x + r0; b < n; b += 2 * gridDim.x) {
            const size_t i = (size_t)b * P + c;
            const float g = dx[i], v = z[i];
            const float dz = v > 0.f ? g * g3 : 0.f;
            dx[i] = dz;
            sb += dz;
            sg = fmaf(g, (v > 0.f ? v : 0.f) * kBnInfer, sg);
            sbeta += g;
        }
    }
    s_sum[0][threadIdx.x] = sb; s_sum[1][threadIdx.x] = sg; s_sum[2][threadIdx.x] = sbeta;
    __syncthreads();
    if (threadIdx.x < kProjeMaxPitch && c < T.dim)
        for (int r = 0; r < 3; ++r)
            atomicAdd(C.fc_out.g + (size_t)r * P + c, s_sum[r][c] + s_sum[r][c + kProjeMaxPitch]);
    const int gt = blockIdx.x * blockDim.x + threadIdx.x, gs = gridDim.x * blockDim.x;
    for (int r = gt; r < C.K; r += gs) C.fc_w.touched[r] = 1;
    for (int r = gt; r < C.F; r += gs) C.conv.touched[r] = 1;
    if (gt < 2) C.bn_in.touched[gt] = 1;
    if (gt < 3) C.fc_out.touched[gt] = 1;
}

// dA = dz·Wᵀ, taken back through the conv ReLU and dropout in the epilogue and written over A: the ReLU was active and
// the element kept iff A > 0, where dp = dA/keep.  Tile t = (batch tile, input tile).
__global__ void __launch_bounds__(kThreads)
k_conve_fc_dx(ProjeDev T, ConveDev C, int n, const float* __restrict__ dz, float* A) {
    __shared__ __align__(16) float As[kTk * kTld];
    __shared__ __align__(16) float Bs[kTk * kTld];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int mt = (n + kTile - 1) / kTile, nt = (C.lda + kTile - 1) / kTile;
    for (int t = blockIdx.x; t < mt * nt; t += gridDim.x) {
        const int m0 = (t % mt) * kTile, n0 = (t / mt) * kTile;
        float acc[8][8];
        zero_acc(acc);
        for (int k0 = 0; k0 < T.pitch; k0 += kTk) {
            __syncthreads();
            stage_rows_t(As, [&](int i) { return m0 + i < n ? dz + (size_t)(m0 + i) * T.pitch : nullptr; }, k0, T.pitch);
            stage_rows_t(Bs, [&](int i) { return n0 + i < C.K ? C.fc_w.w + (size_t)(n0 + i) * T.pitch : nullptr; }, k0,
                         T.pitch);
            __syncthreads();
            tile_mma(acc, As, Bs, ty, tx);
        }
#pragma unroll
        for (int a = 0; a < 8; ++a) {
            const int m = m0 + ty + 16 * a;
            if (m >= n) continue;
#pragma unroll
            for (int b = 0; b < 8; ++b) {
                const int k = n0 + tx + 16 * b;
                if (k >= C.lda) continue;
                float* p = A + (size_t)m * C.lda + k;
                *p = *p > 0.f ? acc[a][b] / C.keep : 0.f;
            }
        }
    }
}

// the gradients of filter f's taps, bias, γ₂ and β₂ over one split of the batch: tile t = (filter, batch split).
// The conv output q is recomputed from img (nine FMAs) rather than stored: it is needed only for γ₂.
__global__ void __launch_bounds__(kThreads)
k_conve_conv_dw(ProjeDev T, ConveDev C, int n, const float* __restrict__ img, const float* __restrict__ dp, int split) {
    __shared__ float s_red[kWarpsPerBlock][kConvCols];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int D2 = 2 * T.dim, y = C.y, H = 2 * C.x;
    const int bt = (n + split - 1) / split;
    for (int t = blockIdx.x; t < C.F * bt; t += gridDim.x) {
        const int f = t % C.F, b0 = (t / C.F) * split, b1 = min(n, b0 + split);
        const float* k = C.conv.w + (size_t)f * C.conv.pitch;
        const float s2 = k[10] * kBnInfer;
        float acc[kConvCols];
#pragma unroll
        for (int r = 0; r < kConvCols; ++r) acc[r] = 0.f;
        for (int e = threadIdx.x; e < (b1 - b0) * D2; e += blockDim.x) {
            const int b = b0 + e / D2, pos = e % D2, i = pos / y, j = pos - i * y;
            const float g = dp[(size_t)b * C.lda + f * D2 + pos];
            if (g == 0.f) continue;                       // dropped or ReLU inactive: no contribution
            const float* im = img + (size_t)b * D2;
            float nb[9];
            float q = k[9];
#pragma unroll
            for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) {
                    const int ii = i + dy - 1, jj = j + dx - 1;
                    nb[3 * dy + dx] = (ii >= 0 && ii < H && jj >= 0 && jj < y) ? im[ii * y + jj] : 0.f;
                    q = fmaf(k[3 * dy + dx], nb[3 * dy + dx], q);
                }
            const float dq = g * s2;
#pragma unroll
            for (int r = 0; r < 9; ++r) acc[r] = fmaf(dq, nb[r], acc[r]);
            acc[9] += dq;
            acc[10] = fmaf(g, q * kBnInfer, acc[10]);
            acc[11] += g;
        }
#pragma unroll
        for (int r = 0; r < kConvCols; ++r) {
            const float v = warp_sum(acc[r]);
            if (lane == 0) s_red[warp][r] = v;
        }
        __syncthreads();
        if (threadIdx.x < kConvCols) {
            float s = 0.f;
            for (int w = 0; w < kWarpsPerBlock; ++w) s += s_red[w][threadIdx.x];
            atomicAdd(C.conv.g + (size_t)f * C.conv.pitch + threadIdx.x, s);
        }
        __syncthreads();
    }
}

// one CTA per positive: the transposed convolution of dq = dp·γ₂/√(1+ε) back to the image, through the dropout and the
// input BN (γ₁, β₁ column sums), and dê, dr̂ through the tables' normalisation into ent.grad, rel.grad
__global__ void __launch_bounds__(kThreads)
k_conve_conv_dx(ProjeDev T, ConveDev C, const int32_t* __restrict__ ph, const int32_t* __restrict__ pr, int n,
                const float* __restrict__ dp) {
    __shared__ __align__(16) float s_v[2][kProjeMaxPitch];
    __shared__ __align__(16) float s_dv[2][kProjeMaxPitch];
    __shared__ float s_g1[kProjeMaxPitch], s_b1[kProjeMaxPitch];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int d = T.dim, D2 = 2 * d, y = C.y, H = 2 * C.x;
    const uint32_t key0 = dropout_key(C.seed, 0);
    for (int i = threadIdx.x; i < kProjeMaxPitch; i += blockDim.x) {
        s_g1[i] = s_b1[i] = 0.f;
        s_dv[0][i] = s_dv[1][i] = 0.f;                    // columns d … pitch − 1 are pushed as zeros
    }
    for (int b = blockIdx.x; b < n; b += gridDim.x) {
        NRow<1> nr;
        int id = 0;
        if (warp < 2) {
            id = __ldg((warp == 0 ? ph : pr) + b);
            nr = lookup<1>(pick_table(warp == 0, T.ent, T.rel), id, lane);
            if (4 * lane < T.pitch) *reinterpret_cast<float4*>(&s_v[warp][4 * lane]) = nr.x.v[0];
        }
        __syncthreads();
        const float* g = dp + (size_t)b * C.lda;
        for (int e = threadIdx.x; e < D2; e += blockDim.x) {
            const int i = e / y, j = e - i * y, half = e >= d;
            float du = 0.f;
            for (int f = 0; f < C.F; ++f) {
                const float* k = C.conv.w + (size_t)f * C.conv.pitch;
                const float* gf = g + f * D2;
                float s = 0.f;
#pragma unroll
                for (int dy = 0; dy < 3; ++dy) {
                    const int ii = i - dy + 1;                // the output row whose tap dy reads image row i
                    if (ii < 0 || ii >= H) continue;
#pragma unroll
                    for (int dx = 0; dx < 3; ++dx) {
                        const int jj = j - dx + 1;
                        if (jj >= 0 && jj < y) s = fmaf(k[3 * dy + dx], __ldg(gf + ii * y + jj), s);
                    }
                }
                du = fmaf(s, k[10] * kBnInfer, du);
            }
            du = dropout_kept(key0, (uint32_t)(b * D2 + e), C.keep) ? du / C.keep : 0.f;
            atomicAdd(s_g1 + j, du * s_v[half][e - half * d] * kBnInfer);
            atomicAdd(s_b1 + j, du);
            s_dv[half][e - half * d] = du * C.bn_in.w[j] * kBnInfer;
        }
        __syncthreads();
        if (warp < 2) {
            Row<1> gr;
            gr.v[0] = 4 * lane < kProjeMaxPitch ? *reinterpret_cast<const float4*>(&s_dv[warp][4 * lane]) : f4(0.f);
            push<1>(pick_table(warp == 0, T.ent, T.rel), id, lane, gr, nr);
        }
        __syncthreads();
    }
    for (int j = threadIdx.x; j < y; j += blockDim.x) {
        atomicAdd(C.bn_in.g + j, s_g1[j]);
        atomicAdd(C.bn_in.g + C.bn_in.pitch + j, s_b1[j]);
    }
}

// dim_factorization of models/neural/conve.py:10-18: x = the largest divisor of d not above ⌊√d⌋ + 1, y = d / x
static void conve_factor(int d, int* x, int* y) {
    int half = (int)sqrt((double)d) + 1;
    while (d % half > 0) --half;
    *x = half;
    *y = d / half;
}

struct ConveWs {
    size_t first, img, a, z, x, dx, lq, g, total;
    int ldg, lda;
};

// workspace sections: the sampler's first-draw index per class, the dropped image [n, 2d], the dense layer's input
// A [n, lda] (its gradient dp overwrites it in the backward), z, X and dX [n, pitch], log q [S], G [n, ldg]
static ConveWs conve_layout(int n, int num_sampled, int dim, int pitch, int filters, int n_classes) {
    ConveWs w;
    WsCarver c;
    const size_t row = 4 * (size_t)n * pitch;
    w.ldg = round4(num_sampled);
    w.lda = round4(2 * filters * dim);
    w.first = c.take(4 * (size_t)n_classes);
    w.img = c.take(4 * (size_t)n * 2 * dim);
    w.a = c.take(4 * (size_t)n * w.lda);
    w.z = c.take(row);
    w.x = c.take(row);
    w.dx = c.take(row);
    w.lq = c.take(4 * (size_t)num_sampled);
    w.g = c.take(4 * (size_t)n * w.ldg);
    w.total = c.at;
    return w;
}

// The argument checks all three sampled-NCE steps make once their tables have passed their own: cls_b is [C, 1] for
// the C rows of cls_w, 1 ≤ num_sampled ≤ C, n ≥ 0, the sampled set, num_tries and loss_out are given, and so are the
// batch's id arrays when n > 0 (`ids_given`); last the workspace, against the size `layout()` computes from the checked
// shapes.  OEA_OK or the first error; the caller returns early on either, and when n == 0.
template <class Layout>
static int check_head(const oea_table* w, const oea_table* b, int num_sampled, int n, const int32_t* sampled,
                      const int32_t* num_tries, const double* loss_out, bool ids_given, const void* workspace,
                      size_t workspace_bytes, Layout layout) {
    if (b->rows != w->rows || b->dim != 1) return OEA_ERR_SHAPE;
    if (num_sampled < 1 || num_sampled > w->rows) return OEA_ERR_RANGE;
    if (n < 0) return OEA_ERR_SHAPE;
    if (sampled == nullptr || num_tries == nullptr || loss_out == nullptr) return OEA_ERR_NULL;
    if (n > 0 && !ids_given) return OEA_ERR_NULL;
    if (workspace == nullptr || workspace_bytes < layout() || !aligned16(workspace)) return OEA_ERR_WORKSPACE;
    return OEA_OK;
}

}  // namespace oea

using namespace oea;

extern "C" size_t oea_proje_workspace_bytes(int32_t n_pos, int32_t num_sampled, int32_t dim, int32_t n_classes) {
    if (n_pos < 0 || num_sampled < 1 || dim <= 0 || n_classes <= 0) return 0;
    return proje_layout(n_pos, num_sampled, round4(dim), n_classes).total;
}

extern "C" int oea_logu_sample_unique(int32_t range_max, int32_t num_sampled, uint64_t seed, int32_t* sampled,
                                      int32_t* num_tries, void* workspace, size_t workspace_bytes, void* stream) {
    if (range_max < 1 || num_sampled < 1 || num_sampled > range_max) return OEA_ERR_RANGE;
    if (sampled == nullptr || num_tries == nullptr) return OEA_ERR_NULL;
    if (workspace == nullptr || workspace_bytes < 4 * (size_t)range_max || !aligned16(workspace)) return OEA_ERR_WORKSPACE;
    OEA_LAUNCH(k_logu_sample, 1, kThreads, 0, (cudaStream_t)stream, range_max, num_sampled, seed,
               static_cast<int32_t*>(workspace), sampled, num_tries);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_proje_score_fed(const oea_proje* model, const int32_t* pos_h, const int32_t* pos_r,
                                   const int32_t* pos_t, int32_t n_pos, const int32_t* sampled, const int32_t* num_tries,
                                   int32_t num_sampled, void* workspace, size_t workspace_bytes, double* loss_out,
                                   void* stream) {
    if (model == nullptr) return OEA_ERR_NULL;
    const oea_table* tabs[5] = {model->ent, model->rel, model->cls_w, model->cls_b, model->params};
    for (const oea_table* t : tabs) {
        const int rc = check_table(t, true);
        if (rc) return rc;
    }
    const oea_table *ent = model->ent, *rel = model->rel, *w = model->cls_w, *b = model->cls_b, *prm = model->params;
    if (rel->dim != ent->dim || w->dim != ent->dim || rel->pitch != ent->pitch || w->pitch != ent->pitch ||
        prm->pitch != ent->pitch || ent->pitch > kProjeMaxPitch)
        return OEA_ERR_DIM;
    if (prm->rows != 4 || prm->dim != ent->dim) return OEA_ERR_SHAPE;
    ProjeWs L{};
    const int rc = check_head(w, b, num_sampled, n_pos, sampled, num_tries, loss_out, pos_h && pos_r && pos_t,
                              workspace, workspace_bytes,
                              [&] { return (L = proje_layout(n_pos, num_sampled, ent->pitch, w->rows)).total; });
    if (rc != OEA_OK || n_pos == 0) return rc;

    char* ws = static_cast<char*>(workspace);
    float* xh = reinterpret_cast<float*>(ws + L.xh);
    float* xr = reinterpret_cast<float*>(ws + L.xr);
    float* z = reinterpret_cast<float*>(ws + L.z);
    float* x = reinterpret_cast<float*>(ws + L.x);
    float* dx = reinterpret_cast<float*>(ws + L.dx);
    float* dxh = reinterpret_cast<float*>(ws + L.dxh);
    float* dxr = reinterpret_cast<float*>(ws + L.dxr);
    float* stats = reinterpret_cast<float*>(ws + L.stats);
    float* lq = reinterpret_cast<float*>(ws + L.lq);
    float* G = reinterpret_cast<float*>(ws + L.g);
    ProjeDev T;
    T.ent = table_dev(ent); T.rel = table_dev(rel); T.w = table_dev(w); T.b = table_dev(b); T.prm = table_dev(prm);
    T.w.norm = T.b.norm = T.prm.norm = false;             // entity_w, entity_b and the MLP / BN variables: raw
    T.dim = ent->dim; T.pitch = ent->pitch; T.n_classes = w->rows; T.num_sampled = num_sampled; T.ldg = L.ldg;
    cudaStream_t st = (cudaStream_t)stream;
    const int n = n_pos, S = num_sampled;
    const HeadGrids H = head_grids(n, S, L.ldg);
    const int rows_grid = H.rows;
#ifdef OEA_HOST_EMU
    const int col_grid = 2;
#else
    const int col_grid = ent->pitch;
#endif
    OEA_CUDA_TRY(cudaMemsetAsync(dx, 0, 4 * (size_t)n * ent->pitch, st));
    OEA_LAUNCH(k_proje_gather, rows_grid, kThreads, 0, st, T, pos_h, pos_r, n, xh, xr);
    OEA_LAUNCH(k_proje_columns_fwd, col_grid, kThreads, 0, st, T, n, xh, xr, z, x, stats);
    OEA_LAUNCH(k_nce_logq, rows_grid, kThreads, 0, st, sampled, num_tries, T.n_classes, S, lq);
    OEA_LAUNCH(k_nce_logits<GatheredW>, H.lg, kThreads, 0, st, T, n, x, sampled, lq, G, loss_out, GatheredW{});
    OEA_LAUNCH(k_nce_dx<GatheredW>, H.dx, kThreads, 0, st, T, n, G, sampled, H.split_s, dx, GatheredW{});
    OEA_LAUNCH(k_nce_dw<GatheredW>, H.dw, kThreads, 0, st, T, n, G, x, sampled, H.split_b, GatheredW{});
    OEA_LAUNCH(k_nce_true, rows_grid, kThreads, 0, st, T, pos_t, n, x, num_tries, 1.f, dx, loss_out);
    OEA_LAUNCH(k_proje_columns_bwd, col_grid, kThreads, 0, st, T, n, xh, xr, z, dx, stats, dxh, dxr);
    OEA_LAUNCH(k_proje_push, rows_grid, kThreads, 0, st, T, pos_h, pos_r, n, dxh, dxr);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" size_t oea_nce_workspace_bytes(int32_t n, int32_t num_sampled, int32_t dim, int32_t n_classes) {
    if (n < 0 || num_sampled < 1 || dim <= 0 || n_classes <= 0) return 0;
    return nce_layout(n, num_sampled, round4(dim), n_classes).total;
}

extern "C" int oea_nce_score_fed(const oea_nce* model, const int32_t* inputs, const int32_t* labels, int32_t n,
                                 const int32_t* sampled, const int32_t* num_tries, int32_t num_sampled, float loss_scale,
                                 void* workspace, size_t workspace_bytes, double* loss_out, void* stream) {
    if (model == nullptr) return OEA_ERR_NULL;
    const oea_table* tabs[3] = {model->in, model->cls_w, model->cls_b};
    for (const oea_table* t : tabs) {
        const int rc = check_table(t, true);
        if (rc) return rc;
    }
    const oea_table *in = model->in, *w = model->cls_w, *b = model->cls_b;
    if (w->dim != in->dim || w->pitch != in->pitch || in->pitch > kProjeMaxPitch) return OEA_ERR_DIM;
    NceWs L{};
    const int rc = check_head(w, b, num_sampled, n, sampled, num_tries, loss_out, inputs && labels,
                              workspace, workspace_bytes,
                              [&] { return (L = nce_layout(n, num_sampled, in->pitch, w->rows)).total; });
    if (rc != OEA_OK || n == 0) return rc;

    char* ws = static_cast<char*>(workspace);
    float* x = reinterpret_cast<float*>(ws + L.x);
    float* dx = reinterpret_cast<float*>(ws + L.dx);
    float* ws_w = reinterpret_cast<float*>(ws + L.w);
    float* ws_dw = reinterpret_cast<float*>(ws + L.dw);
    float* winv = reinterpret_cast<float*>(ws + L.winv);
    float* wss = reinterpret_cast<float*>(ws + L.wss);
    float* lq = reinterpret_cast<float*>(ws + L.lq);
    float* G = reinterpret_cast<float*>(ws + L.g);
    ProjeDev T{};
    T.ent = table_dev(in); T.w = table_dev(w); T.b = table_dev(b);
    T.b.norm = false;                                     // the biases are a raw [C, 1] variable
    T.dim = in->dim; T.pitch = in->pitch; T.n_classes = w->rows; T.num_sampled = num_sampled; T.ldg = L.ldg;
    const StagedW hw{ws_w, ws_dw, loss_scale};
    cudaStream_t st = (cudaStream_t)stream;
    const int S = num_sampled;
    const HeadGrids H = head_grids(n, S, L.ldg);
#ifdef OEA_HOST_EMU
    const int s_grid = 2;
#else
    const int s_grid = grid_for(S);
#endif
    OEA_CUDA_TRY(cudaMemsetAsync(dx, 0, 4 * (size_t)n * in->pitch, st));
    OEA_LAUNCH(k_nce_stage, s_grid, kThreads, 0, st, T, sampled, ws_w, ws_dw, winv, wss);
    OEA_LAUNCH(k_nce_gather, H.rows, kThreads, 0, st, T, inputs, n, x);
    OEA_LAUNCH(k_nce_logq, H.rows, kThreads, 0, st, sampled, num_tries, T.n_classes, S, lq);
    OEA_LAUNCH(k_nce_logits<StagedW>, H.lg, kThreads, 0, st, T, n, x, sampled, lq, G, loss_out, hw);
    OEA_LAUNCH(k_nce_dx<StagedW>, H.dx, kThreads, 0, st, T, n, G, sampled, H.split_s, dx, hw);
    OEA_LAUNCH(k_nce_dw<StagedW>, H.dw, kThreads, 0, st, T, n, G, x, sampled, H.split_b, hw);
    OEA_LAUNCH(k_nce_true, H.rows, kThreads, 0, st, T, labels, n, x, num_tries, loss_scale, dx, loss_out);
    OEA_LAUNCH(k_nce_w_push, s_grid, kThreads, 0, st, T, sampled, ws_w, ws_dw, winv, wss);
    OEA_LAUNCH(k_nce_in_push, H.rows, kThreads, 0, st, T, inputs, n, dx);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_pairs_draw(const int32_t* pairs, int32_t n_pairs, int32_t batch, uint64_t seed, int32_t epoch,
                              int32_t step, int32_t* first, int32_t* second, void* stream) {
    if (n_pairs < 0 || batch < 0 || batch > n_pairs) return OEA_ERR_RANGE;
    if (batch == 0) return OEA_OK;
    if (pairs == nullptr || first == nullptr || second == nullptr) return OEA_ERR_NULL;
    OEA_LAUNCH_STRIDED(k_pairs_draw, (batch + kThreads - 1) / kThreads, kThreads, 0, (cudaStream_t)stream, pairs,
                       (uint32_t)n_pairs, batch, pairs_key(seed, epoch, step), first, second);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" size_t oea_conve_workspace_bytes(int32_t n_pos, int32_t num_sampled, int32_t dim, int32_t filters,
                                            int32_t n_classes) {
    if (n_pos < 0 || num_sampled < 1 || dim <= 0 || filters < 1 || n_classes <= 0) return 0;
    return conve_layout(n_pos, num_sampled, dim, round4(dim), filters, n_classes).total;
}

extern "C" int oea_conve_score_fed(const oea_conve* model, const int32_t* pos_h, const int32_t* pos_r,
                                   const int32_t* pos_t, int32_t n_pos, const int32_t* sampled, const int32_t* num_tries,
                                   int32_t num_sampled, float keep_prob, uint64_t dropout_seed, void* workspace,
                                   size_t workspace_bytes, double* loss_out, void* stream) {
    if (model == nullptr) return OEA_ERR_NULL;
    const oea_table* tabs[8] = {model->ent, model->rel, model->cls_w, model->cls_b, model->conv, model->bn_in,
                                model->fc_w, model->fc_out};
    for (const oea_table* t : tabs) {
        const int rc = check_table(t, true);
        if (rc) return rc;
    }
    const oea_table *ent = model->ent, *rel = model->rel, *w = model->cls_w, *b = model->cls_b;
    const oea_table *conv = model->conv, *bn_in = model->bn_in, *fc_w = model->fc_w, *fc_out = model->fc_out;
    const int d = ent->dim, P = ent->pitch, F = conv->rows;
    if (rel->dim != d || w->dim != d || rel->pitch != P || w->pitch != P || fc_w->pitch != P || fc_out->pitch != P ||
        P > kProjeMaxPitch)
        return OEA_ERR_DIM;
    if (F < 1) return OEA_ERR_DIM;
    int fx, fy;
    conve_factor(d, &fx, &fy);
    if (conv->dim != kConvCols || bn_in->rows != 2 || bn_in->dim != fy || fc_w->rows != 2 * F * d || fc_w->dim != d ||
        fc_out->rows != 3 || fc_out->dim != d)
        return OEA_ERR_SHAPE;
    if (!(keep_prob > 0.f && keep_prob <= 1.f)) return OEA_ERR_RANGE;
    ConveWs L{};
    const int rc = check_head(w, b, num_sampled, n_pos, sampled, num_tries, loss_out, pos_h && pos_r && pos_t,
                              workspace, workspace_bytes,
                              [&] { return (L = conve_layout(n_pos, num_sampled, d, P, F, w->rows)).total; });
    if (rc != OEA_OK || n_pos == 0) return rc;

    char* ws = static_cast<char*>(workspace);
    float* img = reinterpret_cast<float*>(ws + L.img);
    float* A = reinterpret_cast<float*>(ws + L.a);
    float* z = reinterpret_cast<float*>(ws + L.z);
    float* x = reinterpret_cast<float*>(ws + L.x);
    float* dx = reinterpret_cast<float*>(ws + L.dx);
    float* lq = reinterpret_cast<float*>(ws + L.lq);
    float* G = reinterpret_cast<float*>(ws + L.g);
    ProjeDev T{};
    T.ent = table_dev(ent); T.rel = table_dev(rel); T.w = table_dev(w); T.b = table_dev(b);
    T.w.norm = T.b.norm = false;                          // entity_w and entity_b: raw
    T.dim = d; T.pitch = P; T.n_classes = w->rows; T.num_sampled = num_sampled; T.ldg = L.ldg;
    ConveDev C;
    C.conv = table_dev(conv); C.bn_in = table_dev(bn_in); C.fc_w = table_dev(fc_w); C.fc_out = table_dev(fc_out);
    C.x = fx; C.y = fy; C.F = F; C.K = 2 * F * d; C.lda = L.lda; C.keep = keep_prob; C.seed = dropout_seed;
    // the dense layer on the head's dX and dW kernels: G := A with 2Fd columns at row stride lda (its padding columns
    // are zero, as G's are), W_S := fc_w as a contiguous block.  StagedW ignores the sampled ids.
    ProjeDev Tfc = T;
    Tfc.num_sampled = C.K; Tfc.ldg = L.lda;
    const StagedW fc{C.fc_w.w, C.fc_w.g, 1.f};
    cudaStream_t st = (cudaStream_t)stream;
    const int n = n_pos, S = num_sampled;
    const HeadGrids H = head_grids(n, S, L.ldg), Hfc = head_grids(n, C.K, L.lda);
#ifdef OEA_HOST_EMU
    const int pos_grid = 2, conv_grid = 2, out_grid = 2, bwd_grid = 2, split_conv = 7;
#else
    // split the per-filter sums of the conv backward so that about two CTAs per SM run
    const int sms = sm_count_cached();
    const int conv_parts = (2 * sms + F - 1) / F, split_conv = (n + conv_parts - 1) / conv_parts;
    const int pos_grid = min(n, 8 * sms);
    const int conv_grid = F * ((n + split_conv - 1) / split_conv);
    const int out_grid = min((int)(((size_t)n * P + kThreads - 1) / kThreads), 8 * sms);
    const int bwd_grid = min((n + 1) / 2, sms);           // two rows per block step; one flush of 3·d sums per block
#endif
    OEA_CUDA_TRY(cudaMemsetAsync(z, 0, 4 * (size_t)n * P, st));
    OEA_CUDA_TRY(cudaMemsetAsync(dx, 0, 4 * (size_t)n * P, st));
    OEA_LAUNCH(k_conve_conv_fwd, pos_grid, kThreads, 0, st, T, C, pos_h, pos_r, n, img, A);
    OEA_LAUNCH(k_nce_dx<StagedW>, Hfc.dx, kThreads, 0, st, Tfc, n, A, sampled, Hfc.split_s, z, fc);
    OEA_LAUNCH(k_conve_fc_out, out_grid, kThreads, 0, st, T, C, n, z, x);
    OEA_LAUNCH(k_nce_logq, H.rows, kThreads, 0, st, sampled, num_tries, T.n_classes, S, lq);
    OEA_LAUNCH(k_nce_logits<GatheredW>, H.lg, kThreads, 0, st, T, n, x, sampled, lq, G, loss_out, GatheredW{});
    OEA_LAUNCH(k_nce_dx<GatheredW>, H.dx, kThreads, 0, st, T, n, G, sampled, H.split_s, dx, GatheredW{});
    OEA_LAUNCH(k_nce_dw<GatheredW>, H.dw, kThreads, 0, st, T, n, G, x, sampled, H.split_b, GatheredW{});
    OEA_LAUNCH(k_nce_true, H.rows, kThreads, 0, st, T, pos_t, n, x, num_tries, 1.f, dx, loss_out);
    OEA_LAUNCH(k_conve_fc_out_bwd, bwd_grid, kThreads, 0, st, T, C, n, z, dx);
    OEA_LAUNCH(k_nce_dw<StagedW>, Hfc.dw, kThreads, 0, st, Tfc, n, A, dx, sampled, Hfc.split_b, fc);
    OEA_LAUNCH(k_conve_fc_dx, Hfc.lg, kThreads, 0, st, T, C, n, dx, A);
    OEA_LAUNCH(k_conve_conv_dw, conv_grid, kThreads, 0, st, T, C, n, img, A, split_conv);
    OEA_LAUNCH(k_conve_conv_dx, pos_grid, kThreads, 0, st, T, C, pos_h, pos_r, n, A);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}
