// oea_optim_ext.cu — tf.train.AdadeltaOptimizer (modules/base/optimizers.py:13-15 of the reference) as a dense table
// update.  sm_90a.
//
// TF1 ApplyAdadelta (defaults rho = 0.95, epsilon = 1e-8, both slots start at 0), element-wise and in this order:
//     accum        = rho·accum + (1 − rho)·g²
//     update       = sqrt(accum_update + ε) · rsqrt(accum + ε) · g
//     var         −= lr·update
//     accum_update = rho·accum_update + (1 − rho)·update²
// Unlike Adagrad / SGD the update is NOT row-sparse: a row without gradient still decays both accumulators, so every
// row is visited (as for Adam).  HBM-bound: 4 reads + 3 writes of the table per step (w, g, accum, accum_update in;
// w, accum, accum_update out; g is zeroed: a 4th write) = 32 B per element.  One thread per float4, grid-stride.
#include "oea_rowmath.cuh"

namespace oea {

__global__ void __launch_bounds__(256)
k_rowopt_adadelta(float* __restrict__ w, float* __restrict__ grad, float* __restrict__ accum,
                  float* __restrict__ accum_update, int32_t* __restrict__ touched, int rows, long long n4,
                  float lr, float rho, float eps) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 g = reinterpret_cast<const float4*>(grad)[i];
        float4 a = reinterpret_cast<const float4*>(accum)[i];
        float4 u = reinterpret_cast<const float4*>(accum_update)[i];
        float4 x = reinterpret_cast<const float4*>(w)[i];
        const float g_[4] = {g.x, g.y, g.z, g.w};
        float a_[4] = {a.x, a.y, a.z, a.w}, u_[4] = {u.x, u.y, u.z, u.w}, x_[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            a_[c] = rho * a_[c] + (1.f - rho) * g_[c] * g_[c];
            const float upd = sqrtf(u_[c] + eps) * rsqrtf(a_[c] + eps) * g_[c];
            x_[c] -= lr * upd;
            u_[c] = rho * u_[c] + (1.f - rho) * upd * upd;
        }
        reinterpret_cast<float4*>(w)[i] = make_float4(x_[0], x_[1], x_[2], x_[3]);
        reinterpret_cast<float4*>(accum)[i] = make_float4(a_[0], a_[1], a_[2], a_[3]);
        reinterpret_cast<float4*>(accum_update)[i] = make_float4(u_[0], u_[1], u_[2], u_[3]);
        reinterpret_cast<float4*>(grad)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += stride) touched[r] = 0;
}

}  // namespace oea

using namespace oea;

extern "C" int oea_rowopt_adadelta(const oea_table* t, const oea_opt_cfg* opt, void* stream) {
    int rc = check_table(t, true); if (rc) return rc;
    if (opt == nullptr || t->state1 == nullptr || t->state2 == nullptr) return OEA_ERR_NULL;
    if (opt->kind != OEA_OPT_ADADELTA) return OEA_ERR_KIND;
    const long long n4 = (long long)t->rows * (t->pitch >> 2);
    const long long want = (n4 + 255) / 256;
    const int cap = sm_count_cached() * 8;
    const int grid = (int)(want < 1 ? 1 : (want < cap ? want : cap));
    const float rho = opt->beta1, eps = opt->eps;     // oea_opt_cfg: beta1 carries rho for Adadelta
    OEA_LAUNCH_STRIDED(k_rowopt_adadelta, grid, 256, 0, (cudaStream_t)stream, t->weight, t->grad, t->state1, t->state2,
                       t->touched, t->rows, n4, opt->lr, rho, eps);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}
