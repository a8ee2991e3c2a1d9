// oea_rowopt.cuh — the row optimiser phase shared by the one-launch training steps (oea_triple.cu: the sampled step;
// oea_triple_grouped.cu: the fed step): TF1 Adagrad / SGD on the rows a scorer flagged, in the octet layout.  sm_90a.
#pragma once
#include "oea_rowmath.cuh"

namespace oea {

// Row optimiser over the concatenated row space [ent rows | rel rows] in the octet layout: a warp reads 32 row
// flags at once, then finishes the flagged rows four at a time (octet o takes the o-th flagged row; 12 independent
// 16-byte loads per lane are in flight).  TF1 Adagrad / SGD as in k_rowopt.
struct OptTab {
    float* w;
    float* g;
    float* s1;
    int32_t* touched;
    int rows;
};

template <int KIND>
__device__ __forceinline__ void oct_rowopt_body(const OptTab& A, const OptTab& B, int pitch, float lr, int warp_global,
                                                int n_warps) {
    const int lane = threadIdx.x & 31, oct = lane >> 3, l = lane & 7;
    const int p4 = pitch >> 2;
    const int total = A.rows + B.rows;
    const int n_quads = (total + 3) >> 2;          // work unit: 4 consecutive rows, one per octet
    auto flag_of = [&](int quad) -> int32_t* {
        const int r = 4 * quad + oct;
        if (quad >= n_quads || r >= total) return nullptr;
        return r < A.rows ? A.touched + r : B.touched + (r - A.rows);
    };
    int quad = warp_global;
    int32_t* flag = flag_of(quad);
    int on = (flag != nullptr && l == 0) ? *flag : 0;
    while (quad < n_quads) {
        // the next quad's flag is in flight while this quad's rows are processed
        const int next = quad + n_warps;
        int32_t* nflag = flag_of(next);
        const int non = (nflag != nullptr && l == 0) ? *nflag : 0;
        const bool mine = __shfl_sync(OEA_FULL, on, oct << 3) != 0;
        if (mine) {
            const int rr = 4 * quad + oct;
            const bool first = rr < A.rows;
            const OptTab& T = first ? A : B;
            const size_t off = (size_t)(first ? rr : rr - A.rows) * pitch;
            if (l == 0) *flag = 0;
            for (int q0 = 0; q0 < p4; q0 += 32) {
                float4 g[4], x[4], a[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int q = q0 + l + 8 * i;
                    if (q < p4) {
                        g[i] = *reinterpret_cast<const float4*>(T.g + off + 4 * q);
                        x[i] = *reinterpret_cast<const float4*>(T.w + off + 4 * q);
                        if (KIND == OEA_OPT_ADAGRAD) a[i] = *reinterpret_cast<const float4*>(T.s1 + off + 4 * q);
                    }
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int q = q0 + l + 8 * i;
                    if (q < p4) {
                        if (KIND == OEA_OPT_ADAGRAD) {
                            a[i].x = fmaf(g[i].x, g[i].x, a[i].x); a[i].y = fmaf(g[i].y, g[i].y, a[i].y);
                            a[i].z = fmaf(g[i].z, g[i].z, a[i].z); a[i].w = fmaf(g[i].w, g[i].w, a[i].w);
                            x[i].x -= lr * g[i].x * rsqrtf(a[i].x); x[i].y -= lr * g[i].y * rsqrtf(a[i].y);
                            x[i].z -= lr * g[i].z * rsqrtf(a[i].z); x[i].w -= lr * g[i].w * rsqrtf(a[i].w);
                            *reinterpret_cast<float4*>(T.s1 + off + 4 * q) = a[i];
                        } else {
                            x[i].x -= lr * g[i].x; x[i].y -= lr * g[i].y; x[i].z -= lr * g[i].z; x[i].w -= lr * g[i].w;
                        }
                        *reinterpret_cast<float4*>(T.w + off + 4 * q) = x[i];
                        *reinterpret_cast<float4*>(T.g + off + 4 * q) = f4(0.f);
                    }
                }
            }
        }
        quad = next; flag = nflag; on = non;
    }
}

}  // namespace oea
