// oea_rowopt.cuh — the flagged-row optimiser shared by the one-launch training steps (oea_triple.cu: the sampled steps;
// oea_triple_grouped.cu: the fed steps) and by the two-launch path's k_rowopt_pair: TF1 Adagrad / SGD on the rows a
// scorer flagged, over the concatenated row space [A rows | B rows].  sm_90a.
#pragma once
#include "oea_rowmath.cuh"

namespace oea {

struct OptTab {
    float* w;
    float* g;
    float* s1;
    int32_t* touched;
    int rows;
};

// Row optimiser over [A rows | B rows] (same pitch), flagged rows only; TF1 Adagrad (acc += g², x −= lr·g/√acc) or
// SGD (x −= lr·g), then g = 0 and the flag cleared.  Padding columns are left as they are.
//
// The work unit is a quad of 4 consecutive rows.  Warp w owns quads w, w + n_warps, … : strided, because entity ids
// are ordered by degree and the flagged rows cluster at low ids.  It walks them in windows of 32 quads, lane j taking
// the window's j-th quad and loading its four flags; every flag load of a window is issued before any is used, so a
// window costs one flag latency.  The window's flagged rows (up to 128, from four ballots) are then finished four at a
// time: octet o takes the o-th remaining flagged row, wherever it lies in the window (12 independent 16-byte loads per
// lane in flight).  A quad may straddle the tables when A.rows % 4 != 0, so each row picks its table on its own.
template <int KIND>
__device__ __forceinline__ void rowopt_flagged_body(const OptTab& A, const OptTab& B, int pitch, float lr, int warp_global,
                                                    int n_warps) {
    const int lane = threadIdx.x & 31, oct = lane >> 3, l = lane & 7;
    const int p4 = pitch >> 2;
    const int total = A.rows + B.rows;
    const int n_quads = (total + 3) >> 2;
    for (int w0 = warp_global; w0 < n_quads; w0 += 32 * n_warps) {
        const int quad = w0 + n_warps * lane;
        int32_t f[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = 4 * quad + i;
            f[i] = 0;
            if (quad < n_quads && r < total) f[i] = r < A.rows ? A.touched[r] : B.touched[r - A.rows];
        }
        // bit j of m[i]: row i of the window's j-th quad is flagged.  The ballots also order every lane's flag reads
        // before any flag is cleared below.
        unsigned m[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) m[i] = __ballot_sync(OEA_FULL, f[i] != 0);
        while ((m[0] | m[1] | m[2] | m[3]) != 0u) {
            int pick = -1, skip = oct;           // octet o: the o-th set bit of m[0] … m[3], taken in that order
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int c = __popc(m[i]);
                if (pick < 0 && skip < c) {
                    unsigned mm = m[i];
                    for (int s = 0; s < skip; ++s) mm &= mm - 1u;
                    pick = 32 * i + __ffs((int)mm) - 1;
                } else if (pick < 0) {
                    skip -= c;
                }
            }
#pragma unroll
            for (int s = 0; s < 4; ++s) {        // the four rows taken leave the set
                if (m[0] != 0u) m[0] &= m[0] - 1u;
                else if (m[1] != 0u) m[1] &= m[1] - 1u;
                else if (m[2] != 0u) m[2] &= m[2] - 1u;
                else m[3] &= m[3] - 1u;
            }
            if (pick < 0) continue;
            const int rr = 4 * (w0 + n_warps * (pick & 31)) + (pick >> 5);
            const bool first = rr < A.rows;
            // fields chosen by value: a reference to A or B would put both parameter structs in a stack frame
            float* const tw = first ? A.w : B.w;
            float* const tg = first ? A.g : B.g;
            float* const ts = first ? A.s1 : B.s1;
            int32_t* const tt = first ? A.touched : B.touched;
            const int row = first ? rr : rr - A.rows;
            const size_t off = (size_t)row * pitch;
            if (l == 0) tt[row] = 0;
            for (int q0 = 0; q0 < p4; q0 += 32) {
                float4 g[4], x[4], a[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int q = q0 + l + 8 * i;
                    if (q < p4) {
                        g[i] = *reinterpret_cast<const float4*>(tg + off + 4 * q);
                        x[i] = *reinterpret_cast<const float4*>(tw + off + 4 * q);
                        if (KIND == OEA_OPT_ADAGRAD) a[i] = *reinterpret_cast<const float4*>(ts + off + 4 * q);
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
                            *reinterpret_cast<float4*>(ts + off + 4 * q) = a[i];
                        } else {
                            x[i].x -= lr * g[i].x; x[i].y -= lr * g[i].y; x[i].z -= lr * g[i].z; x[i].w -= lr * g[i].w;
                        }
                        *reinterpret_cast<float4*>(tw + off + 4 * q) = x[i];
                        *reinterpret_cast<float4*>(tg + off + 4 * q) = f4(0.f);
                    }
                }
            }
        }
    }
}

}  // namespace oea
