// oea_match.cu — f-4: stable (Gale–Shapley) alignment on the device over K3's top-`cut` lists.  sm_90a.
//
// Restates modules/finding/alignment.py:171-224 (galeshapley, called by stable_alignment :87-133 with max_iteration =
// cut = 100): suitors (KG1 rows) propose to the head of their preference list; a reviewer (KG2 column) holds the suitor
// it ranks best among its holder and this round's proposers; a rejected proposer strikes the reviewer off its list; a
// DISPLACED holder keeps the reviewer at the head of its list and is rejected there in the next round (as in the
// reference, whose `del matching[r_partner]` does not touch the partner's list).  Within a round the outcome does not
// depend on the order in which the reference walks the suitors, so a round is two data-parallel kernels:
//   propose: every free suitor takes the head of its list and atomicMax-es a packed (similarity, suitor) key into the
//            reviewer's cell, which still holds its current holder's key;
//   resolve: a proposer that now owns the cell becomes the holder (the previous holder is freed), every other proposer
//            advances its list pointer.
// A reviewer ranks suitors by the similarity column (argsort(-sim.T[r])): higher similarity first, equal similarities →
// lower suitor index first (the documented tie rule of this repository; NumPy's argsort leaves it unspecified).
// Only the first `cut` entries of a suitor's list can be reached in `cut` rounds, which is why K3's top-`cut` output is
// the whole input.
#include "oea_rowmath.cuh"

namespace oea {

__device__ __forceinline__ unsigned long long gs_key(float v, int s) {
    unsigned int u = __float_as_uint(v);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);            // order-preserving map of fp32 onto uint32
    return ((unsigned long long)u << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned int)s);
}

__global__ void k_gs_init(int32_t* match, int32_t* ptr, int32_t* holder, unsigned long long* best, int n1, int n2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n1) { match[i] = -1; ptr[i] = 0; }
    if (i < n2) { holder[i] = -1; best[i] = 0ull; }
}

__global__ void k_gs_propose(const int32_t* __restrict__ pref_idx, const float* __restrict__ pref_val, int n1, int cut,
                             const int32_t* __restrict__ match, const int32_t* __restrict__ ptr, int32_t* __restrict__ prop,
                             unsigned long long* __restrict__ best, int32_t* __restrict__ n_prop) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n1) return;
    int r = -1;
    if (match[s] < 0 && ptr[s] < cut) {
        const size_t o = (size_t)s * cut + ptr[s];
        r = pref_idx[o];
        if (r >= 0) { atomicMax(best + r, gs_key(pref_val[o], s)); atomicAdd(n_prop, 1); }
    }
    prop[s] = r;
}

__global__ void k_gs_resolve(int n1, const int32_t* __restrict__ prop, const unsigned long long* __restrict__ best,
                             int32_t* __restrict__ match, int32_t* __restrict__ ptr, int32_t* __restrict__ holder) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n1) return;
    const int r = prop[s];
    if (r < 0) return;
    if ((unsigned int)(best[r] & 0xFFFFFFFFull) == 0xFFFFFFFFu - (unsigned int)s) {
        const int old = holder[r];                   // one winner per reviewer: no race on holder[r]
        if (old >= 0 && old != s) match[old] = -1;   // the displaced suitor did not propose this round: nobody else writes it
        holder[r] = s;
        match[s] = r;
    } else {
        ptr[s] += 1;                                 // rejected: strike this reviewer
    }
}

// Orders an UNORDERED top-k set per row (oea_rows_select_topk's output, k <= 128) into a preference list: gathers the
// similarities from the materialised matrix and sorts (value descending, equal values → lower column first) with a
// 128-slot bitonic network in shared memory, one CTA of 128 threads per row.
__global__ void __launch_bounds__(128)
k_rows_gather_sort(const float* __restrict__ mat, long long ld, int n_rows, int k, int32_t* __restrict__ idx, float* __restrict__ val) {
    __shared__ unsigned long long key[128];
    const int row = blockIdx.x, t = threadIdx.x;
    if (row >= n_rows) return;
    unsigned long long mine = 0ull;                       // padding sorts last (every real key has bit 63 or payload set)
    if (t < k) {
        const int c = idx[(size_t)row * k + t];
        mine = gs_key(__ldg(mat + (size_t)row * ld + c), c);
    }
    key[t] = mine;
    __syncthreads();
    for (int size = 2; size <= 128; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            const int partner = t ^ stride;
            if (partner > t) {
                const bool desc = (t & size) == 0;        // descending blocks first → whole array descending at the end
                const unsigned long long a = key[t], b = key[partner];
                if ((a < b) == desc) { key[t] = b; key[partner] = a; }
            }
            __syncthreads();
        }
    }
    if (t < k) {
        const unsigned long long v = key[t];
        const unsigned int c = 0xFFFFFFFFu - (unsigned int)(v & 0xFFFFFFFFull);
        unsigned int u = (unsigned int)(v >> 32);
        u = (u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u;
        idx[(size_t)row * k + t] = (int32_t)c;
        val[(size_t)row * k + t] = __uint_as_float(u);
    }
}

}  // namespace oea

using namespace oea;

extern "C" int oea_rows_gather_sort(const float* mat, int64_t ld, int32_t n_rows, int32_t k, int32_t* idx, float* val, void* stream) {
    if (!mat || !idx || !val) return OEA_ERR_NULL;
    if (n_rows < 1 || k < 1 || k > 128 || ld < k) return OEA_ERR_RANGE;
    OEA_LAUNCH(k_rows_gather_sort, n_rows, 128, 0, (cudaStream_t)stream, mat, (long long)ld, n_rows, k, idx, val);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" size_t oea_gale_shapley_workspace_bytes(int32_t n1, int32_t n2) {
    if (n1 < 1 || n2 < 1) return 0;
    return (size_t)n2 * 8 + ((size_t)n2 + 2 * (size_t)n1 + 4) * 4 + 64;
}

extern "C" int oea_gale_shapley(const int32_t* pref_idx, const float* pref_val, int32_t n1, int32_t n2, int32_t cut,
                                int32_t max_rounds, int32_t* match, void* workspace, size_t workspace_bytes,
                                int32_t* rounds_host, void* stream) {
    if (!pref_idx || !pref_val || !match || !workspace) return OEA_ERR_NULL;
    if (n1 < 1 || n2 < 1 || cut < 1 || cut > n2 || max_rounds < 0) return OEA_ERR_RANGE;
    if (workspace_bytes < oea_gale_shapley_workspace_bytes(n1, n2)) return OEA_ERR_WORKSPACE;
    if (((uintptr_t)workspace & 7u) != 0) return OEA_ERR_ALIGN;
    cudaStream_t st = (cudaStream_t)stream;
    unsigned long long* best = (unsigned long long*)workspace;
    int32_t* holder = (int32_t*)(best + n2);
    int32_t* ptr = holder + n2;
    int32_t* prop = ptr + n1;
    int32_t* n_prop = prop + n1;
    const int big = n1 > n2 ? n1 : n2;
    OEA_LAUNCH(k_gs_init, (big + 255) / 256, 256, 0, st, match, ptr, holder, best, n1, n2);
    OEA_LAUNCH_CHECK();
    int rounds = 0;
    int32_t h_prop = 0;
    const int grid = (n1 + 255) / 256;
    while (rounds < max_rounds) {
        OEA_CUDA_TRY(cudaMemsetAsync(n_prop, 0, sizeof(int32_t), st));
        OEA_LAUNCH(k_gs_propose, grid, 256, 0, st, pref_idx, pref_val, n1, cut, match, ptr, prop, best, n_prop);
        OEA_LAUNCH(k_gs_resolve, grid, 256, 0, st, n1, prop, best, match, ptr, holder);
        OEA_LAUNCH_CHECK();
        ++rounds;
        // the reference stops as soon as no suitor is free; poll every 4th round (one 4-byte read) and at the end
        if ((rounds & 3) == 0 || rounds == max_rounds) {
            OEA_CUDA_TRY(cudaMemcpyAsync(&h_prop, n_prop, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
            OEA_CUDA_TRY(cudaStreamSynchronize(st));
            if (h_prop == 0) break;
        }
    }
    OEA_CUDA_TRY(cudaStreamSynchronize(st));
    if (rounds_host) *rounds_host = rounds;
    return OEA_OK;
}
