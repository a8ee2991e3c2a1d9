// oea_p2p.cu — path (i) across GPUs: the per-epoch exchange of seed-pair rows (SURVEY §8e, BASELINE.json north_star)
// as direct peer-memory stores over NVLink instead of a library collective.  sm_90a.
//
// The reference has no multi-device code (SURVEY §2a); the exchange mirrors what its single session does implicitly:
// the seed entities of models/basic_model.py:211-236 are the rows both KGs' triples keep coherent.
//
// Every rank owns a WINDOW (one cudaMalloc, exported with cudaIpcGetMemHandle, mapped by every peer):
//     rows  [2 parities][world sources][max_rows][pitch] fp32     staging of published rows
//     flags [2 parities][world sources] uint64                    epoch number of the last complete publication
//     status[4] int32                                             [0] != 0: a wait timed out
// push(epoch): a warp per owned row reads the row from the table and stores it into the slot
//     rows[epoch & 1][rank] of EVERY peer's window (st.global over NVLink, 128-bit); every CTA fences at system scope
//     and takes a ticket; the last CTA publishes flags[epoch & 1][rank] = epoch on every peer with st.release.sys.
// pull(epoch): lanes 0..world-1 of each CTA's first warp acquire the local flags (ld.acquire.sys, bounded spin), the
//     CTA barrier extends the acquire to the whole CTA, then a warp per received row copies staging → table.
// Two parities are enough: a rank publishes epoch e+2 only after it has pulled e+1, which every peer publishes only
// after having pulled e (stream order on each rank: … pull(e), push(e+1) …), so the slot it overwrites has been read.
#include <string.h>
#ifdef OEA_HOST_EMU
#include <atomic>
#include <chrono>
#endif
#include "oea_rowmath.cuh"

namespace oea {

struct XchgLayout {
    size_t rows_bytes, flags_off, status_off, total;
};
__host__ __device__ inline XchgLayout xchg_layout(int world, int max_rows, int pitch) {
    XchgLayout L;
    L.rows_bytes = (size_t)2 * world * max_rows * pitch * sizeof(float);
    L.flags_off = (L.rows_bytes + 255) & ~(size_t)255;
    L.status_off = L.flags_off + (size_t)2 * world * sizeof(unsigned long long);
    L.total = (L.status_off + 4 * sizeof(int32_t) + 255) & ~(size_t)255;
    return L;
}

struct XchgDev {
    char* window[OEA_P2P_MAX_WORLD];
    const int32_t* own_ids;
    const int32_t* slot_ids;
    int32_t* ticket;
    int rank, world, pitch, max_rows, n_own;
};

#ifdef OEA_HOST_EMU   // tests/emu: "peers" are buffers of the same process; plain atomics stand in for the system-scope PTX
inline void st_release_sys(unsigned long long* p, unsigned long long v) { std::atomic_ref<unsigned long long>(*p).store(v, std::memory_order_release); }
inline unsigned long long ld_acquire_sys(const unsigned long long* p) {
    return std::atomic_ref<unsigned long long>(*const_cast<unsigned long long*>(p)).load(std::memory_order_acquire);
}
inline unsigned long long global_ns() {
    return (unsigned long long)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
inline float4 ld_cg4(const float* p) { return *reinterpret_cast<const float4*>(p); }
inline void __threadfence_system() { std::atomic_thread_fence(std::memory_order_seq_cst); }
inline void __nanosleep(unsigned) {}
inline int emu_exchange(int32_t* p, int v) { return std::atomic_ref<int32_t>(*p).exchange(v); }
#define OEA_ATOMIC_EXCH(P, V) emu_exchange((P), (V))
#else
#define OEA_ATOMIC_EXCH(P, V) atomicExch((P), (V))
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ float4 ld_cg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
#endif

// own rows → contiguous [n_own, pitch] (the NCCL variant's send buffer)
__global__ void __launch_bounds__(kThreads)
k_seed_pack(const float* __restrict__ w, int pitch, const int32_t* __restrict__ ids, int n, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int p4 = pitch >> 2;
    for (int i = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); i < n; i += gridDim.x * kWarpsPerBlock) {
        const float* src = w + (size_t)__ldg(ids + i) * pitch;
        float* dst = out + (size_t)i * pitch;
        for (int c = lane; c < p4; c += OEA_WARP) *reinterpret_cast<float4*>(dst + 4 * c) = *reinterpret_cast<const float4*>(src + 4 * c);
    }
}

// staging [world, max_rows, pitch] → table rows slot_ids[g, i] (−1 = padding), skipping this rank's own slot
__device__ __forceinline__ void unpack_body(float* __restrict__ w, int pitch, const float* __restrict__ recv,
                                            const int32_t* __restrict__ slot_ids, int world, int max_rows, int rank) {
    const int lane = threadIdx.x & 31;
    const int p4 = pitch >> 2;
    const int total = world * max_rows;
    for (int s = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); s < total; s += gridDim.x * kWarpsPerBlock) {
        if (s / max_rows == rank) continue;
        const int row = __ldg(slot_ids + s);
        if (row < 0) continue;
        const float* src = recv + (size_t)s * pitch;
        float* dst = w + (size_t)row * pitch;
        for (int c = lane; c < p4; c += OEA_WARP) *reinterpret_cast<float4*>(dst + 4 * c) = ld_cg4(src + 4 * c);
    }
}

__global__ void __launch_bounds__(kThreads)
k_seed_unpack(float* __restrict__ w, int pitch, const float* __restrict__ recv, const int32_t* __restrict__ slot_ids,
              int world, int max_rows, int rank) {
    unpack_body(w, pitch, recv, slot_ids, world, max_rows, rank);
}

__global__ void __launch_bounds__(kThreads)
k_seed_push(XchgDev X, const float* __restrict__ w, unsigned long long epoch) {
    const int lane = threadIdx.x & 31;
    const int p4 = X.pitch >> 2;
    const int parity = (int)(epoch & 1ull);
    const size_t slot_off = ((size_t)(parity * X.world + X.rank) * X.max_rows) * X.pitch * sizeof(float);
    for (int i = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); i < X.n_own; i += gridDim.x * kWarpsPerBlock) {
        const float* src = w + (size_t)__ldg(X.own_ids + i) * X.pitch;
        for (int c = lane; c < p4; c += OEA_WARP) {
            const float4 v = *reinterpret_cast<const float4*>(src + 4 * c);
            for (int g = 0; g < X.world; ++g) {
                if (g == X.rank) continue;
                float* dst = reinterpret_cast<float*>(X.window[g] + slot_off) + (size_t)i * X.pitch;
                *reinterpret_cast<float4*>(dst + 4 * c) = v;
            }
        }
    }
    // publication: all of this CTA's peer stores are ordered before its ticket; the last CTA raises the flags
    __threadfence_system();
    __syncthreads();
    __shared__ int s_last;
    if (threadIdx.x == 0) s_last = atomicAdd(X.ticket, 1) == (int)gridDim.x - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence_system();
    const XchgLayout L = xchg_layout(X.world, X.max_rows, X.pitch);
    if (threadIdx.x < X.world && threadIdx.x != X.rank) {
        unsigned long long* flags = reinterpret_cast<unsigned long long*>(X.window[threadIdx.x] + L.flags_off);
        st_release_sys(flags + parity * X.world + X.rank, epoch);
    }
    if (threadIdx.x == 0) *X.ticket = 0;      // the next push starts from a clean ticket (stream-ordered)
}

__global__ void __launch_bounds__(kThreads)
k_seed_pull(XchgDev X, float* __restrict__ w, unsigned long long epoch, unsigned long long timeout_ns) {
    const XchgLayout L = xchg_layout(X.world, X.max_rows, X.pitch);
    char* win = X.window[X.rank];
    const int parity = (int)(epoch & 1ull);
    if (threadIdx.x < X.world && threadIdx.x != X.rank) {
        const unsigned long long* flag = reinterpret_cast<const unsigned long long*>(win + L.flags_off) + parity * X.world + threadIdx.x;
        const unsigned long long t0 = global_ns();
        while (ld_acquire_sys(flag) < epoch) {
            if (global_ns() - t0 > timeout_ns) {     // a peer never published: report, do not hang the device
                OEA_ATOMIC_EXCH(reinterpret_cast<int32_t*>(win + L.status_off), 1);
                break;
            }
            __nanosleep(200);
        }
    }
    __syncthreads();
    const float* recv = reinterpret_cast<const float*>(win) + (size_t)parity * X.world * X.max_rows * X.pitch;
    unpack_body(w, X.pitch, recv, X.slot_ids, X.world, X.max_rows, X.rank);
}

static int xchg_dev(const oea_seed_xchg* x, XchgDev* out) {
    if (!x) return OEA_ERR_NULL;
    if (x->world < 1 || x->world > OEA_P2P_MAX_WORLD || x->rank < 0 || x->rank >= x->world) return OEA_ERR_RANGE;
    if (x->pitch <= 0 || (x->pitch & 3) != 0 || x->max_rows < 1 || x->n_own < 0 || x->n_own > x->max_rows) return OEA_ERR_DIM;
    if (!x->slot_ids || !x->ticket || (x->n_own > 0 && !x->own_ids)) return OEA_ERR_NULL;
    for (int g = 0; g < x->world; ++g) {
        if (!x->window[g]) return OEA_ERR_NULL;
        out->window[g] = (char*)x->window[g];
    }
    out->own_ids = x->own_ids; out->slot_ids = x->slot_ids; out->ticket = x->ticket;
    out->rank = x->rank; out->world = x->world; out->pitch = x->pitch; out->max_rows = x->max_rows; out->n_own = x->n_own;
    return OEA_OK;
}

}  // namespace oea

using namespace oea;

extern "C" size_t oea_seed_xchg_window_bytes(int32_t world, int32_t max_rows, int32_t pitch) {
    if (world < 1 || max_rows < 1 || pitch < 1) return 0;
    return xchg_layout(world, max_rows, pitch).total;
}

extern "C" int oea_p2p_window_create(size_t bytes, void** dev_ptr, void* handle_out64) {
    if (!dev_ptr || !handle_out64 || bytes == 0) return OEA_ERR_NULL;
    void* p = nullptr;
    OEA_CUDA_TRY(cudaMalloc(&p, bytes));
    cudaError_t e = cudaMemset(p, 0, bytes);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    cudaIpcMemHandle_t h;
    if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) { cudaFree(p); return -(int)e; }
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    memcpy(handle_out64, &h, sizeof(h));
    *dev_ptr = p;
    return OEA_OK;
}

extern "C" int oea_p2p_window_open(const void* handle64, void** peer_ptr) {
    if (!handle64 || !peer_ptr) return OEA_ERR_NULL;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, sizeof(h));
    void* p = nullptr;
    OEA_CUDA_TRY(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    *peer_ptr = p;
    return OEA_OK;
}

extern "C" int oea_p2p_window_close(void* peer_ptr) {
    if (!peer_ptr) return OEA_ERR_NULL;
    OEA_CUDA_TRY(cudaIpcCloseMemHandle(peer_ptr));
    return OEA_OK;
}

extern "C" int oea_p2p_window_destroy(void* dev_ptr) {
    if (!dev_ptr) return OEA_ERR_NULL;
    OEA_CUDA_TRY(cudaFree(dev_ptr));
    return OEA_OK;
}

extern "C" int oea_seed_pack(const float* weight, int32_t pitch, const int32_t* ids, int32_t n, float* out, void* stream) {
    if (n < 0 || pitch <= 0 || (pitch & 3) != 0) return OEA_ERR_DIM;
    if (n == 0) return OEA_OK;
    if (!weight || !ids || !out) return OEA_ERR_NULL;
    OEA_LAUNCH(k_seed_pack, grid_for(n), kThreads, 0, (cudaStream_t)stream, weight, pitch, ids, n, out);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_seed_unpack(float* weight, int32_t pitch, const float* recv, const int32_t* slot_ids, int32_t world,
                               int32_t max_rows, int32_t rank, void* stream) {
    if (world < 1 || max_rows < 1 || pitch <= 0 || (pitch & 3) != 0) return OEA_ERR_DIM;
    if (!weight || !recv || !slot_ids) return OEA_ERR_NULL;
    OEA_LAUNCH(k_seed_unpack, grid_for(world * max_rows), kThreads, 0, (cudaStream_t)stream, weight, pitch, recv, slot_ids, world, max_rows, rank);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_seed_push(const oea_seed_xchg* x, const float* weight, uint64_t epoch, void* stream) {
    XchgDev X;
    int rc = xchg_dev(x, &X); if (rc) return rc;
    if (!weight) return OEA_ERR_NULL;
    if (epoch == 0) return OEA_ERR_RANGE;
    if (X.world == 1) return OEA_OK;
    const int grid = grid_for(X.n_own > 0 ? X.n_own : 1);
    OEA_LAUNCH(k_seed_push, grid, kThreads, 0, (cudaStream_t)stream, X, weight, (unsigned long long)epoch);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_seed_pull(const oea_seed_xchg* x, float* weight, uint64_t epoch, uint64_t timeout_ns, void* stream) {
    XchgDev X;
    int rc = xchg_dev(x, &X); if (rc) return rc;
    if (!weight) return OEA_ERR_NULL;
    if (epoch == 0) return OEA_ERR_RANGE;
    if (X.world == 1) return OEA_OK;
    OEA_LAUNCH(k_seed_pull, grid_for(X.world * X.max_rows), kThreads, 0, (cudaStream_t)stream, X, weight, (unsigned long long)epoch,
               (unsigned long long)timeout_ns);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

extern "C" int oea_seed_xchg_status(const oea_seed_xchg* x, int32_t* status_host) {
    if (!x || !status_host || x->rank < 0 || x->rank >= OEA_P2P_MAX_WORLD || !x->window[x->rank]) return OEA_ERR_NULL;
    const XchgLayout L = xchg_layout(x->world, x->max_rows, x->pitch);
#ifdef OEA_HOST_EMU
    memcpy(status_host, (const char*)x->window[x->rank] + L.status_off, sizeof(int32_t));
#else
    OEA_CUDA_TRY(cudaMemcpy(status_host, (const char*)x->window[x->rank] + L.status_off, sizeof(int32_t), cudaMemcpyDeviceToHost));
#endif
    return OEA_OK;
}
