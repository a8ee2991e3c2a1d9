// oea_sampler.cu — the batch producer of modules/train/batch.py:36-45 / :168-184 on the device: index vectors for the
// fed entry points (oea_triple_score_fed, oea_model_score_fed).  sm_90a.
#include "oea_sampler.cuh"

namespace oea {

// ------------------------------------------------------------------------------------------------
// Batch producer (modules/train/batch.py:36-45 / :168-184) for the fed entry points: one warp per positive writes
// the positive's (h, r, t) and its k negatives as index vectors.  Same positive selection as k_score_sampled.
// sampler 0: sample_negatives<32> (generate_neg_triples_fast).  sampler 1: generate_neg_triples (batch.py:60-86):
// lane j < k owns negative j, flips its own coin per try, draws one candidate WITH replacement, accepts the first
// draw that is not a known triple; after max_try rejections the tail becomes a uniform entity of the KG.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_sample_batch(SampledParams P, int sampler, const float* __restrict__ warm_w, int warm_pitch,
               int32_t* __restrict__ pos_out, int32_t* __restrict__ neg_out) {
    if (P.dev_seed != nullptr) P.seed ^= __ldg(reinterpret_cast<const unsigned long long*>(P.dev_seed));
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const int n_warps = gridDim.x * kWarpsPerBlock;
    const int n_pos = P.n_slice[0] + P.n_slice[1];
    const int k = P.k;
    const size_t n_neg = (size_t)n_pos * k;
    for (int p = warp_global; p < n_pos; p += n_warps) {
        const SampledPositive s = draw_positive<32, true>(P, P.seed, p, lane, false, nullptr, nullptr, pos_out, n_pos);
        const oea_kg_view& kg = P.kg[s.q];
        const int h = s.h, r = s.r, t = s.t;
        if (k == 0) continue;
        int neg_e = 0;
        bool neg_head = false;
        if (sampler == 0) {
            sample_negatives<32>(P, P.seed, kg, true, p, h, r, t, k, lane, neg_e, neg_head);
        } else if (lane < k) {
            const uint32_t base = rng_base(P.seed, (uint32_t)P.step, (uint32_t)p);
            bool done = false;
            for (int tr = 0; tr < P.max_try && !done; ++tr) {
                const bool head = (rng_draw(base, 0x51DEu + (uint32_t)lane * 64u, (uint32_t)tr) >> 31) != 0;
                const int corrupted = head ? h : t;
                const int32_t* list = kg.entities;
                uint32_t C = (uint32_t)kg.n_entities;
                if (kg.cand != nullptr) {
                    if (kg.ent2row == nullptr) {
                        const int32_t* row = kg.cand + (size_t)corrupted * kg.n_cand;
                        if (__ldg(row) >= 0) { list = row; C = (uint32_t)kg.n_cand; }
                    } else {
                        const int row = __ldg(kg.ent2row + corrupted);
                        if (row >= 0) { list = kg.cand + (size_t)row * kg.n_cand; C = (uint32_t)kg.n_cand; }
                    }
                }
                const int e = __ldg(list + bounded32(rng_draw(base, ((uint32_t)tr << 8) | (uint32_t)lane, 0xC0FFEEu), C));
                const uint64_t key = head ? triple_key(e, r, t, P.tset.ent_bits, P.tset.rel_bits)
                                          : triple_key(h, r, e, P.tset.ent_bits, P.tset.rel_bits);
                if (!tset_contains(P.tset, key)) { neg_e = e; neg_head = head; done = true; }
            }
            if (!done) {   // batch.py:82-85: (head, relation, random.choice(entities_list))
                neg_e = __ldg(kg.entities + bounded32(rng_draw(base, 0xFA11u, (uint32_t)lane), (uint32_t)kg.n_entities));
                neg_head = false;
            }
        }
        if (lane < k) {
            if (warm_w != nullptr) prefetch_row_l2(warm_w + (size_t)neg_e * warm_pitch, warm_pitch);   // for the next kernel
            const size_t o = (size_t)p * k + lane;
            neg_out[o] = neg_head ? neg_e : h;
            neg_out[n_neg + o] = r;
            neg_out[2 * n_neg + o] = neg_head ? t : neg_e;
        }
    }
}

}  // namespace oea

using namespace oea;

extern "C" int oea_triple_sample_batch(const oea_kg_view* kg1, const oea_kg_view* kg2, const oea_tripleset* tset,
                                       const oea_sample_cfg* smp, int32_t sampler, const oea_table* warm,
                                       int32_t* pos_hrt, int32_t* neg_hrt, int32_t* n_pos_host, void* stream) {
    SampledParams P;
    int n_pos = 0;
    int rc = sampler_prepare(kg1, kg2, tset, smp, &P, &n_pos); if (rc) return rc;
    if (P.shard_world != 1) return OEA_ERR_RANGE;
    if (sampler != 0 && sampler != 1) return OEA_ERR_KIND;
    if (!pos_hrt || !n_pos_host || (smp->neg_per_pos > 0 && !neg_hrt)) return OEA_ERR_NULL;
    if (warm != nullptr) { rc = check_table(warm, false); if (rc) return rc; }
    if (sampler == 0 && warm == nullptr) return OEA_ERR_NULL;   // the fast sampler always warms the rows it draws
    *n_pos_host = n_pos;
    if (n_pos == 0) return OEA_OK;
    P.diag = 0;
    const float* warm_w = warm ? warm->weight : nullptr;
    const int warm_pitch = warm ? warm->pitch : 0;
    OEA_LAUNCH_STRIDED(k_sample_batch, grid_for(n_pos), kThreads, 0, (cudaStream_t)stream, P, sampler, warm_w, warm_pitch,
                       pos_hrt, neg_hrt);
    OEA_LAUNCH_CHECK();
    return OEA_OK;
}

