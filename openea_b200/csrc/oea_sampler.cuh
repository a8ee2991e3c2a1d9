// oea_sampler.cuh — the on-device batch sampler of path (i), shared by the fused step kernels (oea_triple.cu) and the
// batch producer (oea_sampler.cu): step parameters, the counter RNG, negative sampling of one positive by its warp
// (modules/train/batch.py:89-119), and the host-side slice arithmetic of batch.py:36-53.  sm_90a.
#pragma once
#include <stdlib.h>
#include "oea_rowmath.cuh"

namespace oea {

struct SampledParams {
    oea_kg_view kg[2];
    oea_tripleset tset;
    int n_slice[2];      // positives of this step taken from each KG
    int start[2];        // offset of the slice inside the (permuted) triple list
    int k;               // negatives per positive
    int step;
    int max_try;
    uint64_t seed;
    const uint64_t* dev_seed;   // optional device scalar xor-ed into seed (CUDA-graph replays)
    int shard_rank, shard_world;   // this launch scores the positives p ≡ shard_rank (mod shard_world); 0 / 1 = all
    int diag;            // OEA_DIAG bit mask (measurement only): 1 synthetic negatives (no cand/hash chain),
                         // 2 no gradient output, 4 no negatives, 8 identity permutation
};

// Counter RNG of the sampler: `rng_base` folds (epoch seed, step, positive) once per positive; every draw is one
// pcg32 of the base xor a small counter.
__device__ __forceinline__ uint32_t rng_base(uint64_t seed, uint32_t step, uint32_t p) {
    return pcg32((uint32_t)seed ^ pcg32((uint32_t)(seed >> 32) ^ (step * 0x9E3779B9u)) ^ (p * 0x85EBCA6Bu));
}
__device__ __forceinline__ uint32_t rng_draw(uint32_t base, uint32_t a, uint32_t b) {
    return pcg32(base ^ (a * 0xC2B2AE35u) ^ (b * 0x27D4EB2Fu));
}

// Negative sampling of one positive by its warp (batch.py:89-119): lane j < k ends up owning negative j
// (corrupted entity neg_e, neg_head = head corrupted).  Up to max_try rounds; a round flips ONE coin for all
// still-missing negatives, draws distinct candidate positions for them, keeps the draws that are not known
// triples; the last round keeps everything.
__device__ __forceinline__ void warp_sample_negatives(const SampledParams& P, uint64_t seed, const oea_kg_view& kg, int p, int h, int r,
                                                      int t, int k, int lane, const float* __restrict__ ent_w, int ent_pitch,
                                                      int& neg_e, bool& neg_head) {
    bool need = lane < k;
    const uint32_t base = rng_base(seed, (uint32_t)P.step, (uint32_t)p);
    for (int tr = 0; tr < P.max_try; ++tr) {
        const unsigned missing = __ballot_sync(OEA_FULL, need);
        if (missing == 0u) break;
        const bool head = (rng_draw(base, 0x51DEu, tr) >> 31) != 0;  // np.random.binomial(1, .5)
        const int corrupted = head ? h : t;
        const int32_t* list = kg.entities;
        uint32_t C = (uint32_t)kg.n_entities;
        if (kg.cand != nullptr) {
            if (kg.ent2row == nullptr) {   // candidate matrix indexed by entity id; a row starting with −1 = no list
                const int32_t* row = kg.cand + (size_t)corrupted * kg.n_cand;
                if (__ldg(row) >= 0) { list = row; C = (uint32_t)kg.n_cand; }
            } else {
                const int row = __ldg(kg.ent2row + corrupted);
                if (row >= 0) { list = kg.cand + (size_t)row * kg.n_cand; C = (uint32_t)kg.n_cand; }
            }
        }
        // random.sample(candidates, #missing): distinct positions among the needing lanes
        uint32_t pos = 0;
        bool unsettled = need;
        for (uint32_t redraw = 0; ; ++redraw) {
            if (unsettled) pos = bounded32(rng_draw(base, (tr << 8) | lane, 0xC0FFEEu + redraw), C);
            const unsigned active = __ballot_sync(OEA_FULL, need);
            unsigned same = 0u;
            if (need) same = __match_any_sync(active, pos);
            // the lowest lane of a duplicate group keeps its draw, the others redraw
            unsettled = need && ((same & ((1u << lane) - 1u)) != 0u);
            if (__ballot_sync(OEA_FULL, unsettled) == 0u) break;
        }
        if (need) {
            const int e = __ldg(list + pos);
            // start fetching the candidate's row while the membership probe is in flight (rejections are < 1 %)
            prefetch_row_l2(ent_w + (size_t)e * ent_pitch, ent_pitch);
            bool accept = tr == P.max_try - 1;
            if (!accept) {
                const uint64_t key = head ? triple_key(e, r, t, P.tset.ent_bits, P.tset.rel_bits)
                                          : triple_key(h, r, e, P.tset.ent_bits, P.tset.rel_bits);
                accept = !tset_contains(P.tset, key);
            }
            if (accept) { neg_e = e; neg_head = head; need = false; }
        }
    }
}

}  // namespace oea

inline int check_kg(const oea_kg_view* kg, int k) {
    if (kg == nullptr) return OEA_ERR_NULL;
    if (kg->n_triples < 0 || kg->n_entities < 0) return OEA_ERR_RANGE;
    if (kg->n_triples > 0 && (kg->triples == nullptr || kg->entities == nullptr)) return OEA_ERR_NULL;
    if (kg->n_triples > 0 && kg->n_entities < k) return OEA_ERR_RANGE;  // random.sample would raise
    if (kg->cand != nullptr && kg->n_cand < (k > 1 ? k : 1)) return OEA_ERR_RANGE;
    return OEA_OK;
}

// batch.py:39-42 / :48-53 — slice bounds of one KG for one step, computed as the reference does.
inline void slice_of(int n_triples, int batch_kg, int step, int* start, int* count) {
    long long s = (long long)step * batch_kg, e = s + batch_kg;
    if (e > n_triples) e = n_triples;
    if (s > n_triples) s = n_triples;
    *start = (int)s;
    *count = (int)(e - s > 0 ? e - s : 0);
}

// Slice arithmetic + sampler parameters of one step (batch.py:36-53), shared by every sampling entry point.
inline int sampler_prepare(const oea_kg_view* kg1, const oea_kg_view* kg2, const oea_tripleset* tset,
                           const oea_sample_cfg* smp, oea::SampledParams* Pout, int* n_pos_out_host) {
    using namespace oea;
    if (!smp || !tset || !tset->slots) return OEA_ERR_NULL;
    if (smp->neg_per_pos < 0 || smp->neg_per_pos > 32 || smp->batch_size < 1 || smp->max_try < 1 || smp->step < 0) return OEA_ERR_RANGE;
    if (tset->capacity == 0 || (tset->capacity & (tset->capacity - 1)) != 0) return OEA_ERR_RANGE;
    int rc = check_kg(kg1, smp->neg_per_pos); if (rc) return rc;
    rc = check_kg(kg2, smp->neg_per_pos); if (rc) return rc;
    const long long T = (long long)kg1->n_triples + kg2->n_triples;
    if (T == 0) return OEA_ERR_RANGE;
    // int(len(l1) / (len(l1) + len(l2)) * batch_size): float division, multiply, truncate (batch.py:39)
    const int b1 = (int)((double)kg1->n_triples / (double)T * (double)smp->batch_size);
    const int b2 = smp->batch_size - b1;

    SampledParams& P = *Pout;
    P.kg[0] = *kg1; P.kg[1] = *kg2; P.tset = *tset;
    slice_of(kg1->n_triples, b1, smp->step, &P.start[0], &P.n_slice[0]);
    slice_of(kg2->n_triples, b2, smp->step, &P.start[1], &P.n_slice[1]);
    P.k = smp->neg_per_pos; P.step = smp->step; P.max_try = smp->max_try; P.seed = smp->epoch_seed;
    P.dev_seed = smp->dev_seed;
    if (smp->shard_world < 0 || (smp->shard_world > 1 && (smp->shard_rank < 0 || smp->shard_rank >= smp->shard_world))) return OEA_ERR_RANGE;
    P.shard_world = smp->shard_world > 1 ? smp->shard_world : 1;
    P.shard_rank = smp->shard_world > 1 ? smp->shard_rank : 0;
    {   // measurement-only ablation switches (DESIGN.md §4, "where the time goes"); read once per process
        static int diag_cached = -1;
        if (diag_cached < 0) { const char* dg = getenv("OEA_DIAG"); diag_cached = dg ? atoi(dg) : 0; }
        P.diag = diag_cached;
    }
    *n_pos_out_host = P.n_slice[0] + P.n_slice[1];
    return OEA_OK;
}

