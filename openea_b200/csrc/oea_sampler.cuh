// oea_sampler.cuh — the on-device batch sampler of path (i), shared by the fused step kernels (oea_triple.cu) and the
// batch producer (oea_sampler.cu): step parameters, the counter RNG, the draw of a positive and its debug-dump row,
// negative sampling of one positive by a warp or half-warp (modules/train/batch.py:89-119), and the host-side slice
// arithmetic of batch.py:36-53.  sm_90a.
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

// Positive p of a sampled step (batch.py:36-53), drawn by a group of LANES lanes: the KG q it comes from, its index
// `tri` in that KG's triple list (the Feistel permutation of the step's slice, or the slice itself when `identity`) and
// its (h, r, t), known to every lane of the group.  With `ent` / `rel` given, lanes 0-2 of the group start fetching
// the three rows into L2, to overlap that fetch with the sampling chain.  With WRITE_POS (the batch producer) they
// write (h, r, t) to pos_out[hl·n_pos + p].
struct SampledPositive {
    int q;
    uint32_t tri;
    int h, r, t;
};
template <int LANES, bool WRITE_POS = false>
__device__ __forceinline__ SampledPositive draw_positive(const SampledParams& P, uint64_t seed, int p, int lane, bool identity,
                                                         const TableDev* ent = nullptr, const TableDev* rel = nullptr,
                                                         int32_t* __restrict__ pos_out = nullptr, int n_pos = 0) {
    const int hl = lane & (LANES - 1), hbase = lane & ~(LANES - 1);
    const int q = p < P.n_slice[0] ? 0 : 1;
    const oea_kg_view& kg = P.kg[q];
    const int local = q == 0 ? p : p - P.n_slice[0];
    const uint32_t tri = identity ? (uint32_t)(P.start[q] + local)
                                  : feistel_perm((uint32_t)(P.start[q] + local), (uint32_t)kg.n_triples,
                                                 seed ^ (q ? 0xA5A5A5A5DEADBEEFull : 0x0123456789ABCDEFull));
    int hrt = 0;
    if (hl < 3) {
        hrt = __ldg(kg.triples + 3 * (size_t)tri + hl);
        if (WRITE_POS) pos_out[(size_t)hl * n_pos + p] = hrt;
    }
    const int h = __shfl_sync(OEA_FULL, hrt, hbase);
    const int r = __shfl_sync(OEA_FULL, hrt, hbase + 1);
    const int t = __shfl_sync(OEA_FULL, hrt, hbase + 2);
    if (ent != nullptr && hl < 3) {
        const float* rowp = hl == 1 ? rel->w + (size_t)r * rel->pitch : ent->w + (size_t)(hl == 0 ? h : t) * ent->pitch;
        prefetch_row_l2(rowp, ent->pitch);
    }
    return SampledPositive{q, tri, h, r, t};
}

// Row p of the optional debug dump of a sampled step: the triple index with bit 30 set for KG 2, the group's head
// mask (bit j: negative j corrupts the head; `head_mask` is the warp's ballot) and the k negatives.
template <int LANES>
__device__ __forceinline__ void dump_draws(int32_t* __restrict__ dbg, int p, int k, const SampledPositive& s, unsigned head_mask,
                                           int lane, int neg_e) {
    const int hl = lane & (LANES - 1), hbase = lane & ~(LANES - 1);
    int32_t* row = dbg + (size_t)p * (2 + k);
    if (hl == 0) {
        row[0] = (int32_t)s.tri + (s.q ? (1 << 30) : 0);
        row[1] = (int32_t)(LANES == 32 ? head_mask : (head_mask >> hbase) & ((1u << LANES) - 1u));
    }
    if (hl < k) row[2 + hl] = neg_e;
}

// Negative sampling of one positive by a group of LANES lanes (a warp, or a half-warp of the duo scorer)
// (batch.py:89-119): lane hl < k of the group ends up owning negative hl (corrupted entity neg_e, neg_head = head
// corrupted).  Up to max_try rounds; a round flips ONE coin for all still-missing negatives, draws distinct candidate
// positions for them, keeps the draws that are not known triples; the last round keeps everything.  The counters use
// hl and the distinct-position test compares inside a group only, so a half-warp draws exactly what a warp draws for
// the same positive and seed.  A group that is not `live` samples nothing.
template <int LANES>
__device__ __forceinline__ void sample_negatives(const SampledParams& P, uint64_t seed, const oea_kg_view& kg, bool live, int p,
                                                 int h, int r, int t, int k, int lane, int& neg_e, bool& neg_head) {
    static_assert(LANES == 16 || LANES == 32, "a warp or a half-warp");
    const int hl = lane & (LANES - 1);
    const uint32_t group_bit = (uint32_t)(lane / LANES) << 31;   // C <= 2^31: bit 31 separates the half-warps
    bool need = live && hl < k;
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
            if (unsettled) pos = bounded32(rng_draw(base, (tr << 8) | hl, 0xC0FFEEu + redraw), C);
            const unsigned active = __ballot_sync(OEA_FULL, need);
            unsigned same = 0u;
            if (need) same = __match_any_sync(active, pos | group_bit);
            // the lowest lane of a duplicate group keeps its draw, the others redraw
            unsettled = need && ((same & ((1u << lane) - 1u)) != 0u);
            if (__ballot_sync(OEA_FULL, unsettled) == 0u) break;
        }
        if (need) {
            // No L2 prefetch of the candidate's row here: the scorer's demand loads of it follow within the same
            // positive, and at the 100K step (memory-system throughput bound, DESIGN.md §4) the extra four line
            // requests per negative cost more than the latency they hide.
            const int e = __ldg(list + pos);
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
    if (tset->filter && (tset->filter_words == 0 || (tset->filter_words & (tset->filter_words - 1)) != 0)) return OEA_ERR_RANGE;
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

