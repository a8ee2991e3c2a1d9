/*
 * oea.h — C-ABI of liboea.so, the H100 (sm_90a) engine behind the OpenEA hot path.
 *
 * The reference (nju-websoft/OpenEA) has NO native / FFI layer: its "operator API" is a set of
 * Python callables that bottom out in TensorFlow-1 session.run() and NumPy.  Each entry point
 * below names the reference callable(s) it replaces (file:line under /root/reference/src/openea).
 *
 * Conventions (all entry points):
 *   - extern "C", plain pointers and sizes, no C++/torch types.
 *   - return int: 0 = OEA_OK, >0 = argument error (OEA_ERR_*), <0 = -(cudaError_t).
 *   - device pointers unless the name ends in _host; `stream` is a cudaStream_t passed as void*.
 *   - never allocate or free device memory; the caller owns every buffer (incl. workspaces).
 *   - asynchronous on `stream` unless documented otherwise (the *_host entry points synchronise,
 *     mirroring the synchronous session.run() they replace).
 *   - no CUDA context is created at load time (safe to dlopen in forked workers).
 */
#ifndef OEA_H_
#define OEA_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OEA_ABI_VERSION 1

enum {
    OEA_OK = 0,
    OEA_ERR_NULL = 1,        /* required pointer is NULL */
    OEA_ERR_DIM = 2,         /* dim/pitch/rows out of the supported range */
    OEA_ERR_ALIGN = 3,       /* pointer or pitch not 16-byte aligned */
    OEA_ERR_KIND = 4,        /* unknown score / loss / optimiser / metric kind */
    OEA_ERR_SHAPE = 5,       /* inconsistent batch sizes (e.g. margin loss needs n_neg == n_pos) */
    OEA_ERR_RANGE = 6,       /* k, n_cand, … out of range */
    OEA_ERR_WORKSPACE = 7    /* workspace too small */
};

/* ---- score / loss / optimiser kinds -------------------------------------------------------- */
/* modules/base/losses.py:15-73: `loss_norm == 'L1'` → Σ|h+r−t| ; anything else → Σ(h+r−t)² (squared) */
enum { OEA_SCORE_L1 = 0, OEA_SCORE_L2SQ = 1 };
/* losses.py margin_loss:15, limited_loss:42, logistic_loss:59, positive_loss:30;
 * approaches/bootea.py:197 alignment loss  −Σ log σ(−s)  (OEA_LOSS_LOGSIGMOID, positives only) */
enum { OEA_LOSS_MARGIN = 0, OEA_LOSS_LIMITED = 1, OEA_LOSS_LOGISTIC = 2, OEA_LOSS_POSITIVE = 3,
       OEA_LOSS_LOGSIGMOID = 4 };
/* modules/base/optimizers.py:10-20 (TF1 semantics: Adagrad acc0 = 0.1 and no epsilon; TF-Adam) */
enum { OEA_OPT_SGD = 0, OEA_OPT_ADAGRAD = 1, OEA_OPT_ADAM = 2, OEA_OPT_ADADELTA = 3 };

/* An embedding table as TF holds it: the raw variable + optimiser slots (+ our gradient scratch).
 * Replaces the tf.Variable made by modules/base/initializers.py:9-50; `l2_norm` mirrors the
 * `is_l2_norm` flag: every lookup goes through x·rsqrt(max(Σx², 1e-12)) and the gradient flows
 * back through that normalisation (initializers.py:26,34,41,50).
 * Layout: row-major [rows, pitch] fp32, pitch % 4 == 0, pitch >= dim, padding columns are zero.
 * `grad` must be all-zero and `touched` all-zero between steps (oea_rowopt_apply restores that). */
typedef struct oea_table {
    float*   weight;   /* [rows, pitch] raw variable (NOT normalised) */
    float*   grad;     /* [rows, pitch] gradient accumulator */
    float*   state1;   /* [rows, pitch] Adagrad accumulator / Adam m (NULL for SGD) */
    float*   state2;   /* [rows, pitch] Adam v (NULL otherwise) */
    int32_t* touched;  /* [rows] 0/1 flags: row received gradient this step */
    int32_t  rows;
    int32_t  dim;
    int32_t  pitch;
    int32_t  l2_norm;
} oea_table;

typedef struct oea_loss_cfg {
    int32_t score_kind;   /* OEA_SCORE_* */
    int32_t loss_kind;    /* OEA_LOSS_* */
    float   margin;       /* margin (margin-based) or pos_margin (limited) */
    float   neg_margin;   /* limited */
    float   balance;      /* limited: weight of the negative part (aligne.py:63-65) */
} oea_loss_cfg;

typedef struct oea_opt_cfg {
    int32_t kind;         /* OEA_OPT_* */
    float   lr;
    float   beta1, beta2, eps;  /* Adam (TF defaults .9 / .999 / 1e-8); Adadelta: beta1 = rho (.95), eps = epsilon (1e-8) */
    int32_t t;            /* Adam only: 1-based step count */
} oea_opt_cfg;

/* One KG's share of the training data for the fused on-device sampler.
 * Replaces the Python lists handed to modules/train/batch.py:36-45. */
typedef struct oea_kg_view {
    const int32_t* triples;   /* [n_triples, 3] (h, r, t) */
    int32_t        n_triples;
    const int32_t* entities;  /* [n_entities] entity ids of this KG (uniform candidate list) */
    int32_t        n_entities;
    const int32_t* cand;      /* ε-truncated neighbour lists [cand_rows, n_cand], or NULL */
    const int32_t* ent2row;   /* [ent table rows] entity id → row of `cand`, −1 = no list.  NULL with cand != NULL:
                               * `cand` is indexed by ENTITY ID ([ent table rows, n_cand]) and a row whose first
                               * element is −1 means "no list" (one dependent load less per positive) */
    int32_t        n_cand;
} oea_kg_view;

/* Open-addressing set of packed (h, r, t) keys (triple membership test of batch.py:104-109). */
typedef struct oea_tripleset {
    const uint64_t* slots;    /* [capacity], empty = 0xFFFFFFFFFFFFFFFF */
    uint32_t        capacity; /* power of two */
    uint32_t        ent_bits; /* key = (h << (ent_bits + rel_bits)) | (r << ent_bits) | t */
    uint32_t        rel_bits;
    const uint64_t* filter;   /* optional blocked Bloom filter of the same keys [filter_words] (one word and four bits
                               * per key, tset_filter_hash / tset_filter_bits of oea_common.cuh), or NULL: a key the
                               * filter rejects is absent without probing `slots` */
    uint32_t        filter_words; /* power of two when filter != NULL */
} oea_tripleset;

typedef struct oea_sample_cfg {
    int32_t  batch_size;      /* args.batch_size: positives per step over both KGs */
    int32_t  neg_per_pos;     /* args.neg_triple_num (0..32) */
    int32_t  step;            /* step index inside the epoch */
    int32_t  max_try;         /* batch.py:89 max_try (10) */
    uint64_t epoch_seed;      /* permutation + sampling seed of this epoch */
    const uint64_t* dev_seed; /* optional DEVICE scalar xor-ed into epoch_seed at kernel start: lets a CUDA graph of a
                               * whole epoch (one node pair per step) be replayed with a new seed every epoch */
    int32_t  shard_rank;      /* exact-parity multi-GPU mode (SURVEY 8e): this call scores only the positives p of the   */
    int32_t  shard_world;     /* step's batch with p % shard_world == shard_rank (draws depend on p, not on the shard, so
                               * the union over ranks IS the single-GPU batch); 0 or 1 = the whole batch.  Honoured by
                               * oea_triple_score_sampled; the other sampling entry points require the whole batch. */
} oea_sample_cfg;

/* ---- path (i) across GPUs: peer-memory exchange of seed-pair rows (oea_p2p.cu) ------------------ */
#define OEA_P2P_MAX_WORLD 16
/* One rank's view of the exchange.  window[g] is rank g's window (oea_p2p_window_create on rank g) as mapped in THIS
 * process (window[rank] is the local allocation, the others come from oea_p2p_window_open). */
typedef struct oea_seed_xchg {
    int32_t        rank, world;      /* world <= OEA_P2P_MAX_WORLD */
    int32_t        pitch;            /* floats per row, == the table's pitch */
    int32_t        max_rows;         /* rows per (parity, source rank) slot: max over ranks of the owned-row count */
    void*          window[OEA_P2P_MAX_WORLD];
    const int32_t* own_ids;          /* [n_own] device: the rows this rank owns and publishes, in slot order */
    int32_t        n_own;
    const int32_t* slot_ids;         /* [world, max_rows] device: table row of every received slot, -1 = padding */
    int32_t*       ticket;           /* device int32, zero-initialised (last-CTA election of the push kernel) */
} oea_seed_xchg;

/* ---- misc ---------------------------------------------------------------------------------- */
int         oea_abi_version(void);
const char* oea_error_string(int code);

/* ---- path (i): negative-sampled triple scoring, forward + backward ------------------------- */

/* Fed step, forward+backward only.  Replaces the graph of models/basic_model.py:80-98 /
 * approaches/aligne.py:47-66 / approaches/mtranse.py:46-57 / approaches/bootea.py:190-199 up to
 * compute_gradients: gathers rows, scores, evaluates the loss of modules/base/losses.py and
 * scatter-adds d(loss)/d(raw variable) into ent->grad / rel->grad (setting `touched`).
 * n_neg may be 0 (positive / logsigmoid losses).  *loss_out (device, fp64) is incremented by the
 * batch loss (sum over the batch, as TF's reduce_sum). */
int oea_triple_score_fed(const oea_table* ent, const oea_table* rel,
                         const int32_t* pos_h, const int32_t* pos_r, const int32_t* pos_t, int32_t n_pos,
                         const int32_t* neg_h, const int32_t* neg_r, const int32_t* neg_t, int32_t n_neg,
                         const oea_loss_cfg* loss, double* loss_out, void* stream);

/* oea_triple_score_fed for batches in the reference's layout (batch.py:36-45): the n_neg / n_pos negatives of positive p
 * sit at p·k … p·k+k−1.  One warp scores a positive and its negatives: rows a negative shares with its positive are
 * neither reloaded nor reduced separately (3 + k row loads and reductions per positive instead of 3·(1 + k)); a negative
 * that shares fewer than two rows takes the general path, so every fed batch gives the same result as
 * oea_triple_score_fed (up to fp32 summation order).  Requires n_pos > 0 and n_neg % n_pos == 0. */
int oea_triple_score_fed_grouped(const oea_table* ent, const oea_table* rel,
                                 const int32_t* pos_h, const int32_t* pos_r, const int32_t* pos_t, int32_t n_pos,
                                 const int32_t* neg_h, const int32_t* neg_r, const int32_t* neg_t, int32_t n_neg,
                                 const oea_loss_cfg* loss, double* loss_out, void* stream);

/* Margin loss with a weight per pair: scale · Σ_i w_i · relu(loss->margin + s(pos_i) − s(neg_i)), s by loss->score_kind.
 * w_i = weights[i] (OEA_WEIGHT_DIRECT), 1 / weights[i] (OEA_WEIGHT_RECIPROCAL) or 1 (weights NULL).  Replaces
 * approaches/iptranse.py:170-174 (_generate_transe_alignment_loss; w = similarity of the newly aligned pair) and
 * iptranse.py:176-180 (_generate_path_loss; reciprocal path weights, scale = args.path_parm).  For the path loss the
 * three ids of a "triple" are relation ids (r_x + r_y − r): pass the relation table as BOTH `ent` and `rel`.
 * Accumulates into grad / touched like oea_triple_score_fed; *loss_out (device, fp64) += the weighted batch loss. */
enum { OEA_WEIGHT_DIRECT = 0, OEA_WEIGHT_RECIPROCAL = 1 };
int oea_triple_score_margin_weighted(const oea_table* ent, const oea_table* rel,
                                     const int32_t* pos_h, const int32_t* pos_r, const int32_t* pos_t,
                                     const int32_t* neg_h, const int32_t* neg_r, const int32_t* neg_t, int32_t n,
                                     const float* weights, int32_t weight_mode, float scale,
                                     const oea_loss_cfg* loss, double* loss_out, void* stream);

/* scale · Σ_i w_i · ‖ê[ids_a[i]] − ê[ids_b[i]]‖² over looked-up (normalised when ent->l2_norm) rows, forward + backward
 * into ent->grad / touched.  weights may be NULL (w = 1).  Replaces IMUSE's align loss (approaches/imuse.py:303-306). */
int oea_pair_distance_loss(const oea_table* ent, const int32_t* ids_a, const int32_t* ids_b, int32_t n,
                           const float* weights, float scale, double* loss_out, void* stream);

/* The whole fed step — oea_triple_score_fed_grouped followed by oea_rowopt_apply_pair — as ONE cooperative launch
 * (grouped scoring, grid barrier, row optimiser): session.run([triple_loss, triple_optimizer], feed_dict) of
 * models/basic_model.py:222-232 on device index vectors.  Squared-L2 score, pitch <= 256, Adagrad / SGD; returns
 * OEA_ERR_KIND for anything else (take the two-call path then).  Opt-in on the host-index steps: OEA_FED_FUSED=1. */
int oea_triple_step_fed_grouped(const oea_table* ent, const oea_table* rel,
                                const int32_t* pos_h, const int32_t* pos_r, const int32_t* pos_t, int32_t n_pos,
                                const int32_t* neg_h, const int32_t* neg_r, const int32_t* neg_t, int32_t n_neg,
                                const oea_loss_cfg* loss, const oea_opt_cfg* opt, double* loss_out, void* stream);

/* Optimiser step on a table whose `grad` was filled by a score call.  Replaces
 * optimizer.apply_gradients of modules/base/optimizers.py:4-7.  Adagrad / SGD touch only flagged
 * rows (identical to TF's dense update because untouched rows have g = 0); Adam is dense.
 * Leaves grad = 0 and touched = 0. */
int oea_rowopt_apply(const oea_table* table, const oea_opt_cfg* opt, void* stream);

/* tf.train.AdadeltaOptimizer (optimizers.py:13-15): dense update of every row (both accumulators decay on rows without
 * gradient); state1 = accum, state2 = accum_update, both start at 0; opt->beta1 = rho, opt->eps = epsilon.
 * oea_rowopt_apply dispatches OEA_OPT_ADADELTA here.  Leaves grad = 0 and touched = 0. */
int oea_rowopt_adadelta(const oea_table* table, const oea_opt_cfg* opt, void* stream);

/* The optimiser step of BOTH tables in one launch (Adagrad / SGD; Adam falls back to two dense launches).
 * Same semantics as two oea_rowopt_apply calls. */
int oea_rowopt_apply_pair(const oea_table* a, const oea_table* b, const oea_opt_cfg* opt, void* stream);

/* Fused on-device step: batch slicing + negative sampling of modules/train/batch.py:36-119 and the
 * forward/backward above in ONE kernel (no index buffers).  Positive p of step s is
 * triples[perm_epoch(s·B_kg + p)] with B_1 = ⌊B·T1/(T1+T2)⌋, B_2 = B − B_1 (batch.py:39-42);
 * negatives corrupt head or tail (one Bernoulli(.5) per try for all missing negatives),
 * candidates = ε-truncated list of the corrupted entity or the KG's entity list, sampled without
 * replacement inside a try, rejected when in `tset`, last try accepts unfiltered (batch.py:89-119).
 * neg_per_pos: >= 1 for LIMITED / LOGISTIC, exactly 1 for MARGIN (pairs), 0 for POSITIVE / LOGSIGMOID.
 * dbg_neg: optional [batch_size, 2 + neg_per_pos] int32 dump (triple index, side bitmask, sampled
 * entities) so a test can replay the identical batch through the fed path / the oracle.
 * n_pos_out (device int32, optional) receives the number of positives actually in this step. */
int oea_triple_score_sampled(const oea_table* ent, const oea_table* rel,
                             const oea_kg_view* kg1, const oea_kg_view* kg2, const oea_tripleset* tset,
                             const oea_sample_cfg* smp, const oea_loss_cfg* loss,
                             double* loss_out, int32_t* n_pos_out, int32_t* dbg_neg, void* stream);

/* One whole training step in one call: oea_triple_score_sampled + oea_rowopt_apply_pair (what one
 * session.run([triple_loss, triple_optimizer]) of basic_model.py:224 does, without the feed). */
int oea_triple_step_sampled(const oea_table* ent, const oea_table* rel,
                            const oea_kg_view* kg1, const oea_kg_view* kg2, const oea_tripleset* tset,
                            const oea_sample_cfg* smp, const oea_loss_cfg* loss, const oea_opt_cfg* opt,
                            double* loss_out, int32_t* n_pos_out, void* stream);

/* Reference-facing synchronous step with HOST index buffers (the session.run(feed_dict) boundary of
 * models/basic_model.py:222-232): H2D copy of the six index vectors into `dev_idx_ws`
 * (>= 3·(n_pos+n_neg) int32), score, optimiser step on both tables, D2H of the batch loss,
 * stream synchronise.  Returns the batch loss in *loss_host. */
int oea_triple_step_fed_host(const oea_table* ent, const oea_table* rel,
                             const int32_t* pos_hrt_host, int32_t n_pos,   /* [3, n_pos] h|r|t */
                             const int32_t* neg_hrt_host, int32_t n_neg,   /* [3, n_neg] */
                             const oea_loss_cfg* loss, const oea_opt_cfg* opt,
                             int32_t* dev_idx_ws, double* dev_loss_ws, double* loss_pinned_host,
                             float* loss_host, void* stream);

/* ---- path (i), SURVEY §8f-2: the other score functions of the reference's models/ ------------------------ */

/* Which score function a fed step evaluates and which tables it reads:
 *   TRANSE    Σ|ĥ + r̂ − t̂| or Σ(·)²                              models/trans/transe.py:33-45
 *   TRANSH    the same on e⊥ = e − <e, n̂>n̂, n̂ = l2_normalize(normal_vector[r])   models/trans/transh.py:25-51,
 *                                                                  approaches/bootea_transh.py:57-95
 *   TRANSD    the same on e⊥ = l2_normalize(e + <e, e_p>·r_p)      models/trans/transd.py:26-65
 *   DISTMULT  similarity Σ ĥ∘r̂∘t̂                                  models/semantic/distmult.py:43-59
 *   SIMPLE    (Σ l2n(h_H∘r₁)∘t_T + Σ l2n(t_H∘r₂)∘h_T)/2            models/semantic/simple.py:50-86
 *   ROTATE    Σ_i |ĥ_i·e^{iθ_i} − t̂_i| − γ over (re, im) pairs,      models/semantic/rotate.py:52-110,
 *             θ = r̂·phase                                          approaches/bootea_rotate.py:48-108,149-160
 *   HOLE      similarity σ(<l2n(r̂), ccorr(ĥ, t̂)>), ccorr_k = Σ_i ĥ_i·t̂_{(i+k) mod dim}   models/semantic/hole.py:41-86
 * The similarity models are scored as energies E = −similarity, so OEA_LOSS_LOGISTIC gives their
 * softplus(−score⁺) + softplus(score⁻).  ROTATE's energy is the distance minus γ, so OEA_LOSS_LOGISTIC is the reference's
 * −log σ(γ − d⁺) − log σ(d⁻ − γ) and OEA_LOSS_LOGSIGMOID its alignment loss −log σ(γ − d).
 * ROTATE and HOLE run in fp32 like every other kind (the reference keeps RotatE's variables in float64); the gradient of
 * RotatE's modulus at a zero coordinate is 0 (TF's is NaN there).  HOLE computes the correlation directly, O(dim²).
 *   TRANSR    Σ|l2n(M_r·ĥ) + r̂ − l2n(M_r·t̂)| or Σ(·)², M_r = rel_matrix[r] as d×d     models/trans/transr.py:14-52
 *             (row-major).  The projections are l2-normalised whatever ent's l2_norm says; the matrix never is.  rel_aux
 *             is the matrix table: rows = rel->rows·dim, row r·dim + i = row i of M_r.  Scored by oea_transr_score_fed
 *             only (it needs a workspace); oea_model_score_fed returns OEA_ERR_KIND for it. */
enum { OEA_MODEL_TRANSE = 0, OEA_MODEL_TRANSH = 1, OEA_MODEL_TRANSD = 2, OEA_MODEL_DISTMULT = 3, OEA_MODEL_SIMPLE = 4,
       OEA_MODEL_ROTATE = 5, OEA_MODEL_HOLE = 6, OEA_MODEL_TRANSR = 7 };

typedef struct oea_model {
    int32_t kind;              /* OEA_MODEL_* */
    const oea_table* ent;      /* ent_embeds                                 | SIMPLE: head_ent_embeds | ROTATE: re_ent_embeds */
    const oea_table* rel;      /* rel_embeds                                 | SIMPLE: rel_embeds1 */
    const oea_table* ent_aux;  /* TRANSD: ent_transfer | SIMPLE: tail_ent_embeds | ROTATE: im_ent_embeds | else NULL */
    const oea_table* rel_aux;  /* TRANSH: normal_vector, TRANSD: rel_transfer | SIMPLE: rel_embeds2   | TRANSR: rel_matrix
                                * | else NULL */
    float gamma;               /* ROTATE: γ (args.gamma); ignored by the other kinds */
    float phase;               /* ROTATE: π/ρ with ρ = (γ + 2)/dim, the scale from r̂ to the phase (rotate.py:37,90);
                                * ignored by the other kinds */
} oea_model;

/* oea_triple_score_fed for any oea_model: gathers the 3–6 rows of every triple, scores it, evaluates the loss of
 * modules/base/losses.py and scatter-adds d(loss)/d(raw variable) into the grad of every table involved (setting
 * `touched`).  MARGIN pairs positive i with negative i (n_pos == n_neg).  loss_scale multiplies loss and gradient
 * (1 for TF's reduce_sum losses; 1/(n_pos+n_neg) for DistMult's reduce_mean, distmult.py:58).
 * ROTATE takes every loss but MARGIN (OEA_ERR_KIND); a negative weight other than the positives' (1/k in rotate.py:81)
 * is a second call with only negatives.  HOLE takes only MARGIN (OEA_ERR_KIND otherwise), with n_neg = k·n_pos
 * negatives in the reference layout (those of positive p at p·k … p·k+k−1): Σ_p relu(m + E⁺_p − mean_j E⁻_{p,j})
 * (hole.py:80-84); OEA_ERR_SHAPE when n_pos does not divide n_neg.
 * All tables share dim and pitch, pitch <= 256.  Run oea_rowopt_apply on every table afterwards. */
int oea_model_score_fed(const oea_model* model,
                        const int32_t* pos_h, const int32_t* pos_r, const int32_t* pos_t, int32_t n_pos,
                        const int32_t* neg_h, const int32_t* neg_r, const int32_t* neg_t, int32_t n_neg,
                        const oea_loss_cfg* loss, float loss_scale, double* loss_out, void* stream);

/* TransR's fed step (models/trans/transr.py:14-52), with oea_model_score_fed's semantics, loss kinds, pairing rule and
 * argument checks, for model->kind == OEA_MODEL_TRANSR: the scored triples are grouped by relation on the device, and
 * each chunk of ≤ 64 triples of one relation reads M_r once and reduces its gradient once (red into rel_aux->grad,
 * its d rows flagged in rel_aux->touched).  Entity and relation gradients as every other kind.  FP32 throughout.
 * OEA_ERR_DIM when pitch > 128 or the three tables disagree on pitch; OEA_ERR_SHAPE when rel_aux->rows != rel->rows·dim
 * or rel_aux->dim != dim; OEA_ERR_WORKSPACE when the 16-byte aligned workspace is smaller than
 * oea_transr_workspace_bytes(n_pos, n_neg, dim, rel->rows).  No allocation, no host synchronisation.
 * Run oea_rowopt_apply on the three tables afterwards. */
size_t oea_transr_workspace_bytes(int32_t n_pos, int32_t n_neg, int32_t dim, int32_t n_rel);
int oea_transr_score_fed(const oea_model* model,
                         const int32_t* pos_h, const int32_t* pos_r, const int32_t* pos_t, int32_t n_pos,
                         const int32_t* neg_h, const int32_t* neg_r, const int32_t* neg_t, int32_t n_neg,
                         const oea_loss_cfg* loss, float loss_scale, void* workspace, size_t workspace_bytes,
                         double* loss_out, void* stream);

/* ---- path (i), ProjE (models/neural/proje.py) ---------------------------------------------------------------------- */

/* TF's log_uniform_candidate_sampler(unique=True, range_max) as nce_loss calls it: P(c) = log((c+2)/(c+1)) / log(E+1),
 * draws until num_sampled distinct classes are held.  Writes the classes in draw order to sampled [num_sampled] and the
 * number of draws taken to *num_tries (both device int32; no host synchronisation).  Draw j is a pure function of
 * (seed, j): ⌊exp(u_j·log(E+1))⌋ − 1 mod E with u_j the top 53 bits of mix64(seed ^ mix64(j)) / 2⁵³.
 * OEA_ERR_RANGE unless 1 <= num_sampled <= range_max; OEA_ERR_WORKSPACE when the 16-byte aligned workspace holds fewer
 * than 4·range_max bytes (oea_proje_workspace_bytes covers it). */
int oea_logu_sample_unique(int32_t range_max, int32_t num_sampled, uint64_t seed, int32_t* sampled, int32_t* num_tries,
                           void* workspace, size_t workspace_bytes, void* stream);

/* ProjE's variables (proje.py:36-44, :57-62).  All tables share pitch <= 128.
 *   ent, rel  ent_embeds / rel_embeds, looked up through l2_normalize when their l2_norm is set
 *   cls_w     entity_w [E, d], cls_b entity_b stored as [E, 1]; raw
 *   params    [4, d]: rows mlp/mlp_w, mlp/mlp_bias, the input batch norm's beta (shared by the head and relation
 *             inputs), the output batch norm's beta.  One table: Adam is element-wise and the four share one optimiser. */
typedef struct oea_proje {
    const oea_table* ent;
    const oea_table* rel;
    const oea_table* cls_w;
    const oea_table* cls_b;
    const oea_table* params;
} oea_proje;

/* ProjE's fed step, forward + backward (proje.py:46-74): x_h = ê[h], x_r = r̂[r]; both through a training-mode batch
 * norm (batch moments, biased variance, ε = 1e-3, the shared beta); z = (y_h + y_r)∘mlp_w + mlp_bias; X = the output
 * batch norm of z; loss = Σ_b tf.nn.nce_loss(cls_w, cls_b, label t_b, X_b) over the given sampled set (the whole batch
 * shares it): logits x·w_c + b_c − log q(c) with q(c) = −expm1(num_tries·log1p(−P(c))), or P(c)·num_sampled when
 * *num_tries == num_sampled; sigmoid cross-entropy, true class → 1, sampled → 0, accidental hits kept.
 * *loss_out (device fp64) += the batch loss; every table's grad += d loss / d raw variable, touched rows flagged.
 * FP32 throughout.  OEA_ERR_RANGE unless 1 <= num_sampled <= cls_w->rows; OEA_ERR_DIM when pitch > 128 or the pitches
 * or dims disagree; OEA_ERR_SHAPE when cls_b is not [cls_w->rows, 1] or params not [4, dim]; OEA_ERR_WORKSPACE when the
 * 16-byte aligned workspace is smaller than oea_proje_workspace_bytes(n_pos, num_sampled, dim, cls_w->rows).
 * Run oea_rowopt_apply on the five tables afterwards. */
size_t oea_proje_workspace_bytes(int32_t n_pos, int32_t num_sampled, int32_t dim, int32_t n_classes);
int oea_proje_score_fed(const oea_proje* model, const int32_t* pos_h, const int32_t* pos_r, const int32_t* pos_t,
                        int32_t n_pos, const int32_t* sampled, const int32_t* num_tries, int32_t num_sampled,
                        void* workspace, size_t workspace_bytes, double* loss_out, void* stream);

/* ---- path (i), ConvE (models/neural/conve.py) ---------------------------------------------------------------------- */

/* ConvE's variables (conve.py:42-68 on top of ProjE's proje.py:36-44).  ent, rel, cls_w, cls_b as in oea_proje; every
 * table but cls_b shares pitch <= 128.  With d = dim, (x, y) = dim_factorization(d) (conve.py:10-18) and F = conv->rows:
 *   conv    [F, 12]: row f holds the 3×3 kernel's taps of filter f (conv2d's [3, 3, 1, F] kernel, tap dy·3 + dx), the
 *           conv bias, and the gamma and beta of the batch norm over filters (axis = 1)
 *   bn_in   [2, y]: gamma and beta of the batch norm over the stacked image's columns (axis = −1)
 *   fc_w    [2·F·d, d]: fully_connected's weights (input index f·2d + i·y + j)
 *   fc_out  [3, d]: fully_connected's bias, and gamma and beta of the output batch norm
 * All raw (no l2_normalize); one Adam per table is element-wise, as TF's one optimiser over the separate variables. */
typedef struct oea_conve {
    const oea_table* ent;
    const oea_table* rel;
    const oea_table* cls_w;
    const oea_table* cls_b;
    const oea_table* conv;
    const oea_table* bn_in;
    const oea_table* fc_w;
    const oea_table* fc_out;
} oea_conve;

/* ConvE's fed step, forward + backward (conve.py:42-79): ê[h] and r̂[r] reshaped row-major to x × y and stacked into a
 * [2x, y] image; an inference-mode batch norm (moving mean 0, variance 1, ε = 1e-3: v·γ/√(1+ε) + β) per column;
 * dropout; a 3×3 'same' cross-correlation with F filters and a bias; a batch norm per filter; ReLU; dropout; the
 * flattened [2Fd] vector through fully_connected (ReLU); a batch norm per column → X; then tf.nn.nce_loss over the given
 * sampled set exactly as oea_proje_score_fed scores X.  Dropout keeps element i of mask s (0: the image, 1: the conv
 * output) iff (pcg32(k_s ^ i) >> 8)·2⁻²⁴ < keep_prob with k_s = pcg32(lo(seed) ^ pcg32(hi(seed) + s·0x9E3779B9)), and
 * scales kept elements by 1/keep_prob; keep_prob = 1 is the identity.  *loss_out (device fp64) += the batch loss; every
 * table's grad += d loss / d raw variable, touched rows flagged (all rows of conv, bn_in, fc_w, fc_out).  FP32
 * throughout.  OEA_ERR_RANGE unless 0 < keep_prob <= 1 and 1 <= num_sampled <= cls_w->rows; OEA_ERR_DIM when F < 1,
 * a pitch exceeds 128 or the pitches or dims disagree; OEA_ERR_SHAPE when a tower table is not of the shape above or
 * cls_b is not [cls_w->rows, 1]; OEA_ERR_WORKSPACE when the 16-byte aligned workspace is smaller than
 * oea_conve_workspace_bytes(n_pos, num_sampled, dim, F, cls_w->rows), which also covers oea_logu_sample_unique over
 * cls_w->rows classes.  Run oea_rowopt_apply on the eight tables afterwards. */
size_t oea_conve_workspace_bytes(int32_t n_pos, int32_t num_sampled, int32_t dim, int32_t filters, int32_t n_classes);
int oea_conve_score_fed(const oea_conve* model, const int32_t* pos_h, const int32_t* pos_r, const int32_t* pos_t,
                        int32_t n_pos, const int32_t* sampled, const int32_t* num_tries, int32_t num_sampled,
                        float keep_prob, uint64_t dropout_seed, void* workspace, size_t workspace_bytes,
                        double* loss_out, void* stream);

/* ---- path (i), the general sampled-NCE step (approaches/attr2vec.py) ---------------------------------------------- */

/* The variables of tf.nn.nce_loss applied to an embedding lookup.  in and cls_w share dim and a pitch <= 128; each is
 * looked up through l2_normalize when its own l2_norm is set (Attr2Vec: both, xavier_init(…, True)).  cls_b: the
 * biases stored as [C, 1], raw. */
typedef struct oea_nce {
    const oea_table* in;
    const oea_table* cls_w;
    const oea_table* cls_b;
} oea_nce;

/* loss = loss_scale · Σ_b tf.nn.nce_loss(ŵ, cls_b, label = labels[b], x̂ = in[inputs[b]]) over the given sampled set of
 * oea_logu_sample_unique (the whole batch shares it): logits x̂·ŵ_c + b_c − log q(c) as oea_proje_score_fed, sigmoid
 * cross-entropy, accidental hits kept.  Attr2Vec's reduce_mean is loss_scale = 1/n (attr2vec.py:121-123).
 * *loss_out (device fp64) += loss; the three tables' grad += loss_scale · d loss / d raw variable, touched rows flagged.
 * FP32 throughout.  OEA_ERR_DIM when the pitch exceeds 128 or in and cls_w disagree in dim or pitch; OEA_ERR_SHAPE when
 * cls_b is not [cls_w->rows, 1]; OEA_ERR_RANGE unless 1 <= num_sampled <= cls_w->rows; OEA_ERR_WORKSPACE when the
 * 16-byte aligned workspace is smaller than oea_nce_workspace_bytes(n, num_sampled, dim, cls_w->rows), which also
 * covers oea_logu_sample_unique over cls_w->rows classes.  Run oea_rowopt_apply on the three tables afterwards. */
size_t oea_nce_workspace_bytes(int32_t n, int32_t num_sampled, int32_t dim, int32_t n_classes);
int oea_nce_score_fed(const oea_nce* model, const int32_t* inputs, const int32_t* labels, int32_t n,
                      const int32_t* sampled, const int32_t* num_tries, int32_t num_sampled, float loss_scale,
                      void* workspace, size_t workspace_bytes, double* loss_out, void* stream);

/* random.sample(pairs, batch) of attr2vec.py:150 on the device: first[i], second[i] = pairs[2·r_i], pairs[2·r_i + 1]
 * for r_i = feistel_perm(i, n_pairs, key(seed, epoch, step)), i < batch — a keyed permutation of the rows restricted to
 * its first `batch` positions, so the rows are distinct within a call; it is not a uniformly random subset.
 * pairs: device int32 [n_pairs, 2].  OEA_ERR_RANGE unless 0 <= batch <= n_pairs. */
int oea_pairs_draw(const int32_t* pairs, int32_t n_pairs, int32_t batch, uint64_t seed, int32_t epoch, int32_t step,
                   int32_t* first, int32_t* second, void* stream);

/* The batch producer of modules/train/batch.py:36-45 (generate_relation_triple_batch) / :168-184
 * (generate_triple_label_batch) on the device: writes the index vectors a fed step takes.
 *   pos_hrt [3, n_pos] (h | r | t rows), neg_hrt [3, n_pos·neg_per_pos] (negatives of positive p at p·k … p·k+k−1),
 *   n_pos = positives of this step (slice arithmetic of batch.py:39-42,48-53), returned in *n_pos_host (HOST int).
 * sampler 0 = generate_neg_triples_fast (batch.py:89-119, as in oea_triple_score_sampled);
 * sampler 1 = generate_neg_triples (batch.py:60-86): every negative flips its own coin and draws one candidate
 *             with replacement per try; after max_try rejections the tail is replaced by a uniform entity of the KG.
 * `warm` (optional): an entity table whose sampled rows are prefetched into L2 for the scoring kernel that follows.
 * Both buffers must hold batch_size (·neg_per_pos) columns; their row stride is n_pos (·neg_per_pos). */
int oea_triple_sample_batch(const oea_kg_view* kg1, const oea_kg_view* kg2, const oea_tripleset* tset,
                            const oea_sample_cfg* smp, int32_t sampler, const oea_table* warm,
                            int32_t* pos_hrt, int32_t* neg_hrt, int32_t* n_pos_host, void* stream);

/* The same step as a depth-2 pipeline (oea_pipeline.cu): the H2D copy of step i+1 overlaps the kernels of step i and the
 * host reads step i's loss while step i+1 runs; table updates stay strictly sequential on `compute_stream`.
 * The caller owns everything: two streams, per slot two events (created with cudaEventDisableTiming or not), a device
 * index buffer of >= 3·(n_pos+n_neg) int32, a device fp64 loss scalar and a PINNED host fp64 loss scalar.
 * submit(slot) is asynchronous; collect(slot) blocks until that slot's step has finished and returns its loss.
 * A submitted step's host index buffers must stay untouched until collect() of that step (or of a later one). */
typedef struct oea_fed_pipeline {
    void*    copy_stream;      /* cudaStream_t */
    void*    compute_stream;   /* cudaStream_t */
    void*    ev_copied[2];     /* cudaEvent_t */
    void*    ev_computed[2];   /* cudaEvent_t */
    int32_t* dev_idx[2];
    double*  dev_loss[2];
    double*  host_loss[2];
} oea_fed_pipeline;
int oea_triple_step_fed_host_submit(const oea_table* ent, const oea_table* rel, const oea_fed_pipeline* pipe, int32_t slot,
                                    const int32_t* pos_hrt_host, int32_t n_pos, const int32_t* neg_hrt_host, int32_t n_neg,
                                    const oea_loss_cfg* loss, const oea_opt_cfg* opt);
int oea_triple_step_fed_host_collect(const oea_fed_pipeline* pipe, int32_t slot, float* loss_host);

/* Normalised view of a table (what TF returns for `ent_embeds` when is_l2_norm):
 * out[i, :dim] = normalise(weight[ids[i]]) (ids == NULL → all rows).  Replaces
 * tf.nn.embedding_lookup(self.ent_embeds, ids).eval() of basic_model.py:106-121,185,198-204. */
int oea_table_lookup(const oea_table* table, const int32_t* ids, int32_t n, float* out, int32_t out_pitch,
                     void* stream);

/* Build the triple membership set on device: slots[capacity] (capacity = power of two, >= 2·n) is
 * reset to empty and filled with the packed keys of triples [n,3].  Replaces the Python
 * `relation_triples_set` handed to batch.py:36 (modules/load/kg.py:63). */
int oea_tripleset_build(const int32_t* triples, int32_t n, uint64_t* slots, uint32_t capacity,
                        uint32_t ent_bits, uint32_t rel_bits, void* stream);

/* Backward of oea_table_lookup: grad_rows [n, grad_pitch] = d loss / d (normalised row i); pushes it through
 * the l2_normalize Jacobian of row ids[i] and scatter-adds into table->grad (sets touched).  Together with
 * oea_table_lookup this is tf.nn.embedding_lookup(l2_normalize(var), ids) + its gradient for arbitrary
 * graphs (e.g. modules/base/mapping.py:14-15). */
int oea_table_scatter_grad(const oea_table* table, const int32_t* ids, int32_t n, const float* grad_rows,
                           int32_t grad_pitch, void* stream);

/* modules/base/losses.py on already-gathered rows [n, pitch]: margin_loss:15, positive_loss:30,
 * limited_loss:42, logistic_loss:59 (+ bootea.py:197).  Adds the loss to *loss_out and writes d loss /
 * d row for all six inputs (the tensor-in → scalar-out API of get_loss_func, losses.py:4). */
int oea_loss_rows(const float* ph, const float* pr, const float* pt, int32_t n_pos,
                  const float* nh, const float* nr, const float* nt, int32_t n_neg,
                  int32_t dim, int32_t pitch, const oea_loss_cfg* loss, double* loss_out,
                  float* g_ph, float* g_pr, float* g_pt, float* g_nh, float* g_nr, float* g_nt, void* stream);

/* mapping_loss (modules/base/losses.py:76-80) forward+backward: alpha·(Σ‖e2 − e1·M‖² + Σ(M·Mᵀ − I)²)
 * (alpha = args.alpha of mapping.py:17).  e1/e2 [n, pitch]; M [dim, mpitch].  Adds the loss to
 * *loss_out, writes g_e1 / g_e2 [n, pitch] and ADDS into g_M [dim, mpitch]. */
size_t oea_mapping_workspace_bytes(int32_t dim);
int oea_mapping_fwd_bwd(const float* e1, const float* e2, int32_t n, int32_t dim, int32_t pitch,
                        const float* M, int32_t mpitch, float alpha, double* loss_out,
                        float* g_e1, float* g_e2, float* g_M, void* workspace, size_t workspace_bytes,
                        void* stream);

/* ---- path (iii): all-pairs similarity, CSLS, top-k, rank ----------------------------------- */

/* modules/finding/similarity.py:33-51.  INNER also serves 'cosine' (rows normalised first with
 * oea_rows_normalize).  L1 = 'manhattan' (1 − cityblock), L2 = 'euclidean' (1 − ‖a−b‖₂). */
enum { OEA_METRIC_INNER = 0, OEA_METRIC_L1 = 1, OEA_METRIC_L2 = 2 };

/* E1 [n1, pitch1], E2 [n2, pitch2]: row-major fp32, pitch % 4 == 0, columns >= dim are ZERO.
 * e1_t / e2_t: k-major copies of the operands made by oea_sim_transpose (ld*_t = oea_sim_transpose_ld(n)); the
 * 128×128 tile kernel streams them with 16-byte cp.async in a 3-stage pipeline. */
typedef struct oea_sim_cfg {
    int32_t metric;
    int32_t n1, n2, dim;
    int32_t pitch1, pitch2;
    const float* e1_t;
    const float* e2_t;
    int64_t ld1_t, ld2_t;
} oea_sim_cfg;

/* k-major, zero-padded copy of an operand: out [ceil16(pitch), oea_sim_transpose_ld(n)], out[k][r] = in[r][k]. */
int64_t oea_sim_transpose_ld(int32_t n);
size_t  oea_sim_transpose_bytes(int32_t n, int32_t pitch);
int     oea_sim_transpose(const float* in, int32_t pitch, int32_t n, float* out, void* stream);

/* Per-row k best columns of S (or of the CSLS matrix 2·S − row_off[i] − col_off[j] when the two
 * offset vectors are given; similarity.py:57-77), k <= 32, without materialising S.
 * out_val/out_idx [n1, k] sorted descending (ties: lower column first), out_mean [n1] = mean of the
 * k values (= calculate_nearest_k, similarity.py:80-83); each output may be NULL.
 * Replaces calculate_nearest_k (call with (E1,E2) for rows, (E2,E1) for columns),
 * search_nearest_k (bootstrapping/alignment_finder.py:66-76) and the top-k part of predict(). */
size_t oea_sim_topk_workspace_bytes(const oea_sim_cfg* cfg, int32_t k);
int oea_sim_topk(const oea_sim_cfg* cfg, const float* e1, const float* e2,
                 const float* row_off, const float* col_off, int32_t k,
                 float* out_val, int32_t* out_idx, float* out_mean,
                 void* workspace, size_t workspace_bytes, void* stream);

/* calculate_rank (modules/finding/alignment.py:146-168) without the sort: for every row i,
 * out_top1[i] = argmax_j S'_ij and out_rank[i] = 0-based rank of column gold[i] in descending order
 * (ties: lower column index first).  S' as above. */
size_t oea_sim_rank_workspace_bytes(const oea_sim_cfg* cfg);
int oea_sim_rank(const oea_sim_cfg* cfg, const float* e1, const float* e2,
                 const float* row_off, const float* col_off, const int32_t* gold,
                 int32_t* out_top1, int32_t* out_rank,
                 void* workspace, size_t workspace_bytes, void* stream);

/* Materialise S' into out [n1, ld_out] (sim(), similarity.py:11-54; BootEA.eval_ref_sim_mat,
 * approaches/bootea.py:214-219).  Also the first stage of the large-k neighbour search. */
int oea_sim_matrix(const oea_sim_cfg* cfg, const float* e1, const float* e2,
                   const float* row_off, const float* col_off, float* out, int64_t ld_out, void* stream);
/* oea_sim_matrix for the inner-product metric on the tensor cores (oea_sim_tc.cu): 3xTF32 wgmma with fp32 register
 * accumulators; values agree with oea_sim_matrix to fp32 round-off (not bit for bit: the summation order differs), which
 * is why it is opt-in (OEA_SIM_TC=1 in openea_b200.finding).  Takes the ROW-major operands (e1_t / e2_t are not read);
 * ld_out % 4 == 0.  OEA_ERR_KIND for other metrics. */
int oea_sim_matrix_tc(const oea_sim_cfg* cfg, const float* e1, const float* e2, const float* row_off, const float* col_off,
                      float* out, int64_t ld_out, void* stream);

/* CSLS on a MATERIALISED similarity matrix (from oea_sim_matrix): used when n1·n2·4 B fits in memory, so the
 * contraction runs once instead of three times (similarity.py:57-83, alignment.py:146-168).
 *   oea_matrix_topk_mean: mean of the k (<= 32) largest entries of every row (by_column = 0) or every column
 *                         (by_column = 1) of mat [n_rows, ld] → out_mean [n_rows] / [n_cols]  (= calculate_nearest_k);
 *                         the column form keeps per-row-split partial lists in `workspace` (size from
 *                         oea_matrix_topk_mean_workspace_bytes; the row form needs none);
 *   oea_matrix_rank     : per row arg-max and 0-based rank of column gold[i] of 2·S − row_off[i] − col_off[j]
 *                         (offsets NULL → of S itself); ties: lower column first. */
size_t oea_matrix_topk_mean_workspace_bytes(int32_t n_rows, int32_t n_cols, int32_t k, int32_t by_column);
int oea_matrix_topk_mean(const float* mat, int64_t ld, int32_t n_rows, int32_t n_cols, int32_t k,
                         int32_t by_column, float* out_mean, void* workspace, size_t workspace_bytes, void* stream);
int oea_matrix_rank(const float* mat, int64_t ld, int32_t n_rows, int32_t n_cols, const float* row_off,
                    const float* col_off, const int32_t* gold, int32_t* out_top1, int32_t* out_rank, void* stream);

/* Hits@k counts and rank sums of a 0-based rank vector in one launch (the NumPy reductions of
 * greedy_alignment, alignment.py:55-69): out[i] = #{rank < top_k_host[i]} for i < n_top (<= 8),
 * out[n_top] = Σ(rank+1), out[n_top+1] = Σ 1/(rank+1); device fp64 [n_top + 2], zeroed here. top_k_host is a HOST array. */
int oea_rank_stats(const int32_t* rank, int32_t n, const int32_t* top_k_host, int32_t n_top, double* out, void* stream);

/* sklearn.preprocessing.normalize (similarity.py:30-32) with the rule of scikit-learn >= 1.0: rows scaled to unit L2
 * norm, except that a row whose fp32 norm is below 10·FLT_EPSILON (a zero row, or a non-zero row whose squared norm
 * underflows) is copied unchanged; writes zero padding up to out_pitch. */
int oea_rows_normalize(const float* in, int32_t in_pitch, int32_t n, int32_t dim, float* out, int32_t out_pitch,
                       void* stream);

/* Per-row k LARGEST entries of a materialised matrix, large k (the ε-truncated neighbour search,
 * modules/train/batch.py:157-165: np.argpartition(-sim, k)[:k]).  The set is the first k columns by (value
 * descending, column ascending): of the columns tied at the k-th value the lowest-index ones are taken.  Each row of
 * out_idx [n_rows, k] lists that set in ascending column order, as col_ids[column] (col_ids == NULL → the column
 * index itself); the output is deterministic.  oea_rows_gather_sort orders it by value. */
int oea_rows_select_topk(const float* mat, int64_t ld, int32_t n_rows, int32_t n_cols, int32_t k,
                         const int32_t* col_ids, int32_t* out_idx, void* stream);

/* ---- path (ii): sparse adjacency × dense embeddings (GCN-Align / AliNet / RDGCN aggregation) -------- */

/* CSR matrix: int32 column indices, fp32 values (the tf.SparseTensor supports of gcn_align.py:575-578). */
typedef struct oea_csr {
    const int32_t* rowptr;   /* [n_rows + 1] */
    const int32_t* col;      /* [nnz] */
    const float*   val;      /* [nnz] */
    int32_t        n_rows, n_cols;
    int64_t        nnz;
} oea_csr;

/* Hub rows of a CSR matrix (more than oea_spmm_long_row_threshold() non-zeros; Zipf-degree entities) cut into
 * segments of oea_spmm_segment_nnz() non-zeros, prepared once on the host:
 *   long_rows [n_long] row ids; seg_ptr [n_long + 1] first segment of every hub row; for every segment
 *   seg_row [n_seg] = index into long_rows and seg_start [n_seg] = its first non-zero (absolute position). */
typedef struct oea_spmm_hubs {
    const int32_t* long_rows;
    const int32_t* seg_ptr;
    const int32_t* seg_row;
    const int32_t* seg_start;
    int32_t        n_long, n_seg;
} oea_spmm_hubs;

/* Y[n_rows, d] = A · X[n_cols, d] (+ beta·Y), optional fused epilogues: relu (the `act` of GraphConvolution,
 * gcn_align.py:259-267) or masking by mask_src > 0 (relu backward).  Replaces tf.sparse_tensor_dense_matmul
 * (gcn_align.py:83, alinet.py:581, rdgcn.py:187).  d % 4 == 0, d <= 512.  Rows with at most the threshold run
 * one warp each; hub rows go segment by segment through `workspace` (>= oea_spmm_workspace_bytes(n_seg, d))
 * and are summed in order (deterministic).  With hubs NULL (or n_long == 0) every row runs one warp each, whatever
 * its length: correct, but a hub row then sets the kernel's critical path.
 * The backward pass is the same call on the CSR of Aᵀ. */
int oea_spmm_long_row_threshold(void);
int oea_spmm_segment_nnz(void);
size_t oea_spmm_workspace_bytes(int32_t n_segments, int32_t d);
int oea_spmm_csr(const oea_csr* A, const oea_spmm_hubs* hubs,
                 const float* X, int32_t ldx, float* Y, int32_t ldy, int32_t d,
                 int32_t relu, const float* mask_src, float beta,
                 void* workspace, size_t workspace_bytes, void* stream);

/* Edge-softmax attention over a sparse neighbourhood (AliNetGraphAttentionLayer.call, approaches/alinet.py:656-677;
 * same shape in rdgcn.py:202-215):  alpha_e = softmax over the non-zeros of row i of leaky_relu(a_e·(s1[i] + s2[col e]))
 * (replaces adj*s1, adj*s2ᵀ, tf.sparse_add, tf.nn.leaky_relu, tf.sparse_softmax).  alpha [nnz] is in A's CSR order;
 * the aggregation Σ alpha·M is oea_spmm_csr with alpha as the values.
 * Edge-logit mode (s1 == s2 == NULL): A->val[e] is itself the pre-activation logit of edge e (RDGCN's
 * add_sparse_att_layer, rdgcn.py:202-215: logit_e = dual_transform[relation of e]); in the backward ds1 is then a
 * per-EDGE array [nnz] = d loss / d A->val[e] and ds2 is unused. */
int oea_edge_softmax_fwd(const oea_csr* A, const float* s1, const float* s2, float slope, float* alpha, void* stream);
/* out[e] = <G[row e, :d], M[col e, :d]> on A's pattern (d alpha of the aggregation). */
int oea_sddmm(const oea_csr* A, const float* G, int32_t ldg, const float* M, int32_t ldm, int32_t d, float* out, void* stream);
/* Backward of oea_edge_softmax_fwd: ds1 [n_rows] is written, ds2 [n_cols] is ACCUMULATED into (caller zeroes it). */
int oea_edge_softmax_bwd(const oea_csr* A, const float* s1, const float* s2, float slope, const float* alpha,
                         const float* dalpha, float* ds1, float* ds2, void* stream);

/* align_loss (approaches/gcn_align.py:298-320; rdgcn.py:293-315 has the same form): L1 margin loss over t
 * seed pairs with k negatives per side, mean over 2·k·t, forward + backward.  x [N, ld] are the output
 * embeddings; neg_left/neg_right/neg2_left/neg2_right are [t·k] row ids; *loss_out += loss;
 * grad [N, ld] += d loss / d x (caller zeroes it). */
int oea_align_loss_l1(const float* x, int32_t ld, int32_t dim, const int32_t* left, const int32_t* right, int32_t t,
                      int32_t k, const int32_t* neg_left, const int32_t* neg_right,
                      const int32_t* neg2_left, const int32_t* neg2_right, float gamma,
                      double* loss_out, float* grad, void* stream);

/* ---- path (i) across GPUs (SURVEY section 8e; the reference is single-device: models/basic_model.py:211-236 keeps the
 * seed entities coherent simply by training both KGs' triples in one session) ---------------------------------------
 * Exception to "never allocate": an exchange window must be a whole cudaMalloc allocation to be IPC-exportable, so
 * the library creates and frees it.  create/open/close/destroy and oea_seed_xchg_status are synchronous host calls;
 * pack/unpack/push/pull are asynchronous on `stream`. */
size_t oea_seed_xchg_window_bytes(int32_t world, int32_t max_rows, int32_t pitch);
int oea_p2p_window_create(size_t bytes, void** dev_ptr, void* handle_out64);   /* zero-filled; 64-byte IPC handle out */
int oea_p2p_window_open(const void* handle64, void** peer_ptr);                /* maps a peer's window (lazy peer access) */
int oea_p2p_window_close(void* peer_ptr);
int oea_p2p_window_destroy(void* dev_ptr);
/* Publish this rank's owned rows of `weight` as epoch `epoch` (>= 1, increasing by 1 per call) into every peer's window:
 * one kernel, 128-bit stores over NVLink + a release flag per peer.  No library collective is involved. */
int oea_seed_push(const oea_seed_xchg* x, const float* weight, uint64_t epoch, void* stream);
/* Wait (on the device, at most timeout_ns) until every peer has published `epoch`, then copy the received rows into
 * `weight` (rows owned by this rank are left alone).  A timeout sets the status word instead of hanging. */
int oea_seed_pull(const oea_seed_xchg* x, float* weight, uint64_t epoch, uint64_t timeout_ns, void* stream);
int oea_seed_xchg_status(const oea_seed_xchg* x, int32_t* status_host);        /* 0 = ok, 1 = a pull timed out */
/* The same exchange around a library all-gather (fallback where peer mapping is unavailable): own rows -> contiguous
 * send buffer, and [world, max_rows, pitch] receive buffer -> table rows (skipping `rank`'s own slot). */
int oea_seed_pack(const float* weight, int32_t pitch, const int32_t* ids, int32_t n, float* out, void* stream);
int oea_seed_unpack(float* weight, int32_t pitch, const float* recv, const int32_t* slot_ids, int32_t world,
                    int32_t max_rows, int32_t rank, void* stream);

/* ---- f-4: stable alignment (modules/finding/alignment.py:87-133 stable_alignment, :171-224 galeshapley) ----------
 * Suitor-proposing deferred acceptance over K3's top-`cut` lists: pref_idx / pref_val [n1, cut] are oea_sim_topk's
 * outputs (descending similarity; the reviewer side ranks suitors by the same similarities, ties → lower suitor index).
 * match[s] = reviewer held by suitor s, or -1.  At most max_rounds proposal rounds (the reference passes cut).
 * SYNCHRONOUS: the round loop polls a device counter; *rounds_host (optional) receives the rounds run. */
/* Turns oea_rows_select_topk's unordered per-row sets (k <= 128) into preference lists: val[r, :] = mat[r, idx[r, :]]
 * sorted descending (equal values: lower column first), idx permuted alongside (in place). */
int oea_rows_gather_sort(const float* mat, int64_t ld, int32_t n_rows, int32_t k, int32_t* idx, float* val, void* stream);
size_t oea_gale_shapley_workspace_bytes(int32_t n1, int32_t n2);
int oea_gale_shapley(const int32_t* pref_idx, const float* pref_val, int32_t n1, int32_t n2, int32_t cut,
                     int32_t max_rounds, int32_t* match, void* workspace, size_t workspace_bytes,
                     int32_t* rounds_host, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* OEA_H_ */
