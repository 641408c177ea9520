/* kgrec_b200.h -- C ABI of the H100 (sm_90a) scoring engine for joint KG +
 * recommendation models (TransE / TransH / TransR / TUP / KTUP).
 *
 * The reference (TaoMiner/joint-kg-recommender) is pure Python on PyTorch and
 * has no FFI of its own: its "plugin boundary" for this path is the duck-typed
 * nn.Module protocol of jTransUP/models/{transE,transH,transR,transUP,jTransUP}.py
 * (SURVEY.md section 8b).  Each entry point below replaces the chain of stock
 * torch ops behind one of those methods; the citation on each says which.
 * The Python mirror of the reference classes (joint-kg-recommender_b200/kgrec_b200)
 * binds this header with ctypes -- see INTEGRATION.md.
 *
 * Conventions
 *  - every pointer is a DEVICE pointer unless the name ends in _host;
 *  - tables are fp32 row-major [rows, ld] with ld >= dim (floats);
 *  - index arrays are int32 or int64 (idx_bytes = 4 | 8), as the reference's
 *    drivers pass torch.LongTensor (knowledge_representation.py:179-184);
 *  - all work is enqueued on `stream` (a cudaStream_t); nothing synchronises;
 *  - return value: KGREC_OK or an error code; kgrec_last_error() has the text;
 *  - there is no CPU fallback anywhere behind this header.
 */
#ifndef KGREC_B200_H_
#define KGREC_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KGREC_ABI_VERSION 2

typedef void* kgrec_stream_t; /* cudaStream_t */

enum {
  KGREC_OK = 0,
  KGREC_ERR_INVALID = 1,     /* bad argument (null table, dim, alignment ...)   */
  KGREC_ERR_UNSUPPORTED = 2, /* shape outside what the kernels are built for   */
  KGREC_ERR_CUDA = 3         /* a CUDA runtime call failed                     */
};

/* -model_type values on the hot path (jTransUP/models/base.py:23-25). */
enum {
  KGREC_TRANSE = 0, /* transE.py   score = L(E[h] + R[r] - E[t])                         */
  KGREC_TRANSH = 1, /* transH.py   hyperplane projection by Norm[r] (misc.py:18-19)      */
  KGREC_TRANSR = 2, /* transR.py   d x d matrix Proj[r] (misc.py:21-26)                  */
  KGREC_TUP = 3,    /* transUP.py  user/item + preference induction (transUP.py:105-115) */
  KGREC_KTUP = 4    /* jTransUP.py rec branch (jTransUP.py:124-143); its KG branch is
                       KGREC_TRANSH on the same tables                                   */
};

enum { KGREC_LOSS_MARGIN = 0, /* utils/loss.py:8-16  sum max(pos-neg+margin,0)        */
       KGREC_LOSS_BPR = 1 };  /* utils/loss.py:29-31 mean -logsigmoid(target*(pos-neg)) */

enum { KGREC_SIDE_HEAD = 0,   /* evaluateHead: c = proj(E[t]) - R[r]                    */
       KGREC_SIDE_TAIL = 1,   /* evaluateTail: c = proj(E[h]) + R[r]                    */
       KGREC_SIDE_REC = 2 };  /* evaluate / evaluateRec: users against all items        */

/* The embedding tables of one model instance (the nn.Embedding weights the
 * reference classes own: transE.py:36-40, transH.py:39-45, transR.py:45-51,
 * transUP.py:46-60, jTransUP.py:64-103).  Unused tables are NULL. */
typedef struct kgrec_tables {
  int32_t dim;        /* embedding_size d                                        */
  int32_t ld;         /* leading dimension of every [rows, d] table, in floats   */
  int32_t l1;         /* L1_flag: 1 -> sum|e|, 0 -> sum e^2 (no sqrt)            */
  int32_t use_gumbel; /* use_st_gumbel (TUP / KTUP)                              */
  int64_t n_ent;      /* rows of ent (KTUP: entity_total + 1, last = zero pad)   */
  int64_t n_rel;
  int64_t n_user;
  int64_t n_item;
  int32_t n_pref;     /* preference_total P (KTUP: == n_rel)                     */
  int32_t reserved;
  const float* ent;        /* [n_ent, ld]                                        */
  const float* rel;        /* [n_rel, ld]                                        */
  const float* norm;       /* [n_rel, ld]     TransH, KTUP                       */
  const float* proj;       /* [n_rel, d*d]    TransR, row-major M[a,b]           */
  const float* user;       /* [n_user, ld]                                       */
  const float* item;       /* [n_item, ld]                                       */
  const float* pref;       /* [n_pref, ld]                                       */
  const float* pref_norm;  /* [n_pref, ld]                                       */
  const int32_t* item2ent; /* [n_item] KTUP item -> aligned entity row, unaligned
                              items map to the padding row n_ent-1: the device form
                              of paddingItems (jTransUP.py:114-120)               */
} kgrec_tables;

/* Where the backward kernels put row gradients.
 * mode 0 "slots": one gradient row per gathered row, laid out in gather order --
 *         the value array of an (uncoalesced) sparse COO gradient whose indices
 *         are the input id arrays themselves.  ent: [2n, d] (head slots then tail
 *         slots; KTUP: [n, d] aligned-entity slots), rel / norm / user / item: [n, d].
 * mode 1 "dense": atomically accumulated into caller-zeroed [rows, d] buffers,
 *         the layout the reference's autograd produces (param.grad).
 * proj, pref, pref_norm are always accumulated densely ([n_rel, d*d], [P, d]).
 * For KTUP the gradient of rel / norm equals that of pref / pref_norm
 * (jTransUP.py:253-258) and is written once, to pref / pref_norm. */
typedef struct kgrec_grads {
  int32_t mode;
  int32_t reserved;
  float* ent;
  float* rel;
  float* norm;
  float* proj;
  float* user;
  float* item;
  float* pref;
  float* pref_norm;
} kgrec_grads;

int kgrec_abi_version(void);
const char* kgrec_last_error(void);
/* number of SMs the library sized its grids for on the current device */
int kgrec_sm_count(void);

/* ---- training path ------------------------------------------------------ */

/* model.forward: transE.py:51-63, transH.py:58-71, transR.py:65-78,
 * transUP.py:69-82, jTransUP.py:122-161.
 * KG models: a = h, b = t, c = r.   TUP / KTUP: a = u, b = i, c = NULL.
 * gumbel_u: [n, P] uniform draws for the ST Gumbel-softmax (transUP.py:159-161)
 * or NULL -> drawn in-kernel from Philox4x32-10 keyed by `seed` (only read when
 * tables->use_gumbel).  status (optional, int32[1]) is set non-zero when an
 * index is out of range. */
int kgrec_score_fwd(const kgrec_tables* tables, int model,
                    const void* a, const void* b, const void* c, int idx_bytes, int64_t n,
                    const float* gumbel_u, uint64_t seed,
                    float* scores, int32_t* status, kgrec_stream_t stream);

/* The autograd of the above (reference: losses.backward(),
 * knowledge_representation.py:207): given dLoss/dscore [n] emits row gradients. */
int kgrec_score_bwd(const kgrec_tables* tables, int model,
                    const void* a, const void* b, const void* c, int idx_bytes, int64_t n,
                    const float* gumbel_u, uint64_t seed,
                    const float* grad_scores, const kgrec_grads* grads,
                    kgrec_stream_t stream);

/* Fused positive + sampled-negative scoring with the ranking loss:
 * pos = model(pos ids); neg = model(neg ids); marginLoss / bprLoss
 * (knowledge_representation.py:189-195, item_recommendation.py:171-175).
 * Positive j owns negatives [j*n_neg, (j+1)*n_neg).  The loss is reduced per
 * batch of `batch_pos` positives: loss[b], b < ceil(n_pos / batch_pos) --
 * margin: sum over the batch's pairs; bpr: mean over them.
 * gumbel_u (optional): [n_pos + n_pos*n_neg, P], positives first.
 * workspace: >= kgrec_rank_loss_workspace_bytes(n_pos) bytes. */
int64_t kgrec_rank_loss_workspace_bytes(int64_t n_pos);
int kgrec_rank_loss_fwd(const kgrec_tables* tables, int model,
                        const void* pa, const void* pb, const void* pc,
                        const void* na, const void* nb, const void* nc,
                        int idx_bytes, int64_t n_pos, int32_t n_neg, int64_t batch_pos,
                        int loss_kind, float margin_or_target,
                        const float* gumbel_u, uint64_t seed,
                        float* pos_scores, float* neg_scores, float* loss,
                        void* workspace, int32_t* status, kgrec_stream_t stream);

/* Backward of kgrec_rank_loss_fwd from the saved scores: the per-score
 * coefficients dLoss/dscore are formed in-kernel (loss.py:16, 30-31), scaled by
 * grad_loss (host scalar) times grad_loss_dev[batch] (optional device array, one
 * upstream value per loss batch), and the row gradients written as in
 * kgrec_score_bwd with the positives' slots first: slot arrays are sized for
 * n = n_pos * (1 + n_neg). */
int kgrec_rank_loss_bwd(const kgrec_tables* tables, int model,
                        const void* pa, const void* pb, const void* pc,
                        const void* na, const void* nb, const void* nc,
                        int idx_bytes, int64_t n_pos, int32_t n_neg, int64_t batch_pos,
                        int loss_kind, float margin_or_target,
                        const float* gumbel_u, uint64_t seed,
                        const float* pos_scores, const float* neg_scores, float grad_loss,
                        const float* grad_loss_dev, const kgrec_grads* grads, kgrec_stream_t stream);

/* kgrec_rank_loss_fwd + kgrec_rank_loss_bwd(grad_loss) as ONE call: scores, per-batch losses
 * and the row gradients of grad_loss * sum_b loss[b] -- what a training step of
 * item_recommendation.py:165-181 / knowledgable_recommendation.py needs from the model.
 * TUP / KTUP pairs are scored, differentiated and reduced in a single kernel pass when a
 * positive and its negatives fit one warp's rows (n_neg <= 15, embedding_size <= 128,
 * preference_total <= 32); other shapes and models run the two kernels back to back.
 * Gradient slots as in kgrec_rank_loss_bwd.
 * slot_user_ids / slot_item_ids / slot_ent_ids (optional, int64 [n_pos * (1 + n_neg)], TUP / KTUP
 * only, ent for KTUP): the table row of every gradient slot, i.e. the index arrays of the sparse COO
 * gradients, written by the same pass. */
int kgrec_rank_loss_step(const kgrec_tables* tables, int model,
                         const void* pa, const void* pb, const void* pc,
                         const void* na, const void* nb, const void* nc,
                         int idx_bytes, int64_t n_pos, int32_t n_neg, int64_t batch_pos,
                         int loss_kind, float margin_or_target, float grad_loss,
                         const float* gumbel_u, uint64_t seed,
                         float* pos_scores, float* neg_scores, float* loss,
                         const kgrec_grads* grads,
                         int64_t* slot_user_ids, int64_t* slot_item_ids, int64_t* slot_ent_ids,
                         void* workspace, int32_t* status, kgrec_stream_t stream);

/* The same fused ranking loss in the group-compact negative format (TransE / TransH and the
 * KTUP KG branch).  The reference draws a negative by corrupting the head OR the tail of its
 * positive (utils/data.py:12-56), so negative k of positive j is one int32:
 *     corrupt[j*n_neg + k] >= 0 : (h_j, r_j, corrupt)      tail replaced
 *     corrupt[j*n_neg + k] <  0 : (~corrupt, r_j, t_j)     head replaced
 * Scores and losses equal kgrec_rank_loss_fwd on the expanded triples.  The backward reads
 * (3 + n_neg) rows per group and writes (3 + n_neg) gradient rows, accumulating the shared
 * rows' gradients in registers.  Slot layout (grads->mode 0): ent [n_pos * (2 + n_neg), d],
 * per group: head, tail, corrupted_1 .. corrupted_K; rel and norm [n_pos, d]. */
int kgrec_corrupt_loss_fwd(const kgrec_tables* tables, int model,
                           const void* ph, const void* pt, const void* pr, int idx_bytes, int64_t n_pos,
                           const int32_t* corrupt, int32_t n_neg, int64_t batch_pos,
                           int loss_kind, float margin_or_target,
                           float* pos_scores, float* neg_scores, float* loss,
                           void* workspace, int32_t* status, kgrec_stream_t stream);
int kgrec_corrupt_loss_bwd(const kgrec_tables* tables, int model,
                           const void* ph, const void* pt, const void* pr, int idx_bytes, int64_t n_pos,
                           const int32_t* corrupt, int32_t n_neg, int64_t batch_pos,
                           int loss_kind, float margin_or_target,
                           const float* pos_scores, const float* neg_scores, float grad_loss,
                           const float* grad_loss_dev, const kgrec_grads* grads,
                           int64_t* slot_ent_ids, int64_t* slot_rel_ids,   /* optional, as in kgrec_corrupt_loss_step */
                           kgrec_stream_t stream);

/* Forward + loss + backward of the group-compact ranking loss in ONE pass: scores, per-batch
 * losses and the row gradients of grad_loss * sum_b loss[b] (every reference driver calls
 * backward() on the loss itself, knowledge_representation.py:207, so the upstream is a known
 * scalar).  One gather of (3 + n_neg) rows and (3 + n_neg) gradient rows per group; outputs
 * and slot layout as kgrec_corrupt_loss_fwd / _bwd.
 * slot_ent_ids [n_pos * (2 + n_neg)] / slot_rel_ids [n_pos] (optional, int64): the table row of every
 * gradient slot, i.e. the index array of the sparse COO gradient whose values the slots are
 * (torch.sparse_coo_tensor(ids, slots)); written by the same pass so that no host-side index
 * building is left in a training step.
 * reg_flags = 1 adds the KG drivers' regularisers to each batch loss and to the gradients
 * (knowledge_representation.py:197-204): normLoss (loss.py:21-23) over the entity rows of
 * cat[ph, pt, nh, nt] and the relation rows of cat[pr, nr], and for TransH orthogonalLoss
 * (loss.py:18-19) over (rel, norm) rows of cat[pr, nr] -- every row with the multiplicity it has in
 * those lists.  Margin loss and embedding_size <= 128 only; reg_flags other than 0 / 1 is
 * KGREC_ERR_INVALID, reg_flags 1 with the BPR loss KGREC_ERR_UNSUPPORTED.
 * KGREC_TRANSR is accepted by this entry point as well (embedding_size <= 128, n_neg <= 14,
 * reg_flags 0 or 1; normLoss over the raw ent / rel rows as above, none on proj, as the
 * reference): the relation's d x d matrix is read twice per GROUP and its gradient
 * (grads->proj, always a dense [n_rel, d*d] accumulate) added once per group; the groups are
 * visited in relation order (a counting sort of pr inside the call) so that a CTA's warps share M_r.
 * workspace: >= kgrec_corrupt_loss_step_workspace_bytes(tables, model, n_pos) bytes. */
int64_t kgrec_corrupt_loss_step_workspace_bytes(const kgrec_tables* tables, int model, int64_t n_pos);
int kgrec_corrupt_loss_step(const kgrec_tables* tables, int model,
                            const void* ph, const void* pt, const void* pr, int idx_bytes, int64_t n_pos,
                            const int32_t* corrupt, int32_t n_neg, int64_t batch_pos,
                            int loss_kind, float margin_or_target, float grad_loss, int32_t reg_flags,
                            float* pos_scores, float* neg_scores, float* loss,
                            const kgrec_grads* grads, int64_t* slot_ent_ids, int64_t* slot_rel_ids,
                            void* workspace, int32_t* status, kgrec_stream_t stream);

/* ---- device-side negative sampling (SURVEY 8f, next row 2) --------------------------------
 * The reference draws negatives with per-triple Python rejection loops (utils/data.py:12-85).
 * Known triples / ratings are 64-bit keys in an open-addressing hash set in HBM:
 *   triple key  = (h * n_rel + r) * n_ent + t        rating key = u * n_item + i
 * Draws are Philox4x32-10 keyed by (seed, negative index, attempt): reproducible per seed. */
int64_t kgrec_hashset_capacity(int64_t n_keys);        /* power of two >= 2 n_keys */
int kgrec_hashset_build(const uint64_t* keys, int64_t n, uint64_t* table, int64_t capacity,
                        kgrec_stream_t stream);
/* getTrainTripleBatch + corrupt_head/tail_filter (data.py:12-56): n_neg negatives per positive,
 * head or tail with probability 1/2, uniform entity, redrawn while equal to the original or a
 * known triple (table == NULL: unfiltered).  Output: the group-compact int32 format of
 * kgrec_corrupt_loss_* (>= 0 tail replaced, < 0 head replaced by ~value).  After 64 rejected draws
 * the kernel scans on from the last draw for the first valid id (the reference would keep drawing);
 * if a key has NO valid negative (where the reference never returns) the last draw is emitted and
 * *status (optional int32[1]) is set to 2. */
int kgrec_sample_corrupt(const void* ph, const void* pt, const void* pr, int idx_bytes, int64_t n_pos,
                         int32_t n_neg, int64_t n_ent, int64_t n_rel,
                         const uint64_t* table, int64_t capacity, uint64_t seed,
                         int32_t* corrupt, int32_t* status, kgrec_stream_t stream);
/* getNegRatings (data.py:64-85): n_neg negative items per (user, positive item), uniform,
 * redrawn while equal to the positive or a known item of the user. */
int kgrec_sample_neg_items(const void* u, const void* pi, int idx_bytes, int64_t n, int32_t n_neg,
                           int64_t n_item, const uint64_t* table, int64_t capacity, uint64_t seed,
                           int32_t* neg_items, int32_t* status, kgrec_stream_t stream);

/* ---- sparse-row optimizer (SURVEY 8f, next row 1) -----------------------------------------
 * Replaces the reference's dense optimizer step and clip_grad_norm (utils/trainer.py:63-81,
 * knowledge_representation.py:213; item_recommendation.py:189-192;
 * knowledgable_recommendation.py:398-402) at a cost proportional to the rows the batch touched.
 * Gradients sit in persistent dense accumulators the training kernels wrote with grads->mode 1
 * (all-zero outside a step).  The rows a step touched carry an epoch mark (marks[row] == epoch,
 * int32 [rows], never cleared: the caller bumps the epoch every step); marks == NULL means every
 * row (the small tables: pref / pref_norm / proj, KTUP's rel / norm).  Up to 8 tables per call,
 * one launch for all of them. */
typedef struct kgrec_opt_table {
  float* table;          /* [rows, dim] parameters (contiguous)                                */
  float* acc;            /* [rows, dim] accumulated gradient, zeroed again by kgrec_rows_update */
  float* state1;         /* Adagrad sum / Adam m, or NULL (SGD)                                */
  float* state2;         /* Adam v, or NULL                                                    */
  const int32_t* marks;  /* [rows] epoch marks, or NULL = all rows                             */
  int64_t rows;
  int32_t dim;
  int32_t keep_acc;      /* 1: leave acc as it is (an entry of a LATER call shares it and clears  */
                         /* it).  An update call refuses entries whose accumulators overlap when  */
                         /* one of them clears its own: the other could read it already cleared   */
  int32_t vec;           /* set by the library (128-bit path usable)                           */
  int32_t reserved;
} kgrec_opt_table;

/* One id array of the batch and the mark array of the table it indexes. */
typedef struct kgrec_mark_seg {
  const void* ids;       /* n ids, idx_bytes wide                                              */
  int64_t n;
  int32_t idx_bytes;
  int32_t compact;       /* 1: group-compact corrupted ids (v < 0 names entity ~v)             */
  const int32_t* remap;  /* optional [n_remap] lookup applied first (KTUP: item2ent)           */
  int64_t n_remap;
  int32_t* marks;        /* [rows]                                                             */
  int64_t rows;
} kgrec_mark_seg;

/* marks[id] = epoch for every id of every segment (<= 8 segments, one launch).  An id is first
 * decoded (compact: v < 0 names ~v), then remapped, then range-checked.  An out-of-range id (of the
 * remap, or of the table) marks row 0 -- where the training kernels clamp it and send its gradient --
 * and sets *status (optional int32[1]) to 1; a call with every id in range leaves *status as it is. */
int kgrec_rows_mark(const kgrec_mark_seg* segs_host, int n_segs, int32_t epoch, int32_t* status,
                    kgrec_stream_t stream);
/* adds to *sqnorm the squared L2 norm of the marked accumulator rows of all tables:
 * clip_grad_norm's total norm */
int kgrec_rows_sqnorm(const kgrec_opt_table* tabs_host, int n_tabs, int32_t epoch, float* sqnorm,
                      kgrec_stream_t stream);
/* one optimizer update of every marked row, then its acc row is cleared.  kind 0 SGD, 1 Adagrad
 * (state1 = sum), 2 Adam on the touched rows (state1 = m, state2 = v, step = 1-based count).
 * sqnorm (optional, device): gradients are scaled by min(1, max_norm / (sqrt(*sqnorm) + 1e-6))
 * as clip_grad_norm does. */
int kgrec_rows_update(const kgrec_opt_table* tabs_host, int n_tabs, int32_t epoch, int kind, float lr,
                      float eps, float beta1, float beta2, int64_t step, float weight_decay,
                      const float* sqnorm, float max_norm, kgrec_stream_t stream);

/* ---- row-factored training step of the rec models (TUP / KTUP): soft preferences, or ST-Gumbel with the L2 score ----
 * transUP.py:69-82, 105-115; jTransUP.py:122-161, 250-260.  With raw logits as mixing weights r = RA_u + RA_i and
 * w = WB_u + WB_i with RA_x = hf (x P'^T / 2) P' (WB_x with N'): the [P x d] contractions are done once per DISTINCT
 * row of the step (rows carrying the epoch mark: kgrec_rows_mark must have run on the step's user / item ids with
 * this epoch) instead of once per pair; the pair kernel is O(d).  Positives (pu, pi), negatives ni [n_pos, n_neg]
 * (the user is shared: getNegRatings, utils/data.py:64-85).  Gradients are ADDED to the dense accumulators in `acc`
 * (grads->mode 1: user, item, pref, pref_norm [, ent]; the KTUP caller copies pref / pref_norm's to rel / norm);
 * scores and per-batch losses as kgrec_rank_loss_step.  workspace: kgrec_rec_rows_workspace_floats floats, persistent
 * across steps (first_use = 1 on the first call zero-fills its accumulators).  loss_workspace: n_pos floats.
 * norm_reg_loss (optional, TUP): adds the driver's normLoss over the batch's user rows and cat[pos, neg] item rows
 * (item_recommendation.py:177-179) -- value to *norm_reg_loss, gradient into the same accumulators -- inside the pair kernel.
 * tables->use_gumbel = 1 (squared-L2 score only): the arg-max preference per pair from per-row logit halves, dL/dp_k for
 * every k in O(1) from [P, P] Gram tables, the logit path per distinct row (csrc/train_rec_rows.cu); gumbel_u: optional
 * explicit uniforms [n_pos * (1 + n_neg), P] (positives first, then negatives), else Philox draws keyed by seed.
 * embedding_size % 4 == 0 and <= 128, preference_total <= 32, n_neg <= 31. */
int64_t kgrec_rec_rows_workspace_floats(int64_t n_user, int64_t n_item, int32_t dim, int32_t n_pref, int ktup);
int kgrec_rec_rows_step(const kgrec_tables* tables, int model, const void* pu, const void* pi, const void* ni,
                        int idx_bytes, int64_t n_pos, int32_t n_neg, int64_t batch_pos, int loss_kind,
                        float margin_or_target, float grad_loss, const int32_t* marks_user,
                        const int32_t* marks_item, int32_t epoch, float* workspace, int32_t first_use,
                        const kgrec_grads* acc, float* pos_scores, float* neg_scores, float* loss,
                        void* loss_workspace, float* norm_reg_loss, const float* gumbel_u, uint64_t seed,
                        int32_t* status, kgrec_stream_t stream);

/* ---- device-resident step state: training steps replayed from a CUDA graph -----------------------
 * A replayed graph re-uses every by-value argument it was captured with.  The scalars that change from
 * one training step to the next therefore live in device memory, in one kgrec_step_state, and the
 * `_dev` entry points below read them there instead of taking them by value.  Everything else about a
 * `_dev` call (validation, kernels, results) is that of the entry point it is named after.
 * A step runs:  kgrec_batch_gather  ->  kgrec_step_advance  ->  samplers / loss step / optimizer (_dev),
 * so inside a step `step` is the running step's 1-based count and `epoch` its mark epoch. */
typedef struct kgrec_step_state {
  int64_t step;          /* steps begun so far: Adam's step count t                               */
  uint64_t gumbel_seed;  /* Gumbel-noise seed of step s: gumbel_seed + s                          */
  uint64_t sample_seed;  /* negative-sampler seed of step s: sample_seed + s                      */
  int32_t epoch;         /* epoch mark of the running step (kgrec_rows_mark / _sqnorm / _update)  */
  float lr;              /* learning rate of kgrec_rows_update_dev                                */
} kgrec_step_state;

/* step += 1, epoch += 1, and *cursor += batch when cursor is not NULL (one thread). */
int kgrec_step_advance(kgrec_step_state* state, int64_t* cursor, int64_t batch, kgrec_stream_t stream);
/* out_host[c][j] = cols_host[c][order[*cursor + j]] for j < batch, c < n_cols (<= 4): the batch
 * DeviceTrainIterator cuts from its shuffled visiting order.  The cursor is only read: the
 * kgrec_step_advance that follows moves it (a kernel cannot read and move it without a grid barrier).
 * Positions past n_order and rows outside [0, n_rows) read row 0 and set *status (optional) to 1. */
int kgrec_batch_gather(const int64_t* order, int64_t n_order, const int64_t* cursor, const void* const* cols_host,
                       void* const* out_host, int n_cols, int idx_bytes, int64_t n_rows, int64_t batch,
                       int32_t* status, kgrec_stream_t stream);
/* kgrec_rows_mark / _sqnorm / _update with the epoch, the learning rate and Adam's step (bias terms
 * formed on the device) read from *state */
int kgrec_rows_mark_dev(const kgrec_mark_seg* segs_host, int n_segs, const kgrec_step_state* state, int32_t* status,
                        kgrec_stream_t stream);
int kgrec_rows_sqnorm_dev(const kgrec_opt_table* tabs_host, int n_tabs, const kgrec_step_state* state, float* sqnorm,
                          kgrec_stream_t stream);
int kgrec_rows_update_dev(const kgrec_opt_table* tabs_host, int n_tabs, const kgrec_step_state* state, int kind,
                          float eps, float beta1, float beta2, float weight_decay, const float* sqnorm,
                          float max_norm, kgrec_stream_t stream);

/* ---- exact torch.optim trajectories (utils/trainer.py:63-102) ------------------------------------
 * kgrec_rows_update with every rule of the reference's trainer and its dense row semantics.  Rules are
 * torch.optim's formulas; weight decay is added to the clipped gradient:
 *   kind 0 SGD      state1 = momentum buffer (momentum != 0):  buf = mu buf + g ; p -= lr buf
 *   kind 1 Adagrad  state1 = sum
 *   kind 2 Adam     state1 = m, state2 = v; the bias terms use step_counts[t], the step count of table t
 *                   of the call, which the call advances by one (in the stream, before the sweep) -- as
 *                   torch advances a parameter's step only when the parameter has a gradient
 *   kind 3 RMSprop  (centered = False) state1 = square_avg, state2 = momentum buffer (momentum != 0):
 *                   sq = alpha sq + (1 - alpha) g^2 ; p -= lr g / (sqrt(sq) + eps)  (or via the buffer)
 * rows: KGREC_ROWS_TOUCHED updates the marked rows (as kgrec_rows_update); KGREC_ROWS_ALL updates every
 * row of every table of the call, as torch.optim's dense step does: a marked row with its clipped
 * accumulator (then cleared), an unmarked row with gradient 0 (its accumulator is not read).  It costs
 * O(table) per call.  Plain SGD and Adagrad without weight decay leave a zero-gradient row bit-unchanged,
 * so for them ALL visits the marked rows only. */
enum { KGREC_ROWS_TOUCHED = 0, KGREC_ROWS_ALL = 1 };
typedef struct kgrec_opt_params {
  int32_t kind;          /* 0 SGD, 1 Adagrad, 2 Adam, 3 RMSprop                                    */
  int32_t rows;          /* KGREC_ROWS_TOUCHED | KGREC_ROWS_ALL                                    */
  float lr;              /* kgrec_rows_update_ex only (_ex_dev reads state->lr)                    */
  float eps;
  float beta1, beta2;    /* Adam                                                                   */
  float alpha;           /* RMSprop                                                                */
  float momentum;        /* SGD, RMSprop (0: no buffer)                                            */
  float weight_decay;
  float max_norm;        /* clip, when sqnorm is given                                             */
  int64_t* step_counts;  /* [n_tabs] int64 device counters, one per table of the call (Adam)       */
} kgrec_opt_params;
int kgrec_rows_update_ex(const kgrec_opt_table* tabs_host, int n_tabs, int32_t epoch, const kgrec_opt_params* params_host,
                         const float* sqnorm, kgrec_stream_t stream);
/* the same with the epoch and the learning rate read from *state (a CUDA-graph-capturable step) */
int kgrec_rows_update_ex_dev(const kgrec_opt_table* tabs_host, int n_tabs, const kgrec_step_state* state,
                             const kgrec_opt_params* params_host, const float* sqnorm, kgrec_stream_t stream);
/* the samplers with seed = state->sample_seed + state->step */
int kgrec_sample_corrupt_dev(const void* ph, const void* pt, const void* pr, int idx_bytes, int64_t n_pos,
                             int32_t n_neg, int64_t n_ent, int64_t n_rel, const uint64_t* table, int64_t capacity,
                             const kgrec_step_state* state, int32_t* corrupt, int32_t* status, kgrec_stream_t stream);
int kgrec_sample_neg_items_dev(const void* u, const void* pi, int idx_bytes, int64_t n, int32_t n_neg, int64_t n_item,
                               const uint64_t* table, int64_t capacity, const kgrec_step_state* state,
                               int32_t* neg_items, int32_t* status, kgrec_stream_t stream);
/* kgrec_rank_loss_step / kgrec_rec_rows_step with the Gumbel seed state->gumbel_seed + state->step
 * (read only when tables->use_gumbel and gumbel_u is NULL) and, for the row-factored step, the epoch
 * mark state->epoch */
int kgrec_rank_loss_step_dev(const kgrec_tables* tables, int model,
                             const void* pa, const void* pb, const void* pc,
                             const void* na, const void* nb, const void* nc,
                             int idx_bytes, int64_t n_pos, int32_t n_neg, int64_t batch_pos,
                             int loss_kind, float margin_or_target, float grad_loss,
                             const float* gumbel_u, const kgrec_step_state* state,
                             float* pos_scores, float* neg_scores, float* loss,
                             const kgrec_grads* grads,
                             int64_t* slot_user_ids, int64_t* slot_item_ids, int64_t* slot_ent_ids,
                             void* workspace, int32_t* status, kgrec_stream_t stream);
int kgrec_rec_rows_step_dev(const kgrec_tables* tables, int model, const void* pu, const void* pi, const void* ni,
                            int idx_bytes, int64_t n_pos, int32_t n_neg, int64_t batch_pos, int loss_kind,
                            float margin_or_target, float grad_loss, const int32_t* marks_user,
                            const int32_t* marks_item, const kgrec_step_state* state, float* workspace,
                            int32_t first_use, const kgrec_grads* acc, float* pos_scores, float* neg_scores,
                            float* loss, void* loss_workspace, float* norm_reg_loss, const float* gumbel_u,
                            int32_t* status, kgrec_stream_t stream);

/* ---- the drivers' recommendation-side regularisers (utils/loss.py:18-23) -------------------------
 * item_recommendation.py:177-180: normLoss(user rows) + normLoss(item rows of cat[pos, neg]) +
 * normLoss(pref table) + orthogonalLoss(pref, pref_norm); knowledgable_recommendation.py:343-344:
 * orthogonalLoss(pref, pref_norm).  Each adds scale * value to *loss_out (device float, optional)
 * and scale * gradient to the dense accumulators (optional) the sparse-row optimizer consumes.
 * (The KG drivers' terms over the triples' rows are fused into kgrec_corrupt_loss_step, reg_flags.) */
/* normLoss over table[ids[i]], i < n -- every listed occurrence counts; ids == NULL: rows 0..n-1 */
int kgrec_reg_norm_rows(const float* table, int64_t rows, int32_t dim, const void* ids, int idx_bytes,
                        int64_t n, float scale, float* loss_out, float* acc, int32_t* status,
                        kgrec_stream_t stream);
/* orthogonalLoss(rel, norm) = sum_rows (norm.rel)^2 / |rel|^2 over two whole [rows, dim] tables */
int kgrec_reg_orth_tables(const float* rel, const float* norm, int64_t rows, int32_t dim, float scale,
                          float* loss_out, float* acc_rel, float* acc_norm, kgrec_stream_t stream);

/* ---- full-catalog evaluation path ---------------------------------------- */
/* Common arguments of the three evaluation modes:
 *   model / side   which evaluate* method: KG sides score query (t,r) / (h,r) pairs against
 *                  entities (transE.py:65-105, transH.py:73-121, jTransUP.py:193-247), the
 *                  rec side scores users against items (transUP.py:84-102, jTransUP.py:163-191).
 *   q, r           query ids (tail ids for SIDE_HEAD, head ids for SIDE_TAIL, user ids for
 *                  SIDE_REC) and relation ids (KG sides), nq of them.
 *   qvec           optional explicit query vectors [nq, 2*dim] = (c | w) replacing q / r on
 *                  the KG sides: c = proj(E[q]) -/+ R[r] (transE.py:68-71, transH.py:76-82)
 *                  and the hyperplane normal w.  Required for KGREC_TRANSR, whose catalog
 *                  must already be projected by the relation matrix (misc.py:29-33).
 *   cat, cat_ld, n_cat   the catalog (shard): n_cat contiguous rows of the entity / item
 *                  table (KTUP rec side: the table built by kgrec_ktup_item_table), 16-byte
 *                  aligned, cat_ld % 4 == 0.
 *   id_base        global id of catalog row 0 (shards of a row-partitioned table).
 *   cat_ids        (kgrec_eval_scores, KG sides) optional explicit global id of every catalog
 *                  row, for gathered sub-catalogs (the reference's all_e_ids); a pair's score
 *                  is bit-identical wherever the row sits, given its id.
 *   gumbel_u       rec side with use_gumbel: optional explicit uniform draws
 *                  [nq, n_cat, P] (transUP.py:159-161); NULL -> counter-hash draws from seed. */

/* evaluateHead / evaluateTail / evaluate / evaluateRec producing the full [nq, n_cat]
 * score matrix the unchanged drivers consume.  out has leading dimension ld_out >= n_cat. */
int kgrec_eval_scores(const kgrec_tables* tables, int model, int side,
                      const void* q, const void* r, int idx_bytes, const float* qvec, int64_t nq,
                      const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base,
                      const int32_t* cat_ids, const float* gumbel_u, uint64_t seed,
                      float* out, int64_t ld_out, kgrec_stream_t stream);

/* The same scores reduced on chip to the K best (smallest) per query, replacing the D2H
 * copy + np.argsort walk of utils/misc.py:125-146, 213-229.  Ordering is (score, id)
 * lexicographic.  filter_ptr / filter_ids: optional CSR (ptr [nq+1], ascending global ids)
 * of catalog ids to skip per query (train + other eval files' positives,
 * item_recommendation.py:108-111).  out_keys: [nq, k] uint64 = score bits << 32 | global id,
 * ascending; unused places hold UINT64_MAX.  workspace: kgrec_eval_workspace_bytes(nq, k) -- the
 * per-range partial lists plus [nq] uint32 score bits through which the ranges of a query share
 * their current K-th best (a range skips rows no other range would keep either). */
int64_t kgrec_eval_workspace_bytes(int64_t nq, int32_t k);
int kgrec_eval_topk(const kgrec_tables* tables, int model, int side,
                    const void* q, const void* r, int idx_bytes, const float* qvec, int64_t nq,
                    const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base, int32_t k,
                    const int64_t* filter_ptr, const int32_t* filter_ids,
                    const float* gumbel_u, uint64_t seed,
                    uint64_t* out_keys, void* workspace, int64_t workspace_bytes,
                    kgrec_stream_t stream);

/* K-way merge of per-shard / per-split top-K lists: in [n_lists, nq, k] -> out [nq, k].
 * Run after the NCCL all-gather of per-GPU candidates (the path's one collective). */
int kgrec_merge_topk(const uint64_t* in_keys, int32_t n_lists, int64_t nq, int32_t k,
                     uint64_t* out_keys, kgrec_stream_t stream);

/* Filtered rank of gold ids (getKGPerformance, utils/misc.py:125-146): adds to counts[i]
 * (caller-zeroed) #{ e in catalog shard : (score(q_i, e), e) < (gold_scores[i], gold_ids[i]) }.
 * Counts of different shards add (one all-reduce); the filter / other-gold correction is
 * applied by the caller from the few filtered ids' scores. */
int kgrec_eval_rank_count(const kgrec_tables* tables, int model, int side,
                          const void* q, const void* r, int idx_bytes, const float* qvec, int64_t nq,
                          const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base,
                          const float* gold_scores, const int32_t* gold_ids,
                          int32_t* counts, kgrec_stream_t stream);

/* The same count with the filter applied in the kernel: row i adds
 * #{ e in catalog shard : (score(q_i, e), e) < (gold_scores[i], gold_ids[i]), e not in X_i }
 * where X_i = excl_ids[excl_ptr[excl_row[i]], excl_ptr[excl_row[i] + 1]) holds ascending GLOBAL ids
 * (the query's filter set -- train + other eval files -- and its gold set; the gold itself never
 * counts, the comparison being strict).  Rows that share a query share its exclusion row.  An id is
 * looked up only when its key is below the gold's.  Shard counts still add.  KG sides only (the rec side:
 * kgrec_rec_rank_count); all three arrays are required (an empty exclusion is a CSR of empty rows). */
int kgrec_eval_rank_count_ex(const kgrec_tables* tables, int model, int side,
                             const void* q, const void* r, int idx_bytes, const float* qvec, int64_t nq,
                             const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base,
                             const float* gold_scores, const int32_t* gold_ids, int32_t* counts,
                             const int32_t* excl_row, const int64_t* excl_ptr, const int32_t* excl_ids,
                             kgrec_stream_t stream);

/* Raw and filtered ranks of link prediction from one catalog sweep.  The arguments of kgrec_eval_rank_count_ex
 * (counts -> filt_counts: the same count, bit for bit) plus the query's gold set as a CSR indexed by the same row,
 * G_i = gold_set_ids[gold_ptr[excl_row[i]], gold_ptr[excl_row[i] + 1]) (ascending global ids), and raw_counts:
 *
 *   filt_counts[i] += #{ e in shard : (score(q_i, e), e) < (gold_scores[i], gold_ids[i]), e not in X_i }
 *   raw_counts[i]  += #{ e in shard : (score(q_i, e), e) < (gold_scores[i], gold_ids[i]), e not in G_i }
 *
 * raw is the reference's walk without the filter (fliter_samples = None, utils/misc.py:125-146): only the query's
 * other golds are skipped.  PRECONDITION: every id of G_i is also in X_i (X_i = filter set U gold set, as
 * KGEvaluator builds it); the gold row is searched only for ids the exclusion row holds, so a gold missing from X_i
 * counts in the raw count.  Both arrays caller-zeroed; the counts of catalog shards add.  KG sides only; every
 * array non-NULL and aligned to its element size. */
int kgrec_eval_rank_count_dual(const kgrec_tables* tables, int model, int side,
                               const void* q, const void* r, int idx_bytes, const float* qvec, int64_t nq,
                               const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base,
                               const float* gold_scores, const int32_t* gold_ids, int32_t* filt_counts,
                               const int32_t* excl_row, const int64_t* excl_ptr, const int32_t* excl_ids,
                               const int64_t* gold_ptr, const int32_t* gold_set_ids, int32_t* raw_counts,
                               kgrec_stream_t stream);

/* Rank counts of the recommendation side (TUP / KTUP): where every gold item of a user sits in the whole filtered
 * catalog.  The queries are USERS, one query per user exactly as in kgrec_eval_topk on KGREC_SIDE_REC (q = user ids,
 * or qvec = augmented user rows with cat = the augmented catalog of the same kind: kgrec_pref_aug_rows /
 * kgrec_gumbel_aug_rows; the three paths and their envelopes are those of kgrec_eval_scores).  The hashed ST-Gumbel
 * noise is one draw per (position of the user in the call, global item id, preference), so only a call with the same
 * user list and seed ranks by the scores kgrec_eval_topk / kgrec_eval_scores see.  The golds hang off the query as a
 * CSR: G_q = gold_ids[gold_ptr[q], gold_ptr[q + 1]) (ascending global ids, n_gold = gold_ptr[nq] in all); the filter
 * row F_q = filter_ids[filter_ptr[q], filter_ptr[q + 1]) is the CSR kgrec_eval_topk takes (both NULL: no filter).
 *
 *   counts[j] += #{ e in shard : (score(u_q, e), e) < (score(u_q, g_j), g_j), e not in F_q, e not in G_q }
 *                                                                            gold_ptr[q] <= j < gold_ptr[q + 1]
 *
 * in the (score bits, global id) key order of kgrec_eval_topk, strictly: a gold never counts itself and two golds of
 * one user never count each other.  This is getKGPerformance's rank (utils/misc.py:125-146) in getRecPerformance's
 * order and filter (213-229).  A gold that is itself in F_q (never in the top-n list either) is skipped: the call
 * SETS its count to -1.  Counts (caller-zeroed) of different catalog shards add, so after the sum a skipped gold is
 * negative.
 *
 * The gold scores must be the values the count pass computes itself, bit for bit, noise included.
 * kgrec_rec_gold_scores is therefore a sweep of the same kernels over the shard that stores the score of every
 * (q, g_j) pair it meets: gold_scores[j] (caller-zeroed) is written when g_j lies in the shard, so the arrays of
 * different shards add (scores are >= 0 and every gold lives in one shard).  kgrec_rec_rank_count then sorts each
 * query's gold keys, streams the shard once more and, for every pair below the query's largest gold key, finds by
 * binary search the golds it sorts before; the filter row is searched only for such pairs.  Any number of golds per
 * query.  workspace: kgrec_rec_rank_workspace_bytes(nq, n_gold) bytes, 8-byte aligned.  nq = 0 or n_gold = 0: no-op. */
int kgrec_rec_gold_scores(const kgrec_tables* tables, int model, const void* q, int idx_bytes, const float* qvec,
                          int64_t nq, const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base,
                          const int64_t* gold_ptr, const int32_t* gold_ids, const float* gumbel_u, uint64_t seed,
                          float* gold_scores, kgrec_stream_t stream);
int64_t kgrec_rec_rank_workspace_bytes(int64_t nq, int64_t n_gold);
int kgrec_rec_rank_count(const kgrec_tables* tables, int model, const void* q, int idx_bytes, const float* qvec,
                         int64_t nq, const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base,
                         const int64_t* gold_ptr, const int32_t* gold_ids, int64_t n_gold, const float* gold_scores,
                         const int64_t* filter_ptr, const int32_t* filter_ids, const float* gumbel_u, uint64_t seed,
                         int32_t* counts, void* workspace, int64_t workspace_bytes, kgrec_stream_t stream);

/* Per-user top-n metrics of the rec side (getRecPerformance, utils/misc.py:213-248): keys [nq, k] from
 * kgrec_eval_topk (UINT64_MAX places are not part of the list), gold sets as a CSR (gold_ptr [nq+1],
 * ascending ids).  out [nq, 5] float64 = (f1, precision, recall, hit, ndcg) with precision = hits / list
 * length and ndcg_at_k method 0 (utils/evaluation.py:41-110); a user without a hit gets zeros. */
int kgrec_rec_topk_metrics(const uint64_t* keys, int64_t nq, int32_t k, const int64_t* gold_ptr,
                           const int32_t* gold_ids, double* out, kgrec_stream_t stream);

/* TransR full-catalog evaluation (transR.py:80-128 + projection_transR_pytorch_batch, misc.py:29-33).
 * The reference projects the whole entity table with every query's matrix; queries of one relation
 * share it, so the caller passes the queries SORTED BY RELATION (q / r device arrays, nq of them) with
 * the run boundaries on the host (run g = sorted queries [run_begin_host[g], run_begin_host[g+1]) of
 * relation run_rel_host[g]); per run the catalog shard is projected once by a hand-written FP32 kernel
 * into `workspace` (kgrec_transr_workspace_floats floats, 16-byte aligned) and the distance kernels of
 * the three modes above run on the projected rows.  Outputs / filter CSR / gold arrays are indexed in
 * the sorted query order.  embedding_size % 4 == 0 and <= 128. */
int64_t kgrec_transr_workspace_floats(int64_t nq, int64_t n_cat, int32_t dim);
int kgrec_transr_eval_scores(const kgrec_tables* tables, int side, const void* q, const void* r, int idx_bytes,
                             int64_t nq, const int64_t* run_begin_host, const int64_t* run_rel_host, int32_t n_runs,
                             const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base,
                             const int32_t* cat_ids, float* workspace, float* out, int64_t ld_out,
                             int32_t* status, kgrec_stream_t stream);
int kgrec_transr_eval_topk(const kgrec_tables* tables, int side, const void* q, const void* r, int idx_bytes,
                           int64_t nq, const int64_t* run_begin_host, const int64_t* run_rel_host, int32_t n_runs,
                           const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base, float* workspace,
                           int32_t k, const int64_t* filter_ptr, const int32_t* filter_ids, uint64_t* out_keys,
                           void* topk_workspace, int64_t topk_workspace_bytes, int32_t* status,
                           kgrec_stream_t stream);
int kgrec_transr_eval_rank_count(const kgrec_tables* tables, int side, const void* q, const void* r, int idx_bytes,
                                 int64_t nq, const int64_t* run_begin_host, const int64_t* run_rel_host, int32_t n_runs,
                                 const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base, float* workspace,
                                 const float* gold_scores, const int32_t* gold_ids, int32_t* counts,
                                 int32_t* status, kgrec_stream_t stream);
/* kgrec_eval_rank_count_ex on the projected rows; excl_row is indexed in the sorted query order and
 * holds absolute rows of the exclusion CSR. */
int kgrec_transr_eval_rank_count_ex(const kgrec_tables* tables, int side, const void* q, const void* r, int idx_bytes,
                                    int64_t nq, const int64_t* run_begin_host, const int64_t* run_rel_host, int32_t n_runs,
                                    const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base, float* workspace,
                                    const float* gold_scores, const int32_t* gold_ids, int32_t* counts,
                                    const int32_t* excl_row, const int64_t* excl_ptr, const int32_t* excl_ids,
                                    int32_t* status, kgrec_stream_t stream);
/* kgrec_eval_rank_count_dual on the projected rows: excl_row (sorted query order) indexes both CSRs with
 * absolute rows; filt_counts / raw_counts are in the sorted query order. */
int kgrec_transr_eval_rank_count_dual(const kgrec_tables* tables, int side, const void* q, const void* r, int idx_bytes,
                                      int64_t nq, const int64_t* run_begin_host, const int64_t* run_rel_host, int32_t n_runs,
                                      const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base, float* workspace,
                                      const float* gold_scores, const int32_t* gold_ids, int32_t* filt_counts,
                                      const int32_t* excl_row, const int64_t* excl_ptr, const int32_t* excl_ids,
                                      const int64_t* gold_ptr, const int32_t* gold_set_ids, int32_t* raw_counts,
                                      int32_t* status, kgrec_stream_t stream);

/* Soft-preference rec-side evaluation (use_st_gumbel = 0) on augmented rows: with raw logits as
 * mixing weights (transUP.py:108-113) r and w are linear in the logits, so each table row is
 * augmented ONCE into [x | x +/- XA | -/+ XB | x . XB] (leading dimension kgrec_pref_aug_ld(d))
 * and the pair score needs two cross dots and one distance pass.  Build the query rows
 * (is_query = 1; ids gathers user rows) and the catalog rows (is_query = 0; rows = the item
 * table, or the kgrec_ktup_item_table output), then call kgrec_eval_scores / kgrec_eval_topk
 * with side = KGREC_SIDE_REC, qvec = the augmented query rows and cat = the augmented catalog. */
int32_t kgrec_pref_aug_ld(int32_t dim);
/* 1 when the augmented soft-preference kernel fits this (embedding_size, top-k [0 = score matrix]); where it does
 * not (148 <= d <= 256, or top-k >= 62 at d = 128), evaluate with user / item ids on the plain path instead. */
int32_t kgrec_pref_aug_supported(int32_t dim, int32_t k);
/* 1 when the plain rec-side path (user / item ids, no augmented rows) fits this (embedding_size, preference_total,
 * use_st_gumbel, top-k [0 = score matrix]).  It stages both preference tables whole, so it has a limit in
 * preference_total x embedding_size: at d = 256 and top-k 128, soft preferences fit up to preference_total 25. */
int32_t kgrec_pref_eval_supported(int32_t dim, int32_t n_pref, int32_t use_gumbel, int32_t k);
int kgrec_pref_aug_rows(const kgrec_tables* tables, int model, int is_query,
                        const void* ids, int idx_bytes, const float* rows, int64_t row_ld, int64_t n,
                        float* out, int64_t ld_out, kgrec_stream_t stream);

/* ST-Gumbel rec-side evaluation (use_st_gumbel = 1, squared-L2 score) on augmented rows.  The pair's preference is
 * k* = arg-max_k (u + i).P'_k / 2 + g_k with fresh Gumbel noise per (pair, k) (transUP.py:84-102, 143-170); with
 * r = hf P'_k*, w = hf N'_k*, a = u - i, s = a.w the score |a + r - s w|^2 equals
 * |a|^2 + |r|^2 + 2 a.r + s^2 (|w|^2 - 2) - 2 s r.w, so each table row is augmented ONCE into
 * [x | A_k = x.P'_k / 2 | C_k = x.(hf N'_k) | pad] (leading dimension kgrec_gumbel_aug_ld(d, P)) and a pair costs the
 * distance |u - i|^2 plus a P-step arg-max: no per-pair [P x d] contraction.  Build the catalog rows (ids = NULL, rows
 * = the item table or the kgrec_ktup_item_table output) and the query rows (ids gathers user rows; gconst = the [3 P]
 * constants, which MUST be stored right behind the query rows: qvec + nq * ld), then call kgrec_eval_scores /
 * kgrec_eval_topk with side = KGREC_SIDE_REC, qvec = the query rows, cat = the augmented catalog. */
int32_t kgrec_gumbel_aug_ld(int32_t dim, int32_t n_pref);
/* 1 when the augmented ST-Gumbel kernel fits this (embedding_size, preference_total, top-k [0 = score matrix]) */
int32_t kgrec_gumbel_aug_supported(int32_t dim, int32_t n_pref, int32_t k);
int kgrec_gumbel_aug_rows(const kgrec_tables* tables, int model, const void* ids, int idx_bytes, const float* rows,
                          int64_t row_ld, int64_t n, float* out, int64_t ld_out, float* gconst,
                          kgrec_stream_t stream);

/* KTUP rec-side catalog: out[i] = Item[item_begin + i] + Ent[item2ent[item_begin + i]]
 * (jTransUP.py:177-181), n_items rows with leading dimension ld_out. */
int kgrec_ktup_item_table(const kgrec_tables* tables, int64_t item_begin, int64_t n_items,
                          float* out, int64_t ld_out, kgrec_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* KGREC_B200_H_ */
