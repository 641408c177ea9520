// extern "C" entry points of the training path: argument validation and family dispatch.
#include "train_dev.cuh"

namespace kgrec {

#define KGREC_DECLARE_FAMILY(FAMV)                                                                                       \
  extern template int launch_score_fwd<FAMV>(const kgrec_tables&, const Plan&, const IdxArgs&, int64_t, const float*,   \
                                             SeedRef, float*, int32_t*, cudaStream_t);                                 \
  extern template int launch_rank_loss_fwd<FAMV>(const kgrec_tables&, const Plan&, const IdxArgs&, const LossCfg&,      \
                                                 const float*, SeedRef, float*, float*, float*, int32_t*, cudaStream_t); \
  extern template int launch_score_bwd<FAMV>(const kgrec_tables&, const Plan&, const IdxArgs&, int64_t, const LossCfg&, \
                                             const float*, SeedRef, const BwdArgs&, const kgrec_grads&, cudaStream_t);
KGREC_DECLARE_FAMILY(FAM_E)
KGREC_DECLARE_FAMILY(FAM_H)
KGREC_DECLARE_FAMILY(FAM_R)
KGREC_DECLARE_FAMILY(FAM_REC)

#define KGREC_BY_FAMILY(fam, CALL)                       \
  ((fam) == FAM_E ? CALL<FAM_E> : (fam) == FAM_H ? CALL<FAM_H> : (fam) == FAM_R ? CALL<FAM_R> : CALL<FAM_REC>)

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int make_plan(const kgrec_tables* T, int model, Plan* pl) {
  if (!T) { set_error("tables is NULL"); return KGREC_ERR_INVALID; }
  if (T->dim <= 0 || T->ld < T->dim) { set_error("bad dim/ld (%d/%d)", T->dim, T->ld); return KGREC_ERR_INVALID; }
  if (T->dim > 512) { set_error("embedding_size %d > 512 is not built", T->dim); return KGREC_ERR_UNSUPPORTED; }
  pl->ktup = 0;
  pl->pr = 1;
  pl->smem_fwd = pl->smem_bwd = 0;
  bool ok = true, al = true;
  auto need = [&](const void* p, const char* name) {
    if (!p) { set_error("model %d needs table '%s'", model, name); ok = false; }
    else if (!aligned16(p)) al = false;
  };
  switch (model) {
    case KGREC_TRANSE: pl->fam = FAM_E; need(T->ent, "ent"); need(T->rel, "rel"); break;
    case KGREC_TRANSH: pl->fam = FAM_H; need(T->ent, "ent"); need(T->rel, "rel"); need(T->norm, "norm"); break;
    case KGREC_TRANSR: pl->fam = FAM_R; need(T->ent, "ent"); need(T->rel, "rel"); need(T->proj, "proj"); break;
    case KGREC_KTUP:
      pl->ktup = 1;
      need(T->ent, "ent"); need(T->rel, "rel"); need(T->norm, "norm");
      if (!T->item2ent) { set_error("KTUP needs item2ent"); ok = false; }
      if (ok && T->n_pref != T->n_rel) { set_error("KTUP needs n_pref == n_rel"); return KGREC_ERR_INVALID; }
      /* fallthrough */
    case KGREC_TUP:
      pl->fam = FAM_REC;
      need(T->user, "user"); need(T->item, "item"); need(T->pref, "pref"); need(T->pref_norm, "pref_norm");
      break;
    default: set_error("unknown model %d", model); return KGREC_ERR_INVALID;
  }
  if (!ok) return KGREC_ERR_INVALID;
  pl->vec = al && (T->dim % 4 == 0) && (T->ld % 4 == 0);
  pl->nch = T->dim <= 128 ? 1 : (T->dim <= 256 ? 2 : 4);
  if (!pl->vec && pl->nch == 2) pl->nch = 4;                 // scalar path is built for NCH 1 and 4
  if (pl->fam == FAM_R) pl->smem_fwd = pl->smem_bwd = static_cast<size_t>(kWarpsPerCta) * 128 * pl->nch * sizeof(float);
  if (pl->fam == FAM_REC) {
    const int P = T->n_pref;
    if (P <= 0 || P > kMaxPref) {
      set_error("preference_total %d outside [1, %d]", P, kMaxPref);
      return KGREC_ERR_UNSUPPORTED;
    }
    pl->smem_fwd = (rec_tables_floats(P, T->dim) + static_cast<size_t>(kWarpsPerCta) * 3 * kMaxPref) * sizeof(float);
    pl->smem_bwd = pl->smem_fwd +
                   static_cast<size_t>(kWarpsPerCta) * (3 * pl->nch * 128 + 2 * kMaxPref) * sizeof(float) + 64;
    pl->pr = (P + kWarpsPerCta - 1) / kWarpsPerCta;
    if (pl->smem_bwd > 220 * 1024) { set_error("preference tables do not fit in shared memory"); return KGREC_ERR_UNSUPPORTED; }
  }
  return KGREC_OK;
}

static int check_bwd_plan(const kgrec_tables* T, const Plan& pl) {
  if (pl.fam != FAM_REC) return KGREC_OK;
  const int pmax = pl.nch == 1 ? 64 : (pl.nch == 2 ? 32 : 16);
  if (T->n_pref > pmax) {
    set_error("backward: preference_total %d > %d is not built for embedding_size %d", T->n_pref, pmax, T->dim);
    return KGREC_ERR_UNSUPPORTED;
  }
  return KGREC_OK;
}

static int check_idx(const void* a, const void* b, const void* c, int fam, int idx_bytes) {
  if (idx_bytes != 4 && idx_bytes != 8) { set_error("idx_bytes must be 4 or 8"); return KGREC_ERR_INVALID; }
  if (!a || !b || (fam != FAM_REC && !c)) { set_error("index array is NULL"); return KGREC_ERR_INVALID; }
  return KGREC_OK;
}

static int check_loss(int loss_kind, int64_t n_pos, int32_t n_neg, int64_t batch_pos) {
  if (loss_kind != KGREC_LOSS_MARGIN && loss_kind != KGREC_LOSS_BPR) { set_error("unknown loss %d", loss_kind); return KGREC_ERR_INVALID; }
  if (n_pos < 0 || n_neg < 1 || batch_pos < 1) { set_error("bad n_pos / n_neg / batch_pos"); return KGREC_ERR_INVALID; }
  return KGREC_OK;
}

static int check_grads(const Plan& pl, const kgrec_grads* G) {
  if (!G || (G->mode != 0 && G->mode != 1)) { set_error("bad grads descriptor"); return KGREC_ERR_INVALID; }
  bool ok;
  if (pl.fam == FAM_REC) ok = G->user && G->item && G->pref && G->pref_norm && (!pl.ktup || G->ent);
  else ok = G->ent && G->rel && (pl.fam != FAM_H || G->norm) && (pl.fam != FAM_R || G->proj);
  if (!ok) { set_error("a gradient buffer this model needs is NULL"); return KGREC_ERR_INVALID; }
  return KGREC_OK;
}

}  // namespace kgrec

using namespace kgrec;

extern "C" int kgrec_score_fwd(const kgrec_tables* tables, int model, const void* a, const void* b, const void* c,
                               int idx_bytes, int64_t n, const float* gumbel_u, uint64_t seed, float* scores,
                               int32_t* status, kgrec_stream_t stream) {
  Plan pl;
  int rc = make_plan(tables, model, &pl);
  if (rc) return rc;
  if ((rc = check_idx(a, b, c, pl.fam, idx_bytes))) return rc;
  if (n < 0 || !scores) { set_error("bad n / scores"); return KGREC_ERR_INVALID; }
  if (n == 0) return KGREC_OK;
  const IdxArgs I{a, b, c, nullptr, nullptr, nullptr, idx_bytes == 8};
  return KGREC_BY_FAMILY(pl.fam, launch_score_fwd)(*tables, pl, I, n, gumbel_u, seed, scores, status,
                                                   static_cast<cudaStream_t>(stream));
}

extern "C" int64_t kgrec_rank_loss_workspace_bytes(int64_t n_pos) { return (n_pos > 0 ? n_pos : 1) * 4; }

extern "C" int kgrec_rank_loss_fwd(const kgrec_tables* tables, int model, const void* pa, const void* pb,
                                   const void* pc, const void* na, const void* nb, const void* nc, int idx_bytes,
                                   int64_t n_pos, int32_t n_neg, int64_t batch_pos, int loss_kind,
                                   float margin_or_target, const float* gumbel_u, uint64_t seed, float* pos_scores,
                                   float* neg_scores, float* loss, void* workspace, int32_t* status,
                                   kgrec_stream_t stream) {
  Plan pl;
  int rc = make_plan(tables, model, &pl);
  if (rc) return rc;
  if ((rc = check_idx(pa, pb, pc, pl.fam, idx_bytes)) || (rc = check_idx(na, nb, nc, pl.fam, idx_bytes))) return rc;
  if ((rc = check_loss(loss_kind, n_pos, n_neg, batch_pos))) return rc;
  if (!pos_scores || !neg_scores || !loss || !workspace) { set_error("output / workspace pointer is NULL"); return KGREC_ERR_INVALID; }
  if (n_pos == 0) return KGREC_OK;
  const IdxArgs I{pa, pb, pc, na, nb, nc, idx_bytes == 8};
  const LossCfg L{loss_kind, margin_or_target, n_neg, n_pos, batch_pos};
  float* group_loss = static_cast<float*>(workspace);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  rc = KGREC_BY_FAMILY(pl.fam, launch_rank_loss_fwd)(*tables, pl, I, L, gumbel_u, seed, pos_scores, neg_scores,
                                                     group_loss, status, st);
  if (rc) return rc;
  const int64_t n_batches = (n_pos + batch_pos - 1) / batch_pos;
  k_batch_loss<<<static_cast<unsigned>(n_batches), 256, 0, st>>>(group_loss, L, loss);
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

extern "C" int kgrec_score_bwd(const kgrec_tables* tables, int model, const void* a, const void* b, const void* c,
                               int idx_bytes, int64_t n, const float* gumbel_u, uint64_t seed,
                               const float* grad_scores, const kgrec_grads* grads, kgrec_stream_t stream) {
  Plan pl;
  int rc = make_plan(tables, model, &pl);
  if (rc) return rc;
  if ((rc = check_bwd_plan(tables, pl)) || (rc = check_idx(a, b, c, pl.fam, idx_bytes)) || (rc = check_grads(pl, grads))) return rc;
  if (n < 0 || !grad_scores) { set_error("bad n / grad_scores"); return KGREC_ERR_INVALID; }
  if (n == 0) return KGREC_OK;
  const IdxArgs I{a, b, c, nullptr, nullptr, nullptr, idx_bytes == 8};
  const LossCfg L{0, 0.f, 1, n, n};
  const BwdArgs B{grad_scores, nullptr, nullptr, 1.f, nullptr};
  return KGREC_BY_FAMILY(pl.fam, launch_score_bwd)(*tables, pl, I, n, L, gumbel_u, seed, B, *grads,
                                                   static_cast<cudaStream_t>(stream));
}

extern "C" int kgrec_rank_loss_bwd(const kgrec_tables* tables, int model, const void* pa, const void* pb,
                                   const void* pc, const void* na, const void* nb, const void* nc, int idx_bytes,
                                   int64_t n_pos, int32_t n_neg, int64_t batch_pos, int loss_kind,
                                   float margin_or_target, const float* gumbel_u, uint64_t seed,
                                   const float* pos_scores, const float* neg_scores, float grad_loss,
                                   const float* grad_loss_dev, const kgrec_grads* grads, kgrec_stream_t stream) {
  Plan pl;
  int rc = make_plan(tables, model, &pl);
  if (rc) return rc;
  if ((rc = check_bwd_plan(tables, pl)) || (rc = check_idx(pa, pb, pc, pl.fam, idx_bytes)) ||
      (rc = check_idx(na, nb, nc, pl.fam, idx_bytes)) || (rc = check_grads(pl, grads)))
    return rc;
  if ((rc = check_loss(loss_kind, n_pos, n_neg, batch_pos))) return rc;
  if (!pos_scores || !neg_scores) { set_error("saved scores are NULL"); return KGREC_ERR_INVALID; }
  if (n_pos == 0) return KGREC_OK;
  const IdxArgs I{pa, pb, pc, na, nb, nc, idx_bytes == 8};
  const LossCfg L{loss_kind, margin_or_target, n_neg, n_pos, batch_pos};
  const BwdArgs B{nullptr, pos_scores, neg_scores, grad_loss, grad_loss_dev};
  return KGREC_BY_FAMILY(pl.fam, launch_score_bwd)(*tables, pl, I, n_pos * (1 + static_cast<int64_t>(n_neg)), L,
                                                   gumbel_u, seed, B, *grads, static_cast<cudaStream_t>(stream));
}

static int rank_loss_step(const kgrec_tables* tables, int model, const void* pa, const void* pb, const void* pc,
                          const void* na, const void* nb, const void* nc, int idx_bytes, int64_t n_pos, int32_t n_neg,
                          int64_t batch_pos, int loss_kind, float margin_or_target, float grad_loss,
                          const float* gumbel_u, SeedRef seed, float* pos_scores, float* neg_scores, float* loss,
                          const kgrec_grads* grads, int64_t* slot_user_ids, int64_t* slot_item_ids,
                          int64_t* slot_ent_ids, void* workspace, int32_t* status, kgrec_stream_t stream) {
  Plan pl;
  int rc = make_plan(tables, model, &pl);
  if (rc) return rc;
  if ((rc = check_bwd_plan(tables, pl)) || (rc = check_idx(pa, pb, pc, pl.fam, idx_bytes)) ||
      (rc = check_idx(na, nb, nc, pl.fam, idx_bytes)) || (rc = check_grads(pl, grads)))
    return rc;
  if ((rc = check_loss(loss_kind, n_pos, n_neg, batch_pos))) return rc;
  if (!pos_scores || !neg_scores || !loss || !workspace) { set_error("output / workspace pointer is NULL"); return KGREC_ERR_INVALID; }
  const bool want_ids = slot_user_ids != nullptr;
  if (want_ids && (pl.fam != FAM_REC || !slot_item_ids || (pl.ktup && !slot_ent_ids))) {
    set_error("slot ids: TUP / KTUP only, user + item (+ entity for KTUP) together");
    return KGREC_ERR_INVALID;
  }
  if (n_pos == 0) return KGREC_OK;
  const IdxArgs I{pa, pb, pc, na, nb, nc, idx_bytes == 8};
  const LossCfg L{loss_kind, margin_or_target, n_neg, n_pos, batch_pos};
  float* group_loss = static_cast<float*>(workspace);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t n_batches = (n_pos + batch_pos - 1) / batch_pos;
  rc = -1;
  if (pl.fam == FAM_REC)
    rc = rec_tile_loss_step(*tables, pl, I, L, grad_loss, gumbel_u, seed, pos_scores, neg_scores, group_loss, *grads,
                            want_ids ? slot_user_ids : nullptr, slot_item_ids, slot_ent_ids, status, st);
  if (rc > 0) return rc;
  if (rc < 0) {   // shapes the single-pass kernel is not built for: forward, then backward from the saved scores
    rc = KGREC_BY_FAMILY(pl.fam, launch_rank_loss_fwd)(*tables, pl, I, L, gumbel_u, seed, pos_scores, neg_scores,
                                                       group_loss, status, st);
    if (rc) return rc;
    const BwdArgs B{nullptr, pos_scores, neg_scores, grad_loss, nullptr};
    rc = KGREC_BY_FAMILY(pl.fam, launch_score_bwd)(*tables, pl, I, n_pos * (1 + static_cast<int64_t>(n_neg)), L,
                                                   gumbel_u, seed, B, *grads, st);
    if (rc) return rc;
    if (want_ids && (rc = rec_slot_ids(*tables, pl, I, n_pos, n_pos * (1 + static_cast<int64_t>(n_neg)), slot_user_ids,
                                       slot_item_ids, slot_ent_ids, st)))
      return rc;
  }
  k_batch_loss<<<static_cast<unsigned>(n_batches), 256, 0, st>>>(group_loss, L, loss);
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

extern "C" int kgrec_rank_loss_step(const kgrec_tables* tables, int model, const void* pa, const void* pb,
                                    const void* pc, const void* na, const void* nb, const void* nc, int idx_bytes,
                                    int64_t n_pos, int32_t n_neg, int64_t batch_pos, int loss_kind,
                                    float margin_or_target, float grad_loss, const float* gumbel_u, uint64_t seed,
                                    float* pos_scores, float* neg_scores, float* loss, const kgrec_grads* grads,
                                    int64_t* slot_user_ids, int64_t* slot_item_ids, int64_t* slot_ent_ids,
                                    void* workspace, int32_t* status, kgrec_stream_t stream) {
  return rank_loss_step(tables, model, pa, pb, pc, na, nb, nc, idx_bytes, n_pos, n_neg, batch_pos, loss_kind,
                        margin_or_target, grad_loss, gumbel_u, seed, pos_scores, neg_scores, loss, grads, slot_user_ids,
                        slot_item_ids, slot_ent_ids, workspace, status, stream);
}

extern "C" int kgrec_rank_loss_step_dev(const kgrec_tables* tables, int model, const void* pa, const void* pb,
                                        const void* pc, const void* na, const void* nb, const void* nc, int idx_bytes,
                                        int64_t n_pos, int32_t n_neg, int64_t batch_pos, int loss_kind,
                                        float margin_or_target, float grad_loss, const float* gumbel_u,
                                        const kgrec_step_state* state, float* pos_scores, float* neg_scores,
                                        float* loss, const kgrec_grads* grads, int64_t* slot_user_ids,
                                        int64_t* slot_item_ids, int64_t* slot_ent_ids, void* workspace,
                                        int32_t* status, kgrec_stream_t stream) {
  if (!state) { set_error("step state is NULL"); return KGREC_ERR_INVALID; }
  return rank_loss_step(tables, model, pa, pb, pc, na, nb, nc, idx_bytes, n_pos, n_neg, batch_pos, loss_kind,
                        margin_or_target, grad_loss, gumbel_u, SeedRef(0, state), pos_scores, neg_scores, loss, grads,
                        slot_user_ids, slot_item_ids, slot_ent_ids, workspace, status, stream);
}
