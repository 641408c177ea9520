// Fused gather -> (project | preference-mix) -> residual -> L1/L2 reduce -> ranking loss
// kernels and their sparse-row-gradient backward, for sm_90a.
//
// Mapping: one warp owns one triple / pair.  A row of d floats is spread over the warp
// (Row<NCH,VEC>: 128-bit loads, lane c owns float4 chunk c); all rows of a triple are
// requested back to back before any arithmetic so each warp keeps 3-4 rows (1.2-1.6 KB) in
// flight, and every reduction over d is a shuffle tree.  Nothing is staged through global
// memory between the gather and the score.
//
// Reference arithmetic restated here (CPU form: oracle/kg_oracle.py):
//   transE.py:51-63, transH.py:58-71 (+utils/misc.py:18-19), transR.py:65-78
//   (+misc.py:21-26), transUP.py:69-82,105-115,143-170, jTransUP.py:122-161,250-315,
//   utils/loss.py:8-16,29-31.
#pragma once
#include "common.cuh"

namespace kgrec {

enum { FAM_E = 0, FAM_H = 1, FAM_R = 2, FAM_REC = 3 };

struct LossCfg {
  int kind;           // KGREC_LOSS_*
  float param;        // margin or target
  int n_neg;          // negatives per positive
  int64_t n_pos;
  int64_t batch_pos;  // positives per loss batch
};

struct IdxArgs {
  const void *a, *b, *c;     // flat triples (or positives)
  const void *na, *nb, *nc;  // negatives (fused ranking-loss kernels)
  int is64;
};

struct Plan {
  int fam, nch, ktup;
  bool vec;
  int pr;  // REC backward: preference rows per warp
  size_t smem_fwd, smem_bwd;
};

struct BwdArgs {
  const float* grad_scores;  // explicit upstream, or
  const float* pos_scores;   // saved scores of the fused ranking loss
  const float* neg_scores;
  float grad_loss;             // host scalar, multiplied with
  const float* grad_loss_dev;  // optional per-batch upstream [n_batches] (device)
};

__device__ __forceinline__ float loss_term(const LossCfg& L, float pos, float neg) {
  if (L.kind == KGREC_LOSS_MARGIN) return fmaxf(pos - neg + L.param, 0.f);
  const float x = L.param * (pos - neg);  // -logsigmoid(x) = softplus(-x)
  return fmaxf(-x, 0.f) + log1pf(expf(-fabsf(x)));
}
// d term / d pos  (d term / d neg is the negative)
__device__ __forceinline__ float loss_dpos(const LossCfg& L, float pos, float neg) {
  if (L.kind == KGREC_LOSS_MARGIN) return (pos - neg + L.param > 0.f) ? 1.f : 0.f;
  const float x = L.param * (pos - neg);
  return -L.param / (1.f + expf(x));  // -target * sigmoid(-x)
}
__device__ __forceinline__ float loss_batch_scale(const LossCfg& L, int64_t j) {
  if (L.kind == KGREC_LOSS_MARGIN) return 1.f;  // a sum
  const int64_t b0 = (j / L.batch_pos) * L.batch_pos;
  const int64_t cnt = min(L.batch_pos, L.n_pos - b0);
  return 1.f / (static_cast<float>(cnt) * static_cast<float>(L.n_neg));  // a mean
}
// upstream dLoss/dscore of flat triple i (positives first, then negatives)
__device__ __forceinline__ float upstream_grad(const BwdArgs& B, const LossCfg& L, int64_t i, int lane) {
  if (B.pos_scores == nullptr) return __ldg(B.grad_scores + i);
  if (i < L.n_pos) {
    const float sp = __ldg(B.pos_scores + i);
    float c = 0.f;
    for (int k = lane; k < L.n_neg; k += 32) c += loss_dpos(L, sp, __ldg(B.neg_scores + i * L.n_neg + k));
    const float up = B.grad_loss * (B.grad_loss_dev ? __ldg(B.grad_loss_dev + i / L.batch_pos) : 1.f);
    return warp_sum(c) * loss_batch_scale(L, i) * up;
  }
  const int64_t m = i - L.n_pos, j = m / L.n_neg;
  const float up = B.grad_loss * (B.grad_loss_dev ? __ldg(B.grad_loss_dev + j / L.batch_pos) : 1.f);
  return -loss_dpos(L, __ldg(B.pos_scores + j), __ldg(B.neg_scores + m)) * loss_batch_scale(L, j) * up;
}

// out[k] = scale * sum_j (TA[k][j] a_j + TB[k][j] b_j), k < n_rows; rows read with LOAD
// (shared or global), eight rows per butterfly.  `out` is warp-private shared memory.
template <int NCH, bool VEC, bool GLOBAL, bool TWO>
__device__ __forceinline__ void rows_dot(const float (&a)[NCH * 4], const float* TA, const float (&b)[NCH * 4],
                                         const float* TB, int n_rows, int64_t stride, int d, float scale, float* out,
                                         int lane) {
  using R = Row<NCH, VEC>;
#pragma unroll 1
  for (int g = 0; g < n_rows; g += 8) {
    float vals[8];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const int k = g + kk;
      vals[kk] = 0.f;
      if (k < n_rows) {
        float row[NCH * 4];
        if (GLOBAL) R::load(row, TA + k * stride, d, lane);
        else R::load_s(row, TA + k * stride, d, lane);
        float s = R::dot(row, a);
        if (TWO) {
          if (GLOBAL) R::load(row, TB + k * stride, d, lane);
          else R::load_s(row, TB + k * stride, d, lane);
          s += R::dot(row, b);
        }
        vals[kk] = s;
      }
    }
    const float r = warp_reduce_scatter8(vals, lane);
    const int k = g + (lane >> 2);
    if ((lane & 3) == 0 && k < n_rows) out[k] = r * scale;
  }
  __syncwarp();
}

// ===========================================================================================
// KG families: TransE / TransH / TransR
// ===========================================================================================
template <int FAM, int NCH, bool VEC>
struct KgTriple {
  using R = Row<NCH, VEC>;
  static constexpr int NE = R::NE;
  float h[NE], t[NE], r[NE], w[NE];
  float e[NE];
  float xw;  // (h - t) . w  (TransH)

  __device__ __forceinline__ void load(const kgrec_tables& T, int64_t ih, int64_t it, int64_t ir, int lane) {
    R::load(h, T.ent + ih * T.ld, T.dim, lane);
    R::load(t, T.ent + it * T.ld, T.dim, lane);
    R::load(r, T.rel + ir * T.ld, T.dim, lane);
    if (FAM == FAM_H) R::load(w, T.norm + ir * T.ld, T.dim, lane);
  }

  // score from the loaded rows.  TransR: `m` is the relation's d x d matrix and `scr` a
  // warp-private shared scratch of >= 128 * NCH floats.
  __device__ __forceinline__ float score(const kgrec_tables& T, const float* __restrict__ m, float* scr, int lane) {
    const int d = T.dim;
    if (FAM == FAM_E) {
#pragma unroll
      for (int i = 0; i < NE; ++i) e[i] = h[i] + r[i] - t[i];
    } else if (FAM == FAM_H) {
      float a = R::dot(h, w), b = R::dot(t, w);
      warp_sum2(a, b);
      xw = a - b;
#pragma unroll
      for (int i = 0; i < NE; ++i) e[i] = (h[i] - a * w[i]) + r[i] - (t[i] - b * w[i]);
    } else {
      // e = M (h - t) + r : d row-dot-products, eight per butterfly, through the scratch
      float x[NE];
#pragma unroll
      for (int i = 0; i < NE; ++i) x[i] = h[i] - t[i];
      __syncwarp();
      rows_dot<NCH, VEC, true, false>(x, m, x, nullptr, d, d, d, 1.f, scr, lane);
      R::load_s(e, scr, d, lane);
#pragma unroll
      for (int i = 0; i < NE; ++i) e[i] += r[i];
    }
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < NE; ++i) acc += dist_term(e[i], T.l1);
    return warp_sum(acc);
  }

  // row gradients for upstream g; slot `slot` of n
  __device__ __forceinline__ void backward(const kgrec_tables& T, const kgrec_grads& G, const float* __restrict__ m,
                                           float* scr, int64_t ih, int64_t it, int64_t ir, int64_t slot, int64_t n,
                                           float g, int lane) {
    const int d = T.dim;
    float eps[NE], gx[NE];
#pragma unroll
    for (int i = 0; i < NE; ++i) eps[i] = g * ddist_term(e[i], T.l1);
    if (FAM == FAM_E) {
#pragma unroll
      for (int i = 0; i < NE; ++i) gx[i] = eps[i];
    } else if (FAM == FAM_H) {
      const float ew = warp_sum(R::dot(eps, w));
      float gw[NE];
#pragma unroll
      for (int i = 0; i < NE; ++i) {
        gx[i] = eps[i] - ew * w[i];
        gw[i] = -(ew * (h[i] - t[i]) + xw * eps[i]);
      }
      if (G.mode == 0) R::store_cs(G.norm + slot * d, gw, d, lane);
      else R::red_add(G.norm + ir * d, gw, d, lane);
    } else {
      // gx = M^T eps ; grad_M[a, :] += eps_a * (h - t)
      float x[NE];
#pragma unroll
      for (int i = 0; i < NE; ++i) { x[i] = h[i] - t[i]; gx[i] = 0.f; }
      __syncwarp();
      R::store(scr, eps, d, lane);
      __syncwarp();
      float* gm = G.proj + ir * static_cast<int64_t>(d) * d;
#pragma unroll 2
      for (int a = 0; a < d; ++a) {
        const float ea = scr[a];
        float mr[NE], o[NE];
        R::load(mr, m + static_cast<int64_t>(a) * d, d, lane);
#pragma unroll
        for (int i = 0; i < NE; ++i) { gx[i] = fmaf(ea, mr[i], gx[i]); o[i] = ea * x[i]; }
        R::red_add(gm + static_cast<int64_t>(a) * d, o, d, lane);
      }
    }
    if (G.mode == 0) R::store_cs(G.rel + slot * d, eps, d, lane);
    else R::red_add(G.rel + ir * d, eps, d, lane);
    float ngx[NE];
#pragma unroll
    for (int i = 0; i < NE; ++i) ngx[i] = -gx[i];
    if (G.mode == 0) {
      R::store_cs(G.ent + slot * d, gx, d, lane);
      R::store_cs(G.ent + (n + slot) * d, ngx, d, lane);
    } else {
      R::red_add(G.ent + ih * d, gx, d, lane);
      R::red_add(G.ent + it * d, ngx, d, lane);
    }
  }
};

// ===========================================================================================
// REC family: TUP and the KTUP rec branch
// ===========================================================================================
struct PrefView {
  const float* P;  // smem [n_pref, stride]  (KTUP: pref + rel)
  const float* N;  // smem [n_pref, stride]  (KTUP: pref_norm + norm)
  int n_pref;
  int stride;
  float hf;  // 1 (TUP) or 0.5 (KTUP: jTransUP.py:257-258)
};

// warp-private shared scratch of a REC warp: 3 * kMaxPref floats
//   [0, P)          z   logits (u + i) . P_k / 2
//   [kMaxPref, +P)  v   z + Gumbel noise
//   [2kMaxPref, +P) gp  dLoss/dp
template <int NCH, bool VEC>
struct RecPair {
  using R = Row<NCH, VEC>;
  static constexpr int NE = R::NE;
  float u[NE], it[NE];
  float w[NE], r[NE], e[NE];
  float xw;
  int kstar;

  __device__ __forceinline__ void load_item(const kgrec_tables& T, bool ktup, int64_t ii, int64_t ia, int lane) {
    R::load(it, T.item + ii * T.ld, T.dim, lane);
    if (ktup) {
      float ee[NE];
      R::load(ee, T.ent + ia * T.ld, T.dim, lane);
#pragma unroll
      for (int i = 0; i < NE; ++i) it[i] += ee[i];  // ie = i_e + e_e  (jTransUP.py:133)
    }
  }
  __device__ __forceinline__ void load(const kgrec_tables& T, bool ktup, int64_t iu, int64_t ii, int64_t ia, int lane) {
    R::load(u, T.user + iu * T.ld, T.dim, lane);
    load_item(T, ktup, ii, ia, lane);
  }

  __device__ __forceinline__ float score(const kgrec_tables& T, const PrefView& pv, const float* gu_row, uint64_t seed,
                                         uint64_t pair_id, float* scr, int lane) {
    const int d = T.dim, P = pv.n_pref;
    float s[NE];
#pragma unroll
    for (int i = 0; i < NE; ++i) s[i] = u[i] + it[i];
    __syncwarp();
    rows_dot<NCH, VEC, false, false>(s, pv.P, s, nullptr, P, pv.stride, d, 0.5f, scr, lane);  // transUP.py:108
#pragma unroll
    for (int i = 0; i < NE; ++i) { r[i] = 0.f; w[i] = 0.f; }
    if (T.use_gumbel) {
      // the forward value of the ST estimator is the one-hot arg-max (transUP.py:164-168)
      float best = -INFINITY;
      int bk = 0x7fffffff;
      for (int k = lane; k < P; k += 32) {
        const float v = scr[k] + (gu_row ? gumbel_from_uniform(__ldg(gu_row + k))
                                         : gumbel_fast(philox_uniform_bits(seed, pair_id, static_cast<uint32_t>(k))));
        scr[kMaxPref + k] = v;
        if (v > best) { best = v; bk = k; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(FULL, best, o);
        const int ok = __shfl_xor_sync(FULL, bk, o);
        if (ob > best || (ob == best && ok < bk)) { best = ob; bk = ok; }
      }
      kstar = bk;
      float row[NE];
      R::load_s(row, pv.P + kstar * pv.stride, d, lane);
#pragma unroll
      for (int i = 0; i < NE; ++i) r[i] = pv.hf * row[i];
      R::load_s(row, pv.N + kstar * pv.stride, d, lane);
#pragma unroll
      for (int i = 0; i < NE; ++i) w[i] = pv.hf * row[i];
    } else {
      kstar = -1;
      // raw logits are the mixing weights, no softmax (transUP.py:108-113)
#pragma unroll 2
      for (int k = 0; k < P; ++k) {
        const float zk = scr[k];
        float row[NE];
        R::load_s(row, pv.P + k * pv.stride, d, lane);
#pragma unroll
        for (int i = 0; i < NE; ++i) r[i] = fmaf(zk, row[i], r[i]);
        R::load_s(row, pv.N + k * pv.stride, d, lane);
#pragma unroll
        for (int i = 0; i < NE; ++i) w[i] = fmaf(zk, row[i], w[i]);
      }
#pragma unroll
      for (int i = 0; i < NE; ++i) { r[i] *= pv.hf; w[i] *= pv.hf; }
    }
    float a = R::dot(u, w), b = R::dot(it, w);
    warp_sum2(a, b);
    xw = a - b;
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < NE; ++i) {
      e[i] = (u[i] - a * w[i]) + r[i] - (it[i] - b * w[i]);
      acc += dist_term(e[i], T.l1);
    }
    return warp_sum(acc);
  }

  // Backward for upstream g (score() must have run with the same scratch).  Produces the
  // user / item-side row gradients and leaves in the CTA staging area what the table-gradient
  // accumulation needs: vectors sv = [eps | gw | s] (dpad floats each) and coefficient rows
  // sc = [cA | cB] (kMaxPref each) with cA = hf * p, cB = gz / 2, so that
  //   g_pref[k] += cA[k] eps + cB[k] s ;  g_pref_norm[k] += cA[k] gw.
  __device__ __forceinline__ void backward(const kgrec_tables& T, const PrefView& pv, float g, float* scr, int lane,
                                           float (&gu)[NE], float (&gi)[NE], float* sv, float* sc, int dpad) {
    const int d = T.dim, P = pv.n_pref;
    float eps[NE], gw[NE], gx[NE], s[NE];
#pragma unroll
    for (int i = 0; i < NE; ++i) eps[i] = g * ddist_term(e[i], T.l1);
    const float ew = warp_sum(R::dot(eps, w));
#pragma unroll
    for (int i = 0; i < NE; ++i) {
      gx[i] = eps[i] - ew * w[i];
      gw[i] = -(ew * (u[i] - it[i]) + xw * eps[i]);
      s[i] = u[i] + it[i];
    }
    float* gp = scr + 2 * kMaxPref;
    rows_dot<NCH, VEC, false, true>(eps, pv.P, gw, pv.N, P, pv.stride, d, pv.hf, gp, lane);
    if (T.use_gumbel) {
      // y = softmax(z + noise); gz = y * (gp - <y, gp>)   (backward of transUP.py:162-168)
      const float* v = scr + kMaxPref;
      float mx = -INFINITY;
      for (int k = lane; k < P; k += 32) mx = fmaxf(mx, v[k]);
      mx = warp_max(mx);
      float sum = 0.f, yg = 0.f;
      for (int k = lane; k < P; k += 32) {
        const float ex = expf(v[k] - mx);
        sum += ex;
        yg += ex * gp[k];
      }
      warp_sum2(sum, yg);
      yg /= sum;
      for (int k = lane; k < P; k += 32) {
        const float y = expf(v[k] - mx) / sum;
        sc[k] = (k == kstar) ? pv.hf : 0.f;
        sc[kMaxPref + k] = 0.5f * y * (gp[k] - yg);
      }
    } else {
      for (int k = lane; k < P; k += 32) {
        sc[k] = pv.hf * scr[k];
        sc[kMaxPref + k] = 0.5f * gp[k];
      }
    }
    __syncwarp();
    // gs = sum_k gz_k P_k / 2 = sum_k cB_k P_k
    float gs[NE];
#pragma unroll
    for (int i = 0; i < NE; ++i) gs[i] = 0.f;
#pragma unroll 2
    for (int k = 0; k < P; ++k) {
      const float cb = sc[kMaxPref + k];
      float row[NE];
      R::load_s(row, pv.P + k * pv.stride, d, lane);
#pragma unroll
      for (int i = 0; i < NE; ++i) gs[i] = fmaf(cb, row[i], gs[i]);
    }
#pragma unroll
    for (int i = 0; i < NE; ++i) {
      gu[i] = gx[i] + gs[i];
      gi[i] = -gx[i] + gs[i];
    }
    R::store(sv, eps, dpad, lane);  // lanes past d hold zeros
    R::store(sv + dpad, gw, dpad, lane);
    R::store(sv + 2 * dpad, s, dpad, lane);
  }
};

// CTA prologue: stage the preference tables (KTUP: summed with the relation tables).
__device__ __forceinline__ void stage_pref_tables(const kgrec_tables& T, bool ktup, float* sP, float* sN, int stride) {
  const int d = T.dim, P = T.n_pref;
  for (int idx = threadIdx.x; idx < P * stride; idx += blockDim.x) {
    const int k = idx / stride, j = idx - k * stride;
    float a = 0.f, b = 0.f;
    if (j < d) {
      a = __ldg(T.pref + static_cast<int64_t>(k) * T.ld + j);
      b = __ldg(T.pref_norm + static_cast<int64_t>(k) * T.ld + j);
      if (ktup) {
        a += __ldg(T.rel + static_cast<int64_t>(k) * T.ld + j);
        b += __ldg(T.norm + static_cast<int64_t>(k) * T.ld + j);
      }
    }
    sP[idx] = a;
    sN[idx] = b;
  }
}

// ===========================================================================================
// kernels
// ===========================================================================================
// shared-memory layout helpers
//   KG  (TransR only): [8 warps][128 NCH] scratch
//   REC forward:  sP | sN | [8][3 kMaxPref] scratch
//   REC backward: sP | sN | [8][3 kMaxPref] scratch | [8][3 dpad] sv | [8][2 kMaxPref] sc | [8] flags
__host__ __device__ inline size_t rec_tables_floats(int P, int d) { return static_cast<size_t>(2) * P * ((d + 3) & ~3); }

// ---- flat forward: scores[i] = model(a[i], b[i], c[i]) -----------------------------------
template <int FAM, int NCH, bool VEC>
__global__ void __launch_bounds__(kThreads)
k_score_fwd(const kgrec_tables T, const int ktup, const IdxArgs I, const int64_t n, const float* __restrict__ gumbel_u,
            const SeedRef seed_ref, float* __restrict__ scores, int32_t* status) {
  extern __shared__ __align__(16) float smem[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t first = static_cast<int64_t>(blockIdx.x) * kWarpsPerCta + wid;
  const int64_t step = static_cast<int64_t>(gridDim.x) * kWarpsPerCta;
  if constexpr (FAM == FAM_REC) {
    const uint64_t seed = seed_ref.get();
    const int stride = (T.dim + 3) & ~3;
    float* sP = smem;
    float* sN = smem + T.n_pref * stride;
    float* scr = sN + T.n_pref * stride + wid * 3 * kMaxPref;
    stage_pref_tables(T, ktup, sP, sN, stride);
    __syncthreads();
    const PrefView pv{sP, sN, T.n_pref, stride, ktup ? 0.5f : 1.f};
    for (int64_t i = first; i < n; i += step) {
      const int64_t iu = checked(load_idx(I.a, i, I.is64), T.n_user, status);
      const int64_t ii = checked(load_idx(I.b, i, I.is64), T.n_item, status);
      RecPair<NCH, VEC> p;
      p.load(T, ktup, iu, ii, ktup ? __ldg(T.item2ent + ii) : 0, lane);
      const float s = p.score(T, pv, gumbel_u ? gumbel_u + i * T.n_pref : nullptr, seed, static_cast<uint64_t>(i), scr, lane);
      if (lane == 0) scores[i] = s;
    }
  } else {
    float* scr = smem + wid * 128 * NCH;
    for (int64_t i = first; i < n; i += step) {
      const int64_t ih = checked(load_idx(I.a, i, I.is64), T.n_ent, status);
      const int64_t it = checked(load_idx(I.b, i, I.is64), T.n_ent, status);
      const int64_t ir = checked(load_idx(I.c, i, I.is64), T.n_rel, status);
      KgTriple<FAM, NCH, VEC> t;
      t.load(T, ih, it, ir, lane);
      const float s = t.score(T, FAM == FAM_R ? T.proj + ir * static_cast<int64_t>(T.dim) * T.dim : nullptr, scr, lane);
      if (lane == 0) scores[i] = s;
    }
  }
}

// ---- fused positive + K negatives + ranking-loss terms -------------------------------------
// One warp per positive.  The positive's rows stay in registers; a negative re-reads only
// the rows whose id differs from the positive's (corrupt-head / corrupt-tail sampling,
// utils/data.py:12-56, changes exactly one of them), which brings the traffic per scored
// triple from 3 rows down to (3 + K) / (1 + K).
template <int FAM, int NCH, bool VEC>
__global__ void __launch_bounds__(kThreads)
k_rank_loss_fwd(const kgrec_tables T, const int ktup, const IdxArgs I, const LossCfg L,
                const float* __restrict__ gumbel_u, const SeedRef seed_ref, float* __restrict__ pos_scores,
                float* __restrict__ neg_scores, float* __restrict__ group_loss, int32_t* status) {
  extern __shared__ __align__(16) float smem[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int K = L.n_neg;
  const int64_t first = static_cast<int64_t>(blockIdx.x) * kWarpsPerCta + wid;
  const int64_t step = static_cast<int64_t>(gridDim.x) * kWarpsPerCta;
  using R = Row<NCH, VEC>;
  constexpr int NE = NCH * 4;
  if constexpr (FAM == FAM_REC) {
    const uint64_t seed = seed_ref.get();
    const int stride = (T.dim + 3) & ~3;
    float* sP = smem;
    float* sN = smem + T.n_pref * stride;
    float* scr = sN + T.n_pref * stride + wid * 3 * kMaxPref;
    stage_pref_tables(T, ktup, sP, sN, stride);
    __syncthreads();
    const PrefView pv{sP, sN, T.n_pref, stride, ktup ? 0.5f : 1.f};
    for (int64_t j = first; j < L.n_pos; j += step) {
      const int64_t iu = checked(load_idx(I.a, j, I.is64), T.n_user, status);
      const int64_t ii = checked(load_idx(I.b, j, I.is64), T.n_item, status);
      RecPair<NCH, VEC> p;
      p.load(T, ktup, iu, ii, ktup ? __ldg(T.item2ent + ii) : 0, lane);
      const float sp = p.score(T, pv, gumbel_u ? gumbel_u + j * T.n_pref : nullptr, seed, static_cast<uint64_t>(j), scr, lane);
      if (lane == 0) pos_scores[j] = sp;
      float lsum = 0.f;
      for (int k = 0; k < K; ++k) {
        const int64_t m = j * K + k;
        const int64_t nu = checked(load_idx(I.na, m, I.is64), T.n_user, status);
        const int64_t ni = checked(load_idx(I.nb, m, I.is64), T.n_item, status);
        if (nu != iu) R::load(p.u, T.user + nu * T.ld, T.dim, lane);   // (never, with the reference sampler)
        p.load_item(T, ktup, ni, ktup ? __ldg(T.item2ent + ni) : 0, lane);
        const uint64_t pid = static_cast<uint64_t>(L.n_pos + m);
        const float sn = p.score(T, pv, gumbel_u ? gumbel_u + pid * T.n_pref : nullptr, seed, pid, scr, lane);
        if (lane == 0) neg_scores[m] = sn;
        lsum += loss_term(L, sp, sn);
        if (nu != iu) R::load(p.u, T.user + iu * T.ld, T.dim, lane);
      }
      if (lane == 0) group_loss[j] = lsum;
    }
  } else {
    float* scr = smem + wid * 128 * NCH;
    for (int64_t j = first; j < L.n_pos; j += step) {
      const int64_t ih = checked(load_idx(I.a, j, I.is64), T.n_ent, status);
      const int64_t it = checked(load_idx(I.b, j, I.is64), T.n_ent, status);
      const int64_t ir = checked(load_idx(I.c, j, I.is64), T.n_rel, status);
      // ids of the first negative are requested together with the positive's rows
      int64_t nh = 0, nt = 0, nr = 0;
      if (K > 0) {
        nh = load_idx(I.na, j * K, I.is64);
        nt = load_idx(I.nb, j * K, I.is64);
        nr = load_idx(I.nc, j * K, I.is64);
      }
      KgTriple<FAM, NCH, VEC> p;
      p.load(T, ih, it, ir, lane);
      const float sp = p.score(T, FAM == FAM_R ? T.proj + ir * static_cast<int64_t>(T.dim) * T.dim : nullptr, scr, lane);
      if (lane == 0) pos_scores[j] = sp;
      float lsum = 0.f;
      for (int k = 0; k < K; ++k) {
        const int64_t m = j * K + k;
        nh = checked(nh, T.n_ent, status);
        nt = checked(nt, T.n_ent, status);
        nr = checked(nr, T.n_rel, status);
        KgTriple<FAM, NCH, VEC> q;
        if (nh == ih) {
#pragma unroll
          for (int i = 0; i < NE; ++i) q.h[i] = p.h[i];
        } else R::load(q.h, T.ent + nh * T.ld, T.dim, lane);
        if (nt == it) {
#pragma unroll
          for (int i = 0; i < NE; ++i) q.t[i] = p.t[i];
        } else R::load(q.t, T.ent + nt * T.ld, T.dim, lane);
        if (nr == ir) {
#pragma unroll
          for (int i = 0; i < NE; ++i) { q.r[i] = p.r[i]; if (FAM == FAM_H) q.w[i] = p.w[i]; }
        } else {
          R::load(q.r, T.rel + nr * T.ld, T.dim, lane);
          if (FAM == FAM_H) R::load(q.w, T.norm + nr * T.ld, T.dim, lane);
        }
        const int64_t cr = nr;
        if (k + 1 < K) {   // next negative's ids in flight while this one computes
          nh = load_idx(I.na, m + 1, I.is64);
          nt = load_idx(I.nb, m + 1, I.is64);
          nr = load_idx(I.nc, m + 1, I.is64);
        }
        const float sn = q.score(T, FAM == FAM_R ? T.proj + cr * static_cast<int64_t>(T.dim) * T.dim : nullptr, scr, lane);
        if (lane == 0) neg_scores[m] = sn;
        lsum += loss_term(L, sp, sn);
      }
      if (lane == 0) group_loss[j] = lsum;
    }
  }
}

// ---- backward ------------------------------------------------------------------------------
// Flat over n triples.  The upstream dLoss/dscore is either read from grad_scores or, for the
// fused ranking loss, formed here from the saved scores (upstream_grad).
template <int FAM, int NCH, bool VEC, int PR>
__global__ void __launch_bounds__(kThreads)
k_score_bwd(const kgrec_tables T, const int ktup, const IdxArgs I, const int64_t n, const LossCfg L,
            const float* __restrict__ gumbel_u, const SeedRef seed_ref, const BwdArgs B, const kgrec_grads G) {
  extern __shared__ __align__(16) float smem[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const bool fused = B.pos_scores != nullptr;
  using R = Row<NCH, VEC>;
  constexpr int NE = NCH * 4;

  if constexpr (FAM == FAM_REC) {
    const uint64_t seed = seed_ref.get();
    const int d = T.dim, P = T.n_pref;
    const int stride = (d + 3) & ~3;
    constexpr int dpad = NCH * 128;
    float* sP = smem;
    float* sN = sP + P * stride;
    float* scr_all = sN + P * stride;                        // [8][3 kMaxPref]
    float* sv_all = scr_all + kWarpsPerCta * 3 * kMaxPref;   // [8][3][dpad]
    float* sc_all = sv_all + kWarpsPerCta * 3 * dpad;        // [8][2][kMaxPref]
    int* sact = reinterpret_cast<int*>(sc_all + kWarpsPerCta * 2 * kMaxPref);
    stage_pref_tables(T, ktup, sP, sN, stride);
    __syncthreads();
    const PrefView pv{sP, sN, P, stride, ktup ? 0.5f : 1.f};
    float accp[PR][NE], accn[PR][NE];   // this warp's rows wid, wid + 8, ... of the two table gradients
#pragma unroll
    for (int m = 0; m < PR; ++m)
#pragma unroll
      for (int e = 0; e < NE; ++e) { accp[m][e] = 0.f; accn[m][e] = 0.f; }

    for (int64_t base = static_cast<int64_t>(blockIdx.x) * kWarpsPerCta; base < n;
         base += static_cast<int64_t>(gridDim.x) * kWarpsPerCta) {
      const int64_t i = base + wid;
      if (i < n) {
        const bool isneg = fused && i >= L.n_pos;
        const int64_t li = isneg ? i - L.n_pos : i;
        const int64_t iu = load_idx(isneg ? I.na : I.a, li, I.is64);
        const int64_t ii = load_idx(isneg ? I.nb : I.b, li, I.is64);
        const int64_t ia = ktup ? __ldg(T.item2ent + ii) : 0;
        float* scr = scr_all + wid * 3 * kMaxPref;
        RecPair<NCH, VEC> p;
        p.load(T, ktup, iu, ii, ia, lane);
        p.score(T, pv, gumbel_u ? gumbel_u + i * P : nullptr, seed, static_cast<uint64_t>(i), scr, lane);
        const float g = upstream_grad(B, L, i, lane);
        float gu[NE], gi[NE];
        p.backward(T, pv, g, scr, lane, gu, gi, sv_all + wid * 3 * dpad, sc_all + wid * 2 * kMaxPref, dpad);
        if (G.mode == 0) {
          R::store_cs(G.user + i * d, gu, d, lane);
          R::store_cs(G.item + i * d, gi, d, lane);
          if (ktup) {
            if (ia == T.n_ent - 1) {  // padding row: no gradient (jTransUP.py:96)
#pragma unroll
              for (int e = 0; e < NE; ++e) gi[e] = 0.f;
            }
            R::store_cs(G.ent + i * d, gi, d, lane);
          }
        } else {
          R::red_add(G.user + iu * d, gu, d, lane);
          R::red_add(G.item + ii * d, gi, d, lane);
          if (ktup && ia != T.n_ent - 1) R::red_add(G.ent + ia * d, gi, d, lane);
        }
      }
      if (lane == 0) sact[wid] = (i < n);
      __syncthreads();
      // CTA-wide accumulation of the [P, d] table gradients: a thread-owned register tile
      for (int q = 0; q < kWarpsPerCta; ++q) {
        if (!sact[q]) continue;
        const float* sv = sv_all + q * 3 * dpad;
        const float* sc = sc_all + q * 2 * kMaxPref;
        float ve[NE], vg[NE], vs[NE];
        R::load_s(ve, sv, dpad, lane);
        R::load_s(vg, sv + dpad, dpad, lane);
        R::load_s(vs, sv + 2 * dpad, dpad, lane);
#pragma unroll
        for (int m = 0; m < PR; ++m) {
          const int k = wid + kWarpsPerCta * m;
          if (k < P) {
            const float ca = sc[k], cb = sc[kMaxPref + k];
#pragma unroll
            for (int e = 0; e < NE; ++e) {
              accp[m][e] = fmaf(ca, ve[e], fmaf(cb, vs[e], accp[m][e]));
              accn[m][e] = fmaf(ca, vg[e], accn[m][e]);
            }
          }
        }
      }
      __syncthreads();
    }
#pragma unroll
    for (int m = 0; m < PR; ++m) {
      const int k = wid + kWarpsPerCta * m;
      if (k < P) {
        R::red_add(G.pref + static_cast<int64_t>(k) * d, accp[m], d, lane);
        R::red_add(G.pref_norm + static_cast<int64_t>(k) * d, accn[m], d, lane);
      }
    }
  } else {
    float* scr = smem + wid * 128 * NCH;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * kWarpsPerCta + wid; i < n;
         i += static_cast<int64_t>(gridDim.x) * kWarpsPerCta) {
      const bool isneg = fused && i >= L.n_pos;
      const int64_t li = isneg ? i - L.n_pos : i;
      const int64_t ih = load_idx(isneg ? I.na : I.a, li, I.is64);
      const int64_t it = load_idx(isneg ? I.nb : I.b, li, I.is64);
      const int64_t ir = load_idx(isneg ? I.nc : I.c, li, I.is64);
      const float* m = FAM == FAM_R ? T.proj + ir * static_cast<int64_t>(T.dim) * T.dim : nullptr;
      KgTriple<FAM, NCH, VEC> t;
      t.load(T, ih, it, ir, lane);
      t.score(T, m, scr, lane);
      t.backward(T, G, m, scr, ih, it, ir, i, n, upstream_grad(B, L, i, lane), lane);
    }
  }
}

// per-batch deterministic reduction of the group terms (one CTA per loss batch)
static __global__ void __launch_bounds__(256)
k_batch_loss(const float* __restrict__ group_loss, const LossCfg L, float* __restrict__ loss) {
  __shared__ float part[8];
  const int64_t b0 = static_cast<int64_t>(blockIdx.x) * L.batch_pos;
  const int64_t cnt = min(L.batch_pos, L.n_pos - b0);
  float s = 0.f;
  for (int64_t i = threadIdx.x; i < cnt; i += blockDim.x) s += group_loss[b0 + i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += part[w];
    if (L.kind == KGREC_LOSS_BPR) t /= (static_cast<float>(cnt) * static_cast<float>(L.n_neg));
    loss[blockIdx.x] = t;
  }
}


// ===========================================================================================
// host-side launchers (one explicit instantiation per family, each in its own .cu)
// ===========================================================================================
inline int grid_for(int64_t n_units) {
  const int64_t ctas = (n_units + kWarpsPerCta - 1) / kWarpsPerCta;
  const int64_t cap = static_cast<int64_t>(sm_count()) * 8;  // 8 x 256 threads = one SM's thread capacity
  return static_cast<int>(ctas < 1 ? 1 : (ctas < cap ? ctas : cap));
}

template <typename K>
int set_smem(K kernel, size_t bytes) {
  if (bytes > 48 * 1024)
    KGREC_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes)));
  return KGREC_OK;
}

// variants built: 128-bit path for d <= 128 / 256 / 512, scalar path (d % 4 != 0) for d <= 128 / 512
#define KGREC_DISPATCH_ROW(...)                                                    \
  if (!pl.vec && pl.nch == 1) { constexpr int NCH = 1; constexpr bool VEC = false; __VA_ARGS__ } \
  else if (!pl.vec)     { constexpr int NCH = 4; constexpr bool VEC = false; __VA_ARGS__ } \
  else if (pl.nch == 1) { constexpr int NCH = 1; constexpr bool VEC = true;  __VA_ARGS__ } \
  else if (pl.nch == 2) { constexpr int NCH = 2; constexpr bool VEC = true;  __VA_ARGS__ } \
  else                  { constexpr int NCH = 4; constexpr bool VEC = true;  __VA_ARGS__ }

// TUP / KTUP pairs in large flat batches go through the tile engine (train_rec_tile.cu); these
// return -1 when the shape is outside what it is built for (small n, d > 128, P > 32, unaligned)
// and the one-warp-per-pair kernels below take the call.
int rec_tile_score_fwd(const kgrec_tables& T, const Plan& pl, const IdxArgs& I, int64_t n, const float* gumbel_u,
                       SeedRef seed, float* scores, int32_t* status, cudaStream_t st);
int rec_tile_rank_loss_fwd(const kgrec_tables& T, const Plan& pl, const IdxArgs& I, const LossCfg& L,
                           const float* gumbel_u, SeedRef seed, float* pos_scores, float* neg_scores,
                           float* group_loss, int32_t* status, cudaStream_t st);
int rec_tile_score_bwd(const kgrec_tables& T, const Plan& pl, const IdxArgs& I, int64_t n, const LossCfg& L,
                       const float* gumbel_u, SeedRef seed, const BwdArgs& B, const kgrec_grads& G, cudaStream_t st);
int rec_tile_loss_step(const kgrec_tables& T, const Plan& pl, const IdxArgs& I, const LossCfg& L, float grad_loss,
                       const float* gumbel_u, SeedRef seed, float* pos_scores, float* neg_scores, float* group_loss,
                       const kgrec_grads& G, int64_t* slot_user, int64_t* slot_item, int64_t* slot_ent, int32_t* status,
                       cudaStream_t st);
int rec_slot_ids(const kgrec_tables& T, const Plan& pl, const IdxArgs& I, int64_t n_pos, int64_t n, int64_t* su, int64_t* si,
                 int64_t* se, cudaStream_t st);

template <int FAM>
int launch_score_fwd(const kgrec_tables& T, const Plan& pl, const IdxArgs& I, int64_t n, const float* gumbel_u,
                     SeedRef seed, float* scores, int32_t* status, cudaStream_t st) {
  int rc = KGREC_OK;
  if constexpr (FAM == FAM_REC) {
    if ((rc = rec_tile_score_fwd(T, pl, I, n, gumbel_u, seed, scores, status, st)) >= 0) return rc;
  }
  KGREC_DISPATCH_ROW({
    auto kern = k_score_fwd<FAM, NCH, VEC>;
    if ((rc = set_smem(kern, pl.smem_fwd))) return rc;
    kern<<<grid_for(n), kThreads, pl.smem_fwd, st>>>(T, pl.ktup, I, n, gumbel_u, seed, scores, status);
  })
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

template <int FAM>
int launch_rank_loss_fwd(const kgrec_tables& T, const Plan& pl, const IdxArgs& I, const LossCfg& L,
                         const float* gumbel_u, SeedRef seed, float* pos_scores, float* neg_scores,
                         float* group_loss, int32_t* status, cudaStream_t st) {
  int rc = KGREC_OK;
  if constexpr (FAM == FAM_REC) {
    if ((rc = rec_tile_rank_loss_fwd(T, pl, I, L, gumbel_u, seed, pos_scores, neg_scores, group_loss, status, st)) >= 0)
      return rc;
  }
  KGREC_DISPATCH_ROW({
    auto kern = k_rank_loss_fwd<FAM, NCH, VEC>;
    if ((rc = set_smem(kern, pl.smem_fwd))) return rc;
    kern<<<grid_for(L.n_pos), kThreads, pl.smem_fwd, st>>>(T, pl.ktup, I, L, gumbel_u, seed, pos_scores, neg_scores,
                                                          group_loss, status);
  })
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

template <int FAM>
int launch_score_bwd(const kgrec_tables& T, const Plan& pl, const IdxArgs& I, int64_t n, const LossCfg& L,
                     const float* gumbel_u, SeedRef seed, const BwdArgs& B, const kgrec_grads& G, cudaStream_t st) {
  int rc = KGREC_OK;
  if constexpr (FAM == FAM_REC) {
    if ((rc = rec_tile_score_bwd(T, pl, I, n, L, gumbel_u, seed, B, G, st)) >= 0) return rc;
#define KGREC_BWD_REC(PRV)                                                                                  \
  {                                                                                                         \
    auto kern = k_score_bwd<FAM_REC, NCH, VEC, PRV>;                                                        \
    if ((rc = set_smem(kern, pl.smem_bwd))) return rc;                                                      \
    kern<<<grid_for(n), kThreads, pl.smem_bwd, st>>>(T, pl.ktup, I, n, L, gumbel_u, seed, B, G);            \
  }
    // preference rows per warp: P <= 32 -> 4, P <= 64 -> 8 (d <= 128 only); wide rows: P <= 32 / 16
    KGREC_DISPATCH_ROW({
      if constexpr (NCH == 1) { if (pl.pr <= 4) KGREC_BWD_REC(4) else KGREC_BWD_REC(8) }
      else if constexpr (NCH == 2) KGREC_BWD_REC(4)
      else KGREC_BWD_REC(2)
    })
#undef KGREC_BWD_REC
  } else {
    KGREC_DISPATCH_ROW({
      auto kern = k_score_bwd<FAM, NCH, VEC, 1>;
      if ((rc = set_smem(kern, pl.smem_fwd))) return rc;
      kern<<<grid_for(n), kThreads, pl.smem_fwd, st>>>(T, 0, I, n, L, gumbel_u, seed, B, G);
    })
  }
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

#define KGREC_INSTANTIATE_FAMILY(FAMV)                                                                            \
  template int launch_score_fwd<FAMV>(const kgrec_tables&, const Plan&, const IdxArgs&, int64_t, const float*,    \
                                      SeedRef, float*, int32_t*, cudaStream_t);                                  \
  template int launch_rank_loss_fwd<FAMV>(const kgrec_tables&, const Plan&, const IdxArgs&, const LossCfg&,       \
                                          const float*, SeedRef, float*, float*, float*, int32_t*, cudaStream_t); \
  template int launch_score_bwd<FAMV>(const kgrec_tables&, const Plan&, const IdxArgs&, int64_t, const LossCfg&,  \
                                      const float*, SeedRef, const BwdArgs&, const kgrec_grads&, cudaStream_t);

}  // namespace kgrec
