// Row-factored training step for TUP / KTUP with SOFT preferences (use_st_gumbel = 0: the mode of the reference's shipped
// scripts, transup.sh / ktup.sh `-nouse_st_gumbel`; transUP.py:69-82, 105-115, jTransUP.py:122-161, 250-260).
//
// With raw logits as mixing weights everything the preference induction does is LINEAR in s = u + i':
//     z = s P'^T / 2,   r = hf z P' = RA_u + RA_i,   w = hf z N' = WB_u + WB_i,     RA_x = hf (x P'^T / 2) P',  WB_x likewise with N'
// so the nine [P x d] contractions the pair kernel (train_rec_tile.cu) spends per PAIR can be spent per DISTINCT ROW of a
// step instead -- a step of 256 batches touches each of 50k users ~10 times, each of 6k users of an ml1m-sized rec side ~90
// times (SURVEY 7.3-1 points at the same factorisation for evaluation):
//   k_rows_compact     marked rows (the optimizer's epoch marks) -> a dense list per table
//   k_soft_rows_fwd    per listed row: zx = x P'^T / 2 [P], RA_x, WB_x [d]   (KTUP items: x = item + ent[item2ent], also stored)
//   k_soft_pairs       per group (positive + its negatives, one warp): r, w by two adds; a = u - i', s = a.w,
//                      e = a + r - s w, score, ranking loss, then eps, gx = eps - (eps.w) w, gw = -((eps.w) a + s eps);
//                      O(d) per pair; gradients leave as atomic row adds: gx -> the rows' direct gradient, eps -> G_RA, gw -> G_WB
//   k_soft_rows_bwd    per listed row: g_z = hf (G_RA P'^T + G_WB N'^T), row gradient += g_z P' / 2
//   k_soft_rows_tables the table gradients dP' += hf zx^T G_RA + g_z^T x / 2, dN' += hf zx^T G_WB as a [P x n] . [n x d] product over the
//                      listed rows (a thread owns a column chunk x half of the preferences in registers; one flush per CTA)
// All of it accumulates into the dense accumulators of the sparse-row optimizer (csrc/optim.cu), which then clips and updates.
// Same arithmetic as the pair kernel up to re-association; parity: tests/test_gpu_parity.py::test_sparse_row_optimizer_rec_models.
#include "train_dev.cuh"

namespace kgrec {
namespace {

constexpr int kRowThreads = 256;

__global__ void __launch_bounds__(256)
k_rows_compact(const int32_t* __restrict__ marks, int64_t rows, int32_t epoch_arg, const kgrec_step_state* state,
               int32_t* __restrict__ list, int32_t* __restrict__ count) {
  const int32_t epoch = state ? state->epoch : epoch_arg;
  const int lane = threadIdx.x & 31;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  for (int64_t c = warp; c * 32 < rows; c += n_warps) {
    const int64_t row = c * 32 + lane;
    const bool mine = row < rows && __ldg(marks + row) == epoch;
    const unsigned m = __ballot_sync(FULL, mine);
    if (!m) continue;
    int base = 0;
    if (lane == 0) base = atomicAdd(count, __popc(m));
    base = __shfl_sync(FULL, base, 0);
    if (mine) list[base + __popc(m & ((1u << lane) - 1u))] = static_cast<int32_t>(row);
  }
}

struct SoftRows {                 // one side (users or items) of the rec model
  const float* table;             // [rows, d] parameter rows
  const float* ent;               // KTUP items: entity table, else NULL
  const int32_t* item2ent;
  int64_t n_ent;
  float* x;                       // KTUP items: effective rows item + ent [rows, d]; else NULL (x = table)
  float *ra, *wb;                 // [rows, d]
  float* zx;                      // [rows, P]
  float *g_ra, *g_wb;             // [rows, d] accumulators, zeroed again by the backward
  float* gx;                      // direct row gradient: the table's dense accumulator, or (KTUP items) a work buffer
  float *acc_table, *acc_ent;     // KTUP items: where gx + logit path goes
  const int32_t* list;
  const int32_t* count;
};

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 add4(const float4& a, const float4& b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 sub4(const float4& a, const float4& b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
__device__ __forceinline__ float dot4(const float4& a, const float4& b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w))); }
__device__ __forceinline__ float4 axpy4(float s, const float4& x, const float4& y) {
  return make_float4(fmaf(s, x.x, y.x), fmaf(s, x.y, y.y), fmaf(s, x.z, y.z), fmaf(s, x.w, y.w));
}

// ---- per-row kernels: a thread owns (row, slice) -- 8 rows x 4 slices of interleaved 16-byte chunks per warp, the tile
// kernel's mapping: a table chunk is one broadcast LDS.128 feeding 4 FMAs per preference, a dot over d costs two
// xor-shuffles, nothing is staged per row.  Tables chunk-major in shared memory: chunk c of preference k at [c * PT + k].
template <int PT>
__device__ __forceinline__ void stage_tables_cm(const kgrec_tables& T, int ktup, float4* sP, float4* sN) {
  const int NC = T.dim >> 2, P = T.n_pref;
  for (int idx = threadIdx.x; idx < PT * NC; idx += blockDim.x) {
    const int k = idx / NC, c = idx - k * NC;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (k < P) {
      a = ldg_f4(reinterpret_cast<const float4*>(T.pref + static_cast<int64_t>(k) * T.ld) + c);
      b = ldg_f4(reinterpret_cast<const float4*>(T.pref_norm + static_cast<int64_t>(k) * T.ld) + c);
      if (ktup) {
        const float4 r = ldg_f4(reinterpret_cast<const float4*>(T.rel + static_cast<int64_t>(k) * T.ld) + c);
        const float4 w = ldg_f4(reinterpret_cast<const float4*>(T.norm + static_cast<int64_t>(k) * T.ld) + c);
        a.x += r.x; a.y += r.y; a.z += r.z; a.w += r.w;
        b.x += w.x; b.y += w.y; b.z += w.z; b.w += w.w;
      }
    }
    sP[c * PT + k] = a;
    sN[c * PT + k] = b;
  }
}
__device__ __forceinline__ float qsum4(float v) {   // all-reduce over the 4 slices of a row
  v += __shfl_xor_sync(FULL, v, 8);
  v += __shfl_xor_sync(FULL, v, 16);
  return v;
}
constexpr int kMaxChunks = 8;        // chunks per slice: d <= 128

template <int PT>
__global__ void __launch_bounds__(kRowThreads)
k_soft_rows_fwd(const kgrec_tables T, const int ktup, const SoftRows S) {
  extern __shared__ __align__(16) float sm[];
  const int d = T.dim, P = T.n_pref, NC = d >> 2, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float4* sP = reinterpret_cast<float4*>(sm);
  float4* sN = sP + PT * NC;
  stage_tables_cm<PT>(T, ktup, sP, sN);
  __syncthreads();
  const float hf = ktup ? 0.5f : 1.f;
  const int slot = lane & 7, q = lane >> 3;
  const int n = *S.count;
  for (int base = blockIdx.x * 64; base < n; base += gridDim.x * 64) {
    const int i = base + wid * 8 + slot;
    const bool valid = i < n;
    const int64_t row = valid ? S.list[i] : 0;
    float4 x[kMaxChunks];
    int64_t ia = 0;
    if (S.ent && valid) ia = __ldg(S.item2ent + row);
#pragma unroll
    for (int j = 0; j < kMaxChunks; ++j) {
      const int c = q + 4 * j;
      x[j] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c < NC && valid) {
        x[j] = ldg_f4(reinterpret_cast<const float4*>(S.table + row * T.ld) + c);
        if (S.ent) {
          const float4 e = ldg_f4(reinterpret_cast<const float4*>(S.ent + ia * T.ld) + c);
          x[j].x += e.x; x[j].y += e.y; x[j].z += e.z; x[j].w += e.w;
          reinterpret_cast<float4*>(S.x + row * d)[c] = x[j];
        }
      }
    }
    float z[PT];
#pragma unroll
    for (int k = 0; k < PT; ++k) z[k] = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxChunks; ++j) {
      const int c = q + 4 * j;
      if (c < NC) {
#pragma unroll
        for (int k = 0; k < PT; ++k) z[k] += dot4(x[j], sP[c * PT + k]);
      }
    }
#pragma unroll
    for (int k = 0; k < PT; ++k) {
      z[k] = 0.5f * qsum4(z[k]);
      if (valid && k < P && (k & 3) == q) S.zx[row * P + k] = z[k];
    }
#pragma unroll
    for (int j = 0; j < kMaxChunks; ++j) {
      const int c = q + 4 * j;
      if (c < NC && valid) {
        float4 ra = make_float4(0.f, 0.f, 0.f, 0.f), wb = ra;
#pragma unroll
        for (int k = 0; k < PT; ++k) {
          const float zz = hf * z[k];
          ra = axpy4(zz, sP[c * PT + k], ra);
          wb = axpy4(zz, sN[c * PT + k], wb);
        }
        reinterpret_cast<float4*>(S.ra + row * d)[c] = ra;
        reinterpret_cast<float4*>(S.wb + row * d)[c] = wb;
      }
    }
  }
}

struct SoftPairs {
  const void *pu, *pi, *ni;
  int is64;
  LossCfg L;
  float grad_loss;
  int64_t n_user, n_item;
  const float *xu, *xi;           // effective rows [rows, d] (pitch ldu / ldi)
  int64_t ldu, ldi;
  const float *ra_u, *wb_u, *ra_i, *wb_i;
  float *gx_u, *gx_i, *g_ra_u, *g_wb_u, *g_ra_i, *g_wb_i;
  float *pos_scores, *neg_scores, *group_loss;
  int32_t* status;
  int d, l1;
  // optional: the driver's normLoss over the batch's user rows and cat[pos, neg] item rows (item_recommendation.py:177-179),
  // value added to *reg_loss, gradient 2 x folded into the rows' direct gradient (TUP; the rows are in registers here)
  float* reg_loss;
  float reg_scale;
};

__global__ void __launch_bounds__(kThreads, 4)
k_soft_pairs(const SoftPairs A) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int d = A.d, K = A.L.n_neg;
  const bool act = lane * 4 < d;
  const int64_t n_pos = A.L.n_pos;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  bool bad = false;
  for (int64_t j = static_cast<int64_t>(blockIdx.x) * kWarpsPerCta + wid; j < n_pos; j += static_cast<int64_t>(gridDim.x) * kWarpsPerCta) {
    int64_t iu = load_idx(A.pu, j, A.is64);
    if (static_cast<uint64_t>(iu) >= static_cast<uint64_t>(A.n_user)) { bad = true; iu = 0; }
    // lane m holds the item id of member m (0 = the positive)
    int64_t idm = 0;
    if (lane <= K) {
      idm = lane == 0 ? load_idx(A.pi, j, A.is64) : load_idx(A.ni, j * K + lane - 1, A.is64);
      if (static_cast<uint64_t>(idm) >= static_cast<uint64_t>(A.n_item)) { bad = true; idm = 0; }
    }
    float4 u = z4, rau = z4, wbu = z4;
    if (act) {
      u = ld4(A.xu + iu * A.ldu + 4 * lane);
      rau = ld4(A.ra_u + iu * d + 4 * lane);
      wbu = ld4(A.wb_u + iu * d + 4 * lane);
    }
    float reg_sum = 0.f, my_n2 = 0.f;
    const bool reg = A.reg_loss != nullptr;
    const float n2u = reg ? warp_sum(dot4(u, u)) : 0.f;
    if (reg && n2u > 1.f) reg_sum += n2u - 1.f;
    // pass 1: scores (lane m keeps member m's score and s = a.w)
    float my_score = 0.f, my_s = 0.f;
    for (int m = 0; m <= K; ++m) {
      const int64_t id = __shfl_sync(FULL, idm, m);
      float4 x = z4, r = z4, w = z4;
      if (act) {
        x = ld4(A.xi + id * A.ldi + 4 * lane);
        r = add4(rau, ld4(A.ra_i + id * d + 4 * lane));
        w = add4(wbu, ld4(A.wb_i + id * d + 4 * lane));
      }
      const float4 a = sub4(u, x);
      const float s = warp_sum(dot4(a, w));
      const float4 e = axpy4(-s, w, add4(a, r));
      float sc = dist_term(e.x, A.l1) + dist_term(e.y, A.l1) + dist_term(e.z, A.l1) + dist_term(e.w, A.l1);
      float n2x = reg ? dot4(x, x) : 0.f;
      if (reg) warp_sum2(sc, n2x); else sc = warp_sum(sc);
      if (reg && n2x > 1.f) reg_sum += n2x - 1.f;
      if (lane == m) { my_score = sc; my_s = s; my_n2 = n2x; }
    }
    const float sp = __shfl_sync(FULL, my_score, 0);
    // ranking loss of the group and its derivative (utils/loss.py:8-16, 29-31)
    const float up = A.grad_loss * loss_batch_scale(A.L, j);
    float term = 0.f, dp = 0.f;
    if (lane >= 1 && lane <= K) { term = loss_term(A.L, sp, my_score); dp = loss_dpos(A.L, sp, my_score); }
    const float lsum = warp_sum(term), dsum = warp_sum(dp);
    const float my_g = lane == 0 ? dsum * up : -dp * up;          // dLoss / dscore of member `lane`
    if (lane == 0) { A.pos_scores[j] = sp; A.group_loss[j] = lsum; }
    if (lane >= 1 && lane <= K) A.neg_scores[j * K + lane - 1] = my_score;
    // pass 2: gradients
    float4 gu = z4, gra = z4, gwb = z4;
    for (int m = 0; m <= K; ++m) {
      const float g = __shfl_sync(FULL, my_g, m);
      const bool regx = reg && __shfl_sync(FULL, my_n2, m) > 1.f;
      if (g == 0.f && !regx) continue;                            // warp-uniform (inactive hinge, row inside the unit ball)
      const int64_t id = __shfl_sync(FULL, idm, m);
      const float s = __shfl_sync(FULL, my_s, m);
      float4 x = z4, r = z4, w = z4;
      if (act) {
        x = ld4(A.xi + id * A.ldi + 4 * lane);
        r = add4(rau, ld4(A.ra_i + id * d + 4 * lane));
        w = add4(wbu, ld4(A.wb_i + id * d + 4 * lane));
      }
      const float4 a = sub4(u, x);
      const float4 e = axpy4(-s, w, add4(a, r));
      const float4 eps = make_float4(g * ddist_term(e.x, A.l1), g * ddist_term(e.y, A.l1), g * ddist_term(e.z, A.l1), g * ddist_term(e.w, A.l1));
      const float ew = warp_sum(dot4(eps, w));
      const float4 gx = axpy4(-ew, w, eps);                                       // eps - (eps.w) w
      const float4 gw = make_float4(-fmaf(ew, a.x, s * eps.x), -fmaf(ew, a.y, s * eps.y), -fmaf(ew, a.z, s * eps.z), -fmaf(ew, a.w, s * eps.w));
      gu = add4(gu, gx); gra = add4(gra, eps); gwb = add4(gwb, gw);
      float4 gxi = make_float4(-gx.x, -gx.y, -gx.z, -gx.w);
      if (regx) gxi = axpy4(2.f * A.reg_scale, x, gxi);
      if (act) {
        red_add_f4(A.gx_i + id * d + 4 * lane, gxi.x, gxi.y, gxi.z, gxi.w);
        red_add_f4(A.g_ra_i + id * d + 4 * lane, eps.x, eps.y, eps.z, eps.w);
        red_add_f4(A.g_wb_i + id * d + 4 * lane, gw.x, gw.y, gw.z, gw.w);
      }
    }
    if (reg && n2u > 1.f) gu = axpy4(2.f * A.reg_scale, u, gu);
    if (reg && lane == 0 && reg_sum != 0.f) atomicAdd(A.reg_loss, A.reg_scale * reg_sum);
    if (act) {
      red_add_f4(A.gx_u + iu * d + 4 * lane, gu.x, gu.y, gu.z, gu.w);
      red_add_f4(A.g_ra_u + iu * d + 4 * lane, gra.x, gra.y, gra.z, gra.w);
      red_add_f4(A.g_wb_u + iu * d + 4 * lane, gwb.x, gwb.y, gwb.z, gwb.w);
    }
  }
  if (bad && A.status) *A.status = 1;
}

// backward, part a: g_z = hf (G_RA P'^T + G_WB N'^T) -> cb[row] = g_z / 2, and the row gradient += (g_z / 2) P'
template <int PT>
__global__ void __launch_bounds__(kRowThreads)
k_soft_rows_bwd(const kgrec_tables T, const int ktup, const SoftRows S, float* __restrict__ cb) {
  extern __shared__ __align__(16) float sm[];
  const int d = T.dim, P = T.n_pref, NC = d >> 2, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float4* sP = reinterpret_cast<float4*>(sm);
  float4* sN = sP + PT * NC;
  stage_tables_cm<PT>(T, ktup, sP, sN);
  __syncthreads();
  const float hf = ktup ? 0.5f : 1.f;
  const int slot = lane & 7, q = lane >> 3;
  const int n = *S.count;
  for (int base = blockIdx.x * 64; base < n; base += gridDim.x * 64) {
    const int i = base + wid * 8 + slot;
    const bool valid = i < n;
    const int64_t row = valid ? S.list[i] : 0;
    float gz[PT];
#pragma unroll
    for (int k = 0; k < PT; ++k) gz[k] = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxChunks; ++j) {
      const int c = q + 4 * j;
      if (c < NC && valid) {
        const float4 gra = ld4(S.g_ra + row * d + 4 * c), gwb = ld4(S.g_wb + row * d + 4 * c);
#pragma unroll
        for (int k = 0; k < PT; ++k) gz[k] += dot4(gra, sP[c * PT + k]) + dot4(gwb, sN[c * PT + k]);
      }
    }
#pragma unroll
    for (int k = 0; k < PT; ++k) {
      gz[k] = 0.5f * hf * qsum4(gz[k]);
      if (valid && k < P && (k & 3) == q) cb[row * P + k] = gz[k];
    }
    int64_t ia = 0;
    if (S.acc_table && valid) ia = __ldg(S.item2ent + row);
#pragma unroll
    for (int j = 0; j < kMaxChunks; ++j) {
      const int c = q + 4 * j;
      if (c < NC && valid) {
        float4 gs = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int k = 0; k < PT; ++k) gs = axpy4(gz[k], sP[c * PT + k], gs);
        if (S.acc_table) {                   // KTUP items: direct gradient from the work buffer; item and aligned entity both get the sum
          float4 t = ld4(S.gx + row * d + 4 * c);
          reinterpret_cast<float4*>(S.gx + row * d)[c] = make_float4(0.f, 0.f, 0.f, 0.f);
          t = add4(t, gs);
          float4* ai = reinterpret_cast<float4*>(S.acc_table + row * d) + c;
          *ai = add4(*ai, t);
          if (ia != S.n_ent - 1) red_add_f4(S.acc_ent + ia * d + 4 * c, t.x, t.y, t.z, t.w);     // padding row: no gradient (jTransUP.py:96)
        } else {
          float4* gp = reinterpret_cast<float4*>(S.gx + row * d) + c;
          *gp = add4(*gp, gs);
        }
      }
    }
  }
}

// backward, part b: the [P, d] table gradients as a [P x n] . [n x d] product over the listed rows:
//   dP'[k] += sum_rows hf zx[row][k] G_RA[row] + cb[row][k] x[row];   dN'[k] += sum_rows hf zx[row][k] G_WB[row]
// A thread owns (16-byte column chunk, half of the preferences) in registers over all the rows of its row group.
template <int PT>
__global__ void __launch_bounds__(kRowThreads, (PT <= 20 ? 2 : 1))
k_soft_rows_tables(const kgrec_tables T, const int ktup, const SoftRows S, const float* __restrict__ cb,
                   float* __restrict__ acc_pref, float* __restrict__ acc_pref_norm) {
  constexpr int KH = PT / 2;
  const int d = T.dim, P = T.n_pref, NC = d >> 2;
  const float hf = ktup ? 0.5f : 1.f;
  const int items = NC * 2, ngrp = kRowThreads / items;
  const int grp = threadIdx.x / items, item = threadIdx.x - grp * items;
  const int jc = item % NC, k0 = (item / NC) * KH;
  if (grp >= ngrp) return;
  float4 accP[KH], accN[KH];
#pragma unroll
  for (int k = 0; k < KH; ++k) { accP[k] = make_float4(0.f, 0.f, 0.f, 0.f); accN[k] = accP[k]; }
  const int n = *S.count;
  for (int i = blockIdx.x * ngrp + grp; i < n; i += gridDim.x * ngrp) {
    const int64_t row = S.list[i];
    const float4 gra = ld4(S.g_ra + row * d + 4 * jc), gwb = ld4(S.g_wb + row * d + 4 * jc);
    const float4 x = S.x ? ld4(S.x + row * d + 4 * jc) : ldg_f4(reinterpret_cast<const float4*>(S.table + row * T.ld) + jc);
#pragma unroll
    for (int k = 0; k < KH; ++k) {
      if (k0 + k < P) {
        const float za = hf * __ldg(S.zx + row * P + k0 + k), zb = __ldg(cb + row * P + k0 + k);
        accP[k] = axpy4(za, gra, axpy4(zb, x, accP[k]));
        accN[k] = axpy4(za, gwb, accN[k]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < KH; ++k) {
    if (k0 + k < P) {
      red_add_f4(acc_pref + static_cast<int64_t>(k0 + k) * d + 4 * jc, accP[k].x, accP[k].y, accP[k].z, accP[k].w);
      red_add_f4(acc_pref_norm + static_cast<int64_t>(k0 + k) * d + 4 * jc, accN[k].x, accN[k].y, accN[k].z, accN[k].w);
    }
  }
}

// the per-row accumulators are clean again for the next step
__global__ void __launch_bounds__(256)
k_rows_zero2(const int32_t* __restrict__ list, const int32_t* __restrict__ count, float* __restrict__ a, float* __restrict__ b, int d) {
  const int n = *count, NC = d >> 2;
  const int64_t total = static_cast<int64_t>(n) * NC;
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t row = list[t / NC];
    const int c = static_cast<int>(t % NC);
    reinterpret_cast<float4*>(a + row * d)[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    reinterpret_cast<float4*>(b + row * d)[c] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// =====================================================================================================================
// ST-Gumbel preferences, squared-L2 score (use_st_gumbel = 1, L1_flag = 0): transUP.py:143-170.
// The forward picks ONE preference per pair, k* = arg-max_k z_k + g_k with z = (u + i') P'^T / 2 = A_u + A_i, so r = hf P'_k*,
// w = hf N'_k* are table rows and s = a.w = hf (CN_u[k*] - CN_i[k*]) with CN_x = x N'^T.  The straight-through backward needs
// dL/dp_k = hf (eps . P'_k + gw . N'_k) for EVERY k; with eps = 2 g e (L2) and e = a + r - s w these dots are O(1) from the
// per-row A / CN and the [P, P] Gram tables PP = P' P'^T, NP = N' P'^T, NN = N' N'^T:
//     eps . P'_k = 2 g (2 (A_u - A_i)[k] + hf PP[k*][k] - s hf NP[k*][k])
//     eps . N'_k = 2 g ((CN_u - CN_i)[k] + hf NP[k][k*] - s hf NN[k*][k])
//     gp_k = hf (eps . P'_k - ew (CN_u - CN_i)[k] - s eps . N'_k),      gz = y (gp - <y, gp>),  y = softmax(z + g)
// (lane k of the warp handles preference k).  What is left per pair is O(d): e and gx = eps - ew w.  The one-hot table rows
// dP'_k* += hf eps and dN'_k* += hf gw are NOT added per pair (d-wide atomics on P hot rows): with c1 = 2 g hf, t2 = hf ew + s c1
//     hf eps = c1 (u - i' + R_k* - s W_k*),      hf gw = -t2 (u - i') - s c1 R_k* + s^2 c1 W_k*
// so a pair adds four scalars to per-row coefficient vectors (CK_u[k*] += c1, CK_i[k*] -= c1, DK_u[k*] -= t2, DK_i[k*] += t2)
// and four to per-preference sums (S1..S4[k*] in shared memory), and the d-wide work happens once per DISTINCT row.  The logit
// path -- row gradient += (gz / 2) P', dP' += (gz / 2)^T (u + i') -- is linear in the rows too (GZ_x = sum of the row's gz):
//     dP' += (GZ / 2 + CK)^T X + S1 R - S2 W,        dN' += DK^T X + S3 R + S4 W        (R = hf P', W = hf N').
// =====================================================================================================================
__global__ void __launch_bounds__(256)
k_gumbel_gram(const kgrec_tables T, const int ktup, float* __restrict__ gram) {      // gram: [3][P][P] = PP | NP | NN
  const int d = T.dim, P = T.n_pref, lane = threadIdx.x & 31;
  const int wq = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (wq >= P * P) return;
  const int j = wq / P, k = wq - j * P;
  float pp = 0.f, np = 0.f, nn = 0.f;
  for (int t = lane; t < d; t += 32) {
    float pj = __ldg(T.pref + static_cast<int64_t>(j) * T.ld + t), pk = __ldg(T.pref + static_cast<int64_t>(k) * T.ld + t);
    float nj = __ldg(T.pref_norm + static_cast<int64_t>(j) * T.ld + t), nk = __ldg(T.pref_norm + static_cast<int64_t>(k) * T.ld + t);
    if (ktup) {
      pj += __ldg(T.rel + static_cast<int64_t>(j) * T.ld + t); pk += __ldg(T.rel + static_cast<int64_t>(k) * T.ld + t);
      nj += __ldg(T.norm + static_cast<int64_t>(j) * T.ld + t); nk += __ldg(T.norm + static_cast<int64_t>(k) * T.ld + t);
    }
    pp = fmaf(pj, pk, pp); np = fmaf(nj, pk, np); nn = fmaf(nj, nk, nn);
  }
  warp_sum2(pp, np);
  nn = warp_sum(nn);
  if (lane == 0) { gram[wq] = pp; gram[P * P + wq] = np; gram[2 * P * P + wq] = nn; }
}

struct GumbelRows {
  const float* table; const float* ent; const int32_t* item2ent; int64_t n_ent;
  float* x;                        // KTUP items: effective rows
  float *a, *cn;                   // [rows, P] logit halves x.P'_k / 2 and normal dots x.N'_k
  float *gz;                       // [rows, P] accumulated logit gradients, zeroed again by the backward
  float *ck;                       // [rows, 2, P] coefficients of this row in the one-hot table gradients dP'_k*, dN'_k* (zeroed likewise)
  float *cb, *cbn;                 // [rows, P] gz / 2 + ck and dk: the coefficient matrices of the table-gradient products
  float* gx; float *acc_table, *acc_ent;
  const int32_t* list; const int32_t* count;
};

template <int PT>
__global__ void __launch_bounds__(kRowThreads)
k_gumbel_rows_fwd(const kgrec_tables T, const int ktup, const GumbelRows S) {
  extern __shared__ __align__(16) float sm[];
  const int d = T.dim, P = T.n_pref, NC = d >> 2, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float4* sP = reinterpret_cast<float4*>(sm);
  float4* sN = sP + PT * NC;
  stage_tables_cm<PT>(T, ktup, sP, sN);
  __syncthreads();
  const int slot = lane & 7, q = lane >> 3;
  const int n = *S.count;
  for (int base = blockIdx.x * 64; base < n; base += gridDim.x * 64) {
    const int i = base + wid * 8 + slot;
    const bool valid = i < n;
    const int64_t row = valid ? S.list[i] : 0;
    int64_t ia = 0;
    if (S.ent && valid) ia = __ldg(S.item2ent + row);
    float za[PT], zc[PT];
#pragma unroll
    for (int k = 0; k < PT; ++k) { za[k] = 0.f; zc[k] = 0.f; }
#pragma unroll
    for (int j = 0; j < kMaxChunks; ++j) {
      const int c = q + 4 * j;
      if (c < NC && valid) {
        float4 x = ldg_f4(reinterpret_cast<const float4*>(S.table + row * T.ld) + c);
        if (S.ent) {
          x = add4(x, ldg_f4(reinterpret_cast<const float4*>(S.ent + ia * T.ld) + c));
          reinterpret_cast<float4*>(S.x + row * d)[c] = x;
        }
#pragma unroll
        for (int k = 0; k < PT; ++k) { za[k] += dot4(x, sP[c * PT + k]); zc[k] += dot4(x, sN[c * PT + k]); }
      }
    }
#pragma unroll
    for (int k = 0; k < PT; ++k) {
      const float a = 0.5f * qsum4(za[k]), c = qsum4(zc[k]);
      if (valid && k < P && (k & 3) == q) { S.a[row * P + k] = a; S.cn[row * P + k] = c; }
    }
  }
}

struct GumbelPairs {
  const void *pu, *pi, *ni;
  int is64;
  LossCfg L;
  float grad_loss;
  int64_t n_user, n_item;
  const float *xu, *xi; int64_t ldu, ldi;
  const float *a_u, *cn_u, *a_i, *cn_i;
  float *gx_u, *gx_i, *gz_u, *gz_i, *ck_u, *ck_i;
  float *acc_pref, *acc_pref_norm;
  const float* gram;                 // [3][P][P]
  const float* gumbel_u; SeedRef seed;
  float *pos_scores, *neg_scores, *group_loss;
  int32_t* status;
  kgrec_tables T; int ktup;
  float* reg_loss;                 // TUP driver's normLoss over cat[u], cat[pos items, neg items] (item_recommendation.py:177-179), or NULL
  float reg_scale;
};

__global__ void __launch_bounds__(kThreads, 4)
k_gumbel_pairs(const GumbelPairs A) {
  extern __shared__ __align__(16) float sm[];
  const kgrec_tables& T = A.T;
  const int d = T.dim, P = T.n_pref, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float* sR = sm;                    // [P][d] hf P'
  float* sW = sR + P * d;            // [P][d] hf N'
  float* sS = sW + P * d;            // [4][P] per-preference sums S1..S4 of this CTA
  float* sG = sS + 4 * P;            // [3][P][P]
  float* sV = sG + 3 * P * P + (threadIdx.x >> 5) * (A.L.n_neg + 1) * P;     // this warp's z + noise of every member: [K + 1][P]
  const float hf = A.ktup ? 0.5f : 1.f;
  for (int idx = threadIdx.x; idx < P * d; idx += blockDim.x) {
    const int k = idx / d, j = idx - k * d;
    float a = __ldg(T.pref + static_cast<int64_t>(k) * T.ld + j), b = __ldg(T.pref_norm + static_cast<int64_t>(k) * T.ld + j);
    if (A.ktup) { a += __ldg(T.rel + static_cast<int64_t>(k) * T.ld + j); b += __ldg(T.norm + static_cast<int64_t>(k) * T.ld + j); }
    sR[idx] = hf * a; sW[idx] = hf * b;
  }
  for (int idx = threadIdx.x; idx < 4 * P; idx += blockDim.x) sS[idx] = 0.f;
  for (int idx = threadIdx.x; idx < 3 * P * P; idx += blockDim.x) sG[idx] = __ldg(A.gram + idx);
  __syncthreads();
  const int K = A.L.n_neg;
  const bool act = lane * 4 < d, kl = lane < P;
  const int64_t n_pos = A.L.n_pos;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  bool bad = false;
  // arg-max over the lanes < P with the lowest index among equals (torch.max): one integer redux on the order-preserving
  // key of the float, one ballot
  auto okey = [&](float v) {
    const uint32_t b = __float_as_uint(v);
    return kl ? ((b & 0x80000000u) ? ~b : (b | 0x80000000u)) : 0u;
  };
  auto argmax = [&](float v) {
    const uint32_t key = okey(v);
    const uint32_t mx = __reduce_max_sync(FULL, key);
    return __ffs(__ballot_sync(FULL, key == mx)) - 1;
  };
  for (int64_t j = static_cast<int64_t>(blockIdx.x) * kWarpsPerCta + wid; j < n_pos; j += static_cast<int64_t>(gridDim.x) * kWarpsPerCta) {
    int64_t iu = load_idx(A.pu, j, A.is64);
    if (static_cast<uint64_t>(iu) >= static_cast<uint64_t>(A.n_user)) { bad = true; iu = 0; }
    int64_t idm = 0;
    if (lane <= K) {
      idm = lane == 0 ? load_idx(A.pi, j, A.is64) : load_idx(A.ni, j * K + lane - 1, A.is64);
      if (static_cast<uint64_t>(idm) >= static_cast<uint64_t>(A.n_item)) { bad = true; idm = 0; }
    }
    float4 u = z4;
    if (act) u = ld4(A.xu + iu * A.ldu + 4 * lane);
    const float au = kl ? __ldg(A.a_u + iu * P + lane) : 0.f, cu = kl ? __ldg(A.cn_u + iu * P + lane) : 0.f;
    const bool reg = A.reg_loss != nullptr;
    const float n2u = reg ? warp_sum(dot4(u, u)) : 0.f;
    float reg_sum = (reg && n2u > 1.f) ? n2u - 1.f : 0.f, my_n2 = 0.f;
    // Gumbel noise of the whole group, [K + 1][P]: explicit uniforms (parity runs), or ONE Philox block per four values
    // (all members at once: a Philox call is a warp-wide instruction stream, so it is spent on the group, not per member)
    __syncwarp();
    if (A.gumbel_u) {
      for (int m = 0; m <= K; ++m) {
        const int64_t pid = m == 0 ? j : n_pos + j * K + (m - 1);
        if (kl) sV[m * P + lane] = gumbel_from_uniform(__ldg(A.gumbel_u + pid * P + lane));
      }
    } else {
      const uint64_t seed = A.seed.get();
      const int n_vals = (K + 1) * P;
      for (int b = lane; 4 * b < n_vals; b += 32) {
        const uint4 r = philox4(seed, static_cast<uint64_t>(j), static_cast<uint32_t>(b));
        const uint32_t w4[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int t = 0; t < 4; ++t)
          if (4 * b + t < n_vals) sV[4 * b + t] = gumbel_fast(w4[t]);
      }
    }
    __syncwarp();
    // pass 1: scores; lane m keeps member m's score, k* and s
    float my_score = 0.f, my_s = 0.f;
    int my_k = 0;
    for (int m = 0; m <= K; ++m) {
      const int64_t id = __shfl_sync(FULL, idm, m);
      const float ax = kl ? __ldg(A.a_i + id * P + lane) : 0.f, cx = kl ? __ldg(A.cn_i + id * P + lane) : 0.f;
      float v = 0.f;
      if (kl) { v = au + ax + sV[m * P + lane]; sV[m * P + lane] = v; }          // z + noise, kept for the backward
      const int ks = argmax(v);
      const float s = hf * __shfl_sync(FULL, cu - cx, ks);
      float4 x = z4, r = z4, w = z4;
      if (act) { x = ld4(A.xi + id * A.ldi + 4 * lane); r = ld4(sR + ks * d + 4 * lane); w = ld4(sW + ks * d + 4 * lane); }
      const float4 e = axpy4(-s, w, add4(sub4(u, x), r));
      float sc = dot4(e, e), n2x = reg ? dot4(x, x) : 0.f;
      if (reg) warp_sum2(sc, n2x); else sc = warp_sum(sc);
      if (reg && n2x > 1.f) reg_sum += n2x - 1.f;
      if (lane == m) { my_score = sc; my_s = s; my_k = ks; my_n2 = n2x; }
    }
    const float sp = __shfl_sync(FULL, my_score, 0);
    const float up = A.grad_loss * loss_batch_scale(A.L, j);
    float term = 0.f, dp = 0.f;
    if (lane >= 1 && lane <= K) { term = loss_term(A.L, sp, my_score); dp = loss_dpos(A.L, sp, my_score); }
    const float lsum = warp_sum(term), dsum = warp_sum(dp);
    const float my_g = lane == 0 ? dsum * up : -dp * up;
    if (lane == 0) { A.pos_scores[j] = sp; A.group_loss[j] = lsum; }
    if (lane >= 1 && lane <= K) A.neg_scores[j * K + lane - 1] = my_score;
    // pass 2: gradients
    float4 gu = z4;
    float gzu = 0.f;
    for (int m = 0; m <= K; ++m) {
      const float g = __shfl_sync(FULL, my_g, m);
      const bool regx = reg && __shfl_sync(FULL, my_n2, m) > 1.f;
      if (g == 0.f && !regx) continue;
      const int64_t id = __shfl_sync(FULL, idm, m);
      if (g == 0.f) {              // inactive hinge, row outside the unit ball: the regulariser's gradient only
        if (act) {
          const float4 x = ld4(A.xi + id * A.ldi + 4 * lane);
          const float c = 2.f * A.reg_scale;
          red_add_f4(A.gx_i + id * d + 4 * lane, c * x.x, c * x.y, c * x.z, c * x.w);
        }
        continue;
      }
      const int ks = __shfl_sync(FULL, my_k, m);
      const float s = __shfl_sync(FULL, my_s, m);
      const float ax = kl ? __ldg(A.a_i + id * P + lane) : 0.f, cx = kl ? __ldg(A.cn_i + id * P + lane) : 0.f;
      const float v = kl ? sV[m * P + lane] : 0.f;
      const float mx = __shfl_sync(FULL, v, ks);                  // the arg-max's value
      const float ex = kl ? __expf(v - mx) : 0.f;
      const float y = __fdividef(ex, warp_sum(ex));
      float4 x = z4, r = z4, w = z4;
      if (act) { x = ld4(A.xi + id * A.ldi + 4 * lane); r = ld4(sR + ks * d + 4 * lane); w = ld4(sW + ks * d + 4 * lane); }
      const float4 a = sub4(u, x);
      const float4 e = axpy4(-s, w, add4(a, r));
      const float g2 = 2.f * g;
      const float4 eps = make_float4(g2 * e.x, g2 * e.y, g2 * e.z, g2 * e.w);
      const float ew = warp_sum(dot4(eps, w));
      const float4 gx = axpy4(-ew, w, eps);
      // dL/dp_k for every k (lane k), O(1) from the Gram tables
      float gz = 0.f;
      {
        float gp = 0.f;
        if (kl) {
          const float da = au - ax, dc = cu - cx;
          const float epk = g2 * (2.f * da + hf * sG[ks * P + lane] - s * hf * sG[P * P + ks * P + lane]);
          const float enk = g2 * (dc + hf * sG[P * P + lane * P + ks] - s * hf * sG[2 * P * P + ks * P + lane]);
          gp = hf * (epk - ew * dc - s * enk);
        }
        const float yg = warp_sum(y * gp);
        gz = y * (gp - yg);
      }
      gu = add4(gu, gx);
      gzu += gz;
      if (act) {
        float4 gxi = make_float4(-gx.x, -gx.y, -gx.z, -gx.w);
        if (regx) gxi = axpy4(2.f * A.reg_scale, x, gxi);
        red_add_f4(A.gx_i + id * d + 4 * lane, gxi.x, gxi.y, gxi.z, gxi.w);
      }
      if (lane < 4) {   // one-hot table gradients: eight scalars instead of two d-wide rows (lanes 0/1: user ck/dk, 2/3: item)
        const float c1 = g2 * hf, t2 = fmaf(hf, ew, s * c1);
        const bool usr = lane < 2, isd = lane & 1;
        float* row = usr ? A.ck_u + iu * 2 * P : A.ck_i + id * 2 * P;
        const float v = isd ? t2 : c1;
        atomicAdd(row + (isd ? P : 0) + ks, (usr != isd) ? v : -v);      // ck_u += c1, dk_u -= t2, ck_i -= c1, dk_i += t2
        const float sv = lane == 0 ? c1 : (lane == 1 ? c1 * s : (lane == 2 ? -s * c1 : s * s * c1));
        atomicAdd(sS + lane * P + ks, sv);
      }
      if (kl) atomicAdd(A.gz_i + id * P + lane, gz);
    }
    if (reg && n2u > 1.f) gu = axpy4(2.f * A.reg_scale, u, gu);
    if (reg && lane == 0 && reg_sum != 0.f) atomicAdd(A.reg_loss, A.reg_scale * reg_sum);
    if (act) red_add_f4(A.gx_u + iu * d + 4 * lane, gu.x, gu.y, gu.z, gu.w);
    if (kl && gzu != 0.f) atomicAdd(A.gz_u + iu * P + lane, gzu);
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < P * d; idx += blockDim.x) {        // this CTA's share of S1 R - S2 W and S3 R + S4 W
    const int k = idx / d;
    const float r = sR[idx], w = sW[idx];
    const float dp = sS[k] * r - sS[P + k] * w, dn = sS[2 * P + k] * r + sS[3 * P + k] * w;
    if (dp != 0.f) atomicAdd(A.acc_pref + idx, dp);
    if (dn != 0.f) atomicAdd(A.acc_pref_norm + idx, dn);
  }
  if (bad && A.status) *A.status = 1;
}

// backward per row: cb = GZ / 2 + CK, cbn = DK (accumulators cleared), row gradient += (GZ / 2) P'
template <int PT>
__global__ void __launch_bounds__(kRowThreads)
k_gumbel_rows_bwd(const kgrec_tables T, const int ktup, const GumbelRows S) {
  extern __shared__ __align__(16) float sm[];
  const int d = T.dim, P = T.n_pref, NC = d >> 2, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float4* sP = reinterpret_cast<float4*>(sm);
  float4* sN = sP + PT * NC;
  stage_tables_cm<PT>(T, ktup, sP, sN);
  __syncthreads();
  const int slot = lane & 7, q = lane >> 3;
  const int n = *S.count;
  for (int base = blockIdx.x * 64; base < n; base += gridDim.x * 64) {
    const int i = base + wid * 8 + slot;
    const bool valid = i < n;
    const int64_t row = valid ? S.list[i] : 0;
    float gz[PT];
#pragma unroll
    for (int k = 0; k < PT; ++k) gz[k] = (valid && k < P) ? 0.5f * S.gz[row * P + k] : 0.f;
    __syncwarp();
#pragma unroll
    for (int k = 0; k < PT; ++k)
      if (valid && k < P && (k & 3) == q) {
        S.cb[row * P + k] = gz[k] + S.ck[row * 2 * P + k];
        S.cbn[row * P + k] = S.ck[row * 2 * P + P + k];
        S.gz[row * P + k] = 0.f; S.ck[row * 2 * P + k] = 0.f; S.ck[row * 2 * P + P + k] = 0.f;
      }
    int64_t ia = 0;
    if (S.acc_table && valid) ia = __ldg(S.item2ent + row);
#pragma unroll
    for (int j = 0; j < kMaxChunks; ++j) {
      const int c = q + 4 * j;
      if (c < NC && valid) {
        float4 gs = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int k = 0; k < PT; ++k) gs = axpy4(gz[k], sP[c * PT + k], gs);
        if (S.acc_table) {
          float4 t = ld4(S.gx + row * d + 4 * c);
          reinterpret_cast<float4*>(S.gx + row * d)[c] = make_float4(0.f, 0.f, 0.f, 0.f);
          t = add4(t, gs);
          float4* ai = reinterpret_cast<float4*>(S.acc_table + row * d) + c;
          *ai = add4(*ai, t);
          if (ia != S.n_ent - 1) red_add_f4(S.acc_ent + ia * d + 4 * c, t.x, t.y, t.z, t.w);
        } else {
          float4* gp = reinterpret_cast<float4*>(S.gx + row * d) + c;
          *gp = add4(*gp, gs);
        }
      }
    }
  }
}

// dP'[k] += sum_rows cb[row][k] x[row];  dN'[k] += sum_rows cbn[row][k] x[row]
template <int PT>
__global__ void __launch_bounds__(kRowThreads, (PT <= 20 ? 2 : 1))
k_gumbel_rows_tables(const kgrec_tables T, const GumbelRows S, float* __restrict__ acc_pref, float* __restrict__ acc_pref_norm) {
  constexpr int KH = PT / 2;
  const int d = T.dim, P = T.n_pref, NC = d >> 2;
  const int items = NC * 2, ngrp = kRowThreads / items;
  const int grp = threadIdx.x / items, item = threadIdx.x - grp * items;
  const int jc = item % NC, k0 = (item / NC) * KH;
  if (grp >= ngrp) return;
  float4 accP[KH], accN[KH];
#pragma unroll
  for (int k = 0; k < KH; ++k) { accP[k] = make_float4(0.f, 0.f, 0.f, 0.f); accN[k] = accP[k]; }
  const int n = *S.count;
  for (int i = blockIdx.x * ngrp + grp; i < n; i += gridDim.x * ngrp) {
    const int64_t row = S.list[i];
    const float4 x = S.x ? ld4(S.x + row * d + 4 * jc) : ldg_f4(reinterpret_cast<const float4*>(S.table + row * T.ld) + jc);
#pragma unroll
    for (int k = 0; k < KH; ++k)
      if (k0 + k < P) {
        accP[k] = axpy4(__ldg(S.cb + row * P + k0 + k), x, accP[k]);
        accN[k] = axpy4(__ldg(S.cbn + row * P + k0 + k), x, accN[k]);
      }
  }
#pragma unroll
  for (int k = 0; k < KH; ++k)
    if (k0 + k < P) {
      red_add_f4(acc_pref + static_cast<int64_t>(k0 + k) * d + 4 * jc, accP[k].x, accP[k].y, accP[k].z, accP[k].w);
      red_add_f4(acc_pref_norm + static_cast<int64_t>(k0 + k) * d + 4 * jc, accN[k].x, accN[k].y, accN[k].z, accN[k].w);
    }
}

}  // namespace
}  // namespace kgrec

using namespace kgrec;

extern "C" int64_t kgrec_rec_rows_workspace_floats(int64_t n_user, int64_t n_item, int32_t dim, int32_t n_pref, int ktup) {
  // per side: ra, wb, g_ra, g_wb [rows, d], zx [rows, P], list [rows] (+1 count); KTUP items: x, gx [rows, d]
  const int64_t per = 4 * static_cast<int64_t>(dim) + 8 * static_cast<int64_t>(n_pref) + 8;     // covers the soft and the ST-Gumbel layouts
  return n_user * per + n_item * (per + (ktup ? 2 * static_cast<int64_t>(dim) : 0)) + 3 * static_cast<int64_t>(n_pref) * n_pref + 64;
}

static int rec_rows_step(const kgrec_tables* tables, int model, const void* pu, const void* pi, const void* ni, int idx_bytes,
                         int64_t n_pos, int32_t n_neg, int64_t batch_pos, int loss_kind, float margin_or_target,
                         float grad_loss, const int32_t* marks_user, const int32_t* marks_item, int32_t epoch,
                         const kgrec_step_state* state, float* workspace, int32_t first_use, const kgrec_grads* acc,
                         float* pos_scores, float* neg_scores, float* loss, void* loss_workspace, float* norm_reg_loss,
                         const float* gumbel_u, uint64_t seed, int32_t* status, kgrec_stream_t stream) {
  if (!tables || (model != KGREC_TUP && model != KGREC_KTUP)) { set_error("rec_rows_step: TUP / KTUP"); return KGREC_ERR_INVALID; }
  const kgrec_tables& T = *tables;
  const int d = T.dim, P = T.n_pref;
  const bool ktup = model == KGREC_KTUP;
  if (T.use_gumbel && T.l1) { set_error("rec_rows_step with use_st_gumbel is built for the squared-L2 score (L1_flag = 0)"); return KGREC_ERR_UNSUPPORTED; }
  if (d <= 0 || d > 128 || d % 4 || T.ld != d || P <= 0 || P > 32 || n_neg < 1 || n_neg > 31) {
    set_error("rec_rows_step: embedding_size %% 4 == 0 and <= 128, contiguous tables, preference_total <= 32, 1..31 negatives per positive");
    return KGREC_ERR_UNSUPPORTED;
  }
  if (!T.user || !T.item || !T.pref || !T.pref_norm || (ktup && (!T.ent || !T.rel || !T.norm || !T.item2ent))) { set_error("rec_rows_step: table missing"); return KGREC_ERR_INVALID; }
  if (!pu || !pi || !ni || (idx_bytes != 4 && idx_bytes != 8) || n_pos < 0 || batch_pos < 1 || !marks_user || !marks_item || !workspace || !acc ||
      acc->mode != 1 || !acc->user || !acc->item || !acc->pref || !acc->pref_norm || (ktup && !acc->ent) || !pos_scores || !neg_scores || !loss ||
      !loss_workspace) {
    set_error("rec_rows_step: NULL / bad argument (gradients go to dense accumulators, grads->mode 1)");
    return KGREC_ERR_INVALID;
  }
  if (loss_kind != KGREC_LOSS_MARGIN && loss_kind != KGREC_LOSS_BPR) { set_error("unknown loss %d", loss_kind); return KGREC_ERR_INVALID; }
  if (n_pos == 0) return KGREC_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // carve the workspace
  float* w = workspace;
  auto take = [&](int64_t n) { float* p = w; w += (n + 3) & ~static_cast<int64_t>(3); return p; };
  const int64_t nu = T.n_user, nit = T.n_item;
  const int cap = sm_count() * 8;
  auto grid1 = [&](int64_t units) { const int64_t g = units < 1 ? 1 : units; return static_cast<int>(g < cap ? g : cap); };
  // rows touched: at most min(rows, ids) per side
  const int64_t max_u = nu < n_pos ? nu : n_pos, max_i = nit < n_pos * (1 + n_neg) ? nit : n_pos * (1 + n_neg);
  const int PT = P <= 8 ? 8 : (P <= 20 ? 20 : 32);
  const size_t smem_t = static_cast<size_t>(2) * PT * (d / 4) * sizeof(float4);
  const int rcap = sm_count() * 4;
  auto grid64 = [&](int64_t rows) { const int64_t g = (rows + 63) / 64; return static_cast<int>(g < 1 ? 1 : (g < rcap ? g : rcap)); };
  const int tcap = sm_count() * 2;
  auto gridt = [&](int64_t rows) { const int64_t g = (rows + 31) / 32; return static_cast<int>(g < 1 ? 1 : (g < tcap ? g : tcap)); };
  const int64_t n_batches = (n_pos + batch_pos - 1) / batch_pos;
  if (T.use_gumbel) {
    if (norm_reg_loss && ktup) { set_error("rec_rows_step: the row-norm regulariser is the TUP driver's (item_recommendation.py:177-179)"); return KGREC_ERR_UNSUPPORTED; }
    GumbelRows GU{}, GI{};
    GU.table = T.user; GI.table = T.item;
    GU.a = take(nu * P); GU.cn = take(nu * P); GU.gz = take(nu * P); GU.ck = take(2 * nu * P);
    GU.cb = take(nu * P); GU.cbn = take(nu * P);
    GI.a = take(nit * P); GI.cn = take(nit * P); GI.gz = take(nit * P); GI.ck = take(2 * nit * P);
    GI.cb = take(nit * P); GI.cbn = take(nit * P);
    float* gxb = nullptr;
    if (ktup) { GI.x = take(nit * d); gxb = take(nit * d); }
    int32_t* gl_u = reinterpret_cast<int32_t*>(take(nu));
    int32_t* gl_i = reinterpret_cast<int32_t*>(take(nit));
    int32_t* gcnt = reinterpret_cast<int32_t*>(take(4));
    float* gram = take(3 * static_cast<int64_t>(P) * P);
    if (first_use) {
      KGREC_CUDA_OK(cudaMemsetAsync(GU.gz, 0, sizeof(float) * nu * P, st));
      KGREC_CUDA_OK(cudaMemsetAsync(GU.ck, 0, sizeof(float) * 2 * nu * P, st));
      KGREC_CUDA_OK(cudaMemsetAsync(GI.gz, 0, sizeof(float) * nit * P, st));
      KGREC_CUDA_OK(cudaMemsetAsync(GI.ck, 0, sizeof(float) * 2 * nit * P, st));
      if (ktup) KGREC_CUDA_OK(cudaMemsetAsync(gxb, 0, sizeof(float) * nit * d, st));
    }
    KGREC_CUDA_OK(cudaMemsetAsync(gcnt, 0, 4 * sizeof(int32_t), st));
    GU.list = gl_u; GU.count = gcnt; GI.list = gl_i; GI.count = gcnt + 1;
    GU.gx = acc->user;
    if (ktup) { GI.ent = T.ent; GI.item2ent = T.item2ent; GI.n_ent = T.n_ent; GI.gx = gxb; GI.acc_table = acc->item; GI.acc_ent = acc->ent; }
    else GI.gx = acc->item;
    k_rows_compact<<<grid1((nu + 255) / 256), 256, 0, st>>>(marks_user, nu, epoch, state, gl_u, gcnt);
    k_rows_compact<<<grid1((nit + 255) / 256), 256, 0, st>>>(marks_item, nit, epoch, state, gl_i, gcnt + 1);
    k_gumbel_gram<<<(P * P * 32 + 255) / 256, 256, 0, st>>>(T, ktup ? 1 : 0, gram);
    KGREC_CUDA_OK(cudaGetLastError());
    GumbelPairs A{};
    A.pu = pu; A.pi = pi; A.ni = ni; A.is64 = idx_bytes == 8;
    A.L = LossCfg{loss_kind, margin_or_target, n_neg, n_pos, batch_pos};
    A.grad_loss = grad_loss; A.n_user = nu; A.n_item = nit;
    A.xu = T.user; A.ldu = T.ld; A.xi = ktup ? GI.x : T.item; A.ldi = ktup ? d : T.ld;
    A.a_u = GU.a; A.cn_u = GU.cn; A.a_i = GI.a; A.cn_i = GI.cn;
    A.gx_u = acc->user; A.gx_i = GI.gx; A.gz_u = GU.gz; A.gz_i = GI.gz;
    A.ck_u = GU.ck; A.ck_i = GI.ck;
    A.acc_pref = acc->pref; A.acc_pref_norm = acc->pref_norm; A.gram = gram; A.gumbel_u = gumbel_u; A.seed = SeedRef(seed, state);
    A.pos_scores = pos_scores; A.neg_scores = neg_scores; A.group_loss = static_cast<float*>(loss_workspace);
    A.status = status; A.T = T; A.ktup = ktup ? 1 : 0;
    A.reg_loss = norm_reg_loss; A.reg_scale = 1.f;
    const size_t smem_p = (static_cast<size_t>(2) * P * d + 4 * static_cast<size_t>(P) + 3 * static_cast<size_t>(P) * P +
                           static_cast<size_t>(kWarpsPerCta) * (n_neg + 1) * P) * sizeof(float);
    KGREC_CUDA_OK(cudaFuncSetAttribute(k_gumbel_pairs, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_p)));
    const int64_t pg = (n_pos + kWarpsPerCta - 1) / kWarpsPerCta, pcap = static_cast<int64_t>(sm_count()) * 4;
#define GROWS(PTV)                                                                                                       \
  {                                                                                                                      \
    KGREC_CUDA_OK(cudaFuncSetAttribute(k_gumbel_rows_fwd<PTV>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_t))); \
    KGREC_CUDA_OK(cudaFuncSetAttribute(k_gumbel_rows_bwd<PTV>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_t))); \
    k_gumbel_rows_fwd<PTV><<<grid64(max_u), kRowThreads, smem_t, st>>>(T, ktup ? 1 : 0, GU);                             \
    k_gumbel_rows_fwd<PTV><<<grid64(max_i), kRowThreads, smem_t, st>>>(T, ktup ? 1 : 0, GI);                             \
    k_gumbel_pairs<<<static_cast<int>(pg < pcap ? pg : pcap), kThreads, smem_p, st>>>(A);                                \
    k_gumbel_rows_bwd<PTV><<<grid64(max_u), kRowThreads, smem_t, st>>>(T, ktup ? 1 : 0, GU);                             \
    k_gumbel_rows_bwd<PTV><<<grid64(max_i), kRowThreads, smem_t, st>>>(T, ktup ? 1 : 0, GI);                             \
    k_gumbel_rows_tables<PTV><<<gridt(max_u), kRowThreads, 0, st>>>(T, GU, acc->pref, acc->pref_norm);                   \
    k_gumbel_rows_tables<PTV><<<gridt(max_i), kRowThreads, 0, st>>>(T, GI, acc->pref, acc->pref_norm);                   \
  }
    if (PT == 8) GROWS(8) else if (PT == 20) GROWS(20) else GROWS(32)
#undef GROWS
    KGREC_CUDA_OK(cudaGetLastError());
    k_batch_loss<<<static_cast<unsigned>(n_batches), 256, 0, st>>>(A.group_loss, A.L, loss);
    KGREC_CUDA_OK(cudaGetLastError());
    return KGREC_OK;
  }
  SoftRows U{}, I{};
  U.table = T.user; I.table = T.item;
  U.ra = take(nu * d); U.wb = take(nu * d); U.g_ra = take(nu * d); U.g_wb = take(nu * d); U.zx = take(nu * P);
  I.ra = take(nit * d); I.wb = take(nit * d); I.g_ra = take(nit * d); I.g_wb = take(nit * d); I.zx = take(nit * P);
  float* gx_i_buf = nullptr;
  if (ktup) { I.x = take(nit * d); gx_i_buf = take(nit * d); }
  float* cb_u = take(nu * P);
  float* cb_i = take(nit * P);
  int32_t* list_u = reinterpret_cast<int32_t*>(take(nu));
  int32_t* list_i = reinterpret_cast<int32_t*>(take(nit));
  int32_t* counts = reinterpret_cast<int32_t*>(take(4));
  if (first_use) {        // accumulators start clean; afterwards the backward leaves them clean
    KGREC_CUDA_OK(cudaMemsetAsync(U.g_ra, 0, sizeof(float) * 2 * nu * d, st));
    KGREC_CUDA_OK(cudaMemsetAsync(I.g_ra, 0, sizeof(float) * 2 * nit * d, st));
    if (ktup) KGREC_CUDA_OK(cudaMemsetAsync(gx_i_buf, 0, sizeof(float) * nit * d, st));
  }
  KGREC_CUDA_OK(cudaMemsetAsync(counts, 0, 4 * sizeof(int32_t), st));
  U.list = list_u; U.count = counts; I.list = list_i; I.count = counts + 1;
  U.gx = acc->user;
  if (ktup) {
    I.ent = T.ent; I.item2ent = T.item2ent; I.n_ent = T.n_ent; I.gx = gx_i_buf; I.acc_table = acc->item; I.acc_ent = acc->ent;
  } else {
    I.gx = acc->item;
  }
  k_rows_compact<<<grid1((nu + 255) / 256), 256, 0, st>>>(marks_user, nu, epoch, state, list_u, counts);
  k_rows_compact<<<grid1((nit + 255) / 256), 256, 0, st>>>(marks_item, nit, epoch, state, list_i, counts + 1);
  KGREC_CUDA_OK(cudaGetLastError());
#define ROWS_FWD(PTV)                                                                                                    \
  {                                                                                                                      \
    KGREC_CUDA_OK(cudaFuncSetAttribute(k_soft_rows_fwd<PTV>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_t))); \
    k_soft_rows_fwd<PTV><<<grid64(max_u), kRowThreads, smem_t, st>>>(T, ktup ? 1 : 0, U);                                \
    k_soft_rows_fwd<PTV><<<grid64(max_i), kRowThreads, smem_t, st>>>(T, ktup ? 1 : 0, I);                                \
  }
  if (PT == 8) ROWS_FWD(8) else if (PT == 20) ROWS_FWD(20) else ROWS_FWD(32)
#undef ROWS_FWD
  KGREC_CUDA_OK(cudaGetLastError());
  SoftPairs A{};
  A.pu = pu; A.pi = pi; A.ni = ni; A.is64 = idx_bytes == 8;
  A.L = LossCfg{loss_kind, margin_or_target, n_neg, n_pos, batch_pos};
  A.grad_loss = grad_loss; A.n_user = nu; A.n_item = nit;
  A.xu = T.user; A.ldu = T.ld;
  A.xi = ktup ? I.x : T.item; A.ldi = ktup ? d : T.ld;
  A.ra_u = U.ra; A.wb_u = U.wb; A.ra_i = I.ra; A.wb_i = I.wb;
  A.gx_u = acc->user; A.gx_i = I.gx; A.g_ra_u = U.g_ra; A.g_wb_u = U.g_wb; A.g_ra_i = I.g_ra; A.g_wb_i = I.g_wb;
  A.pos_scores = pos_scores; A.neg_scores = neg_scores; A.group_loss = static_cast<float*>(loss_workspace);
  A.status = status; A.d = d; A.l1 = T.l1;
  A.reg_loss = norm_reg_loss; A.reg_scale = 1.f;
  if (norm_reg_loss && ktup) { set_error("rec_rows_step: the row-norm regulariser is the TUP driver's (item_recommendation.py:177-179)"); return KGREC_ERR_UNSUPPORTED; }
  k_soft_pairs<<<grid_for(n_pos), kThreads, 0, st>>>(A);
  KGREC_CUDA_OK(cudaGetLastError());
#define ROWS_BWD(PTV)                                                                                                    \
  {                                                                                                                      \
    KGREC_CUDA_OK(cudaFuncSetAttribute(k_soft_rows_bwd<PTV>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_t))); \
    k_soft_rows_bwd<PTV><<<grid64(max_u), kRowThreads, smem_t, st>>>(T, ktup ? 1 : 0, U, cb_u);                          \
    k_soft_rows_bwd<PTV><<<grid64(max_i), kRowThreads, smem_t, st>>>(T, ktup ? 1 : 0, I, cb_i);                          \
    k_soft_rows_tables<PTV><<<gridt(max_u), kRowThreads, 0, st>>>(T, ktup ? 1 : 0, U, cb_u, acc->pref, acc->pref_norm);   \
    k_soft_rows_tables<PTV><<<gridt(max_i), kRowThreads, 0, st>>>(T, ktup ? 1 : 0, I, cb_i, acc->pref, acc->pref_norm);   \
  }
  if (PT == 8) ROWS_BWD(8) else if (PT == 20) ROWS_BWD(20) else ROWS_BWD(32)
#undef ROWS_BWD
  k_rows_zero2<<<grid1((max_u * (d / 4) + 255) / 256), 256, 0, st>>>(list_u, counts, U.g_ra, U.g_wb, d);
  k_rows_zero2<<<grid1((max_i * (d / 4) + 255) / 256), 256, 0, st>>>(list_i, counts + 1, I.g_ra, I.g_wb, d);
  KGREC_CUDA_OK(cudaGetLastError());
  k_batch_loss<<<static_cast<unsigned>(n_batches), 256, 0, st>>>(A.group_loss, A.L, loss);
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

extern "C" int kgrec_rec_rows_step(const kgrec_tables* tables, int model, const void* pu, const void* pi, const void* ni, int idx_bytes,
                                   int64_t n_pos, int32_t n_neg, int64_t batch_pos, int loss_kind, float margin_or_target,
                                   float grad_loss, const int32_t* marks_user, const int32_t* marks_item, int32_t epoch,
                                   float* workspace, int32_t first_use, const kgrec_grads* acc, float* pos_scores,
                                   float* neg_scores, float* loss, void* loss_workspace, float* norm_reg_loss,
                                   const float* gumbel_u, uint64_t seed, int32_t* status, kgrec_stream_t stream) {
  return rec_rows_step(tables, model, pu, pi, ni, idx_bytes, n_pos, n_neg, batch_pos, loss_kind, margin_or_target, grad_loss,
                       marks_user, marks_item, epoch, nullptr, workspace, first_use, acc, pos_scores, neg_scores, loss,
                       loss_workspace, norm_reg_loss, gumbel_u, seed, status, stream);
}

extern "C" int kgrec_rec_rows_step_dev(const kgrec_tables* tables, int model, const void* pu, const void* pi, const void* ni,
                                       int idx_bytes, int64_t n_pos, int32_t n_neg, int64_t batch_pos, int loss_kind,
                                       float margin_or_target, float grad_loss, const int32_t* marks_user,
                                       const int32_t* marks_item, const kgrec_step_state* state, float* workspace,
                                       int32_t first_use, const kgrec_grads* acc, float* pos_scores, float* neg_scores,
                                       float* loss, void* loss_workspace, float* norm_reg_loss, const float* gumbel_u,
                                       int32_t* status, kgrec_stream_t stream) {
  if (!state) { set_error("rec_rows_step: step state is NULL"); return KGREC_ERR_INVALID; }
  return rec_rows_step(tables, model, pu, pi, ni, idx_bytes, n_pos, n_neg, batch_pos, loss_kind, margin_or_target, grad_loss,
                       marks_user, marks_item, 0, state, workspace, first_use, acc, pos_scores, neg_scores, loss,
                       loss_workspace, norm_reg_loss, gumbel_u, 0, status, stream);
}
