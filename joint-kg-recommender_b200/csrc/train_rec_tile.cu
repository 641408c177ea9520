// Tile engine for the TUP / KTUP-rec training path (transUP.py:69-82,105-115,143-170,
// jTransUP.py:122-161,250-315; CPU form: oracle/kg_oracle.py tup_score / _tup_pair_grads).
//
// Per scored pair the preference induction is nine [P x d] contractions (logits, the mixed
// relation / normal, dL/dp, the chain through the logits, three table-gradient products):
// ~18 k FMA against ~1.6 KB of HBM traffic, i.e. FP32-pipe bound, and with the tables in shared
// memory the real limiter is shared-memory wavefronts per FMA.  One warp per pair (the first
// design, train_dev.cuh RecPair) re-reads all 2P table rows from shared memory for every pair
// and needs a shuffle tree per dot.  Here a CTA owns a tile of M = 16 x warps pairs whose
// vectors live in shared memory, and
//   * passes A-E: a thread owns a (pair, slice) -- 4 slices of interleaved 16-byte chunks per
//     pair, 2 pairs per thread -- so a table chunk is ONE broadcast LDS.128 feeding 8 FMAs per
//     lane, pair rows are conflict-free LDS.128 (row stride in 16-byte units is odd), and a
//     dot over d costs two xor-shuffles instead of a tree;
//   * pass F (the [P, d] table gradients, a [P x M] . [M x d] contraction over the tile): a
//     thread owns a (16-byte column chunk, half of the preferences) register tile that stays
//     in registers over all the tiles of the CTA and is flushed once with red.global.add.v4.
// Row gradients are staged in shared memory and leave as whole coalesced rows (with the COO row id
// of every slot).  Rows arrive by cp.async, contractions run on fp32 pairs, and in MODE_STEP a
// warp's 16 rows hold whole (positive, negatives) groups so that one launch does forward, ranking
// loss and backward (kgrec_rank_loss_step).  Design notes: DESIGN.md 4.1.
#include <cstdlib>
#include "train_dev.cuh"

namespace kgrec {
namespace {

constexpr int kMP = 2;                       // pairs per thread
constexpr int kPairsPerWarp = 8 * kMP;       // 8 pair slots x 4 slices per warp
constexpr int kMaxWarps = 8;
constexpr int kSmemCap = 227 * 1024;

struct TileArgs {
  kgrec_tables T;
  int ktup;
  const void *a, *b, *na, *nb;   // pair i < n_pos reads (a, b)[i], else (na, nb)[i - n_pos]
  int is64;
  int64_t n, n_pos;
  const float* gumbel_u;
  SeedRef seed;
  float *scores_a, *scores_b;    // forward: i < n_pos -> scores_a[i], else scores_b[i - n_pos]
  int32_t* status;
  LossCfg L;                     // backward
  BwdArgs B;
  kgrec_grads G;
  int lda;                       // shared row stride in floats, lda / 4 odd
  int n_tiles;
  // single-pass step: a warp's 16 rows hold gw whole groups of gsz = 1 + n_neg pairs (the positive,
  // then its negatives), so the ranking loss and its gradient are formed between two passes
  int gsz, gw;
  float* group_loss;
  int64_t *slot_user, *slot_item, *slot_ent;   // optional: table row of every gradient slot (COO indices)
};

enum { MODE_FWD = 0, MODE_BWD = 1, MODE_STEP = 2 };

__device__ __forceinline__ float qsum(float v) {   // all-reduce over the 4 slices of a pair
  v += __shfl_xor_sync(FULL, v, 8);
  v += __shfl_xor_sync(FULL, v, 16);
  return v;
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const uint32_t sa = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}
// fp32 pairs: two round-to-nearest FFMAs (sm_90 has no packed FFMA2; the results are the same)
__device__ __forceinline__ float2 ffma2(const float2& a, const float2& b, const float2& c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 lo(const float4& v) { return make_float2(v.x, v.y); }
__device__ __forceinline__ float2 hi(const float4& v) { return make_float2(v.z, v.w); }
__device__ __forceinline__ float2 dup(float v) { return make_float2(v, v); }
__device__ __forceinline__ void dot4acc2(float2& acc, const float4& a, const float4& b) {
  acc = ffma2(lo(a), lo(b), acc);
  acc = ffma2(hi(a), hi(b), acc);
}
__device__ __forceinline__ void axpy4p(float2& ylo, float2& yhi, const float2& aa, const float4& x) {
  ylo = ffma2(aa, lo(x), ylo);
  yhi = ffma2(aa, hi(x), yhi);
}
__device__ __forceinline__ float dot4acc(const float4& a, const float4& b, float acc) {
  return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, fmaf(a.w, b.w, acc))));
}

// upstream dLoss/dscore of flat pair i, one thread (train_dev.cuh upstream_grad is its warp form)
__device__ __forceinline__ float upstream_one(const BwdArgs& B, const LossCfg& L, int64_t i) {
  if (B.pos_scores == nullptr) return __ldg(B.grad_scores + i);
  if (i < L.n_pos) {
    const float sp = __ldg(B.pos_scores + i);
    float c = 0.f;
    for (int k = 0; k < L.n_neg; ++k) c += loss_dpos(L, sp, __ldg(B.neg_scores + i * L.n_neg + k));
    const float up = B.grad_loss * (B.grad_loss_dev ? __ldg(B.grad_loss_dev + i / L.batch_pos) : 1.f);
    return c * loss_batch_scale(L, i) * up;
  }
  const int64_t m = i - L.n_pos, j = m / L.n_neg;
  const float up = B.grad_loss * (B.grad_loss_dev ? __ldg(B.grad_loss_dev + j / L.batch_pos) : 1.f);
  return -loss_dpos(L, __ldg(B.pos_scores + j), __ldg(B.neg_scores + m)) * loss_batch_scale(L, j) * up;
}

template <int PT> struct KSplit { static constexpr int KH = (PT == 20) ? 10 : 8; };   // preferences per pass-F thread

template <int PT, bool GUMBEL, int MODE>
__global__ void __launch_bounds__(kMaxWarps * 32, 1) k_rec_tile(const TileArgs A) {
  extern __shared__ __align__(16) float smem[];
  constexpr bool BWD = MODE != MODE_FWD;
  constexpr bool STEP = MODE == MODE_STEP;
  constexpr int KH = KSplit<PT>::KH;
  constexpr int KSPLIT = PT / KH;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
  const int slot = lane & 7, q = lane >> 3;
  const int M = nw * kPairsPerWarp;
  const kgrec_tables& T = A.T;
  const int d = T.dim, P = T.n_pref, NC = d >> 2, lda4 = A.lda >> 2;
  const float hf = A.ktup ? 0.5f : 1.f;
  const uint64_t seed = GUMBEL ? A.seed.get() : 0;
  const int l1 = T.l1;

  float4* sP = reinterpret_cast<float4*>(smem);                       // [NC][PT]   (KTUP: pref + rel)
  float4* sN = sP + PT * NC;                                          // [NC][PT]   (KTUP: pref_norm + norm)
  float4* S = sN + PT * NC;                                           // [M][lda4]  u + i      -> user-row gradient
  float4* X = S + M * lda4;                                           // [M][lda4]  u - i      -> gx
  float4* E = X + M * lda4;                                           // [M][lda4]  x + r, eps -> item-row gradient
  float4* W = E + M * lda4;                                           // [M][lda4]  w          -> gw
  float* coef = reinterpret_cast<float*>(W + M * lda4);               // [M][2][PT] cA = hf p, cB = gz / 2
  float* sg = coef + M * 2 * PT;                                      // [M] upstream
  int* sid = reinterpret_cast<int*>(sg + M);                          // [3][M] user, item, aligned entity

  for (int idx = tid; idx < PT * NC; idx += blockDim.x) {
    const int k = idx / NC, c = idx - k * NC;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (k < P) {
      a = ldg_f4(reinterpret_cast<const float4*>(T.pref + static_cast<int64_t>(k) * T.ld) + c);
      b = ldg_f4(reinterpret_cast<const float4*>(T.pref_norm + static_cast<int64_t>(k) * T.ld) + c);
      if (A.ktup) {   // jTransUP.py:253-256
        const float4 r = ldg_f4(reinterpret_cast<const float4*>(T.rel + static_cast<int64_t>(k) * T.ld) + c);
        const float4 w = ldg_f4(reinterpret_cast<const float4*>(T.norm + static_cast<int64_t>(k) * T.ld) + c);
        a.x += r.x; a.y += r.y; a.z += r.z; a.w += r.w;
        b.x += w.x; b.y += w.y; b.z += w.z; b.w += w.w;
      }
    }
    sP[c * PT + k] = a;     // chunk-major: the k-th row of a chunk is an immediate offset
    sN[c * PT + k] = b;
  }

  // pass-F ownership: (column chunk jc, preference block kh), replicated over row groups
  const int items = NC * KSPLIT;
  const int ngrp = blockDim.x / items;
  const int grp = tid / items, item = tid - grp * items;
  const int jc = item % NC, kh = item / NC;
  float2 accP[BWD ? KH / 2 : 1][4], accN[BWD ? KH / 2 : 1][4];   // .x = preference k, .y = k + 1
  if constexpr (BWD) {
#pragma unroll
    for (int k = 0; k < KH / 2; ++k)
#pragma unroll
      for (int e = 0; e < 4; ++e) { accP[k][e] = make_float2(0.f, 0.f); accN[k][e] = accP[k][e]; }
  }

  const int mloc[kMP] = {wid * kPairsPerWarp + slot, wid * kPairsPerWarp + 8 + slot};

  // ids of a tile's rows, one per lane: lanes 0-15 hold the user id of row wid*16 + lane, lanes
  // 16-31 the item id of row wid*16 + lane - 16; -1 past the end.  Fetched one tile ahead.
  // (group, member) of a local row in step mode: fixed per row, so the divisions happen once per thread
  struct RowPos { int gl, tt; };
  auto row_pos = [&](int rl) {
    RowPos p{0, 0};
    if constexpr (STEP) { p.gl = rl / A.gsz; p.tt = rl - p.gl * A.gsz; }
    return p;
  };
  const RowPos rp_a[kMP] = {row_pos(slot), row_pos(8 + slot)};
  const RowPos rp_l = row_pos(lane & 15);
  // flat pair index (positives first, then negatives) of the warp's local row rl of tile t; -1 = none
  auto pair_at = [&](int t, int rl, const RowPos& rp) -> int64_t {
    if (t >= A.n_tiles) return -1;
    if constexpr (STEP) {
      const int64_t j = (static_cast<int64_t>(t) * nw + wid) * A.gw + rp.gl;
      if (rp.gl >= A.gw || j >= A.n_pos) return -1;
      return rp.tt == 0 ? j : A.n_pos + j * (A.gsz - 1) + (rp.tt - 1);
    } else {
      const int64_t i = static_cast<int64_t>(t) * M + wid * kPairsPerWarp + rl;
      return i < A.n ? i : -1;
    }
  };
  auto fetch_ids = [&](int t) -> int64_t {
    const int64_t i = pair_at(t, lane & 15, rp_l);
    if (i < 0) return -1;
    const bool neg = i >= A.n_pos;
    const int64_t li = neg ? i - A.n_pos : i;
    return load_idx(lane < 16 ? (neg ? A.na : A.a) : (neg ? A.nb : A.b), li, A.is64);
  };
  int64_t idv = fetch_ids(blockIdx.x);
  __syncthreads();   // tables staged

  // Rows wid*16 .. wid*16+15 of the tile belong to this warp from the gather to the flush; only
  // pass F reads other warps' rows (two CTA barriers per tile in the backward, none in the forward).
  for (int tile = blockIdx.x; tile < A.n_tiles; tile += gridDim.x) {
    const int64_t pidx[kMP] = {pair_at(tile, slot, rp_a[0]), pair_at(tile, 8 + slot, rp_a[1])};

    // ---- gather: raw rows by cp.async (u -> E, item -> W, aligned entity -> S), all 16 rows of
    // the warp in flight at once, then S = u + i', X = u - i'  (i' = item + entity for KTUP,
    // jTransUP.py:133)
    {
      int64_t id = idv;
      if constexpr (MODE != MODE_BWD) {
        if (id >= 0) id = checked(id, lane < 16 ? T.n_user : T.n_item, A.status);
      }
      int64_t ia = 0;
      if (A.ktup && lane >= 16 && id >= 0) ia = __ldg(T.item2ent + id);
      const int rl = wid * kPairsPerWarp + (lane & 15);
      if (lane < 16) sid[rl] = static_cast<int>(id);
      else { sid[M + rl] = static_cast<int>(id); sid[2 * M + rl] = static_cast<int>(ia); }
      if constexpr (MODE == MODE_BWD) {
        if (lane < 16) sg[rl] = id >= 0 ? upstream_one(A.B, A.L, pair_at(tile, lane & 15, rp_l)) : 0.f;
      }
#pragma unroll 4
      for (int j = 0; j < kPairsPerWarp; ++j) {
        const int64_t iu = __shfl_sync(FULL, id, j), ii = __shfl_sync(FULL, id, 16 + j);
        const int64_t iaj = __shfl_sync(FULL, ia, 16 + j);
        const int r = wid * kPairsPerWarp + j;
        if (iu >= 0 && lane < NC) {
          cp_async16(E + r * lda4 + lane, reinterpret_cast<const float4*>(T.user + iu * T.ld) + lane);
          cp_async16(W + r * lda4 + lane, reinterpret_cast<const float4*>(T.item + ii * T.ld) + lane);
          if (A.ktup) cp_async16(S + r * lda4 + lane, reinterpret_cast<const float4*>(T.ent + iaj * T.ld) + lane);
        }
      }
      cp_async_wait_all();
      idv = fetch_ids(tile + gridDim.x);   // in flight during the compute passes
#pragma unroll 4
      for (int j = 0; j < kPairsPerWarp; ++j) {
        const bool ok = __shfl_sync(FULL, id, j) >= 0;
        const int o = (wid * kPairsPerWarp + j) * lda4 + lane;
        if (lane < NC) {
          float4 u = make_float4(0.f, 0.f, 0.f, 0.f), it = u;
          if (ok) {
            u = E[o];
            it = W[o];
            if (A.ktup) { const float4 e = S[o]; it.x += e.x; it.y += e.y; it.z += e.z; it.w += e.w; }
          }
          S[o] = make_float4(u.x + it.x, u.y + it.y, u.z + it.z, u.w + it.w);
          X[o] = make_float4(u.x - it.x, u.y - it.y, u.z - it.z, u.w - it.w);
        }
      }
      __syncwarp();
    }

    // ---- pass A: logits z_k = (u + i) . P_k / 2   (transUP.py:108)
    float z[kMP][PT];
    {
      float2 z2[kMP][PT];
#pragma unroll
      for (int a = 0; a < kMP; ++a)
#pragma unroll
        for (int k = 0; k < PT; ++k) z2[a][k] = make_float2(0.f, 0.f);
      for (int c = q; c < NC; c += 4) {
        const float4 s0 = S[mloc[0] * lda4 + c], s1 = S[mloc[1] * lda4 + c];
#pragma unroll
        for (int k = 0; k < PT; ++k) {
          const float4 p = sP[c * PT + k];
          dot4acc2(z2[0][k], s0, p);
          dot4acc2(z2[1][k], s1, p);
        }
      }
#pragma unroll
      for (int a = 0; a < kMP; ++a)
#pragma unroll
        for (int k = 0; k < PT; ++k) z[a][k] = 0.5f * qsum(z2[a][k].x + z2[a][k].y);
    }

    // ---- preference weights: raw logits, or the ST-Gumbel arg-max (transUP.py:143-170)
    int kstar[kMP] = {0, 0};
    if constexpr (GUMBEL) {
#pragma unroll
      for (int a = 0; a < kMP; ++a) {
        const int64_t pid = pidx[a];
        float nz[PT / 4];
#pragma unroll
        for (int j = 0; j < PT / 4; ++j) {
          const int k = 4 * j + q;
          nz[j] = 0.f;
          if (k < P && pid >= 0)
            nz[j] = A.gumbel_u ? gumbel_from_uniform(__ldg(A.gumbel_u + pid * P + k))
                               : gumbel_fast(philox_uniform_bits(seed, static_cast<uint64_t>(pid), static_cast<uint32_t>(k)));
        }
        float best = -INFINITY;
#pragma unroll
        for (int k = 0; k < PT; ++k) {
          const float noise = __shfl_sync(FULL, nz[k >> 2], slot + 8 * (k & 3));
          const float v = (k < P) ? z[a][k] + noise : -INFINITY;
          z[a][k] = v;                                   // v = z + noise is what the backward needs
          if (v > best) { best = v; kstar[a] = k; }
        }
      }
    }

    // ---- pass B: r = hf p P, w = hf p N; xw = (u - i) . w; E = x + r; W = w
    float xw[kMP] = {0.f, 0.f};
    for (int c = q; c < NC; c += 4) {
      float4 r4[kMP], w4[kMP];
      if constexpr (GUMBEL) {
#pragma unroll
        for (int a = 0; a < kMP; ++a) {
          r4[a] = sP[c * PT + kstar[a]];
          w4[a] = sN[c * PT + kstar[a]];
        }
      } else {
        float2 rl[kMP], rh[kMP], wl[kMP], wh[kMP];
#pragma unroll
        for (int a = 0; a < kMP; ++a) { rl[a] = make_float2(0.f, 0.f); rh[a] = rl[a]; wl[a] = rl[a]; wh[a] = rl[a]; }
#pragma unroll
        for (int k = 0; k < PT; ++k) {
          const float4 p = sP[c * PT + k], nn = sN[c * PT + k];
#pragma unroll
          for (int a = 0; a < kMP; ++a) {
            const float2 zz = dup(z[a][k]);
            axpy4p(rl[a], rh[a], zz, p);
            axpy4p(wl[a], wh[a], zz, nn);
          }
        }
#pragma unroll
        for (int a = 0; a < kMP; ++a) {
          r4[a] = make_float4(rl[a].x, rl[a].y, rh[a].x, rh[a].y);
          w4[a] = make_float4(wl[a].x, wl[a].y, wh[a].x, wh[a].y);
        }
      }
#pragma unroll
      for (int a = 0; a < kMP; ++a) {
        const float4 x = X[mloc[a] * lda4 + c];
        w4[a].x *= hf; w4[a].y *= hf; w4[a].z *= hf; w4[a].w *= hf;
        xw[a] = dot4acc(x, w4[a], xw[a]);
        W[mloc[a] * lda4 + c] = w4[a];
        E[mloc[a] * lda4 + c] = make_float4(fmaf(hf, r4[a].x, x.x), fmaf(hf, r4[a].y, x.y), fmaf(hf, r4[a].z, x.z), fmaf(hf, r4[a].w, x.w));
      }
    }
#pragma unroll
    for (int a = 0; a < kMP; ++a) xw[a] = qsum(xw[a]);

    // ---- pass C: e = (x + r) - xw w; score = L(e); eps = g dL/de   (own chunks only: no sync)
    float ew[kMP] = {0.f, 0.f}, g[kMP] = {0.f, 0.f};
    if constexpr (MODE != MODE_BWD) {
      float sc[kMP] = {0.f, 0.f};
      for (int c = q; c < NC; c += 4) {
#pragma unroll
        for (int a = 0; a < kMP; ++a) {
          const float4 xr = E[mloc[a] * lda4 + c], w4 = W[mloc[a] * lda4 + c];
          sc[a] += dist_term(fmaf(-xw[a], w4.x, xr.x), l1) + dist_term(fmaf(-xw[a], w4.y, xr.y), l1) +
                   dist_term(fmaf(-xw[a], w4.z, xr.z), l1) + dist_term(fmaf(-xw[a], w4.w, xr.w), l1);
        }
      }
#pragma unroll
      for (int a = 0; a < kMP; ++a) {
        sc[a] = qsum(sc[a]);
        const int64_t i = pidx[a];
        if (q == 0 && i >= 0) {
          if (i < A.n_pos) A.scores_a[i] = sc[a];
          else A.scores_b[i - A.n_pos] = sc[a];
        }
        if constexpr (STEP) {
          if (q == 0) sg[mloc[a]] = sc[a];
        }
      }
      if constexpr (STEP) {
        // ranking loss of the group and its derivative (utils/loss.py:8-16,29-31), scores in sg
        __syncwarp();
        const int K = A.gsz - 1;
#pragma unroll
        for (int a = 0; a < kMP; ++a) {
          const int gl = rp_a[a].gl, tt = rp_a[a].tt;
          const int64_t i = pidx[a];
          if (i >= 0) {
            const int64_t j = (static_cast<int64_t>(tile) * nw + wid) * A.gw + gl;
            const float* gs = sg + wid * kPairsPerWarp + gl * A.gsz;    // [pos, neg_1 .. neg_K]
            const float up = A.B.grad_loss * loss_batch_scale(A.L, j);
            if (tt == 0) {
              float c = 0.f, lsum = 0.f;
              for (int k = 1; k <= K; ++k) { c += loss_dpos(A.L, gs[0], gs[k]); lsum += loss_term(A.L, gs[0], gs[k]); }
              g[a] = c * up;
              if (q == 0) A.group_loss[j] = lsum;
            } else {
              g[a] = -loss_dpos(A.L, gs[0], gs[tt]) * up;
            }
          }
        }
        __syncwarp();
      }
    }
    if constexpr (MODE == MODE_BWD) {
#pragma unroll
      for (int a = 0; a < kMP; ++a) g[a] = sg[mloc[a]];
    }
    if constexpr (BWD) {
      for (int c = q; c < NC; c += 4) {
#pragma unroll
        for (int a = 0; a < kMP; ++a) {
          const float4 xr = E[mloc[a] * lda4 + c], w4 = W[mloc[a] * lda4 + c];
          const float4 e = make_float4(fmaf(-xw[a], w4.x, xr.x), fmaf(-xw[a], w4.y, xr.y), fmaf(-xw[a], w4.z, xr.z), fmaf(-xw[a], w4.w, xr.w));
          const float4 eps = make_float4(g[a] * ddist_term(e.x, l1), g[a] * ddist_term(e.y, l1), g[a] * ddist_term(e.z, l1), g[a] * ddist_term(e.w, l1));
          ew[a] = dot4acc(eps, w4, ew[a]);
          E[mloc[a] * lda4 + c] = eps;
        }
      }
#pragma unroll
      for (int a = 0; a < kMP; ++a) ew[a] = qsum(ew[a]);

      // ---- pass D: gx = eps - ew w, gw = -(ew x + xw eps); gp_k = hf (eps . P_k + gw . N_k)
      float gp[kMP][PT];
      float2 gp2[kMP][PT];
#pragma unroll
      for (int a = 0; a < kMP; ++a)
#pragma unroll
        for (int k = 0; k < PT; ++k) gp2[a][k] = make_float2(0.f, 0.f);
      for (int c = q; c < NC; c += 4) {
        float4 eps[kMP], gw[kMP];
#pragma unroll
        for (int a = 0; a < kMP; ++a) {
          eps[a] = E[mloc[a] * lda4 + c];
          const float4 w4 = W[mloc[a] * lda4 + c], x = X[mloc[a] * lda4 + c];
          gw[a] = make_float4(-fmaf(ew[a], x.x, xw[a] * eps[a].x), -fmaf(ew[a], x.y, xw[a] * eps[a].y),
                              -fmaf(ew[a], x.z, xw[a] * eps[a].z), -fmaf(ew[a], x.w, xw[a] * eps[a].w));
          X[mloc[a] * lda4 + c] = make_float4(fmaf(-ew[a], w4.x, eps[a].x), fmaf(-ew[a], w4.y, eps[a].y),
                                              fmaf(-ew[a], w4.z, eps[a].z), fmaf(-ew[a], w4.w, eps[a].w));
          W[mloc[a] * lda4 + c] = gw[a];
        }
#pragma unroll
        for (int k = 0; k < PT; ++k) {
          const float4 p = sP[c * PT + k], nn = sN[c * PT + k];
#pragma unroll
          for (int a = 0; a < kMP; ++a) { dot4acc2(gp2[a][k], eps[a], p); dot4acc2(gp2[a][k], gw[a], nn); }
        }
      }
#pragma unroll
      for (int a = 0; a < kMP; ++a)
#pragma unroll
        for (int k = 0; k < PT; ++k) gp[a][k] = gp2[a][k].x + gp2[a][k].y;
      // coefficients of the table-gradient contraction and of gs:  cA = hf p, cB = gz / 2
#pragma unroll
      for (int a = 0; a < kMP; ++a) {
        float* ca = coef + mloc[a] * 2 * PT;
        if constexpr (GUMBEL) {
          // y = softmax(z + noise); gz = y (gp - <y, gp>)   (backward of transUP.py:162-168)
          float mx = -INFINITY;
#pragma unroll
          for (int k = 0; k < PT; ++k) mx = fmaxf(mx, z[a][k]);
          float sum = 0.f, yg = 0.f;
#pragma unroll
          for (int k = 0; k < PT; ++k) {
            gp[a][k] = hf * qsum(gp[a][k]);
            const float ex = (k < P) ? __expf(z[a][k] - mx) : 0.f;
            z[a][k] = ex;
            sum += ex;
            yg = fmaf(ex, gp[a][k], yg);
          }
          const float inv = 1.f / sum;
          yg *= inv;
#pragma unroll
          for (int k = 0; k < PT; ++k) {
            gp[a][k] = 0.5f * z[a][k] * inv * (gp[a][k] - yg);
            if ((k & 3) == q) { ca[k] = (k == kstar[a]) ? hf : 0.f; ca[PT + k] = gp[a][k]; }
          }
        } else {
#pragma unroll
          for (int k = 0; k < PT; ++k) {
            gp[a][k] = 0.5f * hf * qsum(gp[a][k]);
            if ((k & 3) == q) { ca[k] = hf * z[a][k]; ca[PT + k] = gp[a][k]; }
          }
        }
      }
      __syncthreads();

      // ---- pass F: g_pref[k] += cA[k] eps + cB[k] s ; g_pref_norm[k] += cA[k] gw  over the tile's pairs
      if (grp < ngrp) {
#pragma unroll 2
        for (int m = grp; m < M; m += ngrp) {   // rows without a pair hold zeros
          const float4 e4 = E[m * lda4 + jc], s4 = S[m * lda4 + jc], g4 = W[m * lda4 + jc];
          const float2* ca = reinterpret_cast<const float2*>(coef + m * 2 * PT + kh * KH);
          const float2* cb = reinterpret_cast<const float2*>(coef + m * 2 * PT + PT + kh * KH);
          const float2 ex = dup(e4.x), ey = dup(e4.y), ez = dup(e4.z), ew2 = dup(e4.w);
          const float2 sx = dup(s4.x), sy = dup(s4.y), sz = dup(s4.z), sw = dup(s4.w);
          const float2 gx2 = dup(g4.x), gy = dup(g4.y), gz = dup(g4.z), gw2 = dup(g4.w);
#pragma unroll
          for (int h = 0; h < KH / 2; ++h) {
            const float2 a2 = ca[h], b2 = cb[h];
            accP[h][0] = ffma2(a2, ex, ffma2(b2, sx, accP[h][0]));
            accP[h][1] = ffma2(a2, ey, ffma2(b2, sy, accP[h][1]));
            accP[h][2] = ffma2(a2, ez, ffma2(b2, sz, accP[h][2]));
            accP[h][3] = ffma2(a2, ew2, ffma2(b2, sw, accP[h][3]));
            accN[h][0] = ffma2(a2, gx2, accN[h][0]);
            accN[h][1] = ffma2(a2, gy, accN[h][1]);
            accN[h][2] = ffma2(a2, gz, accN[h][2]);
            accN[h][3] = ffma2(a2, gw2, accN[h][3]);
          }
        }
      }
      __syncthreads();

      // ---- pass E: gs = sum_k cB_k P_k; user row gradient gx + gs -> S, item row gradient gs - gx -> E
      for (int c = q; c < NC; c += 4) {
        float4 gs[kMP];
        float2 gl[kMP], gh[kMP];
#pragma unroll
        for (int a = 0; a < kMP; ++a) { gl[a] = make_float2(0.f, 0.f); gh[a] = gl[a]; }
#pragma unroll
        for (int k = 0; k < PT; ++k) {
          const float4 p = sP[c * PT + k];
#pragma unroll
          for (int a = 0; a < kMP; ++a) axpy4p(gl[a], gh[a], dup(gp[a][k]), p);
        }
#pragma unroll
        for (int a = 0; a < kMP; ++a) gs[a] = make_float4(gl[a].x, gl[a].y, gh[a].x, gh[a].y);
#pragma unroll
        for (int a = 0; a < kMP; ++a) {
          const float4 gx = X[mloc[a] * lda4 + c];
          S[mloc[a] * lda4 + c] = make_float4(gs[a].x + gx.x, gs[a].y + gx.y, gs[a].z + gx.z, gs[a].w + gx.w);
          E[mloc[a] * lda4 + c] = make_float4(gs[a].x - gx.x, gs[a].y - gx.y, gs[a].z - gx.z, gs[a].w - gx.w);
        }
      }
      __syncwarp();

      // ---- flush the row gradients: whole rows, the warp's own 16
      RowPos fp{0, 0};
      for (int j = 0; j < kPairsPerWarp; ++j) {
        const int r = wid * kPairsPerWarp + j;
        const int64_t i = pair_at(tile, j, fp);
        if constexpr (STEP) { if (++fp.tt == A.gsz) { fp.tt = 0; ++fp.gl; } }
        if (i < 0 || lane >= NC) continue;
        const float4 gu = S[r * lda4 + lane];
        float4 gi = E[r * lda4 + lane];
        const int ia = sid[2 * M + r];
        const bool pad = A.ktup && ia == T.n_ent - 1;     // padding row: no gradient (jTransUP.py:96)
        if (A.slot_user && lane == 0) {
          A.slot_user[i] = sid[r];
          A.slot_item[i] = sid[M + r];
          if (A.ktup) A.slot_ent[i] = ia;
        }
        if (A.G.mode == 0) {
          __stcs(reinterpret_cast<float4*>(A.G.user + i * d) + lane, gu);
          __stcs(reinterpret_cast<float4*>(A.G.item + i * d) + lane, gi);
          if (A.ktup) {
            if (pad) gi = make_float4(0.f, 0.f, 0.f, 0.f);
            __stcs(reinterpret_cast<float4*>(A.G.ent + i * d) + lane, gi);
          }
        } else {
          red_add_f4(A.G.user + static_cast<int64_t>(sid[r]) * d + 4 * lane, gu.x, gu.y, gu.z, gu.w);
          red_add_f4(A.G.item + static_cast<int64_t>(sid[M + r]) * d + 4 * lane, gi.x, gi.y, gi.z, gi.w);
          if (A.ktup && !pad) red_add_f4(A.G.ent + static_cast<int64_t>(ia) * d + 4 * lane, gi.x, gi.y, gi.z, gi.w);
        }
      }
      __syncwarp();
    }
  }

  if constexpr (BWD) {
    if (grp < ngrp) {
#pragma unroll
      for (int kk = 0; kk < KH; ++kk) {
        const int k = kh * KH + kk;
        if (k < P) {
          const int h = kk >> 1;
          if (kk & 1) {
            red_add_f4(A.G.pref + static_cast<int64_t>(k) * d + 4 * jc, accP[h][0].y, accP[h][1].y, accP[h][2].y, accP[h][3].y);
            red_add_f4(A.G.pref_norm + static_cast<int64_t>(k) * d + 4 * jc, accN[h][0].y, accN[h][1].y, accN[h][2].y, accN[h][3].y);
          } else {
            red_add_f4(A.G.pref + static_cast<int64_t>(k) * d + 4 * jc, accP[h][0].x, accP[h][1].x, accP[h][2].x, accP[h][3].x);
            red_add_f4(A.G.pref_norm + static_cast<int64_t>(k) * d + 4 * jc, accN[h][0].x, accN[h][1].x, accN[h][2].x, accN[h][3].x);
          }
        }
      }
    }
  }
}

// group terms of the ranking loss from the flat scores (the tile forward scores positives and
// negatives in different tiles)
__global__ void __launch_bounds__(256)
k_group_loss(const float* __restrict__ pos, const float* __restrict__ neg, const LossCfg L, float* __restrict__ group_loss) {
  const int64_t j = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j >= L.n_pos) return;
  const float sp = pos[j];
  float s = 0.f;
  for (int k = 0; k < L.n_neg; ++k) s += loss_term(L, sp, neg[j * L.n_neg + k]);
  group_loss[j] = s;
}

// slot row ids when the step runs as two kernels (shapes outside the tile engine)
__global__ void __launch_bounds__(256)
k_rec_slot_ids(const void* a, const void* b, const void* na, const void* nb, const int is64, const int64_t n_pos, const int64_t n,
               const int32_t* __restrict__ item2ent, int64_t* __restrict__ su, int64_t* __restrict__ si, int64_t* __restrict__ se) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const bool neg = i >= n_pos;
    const int64_t li = neg ? i - n_pos : i;
    const int64_t iu = load_idx(neg ? na : a, li, is64), ii = load_idx(neg ? nb : b, li, is64);
    su[i] = iu;
    si[i] = ii;
    if (se) se[i] = __ldg(item2ent + ii);
  }
}

struct TilePlan {
  int pt, nw, lda, n_tiles, grid;
  size_t smem;
};

// KGREC_REC_TILE=0 keeps every call on the one-warp-per-pair kernels, =force sends every
// supported shape through the tiles whatever n is (the parity tests run both engines on the
// reference's golden vectors); default: by size.
// n work units (pairs, or whole groups in step mode), upw of them per warp
bool plan_tiles(const kgrec_tables& T, const Plan& pl, int64_t n, int upw, TilePlan* tp) {
  const int d = T.dim, P = T.n_pref;
  if (!pl.vec || d > 128 || P > 32 || n < 1) return false;
  const char* env = getenv("KGREC_REC_TILE");
  const bool force = env && env[0] == 'f';
  if (env && env[0] == '0') return false;
  tp->pt = P <= 8 ? 8 : (P <= 20 ? 20 : 32);
  const int nc = d / 4;
  tp->lda = (nc & 1) ? d : d + 4;
  const size_t fixed = static_cast<size_t>(2) * tp->pt * d * 4;
  const size_t per_warp = static_cast<size_t>(kPairsPerWarp) * (4 * tp->lda + 2 * tp->pt + 4) * 4;
  int nw = static_cast<int>((kSmemCap - fixed) / per_warp);
  if (nw > kMaxWarps) nw = kMaxWarps;
  const int ksplit = tp->pt / (tp->pt == 20 ? 10 : 8);
  const int nw_min = (nc * ksplit + 31) / 32 > 2 ? (nc * ksplit + 31) / 32 : 2;
  const int sms = sm_count();
  // smaller tiles while they still give every SM one; below that the one-warp-per-pair kernels win
  while (nw > nw_min && (n + nw * upw - 1) / (nw * upw) < sms) --nw;
  if (nw < nw_min) return false;
  const int64_t tiles = (n + nw * upw - 1) / (nw * upw);
  if ((tiles < sms && !force) || tiles > 0x7fffffff) return false;
  tp->nw = nw;
  tp->n_tiles = static_cast<int>(tiles);
  tp->grid = static_cast<int>(tiles < sms ? tiles : sms);
  tp->smem = fixed + per_warp * nw;
  return true;
}

template <int MODE>
int launch_tiles(const TileArgs& A, const TilePlan& tp, cudaStream_t st) {
  int rc = KGREC_OK;
#define KGREC_TILE(PTV, GUM)                                                             \
  {                                                                                      \
    auto kern = k_rec_tile<PTV, GUM, MODE>;                                              \
    if ((rc = set_smem(kern, tp.smem))) return rc;                                       \
    kern<<<tp.grid, tp.nw * 32, tp.smem, st>>>(A);                                       \
  }
  const bool gum = A.T.use_gumbel != 0;
  if (tp.pt == 8) { if (gum) KGREC_TILE(8, true) else KGREC_TILE(8, false) }
  else if (tp.pt == 20) { if (gum) KGREC_TILE(20, true) else KGREC_TILE(20, false) }
  else { if (gum) KGREC_TILE(32, true) else KGREC_TILE(32, false) }
#undef KGREC_TILE
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

}  // namespace

// ---- entry points used by the FAM_REC launchers (train_dev.cuh); return -1 = not taken ----
int rec_tile_score_fwd(const kgrec_tables& T, const Plan& pl, const IdxArgs& I, int64_t n, const float* gumbel_u,
                       SeedRef seed, float* scores, int32_t* status, cudaStream_t st) {
  TilePlan tp;
  if (!plan_tiles(T, pl, n, kPairsPerWarp, &tp)) return -1;
  TileArgs A{};
  A.T = T; A.ktup = pl.ktup; A.a = I.a; A.b = I.b; A.na = nullptr; A.nb = nullptr; A.is64 = I.is64;
  A.n = n; A.n_pos = n; A.gumbel_u = gumbel_u; A.seed = seed; A.scores_a = scores; A.scores_b = nullptr;
  A.status = status; A.lda = tp.lda; A.n_tiles = tp.n_tiles;
  return launch_tiles<MODE_FWD>(A, tp, st);
}

int rec_tile_rank_loss_fwd(const kgrec_tables& T, const Plan& pl, const IdxArgs& I, const LossCfg& L,
                           const float* gumbel_u, SeedRef seed, float* pos_scores, float* neg_scores,
                           float* group_loss, int32_t* status, cudaStream_t st) {
  TilePlan tp;
  const int64_t n = L.n_pos * (1 + static_cast<int64_t>(L.n_neg));
  if (!plan_tiles(T, pl, n, kPairsPerWarp, &tp)) return -1;
  TileArgs A{};
  A.T = T; A.ktup = pl.ktup; A.a = I.a; A.b = I.b; A.na = I.na; A.nb = I.nb; A.is64 = I.is64;
  A.n = n; A.n_pos = L.n_pos; A.gumbel_u = gumbel_u; A.seed = seed; A.scores_a = pos_scores; A.scores_b = neg_scores;
  A.status = status; A.lda = tp.lda; A.n_tiles = tp.n_tiles;
  const int rc = launch_tiles<MODE_FWD>(A, tp, st);
  if (rc) return rc;
  k_group_loss<<<static_cast<unsigned>((L.n_pos + 255) / 256), 256, 0, st>>>(pos_scores, neg_scores, L, group_loss);
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

int rec_tile_score_bwd(const kgrec_tables& T, const Plan& pl, const IdxArgs& I, int64_t n, const LossCfg& L,
                       const float* gumbel_u, SeedRef seed, const BwdArgs& B, const kgrec_grads& G, cudaStream_t st) {
  TilePlan tp;
  if (!plan_tiles(T, pl, n, kPairsPerWarp, &tp)) return -1;
  const bool fused = B.pos_scores != nullptr;
  TileArgs A{};
  A.T = T; A.ktup = pl.ktup; A.a = I.a; A.b = I.b; A.na = I.na; A.nb = I.nb; A.is64 = I.is64;
  A.n = n; A.n_pos = fused ? L.n_pos : n; A.gumbel_u = gumbel_u; A.seed = seed;
  A.L = L; A.B = B; A.G = G; A.lda = tp.lda; A.n_tiles = tp.n_tiles;
  return launch_tiles<MODE_BWD>(A, tp, st);
}

// forward + ranking loss + backward in one pass over groups of (positive, its negatives)
int rec_tile_loss_step(const kgrec_tables& T, const Plan& pl, const IdxArgs& I, const LossCfg& L, float grad_loss,
                       const float* gumbel_u, SeedRef seed, float* pos_scores, float* neg_scores, float* group_loss,
                       const kgrec_grads& G, int64_t* slot_user, int64_t* slot_item, int64_t* slot_ent, int32_t* status,
                       cudaStream_t st) {
  if (L.n_neg > kPairsPerWarp - 1) return -1;
  const int gsz = 1 + L.n_neg, gw = kPairsPerWarp / gsz;
  TilePlan tp;
  if (!plan_tiles(T, pl, L.n_pos, gw, &tp)) return -1;
  TileArgs A{};
  A.T = T; A.ktup = pl.ktup; A.a = I.a; A.b = I.b; A.na = I.na; A.nb = I.nb; A.is64 = I.is64;
  A.n = L.n_pos * static_cast<int64_t>(gsz); A.n_pos = L.n_pos; A.gumbel_u = gumbel_u; A.seed = seed;
  A.scores_a = pos_scores; A.scores_b = neg_scores; A.status = status;
  A.L = L; A.B = BwdArgs{nullptr, nullptr, nullptr, grad_loss, nullptr}; A.G = G;
  A.lda = tp.lda; A.n_tiles = tp.n_tiles; A.gsz = gsz; A.gw = gw; A.group_loss = group_loss;
  A.slot_user = slot_user; A.slot_item = slot_item; A.slot_ent = slot_ent;
  return launch_tiles<MODE_STEP>(A, tp, st);
}

int rec_slot_ids(const kgrec_tables& T, const Plan& pl, const IdxArgs& I, int64_t n_pos, int64_t n, int64_t* su, int64_t* si,
                 int64_t* se, cudaStream_t st) {
  const int64_t ctas = (n + 255) / 256, cap = static_cast<int64_t>(sm_count()) * 16;
  k_rec_slot_ids<<<static_cast<unsigned>(ctas < cap ? ctas : cap), 256, 0, st>>>(I.a, I.b, I.na, I.nb, I.is64, n_pos, n,
                                                                                   T.item2ent, su, si, pl.ktup ? se : nullptr);
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

}  // namespace kgrec
