// TransR full-catalog evaluation (SURVEY 8a row a6): TransRModel.evaluateHead / evaluateTail, transR.py:80-128
// with projection_transR_pytorch_batch, utils/misc.py:29-33.
//
// The reference projects the WHOLE entity table with every query's own matrix ([B, d, d] x [d, E], 2 B E d^2
// flop).  Queries that share a relation share the matrix, so the work is done per DISTINCT relation of the
// call: the caller passes the queries sorted by relation with the run boundaries (host array), and for each
// run this file
//   1. projects the catalog shard once with the run's matrix      k_transr_project   [n_cat, d] x M_r^T, FP32
//   2. builds the run's query vectors c = M_r E[q] -/+ R[r]        k_transr_qvec
//   3. runs the distance kernels of eval.cu on (c, projected rows)  kgrec_eval_scores / _topk / _rank_count
// so the filtered top-K and rank-count modes come for free and no library GEMM is involved.  The path's one
// dense contraction is a hand-written register-tiled FP32 kernel on the CUDA cores (north_star: no tensor
// cores -- TF32 would not hold the 1e-4 score tolerance): a persistent CTA keeps M_r^T in shared memory and
// walks 128-row catalog tiles (cp.async, row-major), 8 x 8 accumulators per thread, two CTAs per SM at d <= 100.
#include "common.cuh"

namespace kgrec {

constexpr int kPT = 128;              // catalog rows per tile, and the padded matrix width
constexpr int kPLD = kPT + 4;         // shared-memory row pitch (floats): keeps the transposing stores spread over banks
constexpr int kProjThreads = 256;

// out[n, a] = sum_b cat[n, b] * M[a, b]      (M = Proj[r].view(d, d), row-major: misc.py:25, 32-33)
// Shared memory: Mt[b][a] = M[a][b] (a padded to 128 with zeros, pitch 132) and the catalog tile ROW-MAJOR, Es[n][b] with
// pitch d + 4 floats (an odd number of 16-byte units for d = 100; for other d the few distinct rows a warp reads are
// multicast), copied in with cp.async -- no transposing stores.  A thread owns rows {4 ty.., 64 + 4 ty..} and columns
// {4 tx.., 64 + 4 tx..}: per 4 steps of b it issues 8 + 8 LDS.128 for 256 FMAs.  Sized by d, two CTAs fit an SM at
// d <= 100, so one CTA's tile load overlaps the other's FMA loop.
__global__ void __launch_bounds__(kProjThreads, 2)
k_transr_project(const float* __restrict__ M, const float* __restrict__ cat, int64_t cat_ld, int64_t n_cat, int d,
                 float* __restrict__ out, int64_t out_ld) {
  extern __shared__ __align__(16) float smem[];
  const int epitch = d + 4;
  float* Mt = smem;                   // [d][kPLD]
  float* Es = smem + d * kPLD;        // [kPT][epitch]
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int dq = d >> 2;              // 16-byte chunks per row
  for (int i = tid; i < d * kPLD; i += kProjThreads) Mt[i] = 0.f;
  __syncthreads();
  for (int i = tid; i < d * dq; i += kProjThreads) {
    const int a = i / dq, c = i - a * dq;
    const float4 v = __ldg(reinterpret_cast<const float4*>(M + static_cast<int64_t>(a) * d) + c);
    Mt[(4 * c + 0) * kPLD + a] = v.x; Mt[(4 * c + 1) * kPLD + a] = v.y;
    Mt[(4 * c + 2) * kPLD + a] = v.z; Mt[(4 * c + 3) * kPLD + a] = v.w;
  }
  const int64_t n_tiles = (n_cat + kPT - 1) / kPT;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t n0 = tile * kPT;
    __syncthreads();                  // previous tile's Es is no longer read; Mt is complete
    for (int i = tid; i < kPT * dq; i += kProjThreads) {
      const int n = i / dq, c = i - n * dq;
      float* dst = Es + n * epitch + 4 * c;
      if (n0 + n < n_cat) {
        const uint32_t sa = static_cast<uint32_t>(__cvta_generic_to_shared(dst));
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(cat + (n0 + n) * cat_ld + 4 * c) : "memory");
      } else {
        *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    const bool hi_cols = 64 + 4 * tx < d;
    const float* e_lo = Es + (4 * ty) * epitch;
    const float* e_hi = Es + (64 + 4 * ty) * epitch;
#pragma unroll 1
    for (int k = 0; k < d; k += 4) {
      float4 e[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        e[i] = *reinterpret_cast<const float4*>(e_lo + i * epitch + k);
        e[4 + i] = *reinterpret_cast<const float4*>(e_hi + i * epitch + k);
      }
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const float4 m0 = *reinterpret_cast<const float4*>(Mt + (k + kk) * kPLD + 4 * tx);
        const float4 m1 = *reinterpret_cast<const float4*>(Mt + (k + kk) * kPLD + 64 + 4 * tx);
        const float m[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float ev = kk == 0 ? e[i].x : (kk == 1 ? e[i].y : (kk == 2 ? e[i].z : e[i].w));
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(ev, m[j], acc[i][j]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int64_t n = n0 + (i < 4 ? 4 * ty + i : 64 + 4 * ty + (i - 4));
      if (n >= n_cat) continue;
      float* o = out + n * out_ld;
      if (4 * tx < d) *reinterpret_cast<float4*>(o + 4 * tx) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      if (hi_cols) *reinterpret_cast<float4*>(o + 64 + 4 * tx) = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
    }
  }
}

// qvec[i] = (c | 0) with c = M_r E[q_i] - R[r] (head side: q holds tails, transR.py:84-90) or + R[r] (tail side,
// transR.py:109-115); one warp per query of the run, lanes over the columns of M's rows.
__global__ void __launch_bounds__(kThreads)
k_transr_qvec(const kgrec_tables T, int side, const void* q, int is64, int64_t i0, int64_t n, int64_t rel,
              float* __restrict__ qvec, int32_t* status) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, d = T.dim;
  const float* M = T.proj + rel * static_cast<int64_t>(d) * d;
  const float* rr = T.rel + rel * T.ld;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kWarpsPerCta + wid; i < n; i += static_cast<int64_t>(gridDim.x) * kWarpsPerCta) {
    int64_t e = load_idx(q, i0 + i, is64);
    if (static_cast<uint64_t>(e) >= static_cast<uint64_t>(T.n_ent)) { if (status) *status = 1; e = 0; }
    const float* x = T.ent + e * T.ld;
    float* o = qvec + (i0 + i) * 2 * d;
    for (int a = 0; a < d; ++a) {
      float s = 0.f;
      for (int b = lane; b < d; b += 32) s = fmaf(__ldg(M + static_cast<int64_t>(a) * d + b), __ldg(x + b), s);
      s = warp_sum(s);
      if (lane == 0) o[a] = side == KGREC_SIDE_HEAD ? s - __ldg(rr + a) : s + __ldg(rr + a);
    }
    for (int b = lane; b < d; b += 32) o[d + b] = 0.f;
  }
}

}  // namespace kgrec

using namespace kgrec;

namespace {

struct TransRCall {
  const kgrec_tables* T;
  int side;
  const void *q, *r;
  int idx_bytes;
  int64_t nq;
  const int64_t* run_begin;      // host: run g covers sorted queries [run_begin[g], run_begin[g + 1])
  const int64_t* run_rel;        // host: its relation id
  int32_t n_runs;
  const float* cat;
  int64_t cat_ld, n_cat, id_base;
  float *proj_ws, *qvec_ws;
  int32_t* status;
  cudaStream_t st;
};

int transr_check(const TransRCall& C) {
  const kgrec_tables* T = C.T;
  if (!T || !T->ent || !T->rel || !T->proj) { set_error("TransR eval: ent / rel / proj table missing"); return KGREC_ERR_INVALID; }
  const int d = T->dim;
  if (d <= 0 || d > kPT || d % 4) { set_error("TransR eval: embedding_size %d must be a multiple of 4, <= %d", d, kPT); return KGREC_ERR_UNSUPPORTED; }
  if (!C.q || C.nq <= 0 || !C.run_begin || !C.run_rel || C.n_runs <= 0 || !C.cat || C.n_cat <= 0 || !C.proj_ws || !C.qvec_ws) {
    set_error("TransR eval: NULL / empty argument");
    return KGREC_ERR_INVALID;
  }
  if (C.cat_ld % 4 || C.cat_ld < d || (reinterpret_cast<uintptr_t>(C.cat) & 15u) || (reinterpret_cast<uintptr_t>(C.proj_ws) & 15u) ||
      (reinterpret_cast<uintptr_t>(T->proj) & 15u)) {
    set_error("TransR eval: catalog / workspace / proj table must be 16-byte aligned with leading dimensions multiples of 4");
    return KGREC_ERR_UNSUPPORTED;
  }
  if (C.run_begin[0] != 0 || C.run_begin[C.n_runs] != C.nq) { set_error("TransR eval: run boundaries do not cover the queries"); return KGREC_ERR_INVALID; }
  for (int g = 0; g < C.n_runs; ++g)
    if (C.run_begin[g + 1] <= C.run_begin[g] || C.run_rel[g] < 0 || C.run_rel[g] >= T->n_rel) {
      set_error("TransR eval: bad run %d", g);
      return KGREC_ERR_INVALID;
    }
  return KGREC_OK;
}

// Project the shard and build the query vectors of run g.
int transr_prepare(const TransRCall& C, int g) {
  static bool attr_done = false;
  const int d = C.T->dim;
  const size_t smem = (static_cast<size_t>(d) * kPLD + static_cast<size_t>(kPT) * (d + 4)) * sizeof(float);
  if (!attr_done) {
    KGREC_CUDA_OK(cudaFuncSetAttribute(k_transr_project, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>((2u * kPT * kPLD) * sizeof(float))));
    attr_done = true;
  }
  const int64_t rel = C.run_rel[g], i0 = C.run_begin[g], n = C.run_begin[g + 1] - i0;
  const int64_t tiles = (C.n_cat + kPT - 1) / kPT;
  const int64_t slots = static_cast<int64_t>(sm_count()) * (smem <= 110 * 1024 ? 2 : 1);     // resident CTAs
  const int grid = static_cast<int>(tiles < slots ? tiles : slots);
  k_transr_project<<<grid, kProjThreads, smem, C.st>>>(C.T->proj + rel * static_cast<int64_t>(d) * d, C.cat, C.cat_ld, C.n_cat, d,
                                                      C.proj_ws, d);
  KGREC_CUDA_OK(cudaGetLastError());
  const int64_t ctas = (n + kWarpsPerCta - 1) / kWarpsPerCta;
  k_transr_qvec<<<static_cast<int>(ctas < 4096 ? ctas : 4096), kThreads, 0, C.st>>>(*C.T, C.side, C.q, C.idx_bytes == 8, i0, n, rel,
                                                                                   C.qvec_ws, C.status);
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

}  // namespace

extern "C" int64_t kgrec_transr_workspace_floats(int64_t nq, int64_t n_cat, int32_t dim) {
  return n_cat * dim + nq * 2 * dim;     // projected shard + query vectors
}

#define TRANSR_CALL()                                                                                                   \
  TransRCall C{tables, side, q, r, idx_bytes, nq, run_begin_host, run_rel_host, n_runs, cat, cat_ld, n_cat, id_base,     \
               workspace, workspace ? workspace + n_cat * (tables ? tables->dim : 0) : nullptr, status,                 \
               static_cast<cudaStream_t>(stream)};                                                                      \
  int rc = transr_check(C);                                                                                              \
  if (rc) return rc;

extern "C" int kgrec_transr_eval_scores(const kgrec_tables* tables, int side, const void* q, const void* r, int idx_bytes,
                                        int64_t nq, const int64_t* run_begin_host, const int64_t* run_rel_host, int32_t n_runs,
                                        const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base, const int32_t* cat_ids,
                                        float* workspace, float* out, int64_t ld_out, int32_t* status, kgrec_stream_t stream) {
  TRANSR_CALL();
  if (!out || ld_out < n_cat) { set_error("bad out / ld_out"); return KGREC_ERR_INVALID; }
  const int d = tables->dim;
  for (int g = 0; g < n_runs; ++g) {
    if ((rc = transr_prepare(C, g))) return rc;
    const int64_t i0 = run_begin_host[g], n = run_begin_host[g + 1] - i0;
    rc = kgrec_eval_scores(tables, KGREC_TRANSR, side, nullptr, nullptr, 8, C.qvec_ws + i0 * 2 * d, n, C.proj_ws, d, n_cat, id_base,
                           cat_ids, nullptr, 0, out + i0 * ld_out, ld_out, stream);
    if (rc) return rc;
  }
  return KGREC_OK;
}

extern "C" int kgrec_transr_eval_topk(const kgrec_tables* tables, int side, const void* q, const void* r, int idx_bytes,
                                      int64_t nq, const int64_t* run_begin_host, const int64_t* run_rel_host, int32_t n_runs,
                                      const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base, float* workspace,
                                      int32_t k, const int64_t* filter_ptr, const int32_t* filter_ids, uint64_t* out_keys,
                                      void* topk_workspace, int64_t topk_workspace_bytes, int32_t* status, kgrec_stream_t stream) {
  TRANSR_CALL();
  if (!out_keys) { set_error("out_keys is NULL"); return KGREC_ERR_INVALID; }
  const int d = tables->dim;
  for (int g = 0; g < n_runs; ++g) {
    if ((rc = transr_prepare(C, g))) return rc;
    const int64_t i0 = run_begin_host[g], n = run_begin_host[g + 1] - i0;
    // the CSR's row pointers are absolute offsets into filter_ids, so a run's slice of them is a valid CSR
    rc = kgrec_eval_topk(tables, KGREC_TRANSR, side, nullptr, nullptr, 8, C.qvec_ws + i0 * 2 * d, n, C.proj_ws, d, n_cat, id_base, k,
                         filter_ptr ? filter_ptr + i0 : nullptr, filter_ids, nullptr, 0, out_keys + i0 * k, topk_workspace,
                         topk_workspace_bytes, stream);
    if (rc) return rc;
  }
  return KGREC_OK;
}

extern "C" int kgrec_transr_eval_rank_count(const kgrec_tables* tables, int side, const void* q, const void* r, int idx_bytes,
                                            int64_t nq, const int64_t* run_begin_host, const int64_t* run_rel_host, int32_t n_runs,
                                            const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base, float* workspace,
                                            const float* gold_scores, const int32_t* gold_ids, int32_t* counts, int32_t* status,
                                            kgrec_stream_t stream) {
  TRANSR_CALL();
  if (!gold_scores || !gold_ids || !counts) { set_error("rank_count: NULL argument"); return KGREC_ERR_INVALID; }
  const int d = tables->dim;
  for (int g = 0; g < n_runs; ++g) {
    if ((rc = transr_prepare(C, g))) return rc;
    const int64_t i0 = run_begin_host[g], n = run_begin_host[g + 1] - i0;
    rc = kgrec_eval_rank_count(tables, KGREC_TRANSR, side, nullptr, nullptr, 8, C.qvec_ws + i0 * 2 * d, n, C.proj_ws, d, n_cat, id_base,
                               gold_scores + i0, gold_ids + i0, counts + i0, stream);
    if (rc) return rc;
  }
  return KGREC_OK;
}

extern "C" int kgrec_transr_eval_rank_count_ex(const kgrec_tables* tables, int side, const void* q, const void* r, int idx_bytes,
                                               int64_t nq, const int64_t* run_begin_host, const int64_t* run_rel_host, int32_t n_runs,
                                               const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base, float* workspace,
                                               const float* gold_scores, const int32_t* gold_ids, int32_t* counts,
                                               const int32_t* excl_row, const int64_t* excl_ptr, const int32_t* excl_ids,
                                               int32_t* status, kgrec_stream_t stream) {
  TRANSR_CALL();
  if (!gold_scores || !gold_ids || !counts) { set_error("rank_count: NULL argument"); return KGREC_ERR_INVALID; }
  if (!excl_row || !excl_ptr || !excl_ids) { set_error("rank_count_ex: exclusion CSR (excl_row / excl_ptr / excl_ids) has a NULL array"); return KGREC_ERR_INVALID; }
  if ((reinterpret_cast<uintptr_t>(excl_row) & 3u) || (reinterpret_cast<uintptr_t>(excl_ptr) & 7u) || (reinterpret_cast<uintptr_t>(excl_ids) & 3u)) {
    set_error("rank_count_ex: exclusion CSR arrays are not aligned to their element size");
    return KGREC_ERR_INVALID;
  }
  if (id_base < 0 || id_base + n_cat > 0xffffffffll) { set_error("catalog ids must fit 32 bits"); return KGREC_ERR_INVALID; }
  const int d = tables->dim;
  for (int g = 0; g < n_runs; ++g) {
    if ((rc = transr_prepare(C, g))) return rc;
    const int64_t i0 = run_begin_host[g], n = run_begin_host[g + 1] - i0;
    // excl_row holds absolute rows of the CSR, so a run's slice of it is valid as it stands
    rc = kgrec_eval_rank_count_ex(tables, KGREC_TRANSR, side, nullptr, nullptr, 8, C.qvec_ws + i0 * 2 * d, n, C.proj_ws, d, n_cat,
                                  id_base, gold_scores + i0, gold_ids + i0, counts + i0, excl_row + i0, excl_ptr, excl_ids, stream);
    if (rc) return rc;
  }
  return KGREC_OK;
}

extern "C" int kgrec_transr_eval_rank_count_dual(const kgrec_tables* tables, int side, const void* q, const void* r, int idx_bytes,
                                                 int64_t nq, const int64_t* run_begin_host, const int64_t* run_rel_host, int32_t n_runs,
                                                 const float* cat, int64_t cat_ld, int64_t n_cat, int64_t id_base, float* workspace,
                                                 const float* gold_scores, const int32_t* gold_ids, int32_t* filt_counts,
                                                 const int32_t* excl_row, const int64_t* excl_ptr, const int32_t* excl_ids,
                                                 const int64_t* gold_ptr, const int32_t* gold_set_ids, int32_t* raw_counts,
                                                 int32_t* status, kgrec_stream_t stream) {
  TRANSR_CALL();
  if (!gold_scores || !gold_ids || !filt_counts || !raw_counts) { set_error("rank_count_dual: NULL argument"); return KGREC_ERR_INVALID; }
  if (!excl_row || !excl_ptr || !excl_ids) { set_error("rank_count_ex: exclusion CSR (excl_row / excl_ptr / excl_ids) has a NULL array"); return KGREC_ERR_INVALID; }
  if (!gold_ptr || !gold_set_ids) { set_error("rank_count_dual: gold CSR (gold_ptr / gold_set_ids) has a NULL array"); return KGREC_ERR_INVALID; }
  if ((reinterpret_cast<uintptr_t>(excl_row) & 3u) || (reinterpret_cast<uintptr_t>(excl_ptr) & 7u) || (reinterpret_cast<uintptr_t>(excl_ids) & 3u) ||
      (reinterpret_cast<uintptr_t>(gold_ptr) & 7u) || (reinterpret_cast<uintptr_t>(gold_set_ids) & 3u) ||
      (reinterpret_cast<uintptr_t>(filt_counts) & 3u) || (reinterpret_cast<uintptr_t>(raw_counts) & 3u)) {
    set_error("rank_count_dual: exclusion / gold CSR or count arrays are not aligned to their element size");
    return KGREC_ERR_INVALID;
  }
  if (id_base < 0 || id_base + n_cat > 0xffffffffll) { set_error("catalog ids must fit 32 bits"); return KGREC_ERR_INVALID; }
  const int d = tables->dim;
  for (int g = 0; g < n_runs; ++g) {
    if ((rc = transr_prepare(C, g))) return rc;
    const int64_t i0 = run_begin_host[g], n = run_begin_host[g + 1] - i0;
    rc = kgrec_eval_rank_count_dual(tables, KGREC_TRANSR, side, nullptr, nullptr, 8, C.qvec_ws + i0 * 2 * d, n, C.proj_ws, d, n_cat,
                                    id_base, gold_scores + i0, gold_ids + i0, filt_counts + i0, excl_row + i0, excl_ptr, excl_ids,
                                    gold_ptr, gold_set_ids, raw_counts + i0, stream);
    if (rc) return rc;
  }
  return KGREC_OK;
}
