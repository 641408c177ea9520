// Sparse-row optimizer: the first "next" row of SURVEY 8(f).  Replaces the reference's dense
// torch.optim step + clip_grad_norm (utils/trainer.py:63-81, knowledge_representation.py:213),
// whose cost is O(table) per step, by kernels whose cost is O(rows touched by the batch) plus one
// 4-byte flag per table row.
//
// Layout.  Gradients arrive accumulated per row in a persistent dense accumulator `acc` (the training
// kernels' "dense" gradient mode; it is all-zero outside a step).  Which rows a step touched is recorded
// as an EPOCH MARK: marks[row] = step number, written by k_rows_mark from the batch's own id arrays (plain
// idempotent stores -- duplicates cost nothing, nothing is ever cleared, no atomics).  Two sweeps then
// visit the tables, ALL of them in one launch each:
//   k_rows_sqnorm   sum of |acc[row]|^2 over marked rows            (clip_grad_norm's total norm)
//   k_rows_update   clip scale, weight decay, SGD / Adagrad / Adam on the marked rows, acc row := 0
// A warp reads 32 marks with one coalesced load, ballots, and walks the set bits; a marked row is
// processed with 128-bit loads / stores (lane = 16-byte chunk).  Per step the cost is
// rows * 4 B of marks + touched rows * (2..4 reads + 2..4 writes) of d floats -- at configs[1]
// (100k entities, every row touched) ~0.25 GB, against ~1.3 GB for the id-list + CAS version it replaces.
//
// Exact (torch.optim) trajectories: kgrec_rows_update_ex / _ex_dev add SGD with momentum and RMSprop, per-table Adam
// step counts, and row mode ALL -- every row of every table of the call is updated, as the reference's dense optimizer
// does (utils/trainer.py:63-81): a marked row with its clipped accumulator, an unmarked row with gradient 0 (its
// accumulator is zero and is not read).  ALL is a flat streaming sweep (k_rows_update_all): 128-bit units, several
// units per thread in flight, one launch for every table.  Its cost is O(table) per step, the reference's own.
#include "common.cuh"

namespace kgrec {

enum { OPT_SGD = 0, OPT_ADAGRAD = 1, OPT_ADAM = 2, OPT_RMSPROP = 3 };
constexpr int kMaxOptTables = 8;
constexpr int kMaxMarkSegs = 8;

struct MarkArgs {
  kgrec_mark_seg seg[kMaxMarkSegs];
  int64_t begin[kMaxMarkSegs + 1];      // prefix sums of seg[].n
  int n_segs;
  int32_t epoch;
  const kgrec_step_state* state;        // _dev entry point: the epoch is read here
};

// marks[id] = epoch for every id of every segment.  compact: the group-compact corrupted-id format
// (v < 0 names entity ~v).  remap: ids are looked up first (KTUP: item -> aligned entity row).
__global__ void __launch_bounds__(256) k_rows_mark(const MarkArgs A, int32_t* status) {
  const int64_t total = A.begin[A.n_segs];
  const int32_t epoch = A.state ? A.state->epoch : A.epoch;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    int s = 0;
#pragma unroll
    for (int k = 1; k < kMaxMarkSegs; ++k) s += (k < A.n_segs && i >= A.begin[k]) ? 1 : 0;
    const kgrec_mark_seg& S = A.seg[s];
    int64_t v = load_idx(S.ids, i - A.begin[s], S.idx_bytes == 8);
    if (S.compact && v < 0) v = ~v;
    // out-of-range ids: the training kernels clamp them to row 0 (and raise the status word), so that is where
    // their gradient went -- mark the same row, or its accumulator would never be cleared
    if (S.remap) {
      if (static_cast<uint64_t>(v) >= static_cast<uint64_t>(S.n_remap)) { if (status) *status = 1; v = 0; }
      v = __ldg(S.remap + v);
    }
    if (static_cast<uint64_t>(v) >= static_cast<uint64_t>(S.rows)) { if (status) *status = 1; v = 0; }
    S.marks[v] = epoch;
  }
}

struct SweepArgs {
  kgrec_opt_table tab[kMaxOptTables];
  int64_t chunk_begin[kMaxOptTables + 1];    // prefix sums of ceil(rows / 32)
  int64_t unit_begin[kMaxOptTables + 1];     // prefix sums of rows * dim / (vec ? 4 : 1): the units of the ALL sweep
  int32_t div[kMaxOptTables];                // sweep rows per table row (wide rows are swept in segments)
  int n_tabs;
  int32_t epoch;
  int kind;
  float lr, eps, beta1, beta2, wd, bias1, bias2_sqrt;
  float alpha, momentum;                     // RMSprop's smoothing constant; SGD / RMSprop momentum (0: none)
  int use_s1, use_s2;                        // the rule keeps state1 / state2
  const float* sqnorm;
  float max_norm;
  const kgrec_step_state* state;             // _dev entry points: epoch, lr and Adam's step are read here
  const int64_t* steps;                      // _ex: Adam's step count per table of the call (NULL: the global step)
};

// The scalars of one step: the by-value arguments, or the device step state's
__device__ __forceinline__ int32_t sweep_epoch(const SweepArgs& A) { return A.state ? A.state->epoch : A.epoch; }

// A warp owns 32 consecutive rows of one table: one coalesced load of their marks, a ballot, and the marked rows are
// handed out kRowsInFlight at a time -- f gets the batch so that it can issue the loads of all its rows before the
// first use (the sweeps are latency-bound: a row is three dependent-free loads, a few flops, three stores).
constexpr int kRowsInFlight = 4;

template <typename F>
__device__ __forceinline__ void sweep_rows(const SweepArgs& A, int32_t epoch, F&& f) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  const int64_t total = A.chunk_begin[A.n_tabs];
  for (int64_t c = warp; c < total; c += n_warps) {
    int t = 0;
#pragma unroll
    for (int k = 1; k < kMaxOptTables; ++k) t += (k < A.n_tabs && c >= A.chunk_begin[k]) ? 1 : 0;
    const kgrec_opt_table& T = A.tab[t];
    const int64_t row0 = (c - A.chunk_begin[t]) * 32;
    const int64_t row = row0 + lane;
    bool mine = row < T.rows;
    if (mine && T.marks) mine = __ldg(T.marks + row / A.div[t]) == epoch;
    unsigned m = __ballot_sync(FULL, mine);
    while (m) {
      int64_t rows[kRowsInFlight];
      int n = 0;
#pragma unroll
      for (int i = 0; i < kRowsInFlight; ++i) {
        rows[i] = row0;
        if (m) { rows[i] = row0 + (__ffs(m) - 1); m &= m - 1; n = i + 1; }
      }
      f(T, t, rows, n, lane);
    }
  }
}

__global__ void __launch_bounds__(256) k_rows_sqnorm(const SweepArgs A, float* out) {
  float local = 0.f;
  sweep_rows(A, sweep_epoch(A), [&](const kgrec_opt_table& T, int, const int64_t (&rows)[kRowsInFlight], int n, int lane) {
    const int nch = (T.dim + 3) >> 2;
    for (int ch = lane; ch < nch; ch += 32) {
      if (T.vec) {
        float4 v[kRowsInFlight];
#pragma unroll
        for (int i = 0; i < kRowsInFlight; ++i)
          v[i] = i < n ? *reinterpret_cast<const float4*>(T.acc + rows[i] * T.dim + ch * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int i = 0; i < kRowsInFlight; ++i)
          local = fmaf(v[i].x, v[i].x, fmaf(v[i].y, v[i].y, fmaf(v[i].z, v[i].z, fmaf(v[i].w, v[i].w, local))));
      } else {
        for (int i = 0; i < n; ++i)
          for (int e = 0; e < 4 && ch * 4 + e < T.dim; ++e) { const float g = T.acc[rows[i] * T.dim + ch * 4 + e]; local = fmaf(g, g, local); }
      }
    }
  });
  local = warp_sum(local);
  __shared__ float part[8];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) part[wid] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += part[w];
    if (t != 0.f) atomicAdd(out, t);
  }
}

struct StepScalars { float lr, bias1, bias2_sqrt; };

__device__ __forceinline__ float opt_elem(const SweepArgs& A, const StepScalars& S, float pv, float gv, float* s1, float* s2) {
  if (A.wd != 0.f) gv = fmaf(A.wd, pv, gv);          // weight_decay = l2_lambda, on the rows the call updates
  if (A.kind == OPT_SGD) {
    if (A.momentum == 0.f) return pv - S.lr * gv;
    const float b = __fmul_rn(A.momentum, *s1) + gv;  // torch.optim.SGD: buf = mu buf + g (a zero buf: g) ; p -= lr buf
    *s1 = b;
    return pv - S.lr * b;
  }
  if (A.kind == OPT_ADAGRAD) {                        // torch.optim.Adagrad: sum += g^2 ; p -= lr g / (sqrt(sum) + eps)
    const float s = fmaf(gv, gv, *s1);
    *s1 = s;
    return pv - S.lr * gv / (sqrtf(s) + A.eps);
  }
  if (A.kind == OPT_RMSPROP) {                        // torch.optim.RMSprop, centered=False: sq = a sq + (1 - a) g^2
    const float sq = fmaf((1.f - A.alpha) * gv, gv, __fmul_rn(A.alpha, *s1));
    *s1 = sq;
    const float q = gv / (sqrtf(sq) + A.eps);
    if (A.momentum == 0.f) return pv - S.lr * q;      // p -= lr g / (sqrt(sq) + eps)
    const float b = __fmul_rn(A.momentum, *s2) + q;   // buf = mu buf + g / (sqrt(sq) + eps) ; p -= lr buf
    *s2 = b;
    return pv - S.lr * b;
  }
  const float m = A.beta1 * *s1 + (1.f - A.beta1) * gv;          // torch.optim.Adam on the touched rows ("lazy")
  const float v = A.beta2 * *s2 + (1.f - A.beta2) * gv * gv;
  *s1 = m;
  *s2 = v;
  return pv - (S.lr / S.bias1) * m / (sqrtf(v) / S.bias2_sqrt + A.eps);
}

// Adam's bias terms of every table of the call from its own step count (the _ex entry points), in shared memory
struct TableBias { float bias1[kMaxOptTables], bias2_sqrt[kMaxOptTables]; };

__device__ __forceinline__ void table_bias(const SweepArgs& A, TableBias& B) {
  if (threadIdx.x < A.n_tabs) {
    const float t = static_cast<float>(A.steps[threadIdx.x]);
    B.bias1[threadIdx.x] = 1.f - powf(A.beta1, t);
    B.bias2_sqrt[threadIdx.x] = sqrtf(1.f - powf(A.beta2, t));
  }
  __syncthreads();
}

__device__ __forceinline__ StepScalars table_scalars(const SweepArgs& A, const StepScalars& S, const TableBias& B, int t) {
  float b1 = S.bias1, b2 = S.bias2_sqrt;
  if (A.steps) { b1 = B.bias1[t]; b2 = B.bias2_sqrt[t]; }
  return StepScalars{S.lr, b1, b2};
}

__global__ void __launch_bounds__(256) k_rows_update(const SweepArgs A) {
  float scale = 1.f;
  if (A.sqnorm) scale = fminf(1.f, A.max_norm / (sqrtf(__ldg(A.sqnorm)) + 1e-6f));   // clip_grad_norm's coefficient
  StepScalars S0{A.lr, A.bias1, A.bias2_sqrt};
  if (A.state) {          // the host formulas of kgrec_rows_update, on the device
    const float t = static_cast<float>(A.state->step);
    S0.lr = A.state->lr;
    S0.bias1 = 1.f - powf(A.beta1, t);
    S0.bias2_sqrt = sqrtf(1.f - powf(A.beta2, t));
  }
  __shared__ TableBias B;
  if (A.steps) table_bias(A, B);
  sweep_rows(A, sweep_epoch(A), [&](const kgrec_opt_table& T, int t, const int64_t (&rows)[kRowsInFlight], int n, int lane) {
    const StepScalars S = table_scalars(A, S0, B, t);
    const int nch = (T.dim + 3) >> 2;
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int ch = lane; ch < nch; ch += 32) {
      if (T.vec) {
        float4 g[kRowsInFlight], p[kRowsInFlight], a[kRowsInFlight], b[kRowsInFlight];
#pragma unroll
        for (int i = 0; i < kRowsInFlight; ++i) {            // every load of the batch leaves before the first use
          const int64_t o = rows[i] * T.dim + ch * 4;
          g[i] = p[i] = a[i] = b[i] = z4;
          if (i < n) {
            g[i] = *reinterpret_cast<const float4*>(T.acc + o);
            p[i] = *reinterpret_cast<const float4*>(T.table + o);
            if (A.use_s1) a[i] = *reinterpret_cast<const float4*>(T.state1 + o);
            if (A.use_s2) b[i] = *reinterpret_cast<const float4*>(T.state2 + o);
          }
        }
#pragma unroll
        for (int i = 0; i < kRowsInFlight; ++i) {
          if (i >= n) continue;
          const int64_t o = rows[i] * T.dim + ch * 4;
          p[i].x = opt_elem(A, S, p[i].x, g[i].x * scale, &a[i].x, &b[i].x);
          p[i].y = opt_elem(A, S, p[i].y, g[i].y * scale, &a[i].y, &b[i].y);
          p[i].z = opt_elem(A, S, p[i].z, g[i].z * scale, &a[i].z, &b[i].z);
          p[i].w = opt_elem(A, S, p[i].w, g[i].w * scale, &a[i].w, &b[i].w);
          if (!T.keep_acc) *reinterpret_cast<float4*>(T.acc + o) = z4;                   // zero again after the step
          *reinterpret_cast<float4*>(T.table + o) = p[i];
          if (A.use_s1) *reinterpret_cast<float4*>(T.state1 + o) = a[i];
          if (A.use_s2) *reinterpret_cast<float4*>(T.state2 + o) = b[i];
        }
      } else {
#pragma unroll
        for (int i = 0; i < kRowsInFlight; ++i)
          for (int e = 0; i < n && e < 4 && ch * 4 + e < T.dim; ++e) {
            const int64_t o = rows[i] * T.dim + ch * 4 + e;
            const float g = T.acc[o];
            if (!T.keep_acc) T.acc[o] = 0.f;
            float a = A.use_s1 ? T.state1[o] : 0.f, b = A.use_s2 ? T.state2[o] : 0.f;
            T.table[o] = opt_elem(A, S, T.table[o], g * scale, &a, &b);
            if (A.use_s1) T.state1[o] = a;
            if (A.use_s2) T.state2[o] = b;
          }
      }
    }
  });
}

// Row mode ALL: every row of every table.  The tables are one flat array of units -- a float4 (vec tables) or a float
// (the scalar path) -- walked grid-stride, kAllUnroll units a thread in flight: marks, parameters and state are loaded
// for all of them, then the accumulators of the marked ones, then the rule runs and everything is stored.  An unmarked
// row's gradient is 0: its accumulator is neither read nor written.
constexpr int kAllUnroll = 4;

__device__ __forceinline__ float4 ld_unit(const float* base, int64_t o, bool vec) {
  return vec ? *reinterpret_cast<const float4*>(base + o) : make_float4(base[o], 0.f, 0.f, 0.f);
}

__device__ __forceinline__ void st_unit(float* base, int64_t o, bool vec, const float4& v) {
  if (vec) *reinterpret_cast<float4*>(base + o) = v;
  else base[o] = v.x;
}

__global__ void __launch_bounds__(256) k_rows_update_all(const SweepArgs A) {
  float scale = 1.f;
  if (A.sqnorm) scale = fminf(1.f, A.max_norm / (sqrtf(__ldg(A.sqnorm)) + 1e-6f));   // clip_grad_norm's coefficient
  StepScalars S0{A.lr, A.bias1, A.bias2_sqrt};
  if (A.state) S0.lr = A.state->lr;
  __shared__ TableBias B;
  if (A.steps) table_bias(A, B);
  const int32_t epoch = sweep_epoch(A);
  const int64_t total = A.unit_begin[A.n_tabs];
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int64_t base = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; base < total; base += kAllUnroll * stride) {
    int tab[kAllUnroll];
    int64_t off[kAllUnroll];
    bool on[kAllUnroll], marked[kAllUnroll];
    float4 p[kAllUnroll], a[kAllUnroll], b[kAllUnroll], g[kAllUnroll];
#pragma unroll
    for (int i = 0; i < kAllUnroll; ++i) {           // marks, parameters and state of every unit first
      const int64_t u = base + i * stride;
      on[i] = u < total;
      int t = 0;
#pragma unroll
      for (int k = 1; k < kMaxOptTables; ++k) t += (k < A.n_tabs && u >= A.unit_begin[k]) ? 1 : 0;
      tab[i] = t;
      const kgrec_opt_table& T = A.tab[t];
      const int64_t local = u - A.unit_begin[t];
      const int64_t per_row = T.vec ? (T.dim >> 2) : T.dim;
      const int64_t row = local < 0xFFFFFFFFll ? static_cast<int64_t>(static_cast<uint32_t>(local) / static_cast<uint32_t>(per_row))
                                               : local / per_row;
      off[i] = T.vec ? local * 4 : local;
      marked[i] = false;
      p[i] = a[i] = b[i] = g[i] = z4;
      if (on[i]) {
        marked[i] = !T.marks || __ldg(T.marks + (A.div[t] == 1 ? row : row / A.div[t])) == epoch;
        p[i] = ld_unit(T.table, off[i], T.vec);
        if (A.use_s1) a[i] = ld_unit(T.state1, off[i], T.vec);
        if (A.use_s2) b[i] = ld_unit(T.state2, off[i], T.vec);
      }
    }
#pragma unroll
    for (int i = 0; i < kAllUnroll; ++i)              // then the gradients of the marked units
      if (marked[i]) g[i] = ld_unit(A.tab[tab[i]].acc, off[i], A.tab[tab[i]].vec);
#pragma unroll
    for (int i = 0; i < kAllUnroll; ++i) {
      if (!on[i]) continue;
      const kgrec_opt_table& T = A.tab[tab[i]];
      const StepScalars S = table_scalars(A, S0, B, tab[i]);
      p[i].x = opt_elem(A, S, p[i].x, g[i].x * scale, &a[i].x, &b[i].x);
      if (T.vec) {
        p[i].y = opt_elem(A, S, p[i].y, g[i].y * scale, &a[i].y, &b[i].y);
        p[i].z = opt_elem(A, S, p[i].z, g[i].z * scale, &a[i].z, &b[i].z);
        p[i].w = opt_elem(A, S, p[i].w, g[i].w * scale, &a[i].w, &b[i].w);
      }
      if (marked[i] && !T.keep_acc) st_unit(T.acc, off[i], T.vec, z4);
      st_unit(T.table, off[i], T.vec, p[i]);
      if (A.use_s1) st_unit(T.state1, off[i], T.vec, a[i]);
      if (A.use_s2) st_unit(T.state2, off[i], T.vec, b[i]);
    }
  }
}

// Adam's per-table step counts: +1 for every table of the call, ordered in the stream ahead of the sweep that reads them
__global__ void k_step_counts(int64_t* steps, int n_tabs) {
  if (threadIdx.x < n_tabs) steps[threadIdx.x] += 1;
}

}  // namespace kgrec

using namespace kgrec;

static int sweep_args(const kgrec_opt_table* tabs, int n_tabs, int32_t epoch, int need_table, SweepArgs& A) {
  if (!tabs || n_tabs < 1 || n_tabs > kMaxOptTables) {
    set_error("sparse row optimizer: 1..%d tables per call", kMaxOptTables);
    return KGREC_ERR_INVALID;
  }
  A = SweepArgs{};
  A.n_tabs = n_tabs;
  A.epoch = epoch;
  for (int t = 0; t < n_tabs; ++t) {
    kgrec_opt_table T = tabs[t];
    if (!T.acc || T.rows <= 0 || T.dim <= 0 || (need_table && !T.table)) {
      set_error("sparse row optimizer: table %d has no accumulator / parameter / shape", t);
      return KGREC_ERR_INVALID;
    }
    T.vec = (T.dim % 4 == 0) && (reinterpret_cast<uintptr_t>(T.acc) % 16 == 0) &&
            (!T.table || reinterpret_cast<uintptr_t>(T.table) % 16 == 0) &&
            (!T.state1 || reinterpret_cast<uintptr_t>(T.state1) % 16 == 0) &&
            (!T.state2 || reinterpret_cast<uintptr_t>(T.state2) % 16 == 0);
    // wide rows (TransR's d x d matrices: 10^4 floats per row, a few hundred rows) are swept as rows of a segment each, or
    // a handful of warps would walk the whole table
    A.div[t] = 1;
    if (T.dim > 512)
      for (int seg = 512; seg >= 64; seg -= 4)
        if (T.dim % seg == 0) { A.div[t] = T.dim / seg; T.rows *= A.div[t]; T.dim = seg; break; }
    A.tab[t] = T;
    A.chunk_begin[t + 1] = A.chunk_begin[t] + (T.rows + 31) / 32;
    A.unit_begin[t + 1] = A.unit_begin[t] + T.rows * T.dim / (T.vec ? 4 : 1);
  }
  for (int t = n_tabs; t < kMaxOptTables; ++t) {
    A.chunk_begin[t + 1] = A.chunk_begin[n_tabs];
    A.unit_begin[t + 1] = A.unit_begin[n_tabs];
  }
  // An update clears an entry's accumulator rows as it consumes them, and the warps of all the entries of a call run
  // concurrently: another entry of the same call reading that memory could see it cleared already.  keep_acc = 1
  // shares an accumulator with an entry of a later call only.
  if (need_table)
    for (int t = 0; t < n_tabs; ++t)
      for (int o = 0; o < n_tabs; ++o) {
        if (o == t || tabs[o].keep_acc) continue;
        const uintptr_t t0 = reinterpret_cast<uintptr_t>(tabs[t].acc), o0 = reinterpret_cast<uintptr_t>(tabs[o].acc);
        const uintptr_t t1 = t0 + static_cast<uintptr_t>(tabs[t].rows) * tabs[t].dim * sizeof(float);
        const uintptr_t o1 = o0 + static_cast<uintptr_t>(tabs[o].rows) * tabs[o].dim * sizeof(float);
        if (t0 < o1 && o0 < t1) {
          set_error("sparse row optimizer: table %d reads the accumulator that table %d of the same call clears "
                    "(keep_acc = 0); an accumulator cleared by one entry is read by no other entry of the call", t, o);
          return KGREC_ERR_INVALID;
        }
      }
  return KGREC_OK;
}

static int sweep_grid(const SweepArgs& A) {
  const int64_t warps = A.chunk_begin[A.n_tabs], ctas = (warps + 7) / 8, cap = static_cast<int64_t>(sm_count()) * 8;
  return static_cast<int>(ctas < 1 ? 1 : (ctas < cap ? ctas : cap));
}

static int rows_mark(const kgrec_mark_seg* segs, int n_segs, int32_t epoch, const kgrec_step_state* state,
                     int32_t* status, kgrec_stream_t stream) {
  if (!segs || n_segs < 1 || n_segs > kMaxMarkSegs) {
    set_error("kgrec_rows_mark: 1..%d id segments per call", kMaxMarkSegs);
    return KGREC_ERR_INVALID;
  }
  MarkArgs A{};
  A.n_segs = n_segs;
  A.epoch = epoch;
  A.state = state;
  for (int s = 0; s < n_segs; ++s) {
    const kgrec_mark_seg& S = segs[s];
    if (S.n < 0 || (S.n > 0 && (!S.ids || !S.marks)) || (S.idx_bytes != 4 && S.idx_bytes != 8) || S.rows <= 0) {
      set_error("kgrec_rows_mark: bad segment %d", s);
      return KGREC_ERR_INVALID;
    }
    A.seg[s] = S;
    A.begin[s + 1] = A.begin[s] + S.n;
  }
  for (int s = n_segs; s < kMaxMarkSegs; ++s) A.begin[s + 1] = A.begin[n_segs];
  const int64_t total = A.begin[n_segs];
  if (total == 0) return KGREC_OK;
  const int64_t blocks = (total + 255) / 256, cap = static_cast<int64_t>(sm_count()) * 16;
  k_rows_mark<<<static_cast<int>(blocks < cap ? blocks : cap), 256, 0, static_cast<cudaStream_t>(stream)>>>(A, status);
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

static int rows_sqnorm(const kgrec_opt_table* tabs, int n_tabs, int32_t epoch, const kgrec_step_state* state, float* sqnorm,
                       kgrec_stream_t stream) {
  SweepArgs A;
  int rc = sweep_args(tabs, n_tabs, epoch, 0, A);
  if (rc) return rc;
  A.state = state;
  if (!sqnorm) { set_error("sqnorm is NULL"); return KGREC_ERR_INVALID; }
  k_rows_sqnorm<<<sweep_grid(A), 256, 0, static_cast<cudaStream_t>(stream)>>>(A, sqnorm);
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

static int rows_update(const kgrec_opt_table* tabs, int n_tabs, int32_t epoch, const kgrec_step_state* state, int kind,
                       float lr, float eps, float beta1, float beta2, int64_t step, float weight_decay,
                       const float* sqnorm, float max_norm, kgrec_stream_t stream) {
  SweepArgs A;
  int rc = sweep_args(tabs, n_tabs, epoch, 1, A);
  if (rc) return rc;
  if (kind < OPT_SGD || kind > OPT_ADAM) { set_error("sparse row optimizer: unknown kind %d", kind); return KGREC_ERR_INVALID; }
  for (int t = 0; t < n_tabs; ++t)
    if ((kind != OPT_SGD && !tabs[t].state1) || (kind == OPT_ADAM && !tabs[t].state2)) {
      set_error("sparse row optimizer: state missing for optimizer kind %d (table %d)", kind, t);
      return KGREC_ERR_INVALID;
    }
  A.kind = kind; A.lr = lr; A.eps = eps; A.beta1 = beta1; A.beta2 = beta2; A.wd = weight_decay;
  A.use_s1 = kind != OPT_SGD;
  A.use_s2 = kind == OPT_ADAM;
  A.bias1 = 1.f - powf(beta1, static_cast<float>(step));
  A.bias2_sqrt = sqrtf(1.f - powf(beta2, static_cast<float>(step)));
  A.sqnorm = sqnorm; A.max_norm = max_norm; A.state = state;
  k_rows_update<<<sweep_grid(A), 256, 0, static_cast<cudaStream_t>(stream)>>>(A);
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

// kgrec_rows_update_ex / _ex_dev: every rule, either row mode, Adam's step count per table
static int rows_update_ex(const kgrec_opt_table* tabs, int n_tabs, int32_t epoch, const kgrec_step_state* state,
                          const kgrec_opt_params* P, const float* sqnorm, kgrec_stream_t stream) {
  if (!P) { set_error("sparse row optimizer: params is NULL"); return KGREC_ERR_INVALID; }
  SweepArgs A;
  int rc = sweep_args(tabs, n_tabs, epoch, 1, A);
  if (rc) return rc;
  const int kind = P->kind;
  if (kind < OPT_SGD || kind > OPT_RMSPROP) { set_error("sparse row optimizer: unknown kind %d", kind); return KGREC_ERR_INVALID; }
  if (P->rows != KGREC_ROWS_TOUCHED && P->rows != KGREC_ROWS_ALL) {
    set_error("sparse row optimizer: unknown row mode %d", P->rows);
    return KGREC_ERR_INVALID;
  }
  A.use_s1 = kind != OPT_SGD || P->momentum != 0.f;
  A.use_s2 = kind == OPT_ADAM || (kind == OPT_RMSPROP && P->momentum != 0.f);
  for (int t = 0; t < n_tabs; ++t)
    if ((A.use_s1 && !tabs[t].state1) || (A.use_s2 && !tabs[t].state2)) {
      set_error("sparse row optimizer: state missing for optimizer kind %d, momentum %g (table %d)", kind,
                static_cast<double>(P->momentum), t);
      return KGREC_ERR_INVALID;
    }
  if (kind == OPT_ADAM && !P->step_counts) {
    set_error("sparse row optimizer: Adam needs its per-table step counts (step_counts is NULL)");
    return KGREC_ERR_INVALID;
  }
  A.kind = kind; A.lr = P->lr; A.eps = P->eps; A.beta1 = P->beta1; A.beta2 = P->beta2; A.wd = P->weight_decay;
  A.alpha = P->alpha; A.momentum = P->momentum;
  A.sqnorm = sqnorm; A.max_norm = P->max_norm; A.state = state; A.steps = P->step_counts;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (P->step_counts) {
    k_step_counts<<<1, 32, 0, s>>>(P->step_counts, n_tabs);
    KGREC_CUDA_OK(cudaGetLastError());
  }
  // a zero gradient leaves a row bit-unchanged under plain SGD and Adagrad without weight decay: ALL then only costs
  // more, and the marked rows are enough
  const bool all = P->rows == KGREC_ROWS_ALL &&
                   !(((kind == OPT_SGD && P->momentum == 0.f) || kind == OPT_ADAGRAD) && P->weight_decay == 0.f);
  if (all) {
    const int64_t units = A.unit_begin[n_tabs];
    const int64_t blocks = (units + 256 * kAllUnroll - 1) / (256 * kAllUnroll), cap = static_cast<int64_t>(sm_count()) * 8;
    k_rows_update_all<<<static_cast<int>(blocks < 1 ? 1 : (blocks < cap ? blocks : cap)), 256, 0, s>>>(A);
  } else {
    k_rows_update<<<sweep_grid(A), 256, 0, s>>>(A);
  }
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

extern "C" int kgrec_rows_mark(const kgrec_mark_seg* segs, int n_segs, int32_t epoch, int32_t* status,
                               kgrec_stream_t stream) {
  return rows_mark(segs, n_segs, epoch, nullptr, status, stream);
}

extern "C" int kgrec_rows_sqnorm(const kgrec_opt_table* tabs, int n_tabs, int32_t epoch, float* sqnorm,
                                 kgrec_stream_t stream) {
  return rows_sqnorm(tabs, n_tabs, epoch, nullptr, sqnorm, stream);
}

extern "C" int kgrec_rows_update(const kgrec_opt_table* tabs, int n_tabs, int32_t epoch, int kind, float lr, float eps,
                                 float beta1, float beta2, int64_t step, float weight_decay, const float* sqnorm,
                                 float max_norm, kgrec_stream_t stream) {
  return rows_update(tabs, n_tabs, epoch, nullptr, kind, lr, eps, beta1, beta2, step, weight_decay, sqnorm, max_norm, stream);
}

extern "C" int kgrec_rows_mark_dev(const kgrec_mark_seg* segs, int n_segs, const kgrec_step_state* state, int32_t* status,
                                   kgrec_stream_t stream) {
  if (!state) { set_error("kgrec_rows_mark_dev: step state is NULL"); return KGREC_ERR_INVALID; }
  return rows_mark(segs, n_segs, 0, state, status, stream);
}

extern "C" int kgrec_rows_sqnorm_dev(const kgrec_opt_table* tabs, int n_tabs, const kgrec_step_state* state, float* sqnorm,
                                     kgrec_stream_t stream) {
  if (!state) { set_error("sparse row optimizer: step state is NULL"); return KGREC_ERR_INVALID; }
  return rows_sqnorm(tabs, n_tabs, 0, state, sqnorm, stream);
}

extern "C" int kgrec_rows_update_dev(const kgrec_opt_table* tabs, int n_tabs, const kgrec_step_state* state, int kind,
                                     float eps, float beta1, float beta2, float weight_decay, const float* sqnorm,
                                     float max_norm, kgrec_stream_t stream) {
  if (!state) { set_error("sparse row optimizer: step state is NULL"); return KGREC_ERR_INVALID; }
  return rows_update(tabs, n_tabs, 0, state, kind, 0.f, eps, beta1, beta2, 1, weight_decay, sqnorm, max_norm, stream);
}

extern "C" int kgrec_rows_update_ex(const kgrec_opt_table* tabs, int n_tabs, int32_t epoch, const kgrec_opt_params* params,
                                    const float* sqnorm, kgrec_stream_t stream) {
  return rows_update_ex(tabs, n_tabs, epoch, nullptr, params, sqnorm, stream);
}

extern "C" int kgrec_rows_update_ex_dev(const kgrec_opt_table* tabs, int n_tabs, const kgrec_step_state* state,
                                        const kgrec_opt_params* params, const float* sqnorm, kgrec_stream_t stream) {
  if (!state) { set_error("sparse row optimizer: step state is NULL"); return KGREC_ERR_INVALID; }
  return rows_update_ex(tabs, n_tabs, 0, state, params, sqnorm, stream);
}
