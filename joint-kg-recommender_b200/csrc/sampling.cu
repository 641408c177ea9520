// Device-side negative sampling: SURVEY 8(f) next row 2.
//
// Restates the reference's samplers (utils/data.py):
//   getTrainTripleBatch :12-18  each negative corrupts the head or the tail with probability 1/2
//   corrupt_head_filter :23-38  uniform entity, redrawn while it equals the original head or the
//   corrupt_tail_filter :43-56  corrupted triple is a known one (train / valid / test dicts)
//   getNegRatings       :64-85  uniform item, redrawn while it equals the positive item or is a
//                               known item of the user (the reference's additional "no item twice
//                               in one batch" rule, data.py:66,79-82, is a host-loop artefact that
//                               cannot hold for batches larger than the catalog and is not kept)
// Known triples / ratings live in an open-addressing hash set of 64-bit keys in HBM; draws come
// from Philox4x32-10 keyed by (seed, negative index, attempt), so a batch is reproducible.
// The KG sampler emits the group-compact format of train_group.cu directly.
#include "common.cuh"

namespace kgrec {

constexpr uint64_t kEmptyKey = ~0ull;

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {   // splitmix64 finaliser
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27; x *= 0x94d049bb133111ebull;
  x ^= x >> 31;
  return x;
}

__global__ void __launch_bounds__(256) k_hashset_insert(const uint64_t* __restrict__ keys, int64_t n, uint64_t* table, uint64_t mask) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const uint64_t key = keys[i];
    uint64_t slot = mix64(key) & mask;
    while (true) {
      const uint64_t prev = atomicCAS(reinterpret_cast<unsigned long long*>(table + slot), kEmptyKey, key);
      if (prev == kEmptyKey || prev == key) break;
      slot = (slot + 1) & mask;
    }
  }
}

__device__ __forceinline__ bool hashset_contains(const uint64_t* __restrict__ table, uint64_t mask, uint64_t key) {
  uint64_t slot = mix64(key) & mask;
  while (true) {
    const uint64_t v = __ldg(table + slot);
    if (v == key) return true;
    if (v == kEmptyKey) return false;
    slot = (slot + 1) & mask;
  }
}

__device__ __forceinline__ uint64_t triple_key(uint64_t h, uint64_t r, uint64_t t, uint64_t n_ent, uint64_t n_rel) {
  return (h * n_rel + r) * n_ent + t;
}

struct SampleArgs {
  const void *a, *b, *c;     // positives: (h, t, r) or (u, i, -)
  int is64;
  int64_t n_pos; int n_neg;
  int64_t n_cat;             // entities or items
  int64_t n_rel;
  const uint64_t* table; uint64_t mask;   // table == nullptr: unfiltered
  uint64_t seed;
  int32_t* out;
  int32_t* status;           // optional: set to 2 when a key has no valid negative at all
  const kgrec_step_state* state;   // _dev entry points: seed = state->sample_seed + state->step
};

__device__ __forceinline__ uint64_t sample_seed(const SampleArgs& A) {
  return A.state ? A.state->sample_seed + static_cast<uint64_t>(A.state->step) : A.seed;
}

constexpr int kMaxAttempts = 64;

__global__ void __launch_bounds__(256) k_sample_corrupt(const SampleArgs A) {
  const int64_t total = A.n_pos * A.n_neg;
  const uint64_t seed = sample_seed(A);
  for (int64_t m = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; m < total; m += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t j = m / A.n_neg;
    const uint64_t h = static_cast<uint64_t>(load_idx(A.a, j, A.is64)), t = static_cast<uint64_t>(load_idx(A.b, j, A.is64));
    const uint64_t r = static_cast<uint64_t>(load_idx(A.c, j, A.is64));
    const bool head = philox_uniform_bits(seed, static_cast<uint64_t>(m), 0xffffffffu) & 1u;      // random.random() < 0.5
    uint32_t ent = 0;
    auto valid = [&](uint32_t e) {
      if (e == (head ? h : t)) return false;
      if (A.table) {
        const uint64_t key = head ? triple_key(e, r, t, A.n_cat, A.n_rel) : triple_key(h, r, e, A.n_cat, A.n_rel);
        if (hashset_contains(A.table, A.mask, key)) return false;
      }
      return true;
    };
    bool found = false;
    for (int attempt = 0; attempt < kMaxAttempts && !found; ++attempt) {
      const uint32_t bits = philox_uniform_bits(seed, static_cast<uint64_t>(m), static_cast<uint32_t>(attempt));
      ent = static_cast<uint32_t>((static_cast<uint64_t>(bits) * static_cast<uint64_t>(A.n_cat)) >> 32);   // randrange(entityTotal)
      found = valid(ent);
    }
    // The reference loops until a draw is valid (data.py:23-56).  After kMaxAttempts rejections (a key whose valid set
    // is a tiny share of the catalog) fall back to a scan from the last draw for the first valid id; if there is none
    // at all -- where the reference would never return -- the last draw is emitted and A.status is raised.
    for (int64_t s = 1; s < A.n_cat && !found; ++s) {
      const uint32_t e = static_cast<uint32_t>((static_cast<uint64_t>(ent) + s) % static_cast<uint64_t>(A.n_cat));
      if (valid(e)) { ent = e; found = true; }
    }
    if (!found && A.status) *A.status = 2;
    A.out[m] = head ? ~static_cast<int32_t>(ent) : static_cast<int32_t>(ent);
  }
}

__global__ void __launch_bounds__(256) k_sample_items(const SampleArgs A) {
  const int64_t total = A.n_pos * A.n_neg;
  const uint64_t seed = sample_seed(A);
  for (int64_t m = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; m < total; m += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t j = m / A.n_neg;
    const uint64_t u = static_cast<uint64_t>(load_idx(A.a, j, A.is64)), pi = static_cast<uint64_t>(load_idx(A.b, j, A.is64));
    uint32_t it = 0;
    auto valid = [&](uint32_t e) {
      return e != pi && !(A.table && hashset_contains(A.table, A.mask, u * static_cast<uint64_t>(A.n_cat) + e));
    };
    bool found = false;
    for (int attempt = 0; attempt < kMaxAttempts && !found; ++attempt) {
      const uint32_t bits = philox_uniform_bits(seed, static_cast<uint64_t>(m), static_cast<uint32_t>(attempt));
      it = static_cast<uint32_t>((static_cast<uint64_t>(bits) * static_cast<uint64_t>(A.n_cat)) >> 32);
      found = valid(it);
    }
    for (int64_t s = 1; s < A.n_cat && !found; ++s) {      // dense users: scan on from the last draw (see k_sample_corrupt)
      const uint32_t e = static_cast<uint32_t>((static_cast<uint64_t>(it) + s) % static_cast<uint64_t>(A.n_cat));
      if (valid(e)) { it = e; found = true; }
    }
    if (!found && A.status) *A.status = 2;
    A.out[m] = static_cast<int32_t>(it);
  }
}

static int grid1d(int64_t n) {
  const int64_t b = (n + 255) / 256, cap = static_cast<int64_t>(sm_count()) * 16;
  return static_cast<int>(b < 1 ? 1 : (b < cap ? b : cap));
}

}  // namespace kgrec

using namespace kgrec;

extern "C" int64_t kgrec_hashset_capacity(int64_t n_keys) {
  int64_t cap = 1024;
  while (cap < 2 * n_keys) cap <<= 1;      // load factor <= 0.5
  return cap;
}

extern "C" int kgrec_hashset_build(const uint64_t* keys, int64_t n, uint64_t* table, int64_t capacity, kgrec_stream_t stream) {
  if (!table || capacity < 2 || (capacity & (capacity - 1)) || n < 0 || (n > 0 && !keys) || 2 * n > capacity) {
    set_error("hashset_build: capacity must be a power of two >= 2 n");
    return KGREC_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  KGREC_CUDA_OK(cudaMemsetAsync(table, 0xff, static_cast<size_t>(capacity) * sizeof(uint64_t), st));
  if (n > 0) k_hashset_insert<<<grid1d(n), 256, 0, st>>>(keys, n, table, static_cast<uint64_t>(capacity - 1));
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

static int sample_check(const void* a, const void* b, int idx_bytes, int64_t n_pos, int32_t n_neg, int64_t n_cat,
                        const uint64_t* table, int64_t capacity, const int32_t* out) {
  if (!a || !b || !out || (idx_bytes != 4 && idx_bytes != 8) || n_pos < 0 || n_neg < 1 || n_cat < 2 || n_cat > 0x7fffffffll) {
    set_error("negative sampler: bad arguments");
    return KGREC_ERR_INVALID;
  }
  if (table && (capacity < 2 || (capacity & (capacity - 1)))) { set_error("negative sampler: bad hash set capacity"); return KGREC_ERR_INVALID; }
  return KGREC_OK;
}

static int sample_corrupt(const void* ph, const void* pt, const void* pr, int idx_bytes, int64_t n_pos, int32_t n_neg,
                          int64_t n_ent, int64_t n_rel, const uint64_t* table, int64_t capacity, uint64_t seed,
                          const kgrec_step_state* state, int32_t* corrupt, int32_t* status, kgrec_stream_t stream) {
  int rc = sample_check(ph, pt, idx_bytes, n_pos, n_neg, n_ent, table, capacity, corrupt);
  if (rc) return rc;
  if (!pr || n_rel < 1) { set_error("negative sampler: relations missing"); return KGREC_ERR_INVALID; }
  if (n_pos == 0) return KGREC_OK;
  const SampleArgs A{ph, pt, pr, idx_bytes == 8, n_pos, n_neg, n_ent, n_rel, table, table ? static_cast<uint64_t>(capacity - 1) : 0, seed, corrupt, status, state};
  k_sample_corrupt<<<grid1d(n_pos * n_neg), 256, 0, static_cast<cudaStream_t>(stream)>>>(A);
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

static int sample_neg_items(const void* u, const void* pi, int idx_bytes, int64_t n, int32_t n_neg, int64_t n_item,
                            const uint64_t* table, int64_t capacity, uint64_t seed, const kgrec_step_state* state,
                            int32_t* neg_items, int32_t* status, kgrec_stream_t stream) {
  int rc = sample_check(u, pi, idx_bytes, n, n_neg, n_item, table, capacity, neg_items);
  if (rc) return rc;
  if (n == 0) return KGREC_OK;
  const SampleArgs A{u, pi, nullptr, idx_bytes == 8, n, n_neg, n_item, 1, table, table ? static_cast<uint64_t>(capacity - 1) : 0, seed, neg_items, status, state};
  k_sample_items<<<grid1d(n * n_neg), 256, 0, static_cast<cudaStream_t>(stream)>>>(A);
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

extern "C" int kgrec_sample_corrupt(const void* ph, const void* pt, const void* pr, int idx_bytes, int64_t n_pos,
                                    int32_t n_neg, int64_t n_ent, int64_t n_rel, const uint64_t* table,
                                    int64_t capacity, uint64_t seed, int32_t* corrupt, int32_t* status, kgrec_stream_t stream) {
  return sample_corrupt(ph, pt, pr, idx_bytes, n_pos, n_neg, n_ent, n_rel, table, capacity, seed, nullptr, corrupt, status, stream);
}

extern "C" int kgrec_sample_neg_items(const void* u, const void* pi, int idx_bytes, int64_t n, int32_t n_neg, int64_t n_item,
                                      const uint64_t* table, int64_t capacity, uint64_t seed, int32_t* neg_items,
                                      int32_t* status, kgrec_stream_t stream) {
  return sample_neg_items(u, pi, idx_bytes, n, n_neg, n_item, table, capacity, seed, nullptr, neg_items, status, stream);
}

extern "C" int kgrec_sample_corrupt_dev(const void* ph, const void* pt, const void* pr, int idx_bytes, int64_t n_pos,
                                        int32_t n_neg, int64_t n_ent, int64_t n_rel, const uint64_t* table,
                                        int64_t capacity, const kgrec_step_state* state, int32_t* corrupt, int32_t* status,
                                        kgrec_stream_t stream) {
  if (!state) { set_error("negative sampler: step state is NULL"); return KGREC_ERR_INVALID; }
  return sample_corrupt(ph, pt, pr, idx_bytes, n_pos, n_neg, n_ent, n_rel, table, capacity, 0, state, corrupt, status, stream);
}

extern "C" int kgrec_sample_neg_items_dev(const void* u, const void* pi, int idx_bytes, int64_t n, int32_t n_neg,
                                          int64_t n_item, const uint64_t* table, int64_t capacity,
                                          const kgrec_step_state* state, int32_t* neg_items, int32_t* status,
                                          kgrec_stream_t stream) {
  if (!state) { set_error("negative sampler: step state is NULL"); return KGREC_ERR_INVALID; }
  return sample_neg_items(u, pi, idx_bytes, n, n_neg, n_item, table, capacity, 0, state, neg_items, status, stream);
}
