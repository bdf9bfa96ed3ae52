// A device group accumulator (obgpu_groups): merges, by value, the groups that obgpu_result_group_by_columns / _values left on
// results -- one per page batch, from any ctx of the device -- into one set of groups, as if every row had been in one batch.
// A result's groups are a self-contained device buffer (gvals::GroupBuf: keys, aggregates, NULL flags and a key heap holding
// copies of the string bytes), so an add never reads a batch image and the batch may be closed once its groups are added.
//   storage  per group: each column's key (an integer's order key, or a string's offset into the accumulator's own heap and its
//            length) and NULL flag, and the aggregates as [lo, hi] pairs: COUNT / SUM 128-bit, MIN / MAX the order key (sign bit
//            flipped as gvals::order_key flips it) and a seen flag. An open-addressing table of group index + 1 (0: empty), at
//            least twice the capacity, keyed by the tuple: integers hash their order key, strings their bytes, NULL a constant.
//   grow     before an add, from the result's n_groups and key_bytes (known on the host): capacity doubles from kInitGroups,
//            the table is rebuilt from the existing groups by insert_kernel; the heap doubles. New storage is allocated before
//            the old is freed, so a failed allocation leaves the accumulator as it was.
//   add      add_kernel, one thread per incoming group. The groups of one result are distinct tuples, so within one add no two
//            threads insert the same tuple and no two threads touch the same accumulator group: the aggregates fold with plain
//            read-modify-write, and a slot claimed during the same add (kLocked, or an index past the groups before the add)
//            always holds another tuple and is passed over without comparing. New groups take an index from a counter and copy
//            their string bytes to the heap at offsets from a bump counter.
//   fetch    the order is made at fetch time, not per add: cub::DeviceMergeSort of the group indices by TupleLess (per column:
//            NULL last, integers by order key, strings bytewise as gvals::StrLess), the string lengths in that order scanned
//            into offsets, then gather_kernel writes the gvals::GroupBuf layout, cached until the next add. The tuples are
//            distinct, so the order is unique and does not depend on thread timing or on the order of the adds.
#pragma once

namespace gmerge {

constexpr int kThreads = 256;
constexpr int64_t kInitGroups = 1024;              // the first capacity; it doubles
constexpr int64_t kMaxGroups = (1ll << 31) - 1;    // the most groups an accumulator holds
constexpr int64_t kInitHeap = 64 << 10;            // the first key heap; it doubles
constexpr uint32_t kLocked = 0xffffffffu;          // a table slot being claimed in the current add
enum : int { CTR_GROUPS, CTR_HEAP, CTR_COL_BYTES, CTR_STATUS = CTR_COL_BYTES + gvals::kMaxGroupCols, CTR_N };

// the accumulator's groups on the device, capacity cap
struct Store {
  uint64_t *key;               // [n_cols][cap]: integer order key, or string heap offset
  uint32_t *len;               // [n_cols][cap]: string key bytes
  uint8_t *null;               // [n_cols][cap]
  unsigned long long *acc;     // [n_aggs][cap][2]
  uint8_t *heap;
  int64_t cap;
  int n_cols, n_aggs;
  uint32_t str_mask;
};

// byte offsets of a Store's arrays in its one allocation
struct StoreLayout {
  size_t len, null, acc, end;
  StoreLayout(int64_t cap, int n_cols, int n_aggs) {
    len = (size_t)n_cols * (size_t)cap * 8;
    null = len + (size_t)n_cols * (size_t)cap * 4;
    acc = (null + (size_t)n_cols * (size_t)cap + 15) & ~(size_t)15;
    end = acc + (size_t)n_aggs * (size_t)cap * 16;
  }
};

// one column's key of a group: the order key of an integer, or a string's bytes at base + off
struct Cell {
  bool null;
  uint64_t key;
  const uint8_t *base;
  uint64_t off;
  uint32_t len;
};

__device__ __forceinline__ Cell stored_cell(const Store &s, int c, int64_t g) {
  const int64_t i = (int64_t)c * s.cap + g;
  return Cell{s.null[i] != 0, s.key[i], s.heap, s.key[i], s.len[i]};
}

// a result's group q in its GroupBuf (ng groups): integer keys are value images, turned into order keys here
struct InGroups {
  const int64_t *keys;         // [n_cols][ng + 1]
  const int64_t *out;          // [n_aggs][ng][2]
  const uint8_t *nulls;        // [n_cols][ng]
  const uint8_t *heap;
  int64_t ng;
};

__device__ __forceinline__ Cell in_cell(const InGroups &in, uint32_t str_mask, uint32_t sgn_key, int c, int64_t q) {
  const int64_t *k = in.keys + c * (in.ng + 1);
  const bool null = in.nulls[c * in.ng + q] != 0;
  if ((str_mask >> c) & 1u) return Cell{null, 0, in.heap, (uint64_t)k[q], (uint32_t)(k[q + 1] - k[q])};
  return Cell{null, (uint64_t)k[q] ^ ((uint64_t)((sgn_key >> c) & 1u) << 63), nullptr, 0, 0};
}

__device__ __forceinline__ uint64_t cell_hash(const Cell &x, bool str) {
  if (x.null) return 0x5851F42D4C957F2Dull;
  return str ? bcodes::str_hash(x.base, x.off, x.len) : bcodes::int_hash(x.key);
}

// bytewise as unsigned bytes, 8 at a time big-endian: < 0, 0, > 0; equal up to the shorter: the shorter first
__device__ __forceinline__ int str_cmp(const Cell &x, const Cell &y) {
  const uint32_t m = x.len < y.len ? x.len : y.len;
  for (uint32_t i = 0; i < m; i += 8u) {
    const uint32_t nb = m - i < 8u ? m - i : 8u;
    const uint64_t bx = gvals::bswap64(bcodes::img_bytes(x.base, x.off, i, nb)), by = gvals::bswap64(bcodes::img_bytes(y.base, y.off, i, nb));
    if (bx != by) return bx < by ? -1 : 1;
  }
  return x.len == y.len ? 0 : x.len < y.len ? -1 : 1;
}

// one column's order: NULL last, integers by order key, strings bytewise
__device__ __forceinline__ int cell_cmp(const Cell &x, const Cell &y, bool str) {
  if (x.null || y.null) return (int)x.null - (int)y.null;
  if (str) return str_cmp(x, y);
  return x.key == y.key ? 0 : x.key < y.key ? -1 : 1;
}

// Slot for a tuple of hash h. A slot holding a group from an earlier add (index < n_before) is offered to eq; a slot claimed
// in this add holds another tuple and is passed over. Returns the slot and sets *claimed when an empty slot was claimed (it then
// holds kLocked until the caller stores the group's index + 1); ~0 when the table is full.
template <class Eq>
__device__ __forceinline__ uint64_t find_or_claim(uint32_t *table, uint64_t mask, uint64_t h, int64_t n_before, Eq eq, bool *claimed) {
  uint64_t slot = h & mask;
  for (uint64_t k = 0; k <= mask; ++k, slot = (slot + 1u) & mask) {
    uint32_t cur = *(volatile uint32_t *)&table[slot];
    if (cur == 0u) {
      cur = atomicCAS(&table[slot], 0u, kLocked);
      if (cur == 0u) {
        *claimed = true;
        return slot;
      }
    }
    if (cur == kLocked || (int64_t)cur - 1 >= n_before) continue;
    if (eq((int64_t)cur - 1)) {
      *claimed = false;
      return slot;
    }
  }
  return ~0ull;
}

__device__ __forceinline__ uint64_t tuple_hash(const Cell (&t)[gvals::kMaxGroupCols], int n_cols, uint32_t str_mask) {
  uint64_t h = 0x243F6A8885A308D3ull;
  for (int c = 0; c < n_cols; ++c) {
    h = (h ^ cell_hash(t[c], (str_mask >> c) & 1u)) * 0xD6E8FEB86659FD93ull;
    h ^= h >> 29;
  }
  return h ^ (h >> 32);
}

// the existing groups [0, n) into an empty table (a rebuild after growth): every tuple is distinct, nothing is compared
__global__ void __launch_bounds__(kThreads) insert_kernel(const __grid_constant__ Store s, int64_t n, uint32_t *table, uint64_t mask,
                                                          unsigned long long *ctr) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  Cell t[gvals::kMaxGroupCols];
  for (int c = 0; c < s.n_cols; ++c) t[c] = stored_cell(s, c, g);
  bool claimed = false;
  const uint64_t slot = find_or_claim(table, mask, tuple_hash(t, s.n_cols, s.str_mask), 0, [](int64_t) { return false; }, &claimed);
  if (slot == ~0ull) { atomicOr(&ctr[CTR_STATUS], 1ull); return; }
  table[slot] = (uint32_t)(g + 1);
}

struct AddArgs {
  Store s;
  uint32_t *table;
  uint64_t mask;
  InGroups in;
  int32_t kind[16];
  uint32_t sgn_key, sgn_agg;   // bit c: group column c's order key has its sign bit flipped; bit k: aggregate k's MIN / MAX key
  int64_t n_before;            // groups before this add
  unsigned long long *ctr;     // CTR_*
};

// incoming group q -> its accumulator group: folded into an equal tuple's, or a new group
__global__ void __launch_bounds__(kThreads) add_kernel(const __grid_constant__ AddArgs p) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= p.in.ng) return;
  const Store &s = p.s;
  Cell t[gvals::kMaxGroupCols];
  for (int c = 0; c < s.n_cols; ++c) t[c] = in_cell(p.in, s.str_mask, p.sgn_key, c, q);
  const auto eq = [&](int64_t g) {
    for (int c = 0; c < s.n_cols; ++c)
      if (cell_cmp(t[c], stored_cell(s, c, g), (s.str_mask >> c) & 1u) != 0) return false;
    return true;
  };
  bool claimed = false;
  const uint64_t slot = find_or_claim(p.table, p.mask, tuple_hash(t, s.n_cols, s.str_mask), p.n_before, eq, &claimed);
  if (slot == ~0ull) { atomicOr(&p.ctr[CTR_STATUS], 1ull); return; }
  if (claimed) {
    const int64_t g = (int64_t)atomicAdd(&p.ctr[CTR_GROUPS], 1ull);
    for (int c = 0; c < s.n_cols; ++c) {
      const int64_t i = (int64_t)c * s.cap + g;
      s.null[i] = t[c].null ? 1 : 0;
      if ((s.str_mask >> c) & 1u) {
        const uint64_t o = atomicAdd(&p.ctr[CTR_HEAP], (unsigned long long)t[c].len);
        atomicAdd(&p.ctr[CTR_COL_BYTES + c], (unsigned long long)t[c].len);
        for (uint32_t b = 0; b < t[c].len; ++b) s.heap[o + b] = t[c].base[t[c].off + b];
        s.key[i] = o;
        s.len[i] = t[c].len;
      } else {
        s.key[i] = t[c].null ? 0 : t[c].key;
        s.len[i] = 0;
      }
    }
    for (int k = 0; k < s.n_aggs; ++k) {
      const int64_t *v = p.in.out + ((int64_t)k * p.in.ng + q) * 2;
      unsigned long long *a = s.acc + ((int64_t)k * s.cap + g) * 2;
      const bool mm = p.kind[k] == OBGPU_AGG_MIN || p.kind[k] == OBGPU_AGG_MAX;
      a[0] = mm && v[1] ? (uint64_t)v[0] ^ ((uint64_t)((p.sgn_agg >> k) & 1u) << 63) : (uint64_t)v[0];
      a[1] = (uint64_t)v[1];
    }
    p.table[slot] = (uint32_t)(g + 1);
    return;
  }
  const int64_t g = (int64_t)p.table[slot] - 1;
  for (int k = 0; k < s.n_aggs; ++k) {
    const int64_t *v = p.in.out + ((int64_t)k * p.in.ng + q) * 2;
    unsigned long long *a = s.acc + ((int64_t)k * s.cap + g) * 2;
    if (p.kind[k] == OBGPU_AGG_MIN || p.kind[k] == OBGPU_AGG_MAX) {
      if (!v[1]) continue;
      const uint64_t key = (uint64_t)v[0] ^ ((uint64_t)((p.sgn_agg >> k) & 1u) << 63);
      if (!a[1] || (p.kind[k] == OBGPU_AGG_MIN ? key < a[0] : key > a[0])) a[0] = key;
      a[1] = 1ull;
      continue;
    }
    const uint64_t lo = a[0] + (uint64_t)v[0];   // 128-bit add: the low word's carry into the high word
    a[1] += (uint64_t)v[1] + (lo < a[0] ? 1ull : 0ull);
    a[0] = lo;
  }
}

// group indices in tuple order
struct TupleLess {
  Store s;
  __device__ bool operator()(uint32_t x, uint32_t y) const {
    for (int c = 0; c < s.n_cols; ++c) {
      const int r = cell_cmp(stored_cell(s, c, x), stored_cell(s, c, y), (s.str_mask >> c) & 1u);
      if (r) return r < 0;
    }
    return false;
  }
};

// string column c's key bytes of the q-th group in order, at slen[c][q]
__global__ void sorted_lens_kernel(const __grid_constant__ Store s, const uint32_t *order, int64_t n, int64_t *slen) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  for (int c = 0; c < s.n_cols; ++c)
    if ((s.str_mask >> c) & 1u) slen[c * n + q] = s.len[(int64_t)c * s.cap + order[q]];
}

struct GatherArgs {
  Store s;
  const uint32_t *order;
  int64_t n;
  int32_t kind[16];
  uint32_t sgn_key, sgn_agg;
  const int64_t *soff;         // [n_cols][n]: string column c's offset of the q-th group's bytes
  int64_t base[gvals::kMaxGroupCols];   // heap offset of string column c's first byte
  int64_t *keys;               // the GroupBuf's
  int64_t *out;
  uint8_t *nulls, *heap;
};

// the q-th group in order into the GroupBuf layout, exactly as gvals::gather_kernel writes it
__global__ void __launch_bounds__(kThreads) gather_kernel(const __grid_constant__ GatherArgs p) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= p.n) return;
  const Store &s = p.s;
  const int64_t g = p.order[q];
  for (int c = 0; c < s.n_cols; ++c) {
    const Cell x = stored_cell(s, c, g);
    int64_t *keys = p.keys + c * (p.n + 1);
    p.nulls[c * p.n + q] = x.null ? 1 : 0;
    if ((s.str_mask >> c) & 1u) {
      const int64_t o = p.base[c] + p.soff[c * p.n + q];
      keys[q] = o;
      if (q + 1 == p.n) keys[q + 1] = o + x.len;
      for (uint32_t b = 0; b < x.len; ++b) p.heap[o + b] = s.heap[x.off + b];
    } else {
      keys[q] = x.null ? 0 : (int64_t)(x.key ^ ((uint64_t)((p.sgn_key >> c) & 1u) << 63));
    }
  }
  for (int k = 0; k < s.n_aggs; ++k) {
    const unsigned long long *a = s.acc + ((int64_t)k * s.cap + g) * 2;
    int64_t *o = p.out + ((int64_t)k * p.n + q) * 2;
    uint64_t lo = a[0];
    if (p.kind[k] == OBGPU_AGG_MIN || p.kind[k] == OBGPU_AGG_MAX) lo = a[1] ? lo ^ ((uint64_t)((p.sgn_agg >> k) & 1u) << 63) : 0ull;
    o[0] = (int64_t)lo;
    o[1] = (int64_t)a[1];
  }
}

}  // namespace gmerge

struct obgpu_groups {
  obgpu_ctx *ctx = nullptr;    // the caller's: fetch errors and launches are counted there
  // the accumulator's own stream (device and stream only, for Scratch and CUDA_TRY): an add waits for the accumulator's work, not
  // for whatever else the caller's ctx has queued, e.g. the scan of another page batch of the same pipeline
  obgpu_ctx own;
  int32_t n_cols = 0, n_aggs = 0;
  int32_t kind[16] = {0}, agg_col[16] = {0};
  // set by the first add: each group column's and aggregate column's obj_type, and what they imply
  bool typed = false;
  int32_t key_type[gvals::kMaxGroupCols] = {0}, agg_type[16] = {0};
  uint32_t str_mask = 0, sgn_key = 0, sgn_agg = 0;
  int64_t n = 0, cap = 0, heap_cap = 0, heap_used = 0;
  int64_t col_bytes[gvals::kMaxGroupCols] = {0};
  void *d_store = nullptr;     // gmerge::StoreLayout(cap)
  uint32_t *d_table = nullptr; // 2 x cap slots
  uint8_t *d_heap = nullptr;   // heap_cap + 16 bytes (img_bytes reads up to 16 bytes past a key)
  unsigned long long *d_ctr = nullptr;   // gmerge::CTR_*
  void *d_gv = nullptr;        // the groups in order (gvals::GroupBuf), cached by fetch until the next add
};

namespace gmerge {

static Store store_of(const obgpu_groups *g, void *base, int64_t cap, uint8_t *heap) {
  const StoreLayout l(cap, g->n_cols, g->n_aggs);
  uint8_t *b = (uint8_t *)base;
  return Store{(uint64_t *)b, (uint32_t *)(b + l.len), b + l.null, (unsigned long long *)(b + l.acc), heap, cap, g->n_cols, g->n_aggs,
               g->str_mask};
}

// room for `more` groups and `more_bytes` key bytes; on failure the accumulator is as it was. Errors go to ectx.
static int grow(obgpu_groups *g, obgpu_ctx *ectx, int64_t more, int64_t more_bytes) {
  obgpu_ctx *ctx = &g->own;
  if (g->heap_used + more_bytes > g->heap_cap) {
    int64_t hc = std::max<int64_t>(kInitHeap, g->heap_cap);
    while (hc < g->heap_used + more_bytes) hc *= 2;
    Scratch h(ctx);
    CUDA_TRY(ectx, h.alloc((size_t)hc + 16));
    if (g->heap_used > 0) CUDA_TRY(ectx, cudaMemcpyAsync(h.p, g->d_heap, (size_t)g->heap_used, cudaMemcpyDeviceToDevice, ctx->stream));
    if (g->d_heap) cudaFreeAsync(g->d_heap, ctx->stream);
    g->d_heap = (uint8_t *)h.release();
    g->heap_cap = hc;
  }
  if (g->n + more <= g->cap) return OBGPU_SUCCESS;
  int64_t cap = std::max<int64_t>(kInitGroups, g->cap);
  while (cap < g->n + more) cap *= 2;
  const StoreLayout nl(cap, g->n_cols, g->n_aggs);
  Scratch sm(ctx);
  const size_t o_store = sm.take(nl.end), o_table = sm.take((size_t)cap * 2 * 4);
  CUDA_TRY(ectx, sm.alloc());
  const Store ns = store_of(g, sm.p + o_store, cap, g->d_heap);
  uint32_t *table = sm.at<uint32_t>(o_table);
  CUDA_TRY(ectx, cudaMemsetAsync(table, 0, (size_t)cap * 2 * 4, ctx->stream));
  if (g->n > 0) {
    const Store os = store_of(g, g->d_store, g->cap, g->d_heap);
    const size_t n = (size_t)g->n;
    for (int c = 0; c < g->n_cols; ++c) {
      CUDA_TRY(ectx, cudaMemcpyAsync(ns.key + (size_t)c * cap, os.key + (size_t)c * g->cap, n * 8, cudaMemcpyDeviceToDevice, ctx->stream));
      CUDA_TRY(ectx, cudaMemcpyAsync(ns.len + (size_t)c * cap, os.len + (size_t)c * g->cap, n * 4, cudaMemcpyDeviceToDevice, ctx->stream));
      CUDA_TRY(ectx, cudaMemcpyAsync(ns.null + (size_t)c * cap, os.null + (size_t)c * g->cap, n, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    for (int k = 0; k < g->n_aggs; ++k)
      CUDA_TRY(ectx, cudaMemcpyAsync(ns.acc + (size_t)k * cap * 2, os.acc + (size_t)k * g->cap * 2, n * 16, cudaMemcpyDeviceToDevice, ctx->stream));
    insert_kernel<<<(unsigned)((g->n + kThreads - 1) / kThreads), kThreads, 0, ctx->stream>>>(ns, g->n, table, (uint64_t)cap * 2 - 1, g->d_ctr);
    ectx->launches++;
    CUDA_TRY(ectx, cudaGetLastError());
  }
  if (g->d_store) cudaFreeAsync(g->d_store, ctx->stream);
  g->d_store = sm.release();
  g->d_table = table;
  g->cap = cap;
  return OBGPU_SUCCESS;
}

}  // namespace gmerge

extern "C" {

int obgpu_groups_create(obgpu_ctx *ctx, int32_t n_group_cols, const obgpu_group_agg *aggs, int32_t n_aggs, obgpu_groups **out) {
  if (!ctx || !out || n_group_cols < 1 || n_group_cols > gvals::kMaxGroupCols || !aggs || n_aggs < 1 || n_aggs > 16) return OBGPU_INVALID_ARGUMENT;
  std::unique_ptr<obgpu_groups> g(new (std::nothrow) obgpu_groups());
  if (!g) return OBGPU_ALLOCATE_MEMORY_FAILED;
  g->ctx = ctx;
  g->n_cols = n_group_cols;
  g->n_aggs = n_aggs;
  for (int k = 0; k < n_aggs; ++k) {
    g->kind[k] = aggs[k].kind;
    g->agg_col[k] = aggs[k].col;
  }
  cudaSetDevice(ctx->device);
  g->own.device = ctx->device;
  g->own.sm_count = ctx->sm_count;
  CUDA_TRY(ctx, cudaStreamCreateWithFlags(&g->own.own_stream, cudaStreamNonBlocking));
  g->own.stream = g->own.own_stream;
  const cudaError_t e = cudaMallocAsync((void **)&g->d_ctr, gmerge::CTR_N * 8, g->own.stream);
  if (e != cudaSuccess || cudaMemsetAsync(g->d_ctr, 0, gmerge::CTR_N * 8, g->own.stream) != cudaSuccess) {
    ctx->err = std::string("obgpu_groups_create: ") + cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError());
    obgpu_groups_free(g.release());
    return e == cudaErrorMemoryAllocation ? OBGPU_ALLOCATE_MEMORY_FAILED : OBGPU_ERR_SYS;
  }
  *out = g.release();
  return OBGPU_SUCCESS;
}

void obgpu_groups_free(obgpu_groups *g) {
  if (!g) return;
  cudaSetDevice(g->ctx->device);
  if (g->own.stream) {
    for (void *p : {(void *)g->d_store, (void *)g->d_heap, (void *)g->d_ctr, g->d_gv})
      if (p) cudaFreeAsync(p, g->own.stream);
    cudaStreamDestroy(g->own.stream);   // its resources go once the frees queued on it have run
  }
  delete g;
}

int obgpu_groups_add(obgpu_groups *g, obgpu_result *r) {
  if (!g || !r || r->gv_groups < 0 || r->ctx->device != g->ctx->device) return OBGPU_INVALID_ARGUMENT;
  obgpu_ctx *ectx = r->ctx;   // the caller's ctx: errors and launches are counted there
  if (r->gv_n_cols != g->n_cols || r->gv_n_aggs != g->n_aggs) {
    ectx->err = "the result's groups have another number of group columns or aggregates than the accumulator";
    return OBGPU_NOT_SUPPORTED;
  }
  for (int k = 0; k < g->n_aggs; ++k)
    if (r->gv_kind[k] != g->kind[k] || r->gv_agg_col[k] != g->agg_col[k]) {
      ectx->err = "aggregate " + std::to_string(k) + " of the result's groups differs from the accumulator's";
      return OBGPU_NOT_SUPPORTED;
    }
  if (g->typed) {
    for (int c = 0; c < g->n_cols; ++c)
      if (r->gv_key_type[c] != g->key_type[c]) {
        ectx->err = "group column " + std::to_string(c) + " has another obj_type than in the first add";
        return OBGPU_NOT_SUPPORTED;
      }
    for (int k = 0; k < g->n_aggs; ++k)
      if (r->gv_agg_type[k] != g->agg_type[k]) {
        ectx->err = "the column of aggregate " + std::to_string(k) + " has another obj_type than in the first add";
        return OBGPU_NOT_SUPPORTED;
      }
  }
  const int64_t ng = r->gv_groups, kb = r->gv_key_bytes;
  if (g->n + ng > gmerge::kMaxGroups) {
    ectx->err = "the accumulator would hold more than 2^31 - 1 groups";
    return OBGPU_NOT_SUPPORTED;
  }
  cudaSetDevice(g->ctx->device);
  CUDA_TRY(ectx, cudaStreamSynchronize(r->ctx->stream));   // the result's groups are written on its own stream
  // growing rebuilds only groups of earlier adds, so the first add's types may be taken once it has room
  if (ng > 0)
    if (const int ret = gmerge::grow(g, ectx, ng, kb); ret != OBGPU_SUCCESS) return ret;
  if (!g->typed) {
    g->typed = true;
    for (int c = 0; c < g->n_cols; ++c) g->key_type[c] = r->gv_key_type[c];
    for (int k = 0; k < g->n_aggs; ++k) g->agg_type[k] = r->gv_agg_type[k];
    g->str_mask = r->gv_str_mask;
    g->sgn_key = r->gv_sgn_key;
    g->sgn_agg = r->gv_sgn_agg;
  }
  if (ng == 0) return OBGPU_SUCCESS;
  obgpu_ctx *ctx = &g->own;
  const gvals::GroupBuf lay(ng, g->n_cols, g->n_aggs, kb);
  const uint8_t *gv = (const uint8_t *)r->d_gv;
  gmerge::AddArgs p{};
  p.s = gmerge::store_of(g, g->d_store, g->cap, g->d_heap);
  p.table = g->d_table;
  p.mask = (uint64_t)g->cap * 2 - 1;
  p.in = gmerge::InGroups{(const int64_t *)gv, (const int64_t *)(gv + lay.out), gv + lay.nulls, gv + lay.heap, ng};
  for (int k = 0; k < g->n_aggs; ++k) p.kind[k] = g->kind[k];
  p.sgn_key = g->sgn_key;
  p.sgn_agg = g->sgn_agg;
  p.n_before = g->n;
  p.ctr = g->d_ctr;
  gmerge::add_kernel<<<(unsigned)((ng + gmerge::kThreads - 1) / gmerge::kThreads), gmerge::kThreads, 0, ctx->stream>>>(p);
  ectx->launches++;
  CUDA_TRY(ectx, cudaGetLastError());
  if (g->d_gv) cudaFreeAsync(g->d_gv, ctx->stream);
  g->d_gv = nullptr;
  unsigned long long *hc = (unsigned long long *)ectx->h_pinned;
  CUDA_TRY(ectx, cudaMemcpyAsync(hc, g->d_ctr, gmerge::CTR_N * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ectx, cudaStreamSynchronize(ctx->stream));
  if (hc[gmerge::CTR_STATUS]) { ectx->err = "group accumulator table full"; return OBGPU_ERR_UNEXPECTED; }
  g->n = (int64_t)hc[gmerge::CTR_GROUPS];
  g->heap_used = (int64_t)hc[gmerge::CTR_HEAP];
  for (int c = 0; c < g->n_cols; ++c) g->col_bytes[c] = (int64_t)hc[gmerge::CTR_COL_BYTES + c];
  return OBGPU_SUCCESS;
}

int obgpu_groups_info(obgpu_groups *g, int64_t *n_groups, int64_t *key_bytes, int32_t *obj_types, int32_t *datum_lens) {
  if (!g) return OBGPU_INVALID_ARGUMENT;
  if (n_groups) *n_groups = g->n;
  if (key_bytes) *key_bytes = g->heap_used;
  for (int c = 0; c < g->n_cols; ++c) {
    const uint8_t t = (uint8_t)g->key_type[c];
    if (obj_types) obj_types[c] = g->key_type[c];
    if (datum_lens) datum_lens[c] = !g->typed ? -1 : (g->str_mask >> c) & 1u ? 0 : obf::datum_len_of(t);
  }
  return OBGPU_SUCCESS;
}

}  // extern "C"

namespace gmerge {

// the n groups of s in tuple order, as a new GroupBuf (*gv, allocated here on ctx's stream): a CUB merge sort of the group
// indices by TupleLess, the string lengths in that order scanned into offsets, then gather_kernel. col_bytes[c]: string column
// c's key bytes over the n groups. The accumulator's fetch and the hash fold over decoded cells (gcells) both end here.
static int sorted_groups(obgpu_ctx *ctx, const Store &s, int64_t n, const int32_t *kind, uint32_t sgn_key, uint32_t sgn_agg,
                         const int64_t *col_bytes, void **gv) {
  int64_t kb = 0;
  for (int c = 0; c < s.n_cols; ++c) kb += col_bytes[c];
  const gvals::GroupBuf lay(n, s.n_cols, s.n_aggs, kb);
  Scratch out(ctx);
  CUDA_TRY(ctx, out.alloc(lay.end));
  CUDA_TRY(ctx, cudaMemsetAsync(out.p, 0, lay.out, ctx->stream));   // no group: offsets {0}; integer columns' last slot 0
  if (n > 0) {
    size_t t_sort = 0, t_scan = 0;
    CUDA_TRY(ctx, cub::DeviceMergeSort::SortKeys(nullptr, t_sort, (uint32_t *)nullptr, n, TupleLess{s}, ctx->stream));
    if (s.str_mask) CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(nullptr, t_scan, (const int64_t *)nullptr, (int64_t *)nullptr, n, ctx->stream));
    // [order][string lengths, offsets: n_cols x n][sort temporaries][scan temporaries]
    Scratch tmp(ctx);
    const size_t o_order = tmp.take((size_t)n * 4), o_slen = tmp.take((size_t)s.n_cols * n * 8), o_soff = tmp.take((size_t)s.n_cols * n * 8);
    const size_t o_sort = tmp.take(t_sort), o_scan = tmp.take(t_scan);
    CUDA_TRY(ctx, tmp.alloc());
    uint32_t *order = tmp.at<uint32_t>(o_order);
    int64_t *slen = tmp.at<int64_t>(o_slen), *soff = tmp.at<int64_t>(o_soff);
    const unsigned grid = (unsigned)((n + kThreads - 1) / kThreads);
    gvals::iota_kernel<<<grid, kThreads, 0, ctx->stream>>>(order, (int)n);
    CUDA_TRY(ctx, cub::DeviceMergeSort::SortKeys(tmp.p + o_sort, t_sort, order, n, TupleLess{s}, ctx->stream));
    GatherArgs p{};
    if (s.str_mask) {
      sorted_lens_kernel<<<grid, kThreads, 0, ctx->stream>>>(s, order, n, slen);
      ctx->launches++;
      for (int c = 0; c < s.n_cols; ++c)
        if ((s.str_mask >> c) & 1u) CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(tmp.p + o_scan, t_scan, slen + c * n, soff + c * n, n, ctx->stream));
    }
    int64_t base = 0;
    for (int c = 0; c < s.n_cols; ++c) {   // each string column's bytes follow the previous one's
      p.base[c] = base;
      base += col_bytes[c];
    }
    p.s = s;
    p.order = order;
    p.n = n;
    for (int k = 0; k < s.n_aggs; ++k) p.kind[k] = kind[k];
    p.sgn_key = sgn_key;
    p.sgn_agg = sgn_agg;
    p.soff = soff;
    p.keys = out.at<int64_t>(0);
    p.out = out.at<int64_t>(lay.out);
    p.nulls = out.at<uint8_t>(lay.nulls);
    p.heap = out.at<uint8_t>(lay.heap);
    gather_kernel<<<grid, kThreads, 0, ctx->stream>>>(p);
    ctx->launches += 2;
    CUDA_TRY(ctx, cudaGetLastError());
  }
  *gv = out.release();
  return OBGPU_SUCCESS;
}

// obgpu_groups_fetch on the accumulator's own stream (errors and launches land in g->own)
static int fetch(obgpu_groups *g, int64_t *host_keys, uint8_t *host_key_nulls, void *host_key_heap, int64_t *host_out) {
  obgpu_ctx *ctx = &g->own;
  if (!g->d_gv)
    if (const int ret = sorted_groups(ctx, store_of(g, g->d_store, g->cap, g->d_heap), g->n, g->kind, g->sgn_key, g->sgn_agg, g->col_bytes,
                                      &g->d_gv);
        ret != OBGPU_SUCCESS)
      return ret;
  return gvals::copy_groups(ctx, (const uint8_t *)g->d_gv, g->n, g->n_cols, g->n_aggs, g->heap_used, host_keys, host_key_nulls, host_key_heap,
                            host_out);
}

}  // namespace gmerge

extern "C" {

int obgpu_groups_fetch(obgpu_groups *g, int64_t *host_keys, uint8_t *host_key_nulls, void *host_key_heap, int64_t *host_out) {
  if (!g || !host_keys || !host_key_nulls || !host_out || (g->heap_used > 0 && !host_key_heap)) return OBGPU_INVALID_ARGUMENT;
  cudaSetDevice(g->ctx->device);
  const int64_t launches0 = g->own.launches;
  const int ret = gmerge::fetch(g, host_keys, host_key_nulls, host_key_heap, host_out);
  g->ctx->launches += g->own.launches - launches0;
  if (ret != OBGPU_SUCCESS) g->ctx->err = g->own.err;
  return ret;
}

}  // extern "C"
