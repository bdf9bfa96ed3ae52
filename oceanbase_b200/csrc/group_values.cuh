// GROUP BY over a whole scan with one group per distinct VALUE of the group column across the page batch
// (obgpu_result_group_by_values), or per distinct TUPLE of values of 1..4 group columns (obgpu_result_group_by_columns).
// obgpu_result_group_by keeps the reference's granularity -- one group per (block, dictionary entry) -- and leaves the merge by
// value to the caller, which at millions of small blocks means millions of groups and calls. Here the merge happens on the device
// and only the groups cross PCIe.
// Per group column (column_stages; a column named twice is staged twice):
//   keys     one warp per block, lanes over the group column's dictionary entries read through the plans (dict_int + cmp_image,
//            dict_str): each entry goes into the batch codes' open-addressing table (bcodes::probe) -- one slot per distinct
//            value, whatever the block's entry width, base or format. A block whose plan is not dictionary coded sets a status bit.
//                                                            -- the host reads the distinct count: above 65 536, NOT_SUPPORTED --
//   number   bcodes::number_kernel: occupied slots -> codes 0..n_keys-1 (in no fixed order) and the code table
//   order    the codes sorted by key: integers by cub::DeviceRadixSort on the order-preserving 64-bit key (the MIN / MAX key:
//            sign bit flipped for signed and narrow classes), strings by cub::DeviceMergeSort comparing the image bytes as
//            unsigned bytes, a proper prefix first -> code_rank[code] = rank. Keys are distinct, so the order is unique.
// Over the selected rows:
//   id       a row's group is the mixed-radix number of its column ranks, column 0 most significant, radix G_c = n_keys_c + 1
//            with NULL as rank n_keys_c: ascending id is the lexicographic order of the tuples. P = prod G_c ids in all.
//   fold     a grid of CTAs, one warp per block at a time: each group column's dictionary entries -> ranks once (a per-warp
//            shared array per column; a dictionary larger than that probes per row), then the selected rows of the result's
//            bitmap words, folded per group. A hidden COUNT(*) (aggregate 0) marks the non-empty groups. Three paths, by P:
//              shared  P x (n_aggs + 1) x 16 B <= kSharedAccBudget: CTA-private shared accumulators indexed by id, flushed once
//                      per CTA with global atomics
//              global  P <= kDenseGroups: global accumulators indexed by id
//              hashed  otherwise: a first pass inserts every row's id into an open-addressing table of ids (id + 1, 0 empty)
//                      -- the host reads the distinct count: above kHashGroups, NOT_SUPPORTED -- the occupied slots are
//                      listed and sorted by id (cub::DeviceRadixSort), so group g is the g-th smallest id, and a second pass
//                      folds each row into global accumulators at probe -> slot -> group
//   compact  a prefix over the non-empty groups (and, per string column, their key lengths) -- the host reads the totals --
//            then one gather into the result's group buffer: per column the keys (the value's 64-bit image, or offsets + a key
//            heap whose bytes come from the batch's device image, the only copy of them for batches opened from stored or macro
//            blocks) and NULL flags, and the aggregates, MIN / MAX keys turned back into values.
#pragma once

#include <memory>

#include <cub/device/device_merge_sort.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace gvals {

constexpr int kWarpsPerCta = 8;
constexpr int kThreads = 32 * kWarpsPerCta;
constexpr int kMaxGroupCols = 4;
constexpr uint32_t kRankCap = 256;                // dictionary entries a warp maps to ranks in shared memory; larger: probe per row
constexpr size_t kRankBytes = (size_t)kWarpsPerCta * kRankCap * 4;   // a CTA's rank arrays of one group column
constexpr size_t kSharedAccBudget = 48u << 10;    // CTA-private accumulators, P x (n_aggs + 1) x 16 bytes, when they fit
constexpr size_t kMaxFoldSmem = kMaxGroupCols * kRankBytes + kSharedAccBudget;   // the most dynamic shared memory a fold launch takes
constexpr uint64_t kDenseGroups = 1ull << 20;     // the most ids the global path indexes directly; more: hashed
constexpr uint32_t kHashSlots = 1u << 23;         // the hashed path's id table (64 MiB)
constexpr uint32_t kHashGroups = 1u << 22;        // the most distinct ids the hashed path takes: the table at most half full
enum : int { ST_LONG_KEY = 8 };                   // a string entry of 65 536 bytes or more: no key (bcodes::key_of keeps 16 bits)
enum : int { ONE_INT, ONE_STR, MULTI };           // fold_kernel's group columns: one integer, one string, or 1..4 of any kind
enum : int { PATH_SHARED, PATH_GLOBAL, PATH_HASH_INSERT, PATH_HASH_FOLD };
// why group_by_columns refused with OBGPU_NOT_SUPPORTED: WHY_OTHER for the refusals every GROUP BY shares (class, aggregates);
// the others are limits of the dictionary fold that the hash fold over decoded cells (group_cells.cuh) does not have
enum : int { WHY_OTHER, WHY_NOT_DICT, WHY_VALUE_CAP, WHY_LONG_KEY, WHY_IMAGE, WHY_TUPLE_CAP };

// the order-preserving key of an integer value: its compare image, sign bit flipped for signed and narrow classes (the MIN / MAX key)
__device__ __forceinline__ uint64_t order_key(const ColDesc &d, uint64_t v) {
  const uint64_t img = (uint64_t)cmp_image(d, v);
  return (d.sc == 1 || d.elem_len < 8) ? img ^ (1ull << 63) : img;
}

// entry e of a dictionary-coded plan as the table keys it: (image offset, length) of a string, or the integer's order key
template <bool STR>
__device__ __forceinline__ void entry_key(const BlockView &bv, const ColDesc &d, uint64_t off, uint32_t e, uint64_t &abs, uint32_t &len,
                                          uint64_t &v) {
  if (STR) {
    uint32_t cell;
    dict_str(bv.s, d, e, cell, len);
    abs = off + cell;
  } else {
    v = order_key(d, dict_int(bv.s, d, e));
  }
}

template <bool STR>
__global__ void __launch_bounds__(kThreads) keys_kernel(dictops::BlkArgs a, int n, int col, unsigned long long *table, unsigned int *counters,
                                                        int *status) {
  const int b = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= n) return;
  BlockView bv;
  ColDesc d;
  if (!dictops::load_plan(a, b, col, bv, d) || (d.sc == 5) != STR) {
    if (lane == 0) atomicOr(status, ST_UNSUPPORTED);
    return;
  }
  const uint64_t off = a.recs[b].off;
  for (uint32_t e = (uint32_t)lane; e < d.dict_count; e += 32u) {
    if (*(volatile unsigned int *)&counters[0] > (unsigned int)bcodes::kMaxCodes) return;   // over the cap: refused
    uint64_t abs = 0, v = 0;
    uint32_t len = 0;
    entry_key<STR>(bv, d, off, e, abs, len, v);
    if (STR && len > 0xffffu) { atomicOr(status, ST_LONG_KEY); return; }
    if (bcodes::probe<STR>(a.image, table, abs, len, v, true, counters) == bcodes::kNoSlot) { atomicOr(&counters[1], 1u); return; }
  }
}

__global__ void iota_kernel(uint32_t *codes, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) codes[i] = (uint32_t)i;
}

__device__ __forceinline__ uint64_t bswap64(uint64_t x) {
  return ((uint64_t)__byte_perm((uint32_t)x, 0u, 0x0123) << 32) | __byte_perm((uint32_t)(x >> 32), 0u, 0x0123);
}

// string codes in key order: bytes compared as unsigned, 8 at a time big-endian; equal up to the shorter: the shorter first
struct StrLess {
  const uint8_t *image;
  const uint64_t *code_table;
  __device__ bool operator()(uint32_t x, uint32_t y) const {
    const uint64_t kx = code_table[x], ky = code_table[y];
    const uint64_t ax = bcodes::key_abs(kx), ay = bcodes::key_abs(ky);
    const uint32_t lx = bcodes::key_len(kx), ly = bcodes::key_len(ky), m = lx < ly ? lx : ly;
    for (uint32_t i = 0; i < m; i += 8u) {
      const uint32_t nb = m - i < 8u ? m - i : 8u;
      const uint64_t bx = bswap64(bcodes::img_bytes(image, ax, i, nb)), by = bswap64(bcodes::img_bytes(image, ay, i, nb));
      if (bx != by) return bx < by;
    }
    return lx < ly;
  }
};

__global__ void rank_kernel(const uint32_t *sorted_codes, const uint64_t *code_table, int n, uint32_t *code_rank, uint64_t *rank_key) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t c = sorted_codes[i];
  code_rank[c] = (uint32_t)i;
  rank_key[i] = code_table[c];
}

// the caller's 1..16 aggregates behind the hidden COUNT(*) of aggregate 0
struct FoldAggs {
  int32_t n;
  int32_t kind[17], col[17];
};

// one group column as the fold reads it: its value table (column_stages) and the rank of each slot's value
struct GroupCol {
  const unsigned long long *table;
  const uint16_t *slot_code;
  const uint32_t *code_rank;
  uint32_t n_keys;                     // rank n_keys: NULL
  int32_t col;
  bool str;
};

struct FoldArgs {
  dictops::BlkArgs a;
  int n_blocks, n_cols;
  FoldAggs aggs;
  const uint32_t *bitmap;              // nullptr: every row
  GroupCol gc[kMaxGroupCols];
  int64_t G;                           // accumulator groups: P (shared, global) or the distinct ids (hashed fold)
  unsigned long long *ids;             // hashed: the id table, id + 1 per occupied slot
  unsigned int *id_ctr;                // hashed: [ids inserted, table full]
  const uint32_t *slot_group;          // hashed fold: id slot -> group
  unsigned long long *acc;             // [aggs.n][G][2]
  int *status;
};

template <bool STR>
__device__ __forceinline__ uint32_t entry_rank(const FoldArgs &p, const GroupCol &q, const BlockView &bv, const ColDesc &d, uint64_t off,
                                               uint32_t e) {
  uint64_t abs = 0, v = 0;
  uint32_t len = 0;
  entry_key<STR>(bv, d, off, e, abs, len, v);
  const uint32_t slot = bcodes::probe<STR>(p.a.image, const_cast<unsigned long long *>(q.table), abs, len, v, false, nullptr);
  if (slot == bcodes::kNoSlot) { atomicOr(p.status, ST_CORRUPT); return q.n_keys; }
  return q.code_rank[q.slot_code[slot]];
}

template <int COLS>
__device__ __forceinline__ uint32_t col_rank(const FoldArgs &p, const GroupCol &q, const BlockView &bv, const ColDesc &d, uint64_t off,
                                             uint32_t e) {
  if (COLS == ONE_STR || (COLS == MULTI && q.str)) return entry_rank<true>(p, q, bv, d, off, e);
  return entry_rank<false>(p, q, bv, d, off, e);
}

// slot of composite id in the hashed path's table: found, or (insert) claimed; kNoSlot when absent (not inserting) or full
__device__ __forceinline__ uint32_t id_slot(unsigned long long *ids, uint64_t id, bool insert, unsigned int *ctr) {
  const unsigned long long key = id + 1ull;
  uint32_t slot = (uint32_t)bcodes::int_hash(id) & (kHashSlots - 1u);
  for (uint32_t k = 0; k < kHashSlots; ++k, slot = (slot + 1u) & (kHashSlots - 1u)) {
    unsigned long long cur = *(volatile unsigned long long *)&ids[slot];
    if (cur == 0ull) {
      if (!insert) return bcodes::kNoSlot;
      cur = atomicCAS(&ids[slot], 0ull, key);
      if (cur == 0ull) {
        atomicAdd(&ctr[0], 1u);
        return slot;
      }
    }
    if (cur == key) return slot;
  }
  return bcodes::kNoSlot;
}

// PATH_SHARED: fold into CTA-private accumulators (dynamic shared memory past the warps' rank arrays), flushed at the end.
// PATH_HASH_INSERT only inserts the selected rows' ids; PATH_HASH_FOLD finds each row's group through them.
template <int COLS, int PATH>
__global__ void __maxnreg__(96) fold_kernel(const __grid_constant__ FoldArgs p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nc = COLS == MULTI ? p.n_cols : 1;
  uint32_t *ranks = (uint32_t *)g_smem + warp * kRankCap;   // group column c's: at + c * kWarpsPerCta * kRankCap
  const int64_t G = p.G, n_acc = (int64_t)p.aggs.n * G;
  unsigned long long *acc = p.acc;
  if (PATH == PATH_SHARED) {
    acc = (unsigned long long *)(g_smem + nc * kRankBytes);
    for (int64_t i = threadIdx.x; i < n_acc; i += blockDim.x) {
      acc[2 * i] = p.aggs.kind[i / G] == OBGPU_AGG_MIN ? ~0ull : 0ull;
      acc[2 * i + 1] = 0ull;
    }
    __syncthreads();
  }
  for (int b = blockIdx.x * kWarpsPerCta + warp; b < p.n_blocks; b += gridDim.x * kWarpsPerCta) {
    BlockView bv;
    ColDesc gd;
    const BlockRec rec = p.a.recs[b];
    bool ok = true;
    for (int c = 0; c < nc && ok; ++c) {
      const GroupCol &q = p.gc[c];
      ok = dictops::load_plan(p.a, b, q.col, bv, gd);
      if (ok && gd.dict_count <= kRankCap)
        for (uint32_t e = (uint32_t)lane; e < gd.dict_count; e += 32u) ranks[c * (kWarpsPerCta * kRankCap) + e] = col_rank<COLS>(p, q, bv, gd, rec.off, e);
    }
    if (!ok) { if (lane == 0) atomicOr(p.status, ST_UNSUPPORTED); continue; }
    const bool in_smem = gd.dict_count <= kRankCap;
    __syncwarp();
    for (uint32_t r0 = 0; r0 < bv.row_count; r0 += 32u) {
      const uint32_t r = r0 + (uint32_t)lane;
      bool sel = r < bv.row_count;
      if (p.bitmap) sel = sel && ((p.bitmap[rec.bm_word_off + (r0 >> 5)] >> lane) & 1u);
      if (PATH == PATH_HASH_INSERT) sel = sel && *(volatile unsigned int *)&p.id_ctr[0] <= kHashGroups;   // over the cap: refused
      if (!sel) continue;
      uint64_t id;
      if (COLS != MULTI) {
        const uint32_t ref = ref_of(bv.s, gd, nullptr, r);
        id = ref >= gd.dict_count ? p.gc[0].n_keys : in_smem ? ranks[ref] : col_rank<COLS>(p, p.gc[0], bv, gd, rec.off, ref);
      } else {
        id = 0;
        for (int c = 0; c < nc; ++c) {
          const GroupCol &q = p.gc[c];
          const ColDesc d = p.a.plans[(int64_t)b * p.a.max_cols + q.col];
          const uint32_t ref = ref_of(bv.s, d, nullptr, r);
          const uint32_t rk = ref >= d.dict_count             ? q.n_keys
                              : d.dict_count <= kRankCap      ? ranks[c * (kWarpsPerCta * kRankCap) + ref]
                                                              : col_rank<COLS>(p, q, bv, d, rec.off, ref);
          id = id * ((uint64_t)q.n_keys + 1ull) + rk;
        }
      }
      if (PATH == PATH_HASH_INSERT) {
        if (id_slot(p.ids, id, true, p.id_ctr) == bcodes::kNoSlot) atomicOr(&p.id_ctr[1], 1u);
        continue;
      }
      int64_t g = (int64_t)id;
      if (PATH == PATH_HASH_FOLD) {
        const uint32_t s = id_slot(p.ids, id, false, nullptr);
        if (s == bcodes::kNoSlot) { atomicOr(p.status, ST_CORRUPT); continue; }
        g = p.slot_group[s];
      }
      for (int k = 0; k < p.aggs.n; ++k) {
        unsigned long long *c = acc + ((int64_t)k * G + g) * 2;
        if (p.aggs.col[k] < 0) { atomicAdd(&c[0], 1ull); continue; }   // COUNT(*), the hidden one included
        const ColDesc d = p.a.plans[(int64_t)b * p.a.max_cols + p.aggs.col[k]];
        if (!d.ok || d.sc == 5) { atomicOr(p.status, ST_UNSUPPORTED); continue; }
        bool is_null;
        const uint64_t v = int_cell(bv, d, nullptr, r, is_null);
        if (is_null) continue;
        dictops::accumulate(c, p.aggs.kind[k], (long long)cmp_image(d, v), d.sc == 1 || d.elem_len < 8);
      }
    }
    __syncwarp();   // the next block's ranks overwrite these
  }
  if (PATH != PATH_SHARED) return;
  __syncthreads();
  for (int64_t i = threadIdx.x; i < n_acc; i += blockDim.x) {
    const int kind = p.aggs.kind[i / G];
    const unsigned long long lo = acc[2 * i], hi = acc[2 * i + 1];
    unsigned long long *o = p.acc + 2 * i;
    if (kind == OBGPU_AGG_MIN || kind == OBGPU_AGG_MAX) {
      if (!hi) continue;
      if (kind == OBGPU_AGG_MIN) atomicMin(&o[0], lo); else atomicMax(&o[0], lo);
      atomicOr(&o[1], 1ull);
      continue;
    }
    if (!(lo | hi)) continue;
    const unsigned long long old = atomicAdd(&o[0], lo), carry = old + lo < old ? 1ull : 0ull;
    if (hi + carry) atomicAdd(&o[1], hi + carry);   // 128-bit add: low word's carry into the high word
  }
}

// the hashed path's occupied id slots, listed in no fixed order ([0]: how many)
__global__ void id_list_kernel(const unsigned long long *ids, unsigned int *ctr, uint64_t *list_id, uint32_t *list_slot) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= kHashSlots || ids[s] == 0ull) return;
  const uint32_t i = atomicAdd(ctr, 1u);
  list_id[i] = ids[s] - 1ull;
  list_slot[i] = s;
}

// sorted by id: slot -> group
__global__ void id_group_kernel(const uint32_t *sorted_slot, int64_t n, uint32_t *slot_group) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) slot_group[sorted_slot[i]] = (uint32_t)i;
}

// one group column as the compaction reads it
struct KeyCol {
  const uint64_t *rank_key;            // rank -> the value's key (the order key, or a string's image offset and length)
  uint64_t radix;                      // n_keys + 1
  int64_t base;                        // strings: heap offset of the column's first byte
  bool str, sgn_key;
};

struct Groups {
  int n_cols;
  KeyCol kc[kMaxGroupCols];
  const uint64_t *group_id;            // hashed: group -> id; dense: nullptr, the id is the group
};

// group g's rank in each column
__device__ __forceinline__ void ranks_of(const Groups &k, int64_t g, uint64_t (&r)[kMaxGroupCols]) {
  uint64_t id = k.group_id ? k.group_id[g] : (uint64_t)g;
#pragma unroll
  for (int c = kMaxGroupCols - 1; c >= 0; --c) {
    if (c >= k.n_cols) continue;
    r[c] = id % k.kc[c].radix;
    id /= k.kc[c].radix;
  }
}

// group g is kept when its hidden COUNT(*) is not zero; lens[c][g] its key bytes in string column c
__global__ void flags_kernel(const unsigned long long *acc, int64_t G, const __grid_constant__ Groups k, int32_t *flags, int64_t *lens) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const bool keep = acc[2 * g] != 0ull;
  flags[g] = keep ? 1 : 0;
  uint64_t r[kMaxGroupCols];
  ranks_of(k, g, r);
#pragma unroll
  for (int c = 0; c < kMaxGroupCols; ++c)
    if (c < k.n_cols && k.kc[c].str)
      lens[c * G + g] = keep && r[c] + 1 < k.kc[c].radix ? (int64_t)bcodes::key_len(k.kc[c].rank_key[r[c]]) : 0;
}

// [n_groups, has NULL group (one column), key bytes of string column c at 2 + c]
__global__ void totals_kernel(const int32_t *flags, const int32_t *pos, const int64_t *lens, const int64_t *koff, int64_t G, uint32_t str_mask,
                              int64_t *tot) {
  tot[0] = (int64_t)pos[G - 1] + flags[G - 1];
  tot[1] = flags[G - 1];
  for (int c = 0; c < kMaxGroupCols; ++c) tot[2 + c] = (str_mask >> c) & 1u ? koff[c * G + G - 1] + lens[c * G + G - 1] : 0;
}

struct GatherArgs {
  const unsigned long long *acc;
  int64_t G, n_groups;
  int n_aggs;
  int32_t kind[16];
  uint32_t sgn_agg;         // bit k: MIN / MAX key of aggregate k has its sign bit flipped
  Groups k;
  const int32_t *flags, *pos;
  const int64_t *lens, *koff;   // [n_cols][G]
  const uint8_t *image;
  int64_t *keys;            // [n_cols][n_groups + 1]: integers' images, or strings' heap offsets
  uint8_t *nulls;           // [n_cols][n_groups]
  uint8_t *heap;
  int64_t *out;             // [n_aggs][n_groups][2]
};

__global__ void gather_kernel(const __grid_constant__ GatherArgs p) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= p.G || !p.flags[g]) return;
  const int64_t q = p.pos[g];
  uint64_t r[kMaxGroupCols];
  ranks_of(p.k, g, r);
#pragma unroll
  for (int c = 0; c < kMaxGroupCols; ++c) {
    if (c >= p.k.n_cols) continue;
    const KeyCol &kc = p.k.kc[c];
    int64_t *keys = p.keys + c * (p.n_groups + 1);
    const bool null_key = r[c] + 1 == kc.radix;
    p.nulls[c * p.n_groups + q] = null_key ? 1 : 0;
    if (kc.str) {
      const int64_t o = kc.base + p.koff[c * p.G + g], len = p.lens[c * p.G + g];
      keys[q] = o;
      if (q + 1 == p.n_groups) keys[q + 1] = o + len;
      if (!null_key) {
        const uint64_t abs = bcodes::key_abs(kc.rank_key[r[c]]);
        for (int64_t i = 0; i < len; ++i) p.heap[o + i] = p.image[abs + i];
      }
    } else if (null_key) {
      keys[q] = 0;
    } else {
      const uint64_t key = kc.rank_key[r[c]];
      keys[q] = (int64_t)(kc.sgn_key ? key ^ (1ull << 63) : key);
    }
  }
  for (int k = 0; k < p.n_aggs; ++k) {
    const unsigned long long *a = p.acc + ((int64_t)(k + 1) * p.G + g) * 2;
    int64_t *o = p.out + ((int64_t)k * p.n_groups + q) * 2;
    uint64_t lo = a[0], hi = a[1];
    if (p.kind[k] == OBGPU_AGG_MIN || p.kind[k] == OBGPU_AGG_MAX) {
      if (!hi) lo = 0;
      else if ((p.sgn_agg >> k) & 1u) lo ^= 1ull << 63;
    }
    o[0] = (int64_t)lo;
    o[1] = (int64_t)hi;
  }
}

using FoldFn = void (*)(const FoldArgs);

template <int COLS>
FoldFn fold_fn(int path) {
  if constexpr (COLS == MULTI) {
    if (path == PATH_HASH_INSERT) return fold_kernel<MULTI, PATH_HASH_INSERT>;
    if (path == PATH_HASH_FOLD) return fold_kernel<MULTI, PATH_HASH_FOLD>;
  }
  return path == PATH_SHARED ? fold_kernel<COLS, PATH_SHARED> : fold_kernel<COLS, PATH_GLOBAL>;
}

// one group column's keys -> number -> order, in scratch of its own
struct ColStage {
  Scratch mem;
  GroupCol dev{};
  const uint64_t *rank_key = nullptr;
  bool sgn_key = false;
  explicit ColStage(obgpu_ctx *c) : mem(c) {}
};

// the order key of a group column of obj_type t has its sign bit flipped (gvals::order_key)
static bool key_sgn(uint8_t t) { return obf::store_class_of(t) == 1 || obf::datum_len_of(t) < 8; }

static int column_stages(obgpu_ctx *ctx, obgpu_batch *b, int32_t col, ColStage &cs, int *why) {
  const uint8_t gt = b->col_types[(size_t)col];
  const int gsc = gt == 0xff ? 0 : obf::store_class_of(gt);
  if (gsc != 1 && gsc != 2 && gsc != 5) { ctx->err = "group-by column is not an integer or string column in every micro block"; return OBGPU_NOT_SUPPORTED; }
  const bool str = gsc == 5;
  if (str && b->image_size >= (int64_t)1 << 37) {
    *why = WHY_IMAGE;
    ctx->err = "string group keys address images below 2^37 bytes";
    return OBGPU_NOT_SUPPORTED;
  }
  const int n = b->n_blocks;
  size_t t_sort = 0;   // cub's temporaries, sized for the most keys
  if (str)
    CUDA_TRY(ctx, cub::DeviceMergeSort::SortKeys(nullptr, t_sort, (uint32_t *)nullptr, (int64_t)bcodes::kMaxCodes, StrLess{}, ctx->stream));
  else
    CUDA_TRY(ctx, cub::DeviceRadixSort::SortPairs(nullptr, t_sort, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const uint32_t *)nullptr,
                                                  (uint32_t *)nullptr, bcodes::kMaxCodes, 0, 64, ctx->stream));
  // [status][counters][table][slot -> code][code table][codes, sorted codes][sorted keys][code -> rank][rank -> key][sort temporaries]
  Scratch &tmp = cs.mem;
  const size_t o_status = tmp.take(64), o_ctr = tmp.take(32);
  const size_t o_table = tmp.take((size_t)bcodes::kTableSlots * 8), o_slot = tmp.take((size_t)bcodes::kTableSlots * 2 + 16);
  const size_t o_ctab = tmp.take((size_t)bcodes::kMaxCodes * 8), o_codes = tmp.take((size_t)bcodes::kMaxCodes * 4);
  const size_t o_scodes = tmp.take((size_t)bcodes::kMaxCodes * 4), o_skeys = tmp.take((size_t)bcodes::kMaxCodes * 8);
  const size_t o_rank = tmp.take((size_t)bcodes::kMaxCodes * 4), o_rkey = tmp.take((size_t)bcodes::kMaxCodes * 8);
  const size_t o_sort = tmp.take(t_sort);
  CUDA_TRY(ctx, tmp.alloc());
  int *d_status = tmp.at<int>(o_status);
  unsigned int *ctr = tmp.at<unsigned int>(o_ctr);   // [entries inserted, table full, codes numbered, integer 2^64 - 1 seen]
  unsigned long long *table = tmp.at<unsigned long long>(o_table);
  uint64_t *code_table = tmp.at<uint64_t>(o_ctab);
  CUDA_TRY(ctx, cudaMemsetAsync(tmp.p, 0, o_slot, ctx->stream));   // status, counters, table
  const dictops::BlkArgs a{b->d_image, b->d_recs, b->d_plans, (int32_t)b->max_cols};
  if (n > 0) {
    const unsigned key_grid = (unsigned)((n + kWarpsPerCta - 1) / kWarpsPerCta);
    (str ? keys_kernel<true> : keys_kernel<false>)<<<key_grid, kThreads, 0, ctx->stream>>>(a, n, col, table, ctr, d_status);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
  }
  int32_t *hs = (int32_t *)ctx->h_pinned;
  CUDA_TRY(ctx, cudaMemcpyAsync(hs, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(hs + 1, ctr, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (hs[0] & ST_UNSUPPORTED) {
    *why = WHY_NOT_DICT;
    ctx->err = "group-by column is not dictionary coded in every micro block";
    return OBGPU_NOT_SUPPORTED;
  }
  if (hs[0] & ST_LONG_KEY) { *why = WHY_LONG_KEY; ctx->err = "group-by string of 65536 bytes or more"; return OBGPU_NOT_SUPPORTED; }
  if (hs[0]) return check_status(ctx, hs[0]);
  if (hs[2] || (uint32_t)hs[1] > (uint32_t)bcodes::kMaxCodes) {
    *why = WHY_VALUE_CAP;
    ctx->err = "more than 65536 distinct group-by values in the batch";
    return OBGPU_NOT_SUPPORTED;
  }
  const int n_keys = hs[1];
  uint32_t *code_rank = tmp.at<uint32_t>(o_rank);
  uint64_t *rank_key = tmp.at<uint64_t>(o_rkey);
  if (n_keys > 0) {
    uint32_t *codes = tmp.at<uint32_t>(o_codes), *sorted = tmp.at<uint32_t>(o_scodes);
    bcodes::number_kernel<<<bcodes::kTableSlots / 256 + 1, 256, 0, ctx->stream>>>(table, str, ctr, tmp.at<uint16_t>(o_slot), code_table);
    iota_kernel<<<(n_keys + 255) / 256, 256, 0, ctx->stream>>>(codes, n_keys);
    ctx->launches += 2;
    if (str) {
      CUDA_TRY(ctx, cudaMemcpyAsync(sorted, codes, (size_t)n_keys * 4, cudaMemcpyDeviceToDevice, ctx->stream));
      CUDA_TRY(ctx, cub::DeviceMergeSort::SortKeys(tmp.p + o_sort, t_sort, sorted, (int64_t)n_keys, StrLess{b->d_image, code_table}, ctx->stream));
    } else {
      CUDA_TRY(ctx, cub::DeviceRadixSort::SortPairs(tmp.p + o_sort, t_sort, (const uint64_t *)code_table, tmp.at<uint64_t>(o_skeys),
                                                    (const uint32_t *)codes, sorted, n_keys, 0, 64, ctx->stream));
    }
    rank_kernel<<<(n_keys + 255) / 256, 256, 0, ctx->stream>>>(sorted, code_table, n_keys, code_rank, rank_key);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
  }
  cs.dev = GroupCol{table, tmp.at<uint16_t>(o_slot), code_rank, (uint32_t)n_keys, col, str};
  cs.rank_key = rank_key;
  cs.sgn_key = key_sgn(gt);
  return OBGPU_SUCCESS;
}

// byte offsets in the result's group buffer: [keys: n_cols x (n_groups + 1)][aggregates][NULL flags: n_cols x n_groups][key heap]
struct GroupBuf {
  size_t out, nulls, heap, end;
  GroupBuf(int64_t ng, int n_cols, int n_aggs, int64_t key_bytes) {
    out = (size_t)n_cols * ((size_t)ng + 1) * 8;
    nulls = out + (size_t)n_aggs * (size_t)ng * 16;
    heap = nulls + (((size_t)n_cols * (size_t)ng + 15) & ~(size_t)15);
    end = heap + (size_t)key_bytes + 16;
  }
};

// the result's group slot <- groups in the GroupBuf layout at gv (the slot takes gv over)
static void set_groups(obgpu_result *r, void *gv, int64_t ng, int64_t kb, const int32_t *cols, int n_cols, const obgpu_group_agg *aggs,
                       int n_aggs, uint32_t str_mask, uint32_t sgn_agg) {
  const obgpu_batch *b = r->batch;
  r->d_gv = gv;
  r->gv_groups = ng;
  r->gv_key_bytes = kb;
  r->gv_n_aggs = n_aggs;
  r->gv_n_cols = n_cols;
  r->gv_str_mask = str_mask;
  for (int k = 0; k < n_aggs; ++k) {
    r->gv_kind[k] = aggs[k].kind;
    r->gv_agg_col[k] = aggs[k].col;
    r->gv_agg_type[k] = aggs[k].col >= 0 ? b->col_types[(size_t)aggs[k].col] : -1;
  }
  r->gv_sgn_key = 0;
  for (int c = 0; c < n_cols; ++c) {
    r->gv_key_type[c] = b->col_types[(size_t)cols[c]];
    if (key_sgn((uint8_t)r->gv_key_type[c])) r->gv_sgn_key |= 1u << c;
  }
  r->gv_sgn_agg = sgn_agg;
}

// the aggregates every GROUP BY folds: COUNT / SUM / MIN / MAX over integer-class columns or COUNT(*); *sgn_agg: bit k when
// aggregate k's MIN / MAX key has its sign bit flipped
static int check_aggs(obgpu_ctx *ctx, const obgpu_batch *b, const obgpu_group_agg *aggs, int32_t n_aggs, uint32_t *sgn_agg) {
  *sgn_agg = 0;
  for (int k = 0; k < n_aggs; ++k) {
    if (aggs[k].kind < OBGPU_AGG_COUNT || aggs[k].kind > OBGPU_AGG_MAX || aggs[k].kind == OBGPU_AGG_SUM_PRODUCT) return OBGPU_NOT_SUPPORTED;
    if (aggs[k].col >= (int32_t)b->max_cols || (aggs[k].col < 0 && aggs[k].kind != OBGPU_AGG_COUNT)) return OBGPU_INVALID_ARGUMENT;
    if (aggs[k].col >= 0) {
      const uint8_t t = b->col_types[(size_t)aggs[k].col];
      const int sc = t == 0xff ? 0 : obf::store_class_of(t);
      if (sc != 1 && sc != 2) { ctx->err = "aggregates fold integer-class columns only"; return OBGPU_NOT_SUPPORTED; }
      if (obf::store_class_of(t) == 1 || obf::datum_len_of(t) < 8) *sgn_agg |= 1u << k;
    }
  }
  return OBGPU_SUCCESS;
}

// the scan's own status first, then the previous call's groups dropped: a refused call leaves none
static int begin_groups(obgpu_result *r) {
  if (!r) return OBGPU_INVALID_ARGUMENT;
  obgpu_result_info info;
  const int ret = obgpu_result_info_get(r, &info);
  if (ret != OBGPU_SUCCESS && ret != OBGPU_BUF_NOT_ENOUGH) return ret;
  cudaSetDevice(r->ctx->device);
  if (r->d_gv) cudaFreeAsync(r->d_gv, r->ctx->stream);
  r->d_gv = nullptr;
  r->gv_groups = -1;
  return OBGPU_SUCCESS;
}

// GROUP BY the tuple of cols[0..n_cols) (arguments checked by the caller but the aggregates); *has_null: the last group's first
// key is NULL; *why: the reason of an OBGPU_NOT_SUPPORTED (WHY_*)
static int group_by_columns(obgpu_result *r, const int32_t *cols, int n_cols, const obgpu_group_agg *aggs, int32_t n_aggs, int64_t *n_groups,
                            int64_t *key_bytes, int32_t *has_null, int *why) {
  *why = WHY_OTHER;
  obgpu_batch *b = r->batch;
  obgpu_ctx *ctx = r->ctx;
  FoldAggs ga{};
  ga.n = n_aggs + 1;
  ga.kind[0] = OBGPU_AGG_COUNT;
  ga.col[0] = -1;
  GatherArgs gp{};
  gp.n_aggs = n_aggs;
  if (const int ret = check_aggs(ctx, b, aggs, n_aggs, &gp.sgn_agg); ret != OBGPU_SUCCESS) return ret;
  for (int k = 0; k < n_aggs; ++k) {
    ga.kind[k + 1] = gp.kind[k] = aggs[k].kind;
    ga.col[k + 1] = aggs[k].col;
  }
  std::unique_ptr<ColStage> st[kMaxGroupCols];
  FoldArgs fp{};
  unsigned __int128 P = 1;   // composite ids
  uint32_t str_mask = 0;
  for (int c = 0; c < n_cols; ++c) {
    st[c] = std::make_unique<ColStage>(ctx);
    if (const int ret = column_stages(ctx, b, cols[c], *st[c], why); ret != OBGPU_SUCCESS) return ret;
    fp.gc[c] = st[c]->dev;
    gp.k.kc[c] = KeyCol{st[c]->rank_key, (uint64_t)st[c]->dev.n_keys + 1, 0, st[c]->dev.str, st[c]->sgn_key};
    if (st[c]->dev.str) str_mask |= 1u << c;
    P *= (uint64_t)st[c]->dev.n_keys + 1;
    if (P >= (unsigned __int128)~0ull) { *why = WHY_TUPLE_CAP; ctx->err = "2^64 - 1 or more composite group ids"; return OBGPU_NOT_SUPPORTED; }
  }
  gp.k.n_cols = n_cols;
  const int path = (uint64_t)P <= kDenseGroups && (uint64_t)P * (uint64_t)ga.n * 16 <= kSharedAccBudget ? PATH_SHARED
                   : (uint64_t)P <= kDenseGroups                                                           ? PATH_GLOBAL
                                                                                                           : PATH_HASH_FOLD;
  const int n = b->n_blocks;
  const unsigned key_grid = (unsigned)((n + kWarpsPerCta - 1) / kWarpsPerCta);
  fp.a = dictops::BlkArgs{b->d_image, b->d_recs, b->d_plans, (int32_t)b->max_cols};
  fp.n_blocks = n;
  fp.n_cols = n_cols;
  fp.aggs = ga;
  fp.bitmap = r->no_filter ? nullptr : r->d_bitmap;
  const size_t rank_smem = (size_t)n_cols * kRankBytes;
  const auto launch = [&](int pth, size_t acc_smem) -> int {
    const FoldFn fold = n_cols > 1 ? fold_fn<MULTI>(pth) : fp.gc[0].str ? fold_fn<ONE_STR>(pth) : fold_fn<ONE_INT>(pth);
    const size_t smem = rank_smem + acc_smem;
    // the attribute is the kernel's, shared by every ctx and thread of the process: always the one largest value any launch
    // needs, so that concurrent calls (one per pipeline worker) never lower it under another's launch
    CUDA_TRY(ctx, cudaFuncSetAttribute(fold, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxFoldSmem));
    unsigned grid = key_grid;
    if (pth == PATH_SHARED) {   // few CTAs, each folding many blocks: one flush per resident CTA
      int per_sm = 0;
      CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fold, kThreads, smem));
      grid = std::min(grid, (unsigned)std::max(per_sm, 1) * (unsigned)ctx->sm_count);
    }
    fold<<<grid, kThreads, smem, ctx->stream>>>(fp);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return OBGPU_SUCCESS;
  };
  // [status][hashed: id counters, id table, slot -> group]
  Scratch fm(ctx);
  const size_t o_status = fm.take(64), o_idctr = fm.take(64);
  const size_t o_ids = path == PATH_HASH_FOLD ? fm.take((size_t)kHashSlots * 8) : 0;
  const size_t o_sgroup = path == PATH_HASH_FOLD ? fm.take((size_t)kHashSlots * 4) : 0;
  CUDA_TRY(ctx, fm.alloc());
  int *d_status = fm.at<int>(o_status);
  fp.status = d_status;
  CUDA_TRY(ctx, cudaMemsetAsync(fm.p, 0, path == PATH_HASH_FOLD ? o_sgroup : fm.bytes, ctx->stream));   // status, counters, id table
  int64_t G = (int64_t)(uint64_t)P;
  Scratch hs(ctx);   // hashed: [listed ids, sorted][listed slots, sorted][sort temporaries]
  uint64_t *group_id = nullptr;
  if (path == PATH_HASH_FOLD) {
    unsigned int *id_ctr = fm.at<unsigned int>(o_idctr);   // [ids inserted, table full, ids listed]
    fp.ids = fm.at<unsigned long long>(o_ids);
    fp.id_ctr = id_ctr;
    fp.slot_group = fm.at<uint32_t>(o_sgroup);
    if (n > 0)
      if (const int ret = launch(PATH_HASH_INSERT, 0); ret != OBGPU_SUCCESS) return ret;
    uint32_t *hc = (uint32_t *)ctx->h_pinned;
    CUDA_TRY(ctx, cudaMemcpyAsync(hc, id_ctr, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(hc + 2, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    if (hc[2]) return check_status(ctx, (int)hc[2]);
    if (hc[1] || hc[0] > kHashGroups) {
      *why = WHY_TUPLE_CAP;
      ctx->err = "more than 4194304 distinct group-by tuples in the selected rows";
      return OBGPU_NOT_SUPPORTED;
    }
    G = hc[0];
    if (G > 0) {
      int end_bit = 0;
      while (end_bit < 64 && ((uint64_t)P - 1) >> end_bit) ++end_bit;
      size_t t_sort = 0;
      CUDA_TRY(ctx, cub::DeviceRadixSort::SortPairs(nullptr, t_sort, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const uint32_t *)nullptr,
                                                    (uint32_t *)nullptr, G, 0, end_bit, ctx->stream));
      const size_t o_lid = hs.take((size_t)G * 8), o_sid = hs.take((size_t)G * 8), o_lslot = hs.take((size_t)G * 4);
      const size_t o_sslot = hs.take((size_t)G * 4), o_sort = hs.take(t_sort);
      CUDA_TRY(ctx, hs.alloc());
      id_list_kernel<<<kHashSlots / 256, 256, 0, ctx->stream>>>(fp.ids, id_ctr + 2, hs.at<uint64_t>(o_lid), hs.at<uint32_t>(o_lslot));
      CUDA_TRY(ctx, cub::DeviceRadixSort::SortPairs(hs.p + o_sort, t_sort, hs.at<const uint64_t>(o_lid), hs.at<uint64_t>(o_sid),
                                                    hs.at<const uint32_t>(o_lslot), hs.at<uint32_t>(o_sslot), G, 0, end_bit, ctx->stream));
      id_group_kernel<<<(unsigned)((G + 255) / 256), 256, 0, ctx->stream>>>(hs.at<const uint32_t>(o_sslot), G, const_cast<uint32_t *>(fp.slot_group));
      ctx->launches += 2;
      CUDA_TRY(ctx, cudaGetLastError());
      group_id = hs.at<uint64_t>(o_sid);
    }
  }
  gp.k.group_id = group_id;
  fp.G = G;
  int64_t ng = 0, kb = 0, col_bytes[kMaxGroupCols] = {0};
  int32_t null_last = 0;
  Scratch accm(ctx), cm(ctx);
  if (G > 0) {
    // accumulators [n_aggs + 1][G][2], MIN from the largest key
    const size_t acc_bytes = (size_t)ga.n * (size_t)G * 16;
    CUDA_TRY(ctx, accm.alloc(acc_bytes));
    unsigned long long *acc = accm.at<unsigned long long>(0);
    CUDA_TRY(ctx, cudaMemsetAsync(acc, 0, acc_bytes, ctx->stream));
    for (int k = 1; k < ga.n; ++k)
      if (ga.kind[k] == OBGPU_AGG_MIN) CUDA_TRY(ctx, cudaMemset2DAsync(acc + (size_t)k * G * 2, 16, 0xff, 8, (size_t)G, ctx->stream));
    fp.acc = acc;
    if (n > 0)
      if (const int ret = launch(path, path == PATH_SHARED ? acc_bytes : 0); ret != OBGPU_SUCCESS) return ret;
    // [totals][flags, positions][lengths, offsets: n_cols x G][scan temporaries]
    size_t t_scan = 0, t_scan64 = 0;
    CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(nullptr, t_scan, (const int32_t *)nullptr, (int32_t *)nullptr, G, ctx->stream));
    if (str_mask) CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(nullptr, t_scan64, (const int64_t *)nullptr, (int64_t *)nullptr, G, ctx->stream));
    const size_t o_tot = cm.take(64), o_flags = cm.take((size_t)G * 4), o_pos = cm.take((size_t)G * 4);
    const size_t o_lens = cm.take((size_t)n_cols * G * 8), o_koff = cm.take((size_t)n_cols * G * 8);
    const size_t o_scan = cm.take(t_scan), o_scan64 = cm.take(t_scan64);
    CUDA_TRY(ctx, cm.alloc());
    int32_t *flags = cm.at<int32_t>(o_flags), *pos = cm.at<int32_t>(o_pos);
    int64_t *lens = cm.at<int64_t>(o_lens), *koff = cm.at<int64_t>(o_koff), *tot = cm.at<int64_t>(o_tot);
    flags_kernel<<<(unsigned)((G + 255) / 256), 256, 0, ctx->stream>>>(acc, G, gp.k, flags, lens);
    CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(cm.p + o_scan, t_scan, flags, pos, G, ctx->stream));
    for (int c = 0; c < n_cols; ++c)
      if ((str_mask >> c) & 1u)
        CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(cm.p + o_scan64, t_scan64, lens + (size_t)c * G, koff + (size_t)c * G, G, ctx->stream));
    totals_kernel<<<1, 1, 0, ctx->stream>>>(flags, pos, lens, koff, G, str_mask, tot);
    ctx->launches += 2;
    CUDA_TRY(ctx, cudaGetLastError());
    int64_t *ht = (int64_t *)ctx->h_pinned;
    CUDA_TRY(ctx, cudaMemcpyAsync(ht, tot, 48, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(ht + 6, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    if (const int32_t s = (int32_t)ht[6]) return check_status(ctx, s);
    ng = ht[0];
    null_last = (int32_t)ht[1];
    for (int c = 0; c < n_cols; ++c) {
      col_bytes[c] = ht[2 + c];
      gp.k.kc[c].base = kb;   // each string column's bytes follow the previous one's
      kb += col_bytes[c];
    }
    gp.flags = flags;
    gp.pos = pos;
    gp.lens = lens;
    gp.koff = koff;
  }
  // the result's groups (GroupBuf)
  const GroupBuf lay(ng, n_cols, n_aggs, kb);
  void *gv = nullptr;
  CUDA_TRY(ctx, cudaMallocAsync(&gv, lay.end, ctx->stream));
  if (const cudaError_t e = cudaMemsetAsync(gv, 0, lay.out, ctx->stream); e != cudaSuccess) {   // no group: offsets {0}
    cudaFreeAsync(gv, ctx->stream);
    ctx->err = std::string("cudaMemsetAsync: ") + cudaGetErrorString(e);
    return OBGPU_ERR_SYS;
  }
  if (G > 0) {
    gp.acc = fp.acc;
    gp.G = G;
    gp.n_groups = ng;
    gp.image = b->d_image;
    gp.keys = (int64_t *)gv;
    gp.out = (int64_t *)((uint8_t *)gv + lay.out);
    gp.nulls = (uint8_t *)gv + lay.nulls;
    gp.heap = (uint8_t *)gv + lay.heap;
    gather_kernel<<<(unsigned)((G + 255) / 256), 256, 0, ctx->stream>>>(gp);
    ctx->launches++;
    if (const cudaError_t e = cudaGetLastError(); e != cudaSuccess) {
      cudaFreeAsync(gv, ctx->stream);
      ctx->err = std::string("gather_kernel: ") + cudaGetErrorString(e);
      return OBGPU_ERR_SYS;
    }
  }
  set_groups(r, gv, ng, kb, cols, n_cols, aggs, n_aggs, str_mask, gp.sgn_agg);
  *n_groups = ng;
  *key_bytes = kb;
  if (has_null) *has_null = null_last;
  return OBGPU_SUCCESS;
}

// groups in the GroupBuf layout at gv -> the host layout of obgpu_result_fetch_group_columns; one synchronisation
static int copy_groups(obgpu_ctx *ctx, const uint8_t *gv, int64_t ng, int n_cols, int n_aggs, int64_t key_bytes, int64_t *host_keys,
                       uint8_t *host_key_nulls, void *host_key_heap, int64_t *host_out) {
  const GroupBuf lay(ng, n_cols, n_aggs, key_bytes);
  CUDA_TRY(ctx, cudaMemcpyAsync(host_keys, gv, lay.out, cudaMemcpyDeviceToHost, ctx->stream));
  if (ng > 0) {
    CUDA_TRY(ctx, cudaMemcpyAsync(host_out, gv + lay.out, lay.nulls - lay.out, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(host_key_nulls, gv + lay.nulls, (size_t)n_cols * (size_t)ng, cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (key_bytes > 0) CUDA_TRY(ctx, cudaMemcpyAsync(host_key_heap, gv + lay.heap, (size_t)key_bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return OBGPU_SUCCESS;
}

}  // namespace gvals

extern "C" {

int obgpu_result_group_by_values(obgpu_result *r, int32_t group_col, const obgpu_group_agg *aggs, int32_t n_aggs, int64_t *n_groups,
                                 int64_t *key_bytes, int32_t *has_null_group) {
  if (const int ret = gvals::begin_groups(r); ret != OBGPU_SUCCESS) return ret;
  if (group_col < 0 || (uint32_t)group_col >= r->batch->max_cols || n_aggs < 1 || n_aggs > 16 || !aggs || !n_groups || !key_bytes ||
      !has_null_group)
    return OBGPU_INVALID_ARGUMENT;
  int why = 0;
  return gvals::group_by_columns(r, &group_col, 1, aggs, n_aggs, n_groups, key_bytes, has_null_group, &why);
}

int obgpu_result_group_by_columns(obgpu_result *r, const int32_t *group_cols, int32_t n_group_cols, const obgpu_group_agg *aggs,
                                  int32_t n_aggs, int64_t *n_groups, int64_t *key_bytes) {
  if (const int ret = gvals::begin_groups(r); ret != OBGPU_SUCCESS) return ret;
  if (!group_cols || n_group_cols < 1 || n_group_cols > gvals::kMaxGroupCols || n_aggs < 1 || n_aggs > 16 || !aggs || !n_groups || !key_bytes)
    return OBGPU_INVALID_ARGUMENT;
  for (int c = 0; c < n_group_cols; ++c)
    if (group_cols[c] < 0 || (uint32_t)group_cols[c] >= r->batch->max_cols) return OBGPU_INVALID_ARGUMENT;
  int why = 0;
  return gvals::group_by_columns(r, group_cols, n_group_cols, aggs, n_aggs, n_groups, key_bytes, nullptr, &why);
}

int obgpu_result_fetch_groups(obgpu_result *r, int64_t *host_keys, void *host_key_heap, int64_t *host_out) {
  const bool str = r && (r->gv_str_mask & 1u);
  if (!r || r->gv_groups < 0 || r->gv_n_cols != 1 || !host_keys || !host_out || (str && r->gv_key_bytes > 0 && !host_key_heap))
    return OBGPU_INVALID_ARGUMENT;
  obgpu_ctx *ctx = r->ctx;
  cudaSetDevice(ctx->device);
  const int64_t ng = r->gv_groups;
  const gvals::GroupBuf lay(ng, 1, r->gv_n_aggs, r->gv_key_bytes);
  const uint8_t *gv = (const uint8_t *)r->d_gv;
  CUDA_TRY(ctx, cudaMemcpyAsync(host_keys, gv, (size_t)(str ? ng + 1 : ng) * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (lay.nulls > lay.out) CUDA_TRY(ctx, cudaMemcpyAsync(host_out, gv + lay.out, lay.nulls - lay.out, cudaMemcpyDeviceToHost, ctx->stream));
  if (str && r->gv_key_bytes > 0)
    CUDA_TRY(ctx, cudaMemcpyAsync(host_key_heap, gv + lay.heap, (size_t)r->gv_key_bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return OBGPU_SUCCESS;
}

int obgpu_result_fetch_group_columns(obgpu_result *r, int64_t *host_keys, uint8_t *host_key_nulls, void *host_key_heap, int64_t *host_out) {
  if (!r || r->gv_groups < 0 || !host_keys || !host_key_nulls || !host_out || (r->gv_key_bytes > 0 && !host_key_heap))
    return OBGPU_INVALID_ARGUMENT;
  cudaSetDevice(r->ctx->device);
  return gvals::copy_groups(r->ctx, (const uint8_t *)r->d_gv, r->gv_groups, r->gv_n_cols, r->gv_n_aggs, r->gv_key_bytes, host_keys,
                            host_key_nulls, host_key_heap, host_out);
}

}  // extern "C"
