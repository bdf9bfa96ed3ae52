// GROUP BY 1..4 columns of ANY encoding over a whole scan: the hash fold over decoded cells behind obgpu_result_group_by_any.
// The dictionary fold (group_values.cuh) needs every group column dictionary coded in every block and caps values, tuples, key
// lengths and image size; here each selected row's key is read through the block's decode plan (int_cell / str_cell, as
// topn::read_cell reads it), so any encoding the scan decodes works, and nothing is capped but the 2^31 - 1 groups of GroupBuf.
//   check    topn::check_kernel: every block's plan of every group and aggregate column decodes the column's class.
//   fold     one warp per block, grid-stride; each block's record and view are loaded once. Per selected row (the result's bitmap
//            words, or every row without a filter) the tuple of cells: an integer's gvals::order_key, a string's image offset
//            and length, a NULL flag; hashed with gmerge::tuple_hash into an open-addressing table of group index + 1 (0: empty),
//            2 x capacity slots rounded up to a power of two. A new tuple's thread claims an empty slot (CAS to kLocked), takes
//            an index from a counter, writes its cells into a gmerge::Store whose heap is the batch image, fences and publishes
//            index + 1. Many rows carry one tuple, so a prober that meets kLocked waits for the publish and compares.
//            Aggregates [n_aggs][cap][2] as dictops::accumulate folds them (COUNT / SUM in 128 bits, MIN / MAX order key and a
//            seen flag); a claimed group has a row, so no hidden COUNT(*). Lanes of a warp on one group (__match_any_sync)
//            combine their rows first and the lowest issues one atomic per aggregate (two for MIN / MAX).
//   capacity first min(selected rows, 2^20) groups; a claim past capacity sets a flag, the fold stops, and the host folds again
//            once with capacity = selected rows, which no batch can exceed: at most two folds, and a low-cardinality scan never
//            allocates per-row memory.
//   order    gmerge::sorted_groups: the accumulator's TupleLess sort and gather into the result's GroupBuf, which is byte for byte
//            what the dictionary fold writes for the same rows.
#pragma once

namespace gcells {

constexpr int kWarps = 8;
constexpr int kThreads = 32 * kWarps;
constexpr int64_t kFirstGroups = 1ll << 20;    // the first fold's capacity (selected rows, when fewer)
constexpr uint32_t kFull = 0xfffffffeu;        // a slot claimed past capacity: holds no group
enum : int { CTR_GROUPS, CTR_FULL, CTR_COL_BYTES, CTR_N = CTR_COL_BYTES + gvals::kMaxGroupCols };

struct FoldArgs {
  dictops::BlkArgs a;
  int n_blocks;
  int32_t col[gvals::kMaxGroupCols];
  const uint32_t *bitmap;          // nullptr: every row
  int32_t kind[16], agg_col[16];
  gmerge::Store s;                 // heap: the batch image
  uint32_t *table;
  uint64_t mask;
  unsigned long long *ctr;         // CTR_*
};

// group g's cell of column c as the claimer wrote it: read past L1, which may hold the line from before the publish
__device__ __forceinline__ gmerge::Cell published_cell(const gmerge::Store &s, int c, int64_t g) {
  const int64_t i = (int64_t)c * s.cap + g;
  const uint64_t key = __ldcg((const unsigned long long *)&s.key[i]);
  return gmerge::Cell{__ldcg(&s.null[i]) != 0, key, s.heap, key, __ldcg(&s.len[i])};
}

// the group of tuple t: found, or claimed and written; -1 past capacity
__device__ __forceinline__ int64_t group_of(const FoldArgs &p, const gmerge::Cell (&t)[gvals::kMaxGroupCols]) {
  const gmerge::Store &s = p.s;
  uint64_t slot = gmerge::tuple_hash(t, s.n_cols, s.str_mask) & p.mask;
  for (uint64_t k = 0; k <= p.mask; ++k, slot = (slot + 1u) & p.mask) {
    uint32_t cur = *(volatile uint32_t *)&p.table[slot];
    if (cur == 0u) {
      cur = atomicCAS(&p.table[slot], 0u, gmerge::kLocked);
      if (cur == 0u) {
        const uint64_t g = atomicAdd(&p.ctr[CTR_GROUPS], 1ull);
        if (g >= (uint64_t)s.cap) {
          atomicOr(&p.ctr[CTR_FULL], 1ull);
          atomicExch(&p.table[slot], kFull);
          return -1;
        }
        for (int c = 0; c < s.n_cols; ++c) {
          const int64_t i = (int64_t)c * s.cap + (int64_t)g;
          s.null[i] = t[c].null ? 1 : 0;
          s.key[i] = t[c].null ? 0 : (((s.str_mask >> c) & 1u) ? t[c].off : t[c].key);
          s.len[i] = t[c].len;
          if (((s.str_mask >> c) & 1u) && t[c].len) atomicAdd(&p.ctr[CTR_COL_BYTES + c], (unsigned long long)t[c].len);
        }
        __threadfence();   // the cells before the index: a prober that sees the index sees them
        atomicExch(&p.table[slot], (uint32_t)g + 1u);
        return (int64_t)g;
      }
    }
    // Unlike gmerge::find_or_claim, whose tuples within one add are distinct, rows here repeat tuples: a slot still being
    // claimed may hold this very tuple, so passing over it would make a second group of it. Wait for its publish. The claimer
    // may be a lane of this warp; independent thread scheduling (sm_70 and later) lets it run while this lane spins, and it
    // waits on nothing between its CAS and its publish, so the wait always ends.
    while (cur == gmerge::kLocked) cur = *(volatile uint32_t *)&p.table[slot];
    if (cur == kFull) return -1;
    __threadfence();
    const int64_t g = (int64_t)cur - 1;
    bool eq = true;
    for (int c = 0; c < s.n_cols && eq; ++c) eq = gmerge::cell_cmp(t[c], published_cell(s, c, g), (s.str_mask >> c) & 1u) == 0;
    if (eq) return g;
  }
  atomicOr(&p.ctr[CTR_FULL], 1ull);
  return -1;
}

// the peers' (lanes of one group) sum of a 128-bit value lo + hi * 2^64, hi 0 or ~0: 16-bit limbs add without overflow in 32
// bits, and the carries of the limb sums go into the high word
__device__ __forceinline__ void peer_sum(uint32_t peers, uint64_t lo, bool neg, uint64_t &sum_lo, uint64_t &sum_hi) {
  const uint64_t s0 = __reduce_add_sync(peers, (uint32_t)(lo & 0xffffu)), s1 = __reduce_add_sync(peers, (uint32_t)((lo >> 16) & 0xffffu));
  const uint64_t s2 = __reduce_add_sync(peers, (uint32_t)((lo >> 32) & 0xffffu)), s3 = __reduce_add_sync(peers, (uint32_t)(lo >> 48));
  const uint64_t n_neg = __reduce_add_sync(peers, neg ? 1u : 0u);
  const uint64_t t = s0 + (s1 << 16) + (s2 << 32);   // < 2^54
  sum_lo = t + ((s3 & 0xffffu) << 48);
  sum_hi = (s3 >> 16) + (sum_lo < t ? 1ull : 0ull) - n_neg;
}

// the peers' MIN / MAX of 64-bit keys, by the high then the low halves; lanes without a key hold the identity
__device__ __forceinline__ uint64_t peer_minmax(uint32_t peers, bool has, uint64_t key, bool is_min) {
  const uint32_t id = is_min ? ~0u : 0u, h = has ? (uint32_t)(key >> 32) : id;
  const uint32_t hi = is_min ? __reduce_min_sync(peers, h) : __reduce_max_sync(peers, h);
  const uint32_t l = has && h == hi ? (uint32_t)key : id;
  const uint32_t lo = is_min ? __reduce_min_sync(peers, l) : __reduce_max_sync(peers, l);
  return ((uint64_t)hi << 32) | lo;
}

__global__ void __launch_bounds__(kThreads) fold_kernel(const __grid_constant__ FoldArgs p) {
  const int lane = threadIdx.x & 31;
  const gmerge::Store &s = p.s;
  for (int b = blockIdx.x * kWarps + (threadIdx.x >> 5); b < p.n_blocks; b += gridDim.x * kWarps) {
    unsigned long long full = lane == 0 ? *(volatile unsigned long long *)&p.ctr[CTR_FULL] : 0ull;
    if (__shfl_sync(~0u, full, 0)) return;   // past capacity: the host folds again
    const BlockRec rec = p.a.recs[b];
    BlockView bv;
    view_from_rec(rec, p.a.image + rec.off, bv);
    const ColDesc *plans = p.a.plans + (int64_t)b * p.a.max_cols;
    for (uint32_t r0 = 0; r0 < bv.row_count; r0 += 32u) {
      const uint32_t r = r0 + (uint32_t)lane;
      bool sel = r < bv.row_count;
      if (p.bitmap) sel = sel && ((p.bitmap[rec.bm_word_off + (r0 >> 5)] >> lane) & 1u);
      int64_t g = -1;
      if (sel) {
        gmerge::Cell t[gvals::kMaxGroupCols];
        for (int c = 0; c < s.n_cols; ++c) {
          const ColDesc d = plans[p.col[c]];
          bool null = false;
          if ((s.str_mask >> c) & 1u) {
            uint32_t cell = 0, len = 0;
            str_cell(bv, d, nullptr, r, cell, len, null);
            t[c] = gmerge::Cell{null, 0, p.a.image, rec.off + cell, null ? 0u : len};
          } else {
            const uint64_t v = int_cell(bv, d, nullptr, r, null);
            t[c] = gmerge::Cell{null, null ? 0ull : gvals::order_key(d, v), nullptr, 0, 0};
          }
        }
        g = group_of(p, t);
      }
      __syncwarp();
      const uint32_t peers = __match_any_sync(~0u, (uint32_t)g);   // -1: no group, those lanes fold nothing
      const bool leader = g >= 0 && lane == __ffs(peers) - 1;
      for (int k = 0; k < s.n_aggs; ++k) {
        const int kind = p.kind[k];
        bool has = g >= 0, sgn = false;   // sgn: dictops::accumulate's flag, signed or narrow
        uint64_t v = 0;
        if (has && p.agg_col[k] >= 0) {
          const ColDesc d = plans[p.agg_col[k]];
          bool null = false;
          v = (uint64_t)cmp_image(d, int_cell(bv, d, nullptr, r, null));
          has = !null;
          sgn = d.sc == 1 || d.elem_len < 8;
        }
        unsigned long long *a = s.acc + ((int64_t)k * s.cap + (g < 0 ? 0 : g)) * 2;
        if (kind == OBGPU_AGG_COUNT) {
          const uint32_t n = __reduce_add_sync(peers, has ? 1u : 0u);
          if (leader && n) atomicAdd(&a[0], (unsigned long long)n);
        } else if (kind == OBGPU_AGG_SUM) {
          uint64_t lo, hi;
          peer_sum(peers, has ? v : 0ull, has && sgn && (int64_t)v < 0, lo, hi);
          if (leader) {
            const unsigned long long old = atomicAdd(&a[0], lo), carry = old + lo < old ? 1ull : 0ull;
            if (hi + carry) atomicAdd(&a[1], hi + carry);   // 128-bit add: the low word's carry into the high word
          }
        } else {
          const bool is_min = kind == OBGPU_AGG_MIN;
          const uint64_t m = peer_minmax(peers, has, sgn ? v ^ (1ull << 63) : v, is_min);
          const uint32_t seen = __reduce_or_sync(peers, has ? 1u : 0u);
          if (leader && seen) {
            if (is_min) atomicMin(&a[0], m); else atomicMax(&a[0], m);
            atomicOr(&a[1], 1ull);
          }
        }
      }
    }
  }
}

// GROUP BY the tuple of cols[0..n_cols) over decoded cells (arguments checked by the caller; aggregates by gvals::check_aggs)
static int group_by_cells(obgpu_result *r, int64_t n_sel, const int32_t *cols, int n_cols, const obgpu_group_agg *aggs, int32_t n_aggs,
                          int64_t *n_groups, int64_t *key_bytes) {
  obgpu_batch *b = r->batch;
  obgpu_ctx *ctx = r->ctx;
  FoldArgs fp{};
  uint32_t sgn_agg = 0, sgn_key = 0;
  if (const int ret = gvals::check_aggs(ctx, b, aggs, n_aggs, &sgn_agg); ret != OBGPU_SUCCESS) return ret;
  topn::Cols cc{};
  cc.a = dictops::BlkArgs{b->d_image, b->d_recs, b->d_plans, (int32_t)b->max_cols};
  uint32_t str_mask = 0;
  for (int c = 0; c < n_cols; ++c) {
    const uint8_t t = b->col_types[(size_t)cols[c]];
    const int sc = t == 0xff ? 0 : obf::store_class_of(t);
    if (sc != 1 && sc != 2 && sc != 5) { ctx->err = "group-by column is not an integer or string column in every micro block"; return OBGPU_NOT_SUPPORTED; }
    if (sc == 5) str_mask |= 1u << c;
    if (gvals::key_sgn(t)) sgn_key |= 1u << c;
    cc.col[cc.n] = fp.col[c] = cols[c];
    cc.str[cc.n++] = sc == 5;
  }
  for (int k = 0; k < n_aggs; ++k) {
    fp.kind[k] = aggs[k].kind;
    fp.agg_col[k] = aggs[k].col;
    if (aggs[k].col >= 0) {
      cc.col[cc.n] = aggs[k].col;
      cc.str[cc.n++] = 0;
    }
  }
  const int nb = b->n_blocks;
  fp.a = cc.a;
  fp.n_blocks = nb;
  fp.bitmap = r->no_filter ? nullptr : r->d_bitmap;
  Scratch cm(ctx);   // [status][counters]
  const size_t o_status = cm.take(64), o_ctr = cm.take(CTR_N * 8);
  CUDA_TRY(ctx, cm.alloc());
  int *d_status = cm.at<int>(o_status);
  fp.ctr = cm.at<unsigned long long>(o_ctr);
  CUDA_TRY(ctx, cudaMemsetAsync(cm.p, 0, cm.bytes, ctx->stream));
  unsigned long long *hc = (unsigned long long *)ctx->h_pinned;   // [status][CTR_*]
  if (nb > 0) {   // the fold decodes only plans the check passed
    topn::check_kernel<<<(unsigned)((nb + 255) / 256), 256, 0, ctx->stream>>>(cc, nb, d_status);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaMemcpyAsync(hc, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    if (const int st = (int)(uint32_t)hc[0]) return check_status(ctx, st);
  }
  int64_t cap = std::min(kFirstGroups, n_sel);
  for (;;) {
    // the store [keys, lengths, NULL flags, aggregates] and the table, 2 x cap slots rounded up to a power of two
    const gmerge::StoreLayout sl(std::max<int64_t>(cap, 1), n_cols, n_aggs);
    uint64_t slots = 2;
    while (slots < 2 * (uint64_t)std::max<int64_t>(cap, 1)) slots *= 2;
    Scratch sm(ctx);
    const size_t o_store = sm.take(sl.end), o_table = sm.take(slots * 4);
    CUDA_TRY(ctx, sm.alloc());
    uint8_t *base = sm.at<uint8_t>(o_store);
    fp.s = gmerge::Store{(uint64_t *)base, (uint32_t *)(base + sl.len), base + sl.null, (unsigned long long *)(base + sl.acc),
                         const_cast<uint8_t *>(b->d_image), std::max<int64_t>(cap, 1), n_cols, n_aggs, str_mask};   // read only
    fp.table = sm.at<uint32_t>(o_table);
    fp.mask = slots - 1;
    CUDA_TRY(ctx, cudaMemsetAsync(fp.table, 0, slots * 4, ctx->stream));
    CUDA_TRY(ctx, cudaMemsetAsync(fp.s.acc, 0, sl.end - sl.acc, ctx->stream));
    for (int k = 0; k < n_aggs; ++k)   // MIN from the largest key
      if (aggs[k].kind == OBGPU_AGG_MIN) CUDA_TRY(ctx, cudaMemset2DAsync(fp.s.acc + (size_t)k * fp.s.cap * 2, 16, 0xff, 8, (size_t)fp.s.cap, ctx->stream));
    CUDA_TRY(ctx, cudaMemsetAsync(fp.ctr, 0, CTR_N * 8, ctx->stream));
    if (nb > 0 && n_sel > 0) {
      int per_sm = 0;
      CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fold_kernel, kThreads, 0));
      const unsigned grid = (unsigned)std::min<int64_t>((nb + kWarps - 1) / kWarps, (int64_t)std::max(per_sm, 1) * ctx->sm_count);
      fold_kernel<<<grid, kThreads, 0, ctx->stream>>>(fp);
      ctx->launches++;
      CUDA_TRY(ctx, cudaGetLastError());
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(hc, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(hc + 1, fp.ctr, CTR_N * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    if (const int st = (int)(uint32_t)hc[0]) return check_status(ctx, st);
    if (hc[1 + CTR_FULL]) {
      const int64_t exact = std::min(n_sel, gmerge::kMaxGroups);
      if (cap < exact) { cap = exact; continue; }   // the one refold, at a capacity no batch can exceed
      ctx->err = n_sel > gmerge::kMaxGroups ? "more than 2^31 - 1 groups" : "group table full";
      return n_sel > gmerge::kMaxGroups ? OBGPU_NOT_SUPPORTED : OBGPU_ERR_UNEXPECTED;
    }
    const int64_t ng = (int64_t)hc[1 + CTR_GROUPS];
    int64_t col_bytes[gvals::kMaxGroupCols] = {0}, kb = 0;
    for (int c = 0; c < n_cols; ++c) kb += col_bytes[c] = (int64_t)hc[1 + CTR_COL_BYTES + c];
    void *gv = nullptr;
    if (const int ret = gmerge::sorted_groups(ctx, fp.s, ng, fp.kind, sgn_key, sgn_agg, col_bytes, &gv); ret != OBGPU_SUCCESS) return ret;
    gvals::set_groups(r, gv, ng, kb, cols, n_cols, aggs, n_aggs, str_mask, sgn_agg);
    *n_groups = ng;
    *key_bytes = kb;
    return OBGPU_SUCCESS;
  }
}

}  // namespace gcells

extern "C" {

int obgpu_result_group_by_any(obgpu_result *r, const int32_t *group_cols, int32_t n_group_cols, const obgpu_group_agg *aggs, int32_t n_aggs,
                              int64_t *n_groups, int64_t *key_bytes, int32_t *path) {
  if (const int ret = gvals::begin_groups(r); ret != OBGPU_SUCCESS) return ret;
  if (!group_cols || n_group_cols < 1 || n_group_cols > gvals::kMaxGroupCols || n_aggs < 1 || n_aggs > 16 || !aggs || !n_groups || !key_bytes)
    return OBGPU_INVALID_ARGUMENT;
  for (int c = 0; c < n_group_cols; ++c)
    if (group_cols[c] < 0 || (uint32_t)group_cols[c] >= r->batch->max_cols) return OBGPU_INVALID_ARGUMENT;
  int why = gvals::WHY_OTHER;
  const int ret = gvals::group_by_columns(r, group_cols, n_group_cols, aggs, n_aggs, n_groups, key_bytes, nullptr, &why);
  if (ret != OBGPU_NOT_SUPPORTED || why == gvals::WHY_OTHER) {
    if (path) *path = ret == OBGPU_SUCCESS ? OBGPU_GROUP_PATH_DICT : 0;
    return ret;
  }
  obgpu_result_info info;
  if (const int ir = obgpu_result_info_get(r, &info); ir != OBGPU_SUCCESS && ir != OBGPU_BUF_NOT_ENOUGH) return ir;
  const int cr = gcells::group_by_cells(r, info.selected_rows, group_cols, n_group_cols, aggs, n_aggs, n_groups, key_bytes);
  if (path) *path = cr == OBGPU_SUCCESS ? OBGPU_GROUP_PATH_CELLS : 0;
  return cr;
}

}  // extern "C"
