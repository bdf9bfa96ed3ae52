// GROUP BY over a whole scan with one group per distinct VALUE of the group column across the page batch
// (obgpu_result_group_by_values). obgpu_result_group_by keeps the reference's granularity -- one group per (block, dictionary
// entry) -- and leaves the merge by value to the caller, which at millions of small blocks means millions of groups and calls.
// Here the merge happens on the device and only the groups cross PCIe (at most 65 537 of them).
//   keys     one warp per block, lanes over the group column's dictionary entries read through the plans (dict_int + cmp_image,
//            dict_str): each entry goes into the batch codes' open-addressing table (bcodes::probe) -- one slot per distinct
//            value, whatever the block's entry width, base or format. A block whose plan is not dictionary coded sets a status bit.
//                                                            -- the host reads the distinct count: above 65 536, NOT_SUPPORTED --
//   number   bcodes::number_kernel: occupied slots -> codes 0..n_keys-1 (in no fixed order) and the code table
//   order    the codes sorted by key: integers by cub::DeviceRadixSort on the order-preserving 64-bit key (the MIN / MAX key:
//            sign bit flipped for signed and narrow classes), strings by cub::DeviceMergeSort comparing the image bytes as
//            unsigned bytes, a proper prefix first -> code_rank[code] = rank. Keys are distinct, so the order is unique.
//   fold     a grid of CTAs, one warp per block at a time: the block's dictionary entries -> ranks once (per-warp shared array;
//            a dictionary larger than that probes per row), then the selected rows of the result's bitmap words, folded per rank
//            into CTA-private shared accumulators flushed once per CTA with global atomics when they fit kSharedAccBudget, else
//            straight into global accumulators. A hidden COUNT(*) (aggregate 0) marks the non-empty groups.
//   compact  a prefix over the non-empty groups (and, for strings, their key lengths)  -- the host reads the totals --
//            then one gather into the result's group buffer: keys (the value's 64-bit image, or offsets + a key heap whose bytes
//            come from the batch's device image, the only copy of them for batches opened from stored or macro blocks) and the
//            aggregates, MIN / MAX keys turned back into values.
#pragma once

#include <cub/device/device_merge_sort.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace gvals {

constexpr int kWarpsPerCta = 8;
constexpr int kThreads = 32 * kWarpsPerCta;
constexpr uint32_t kRankCap = 256;                // dictionary entries a warp maps to ranks in shared memory; larger: probe per row
constexpr size_t kSharedAccBudget = 48u << 10;    // CTA-private accumulators, (n_keys + 1) x (n_aggs + 1) x 16 bytes, when they fit
enum : int { ST_LONG_KEY = 8 };                   // a string entry of 65 536 bytes or more: no key (bcodes::key_of keeps 16 bits)

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

struct FoldArgs {
  dictops::BlkArgs a;
  int n_blocks, col;
  FoldAggs aggs;
  const uint32_t *bitmap;              // nullptr: every row
  const unsigned long long *table;
  const uint16_t *slot_code;
  const uint32_t *code_rank;
  uint32_t n_keys;                     // rank n_keys: the NULL group
  unsigned long long *acc;             // [aggs.n][n_keys + 1][2]
  int *status;
};

template <bool STR>
__device__ __forceinline__ uint32_t entry_rank(const FoldArgs &p, const BlockView &bv, const ColDesc &d, uint64_t off, uint32_t e) {
  uint64_t abs = 0, v = 0;
  uint32_t len = 0;
  entry_key<STR>(bv, d, off, e, abs, len, v);
  const uint32_t slot = bcodes::probe<STR>(p.a.image, const_cast<unsigned long long *>(p.table), abs, len, v, false, nullptr);
  if (slot == bcodes::kNoSlot) { atomicOr(p.status, ST_CORRUPT); return p.n_keys; }
  return p.code_rank[p.slot_code[slot]];
}

// SHARED: fold into CTA-private accumulators (dynamic shared memory past the warps' rank arrays), flushed at the end
template <bool STR, bool SHARED>
__global__ void __maxnreg__(96) fold_kernel(const __grid_constant__ FoldArgs p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t *ranks = (uint32_t *)g_smem + warp * kRankCap;
  const int64_t G = (int64_t)p.n_keys + 1, n_acc = (int64_t)p.aggs.n * G;
  unsigned long long *acc = p.acc;
  if (SHARED) {
    acc = (unsigned long long *)(g_smem + kWarpsPerCta * kRankCap * 4);
    for (int64_t i = threadIdx.x; i < n_acc; i += blockDim.x) {
      acc[2 * i] = p.aggs.kind[i / G] == OBGPU_AGG_MIN ? ~0ull : 0ull;
      acc[2 * i + 1] = 0ull;
    }
    __syncthreads();
  }
  for (int b = blockIdx.x * kWarpsPerCta + warp; b < p.n_blocks; b += gridDim.x * kWarpsPerCta) {
    BlockView bv;
    ColDesc gd;
    if (!dictops::load_plan(p.a, b, p.col, bv, gd)) { if (lane == 0) atomicOr(p.status, ST_UNSUPPORTED); continue; }
    const BlockRec rec = p.a.recs[b];
    const bool in_smem = gd.dict_count <= kRankCap;
    if (in_smem)
      for (uint32_t e = (uint32_t)lane; e < gd.dict_count; e += 32u) ranks[e] = entry_rank<STR>(p, bv, gd, rec.off, e);
    __syncwarp();
    for (uint32_t r0 = 0; r0 < bv.row_count; r0 += 32u) {
      const uint32_t r = r0 + (uint32_t)lane;
      bool sel = r < bv.row_count;
      if (p.bitmap) sel = sel && ((p.bitmap[rec.bm_word_off + (r0 >> 5)] >> lane) & 1u);
      if (!sel) continue;
      const uint32_t ref = ref_of(bv.s, gd, nullptr, r);
      const uint32_t g = ref >= gd.dict_count ? p.n_keys : in_smem ? ranks[ref] : entry_rank<STR>(p, bv, gd, rec.off, ref);
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
  if (!SHARED) return;
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

// group g is kept when its hidden COUNT(*) is not zero; lens[g] its key bytes (strings)
__global__ void flags_kernel(const unsigned long long *acc, int64_t G, bool str, const uint64_t *rank_key, int32_t *flags, int64_t *lens) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const bool keep = acc[2 * g] != 0ull;
  flags[g] = keep ? 1 : 0;
  lens[g] = keep && str && g + 1 < G ? (int64_t)bcodes::key_len(rank_key[g]) : 0;
}

// [n_groups, key bytes, has NULL group]
__global__ void totals_kernel(const int32_t *flags, const int32_t *pos, const int64_t *lens, const int64_t *koff, int64_t G, int64_t *tot) {
  tot[0] = (int64_t)pos[G - 1] + flags[G - 1];
  tot[1] = koff[G - 1] + lens[G - 1];
  tot[2] = flags[G - 1];
}

struct GatherArgs {
  const unsigned long long *acc;
  int64_t G, n_groups;
  int n_aggs;
  int32_t kind[16];
  uint32_t sgn_agg;         // bit k: MIN / MAX key of aggregate k has its sign bit flipped
  bool str, sgn_key;
  const int32_t *flags, *pos;
  const int64_t *lens, *koff;
  const uint64_t *rank_key;
  const uint8_t *image;
  int64_t *keys;            // integers: [n_groups] images; strings: [n_groups + 1] heap offsets
  uint8_t *heap;
  int64_t *out;             // [n_aggs][n_groups][2]
};

__global__ void gather_kernel(const __grid_constant__ GatherArgs p) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= p.G || !p.flags[g]) return;
  const int64_t q = p.pos[g];
  const bool null_group = g + 1 == p.G;
  if (p.str) {
    p.keys[q] = p.koff[g];
    if (q + 1 == p.n_groups) p.keys[q + 1] = p.koff[g] + p.lens[g];
    if (!null_group) {
      const uint64_t abs = bcodes::key_abs(p.rank_key[g]);
      for (int64_t i = 0; i < p.lens[g]; ++i) p.heap[p.koff[g] + i] = p.image[abs + i];
    }
  } else {
    p.keys[q] = null_group ? 0 : (int64_t)(p.sgn_key ? p.rank_key[g] ^ (1ull << 63) : p.rank_key[g]);
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

}  // namespace gvals

extern "C" {

int obgpu_result_group_by_values(obgpu_result *r, int32_t group_col, const obgpu_group_agg *aggs, int32_t n_aggs, int64_t *n_groups,
                                 int64_t *key_bytes, int32_t *has_null_group) {
  if (!r) return OBGPU_INVALID_ARGUMENT;
  {
    obgpu_result_info info;
    const int ret = obgpu_result_info_get(r, &info);   // the scan's own status first
    if (ret != OBGPU_SUCCESS && ret != OBGPU_BUF_NOT_ENOUGH) return ret;
  }
  obgpu_batch *b = r->batch;
  obgpu_ctx *ctx = r->ctx;
  cudaSetDevice(ctx->device);
  if (r->d_gv) cudaFreeAsync(r->d_gv, ctx->stream);   // the previous call's groups
  r->d_gv = nullptr;
  r->gv_groups = -1;
  if (group_col < 0 || (uint32_t)group_col >= b->max_cols || n_aggs < 1 || n_aggs > 16 || !aggs || !n_groups || !key_bytes || !has_null_group)
    return OBGPU_INVALID_ARGUMENT;
  gvals::FoldAggs ga{};
  ga.n = n_aggs + 1;
  ga.kind[0] = OBGPU_AGG_COUNT;
  ga.col[0] = -1;
  gvals::GatherArgs gp{};
  gp.n_aggs = n_aggs;
  for (int k = 0; k < n_aggs; ++k) {
    if (aggs[k].kind < OBGPU_AGG_COUNT || aggs[k].kind > OBGPU_AGG_MAX || aggs[k].kind == OBGPU_AGG_SUM_PRODUCT) return OBGPU_NOT_SUPPORTED;
    if (aggs[k].col >= (int32_t)b->max_cols || (aggs[k].col < 0 && aggs[k].kind != OBGPU_AGG_COUNT)) return OBGPU_INVALID_ARGUMENT;
    if (aggs[k].col >= 0) {
      const uint8_t t = b->col_types[(size_t)aggs[k].col];
      const int sc = t == 0xff ? 0 : obf::store_class_of(t);
      if (sc != 1 && sc != 2) { ctx->err = "aggregates fold integer-class columns only"; return OBGPU_NOT_SUPPORTED; }
      if (obf::store_class_of(t) == 1 || obf::datum_len_of(t) < 8) gp.sgn_agg |= 1u << k;
    }
    ga.kind[k + 1] = gp.kind[k] = aggs[k].kind;
    ga.col[k + 1] = aggs[k].col;
  }
  const uint8_t gt = b->col_types[(size_t)group_col];
  const int gsc = gt == 0xff ? 0 : obf::store_class_of(gt);
  if (gsc != 1 && gsc != 2 && gsc != 5) { ctx->err = "group-by column is not an integer or string column in every micro block"; return OBGPU_NOT_SUPPORTED; }
  const bool str = gsc == 5;
  if (str && b->image_size >= (int64_t)1 << 37) { ctx->err = "string group keys address images below 2^37 bytes"; return OBGPU_NOT_SUPPORTED; }
  gp.str = str;
  gp.sgn_key = gsc == 1 || obf::datum_len_of(gt) < 8;
  const int n = b->n_blocks;
  const int64_t Gmax = (int64_t)bcodes::kMaxCodes + 1;
  // cub's temporaries, sized for the most keys
  size_t t_sort = 0, t_scan = 0, t_scan64 = 0;
  if (str)
    CUDA_TRY(ctx, cub::DeviceMergeSort::SortKeys(nullptr, t_sort, (uint32_t *)nullptr, (int64_t)bcodes::kMaxCodes, gvals::StrLess{}, ctx->stream));
  else
    CUDA_TRY(ctx, cub::DeviceRadixSort::SortPairs(nullptr, t_sort, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const uint32_t *)nullptr,
                                                  (uint32_t *)nullptr, bcodes::kMaxCodes, 0, 64, ctx->stream));
  CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(nullptr, t_scan, (const int32_t *)nullptr, (int32_t *)nullptr, Gmax, ctx->stream));
  CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(nullptr, t_scan64, (const int64_t *)nullptr, (int64_t *)nullptr, Gmax, ctx->stream));
  // temporaries: [status][counters][totals][table][slot -> code][code table][codes, sorted codes][sorted keys][code -> rank]
  // [rank -> key][flags, positions][lengths, offsets][sort / scan temporaries]
  Scratch tmp(ctx);
  const size_t o_status = tmp.take(64), o_ctr = tmp.take(32), o_tot = tmp.take(32);
  const size_t o_table = tmp.take((size_t)bcodes::kTableSlots * 8), o_slot = tmp.take((size_t)bcodes::kTableSlots * 2 + 16);
  const size_t o_ctab = tmp.take((size_t)bcodes::kMaxCodes * 8), o_codes = tmp.take((size_t)bcodes::kMaxCodes * 4);
  const size_t o_scodes = tmp.take((size_t)bcodes::kMaxCodes * 4), o_skeys = tmp.take((size_t)bcodes::kMaxCodes * 8);
  const size_t o_rank = tmp.take((size_t)bcodes::kMaxCodes * 4), o_rkey = tmp.take((size_t)bcodes::kMaxCodes * 8);
  const size_t o_flags = tmp.take((size_t)Gmax * 4), o_pos = tmp.take((size_t)Gmax * 4);
  const size_t o_lens = tmp.take((size_t)Gmax * 8), o_koff = tmp.take((size_t)Gmax * 8);
  const size_t o_sort = tmp.take(t_sort), o_scan = tmp.take(t_scan), o_scan64 = tmp.take(t_scan64);
  CUDA_TRY(ctx, tmp.alloc());
  int *d_status = tmp.at<int>(o_status);
  unsigned int *ctr = tmp.at<unsigned int>(o_ctr);   // [entries inserted, table full, codes numbered, integer 2^64 - 1 seen]
  unsigned long long *table = tmp.at<unsigned long long>(o_table);
  uint64_t *code_table = tmp.at<uint64_t>(o_ctab);
  CUDA_TRY(ctx, cudaMemsetAsync(tmp.p, 0, o_slot, ctx->stream));   // status, counters, totals, table
  const dictops::BlkArgs a{b->d_image, b->d_recs, b->d_plans, (int32_t)b->max_cols};
  const unsigned key_grid = (unsigned)((n + gvals::kWarpsPerCta - 1) / gvals::kWarpsPerCta);
  if (n > 0) {
    (str ? gvals::keys_kernel<true> : gvals::keys_kernel<false>)<<<key_grid, gvals::kThreads, 0, ctx->stream>>>(a, n, group_col, table, ctr, d_status);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
  }
  int32_t *hs = (int32_t *)ctx->h_pinned;
  CUDA_TRY(ctx, cudaMemcpyAsync(hs, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(hs + 1, ctr, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (hs[0] & ST_UNSUPPORTED) { ctx->err = "group-by column is not dictionary coded in every micro block"; return OBGPU_NOT_SUPPORTED; }
  if (hs[0] & gvals::ST_LONG_KEY) { ctx->err = "group-by string of 65536 bytes or more"; return OBGPU_NOT_SUPPORTED; }
  if (hs[0]) return check_status(ctx, hs[0]);
  if (hs[2] || (uint32_t)hs[1] > (uint32_t)bcodes::kMaxCodes) { ctx->err = "more than 65536 distinct group-by values in the batch"; return OBGPU_NOT_SUPPORTED; }
  const int n_keys = hs[1];
  const int64_t G = (int64_t)n_keys + 1;
  uint32_t *code_rank = tmp.at<uint32_t>(o_rank);
  uint64_t *rank_key = tmp.at<uint64_t>(o_rkey);
  if (n_keys > 0) {
    uint16_t *slot_code = tmp.at<uint16_t>(o_slot);
    uint32_t *codes = tmp.at<uint32_t>(o_codes), *sorted = tmp.at<uint32_t>(o_scodes);
    bcodes::number_kernel<<<bcodes::kTableSlots / 256 + 1, 256, 0, ctx->stream>>>(table, str, ctr, slot_code, code_table);
    gvals::iota_kernel<<<(n_keys + 255) / 256, 256, 0, ctx->stream>>>(codes, n_keys);
    ctx->launches += 2;
    if (str) {
      CUDA_TRY(ctx, cudaMemcpyAsync(sorted, codes, (size_t)n_keys * 4, cudaMemcpyDeviceToDevice, ctx->stream));
      CUDA_TRY(ctx, cub::DeviceMergeSort::SortKeys(tmp.p + o_sort, t_sort, sorted, (int64_t)n_keys, gvals::StrLess{b->d_image, code_table}, ctx->stream));
    } else {
      CUDA_TRY(ctx, cub::DeviceRadixSort::SortPairs(tmp.p + o_sort, t_sort, (const uint64_t *)code_table, tmp.at<uint64_t>(o_skeys),
                                                    (const uint32_t *)codes, sorted, n_keys, 0, 64, ctx->stream));
    }
    gvals::rank_kernel<<<(n_keys + 255) / 256, 256, 0, ctx->stream>>>(sorted, code_table, n_keys, code_rank, rank_key);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
  }
  // accumulators [n_aggs + 1][G][2], MIN from the largest key
  const size_t acc_bytes = (size_t)ga.n * (size_t)G * 16;
  Scratch accm(ctx);
  CUDA_TRY(ctx, accm.alloc(acc_bytes));
  unsigned long long *acc = accm.at<unsigned long long>(0);
  CUDA_TRY(ctx, cudaMemsetAsync(acc, 0, acc_bytes, ctx->stream));
  for (int k = 1; k < ga.n; ++k)
    if (ga.kind[k] == OBGPU_AGG_MIN) CUDA_TRY(ctx, cudaMemset2DAsync(acc + (size_t)k * G * 2, 16, 0xff, 8, (size_t)G, ctx->stream));
  if (n > 0) {
    const gvals::FoldArgs fp{a, n, group_col, ga, r->no_filter ? nullptr : r->d_bitmap, table, tmp.at<uint16_t>(o_slot), code_rank, (uint32_t)n_keys, acc,
                             d_status};
    const bool shared = acc_bytes <= gvals::kSharedAccBudget;
    const size_t smem = (size_t)gvals::kWarpsPerCta * gvals::kRankCap * 4 + (shared ? acc_bytes : 0);
    const auto fold = str ? (shared ? gvals::fold_kernel<true, true> : gvals::fold_kernel<true, false>)
                          : (shared ? gvals::fold_kernel<false, true> : gvals::fold_kernel<false, false>);
    CUDA_TRY(ctx, cudaFuncSetAttribute(fold, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    unsigned grid = key_grid;
    if (shared) {   // few CTAs, each folding many blocks: one flush per resident CTA
      int per_sm = 0;
      CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fold, gvals::kThreads, smem));
      grid = std::min(grid, (unsigned)std::max(per_sm, 1) * (unsigned)ctx->sm_count);
    }
    fold<<<grid, gvals::kThreads, smem, ctx->stream>>>(fp);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
  }
  int32_t *flags = tmp.at<int32_t>(o_flags), *pos = tmp.at<int32_t>(o_pos);
  int64_t *lens = tmp.at<int64_t>(o_lens), *koff = tmp.at<int64_t>(o_koff), *tot = tmp.at<int64_t>(o_tot);
  gvals::flags_kernel<<<(unsigned)((G + 255) / 256), 256, 0, ctx->stream>>>(acc, G, str, rank_key, flags, lens);
  CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(tmp.p + o_scan, t_scan, flags, pos, G, ctx->stream));
  CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(tmp.p + o_scan64, t_scan64, lens, koff, G, ctx->stream));
  gvals::totals_kernel<<<1, 1, 0, ctx->stream>>>(flags, pos, lens, koff, G, tot);
  ctx->launches += 2;
  CUDA_TRY(ctx, cudaGetLastError());
  int64_t *ht = (int64_t *)ctx->h_pinned;
  CUDA_TRY(ctx, cudaMemcpyAsync(ht, tot, 24, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(ht + 3, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  const int64_t ng = ht[0], kb = ht[1];
  const int32_t has_null = (int32_t)ht[2], st = (int32_t)ht[3];
  if (st) return check_status(ctx, st);
  // the result's groups: [keys: images, or n_groups + 1 offsets][aggregates][key heap]
  const size_t keys_bytes = ((size_t)ng + 1) * 8, out_bytes = (size_t)n_aggs * (size_t)ng * 16;
  void *gv = nullptr;
  CUDA_TRY(ctx, cudaMallocAsync(&gv, keys_bytes + out_bytes + (size_t)kb + 16, ctx->stream));
  if (const cudaError_t e = cudaMemsetAsync(gv, 0, keys_bytes, ctx->stream); e != cudaSuccess) {   // no group: offsets {0}
    cudaFreeAsync(gv, ctx->stream);
    ctx->err = std::string("cudaMemsetAsync: ") + cudaGetErrorString(e);
    return OBGPU_ERR_SYS;
  }
  gp.acc = acc;
  gp.G = G;
  gp.n_groups = ng;
  gp.flags = flags;
  gp.pos = pos;
  gp.lens = lens;
  gp.koff = koff;
  gp.rank_key = rank_key;
  gp.image = b->d_image;
  gp.keys = (int64_t *)gv;
  gp.out = (int64_t *)((uint8_t *)gv + keys_bytes);
  gp.heap = (uint8_t *)gv + keys_bytes + out_bytes;
  gvals::gather_kernel<<<(unsigned)((G + 255) / 256), 256, 0, ctx->stream>>>(gp);
  ctx->launches++;
  if (const cudaError_t e = cudaGetLastError(); e != cudaSuccess) {
    cudaFreeAsync(gv, ctx->stream);
    ctx->err = std::string("gather_kernel: ") + cudaGetErrorString(e);
    return OBGPU_ERR_SYS;
  }
  r->d_gv = gv;
  r->gv_groups = ng;
  r->gv_key_bytes = kb;
  r->gv_n_aggs = n_aggs;
  r->gv_str = str;
  *n_groups = ng;
  *key_bytes = str ? kb : 0;
  *has_null_group = has_null;
  return OBGPU_SUCCESS;
}

int obgpu_result_fetch_groups(obgpu_result *r, int64_t *host_keys, void *host_key_heap, int64_t *host_out) {
  if (!r || r->gv_groups < 0 || !host_keys || !host_out || (r->gv_str && r->gv_key_bytes > 0 && !host_key_heap)) return OBGPU_INVALID_ARGUMENT;
  obgpu_ctx *ctx = r->ctx;
  cudaSetDevice(ctx->device);
  const int64_t ng = r->gv_groups;
  const size_t keys_bytes = ((size_t)ng + 1) * 8, out_bytes = (size_t)r->gv_n_aggs * (size_t)ng * 16;
  const uint8_t *gv = (const uint8_t *)r->d_gv;
  CUDA_TRY(ctx, cudaMemcpyAsync(host_keys, gv, (size_t)(r->gv_str ? ng + 1 : ng) * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (out_bytes) CUDA_TRY(ctx, cudaMemcpyAsync(host_out, gv + keys_bytes, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));
  if (r->gv_str && r->gv_key_bytes > 0)
    CUDA_TRY(ctx, cudaMemcpyAsync(host_key_heap, gv + keys_bytes + out_bytes, (size_t)r->gv_key_bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return OBGPU_SUCCESS;
}

}  // extern "C"
