// Dictionary surface of a micro-block: what the reference exposes for pushdown GROUP BY and for black filters on one
// dictionary-coded column.
//   ObIMicroBlockReader::get_distinct_count / read_distinct / read_reference / get_group_by_aggregate_result
//     (encoding/ob_micro_block_decoder.cpp:2263-2400; ObDictDecoder::get_distinct_count / batch_read_distinct /
//      read_reference, encoding/ob_dict_decoder.cpp:1681-1830; ObGroupByCell::eval_batch, access/ob_pushdown_aggregate*.h)
//   ObMicroBlockDecoder::filter_black_filter_batch -> ObDictDecoder::pushdown_operator(black filter): the SQL expression
//     is evaluated on the DISTINCT values and rows test their ref (encoding/ob_micro_block_decoder.cpp:1822-1859,
//     can_apply_black ob_micro_block_decoder.h:332-337). Only the caller can evaluate the expression, so the entry
//     takes the per-entry verdicts it computed from read_distinct's output.
// Works on every dictionary-coded plan (DICT, RLE, CONST with a dictionary; PAX and CS): group id = ref, ref ==
// distinct count is the NULL group.
#pragma once

namespace dictops {

struct BlkArgs {
  const uint8_t *image;
  const BlockRec *recs;
  const ColDesc *plans;
  int32_t max_cols;
};

__device__ __forceinline__ bool load_plan(const BlkArgs &a, int block, int col, BlockView &bv, ColDesc &d) {
  const BlockRec rec = a.recs[block];
  view_from_rec(rec, a.image + rec.off, bv);
  d = a.plans[(int64_t)block * a.max_cols + col];
  return bv.ok && d.ok && is_dict_kind(d);
}

// read_distinct: entry i -> value image (integers) or (block offset, length) of the cell (strings)
__global__ void __launch_bounds__(128) read_distinct_kernel(BlkArgs a, int block, int col, uint64_t *vals, int32_t *lens, int *status) {
  BlockView bv;
  ColDesc d;
  if (!load_plan(a, block, col, bv, d)) { if (threadIdx.x == 0) atomicOr(status, ST_UNSUPPORTED); return; }
  for (uint32_t i = threadIdx.x; i < d.dict_count; i += blockDim.x) {
    if (d.sc == 5) {
      uint32_t cell, len;
      dict_str(bv.s, d, i, cell, len);
      vals[i] = cell;
      lens[i] = (int32_t)len;
    } else {
      vals[i] = dict_int(bv.s, d, i);
    }
  }
}

// read_reference: ref of every listed row (NULL / NOP rows: the distinct count)
__global__ void __launch_bounds__(128) read_reference_kernel(BlkArgs a, int block, int col, const int32_t *row_ids, int64_t row_cap,
                                                             uint32_t *refs, int *status) {
  BlockView bv;
  ColDesc d;
  if (!load_plan(a, block, col, bv, d)) { if (threadIdx.x == 0) atomicOr(status, ST_UNSUPPORTED); return; }
  for (int64_t i = threadIdx.x; i < row_cap; i += blockDim.x) {
    const int32_t r = row_ids[i];
    if (r < 0 || (uint32_t)r >= bv.row_count) { atomicOr(status, ST_CORRUPT); continue; }
    const uint32_t ref = ref_of(bv.s, d, nullptr, (uint32_t)r);
    refs[i] = ref < d.dict_count ? ref : d.dict_count;
  }
}

// rows [start, start + count) against per-entry verdicts -> ObBitmap bytes
__global__ void __launch_bounds__(128) dict_pass_kernel(BlkArgs a, int block, int col, const uint8_t *entry_pass, int64_t n_entries, int null_pass,
                                                        int64_t start, int64_t count, uint8_t *out, int *status) {
  BlockView bv;
  ColDesc d;
  if (!load_plan(a, block, col, bv, d) || (int64_t)d.dict_count != n_entries || start + count > (int64_t)bv.row_count) {
    if (threadIdx.x == 0) atomicOr(status, d.ok && bv.ok && is_dict_kind(d) ? ST_CORRUPT : ST_UNSUPPORTED);
    return;
  }
  for (int64_t i = threadIdx.x; i < count; i += blockDim.x) {
    const uint32_t ref = ref_of(bv.s, d, nullptr, (uint32_t)(start + i));
    out[i] = ref < d.dict_count ? (entry_pass[ref] != 0) : (null_pass != 0 && ref == d.dict_count);
  }
}

struct GroupAggs {
  int32_t n;
  int32_t kind[16], col[16];
};

__device__ __forceinline__ void accumulate(unsigned long long *acc /* [2] */, int kind, long long v, bool sgn_or_narrow) {
  if (kind == OBGPU_AGG_COUNT) { atomicAdd(&acc[0], 1ull); return; }
  if (kind == OBGPU_AGG_SUM) {
    const unsigned long long lo = (unsigned long long)v, old = atomicAdd(&acc[0], lo);
    unsigned long long hi = (sgn_or_narrow && v < 0) ? ~0ull : 0ull;
    if (old + lo < old) hi += 1ull;
    if (hi) atomicAdd(&acc[1], hi);
    return;
  }
  const unsigned long long key = sgn_or_narrow ? (unsigned long long)v ^ (1ull << 63) : (unsigned long long)v;
  if (kind == OBGPU_AGG_MIN) atomicMin(&acc[0], key); else atomicMax(&acc[0], key);
  atomicOr(&acc[1], 1ull);
}

// One warp per block: the listed rows (row_ids; or the rows of the selection bitmap) are folded into per-ref accumulators
// out[(agg * n_groups_total + group_off[block] + ref) * 2].
__global__ void __launch_bounds__(128) group_by_kernel(BlkArgs a, int block0, int n_blocks, int group_col, GroupAggs aggs, const int32_t *row_ids,
                                                       int64_t row_cap, const uint32_t *bitmap_words, const int64_t *group_off,
                                                       int64_t n_groups_total, unsigned long long *out, int *status) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int bi = blockIdx.x * (blockDim.x >> 5) + warp;
  if (bi >= n_blocks) return;
  const int block = block0 + bi;
  BlockView bv;
  ColDesc gd;
  if (!load_plan(a, block, group_col, bv, gd)) { if (lane == 0) atomicOr(status, ST_UNSUPPORTED); return; }
  const BlockRec rec = a.recs[block];
  const int64_t goff = group_off[bi];
  const int64_t nrows = row_ids ? row_cap : (int64_t)bv.row_count;
  for (int64_t i = lane; i < nrows; i += 32) {
    uint32_t r;
    if (row_ids) {
      const int32_t rr = row_ids[i];
      if (rr < 0 || (uint32_t)rr >= bv.row_count) { atomicOr(status, ST_CORRUPT); continue; }
      r = (uint32_t)rr;
    } else {
      r = (uint32_t)i;
      if (bitmap_words && !((bitmap_words[rec.bm_word_off + (r >> 5)] >> (r & 31u)) & 1u)) continue;
    }
    uint32_t ref = ref_of(bv.s, gd, nullptr, r);
    if (ref > gd.dict_count) ref = gd.dict_count;
    for (int k = 0; k < aggs.n; ++k) {
      unsigned long long *acc = out + ((int64_t)k * n_groups_total + goff + ref) * 2;
      if (aggs.kind[k] == OBGPU_AGG_COUNT && aggs.col[k] < 0) { atomicAdd(&acc[0], 1ull); continue; }   // COUNT(*)
      const ColDesc d = a.plans[(int64_t)block * a.max_cols + aggs.col[k]];
      if (!d.ok || d.sc == 5) { atomicOr(status, ST_UNSUPPORTED); continue; }
      bool is_null;
      const uint64_t v = int_cell(bv, d, nullptr, r, is_null);
      if (is_null) continue;
      const bool sgn = d.sc == 1 || d.elem_len < 8;
      accumulate(acc, aggs.kind[k], (long long)cmp_image(d, v), sgn);
    }
  }
}

}  // namespace dictops

namespace {

struct DictCall {
  obgpu_ctx *ctx;
  dictops::BlkArgs a;
  int *d_status = nullptr;
};

int dict_call_begin(obgpu_batch *b, int32_t block, int32_t col, DictCall &c) {
  if (!b || block < 0 || block >= b->n_blocks || col < 0 || (uint32_t)col >= b->max_cols) return OBGPU_INVALID_ARGUMENT;
  c.ctx = b->ctx;
  cudaSetDevice(c.ctx->device);
  c.a = dictops::BlkArgs{b->d_image, b->d_recs, b->d_plans, (int32_t)b->max_cols};
  return OBGPU_SUCCESS;
}

// the (block, col) plan on the host: its dictionary size; NOT_SUPPORTED when the column is not dictionary coded there
int host_plan(obgpu_batch *b, int32_t block, int32_t col, ColDesc &d) {
  obgpu_ctx *ctx = b->ctx;
  CUDA_TRY(ctx, cudaMemcpyAsync(&d, b->d_plans + (int64_t)block * b->max_cols + col, sizeof(ColDesc), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (!d.ok || !(d.kind == K_DICT || d.kind == K_RLE || d.kind == K_CONST)) {
    ctx->err = "column is not dictionary coded in this micro block";
    return OBGPU_NOT_SUPPORTED;
  }
  return OBGPU_SUCCESS;
}

}  // namespace

extern "C" {

int obgpu_batch_column_type(const obgpu_batch *b, int32_t col, int32_t *obj_type, int32_t *datum_len) {
  if (!b || col < 0 || (size_t)col >= b->col_types.size()) return OBGPU_INVALID_ARGUMENT;
  const uint8_t t = b->col_types[(size_t)col];
  if (obj_type) *obj_type = t;
  if (datum_len) {
    const int sc = obf::store_class_of(t);
    if (sc == 0) return OBGPU_NOT_SUPPORTED;
    *datum_len = sc == 5 ? 0 : obf::datum_len_of(t);
  }
  return OBGPU_SUCCESS;
}

int obgpu_block_distinct_count(obgpu_batch *b, int32_t block, int32_t col, int64_t *count) {
  DictCall c;
  int ret = dict_call_begin(b, block, col, c);
  if (ret != OBGPU_SUCCESS || !count) return ret != OBGPU_SUCCESS ? ret : OBGPU_INVALID_ARGUMENT;
  ColDesc d;
  if ((ret = host_plan(b, block, col, d)) != OBGPU_SUCCESS) return ret;
  *count = d.dict_count;
  return OBGPU_SUCCESS;
}

int obgpu_block_read_distinct(obgpu_batch *b, int32_t block, int32_t col, uint64_t string_base, uint64_t *vals, int32_t *lens, int64_t cap,
                              int64_t *count) {
  DictCall c;
  int ret = dict_call_begin(b, block, col, c);
  if (ret != OBGPU_SUCCESS || !vals || !count) return ret != OBGPU_SUCCESS ? ret : OBGPU_INVALID_ARGUMENT;
  ColDesc d;
  if ((ret = host_plan(b, block, col, d)) != OBGPU_SUCCESS) return ret;
  *count = d.dict_count;
  if ((int64_t)d.dict_count > cap) return OBGPU_BUF_NOT_ENOUGH;
  if (d.sc == 5 && !lens) return OBGPU_INVALID_ARGUMENT;
  if (d.dict_count == 0) return OBGPU_SUCCESS;
  obgpu_ctx *ctx = c.ctx;
  Scratch tmp(ctx);
  const size_t n = d.dict_count;
  const size_t o_status = tmp.take(64, 8), o_vals = tmp.take(n * 8, 8), o_lens = tmp.take(n * 4, 4);
  CUDA_TRY(ctx, tmp.alloc());
  int *d_status = tmp.at<int>(o_status);
  uint64_t *d_vals = tmp.at<uint64_t>(o_vals);
  int32_t *d_lens = tmp.at<int32_t>(o_lens);
  CUDA_TRY(ctx, cudaMemsetAsync(tmp.p, 0, 64, ctx->stream));
  dictops::read_distinct_kernel<<<1, 128, 0, ctx->stream>>>(c.a, block, col, d_vals, d_lens, d_status);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  int st = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&st, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(vals, d_vals, n * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (d.sc == 5) CUDA_TRY(ctx, cudaMemcpyAsync(lens, d_lens, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (st) return check_status(ctx, st);
  if (d.sc == 5) {   // block offsets of the cells -> addresses in the caller's image
    uint64_t base = string_base + (uint64_t)b->offsets[(size_t)block];
    if (b->d_xf) {   // restated batch (CS stream codecs): where the block and its string area came from
      obcs::XformRec x;
      CUDA_TRY(ctx, cudaMemcpyAsync(&x, b->d_xf + block, sizeof(x), cudaMemcpyDeviceToHost, ctx->stream));
      CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
      base = string_base + x.orig_off + (uint64_t)x.str_delta;
    }
    for (size_t i = 0; i < n; ++i) vals[i] += base;
  }
  return OBGPU_SUCCESS;
}

int obgpu_block_read_reference(obgpu_batch *b, int32_t block, int32_t col, const int32_t *row_ids, int64_t row_cap, uint32_t *refs) {
  DictCall c;
  int ret = dict_call_begin(b, block, col, c);
  if (ret != OBGPU_SUCCESS || !row_ids || !refs || row_cap < 0) return ret != OBGPU_SUCCESS ? ret : OBGPU_INVALID_ARGUMENT;
  if (row_cap == 0) return OBGPU_SUCCESS;
  obgpu_ctx *ctx = c.ctx;
  Scratch tmp(ctx);
  const size_t o_status = tmp.take(64, 4), o_rid = tmp.take((size_t)row_cap * 4, 4), o_refs = tmp.take((size_t)row_cap * 4, 4);
  CUDA_TRY(ctx, tmp.alloc());
  int *d_status = tmp.at<int>(o_status);
  int32_t *d_rid = tmp.at<int32_t>(o_rid);
  uint32_t *d_refs = tmp.at<uint32_t>(o_refs);
  CUDA_TRY(ctx, cudaMemsetAsync(tmp.p, 0, 64, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(d_rid, row_ids, (size_t)row_cap * 4, cudaMemcpyHostToDevice, ctx->stream));
  dictops::read_reference_kernel<<<1, 128, 0, ctx->stream>>>(c.a, block, col, d_rid, row_cap, d_refs, d_status);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  int st = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&st, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(refs, d_refs, (size_t)row_cap * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return check_status(ctx, st);
}

int obgpu_filter_dict_pass(obgpu_batch *b, int32_t block, int32_t col, const uint8_t *entry_pass, int64_t n_entries, int32_t null_pass,
                           int64_t start, int64_t count, uint8_t *result_bitmap) {
  DictCall c;
  int ret = dict_call_begin(b, block, col, c);
  if (ret != OBGPU_SUCCESS || (!entry_pass && n_entries > 0) || n_entries < 0 || start < 0 || count < 0 || !result_bitmap ||
      start + count > (int64_t)b->row_count[(size_t)block])
    return ret != OBGPU_SUCCESS ? ret : OBGPU_INVALID_ARGUMENT;
  {
    ColDesc d;
    if ((ret = host_plan(b, block, col, d)) != OBGPU_SUCCESS) return ret;
    if ((int64_t)d.dict_count != n_entries) {
      c.ctx->err = "one verdict per distinct value is needed";
      return OBGPU_INVALID_ARGUMENT;
    }
  }
  if (count == 0) return OBGPU_SUCCESS;
  obgpu_ctx *ctx = c.ctx;
  Scratch tmp(ctx);
  tmp.take(64, 64);   // status
  const size_t o_pass = tmp.take((size_t)n_entries + 64, 64), o_out = tmp.take((size_t)count, 64);
  CUDA_TRY(ctx, tmp.alloc());
  uint8_t *base = tmp.p;
  CUDA_TRY(ctx, cudaMemsetAsync(base, 0, 64, ctx->stream));
  if (n_entries) CUDA_TRY(ctx, cudaMemcpyAsync(base + o_pass, entry_pass, (size_t)n_entries, cudaMemcpyHostToDevice, ctx->stream));
  dictops::dict_pass_kernel<<<1, 128, 0, ctx->stream>>>(c.a, block, col, base + o_pass, n_entries, null_pass, start, count, base + o_out, (int *)base);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  int st = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&st, base, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(result_bitmap, base + o_out, (size_t)count, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return check_status(ctx, st);
}

static int group_by_common(obgpu_batch *b, int32_t block0, int32_t n_blocks, int32_t group_col, const obgpu_group_agg *aggs, int32_t n_aggs,
                           const int32_t *row_ids, int64_t row_cap, const uint32_t *d_bitmap, int64_t *host_group_off, int64_t *host_out,
                           int64_t out_cap_groups, int64_t *total_groups) {
  if (!b || block0 < 0 || n_blocks <= 0 || block0 + n_blocks > b->n_blocks || group_col < 0 || (uint32_t)group_col >= b->max_cols ||
      n_aggs < 1 || n_aggs > 16 || !aggs || !host_out || !total_groups)
    return OBGPU_INVALID_ARGUMENT;
  obgpu_ctx *ctx = b->ctx;
  cudaSetDevice(ctx->device);
  dictops::GroupAggs ga{};
  ga.n = n_aggs;
  for (int k = 0; k < n_aggs; ++k) {
    if (aggs[k].kind < OBGPU_AGG_COUNT || aggs[k].kind > OBGPU_AGG_MAX || aggs[k].kind == OBGPU_AGG_SUM_PRODUCT) return OBGPU_NOT_SUPPORTED;
    if (aggs[k].col >= (int32_t)b->max_cols || (aggs[k].col < 0 && aggs[k].kind != OBGPU_AGG_COUNT)) return OBGPU_INVALID_ARGUMENT;
    ga.kind[k] = aggs[k].kind;
    ga.col[k] = aggs[k].col;
  }
  // groups of a block = its dictionary entries + the NULL group: sizes from the plans
  std::vector<ColDesc> plans((size_t)n_blocks);
  CUDA_TRY(ctx, cudaMemcpy2DAsync(plans.data(), sizeof(ColDesc), b->d_plans + (int64_t)block0 * b->max_cols + group_col,
                                  sizeof(ColDesc) * b->max_cols, sizeof(ColDesc), (size_t)n_blocks, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  std::vector<int64_t> goff((size_t)n_blocks + 1, 0);
  for (int32_t i = 0; i < n_blocks; ++i) {
    const ColDesc &d = plans[(size_t)i];
    if (!d.ok || !(d.kind == K_DICT || d.kind == K_RLE || d.kind == K_CONST)) {
      ctx->err = "group-by column is not dictionary coded in every micro block";
      return OBGPU_NOT_SUPPORTED;
    }
    goff[(size_t)i + 1] = goff[(size_t)i] + (int64_t)d.dict_count + 1;
  }
  const int64_t G = goff[(size_t)n_blocks];
  *total_groups = G;
  if (host_group_off) memcpy(host_group_off, goff.data(), ((size_t)n_blocks + 1) * 8);
  if (G > out_cap_groups) return OBGPU_BUF_NOT_ENOUGH;
  Scratch tmp(ctx);
  tmp.take(64, 64);   // status
  const size_t o_goff = tmp.take(((size_t)n_blocks + 1) * 8, 64), o_rid = tmp.take((size_t)(row_ids ? row_cap : 0) * 4, 64);
  const size_t out_bytes = (size_t)n_aggs * (size_t)G * 16, o_out = tmp.take(out_bytes, 64);
  CUDA_TRY(ctx, tmp.alloc());
  uint8_t *base = tmp.p;
  CUDA_TRY(ctx, cudaMemsetAsync(base, 0, o_out + out_bytes, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(base + o_goff, goff.data(), ((size_t)n_blocks + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
  if (row_ids && row_cap > 0) CUDA_TRY(ctx, cudaMemcpyAsync(base + o_rid, row_ids, (size_t)row_cap * 4, cudaMemcpyHostToDevice, ctx->stream));
  unsigned long long *d_out = (unsigned long long *)(base + o_out);
  for (int k = 0; k < n_aggs; ++k)   // MIN starts from the largest key
    if (aggs[k].kind == OBGPU_AGG_MIN) CUDA_TRY(ctx, cudaMemset2DAsync(d_out + (size_t)k * G * 2, 16, 0xff, 8, (size_t)G, ctx->stream));
  const dictops::BlkArgs a{b->d_image, b->d_recs, b->d_plans, (int32_t)b->max_cols};
  dictops::group_by_kernel<<<(unsigned)((n_blocks + 3) / 4), 128, 0, ctx->stream>>>(a, block0, n_blocks, group_col, ga, row_ids ? (const int32_t *)(base + o_rid) : nullptr,
                                                                                 row_cap, d_bitmap, (const int64_t *)(base + o_goff), G, d_out, (int *)base);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  int st = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&st, base, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(host_out, d_out, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (st) return check_status(ctx, st);
  // MIN / MAX: order-preserving keys back to values (sign bit flipped for signed / narrow columns)
  for (int k = 0; k < n_aggs; ++k) {
    if (aggs[k].kind != OBGPU_AGG_MIN && aggs[k].kind != OBGPU_AGG_MAX) continue;
    const uint8_t t = b->col_types[(size_t)aggs[k].col];
    const bool sgn = obf::store_class_of(t) == 1 || obf::datum_len_of(t) < 8;
    for (int64_t g = 0; g < G; ++g) {
      int64_t *o = host_out + ((size_t)k * (size_t)G + (size_t)g) * 2;
      if (!o[1]) { o[0] = 0; continue; }
      if (sgn) o[0] = (int64_t)((uint64_t)o[0] ^ (1ull << 63));
    }
  }
  return OBGPU_SUCCESS;
}

int obgpu_block_group_by(obgpu_batch *b, int32_t block, int32_t group_col, const obgpu_group_agg *aggs, int32_t n_aggs, const int32_t *row_ids,
                         int64_t row_cap, int64_t *host_out, int64_t out_cap_groups, int64_t *n_groups) {
  if (!row_ids || row_cap < 0) return OBGPU_INVALID_ARGUMENT;
  return group_by_common(b, block, 1, group_col, aggs, n_aggs, row_ids, row_cap, nullptr, nullptr, host_out, out_cap_groups, n_groups);
}

int obgpu_result_group_by(obgpu_result *r, int32_t group_col, const obgpu_group_agg *aggs, int32_t n_aggs, int64_t *host_group_off,
                          int64_t *host_out, int64_t out_cap_groups, int64_t *total_groups) {
  if (!r) return OBGPU_INVALID_ARGUMENT;
  {
    obgpu_result_info info;
    const int ret = obgpu_result_info_get(r, &info);   // the scan's own status first
    if (ret != OBGPU_SUCCESS && ret != OBGPU_BUF_NOT_ENOUGH) return ret;
  }
  return group_by_common(r->batch, 0, r->batch->n_blocks, group_col, aggs, n_aggs, nullptr, 0, r->no_filter ? nullptr : r->d_bitmap, host_group_off,
                         host_out, out_cap_groups, total_groups);
}

}  // extern "C"
