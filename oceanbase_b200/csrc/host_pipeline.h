// Host-buffer scan pipeline (include/obgpu_pipeline.h): page batches of a host image flow through n_streams worker
// threads, each with its own obgpu_ctx (= CUDA stream): open (H2D + index kernel) -> scan -> fetch (D2H) through the
// public C-ABI of this library. No CUDA calls of its own.
#pragma once
#include <atomic>
#include <memory>
#include <mutex>
#include <thread>

#include "../../include/obgpu_pipeline.h"

struct obgpu_pipeline {
  int device = 0;
  std::vector<obgpu_ctx *> ctxs;
  std::string err;
  // obgpu_pipeline_top_rows: its rows as a fetch buffer (topn::TopBuf) on ctxs[0], kept for obgpu_pipeline_fetch_top_rows;
  // top_rows < 0: none
  void *d_top = nullptr;
  int64_t top_rows = -1, top_heap = 0;
  int32_t top_n_out = 0;
};

namespace obpipe {

inline void batch_bounds(int32_t n_blocks, int32_t bpb, int32_t ramp, std::vector<int32_t> &bounds) {
  bounds.assign(1, 0);
  int32_t b0 = 0;
  for (int32_t k = ramp; k > 0; --k) {
    const int32_t step = std::max(1, k < 32 ? bpb >> k : 0);   // a shift by 32 or more is undefined: the ramp step is then 1
    if (b0 + step >= n_blocks) break;
    b0 += step;
    bounds.push_back(b0);
  }
  while (b0 < n_blocks) {
    b0 = std::min(n_blocks, b0 + bpb);
    bounds.push_back(b0);
  }
}

inline int32_t default_bpb(const obgpu_host_scan_spec *s) { return s->blocks_per_batch > 0 ? s->blocks_per_batch : std::max(1, s->n_blocks / 12); }

// rows of a block without touching the device: the micro header's row_count_ (ob_micro_block_header.h:97-153)
inline int64_t header_rows(const uint8_t *blk) { uint32_t r; memcpy(&r, blk + 16, 4); return r; }

// compressor_type of a spec: 0 (plain blocks) or one obgpu_batch_open_compressed decodes
inline bool compressor_ok(int32_t c) {
  return c == 0 || c == OBGPU_COMPRESSOR_NONE || c == OBGPU_COMPRESSOR_LZ4 || c == OBGPU_COMPRESSOR_ZLIB || c == OBGPU_COMPRESSOR_ZSTD_1_3_8 ||
         c == OBGPU_COMPRESSOR_LZ4_1_9_1;
}

// opens blocks [b0, b1) of the spec as a page batch (the image rebased to the batch's first block) and attaches their skip
// index; *lo / *hi: the batch's byte range of the image
inline int open_batch(obgpu_ctx *ctx, const obgpu_host_scan_spec *s, int32_t b0, int32_t b1, int64_t *lo, int64_t *hi, obgpu_batch **out) {
  *lo = s->offsets[b0];
  *hi = b1 < s->n_blocks ? s->offsets[b1] : s->image_size;
  std::vector<int64_t> offs((size_t)(b1 - b0));
  for (int32_t i = b0; i < b1; ++i) offs[(size_t)(i - b0)] = s->offsets[i] - *lo;
  const uint8_t *img = (const uint8_t *)s->image + *lo;
  obgpu_batch *batch = nullptr;
  int ret = s->compressor_type ? obgpu_batch_open_compressed(ctx, img, *hi - *lo, offs.data(), s->sizes + b0, b1 - b0, 0, s->compressor_type, &batch)
            : s->zero_copy     ? obgpu_batch_open(ctx, img, *hi - *lo, offs.data(), s->sizes + b0, b1 - b0, 1, img, &batch)   // the pinned host image IS the device image
                               : obgpu_batch_open(ctx, img, *hi - *lo, offs.data(), s->sizes + b0, b1 - b0, 0, nullptr, &batch);
  if (ret != OBGPU_SUCCESS) return ret;
  batch->codes_allowed = false;   // scanned once: batch string codes would cost more than they save
  if (s->agg_rows && s->agg_off) {   // offsets keep their table-wide base: the entry rebases them
    ret = obgpu_batch_set_agg_rows(batch, s->agg_rows, s->agg_off + b0);
    if (ret != OBGPU_SUCCESS) {
      obgpu_batch_close(batch);
      return ret;
    }
  }
  *out = batch;
  return OBGPU_SUCCESS;
}

// what obgpu_pipeline_scan and obgpu_pipeline_group_by refuse alike before any batch is opened
inline int check_source(obgpu_pipeline *p, const obgpu_host_scan_spec *s) {
  if (!compressor_ok(s->compressor_type)) {
    p->err = "compressor_type " + std::to_string(s->compressor_type) + " is not decoded on the device";
    return OBGPU_NOT_SUPPORTED;
  }
  if (s->compressor_type && s->zero_copy) {
    p->err = "zero_copy with a compressor: the decoder reads every stored byte";
    return OBGPU_NOT_SUPPORTED;
  }
  return OBGPU_SUCCESS;
}

inline void add128(int64_t acc[2], int64_t lo, int64_t hi) {
  const uint64_t nlo = (uint64_t)acc[0] + (uint64_t)lo;
  acc[1] = (int64_t)((uint64_t)acc[1] + (uint64_t)hi + (nlo < (uint64_t)acc[0] ? 1u : 0u));
  acc[0] = (int64_t)nlo;
}

}  // namespace obpipe

extern "C" {

int obgpu_pipeline_create(int device, int32_t n_streams, obgpu_pipeline **out) {
  if (!out || n_streams < 1 || n_streams > 16) return OBGPU_INVALID_ARGUMENT;
  obgpu_pipeline *p = new (std::nothrow) obgpu_pipeline();
  if (!p) return OBGPU_ALLOCATE_MEMORY_FAILED;
  p->device = device;
  for (int32_t i = 0; i < n_streams; ++i) {
    obgpu_ctx *c = nullptr;
    const int ret = obgpu_ctx_create(device, &c);
    if (ret != OBGPU_SUCCESS) {
      obgpu_pipeline_destroy(p);
      return ret;
    }
    p->ctxs.push_back(c);
  }
  *out = p;
  return OBGPU_SUCCESS;
}

void obgpu_pipeline_destroy(obgpu_pipeline *p) {
  if (!p) return;
  if (p->d_top) {
    cudaSetDevice(p->device);
    cudaFree(p->d_top);
  }
  for (obgpu_ctx *c : p->ctxs) obgpu_ctx_destroy(c);
  delete p;
}

const char *obgpu_pipeline_last_error(const obgpu_pipeline *p) { return p ? p->err.c_str() : ""; }

int obgpu_pipeline_plan(const obgpu_host_scan_spec *s, int32_t *n_batches, int64_t *rows_cap_needed_hint) {
  if (!s || !n_batches || s->n_blocks <= 0 || !s->image || !s->offsets || !s->sizes) return OBGPU_INVALID_ARGUMENT;
  std::vector<int32_t> bounds;
  obpipe::batch_bounds(s->n_blocks, obpipe::default_bpb(s), std::max(0, s->ramp), bounds);
  *n_batches = (int32_t)bounds.size() - 1;
  if (rows_cap_needed_hint) {
    const double hint = s->selectivity_hint > 0 ? std::min(1.0, s->selectivity_hint) : 1.0;
    int64_t cap = 0;
    for (size_t b = 0; b + 1 < bounds.size(); ++b) {
      int64_t rows = 0;
      for (int32_t i = bounds[b]; i < bounds[b + 1]; ++i) rows += obpipe::header_rows((const uint8_t *)s->image + s->offsets[i]);
      cap += (((int64_t)((double)rows * hint) + 1024) + 63) & ~63ll;
    }
    *rows_cap_needed_hint = cap;
  }
  return OBGPU_SUCCESS;
}

int obgpu_pipeline_scan(obgpu_pipeline *p, const obgpu_host_scan_spec *s, obgpu_host_scan_result *res) {
  if (!p || !s || !res || s->n_blocks <= 0 || !s->image || !s->offsets || !s->sizes || s->n_proj < 0 || s->n_aggs < 0 || s->n_aggs > 16)
    return OBGPU_INVALID_ARGUMENT;
  if (!s->no_row_output && s->n_proj > 0 && (!s->out_data || !s->out_nulls)) return OBGPU_INVALID_ARGUMENT;
  if (const int ret = obpipe::check_source(p, s); ret != OBGPU_SUCCESS) return ret;
  const bool heaps = s->out_heap && !s->no_row_output;
  if (heaps)
    for (int32_t c = 0; c < s->n_proj; ++c)
      if (s->out_heap[c] && !s->out_heap_cap) return OBGPU_INVALID_ARGUMENT;
  std::vector<int32_t> bounds;
  obpipe::batch_bounds(s->n_blocks, obpipe::default_bpb(s), std::max(0, s->ramp), bounds);
  const int32_t nb = (int32_t)bounds.size() - 1;
  if (nb > res->n_batches_cap || !res->batch_row_begin || !res->batch_rows) return OBGPU_BUF_NOT_ENOUGH;
  const double hint = s->selectivity_hint > 0 ? std::min(1.0, s->selectivity_hint) : 1.0;
  // output slices: 64-row aligned so that every slice owns whole NULL words
  std::vector<int64_t> slice_cap((size_t)nb), rows_in((size_t)nb);
  int64_t pos = 0;
  for (int32_t b = 0; b < nb; ++b) {
    int64_t rows = 0;
    for (int32_t i = bounds[(size_t)b]; i < bounds[(size_t)b + 1]; ++i) rows += obpipe::header_rows((const uint8_t *)s->image + s->offsets[i]);
    rows_in[(size_t)b] = rows;
    slice_cap[(size_t)b] = std::min<int64_t>(rows, (int64_t)((double)rows * hint) + 1024);
    res->batch_row_begin[b] = pos;
    if (res->batch_block_begin) res->batch_block_begin[b] = bounds[(size_t)b];
    pos += (slice_cap[(size_t)b] + 63) & ~63ll;
  }
  if (res->batch_block_begin) res->batch_block_begin[nb] = s->n_blocks;
  // row ids are copied out row by row as the projected columns are: a scan that asks for them needs the slices too
  const bool row_output = (!s->no_row_output && s->n_proj > 0) || s->out_row_ids;
  if (row_output && pos > s->out_cap_rows) {
    p->err = "output buffers too small for the planned slices (obgpu_pipeline_plan)";
    return OBGPU_BUF_NOT_ENOUGH;
  }
  res->n_batches = nb;
  res->total_rows = res->selected_rows = 0;
  res->h2d_bytes = res->d2h_bytes = res->kernel_launches = 0;
  memset(res->agg_out, 0, sizeof(res->agg_out));
  for (int a = 0; a < s->n_aggs; ++a)
    if (s->aggs[a].kind == OBGPU_AGG_MIN || s->aggs[a].kind == OBGPU_AGG_MAX) res->agg_out[a][1] = 0;

  std::atomic<int32_t> next{0};
  std::atomic<int64_t> tail{pos};   // spare rows after the planned slices: overflowing batches move there
  std::atomic<int> first_err{OBGPU_SUCCESS};
  std::mutex mu;   // result totals / aggregates / error text
  // heap columns: every batch claims a slice of each heap, as overflowing batches claim tail rows
  std::unique_ptr<std::atomic<int64_t>[]> heap_used(new std::atomic<int64_t>[(size_t)std::max(1, s->n_proj)]);
  for (int32_t c = 0; c < s->n_proj; ++c) heap_used[c] = 0;
  std::vector<int64_t> launches0;
  for (obgpu_ctx *c : p->ctxs) launches0.push_back(obgpu_ctx_launch_count(c));

  auto worker = [&](obgpu_ctx *ctx) {
    for (;;) {
      const int32_t b = next.fetch_add(1);
      if (b >= nb || first_err.load() != OBGPU_SUCCESS) return;
      const int32_t b0 = bounds[(size_t)b], b1 = bounds[(size_t)b + 1];
      int64_t lo = 0, hi = 0;
      obgpu_batch *batch = nullptr;
      obgpu_result *r = nullptr;
      auto fail = [&](int code) {
        int expected = OBGPU_SUCCESS;
        if (first_err.compare_exchange_strong(expected, code)) {
          std::lock_guard<std::mutex> g(mu);
          p->err = obgpu_ctx_last_error(ctx);
        }
        if (r) obgpu_result_free(r);
        if (batch) obgpu_batch_close(batch);
      };
      int ret = obpipe::open_batch(ctx, s, b0, b1, &lo, &hi, &batch);
      if (ret != OBGPU_SUCCESS) { fail(ret); return; }
      std::vector<int32_t> heap_cols;   // projected string columns whose bytes go to a heap
      if (!s->no_row_output) {
        // a string column whose values the device rebuilt (HEX_PACKING / STRING_DIFF / STRING_PREFIX) or decoded (compressed
        // blocks) has no bytes in the caller's image to point at: such projections need a heap
        for (int32_t c = 0; c < s->n_proj; ++c) {
          int32_t obj_type = 0, datum_len = -1, rebuilt = 0;
          const bool is_string = obgpu_batch_column_type(batch, s->proj_cols[c], &obj_type, &datum_len) == OBGPU_SUCCESS && datum_len == 0;
          if (is_string && heaps && s->out_heap[c]) {
            heap_cols.push_back(c);
            continue;
          }
          if (is_string && s->compressor_type) {
            ctx->err = "projected column " + std::to_string(c) + " (store index " + std::to_string(s->proj_cols[c]) +
                       ") is a string column of compressed blocks: give it a heap (out_heap)";
            fail(OBGPU_NOT_SUPPORTED);
            return;
          }
          if (obgpu_batch_column_materialised(batch, s->proj_cols[c], &rebuilt) == OBGPU_SUCCESS && rebuilt) {
            ctx->err = "projected column " + std::to_string(c) +
                       " is HEX_PACKING / STRING_DIFF / STRING_PREFIX coded: give it a heap (out_heap) or use obgpu_result_fetch_strings";
            fail(OBGPU_NOT_SUPPORTED);
            return;
          }
        }
      }
      obgpu_scan_spec spec{};
      spec.filter = s->filter;
      spec.proj_cols = s->proj_cols;
      spec.n_proj = s->n_proj;
      spec.string_base = s->string_base + (uint64_t)lo;   // block offsets were rebased by lo
      spec.want_row_ids = s->out_row_ids ? 1 : 0;
      spec.max_selected_rows = std::max<int64_t>(1, slice_cap[(size_t)b]);
      obgpu_result_info info{};
      ret = obgpu_scan(batch, &spec, &r);
      if (ret == OBGPU_SUCCESS) ret = obgpu_result_info_get(r, &info);
      if (ret == OBGPU_BUF_NOT_ENOUGH && !row_output) {
        // nothing is copied out row by row: re-run with the exact capacity
        obgpu_result_free(r);
        r = nullptr;
        spec.max_selected_rows = info.selected_rows;
        ret = obgpu_scan(batch, &spec, &r);
        if (ret == OBGPU_SUCCESS) ret = obgpu_result_info_get(r, &info);
      }
      if (ret == OBGPU_BUF_NOT_ENOUGH) {
        // the slice planned from the selectivity hint is too small: exact re-run into a slice taken from the tail of the
        // output buffers (batches stay dense; batch_row_begin says where each one landed)
        obgpu_result_free(r);
        r = nullptr;
        const int64_t need = (info.selected_rows + 63) & ~63ll;
        const int64_t start = tail.fetch_add(need);
        if (start + need > s->out_cap_rows) {
          fail(OBGPU_BUF_NOT_ENOUGH);
          return;
        }
        res->batch_row_begin[b] = start;
        spec.max_selected_rows = info.selected_rows;
        ret = obgpu_scan(batch, &spec, &r);
        if (ret == OBGPU_SUCCESS) ret = obgpu_result_info_get(r, &info);
      }
      if (ret != OBGPU_SUCCESS) { fail(ret); return; }
      const int64_t n = info.selected_rows, row0 = res->batch_row_begin[b];
      int64_t d2h = 0;
      if (!s->no_row_output && s->n_proj > 0 && n > 0) {
        const int32_t nh = (int32_t)heap_cols.size();
        std::vector<int64_t> hbytes((size_t)nh), hstart((size_t)nh);
        if (nh > 0) {
          ret = obgpu_result_string_bytes(r, nh, heap_cols.data(), 0, n, hbytes.data());
          if (ret != OBGPU_SUCCESS) { fail(ret); return; }
          for (int32_t j = 0; j < nh; ++j) {
            const int32_t c = heap_cols[(size_t)j];
            hstart[(size_t)j] = heap_used[c].fetch_add(hbytes[(size_t)j]);
            if (hstart[(size_t)j] + hbytes[(size_t)j] > s->out_heap_cap[c]) {
              ctx->err = "string heap of projected column " + std::to_string(c) + " is too small (out_heap_cap)";
              fail(OBGPU_BUF_NOT_ENOUGH);
              return;
            }
          }
        }
        std::vector<int32_t> idx((size_t)s->n_proj);
        std::vector<void *> hd((size_t)s->n_proj), ha((size_t)s->n_proj);
        std::vector<uint64_t *> hn((size_t)s->n_proj);
        for (int32_t c = 0; c < s->n_proj; ++c) {
          obgpu_result_col col{};
          obgpu_result_col_get(r, c, &col);
          idx[(size_t)c] = c;
          hd[(size_t)c] = s->out_data[c] ? (uint8_t *)s->out_data[c] + row0 * (col.is_string ? 8 : col.elem_len) : nullptr;
          ha[(size_t)c] = (col.is_string && s->out_lens && s->out_lens[c]) ? (void *)(s->out_lens[c] + row0) : nullptr;
          hn[(size_t)c] = s->out_nulls[c] ? s->out_nulls[c] + row0 / 64 : nullptr;
          d2h += n * (col.is_string ? 12 : col.elem_len) + (n + 63) / 64 * 8;
        }
        std::vector<void *> hh((size_t)nh);
        std::vector<uint64_t *> hp((size_t)nh);
        for (int32_t j = 0; j < nh; ++j) {   // heap columns: only lengths and NULL words come back here, the pointers below
          const int32_t c = heap_cols[(size_t)j];
          hp[(size_t)j] = (uint64_t *)hd[(size_t)c];
          hd[(size_t)c] = nullptr;
          hh[(size_t)j] = (uint8_t *)s->out_heap[c] + hstart[(size_t)j];
          d2h += hbytes[(size_t)j];
        }
        ret = obgpu_result_fetch_cols(r, s->n_proj, idx.data(), 0, n, hd.data(), ha.data(), hn.data());
        if (ret == OBGPU_SUCCESS && nh > 0) ret = obgpu_result_fetch_string_heap(r, nh, heap_cols.data(), 0, n, hh.data(), hp.data());
        if (ret != OBGPU_SUCCESS) { fail(ret); return; }
      }
      if (s->out_row_ids && n > 0) {
        ret = obgpu_result_fetch_row_ids(r, 0, n, s->out_row_ids + row0);
        if (ret != OBGPU_SUCCESS) { fail(ret); return; }
        d2h += n * 4;
      }
      if (s->out_block_begin && s->out_block_count) {
        std::vector<int64_t> so((size_t)(b1 - b0) + 1);
        ret = obgpu_result_fetch_sel_offsets(r, so.data());
        if (ret != OBGPU_SUCCESS) { fail(ret); return; }
        for (int32_t i = b0; i < b1; ++i) {
          s->out_block_begin[i] = row0 + so[(size_t)(i - b0)];
          s->out_block_count[i] = so[(size_t)(i - b0) + 1] - so[(size_t)(i - b0)];
        }
        d2h += (int64_t)so.size() * 8;
      }
      int64_t agg[16][2];
      for (int a = 0; a < s->n_aggs; ++a) {
        ret = obgpu_result_aggregate(r, s->aggs[a].kind, s->aggs[a].col_a, s->aggs[a].col_b, agg[a]);
        if (ret != OBGPU_SUCCESS) { fail(ret); return; }
        d2h += 16;
      }
      {
        std::lock_guard<std::mutex> g(mu);
        res->batch_rows[b] = n;
        res->total_rows += info.total_rows;
        res->selected_rows += n;
        if (!s->zero_copy) res->h2d_bytes += hi - lo;   // zero copy: the kernels read what they reference, the library copies nothing
        res->d2h_bytes += d2h;
        for (int a = 0; a < s->n_aggs; ++a) {
          const int kind = s->aggs[a].kind;
          if (kind == OBGPU_AGG_MIN || kind == OBGPU_AGG_MAX) {
            if (!agg[a][1]) continue;
            // the C-ABI returns MIN / MAX as a signed or unsigned 64-bit value in the column's own order; the column
            // class is the same for every batch, so comparing in the signed order of the first value seen is not
            // enough for unsigned 64-bit columns: keep both and let obgpu_result_col_get's obj_type decide
            obgpu_result_col col{};
            obgpu_result_col_get(r, s->aggs[a].col_a, &col);
            const bool uns = col.obj_type >= OBGPU_OBJ_UTINYINT && col.obj_type <= OBGPU_OBJ_UINT64;
            bool better = !res->agg_out[a][1];
            if (!better) {
              if (uns) better = kind == OBGPU_AGG_MIN ? (uint64_t)agg[a][0] < (uint64_t)res->agg_out[a][0] : (uint64_t)agg[a][0] > (uint64_t)res->agg_out[a][0];
              else better = kind == OBGPU_AGG_MIN ? agg[a][0] < res->agg_out[a][0] : agg[a][0] > res->agg_out[a][0];
            }
            if (better) { res->agg_out[a][0] = agg[a][0]; res->agg_out[a][1] = 1; }
          } else {
            obpipe::add128(res->agg_out[a], agg[a][0], agg[a][1]);
          }
        }
      }
      obgpu_result_free(r);
      obgpu_batch_close(batch);
    }
  };
  std::vector<std::thread> th;
  for (size_t i = 1; i < p->ctxs.size(); ++i) th.emplace_back(worker, p->ctxs[i]);
  worker(p->ctxs[0]);
  for (auto &t : th) t.join();
  if (s->out_heap_used)
    for (int32_t c = 0; c < s->n_proj; ++c) s->out_heap_used[c] = heap_used[c].load();
  for (size_t i = 0; i < p->ctxs.size(); ++i) {
    obgpu_ctx_synchronize(p->ctxs[i]);
    res->kernel_launches += obgpu_ctx_launch_count(p->ctxs[i]) - launches0[i];
  }
  return first_err.load();
}

}  // extern "C"

namespace obpipe {

// GROUP BY through the pipeline: each worker opens its batch, scans it with nothing projected, groups it with
// group_batch(result, &n_groups, &key_bytes) and adds the groups to one accumulator under the mutex
template <class GroupBatch>
static int group_by(obgpu_pipeline *p, const obgpu_host_scan_spec *s, const int32_t *group_cols, int32_t n_group_cols,
                    const obgpu_group_agg *aggs, int32_t n_aggs, obgpu_host_scan_result *res, obgpu_groups **out, GroupBatch group_batch) {
  if (!p || !s || !res || !out || s->n_blocks <= 0 || !s->image || !s->offsets || !s->sizes || !group_cols || n_group_cols < 1 ||
      n_group_cols > gvals::kMaxGroupCols || !aggs || n_aggs < 1 || n_aggs > 16)
    return OBGPU_INVALID_ARGUMENT;
  *out = nullptr;
  if (!s->no_row_output || s->out_row_ids || s->out_block_begin || s->out_block_count || s->n_aggs != 0) {
    p->err = "a GROUP BY through the pipeline returns groups only: no_row_output 1, no row ids, block tables or scalar aggregates";
    return OBGPU_INVALID_ARGUMENT;
  }
  if (const int ret = obpipe::check_source(p, s); ret != OBGPU_SUCCESS) return ret;
  std::vector<int32_t> bounds;
  obpipe::batch_bounds(s->n_blocks, obpipe::default_bpb(s), std::max(0, s->ramp), bounds);
  const int32_t nb = (int32_t)bounds.size() - 1;
  if (nb > res->n_batches_cap || !res->batch_row_begin || !res->batch_rows) return OBGPU_BUF_NOT_ENOUGH;
  obgpu_groups *acc = nullptr;
  if (const int ret = obgpu_groups_create(p->ctxs[0], n_group_cols, aggs, n_aggs, &acc); ret != OBGPU_SUCCESS) {
    p->err = obgpu_ctx_last_error(p->ctxs[0]);
    return ret;
  }
  for (int32_t b = 0; b < nb; ++b) {
    res->batch_row_begin[b] = 0;
    if (res->batch_block_begin) res->batch_block_begin[b] = bounds[(size_t)b];
  }
  if (res->batch_block_begin) res->batch_block_begin[nb] = s->n_blocks;
  res->n_batches = nb;
  res->total_rows = res->selected_rows = 0;
  res->h2d_bytes = res->d2h_bytes = res->kernel_launches = 0;
  memset(res->agg_out, 0, sizeof(res->agg_out));

  std::atomic<int32_t> next{0};
  std::atomic<int> first_err{OBGPU_SUCCESS};
  std::mutex mu;   // the accumulator, result totals, error text
  std::vector<int64_t> launches0;
  for (obgpu_ctx *c : p->ctxs) launches0.push_back(obgpu_ctx_launch_count(c));

  auto worker = [&](obgpu_ctx *ctx) {
    for (;;) {
      const int32_t b = next.fetch_add(1);
      if (b >= nb || first_err.load() != OBGPU_SUCCESS) return;
      int64_t lo = 0, hi = 0;
      obgpu_batch *batch = nullptr;
      obgpu_result *r = nullptr;
      obgpu_result_info info{};
      int ret = obpipe::open_batch(ctx, s, bounds[(size_t)b], bounds[(size_t)b + 1], &lo, &hi, &batch);
      if (ret == OBGPU_SUCCESS) {
        obgpu_scan_spec spec{};   // nothing projected; the capacity is the batch's rows
        spec.filter = s->filter;
        ret = obgpu_scan(batch, &spec, &r);
      }
      if (ret == OBGPU_SUCCESS) ret = obgpu_result_info_get(r, &info);
      int64_t ng = 0, kb = 0;
      if (ret == OBGPU_SUCCESS) ret = group_batch(r, &ng, &kb);
      if (ret == OBGPU_SUCCESS) {
        std::lock_guard<std::mutex> g(mu);
        if (first_err.load() == OBGPU_SUCCESS) ret = obgpu_groups_add(acc, r);
        if (ret == OBGPU_SUCCESS) {
          res->batch_rows[b] = info.selected_rows;
          res->total_rows += info.total_rows;
          res->selected_rows += info.selected_rows;
          if (!s->zero_copy) res->h2d_bytes += hi - lo;   // zero copy: the kernels read what they reference, the library copies nothing
        }
      }
      if (ret != OBGPU_SUCCESS) {
        int expected = OBGPU_SUCCESS;
        if (first_err.compare_exchange_strong(expected, ret)) {
          std::lock_guard<std::mutex> g(mu);
          p->err = obgpu_ctx_last_error(ctx);
        }
      }
      if (r) obgpu_result_free(r);
      if (batch) obgpu_batch_close(batch);
      if (ret != OBGPU_SUCCESS) return;
    }
  };
  std::vector<std::thread> th;
  for (size_t i = 1; i < p->ctxs.size(); ++i) th.emplace_back(worker, p->ctxs[i]);
  worker(p->ctxs[0]);
  for (auto &t : th) t.join();
  for (size_t i = 0; i < p->ctxs.size(); ++i) {
    obgpu_ctx_synchronize(p->ctxs[i]);
    res->kernel_launches += obgpu_ctx_launch_count(p->ctxs[i]) - launches0[i];
  }
  if (first_err.load() != OBGPU_SUCCESS) {
    obgpu_groups_free(acc);
    return first_err.load();
  }
  *out = acc;
  return OBGPU_SUCCESS;
}

}  // namespace obpipe

extern "C" {

int obgpu_pipeline_group_by(obgpu_pipeline *p, const obgpu_host_scan_spec *s, const int32_t *group_cols, int32_t n_group_cols,
                            const obgpu_group_agg *aggs, int32_t n_aggs, obgpu_host_scan_result *res, obgpu_groups **out) {
  return obpipe::group_by(p, s, group_cols, n_group_cols, aggs, n_aggs, res, out, [&](obgpu_result *r, int64_t *ng, int64_t *kb) {
    return obgpu_result_group_by_columns(r, group_cols, n_group_cols, aggs, n_aggs, ng, kb);
  });
}

int obgpu_pipeline_group_by_any(obgpu_pipeline *p, const obgpu_host_scan_spec *s, const int32_t *group_cols, int32_t n_group_cols,
                                const obgpu_group_agg *aggs, int32_t n_aggs, obgpu_host_scan_result *res, obgpu_groups **out,
                                int32_t *cells_batches) {
  std::atomic<int32_t> cells{0};
  const int ret = obpipe::group_by(p, s, group_cols, n_group_cols, aggs, n_aggs, res, out, [&](obgpu_result *r, int64_t *ng, int64_t *kb) {
    int32_t path = 0;
    const int gr = obgpu_result_group_by_any(r, group_cols, n_group_cols, aggs, n_aggs, ng, kb, &path);
    if (path == OBGPU_GROUP_PATH_CELLS) cells.fetch_add(1);
    return gr;
  });
  if (cells_batches) *cells_batches = ret == OBGPU_SUCCESS ? cells.load() : 0;
  return ret;
}

int obgpu_pipeline_top_rows(obgpu_pipeline *p, const obgpu_host_scan_spec *s, const obgpu_sort_key *keys, int32_t n_keys,
                            const int32_t *out_cols, int32_t n_out, int64_t k, obgpu_host_scan_result *res, int64_t *n_rows,
                            int64_t *heap_bytes) {
  if (!p) return OBGPU_INVALID_ARGUMENT;
  cudaSetDevice(p->device);
  if (p->d_top) cudaFree(p->d_top);   // a refused call leaves no rows
  p->d_top = nullptr;
  p->top_rows = -1;
  p->top_heap = 0;
  p->top_n_out = 0;
  if (!s || !res || s->n_blocks <= 0 || !s->image || !s->offsets || !s->sizes) return OBGPU_INVALID_ARGUMENT;
  if (const int a = topn::check_args(keys, n_keys, out_cols, n_out, k, n_rows, heap_bytes, 1u << 30); a != OBGPU_SUCCESS) {
    if (a == OBGPU_NOT_SUPPORTED) p->err = "top rows: k above 65536";
    return a;
  }
  if (!s->no_row_output || s->out_row_ids || s->out_block_begin || s->out_block_count || s->n_aggs != 0) {
    p->err = "top rows through the pipeline return rows only: no_row_output 1, no row ids, block tables or scalar aggregates";
    return OBGPU_INVALID_ARGUMENT;
  }
  if (const int ret = obpipe::check_source(p, s); ret != OBGPU_SUCCESS) return ret;
  std::vector<int32_t> bounds;
  obpipe::batch_bounds(s->n_blocks, obpipe::default_bpb(s), std::max(0, s->ramp), bounds);
  const int32_t nb = (int32_t)bounds.size() - 1;
  if (nb > res->n_batches_cap || !res->batch_row_begin || !res->batch_rows) return OBGPU_BUF_NOT_ENOUGH;
  for (int32_t b = 0; b < nb; ++b) {
    res->batch_row_begin[b] = 0;
    if (res->batch_block_begin) res->batch_block_begin[b] = bounds[(size_t)b];
  }
  if (res->batch_block_begin) res->batch_block_begin[nb] = s->n_blocks;
  res->n_batches = nb;
  res->total_rows = res->selected_rows = 0;
  res->h2d_bytes = res->d2h_bytes = res->kernel_launches = 0;
  memset(res->agg_out, 0, sizeof(res->agg_out));
  topn::Key key[topn::kMaxKeys]{};
  for (int i = 0; i < n_keys; ++i) key[i] = topn::Key{keys[i].col, keys[i].desc ? 1 : 0, keys[i].nulls_first ? 1 : 0, 0};

  std::atomic<int32_t> next{0};
  std::atomic<int> first_err{OBGPU_SUCCESS};
  std::mutex mu;   // the merged set, its column facts, result totals, error text
  topn::TopSet acc;                 // the rows so far, positions table-wide; one ctx's memory, complete whenever mu is free
  obgpu_ctx *acc_ctx = nullptr;
  bool have = false;                // a batch has set the column facts below
  uint32_t str_mask = 0, sgn_mask = 0;
  int32_t types[topn::kMaxKeys + topn::kMaxOut] = {0}, col_str[topn::kMaxKeys + topn::kMaxOut] = {0};
  std::vector<int64_t> launches0;
  for (obgpu_ctx *c : p->ctxs) launches0.push_back(obgpu_ctx_launch_count(c));

  auto worker = [&](obgpu_ctx *ctx) {
    for (;;) {
      const int32_t b = next.fetch_add(1);
      if (b >= nb || first_err.load() != OBGPU_SUCCESS) return;
      int64_t lo = 0, hi = 0;
      obgpu_batch *batch = nullptr;
      obgpu_result *r = nullptr;
      obgpu_result_info info{};
      int ret = obpipe::open_batch(ctx, s, bounds[(size_t)b], bounds[(size_t)b + 1], &lo, &hi, &batch);
      if (ret == OBGPU_SUCCESS) {
        obgpu_scan_spec spec{};   // nothing projected; the capacity is the batch's rows
        spec.filter = s->filter;
        ret = obgpu_scan(batch, &spec, &r);
      }
      if (ret == OBGPU_SUCCESS) ret = obgpu_result_info_get(r, &info);
      int64_t nr = 0, hb = 0;
      if (ret == OBGPU_SUCCESS) ret = obgpu_result_top_rows(r, keys, n_keys, out_cols, n_out, k, &nr, &hb);
      if (ret == OBGPU_SUCCESS) {
        std::lock_guard<std::mutex> g(mu);
        const int n_cols = n_keys + n_out;
        if (!have) {
          have = true;
          str_mask = r->top_str;
          sgn_mask = r->top_sgn;
          for (int c = 0; c < n_cols; ++c) types[c] = r->tset_types[c];
        } else if (r->top_str != str_mask || r->top_sgn != sgn_mask || memcmp(types, r->tset_types, sizeof(int32_t) * (size_t)n_cols) != 0) {
          ctx->err = "top rows: a key or output column has another obj_type in another page batch";
          ret = OBGPU_NOT_SUPPORTED;
        }
        if (ret == OBGPU_SUCCESS && first_err.load() == OBGPU_SUCCESS) {
          const topn::TopSet bs = topn::set_of(r);
          for (int c = 0; c < n_cols; ++c) {
            const int sc = obf::store_class_of((uint8_t)types[c]);
            col_str[c] = sc == 5;
            if (c < n_keys) key[c].str = sc == 5;
          }
          // acc (table-wide positions) and this batch's rows (blocks + the batch's first block), k kept; synchronous, so that
          // acc is complete for the next worker and the result may go
          topn::TopSet merged;
          ret = topn::order_sets(ctx, acc, bs, (uint64_t)bounds[(size_t)b], n_keys, key, col_str, k, merged);
          if (ret == OBGPU_SUCCESS && cudaStreamSynchronize(ctx->stream) != cudaSuccess) {
            ctx->err = "top rows: the merge failed";
            ret = OBGPU_ERR_SYS;
          }
          if (ret == OBGPU_SUCCESS) {
            if (acc.mem) topn::free_set(ctx, acc);   // acc_ctx's work on it finished before it was released
            acc = merged;
            acc_ctx = ctx;
            res->batch_rows[b] = info.selected_rows;
            res->total_rows += info.total_rows;
            res->selected_rows += info.selected_rows;
            if (!s->zero_copy) res->h2d_bytes += hi - lo;
          } else {
            topn::free_set(ctx, merged);
          }
        }
      }
      if (ret != OBGPU_SUCCESS) {
        int expected = OBGPU_SUCCESS;
        if (first_err.compare_exchange_strong(expected, ret)) {
          std::lock_guard<std::mutex> g(mu);
          p->err = obgpu_ctx_last_error(ctx);
        }
      }
      if (r) obgpu_result_free(r);
      if (batch) obgpu_batch_close(batch);
      if (ret != OBGPU_SUCCESS) return;
    }
  };
  std::vector<std::thread> th;
  for (size_t i = 1; i < p->ctxs.size(); ++i) th.emplace_back(worker, p->ctxs[i]);
  worker(p->ctxs[0]);
  for (auto &t : th) t.join();
  for (size_t i = 0; i < p->ctxs.size(); ++i) obgpu_ctx_synchronize(p->ctxs[i]);
  int ret = first_err.load();
  obgpu_ctx *c0 = p->ctxs[0];
  if (ret == OBGPU_SUCCESS) {   // no batch selected a row: the set is empty
    void *buf = nullptr;
    int64_t heap = 0;
    ret = topn::emit(c0, acc, n_keys, n_out, str_mask, sgn_mask, &buf, &heap);
    if (ret == OBGPU_SUCCESS) {
      p->d_top = buf;
      p->top_rows = acc.n;
      p->top_heap = heap;
      p->top_n_out = n_out;
      *n_rows = acc.n;
      *heap_bytes = heap;
    } else {
      p->err = obgpu_ctx_last_error(c0);
    }
  }
  if (acc.mem) topn::free_set(c0, acc);
  for (size_t i = 0; i < p->ctxs.size(); ++i) {
    obgpu_ctx_synchronize(p->ctxs[i]);
    res->kernel_launches += obgpu_ctx_launch_count(p->ctxs[i]) - launches0[i];
  }
  (void)acc_ctx;
  return ret;
}

int obgpu_pipeline_fetch_top_rows(obgpu_pipeline *p, int32_t *host_block, int32_t *host_row, int64_t *host_vals, uint8_t *host_nulls,
                                  void *host_heap) {
  if (!p || p->top_rows < 0 || !host_block || !host_row || (p->top_n_out > 0 && (!host_vals || !host_nulls)) || (p->top_heap > 0 && !host_heap))
    return OBGPU_INVALID_ARGUMENT;
  cudaSetDevice(p->device);
  const int ret = topn::fetch(p->ctxs[0], p->d_top, p->top_rows, p->top_n_out, p->top_heap, host_block, host_row, host_vals, host_nulls, host_heap);
  if (ret != OBGPU_SUCCESS) p->err = obgpu_ctx_last_error(p->ctxs[0]);
  return ret;
}

}  // extern "C"
