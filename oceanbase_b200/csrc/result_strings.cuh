// Bytes of projected string cells as a dense heap: obgpu_result_fetch_strings (the selected rows of a scan) and
// obgpu_project_strings (one block, a row list). Needed for the columns whose values exist only on the device -- HEX_PACKING /
// STRING_DIFF / STRING_PREFIX, rebuilt at batch open (mat_codecs.cuh) -- and usable for every string column (the caller then gets
// bytes instead of pointers into its own image). Same pattern as the merge's string materialisation: lengths -> exclusive scan ->
// one warp per row copies the cell.
#pragma once

namespace resstr {

// The string columns one pass covers. Entry k of a pass over n columns and `rows` rows is row k % rows of column k / rows: the
// columns' cells form one concatenated array, so one launch and one prefix serve every column.
struct Cols {
  const uint64_t *ptrs[kMaxProj];    // projected pointers (string_base + cell offset in the caller's image)
  const int32_t *lens[kMaxProj];     // <= 0 for NULL rows
  const uint32_t *nulls[kMaxProj];   // NULL bits over the dense rows
  uint64_t host_base[kMaxProj];      // gather with row pointers: host address of the column's heap minus the column's first byte offset
};

// where the cell of every entry starts inside the batch's device image: the block of a dense output row by binary search in the
// per-block prefix, the cell offset from the pointer the projection reported (string_base + the block's place in the caller's image).
// Also writes the entry's length (0 for NULL rows) into cat_len, the input of the prefix.
__global__ void __launch_bounds__(256) src_off_kernel(Cols c, int64_t row_begin, int64_t rows, int64_t n,
                                                      const int64_t *__restrict__ sel_offset, int n_blocks, const BlockRec *__restrict__ recs,
                                                      const obcs::XformRec *__restrict__ xf, uint64_t string_base, uint64_t *__restrict__ src_off,
                                                      int32_t *__restrict__ cat_len, int *__restrict__ status) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int64_t j = k / rows;
  const int64_t row = row_begin + (k - j * rows);
  const int32_t len = c.lens[j][row];
  src_off[k] = 0;
  cat_len[k] = len > 0 ? len : 0;
  if (len <= 0) return;
  int lo = 0, hi = n_blocks;   // last block whose first output row is <= row
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (sel_offset[mid] <= row) lo = mid; else hi = mid;
  }
  const BlockRec rec = recs[lo];
  const uint64_t base = string_base + (xf ? xf[lo].orig_off + (uint64_t)xf[lo].str_delta : rec.off);
  const uint64_t cell = c.ptrs[j][row] - base;
  if (cell + (uint64_t)len > (uint64_t)rec.size) { atomicOr(status, ST_CORRUPT); return; }
  src_off[k] = rec.off + cell;
}

// one warp per entry copies its cell to heap + off[k]. row_ptrs != nullptr: lane 0 also writes the entry's final host address,
// c.host_base[column] + off[k], or 0 for a NULL row (c.nulls; rows / row_begin place the entry in its column)
__global__ void __launch_bounds__(256) gather_kernel(const uint8_t *__restrict__ image, const uint64_t *__restrict__ src_off,
                                                     const int32_t *__restrict__ lens, int64_t n, const int64_t *__restrict__ off,
                                                     uint8_t *__restrict__ heap, Cols c, int64_t row_begin, int64_t rows,
                                                     uint64_t *__restrict__ row_ptrs) {
  const int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (k >= n) return;
  const int32_t len = lens[k];
  const int64_t o = off[k];
  if (row_ptrs && lane == 0) {
    const int64_t j = k / rows;
    const int64_t row = row_begin + (k - j * rows);
    const bool is_null = (c.nulls[j][row >> 5] >> (row & 31)) & 1u;
    row_ptrs[k] = is_null ? 0 : c.host_base[j] + (uint64_t)o;
  }
  if (len <= 0) return;
  const uint8_t *src = image + src_off[k];
  uint8_t *dst = heap + o;
  for (int32_t i = lane; i < len; i += 32) dst[i] = src[i];
}

// device buffer of a pass over n entries, reserved in s: status word, source offsets, lengths, byte offsets (n + 1), prefix chunk totals
struct Layout {
  size_t o_src, o_len, o_off, o_chunk;
  Layout(Scratch &s, int64_t n) {
    s.take(256);
    o_src = s.take((size_t)n * 8);
    o_len = s.take((size_t)n * 4);
    o_off = s.take(((size_t)n + 1) * 8);
    o_chunk = s.take(((size_t)(n / kPrefixChunk) + 3) * 8);
  }
};

}  // namespace resstr

namespace {

// lens (device, int32, 0 for NULL rows) -> exclusive prefix off[n + 1] in scratch + o_off: two launches
void prefix_lens(obgpu_ctx *ctx, const int32_t *d_lens, int64_t n, uint8_t *scratch, size_t o_off, size_t o_chunk) {
  const int n_chunks = (int)((n + kPrefixChunk - 1) / kPrefixChunk);
  int64_t *d_off = (int64_t *)(scratch + o_off);
  obgpu_prefix_local_kernel<<<n_chunks, 256, 0, ctx->stream>>>((const uint32_t *)d_lens, (int)n, d_off, (unsigned long long *)(scratch + o_chunk));
  obgpu_prefix_fix_kernel<<<n_chunks + 1, 256, 0, ctx->stream>>>((int)n, n_chunks, d_off, (const unsigned long long *)(scratch + o_chunk));
  ctx->launches += 2;
}

// lens (device, int32, 0 for NULL rows) + src offsets (device) -> host offsets [n + 1] and heap
int gather_to_host(obgpu_ctx *ctx, const uint8_t *d_image, const uint64_t *d_src_off, const int32_t *d_lens, int64_t n, void *host_heap,
                   int64_t heap_cap, int64_t *host_off, int64_t *heap_bytes, uint8_t *scratch, size_t o_off, size_t o_chunk) {
  prefix_lens(ctx, d_lens, n, scratch, o_off, o_chunk);
  const int64_t *d_off = (const int64_t *)(scratch + o_off);
  CUDA_TRY(ctx, cudaMemcpyAsync(host_off, d_off, ((size_t)n + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  const int64_t total = host_off[n];
  *heap_bytes = total;
  if (total > heap_cap || (total > 0 && !host_heap)) return OBGPU_BUF_NOT_ENOUGH;
  if (total == 0) return OBGPU_SUCCESS;
  Scratch heap(ctx);
  CUDA_TRY(ctx, heap.alloc((size_t)total + 16));
  resstr::gather_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, ctx->stream>>>(d_image, d_src_off, d_lens, n, d_off, heap.p, resstr::Cols{}, 0,
                                                                                   n, nullptr);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  CUDA_TRY(ctx, cudaMemcpyAsync(host_heap, heap.p, (size_t)total, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return OBGPU_SUCCESS;
}

// checks of a string call over projected columns cols[0..n) and rows [row_begin, row_begin + row_count) of a scan; fills the
// pass's column table
int string_cols(obgpu_result *r, int32_t n, const int32_t *cols, int64_t row_begin, int64_t row_count, resstr::Cols *tab) {
  if (!r || n < 1 || n > kMaxProj || !cols || row_begin < 0 || row_count < 0 || row_begin + row_count > r->cap) return OBGPU_INVALID_ARGUMENT;
  obgpu_ctx *ctx = r->ctx;
  if ((int64_t)n * row_count >= (int64_t)INT32_MAX) { ctx->err = "too many string cells for one call"; return OBGPU_INVALID_ARGUMENT; }
  for (int32_t j = 0; j < n; ++j) {
    if (cols[j] < 0 || cols[j] >= r->n_proj) return OBGPU_INVALID_ARGUMENT;
    const ResultCol &c = r->cols[cols[j]];
    if (!c.is_string) { ctx->err = "not a string column"; return OBGPU_INVALID_ARGUMENT; }
    tab->ptrs[j] = (const uint64_t *)c.data;
    tab->lens[j] = c.lens;
    tab->nulls[j] = c.nulls;
  }
  obgpu_result_info info;
  const int ret = obgpu_result_info_get(r, &info);
  if (ret != OBGPU_SUCCESS) return ret;
  if (row_begin + row_count > info.selected_rows) return OBGPU_INVALID_ARGUMENT;
  return OBGPU_SUCCESS;
}

// the src-offset launch of a pass over n columns x rows rows into scratch t (laid out by resstr::Layout)
int launch_src_off(obgpu_result *r, const resstr::Cols &tab, int64_t row_begin, int64_t rows, int64_t n, uint8_t *t, const resstr::Layout &L) {
  obgpu_ctx *ctx = r->ctx;
  obgpu_batch *b = r->batch;
  CUDA_TRY(ctx, cudaMemsetAsync(t, 0, 256, ctx->stream));
  resstr::src_off_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(tab, row_begin, rows, n, r->d_sel_offset, b->n_blocks, b->d_recs, b->d_xf,
                                                                              r->string_base, (uint64_t *)(t + L.o_src), (int32_t *)(t + L.o_len),
                                                                              (int *)t);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  return OBGPU_SUCCESS;
}

}  // namespace

extern "C" {

int obgpu_batch_column_materialised(const obgpu_batch *b, int32_t col, int32_t *materialised) {
  if (!b || !materialised || col < 0 || (size_t)col >= b->col_mat.size()) return OBGPU_INVALID_ARGUMENT;
  *materialised = b->col_mat[(size_t)col];
  return OBGPU_SUCCESS;
}

int obgpu_result_fetch_strings(obgpu_result *r, int32_t i, int64_t row_begin, int64_t row_count, void *host_heap, int64_t heap_cap,
                               int64_t *host_off, int64_t *heap_bytes) {
  if (!r || i < 0 || i >= r->n_proj || !host_off || !heap_bytes) return OBGPU_INVALID_ARGUMENT;
  resstr::Cols tab{};
  int ret = string_cols(r, 1, &i, row_begin, row_count, &tab);
  if (ret != OBGPU_SUCCESS) return ret;
  obgpu_ctx *ctx = r->ctx;
  cudaSetDevice(ctx->device);
  host_off[0] = 0;
  *heap_bytes = 0;
  if (row_count == 0) return OBGPU_SUCCESS;
  const int64_t n = row_count;
  Scratch tmp(ctx);
  const resstr::Layout L(tmp, n);
  CUDA_TRY(ctx, tmp.alloc());
  uint8_t *t = tmp.p;
  ret = launch_src_off(r, tab, row_begin, n, n, t, L);
  if (ret != OBGPU_SUCCESS) return ret;
  ret = gather_to_host(ctx, r->batch->d_image, (const uint64_t *)(t + L.o_src), (const int32_t *)(t + L.o_len), n, host_heap, heap_cap, host_off,
                       heap_bytes, t, L.o_off, L.o_chunk);
  if (ret != OBGPU_SUCCESS) return ret;
  int st = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&st, t, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return check_status(ctx, st);
}

int obgpu_result_string_bytes(obgpu_result *r, int32_t n, const int32_t *cols, int64_t row_begin, int64_t row_count, int64_t *bytes) {
  if (!bytes) return OBGPU_INVALID_ARGUMENT;
  resstr::Cols tab{};
  int ret = string_cols(r, n, cols, row_begin, row_count, &tab);
  if (ret != OBGPU_SUCCESS) return ret;
  obgpu_ctx *ctx = r->ctx;
  cudaSetDevice(ctx->device);
  r->str_n = 0;   // no fetch may follow a failed call
  if (r->d_str) {
    cudaFreeAsync(r->d_str, ctx->stream);
    r->d_str = nullptr;
  }
  const int64_t m = (int64_t)n * row_count;
  std::fill(r->str_col_off, r->str_col_off + n + 1, 0);
  if (m > 0) {
    Scratch str(ctx);
    const resstr::Layout L(str, m);
    CUDA_TRY(ctx, str.alloc());
    uint8_t *t = str.p;
    ret = launch_src_off(r, tab, row_begin, row_count, m, t, L);
    if (ret != OBGPU_SUCCESS) return ret;
    prefix_lens(ctx, (const int32_t *)(t + L.o_len), m, t, L.o_off, L.o_chunk);
    // the only values that come back: the status word and each column's first byte offset (+ the grand total)
    const int64_t *d_off = (const int64_t *)(t + L.o_off);
    int st = 0;
    CUDA_TRY(ctx, cudaMemcpyAsync(&st, t, 4, cudaMemcpyDeviceToHost, ctx->stream));
    for (int32_t j = 0; j <= n; ++j)
      CUDA_TRY(ctx, cudaMemcpyAsync(&r->str_col_off[j], d_off + (int64_t)j * row_count, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    ret = check_status(ctx, st);
    if (ret != OBGPU_SUCCESS) return ret;
    r->d_str = str.release();
  }
  for (int32_t j = 0; j < n; ++j) {
    bytes[j] = r->str_col_off[j + 1] - r->str_col_off[j];
    r->str_cols[j] = cols[j];
  }
  r->str_n = n;
  r->str_row_begin = row_begin;
  r->str_rows = row_count;
  return OBGPU_SUCCESS;
}

int obgpu_result_fetch_string_heap(obgpu_result *r, int32_t n, const int32_t *cols, int64_t row_begin, int64_t row_count,
                                   void *const *host_heap, uint64_t *const *host_ptrs) {
  if (!r || !cols || !host_heap) return OBGPU_INVALID_ARGUMENT;
  obgpu_ctx *ctx = r->ctx;
  bool same = n == r->str_n && n > 0 && row_begin == r->str_row_begin && row_count == r->str_rows;
  for (int32_t j = 0; same && j < n; ++j) same = cols[j] == r->str_cols[j];
  if (!same) { ctx->err = "columns / rows differ from the last obgpu_result_string_bytes call"; return OBGPU_INVALID_ARGUMENT; }
  const int64_t m = (int64_t)n * row_count;
  if (m == 0) return OBGPU_SUCCESS;
  resstr::Cols tab{};
  bool want_ptrs = false;
  for (int32_t j = 0; j < n; ++j) {
    const int64_t bytes = r->str_col_off[j + 1] - r->str_col_off[j];
    if (bytes > 0 && !host_heap[j]) return OBGPU_INVALID_ARGUMENT;
    tab.nulls[j] = r->cols[cols[j]].nulls;
    tab.host_base[j] = (uint64_t)(uintptr_t)host_heap[j] - (uint64_t)r->str_col_off[j];
    want_ptrs = want_ptrs || (host_ptrs && host_ptrs[j]);
  }
  cudaSetDevice(ctx->device);
  Scratch str(ctx);   // only sized: r->d_str has this layout
  const resstr::Layout L(str, m);
  const uint8_t *t = (const uint8_t *)r->d_str;
  const int64_t total = r->str_col_off[n] - r->str_col_off[0];
  Scratch tmp(ctx);   // the heap, then the pointer table
  const size_t o_heap = tmp.take((size_t)total + 16, 8), o_ptrs = want_ptrs ? tmp.take((size_t)m * 8, 8) : 0;
  CUDA_TRY(ctx, tmp.alloc());
  uint8_t *d_heap = tmp.at<uint8_t>(o_heap);
  uint64_t *d_ptrs = want_ptrs ? tmp.at<uint64_t>(o_ptrs) : nullptr;
  resstr::gather_kernel<<<(unsigned)((m * 32 + 255) / 256), 256, 0, ctx->stream>>>(
      r->batch->d_image, (const uint64_t *)(t + L.o_src), (const int32_t *)(t + L.o_len), m, (const int64_t *)(t + L.o_off), d_heap, tab,
      row_begin, row_count, d_ptrs);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  for (int32_t j = 0; j < n; ++j) {
    const int64_t bytes = r->str_col_off[j + 1] - r->str_col_off[j];
    if (bytes > 0)
      CUDA_TRY(ctx, cudaMemcpyAsync(host_heap[j], d_heap + r->str_col_off[j], (size_t)bytes, cudaMemcpyDeviceToHost, ctx->stream));
    if (host_ptrs && host_ptrs[j])
      CUDA_TRY(ctx, cudaMemcpyAsync(host_ptrs[j], d_ptrs + (int64_t)j * row_count, (size_t)row_count * 8, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return OBGPU_SUCCESS;
}

int obgpu_project_strings(obgpu_batch *b, int32_t block, int32_t col, const int32_t *row_ids, int64_t row_cap, void *host_heap, int64_t heap_cap,
                          int64_t *host_off, uint64_t *host_nulls, int32_t *has_null, int64_t *heap_bytes) {
  if (!b || !row_ids || row_cap < 0 || !host_off || !heap_bytes || block < 0 || block >= b->n_blocks) return OBGPU_INVALID_ARGUMENT;
  obgpu_ctx *ctx = b->ctx;
  host_off[0] = 0;
  *heap_bytes = 0;
  if (row_cap == 0) return OBGPU_SUCCESS;
  // the ordinary discrete projection with string_base 0 reports every cell at (the block's place in the caller's image) + cell
  std::vector<uint64_t> ptrs((size_t)row_cap, 0), nulls((size_t)(row_cap + 63) / 64, 0);
  std::vector<int32_t> lens((size_t)row_cap, 0);
  int32_t hn = 0;
  int ret = obgpu_project_discrete(b, block, col, row_ids, row_cap, 0, 0, ptrs.data(), lens.data(), nulls.data(), &hn);
  if (ret != OBGPU_SUCCESS) return ret;
  if (host_nulls) memcpy(host_nulls, nulls.data(), nulls.size() * 8);
  if (has_null) *has_null = hn;
  uint64_t base = (uint64_t)b->offsets[(size_t)block];
  if (b->d_xf) {
    obcs::XformRec x;
    CUDA_TRY(ctx, cudaMemcpyAsync(&x, b->d_xf + block, sizeof(x), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    base = x.orig_off + (uint64_t)x.str_delta;
  }
  for (int64_t k = 0; k < row_cap; ++k) {
    const bool is_null = (nulls[(size_t)k / 64] >> (k % 64)) & 1ull;
    if (is_null) { lens[(size_t)k] = 0; ptrs[(size_t)k] = 0; continue; }
    const uint64_t cell = ptrs[(size_t)k] - base;
    if (cell + (uint64_t)lens[(size_t)k] > (uint64_t)b->sizes[(size_t)block]) { ctx->err = "string cell outside its micro block"; return OBGPU_INVALID_DATA; }
    ptrs[(size_t)k] = (uint64_t)b->offsets[(size_t)block] + cell;   // offset inside the batch's device image
  }
  const int64_t n = row_cap;
  Scratch tmp(ctx);
  const size_t o_src = tmp.take((size_t)n * 8), o_len = tmp.take((size_t)n * 4), o_off = tmp.take(((size_t)n + 1) * 8);
  const size_t o_chunk = tmp.take(((size_t)(n / kPrefixChunk) + 3) * 8);
  CUDA_TRY(ctx, tmp.alloc());
  uint8_t *t = tmp.p;
  CUDA_TRY(ctx, cudaMemcpyAsync(t + o_src, ptrs.data(), (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(t + o_len, lens.data(), (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
  return gather_to_host(ctx, b->d_image, (const uint64_t *)(t + o_src), (const int32_t *)(t + o_len), n, host_heap, heap_cap, host_off, heap_bytes, t,
                        o_off, o_chunk);
}

}  // extern "C"
