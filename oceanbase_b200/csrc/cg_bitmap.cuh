// Column-group scans: the selection of a row range as a device-resident bitmap that several page batches share.
//
// Reference: in a column-store table every column group is its own SSTable with its own micro-blocks (different row boundaries per
// group). ObCOSSTableRowsFilter evaluates each pushed-down filter on ITS column group (ObCGScanner::apply_filter,
// column_store/ob_cg_scanner.cpp:273 -> filter_micro_block_in_cg, ob_micro_block_row_scanner.cpp:998), combines the per-group
// results in an ObCGBitmap over the row range (column_store/ob_cg_bitmap.{h,cpp}: bit_and / bit_or / set_bitmap with start_row_id
// offsets) and the projection groups then decode only the rows it selects (ObCGRowScanner::get_next_rows(count, capacity, bitmap),
// ob_cg_scanner.cpp:614). Here: a filter scan of one group's page batch is folded into an obgpu_cg_bitmap
// (obgpu_cg_bitmap_apply_result: set / and / or at the batch's row offset), and obgpu_scan_bitmap projects another group's page
// batch taking that bitmap as its selection -- the per-block packed words the count kernel would have produced are cut out of the
// range bitmap by obgpu_bitmap_slice_kernel, whatever the two groups' block boundaries are.
#pragma once

namespace cgbm {

// One warp per block of the result's batch: the block's packed selection words -> the range bitmap at bit (row_offset + first row
// of the block). A block's 32-row words land at an arbitrary bit position, so every word touches up to two range words, with
// atomics (neighbouring blocks share words). op 0 set, 1 and, 2 or.
__global__ void __launch_bounds__(128) fold_kernel(uint32_t *__restrict__ cg_words, int64_t cg_rows, int64_t row_offset,
                                                   const int64_t *__restrict__ row_start, const uint32_t *__restrict__ rows,
                                                   const int64_t *__restrict__ bm_word_off, int n_blocks,
                                                   const uint32_t *__restrict__ bitmap_words, int all_selected, int op) {
  const int blk = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (blk >= n_blocks) return;
  const uint32_t n = rows[blk];
  const int64_t g0 = row_offset + row_start[blk];
  for (uint32_t w = (uint32_t)lane; w < (n + 31u) / 32u; w += 32u) {
    const uint32_t nb = n - 32u * w >= 32u ? 32u : n - 32u * w;
    const uint32_t valid = nb == 32u ? 0xffffffffu : ((1u << nb) - 1u);
    const uint32_t v = (all_selected ? 0xffffffffu : bitmap_words[bm_word_off[blk] + w]) & valid;
    const int64_t g = g0 + 32ll * w;
    if (g < 0 || g + nb > cg_rows) continue;   // the host checked the extent
    const int64_t i = g >> 5;
    const uint32_t sh = (uint32_t)(g & 31);
    const uint32_t lo_bits = v << sh, lo_mask = valid << sh;
    const uint32_t hi_bits = sh ? v >> (32u - sh) : 0u, hi_mask = sh ? valid >> (32u - sh) : 0u;
    if (op == 0) {
      atomicAnd(&cg_words[i], ~lo_mask);
      atomicOr(&cg_words[i], lo_bits);
      if (hi_mask) { atomicAnd(&cg_words[i + 1], ~hi_mask); atomicOr(&cg_words[i + 1], hi_bits); }
    } else if (op == 1) {
      atomicAnd(&cg_words[i], lo_bits | ~lo_mask);
      if (hi_mask) atomicAnd(&cg_words[i + 1], hi_bits | ~hi_mask);
    } else {
      atomicOr(&cg_words[i], lo_bits);
      if (hi_mask) atomicOr(&cg_words[i + 1], hi_bits);
    }
  }
}

__global__ void __launch_bounds__(256) popcnt_kernel(const uint32_t *__restrict__ w, int64_t from, int64_t to, unsigned long long *out) {
  unsigned long long c = 0;
  const int64_t w0 = from >> 5, w1 = (to + 31) >> 5;
  for (int64_t i = w0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < w1; i += (int64_t)gridDim.x * blockDim.x) {
    uint32_t v = w[i];
    if (i == w0 && (from & 31)) v &= ~((1u << (from & 31)) - 1u);
    if (i == w1 - 1 && (to & 31)) v &= (1u << (to & 31)) - 1u;
    c += __popc(v);
  }
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}

__global__ void __launch_bounds__(256) expand_kernel(const uint32_t *__restrict__ w, int64_t from, int64_t count, uint8_t *__restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) out[i] = (uint8_t)((w[(from + i) >> 5] >> ((from + i) & 31)) & 1u);
}

}  // namespace cgbm

extern "C" {

int obgpu_cg_bitmap_create(obgpu_ctx *ctx, int64_t n_rows, int32_t all_true, obgpu_cg_bitmap **out) {
  if (!ctx || !out || n_rows < 0) return OBGPU_INVALID_ARGUMENT;
  cudaSetDevice(ctx->device);
  std::unique_ptr<obgpu_cg_bitmap> bm(new (std::nothrow) obgpu_cg_bitmap());
  if (!bm) return OBGPU_ALLOCATE_MEMORY_FAILED;
  bm->ctx = ctx;
  bm->n_rows = n_rows;
  const size_t words = (size_t)((n_rows + 31) / 32) + 2;
  Scratch w(ctx);
  CUDA_TRY(ctx, w.alloc(words * 4));
  uint32_t *d_words = w.at<uint32_t>(0);
  CUDA_TRY(ctx, cudaMemsetAsync(d_words, all_true ? 0xff : 0, words * 4, ctx->stream));
  if (all_true && (n_rows & 31)) {   // bits past the range stay clear (popcounts, folds of neighbours)
    const uint32_t last = (1u << (n_rows & 31)) - 1u;
    CUDA_TRY(ctx, cudaMemcpyAsync(d_words + n_rows / 32, &last, 4, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  }
  if (all_true) CUDA_TRY(ctx, cudaMemsetAsync(d_words + (n_rows + 31) / 32, 0, 8, ctx->stream));
  bm->d_words = (uint32_t *)w.release();
  *out = bm.release();
  return OBGPU_SUCCESS;
}

void obgpu_cg_bitmap_free(obgpu_cg_bitmap *bm) {
  if (!bm) return;
  cudaSetDevice(bm->ctx->device);
  if (bm->d_words) cudaFreeAsync(bm->d_words, bm->ctx->stream);
  delete bm;
}

int obgpu_cg_bitmap_apply_result(obgpu_cg_bitmap *bm, obgpu_result *r, int64_t row_offset, int32_t op) {
  if (!bm || !r || op < 0 || op > 2) return OBGPU_INVALID_ARGUMENT;
  obgpu_batch *b = r->batch;
  if (row_offset < 0 || row_offset + b->total_rows > bm->n_rows) return OBGPU_INVALID_ARGUMENT;
  if (bm->ctx != r->ctx) { bm->ctx->err = "the bitmap and the result live on different contexts (streams)"; return OBGPU_INVALID_ARGUMENT; }
  obgpu_ctx *ctx = bm->ctx;
  cudaSetDevice(ctx->device);
  cgbm::fold_kernel<<<(unsigned)(((int64_t)b->n_blocks * 32 + 127) / 128), 128, 0, ctx->stream>>>(
      bm->d_words, bm->n_rows, row_offset, b->d_row_start, b->d_rows, b->d_bm_word_off, b->n_blocks, r->d_bitmap, r->no_filter ? 1 : 0, op);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  return OBGPU_SUCCESS;
}

int obgpu_cg_bitmap_popcnt(obgpu_cg_bitmap *bm, int64_t from, int64_t to, int64_t *count) {
  if (!bm || !count || from < 0 || to < from || to > bm->n_rows) return OBGPU_INVALID_ARGUMENT;
  obgpu_ctx *ctx = bm->ctx;
  cudaSetDevice(ctx->device);
  *count = 0;
  if (to == from) return OBGPU_SUCCESS;
  Scratch tmp(ctx);
  CUDA_TRY(ctx, tmp.alloc(64));
  CUDA_TRY(ctx, cudaMemsetAsync(tmp.p, 0, 64, ctx->stream));
  cgbm::popcnt_kernel<<<std::min<int64_t>(1024, ((to - from) / 32 + 256) / 256), 256, 0, ctx->stream>>>(bm->d_words, from, to, tmp.at<unsigned long long>(0));
  ctx->launches++;
  unsigned long long c = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&c, tmp.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  *count = (int64_t)c;
  return OBGPU_SUCCESS;
}

int obgpu_cg_bitmap_fetch(obgpu_cg_bitmap *bm, int64_t from, int64_t count, uint8_t *host_bitmap_bytes) {
  if (!bm || !host_bitmap_bytes || from < 0 || count < 0 || from + count > bm->n_rows) return OBGPU_INVALID_ARGUMENT;
  if (count == 0) return OBGPU_SUCCESS;
  obgpu_ctx *ctx = bm->ctx;
  cudaSetDevice(ctx->device);
  Scratch tmp(ctx);
  CUDA_TRY(ctx, tmp.alloc((size_t)count));
  cgbm::expand_kernel<<<(unsigned)((count + 255) / 256), 256, 0, ctx->stream>>>(bm->d_words, from, count, tmp.p);
  ctx->launches++;
  CUDA_TRY(ctx, cudaMemcpyAsync(host_bitmap_bytes, tmp.p, (size_t)count, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return OBGPU_SUCCESS;
}

int obgpu_scan_bitmap(obgpu_batch *batch, const obgpu_cg_bitmap *bm, int64_t row_offset, const obgpu_scan_spec *spec, obgpu_result **out) {
  if (!batch || !bm || !spec || !out) return OBGPU_INVALID_ARGUMENT;
  if (row_offset < 0 || row_offset + batch->total_rows > bm->n_rows) return OBGPU_INVALID_ARGUMENT;
  if (bm->ctx != batch->ctx) { batch->ctx->err = "the bitmap and the batch live on different contexts (streams)"; return OBGPU_INVALID_ARGUMENT; }
  return scan_common(batch, spec, bm, row_offset, out);
}

}  // extern "C"
