// Skip-index aggregate rows ON THE DEVICE (obgpu_agg_rows / obgpu_merge_result_agg_rows): per micro-block of the device
// encoder's blocking, the MIN / MAX / NULL_COUNT row ObSkipIndexAggregator hands to the index row (agg_row_buf_), byte for
// byte obgpu_writer_table_agg_rows over the same rows. The row layout and the compare images are ob_agg_row_format.h, the
// code the writer's block_agg_row runs.
// A fixed launch sequence, whatever the block count:
//   reduce  one warp per (block, aggregated column): min / max of the compare keys, NULL count and NOP flag over the block's
//           rows (coalesced loads of the value images and NULL bytes, warp reductions) -> one Rec per (block, column);
//   size    one thread per block sizes its row (obagg::layout); a row above 65535 bytes raises the status word;
//   prefix  obgpu_prefix_local_kernel / obgpu_prefix_fix_kernel: sizes -> row offsets [n_blocks + 1];
//   -- the host reads the total and the status (one synchronisation): the size query ends here --
//   write   one thread per block serializes its row (obagg::write) at its offset;
//   fetch   rows and offsets to the host, one synchronisation.
// One warp reduces a whole block: a block of R rows costs R / 32 dependent load steps on its warp, so very large blocks
// (rows_per_block in the millions) leave the device mostly idle; the encoder's blockings (at most 2^22 rows) are the use.
namespace agg {

constexpr int kThreads = 256;

struct ColSpec {             // one aggregated column, in ascending column index
  const int64_t *vals;
  const uint8_t *nulls;      // 1 NULL, 2 NOP; nullptr: no NULL cell
  uint32_t col_idx;
  uint8_t store_class, datum_len, unsigned_cmp;
};

struct Rec {                 // one (block, column): min / max compare images, NULL count (-1: a NOP cell, nothing aggregated)
  int64_t lo, hi, null_count;
};

__global__ void __launch_bounds__(kThreads) obgpu_agg_reduce_kernel(const ColSpec *__restrict__ cols, int32_t n_agg, int64_t n_blocks,
                                                                     int64_t total_rows, int64_t rows_per_block, Rec *__restrict__ recs) {
  const int64_t w = ((int64_t)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n_blocks * n_agg) return;
  const int32_t k = (int32_t)(w / n_blocks);   // warps of one column are adjacent: neighbouring warps read neighbouring blocks
  const int64_t b = w - (int64_t)k * n_blocks;
  const ColSpec c = cols[k];
  const int64_t r0 = b * rows_per_block, r1 = min(r0 + rows_per_block, total_rows);
  int64_t lo = INT64_MAX, hi = INT64_MIN;
  unsigned long long nulls = 0;
  bool nop = false;
  for (int64_t r = r0 + lane; r < r1; r += 32) {
    const uint8_t e = c.nulls ? __ldcs(c.nulls + r) : (uint8_t)0;
    const int64_t v = obagg::key(obagg::image(__ldcs(c.vals + r), c.store_class, c.datum_len), c.unsigned_cmp);
    if (e) {
      ++nulls;
      nop = nop || e == 2;
    } else {
      lo = min(lo, v);
      hi = max(hi, v);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = min(lo, (int64_t)__shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, (int64_t)__shfl_xor_sync(0xffffffffu, hi, o));
    nulls += __shfl_xor_sync(0xffffffffu, nulls, o);
  }
  nop = __any_sync(0xffffffffu, nop);
  if (lane == 0)
    recs[b * n_agg + k] = Rec{obagg::key(lo, c.unsigned_cmp), obagg::key(hi, c.unsigned_cmp), nop ? -1 : (int64_t)nulls};
}

// Column k of block b's row, as the writer's aggregate_column leaves it
__device__ __forceinline__ obagg::AggCol agg_col(const ColSpec *cols, const Rec *recs, int32_t n_agg, int64_t b, int64_t nrows, int k) {
  const Rec &r = recs[b * n_agg + k];
  obagg::AggCol a{cols[k].col_idx, -1, -1, nullptr, nullptr, 0, 0, 0, 0};
  if (r.null_count >= 0) {
    a.has_null_count = 1;
    a.null_count = r.null_count;
    if (r.null_count < nrows) {
      a.min_len = a.max_len = cols[k].datum_len;
      a.min = (const uint8_t *)&r.lo;
      a.max = (const uint8_t *)&r.hi;
    }
  }
  return a;
}

__global__ void __launch_bounds__(kThreads) obgpu_agg_size_kernel(const ColSpec *__restrict__ cols, const Rec *__restrict__ recs, int32_t n_agg,
                                                                   int64_t n_blocks, int64_t total_rows, int64_t rows_per_block,
                                                                   uint32_t *__restrict__ sizes, unsigned long long *status) {
  const int64_t b = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (b >= n_blocks) return;
  const int64_t nrows = min(rows_per_block, total_rows - b * rows_per_block);
  obagg::Layout l;
  const int64_t size = obagg::layout(n_agg, [&](int k) { return agg_col(cols, recs, n_agg, b, nrows, k); }, l);
  if (size < 0) atomicOr(status, 1ull);
  sizes[b] = size < 0 ? 0u : (uint32_t)size;
}

__global__ void __launch_bounds__(kThreads) obgpu_agg_write_kernel(const ColSpec *__restrict__ cols, const Rec *__restrict__ recs, int32_t n_agg,
                                                                    int64_t n_blocks, int64_t total_rows, int64_t rows_per_block,
                                                                    const int64_t *__restrict__ offsets, uint8_t *__restrict__ out) {
  const int64_t b = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (b >= n_blocks) return;
  const int64_t nrows = min(rows_per_block, total_rows - b * rows_per_block);
  auto col_at = [&](int k) { return agg_col(cols, recs, n_agg, b, nrows, k); };
  obagg::Layout l;
  obagg::layout(n_agg, col_at, l);
  obagg::write(n_agg, col_at, l, out + offsets[b]);
}

}  // namespace agg

static int agg_rows_run(obgpu_ctx *ctx, const obgpu_encode_col *cols, int32_t n_cols, const int32_t *agg_cols, int32_t n_agg,
                        int64_t total_rows, int64_t rows_per_block, void *host_out, int64_t out_cap, int64_t *host_offsets,
                        int64_t *out_size) {
  if (!ctx || !cols || n_cols <= 0 || !agg_cols || n_agg <= 0 || total_rows <= 0 || rows_per_block <= 0 || !out_size ||
      (host_out && !host_offsets))
    return OBGPU_INVALID_ARGUMENT;
  std::vector<agg::ColSpec> spec((size_t)n_agg);
  for (int32_t k = 0; k < n_agg; ++k) {
    const int32_t c = agg_cols[k];
    if (c < 0 || c >= n_cols || c >= (1 << 24)) return OBGPU_INVALID_ARGUMENT;
    const int sc = obf::store_class_of((uint8_t)cols[c].obj_type), dl = obf::datum_len_of((uint8_t)cols[c].obj_type);
    if (sc != 1 && sc != 2) {
      ctx->err = "skip-index aggregate rows on the device: integer-class columns only";
      return OBGPU_NOT_SUPPORTED;
    }
    if (!cols[c].dev_vals) return OBGPU_INVALID_ARGUMENT;
    spec[(size_t)k] = agg::ColSpec{cols[c].dev_vals, cols[c].dev_null, (uint32_t)c, (uint8_t)sc, (uint8_t)dl,
                                   (uint8_t)obagg::unsigned_order(sc, dl)};
  }
  std::sort(spec.begin(), spec.end(), [](const agg::ColSpec &a, const agg::ColSpec &b) { return a.col_idx < b.col_idx; });
  for (size_t k = 1; k < spec.size(); ++k)
    if (spec[k].col_idx == spec[k - 1].col_idx) {
      ctx->err = "agg_cols names a column twice";
      return OBGPU_INVALID_ARGUMENT;
    }
  const int64_t n = (total_rows + rows_per_block - 1) / rows_per_block;
  if (n > 0x7fffffff || n * n_agg > 0x7fffffffll * (agg::kThreads / 32)) return OBGPU_NOT_SUPPORTED;
  cudaSetDevice(ctx->device);
  const int n_chunks = (int)((n + kPrefixChunk - 1) / kPrefixChunk);
  Scratch arena(ctx);
  const size_t o_spec = arena.take((size_t)n_agg * sizeof(agg::ColSpec));
  const size_t o_rec = arena.take((size_t)n * n_agg * sizeof(agg::Rec));
  const size_t o_size = arena.take((size_t)n * 4);
  const size_t o_off = arena.take((size_t)(n + 2) * 8);   // offsets [n + 1], then the status word: one copy reads total + status
  const size_t o_chunk = arena.take((size_t)n_chunks * 8);
  CUDA_TRY(ctx, arena.alloc());
  agg::ColSpec *d_spec = arena.at<agg::ColSpec>(o_spec);
  agg::Rec *d_rec = arena.at<agg::Rec>(o_rec);
  uint32_t *d_size = arena.at<uint32_t>(o_size);
  int64_t *d_off = arena.at<int64_t>(o_off);
  unsigned long long *d_status = (unsigned long long *)(d_off + n + 1), *d_chunk = arena.at<unsigned long long>(o_chunk);
  CUDA_TRY(ctx, cudaMemcpyAsync(d_spec, spec.data(), spec.size() * sizeof(agg::ColSpec), cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaMemsetAsync(d_status, 0, 8, ctx->stream));
  const int64_t warps = n * n_agg;
  const unsigned grid_blocks = (unsigned)((n + agg::kThreads - 1) / agg::kThreads);
  agg::obgpu_agg_reduce_kernel<<<(unsigned)((warps + agg::kThreads / 32 - 1) / (agg::kThreads / 32)), agg::kThreads, 0, ctx->stream>>>(
      d_spec, n_agg, n, total_rows, rows_per_block, d_rec);
  agg::obgpu_agg_size_kernel<<<grid_blocks, agg::kThreads, 0, ctx->stream>>>(d_spec, d_rec, n_agg, n, total_rows, rows_per_block, d_size,
                                                                             d_status);
  obgpu_prefix_local_kernel<<<n_chunks, 256, 0, ctx->stream>>>(d_size, (int)n, d_off, d_chunk);
  obgpu_prefix_fix_kernel<<<n_chunks + 1, 256, 0, ctx->stream>>>((int)n, n_chunks, d_off, d_chunk);
  ctx->launches += 4;
  int64_t *hp = (int64_t *)ctx->h_pinned;
  CUDA_TRY(ctx, cudaGetLastError());
  CUDA_TRY(ctx, cudaMemcpyAsync(hp, d_off + n, 16, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  const int64_t total = hp[0];
  if (hp[1] != 0) {
    ctx->err = "an aggregate row exceeds 65535 bytes";
    return OBGPU_NOT_SUPPORTED;
  }
  *out_size = total;
  if (!host_out) return OBGPU_SUCCESS;
  if (out_cap < total) {
    ctx->err = "output capacity below the aggregate rows' size";
    return OBGPU_BUF_NOT_ENOUGH;
  }
  Scratch rows(ctx);
  CUDA_TRY(ctx, rows.alloc((size_t)std::max<int64_t>(total, 1)));
  agg::obgpu_agg_write_kernel<<<grid_blocks, agg::kThreads, 0, ctx->stream>>>(d_spec, d_rec, n_agg, n, total_rows, rows_per_block, d_off, rows.p);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  CUDA_TRY(ctx, cudaMemcpyAsync(host_out, rows.p, (size_t)total, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(host_offsets, d_off, (size_t)(n + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return OBGPU_SUCCESS;
}

extern "C" {

int obgpu_agg_rows(obgpu_ctx *ctx, const obgpu_encode_col *cols, int32_t n_cols, const int32_t *agg_cols, int32_t n_agg_cols,
                   int64_t total_rows, int64_t rows_per_block, void *host_out, int64_t out_cap, int64_t *host_offsets, int64_t *out_size) {
  return agg_rows_run(ctx, cols, n_cols, agg_cols, n_agg_cols, total_rows, rows_per_block, host_out, out_cap, host_offsets, out_size);
}

int obgpu_merge_result_agg_rows(obgpu_merge_result *res, const int32_t *result_cols, const int32_t *obj_types, int32_t n_cols,
                                const int32_t *agg_cols, int32_t n_agg_cols, int64_t rows_per_block, void *host_out, int64_t out_cap,
                                int64_t *host_offsets, int64_t *out_size) {
  if (!res || !result_cols || !obj_types || n_cols <= 0) return OBGPU_INVALID_ARGUMENT;
  std::vector<obgpu_encode_col> cols;
  int64_t rows = 0;
  const int rc = merge_result_cols(res, result_cols, obj_types, n_cols, cols, rows);
  if (rc != OBGPU_SUCCESS) return rc;
  return agg_rows_run(res->ctx, cols.data(), n_cols, agg_cols, n_agg_cols, rows, rows_per_block, host_out, out_cap, host_offsets, out_size);
}

}  // extern "C"
