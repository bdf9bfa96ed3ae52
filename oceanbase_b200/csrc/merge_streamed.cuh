// Major merge of runs that do not fit in device memory together: range by range, inside the library.
//
// Reference: ObPartitionMajorMerger::merge_partition walks all tables in rowkey order with bounded memory (row iterators over the
// block cache, compaction/ob_partition_merger.cpp:678-829); parallel merge cuts the rowkey space into ranges at block boundaries
// taken from the index tree (ObParallelMergeCtx, ob_partition_parallel_merge_ctx.cpp:187-424). Here a range is one unit of device
// work: the micro-blocks of every run that can hold its rowkeys are opened as a page batch straight from HOST memory (the
// host->device copy), decoded, cut to the range by a binary search on the decoded rowkeys, merged (obgpu_merge_decoded), and handed
// to the caller's sink, which fetches / encodes the rows. n_streams worker threads, each with its own ctx / stream, keep that many
// ranges in flight: the copies of range i + 1 run under the merge and fetch of range i; device memory holds n_streams ranges.
#pragma once
#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <mutex>
#include <thread>

namespace mstream {

// first index with key > bound (upper bound), one thread
__global__ void cut_kernel(const int64_t *key, int64_t n, int64_t lo, int has_lo, int64_t hi, int has_hi, int64_t *out) {
  int64_t a = 0, b = n;
  if (has_lo) { while (a < b) { const int64_t m = (a + b) >> 1; if (key[m] <= lo) a = m + 1; else b = m; } }
  out[0] = has_lo ? a : 0;
  a = 0; b = n;
  if (has_hi) { while (a < b) { const int64_t m = (a + b) >> 1; if (key[m] <= hi) a = m + 1; else b = m; } }
  out[1] = has_hi ? a : n;
}

}  // namespace mstream

extern "C" int obgpu_merge_runs_streamed(int device, int32_t n_streams, const obgpu_stream_run *runs, int32_t n_runs, int32_t rowkey_col,
                                         int32_t flag_col, const int32_t *cols, int32_t n_cols, const int64_t *default_vals,
                                         const uint8_t *default_null, int32_t n_ranges, obgpu_merge_sink sink, void *sink_arg,
                                         int32_t *ranges_done) {
  if (!runs || n_runs <= 0 || n_runs > OBGPU_MERGE_MAX_RUNS || n_cols < 0 || n_cols > 14 || (n_cols > 0 && !cols) || n_ranges <= 0 || !sink)
    return OBGPU_INVALID_ARGUMENT;
  for (int r = 0; r < n_runs; ++r)
    if (!runs[r].image || !runs[r].offsets || !runs[r].sizes || !runs[r].end_keys || runs[r].n_blocks < 0) return OBGPU_INVALID_ARGUMENT;
  // range bounds: quantiles of all block end keys; range i = (bound[i - 1], bound[i]], the first open below, the last open above
  std::vector<int64_t> all;
  for (int r = 0; r < n_runs; ++r) all.insert(all.end(), runs[r].end_keys, runs[r].end_keys + runs[r].n_blocks);
  std::sort(all.begin(), all.end());
  std::vector<int64_t> cuts;
  for (int i = 0; i + 1 < n_ranges && !all.empty(); ++i) {
    const int64_t c = all[std::min(all.size() - 1, all.size() * (size_t)(i + 1) / (size_t)n_ranges)];
    if (cuts.empty() || cuts.back() != c) cuts.push_back(c);
  }
  const int R = (int)cuts.size() + 1;
  if (ranges_done) *ranges_done = 0;
  std::atomic<int> next{0};
  std::atomic<int> first_err{OBGPU_SUCCESS};
  std::mutex mu;
  std::condition_variable cv;
  int delivered = 0;   // ranges handed to the sink so far (they go out in order)
  const int nw = std::max(1, std::min<int>(n_streams, R));
  auto worker = [&]() {
    obgpu_ctx *ctx = nullptr;
    int ret = obgpu_ctx_create(device, &ctx);
    if (ret != OBGPU_SUCCESS) { int e = OBGPU_SUCCESS; first_err.compare_exchange_strong(e, ret); cv.notify_all(); return; }
    const int n_dec = n_cols + 1 + (flag_col >= 0 ? 1 : 0);
    for (;;) {
      const int i = next.fetch_add(1);
      if (i >= R || first_err.load() != OBGPU_SUCCESS) break;
      const bool has_lo = i > 0, has_hi = i + 1 < R;
      const int64_t lo = has_lo ? cuts[(size_t)i - 1] : 0, hi = has_hi ? cuts[(size_t)i] : 0;
      std::vector<obgpu_batch *> batches((size_t)n_runs, nullptr);
      std::vector<obgpu_merge_run> mr((size_t)n_runs);
      std::vector<std::vector<const int64_t *>> vptr((size_t)n_runs);
      std::vector<std::vector<const uint8_t *>> eptr((size_t)n_runs);
      obgpu_merge_result *res = nullptr;
      Scratch cut(ctx);
      std::deque<Scratch> bufs;   // the decoded columns of the runs
      // every run's blocks of the range, opened, decoded and cut to (lo, hi], then merged into res
      ret = [&]() -> int {
        CUDA_TRY(ctx, cut.alloc(16 * (size_t)n_runs + 16));
        int64_t *d_cut = cut.at<int64_t>(0);
        std::vector<int64_t> h_cut((size_t)n_runs * 2, 0);
        for (int r = 0; r < n_runs; ++r) {
          const obgpu_stream_run &sr = runs[r];
          const int64_t *ek = sr.end_keys;
          const int32_t b0 = has_lo ? (int32_t)(std::upper_bound(ek, ek + sr.n_blocks, lo) - ek) : 0;             // first block whose last key > lo
          const int32_t b1 = has_hi ? std::min<int32_t>(sr.n_blocks, (int32_t)(std::lower_bound(ek, ek + sr.n_blocks, hi) - ek) + 1) : sr.n_blocks;
          mr[(size_t)r] = obgpu_merge_run{};
          vptr[(size_t)r].assign((size_t)std::max(n_cols, 1), nullptr);
          eptr[(size_t)r].assign((size_t)std::max(n_cols, 1), nullptr);
          mr[(size_t)r].vals = vptr[(size_t)r].data();
          mr[(size_t)r].ext = eptr[(size_t)r].data();
          if (b0 >= b1) continue;
          const int64_t o0 = sr.offsets[b0], o1 = sr.offsets[b1 - 1] + sr.sizes[b1 - 1];
          std::vector<int64_t> offs((size_t)(b1 - b0));
          for (int32_t k = b0; k < b1; ++k) offs[(size_t)(k - b0)] = sr.offsets[k] - o0;
          int rc = obgpu_batch_open(ctx, (const uint8_t *)sr.image + o0, o1 - o0, offs.data(), sr.sizes + b0, b1 - b0, 0, nullptr, &batches[(size_t)r]);
          if (rc != OBGPU_SUCCESS) return rc;
          int64_t rows = 0;
          obgpu_batch_total_rows(batches[(size_t)r], &rows);
          std::vector<int32_t> dc;
          dc.push_back(rowkey_col);
          if (flag_col >= 0) dc.push_back(flag_col);
          for (int c = 0; c < n_cols; ++c) dc.push_back(cols[c]);
          std::vector<int64_t *> dv((size_t)n_dec);
          std::vector<uint8_t *> de((size_t)n_dec);
          for (int c = 0; c < n_dec; ++c) {
            Scratch &v = bufs.emplace_back(ctx);
            CUDA_TRY(ctx, v.alloc((size_t)rows * 8 + 16));
            Scratch &e = bufs.emplace_back(ctx);
            CUDA_TRY(ctx, e.alloc((size_t)rows + 16));
            dv[(size_t)c] = v.at<int64_t>(0);
            de[(size_t)c] = e.p;
          }
          rc = obgpu_batch_decode_columns(batches[(size_t)r], n_dec, dc.data(), dv.data(), de.data());
          if (rc != OBGPU_SUCCESS) return rc;
          mstream::cut_kernel<<<1, 1, 0, ctx->stream>>>(dv[0], rows, lo, has_lo ? 1 : 0, hi, has_hi ? 1 : 0, d_cut + 2 * r);
          ctx->launches++;
          // the flag column decodes to int64 images: narrow it to the ObDmlFlag byte per row the merge takes
          uint8_t *flag8 = nullptr;
          if (flag_col >= 0) {
            flag8 = de[1];   // the flag column's ext array is not needed (flags are never NULL): reuse it for the narrowed bytes
            mrg::narrow_flag_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, ctx->stream>>>(dv[1], rows, flag8);
            ctx->launches++;
          }
          mr[(size_t)r].key = dv[0];
          mr[(size_t)r].flag = flag8;
          mr[(size_t)r].n = rows;   // cut below
          const int first = flag_col >= 0 ? 2 : 1;
          for (int c = 0; c < n_cols; ++c) { vptr[(size_t)r][(size_t)c] = dv[(size_t)(first + c)]; eptr[(size_t)r][(size_t)c] = de[(size_t)(first + c)]; }
        }
        CUDA_TRY(ctx, cudaMemcpyAsync(h_cut.data(), d_cut, 16 * (size_t)n_runs, cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
        for (int r = 0; r < n_runs; ++r) {
          if (!batches[(size_t)r]) { mr[(size_t)r].n = 0; continue; }
          const int64_t r0 = h_cut[(size_t)2 * r], r1 = h_cut[(size_t)2 * r + 1];
          mr[(size_t)r].n = r1 - r0;
          mr[(size_t)r].key += r0;
          if (mr[(size_t)r].flag) mr[(size_t)r].flag += r0;
          for (int c = 0; c < n_cols; ++c) { vptr[(size_t)r][(size_t)c] += r0; eptr[(size_t)r][(size_t)c] += r0; }
        }
        return obgpu_merge_decoded(ctx, mr.data(), n_runs, n_cols, default_vals, default_null, &res);
      }();
      obgpu_merge_info info{};
      if (ret == OBGPU_SUCCESS) ret = obgpu_merge_result_info(res, &info);
      // ranges leave in order
      {
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [&] { return delivered == i || first_err.load() != OBGPU_SUCCESS; });
        if (ret == OBGPU_SUCCESS && first_err.load() == OBGPU_SUCCESS) ret = sink(sink_arg, i, res);
        if (ret != OBGPU_SUCCESS) { int e = OBGPU_SUCCESS; first_err.compare_exchange_strong(e, ret); }
        ++delivered;
        if (ranges_done && ret == OBGPU_SUCCESS) *ranges_done = delivered;
      }
      cv.notify_all();
      if (res) obgpu_merge_result_free(res);
      for (obgpu_batch *b : batches) if (b) obgpu_batch_close(b);
      if (ret != OBGPU_SUCCESS) break;
    }
    cudaStreamSynchronize(ctx->stream);
    obgpu_ctx_destroy(ctx);
  };
  std::vector<std::thread> th;
  for (int w = 0; w < nw; ++w) th.emplace_back(worker);
  for (auto &t : th) t.join();
  return first_err.load();
}
