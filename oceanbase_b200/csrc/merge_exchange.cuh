// Range-partitioned major merge across the GPUs of one box: the one exchange step of the path, in the library.
//
// Reference: parallel major merge cuts a tablet's rowkey space into ranges at macro-block boundaries and merges every
// range independently, the outputs being concatenated in range order (ObParallelMergeCtx,
// compaction/ob_partition_parallel_merge_ctx.cpp:187-424; ObPartitionMajorMerger::merge_partition per range,
// compaction/ob_partition_merger.cpp:678-829). Here one range per rank:
//   1. every rank samples the rowkeys of the runs it holds (evenly spaced, device kernel)
//   2. ncclAllGather of the candidates -> device radix sort -> world - 1 splitters at the quantiles (all on the device)
//   3. lower_bound of every splitter in every local run (device) -> rows per (run, destination); ncclAllReduce makes the
//      matrix global; ONE device->host copy of it sizes the receive buffers
//   4. slices are packed per (run, destination) and exchanged with grouped ncclSend / ncclRecv over NVLink
//   5. obgpu_merge_decoded on what arrived: rank order is global rowkey order
// Everything between the sizing copy and the merge is enqueued on the ctx stream without host synchronisation.
// NCCL is bound at run time (dlopen of libnccl.so.2): the library has no link-time dependency on it and loads on boxes
// without NCCL; the communicator id travels through the caller's own channel (an RPC in OceanBase, torch.distributed
// in bench.py / the tests).
#pragma once
#include <dlfcn.h>
#include <nccl.h>

#include <cub/device/device_radix_sort.cuh>

struct obgpu_comm {
  obgpu_ctx *ctx = nullptr;
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1;
};

namespace obnccl {

struct Api {
  void *lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};

inline Api &api() {
  static Api a = [] {
    Api x;
    for (const char *name : {"libnccl.so.2", "libnccl.so"}) {
      x.lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
      if (x.lib) break;
    }
    if (!x.lib) return x;
    auto sym = [&](const char *n) { return dlsym(x.lib, n); };
    x.GetUniqueId = (decltype(x.GetUniqueId))sym("ncclGetUniqueId");
    x.CommInitRank = (decltype(x.CommInitRank))sym("ncclCommInitRank");
    x.CommDestroy = (decltype(x.CommDestroy))sym("ncclCommDestroy");
    x.AllGather = (decltype(x.AllGather))sym("ncclAllGather");
    x.AllReduce = (decltype(x.AllReduce))sym("ncclAllReduce");
    x.Send = (decltype(x.Send))sym("ncclSend");
    x.Recv = (decltype(x.Recv))sym("ncclRecv");
    x.GroupStart = (decltype(x.GroupStart))sym("ncclGroupStart");
    x.GroupEnd = (decltype(x.GroupEnd))sym("ncclGroupEnd");
    x.GetErrorString = (decltype(x.GetErrorString))sym("ncclGetErrorString");
    x.ok = x.GetUniqueId && x.CommInitRank && x.CommDestroy && x.AllGather && x.AllReduce && x.Send && x.Recv && x.GroupStart && x.GroupEnd;
    return x;
  }();
  return a;
}

// evenly spaced rowkeys of one run into its candidate slots (INT64_MAX pads the rest)
__global__ void __launch_bounds__(256) sample_kernel(const int64_t *key, int64_t n, int32_t s, int64_t *out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= s) return;
  const int64_t take = n < s ? n : s;
  out[i] = i < take ? key[((int64_t)i * n) / take] : INT64_MAX;
}

// splitter j = sorted candidate at the (j + 1) / world quantile of the valid ones
__global__ void splitter_kernel(const int64_t *sorted, const int64_t *n_valid, int world, int64_t *splitters) {
  const int j = threadIdx.x;
  if (j >= world - 1) return;
  const int64_t v = *n_valid;
  splitters[j] = v > 0 ? sorted[min(v - 1, ((int64_t)(j + 1) * v) / world)] : INT64_MAX;
}

// bounds[q][j + 1] = lower_bound(run q, splitter j); bounds[q][0] = 0, bounds[q][world] = n
struct BoundRuns { const int64_t *key[OBGPU_MERGE_MAX_RUNS]; int64_t n[OBGPU_MERGE_MAX_RUNS]; int32_t index[OBGPU_MERGE_MAX_RUNS]; };
__global__ void bounds_kernel(BoundRuns runs, int n_local, const int64_t *splitters, int world, int64_t *bounds /* [n_local][world + 1] */,
                              long long *cnt /* [n_runs_total][world] */, long long *held /* [n_runs_total] */, long long *owner, int rank) {
  const int q = blockIdx.x, j = threadIdx.x;
  if (q >= n_local || j > world) return;
  const int64_t n = runs.n[q];
  int64_t pos;
  if (j == 0) pos = 0;
  else if (j == world) pos = n;
  else {
    const int64_t s = splitters[j - 1];
    int64_t lo = 0, hi = n;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (runs.key[q][mid] < s) lo = mid + 1; else hi = mid;
    }
    pos = lo;
  }
  bounds[(int64_t)q * (world + 1) + j] = pos;
  __syncthreads();
  if (j < world) cnt[(int64_t)runs.index[q] * world + j] = bounds[(int64_t)q * (world + 1) + j + 1] - bounds[(int64_t)q * (world + 1) + j];
  if (j == 0) { held[runs.index[q]] = 1; owner[runs.index[q]] = rank; }
}

}  // namespace obnccl

extern "C" {

int obgpu_comm_unique_id(void *id_out) {
  if (!id_out) return OBGPU_INVALID_ARGUMENT;
  obnccl::Api &a = obnccl::api();
  if (!a.ok) return OBGPU_NOT_SUPPORTED;
  ncclUniqueId id;
  if (a.GetUniqueId(&id) != ncclSuccess) return OBGPU_ERR_SYS;
  static_assert(sizeof(ncclUniqueId) == OBGPU_COMM_ID_BYTES, "ncclUniqueId is 128 bytes");
  memcpy(id_out, &id, sizeof(id));
  return OBGPU_SUCCESS;
}

int obgpu_comm_create(obgpu_ctx *ctx, const void *id, int32_t rank, int32_t world, obgpu_comm **out) {
  if (!ctx || !id || !out || world < 1 || rank < 0 || rank >= world) return OBGPU_INVALID_ARGUMENT;
  obnccl::Api &a = obnccl::api();
  if (!a.ok) { ctx->err = "NCCL (libnccl.so.2) not found"; return OBGPU_NOT_SUPPORTED; }
  cudaSetDevice(ctx->device);
  obgpu_comm *c = new (std::nothrow) obgpu_comm();
  if (!c) return OBGPU_ALLOCATE_MEMORY_FAILED;
  c->ctx = ctx;
  c->rank = rank;
  c->world = world;
  ncclUniqueId uid;
  memcpy(&uid, id, sizeof(uid));
  const ncclResult_t r = a.CommInitRank(&c->comm, world, uid, rank);
  if (r != ncclSuccess) {
    ctx->err = std::string("ncclCommInitRank: ") + (a.GetErrorString ? a.GetErrorString(r) : "failed");
    delete c;
    return OBGPU_ERR_SYS;
  }
  *out = c;
  return OBGPU_SUCCESS;
}

void obgpu_comm_destroy(obgpu_comm *c) {
  if (!c) return;
  if (c->comm) {
    cudaSetDevice(c->ctx->device);
    cudaStreamSynchronize(c->ctx->stream);
    obnccl::api().CommDestroy(c->comm);
  }
  delete c;
}

int obgpu_merge_decoded_distributed(obgpu_ctx *ctx, obgpu_comm *comm, const obgpu_merge_run *local_runs, const int32_t *run_index,
                                    int32_t n_local, int32_t n_runs_total, int32_t n_cols, int32_t n_more_keys, const int64_t *default_vals,
                                    const uint8_t *default_null, int32_t samples_per_run, obgpu_merge_result **out,
                                    int64_t *splitters_out, int64_t *recv_rows_out) {
  if (!ctx || !comm || comm->ctx != ctx || !out || n_local < 0 || n_runs_total <= 0 || n_runs_total > OBGPU_MERGE_MAX_RUNS ||
      n_local > n_runs_total || (n_local > 0 && (!local_runs || !run_index)) || n_cols < 0 || n_cols > OBGPU_MERGE_MAX_COLS ||
      n_more_keys < 0 || n_more_keys > OBGPU_MERGE_MAX_KEY_COLS - 1 || samples_per_run < 1 || samples_per_run > 65536)
    return OBGPU_INVALID_ARGUMENT;
  for (int q = 0; q < n_local; ++q)
    if (run_index[q] < 0 || run_index[q] >= n_runs_total || local_runs[q].n < 0 || local_runs[q].n_more_keys != n_more_keys) return OBGPU_INVALID_ARGUMENT;
  obnccl::Api &a = obnccl::api();
  const int world = comm->world, rank = comm->rank, S = samples_per_run;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
#define NCCL_TRY(expr)                                                                                                          \
  if (const ncclResult_t r__ = (expr); r__ != ncclSuccess) {                                                                    \
    ctx->err = std::string(#expr) + ": " + (a.GetErrorString ? a.GetErrorString(r__) : "nccl error");                         \
    return OBGPU_ERR_SYS;                                                                                                       \
  } else (void)0
  // every device buffer of the call; freed on the stream when it returns, after the kernels and transfers that use them
  std::deque<Scratch> bufs;
  auto dalloc = [&](size_t bytes, auto *&p) {
    Scratch &s = bufs.emplace_back(ctx);
    const cudaError_t e = s.alloc(bytes);
    p = s.at<std::remove_reference_t<decltype(*p)>>(0);
    return e;
  };
  const size_t slots = (size_t)n_runs_total * S;
  int64_t *d_cand, *d_all, *d_sorted, *d_split, *d_bounds;
  long long *d_tab;   // cnt | held | owner | valid
  CUDA_TRY(ctx, dalloc(slots * 8, d_cand));
  CUDA_TRY(ctx, dalloc(slots * 8 * world, d_all));
  CUDA_TRY(ctx, dalloc(slots * 8 * world, d_sorted));
  CUDA_TRY(ctx, dalloc((size_t)std::max(world - 1, 1) * 8, d_split));
  CUDA_TRY(ctx, dalloc(((size_t)n_runs_total * world + 2 * (size_t)n_runs_total + 2) * 8, d_tab));
  CUDA_TRY(ctx, dalloc((size_t)std::max(n_local, 1) * (world + 1) * 8, d_bounds));
  long long *d_cnt = d_tab, *d_held = d_tab + (size_t)n_runs_total * world, *d_owner = d_held + n_runs_total, *d_valid = d_owner + n_runs_total;
  CUDA_TRY(ctx, cudaMemsetAsync(d_tab, 0, ((size_t)n_runs_total * world + 2 * (size_t)n_runs_total + 2) * 8, st));
  // 1. candidates (slots of runs held elsewhere stay INT64_MAX)
  {
    std::vector<int64_t> fill(slots, INT64_MAX);
    CUDA_TRY(ctx, cudaMemcpyAsync(d_cand, fill.data(), slots * 8, cudaMemcpyHostToDevice, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));   // `fill` is pageable
  }
  long long valid = 0;
  for (int q = 0; q < n_local; ++q) {
    if (local_runs[q].n == 0) continue;
    obnccl::sample_kernel<<<(S + 255) / 256, 256, 0, st>>>(local_runs[q].key, local_runs[q].n, S, d_cand + (size_t)run_index[q] * S);
    ctx->launches++;
    valid += std::min<int64_t>(S, local_runs[q].n);
  }
  CUDA_TRY(ctx, cudaMemcpyAsync(d_valid, &valid, 8, cudaMemcpyHostToDevice, st));
  // 2. gather, sort, splitters -- device only
  NCCL_TRY(a.AllGather(d_cand, d_all, slots, ncclInt64, comm->comm, st));
  NCCL_TRY(a.AllReduce(d_valid, d_valid, 1, ncclInt64, ncclSum, comm->comm, st));
  {
    size_t tmp_bytes = 0;
    CUDA_TRY(ctx, cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, d_all, d_sorted, (int64_t)(slots * world), 0, 64, st));
    uint8_t *d_tmp;
    CUDA_TRY(ctx, dalloc(tmp_bytes, d_tmp));
    CUDA_TRY(ctx, cub::DeviceRadixSort::SortKeys(d_tmp, tmp_bytes, d_all, d_sorted, (int64_t)(slots * world), 0, 64, st));
    ctx->launches += 3;
  }
  if (world > 1) {
    obnccl::splitter_kernel<<<1, 64 >= world ? 64 : 1024, 0, st>>>(d_sorted, (const int64_t *)d_valid, world, d_split);
    ctx->launches++;
  }
  // 3. slice bounds of the local runs, global rows-per-(run, destination) matrix
  if (n_local > 0) {
    obnccl::BoundRuns br{};
    for (int q = 0; q < n_local; ++q) { br.key[q] = local_runs[q].key; br.n[q] = local_runs[q].n; br.index[q] = run_index[q]; }
    obnccl::bounds_kernel<<<n_local, world + 1 <= 32 ? 32 : ((world + 32) & ~31), 0, st>>>(br, n_local, d_split, world, d_bounds, d_cnt, d_held, d_owner, rank);
    ctx->launches++;
  }
  NCCL_TRY(a.AllReduce(d_tab, d_tab, (size_t)n_runs_total * world + 2 * (size_t)n_runs_total, ncclInt64, ncclSum, comm->comm, st));
  std::vector<long long> h_tab((size_t)n_runs_total * world + 2 * (size_t)n_runs_total);
  std::vector<int64_t> h_bounds((size_t)std::max(n_local, 1) * (world + 1)), h_split((size_t)std::max(world - 1, 1));
  CUDA_TRY(ctx, cudaMemcpyAsync(h_tab.data(), d_tab, h_tab.size() * 8, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(h_bounds.data(), d_bounds, h_bounds.size() * 8, cudaMemcpyDeviceToHost, st));
  if (world > 1) CUDA_TRY(ctx, cudaMemcpyAsync(h_split.data(), d_split, (size_t)(world - 1) * 8, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));   // the one sizing synchronisation
  const long long *h_cnt = h_tab.data(), *h_held = h_cnt + (size_t)n_runs_total * world, *h_owner = h_held + n_runs_total;
  for (int q = 0; q < n_runs_total; ++q)
    if (h_held[q] != 1) { ctx->err = "every run index must be held by exactly one rank"; return OBGPU_INVALID_ARGUMENT; }
  if (splitters_out) for (int j = 0; j + 1 < world; ++j) splitters_out[j] = h_split[(size_t)j];
  // 4. pack + exchange. One buffer per (run, peer): [key | vals x n_cols | more_keys x n_more] int64, then [flag | ext x n_cols] bytes
  const size_t n64 = 1 + (size_t)n_cols + (size_t)n_more_keys;
  const size_t row_bytes = 8 * n64 + 1 + (size_t)n_cols;
  struct Xfer { void *buf; size_t bytes; int peer; };
  std::vector<Xfer> sends, recvs;
  std::vector<obgpu_merge_run> runs((size_t)n_runs_total);
  std::vector<std::vector<const int64_t *>> vptr((size_t)n_runs_total), mptr((size_t)n_runs_total);
  std::vector<std::vector<const uint8_t *>> eptr((size_t)n_runs_total);
  std::vector<int> local_of((size_t)n_runs_total, -1);
  for (int q = 0; q < n_local; ++q) local_of[(size_t)run_index[q]] = q;
  for (int g = 0; g < n_runs_total; ++g) {
    obgpu_merge_run &r = runs[(size_t)g];
    r = obgpu_merge_run{};
    r.n_more_keys = n_more_keys;
    vptr[(size_t)g].assign((size_t)n_cols, nullptr);
    eptr[(size_t)g].assign((size_t)n_cols, nullptr);
    mptr[(size_t)g].assign((size_t)n_more_keys, nullptr);
    const int q = local_of[(size_t)g];
    if (q >= 0) {
      const obgpu_merge_run &src = local_runs[q];
      const int64_t *b = h_bounds.data() + (size_t)q * (world + 1);
      for (int j = 0; j < world; ++j) {
        const int64_t lo = b[j], n = b[j + 1] - b[j];
        if (j == rank) {   // stays here: a view of the caller's arrays
          r.n = n;
          r.key = src.key + lo;
          r.flag = src.flag ? src.flag + lo : nullptr;
          for (int c = 0; c < n_cols; ++c) { vptr[(size_t)g][(size_t)c] = src.vals[c] + lo; eptr[(size_t)g][(size_t)c] = src.ext[c] + lo; }
          for (int c = 0; c < n_more_keys; ++c) mptr[(size_t)g][(size_t)c] = src.more_keys[c] + lo;
          continue;
        }
        if (n == 0) continue;
        uint8_t *buf;
        CUDA_TRY(ctx, dalloc((size_t)n * row_bytes, buf));
        int64_t *i64 = (int64_t *)buf;
        uint8_t *u8 = buf + (size_t)n * 8 * n64;
        CUDA_TRY(ctx, cudaMemcpyAsync(i64, src.key + lo, (size_t)n * 8, cudaMemcpyDeviceToDevice, st));
        for (int c = 0; c < n_cols; ++c) CUDA_TRY(ctx, cudaMemcpyAsync(i64 + (size_t)(1 + c) * n, src.vals[c] + lo, (size_t)n * 8, cudaMemcpyDeviceToDevice, st));
        for (int c = 0; c < n_more_keys; ++c) CUDA_TRY(ctx, cudaMemcpyAsync(i64 + (size_t)(1 + n_cols + c) * n, src.more_keys[c] + lo, (size_t)n * 8, cudaMemcpyDeviceToDevice, st));
        if (src.flag) CUDA_TRY(ctx, cudaMemcpyAsync(u8, src.flag + lo, (size_t)n, cudaMemcpyDeviceToDevice, st));
        else CUDA_TRY(ctx, cudaMemsetAsync(u8, OBGPU_DF_INSERT, (size_t)n, st));
        for (int c = 0; c < n_cols; ++c) CUDA_TRY(ctx, cudaMemcpyAsync(u8 + (size_t)(1 + c) * n, src.ext[c] + lo, (size_t)n, cudaMemcpyDeviceToDevice, st));
        sends.push_back(Xfer{buf, (size_t)n * row_bytes, j});
      }
    } else {
      const int64_t n = h_cnt[(size_t)g * world + rank];
      if (n > 0) {
        uint8_t *buf;
        CUDA_TRY(ctx, dalloc((size_t)n * row_bytes, buf));
        const int64_t *i64 = (const int64_t *)buf;
        const uint8_t *u8 = buf + (size_t)n * 8 * n64;
        r.n = n;
        r.key = i64;
        r.flag = u8;
        for (int c = 0; c < n_cols; ++c) { vptr[(size_t)g][(size_t)c] = i64 + (size_t)(1 + c) * n; eptr[(size_t)g][(size_t)c] = u8 + (size_t)(1 + c) * n; }
        for (int c = 0; c < n_more_keys; ++c) mptr[(size_t)g][(size_t)c] = i64 + (size_t)(1 + n_cols + c) * n;
        recvs.push_back(Xfer{buf, (size_t)n * row_bytes, (int)h_owner[g]});
      }
    }
    r.vals = vptr[(size_t)g].data();
    r.ext = eptr[(size_t)g].data();
    r.more_keys = n_more_keys ? mptr[(size_t)g].data() : nullptr;
    if (recv_rows_out) recv_rows_out[g] = r.n;
  }
  if (!sends.empty() || !recvs.empty()) {
    NCCL_TRY(a.GroupStart());
    for (const Xfer &x : sends) NCCL_TRY(a.Send(x.buf, x.bytes, ncclUint8, x.peer, comm->comm, st));
    for (const Xfer &x : recvs) NCCL_TRY(a.Recv(x.buf, x.bytes, ncclUint8, x.peer, comm->comm, st));
    NCCL_TRY(a.GroupEnd());
  }
  // 5. local merge of this rank's range (stream ordered after the exchange)
#undef NCCL_TRY
  return obgpu_merge_decoded(ctx, runs.data(), n_runs_total, n_cols, default_vals, default_null, out);
}

}  // extern "C"
