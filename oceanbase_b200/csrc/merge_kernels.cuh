// merge_kernels.cuh -- major-compaction merge on the device (included at the end of obgpu_scan.cu:
// it uses the batch / ctx internals and the prefix kernels of the scan).
//
// Reference path (include/obgpu_compaction.h has the file:line list): a loser tree pops the run
// heads in (rowkey ascending, newer table first) order, rows of one rowkey are fused newest first,
// delete rows are dropped. Here:
//   1. the K sorted runs are merged PAIRWISE with merge-path tiles (ceil(log2 K) passes over
//      (rowkey, source) pairs, ties resolved "newer run first"), which yields exactly the pop order
//      of the loser tree;
//   2. group heads (first element of a rowkey) decide emit / drop from the newest existing row;
//   3. an exclusive scan of the emit flags gives the dense output index;
//   4. every emitting head fuses its group column by column (first non-NOP cell newest -> oldest,
//      stopping at a delete row, defaults for what stays NOP) and writes the output row.
// HBM-bound: (rowkey, source) pairs are read and written once per pass (16 B per row per pass),
// payload cells are gathered once.
#pragma once
#include <deque>
#include <functional>

#include <cub/device/device_radix_sort.cuh>

namespace mrg {

constexpr int kTile = 2048;     // outputs per CTA in a merge pass
constexpr int kThreads = 256;
constexpr int kVT = kTile / kThreads;
constexpr int kSrcShift = 40;   // source = run << 40 | row index inside the run
constexpr int kFuseTile = 1024;

struct Pair {        // one 2-way merge of a pass: A = [a0, a1), B = [b0, b1) of the input arrays
  int64_t a0, a1, b0, b1, out0;
  int64_t tile0;     // first tile of this pair in the pass's grid
};

struct RunsDev {
  const int64_t *const *key;    // [K]
  const uint8_t *const *flag;   // [K] (entries may be null)
  const int64_t *const *vals;   // [K * n_cols]
  const uint8_t *const *ext;    // [K * n_cols]
  const int64_t *const *more;   // [K * n_more]: rowkey columns after the first (composite rowkeys)
  int32_t n_runs, n_cols, n_more;
};

// Composite rowkeys: the merge passes carry the FIRST rowkey column next to the source; the remaining columns are
// looked up through the source only when the first column ties (ObStorageDatumUtils compares column by column too).
__device__ __forceinline__ int rest_cmp(const RunsDev &r, uint64_t sa, uint64_t sb) {
  const uint64_t idx_mask = (1ull << kSrcShift) - 1;
  const int ra = (int)(sa >> kSrcShift), rb = (int)(sb >> kSrcShift);
  const int64_t ia = (int64_t)(sa & idx_mask), ib = (int64_t)(sb & idx_mask);
  for (int c = 0; c < r.n_more; ++c) {
    const int64_t a = r.more[ra * r.n_more + c][ia], b = r.more[rb * r.n_more + c][ib];
    if (a != b) return a < b ? -1 : 1;
  }
  return 0;
}
__device__ __forceinline__ bool key_less(const RunsDev &r, int64_t ka, uint64_t sa, int64_t kb, uint64_t sb) {
  return ka < kb || (ka == kb && r.n_more > 0 && rest_cmp(r, sa, sb) < 0);
}
__device__ __forceinline__ bool key_equal(const RunsDev &r, int64_t ka, uint64_t sa, int64_t kb, uint64_t sb) {
  return ka == kb && (r.n_more == 0 || rest_cmp(r, sa, sb) == 0);
}

__global__ void __launch_bounds__(256) init_kernel(const int64_t *key, int64_t n, uint64_t run, int64_t *kout,
                                                   uint64_t *sout) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    kout[i] = key[i];
    sout[i] = (run << kSrcShift) | (uint64_t)i;
  }
}

// number of A elements among the first d outputs of merge(A, B), B first on equal keys
__device__ __forceinline__ int64_t merge_path_g(const RunsDev &r, const int64_t *a, const uint64_t *sa, int64_t na,
                                                const int64_t *b, const uint64_t *sb, int64_t nb, int64_t d) {
  int64_t lo = d > nb ? d - nb : 0, hi = d < na ? d : na;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (key_less(r, a[mid], sa[mid], b[d - 1 - mid], sb[d - 1 - mid])) lo = mid + 1; else hi = mid;
  }
  return lo;
}
__device__ __forceinline__ int merge_path_s(const RunsDev &r, const int64_t *a, const uint64_t *sa, int na, const int64_t *b,
                                            const uint64_t *sb, int nb, int d) {
  int lo = d > nb ? d - nb : 0, hi = d < na ? d : na;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (key_less(r, a[mid], sa[mid], b[d - 1 - mid], sb[d - 1 - mid])) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// Merge-path partition: one THREAD per tile start diagonal (all binary searches of a pass in flight together,
// instead of every merge CTA waiting on its own two searches). split[t] = A elements before tile t.
__global__ void __launch_bounds__(256) partition_kernel(const int64_t *__restrict__ kin, const uint64_t *__restrict__ sin, RunsDev runs,
                                                        const Pair *__restrict__ pairs, int n_pairs,
                                                        int64_t n_tiles, int64_t *__restrict__ split) {
  const int64_t tile = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tile >= n_tiles) return;
  int p = 0;
  while (p + 1 < n_pairs && pairs[p + 1].tile0 <= tile) ++p;
  const Pair pr = pairs[p];
  split[tile] = merge_path_g(runs, kin + pr.a0, sin + pr.a0, pr.a1 - pr.a0, kin + pr.b0, sin + pr.b0, pr.b1 - pr.b0,
                             (tile - pr.tile0) * kTile);
}

__global__ void __launch_bounds__(kThreads) pass_kernel(const int64_t *__restrict__ kin, const uint64_t *__restrict__ sin,
                                                        int64_t *__restrict__ kout, uint64_t *__restrict__ sout, RunsDev runs,
                                                        const Pair *__restrict__ pairs, int n_pairs,
                                                        const int64_t *__restrict__ split) {
  __shared__ int64_t s_key[kTile];
  __shared__ uint64_t s_src[kTile];
  const int tid = threadIdx.x;
  int p = 0;
  while (p + 1 < n_pairs && pairs[p + 1].tile0 <= (int64_t)blockIdx.x) ++p;
  const Pair pr = pairs[p];
  const int64_t na = pr.a1 - pr.a0, nb = pr.b1 - pr.b0;
  const int64_t d0 = ((int64_t)blockIdx.x - pr.tile0) * kTile;
  const int64_t d1 = d0 + kTile < na + nb ? d0 + kTile : na + nb;
  // this tile's end split is the next tile's start split, unless the tile closes its pair
  const int64_t i0 = split[blockIdx.x];
  const int64_t i1 = d1 == na + nb ? na : split[blockIdx.x + 1];
  const int64_t j0 = d0 - i0, j1 = d1 - i1;
  const int ca = (int)(i1 - i0), cb = (int)(j1 - j0), total = ca + cb;
  // stage: A part at [0, ca), B part at [ca, ca + cb)
  for (int k = tid; k < total; k += kThreads) {
    const int64_t g = k < ca ? pr.a0 + i0 + k : pr.b0 + j0 + (k - ca);
    s_key[k] = kin[g];
    s_src[k] = sin[g];
  }
  __syncthreads();
  // per-thread merge of kVT consecutive outputs
  const int od0 = tid * kVT < total ? tid * kVT : total;
  const int od1 = od0 + kVT < total ? od0 + kVT : total;
  int ia = merge_path_s(runs, s_key, s_src, ca, s_key + ca, s_src + ca, cb, od0);
  int ib = od0 - ia;
  int64_t rk[kVT];
  uint64_t rs[kVT];
#pragma unroll
  for (int k = 0; k < kVT; ++k) {
    if (od0 + k < od1) {
      const bool take_b = ib < cb && (ia >= ca || !key_less(runs, s_key[ia], s_src[ia], s_key[ca + ib], s_src[ca + ib]));
      const int at = take_b ? ca + ib : ia;
      rk[k] = s_key[at];
      rs[k] = s_src[at];
      if (take_b) ++ib; else ++ia;
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kVT; ++k) {
    if (od0 + k < od1) {
      s_key[od0 + k] = rk[k];
      s_src[od0 + k] = rs[k];
    }
  }
  __syncthreads();
  for (int k = tid; k < total; k += kThreads) {
    kout[pr.out0 + d0 + k] = s_key[k];
    sout[pr.out0 + d0 + k] = s_src[k];
  }
}

// ---- single-pass K-way merge (single-column rowkeys) ------------------------------------------------------------------
// The pairwise passes above read and write every (rowkey, source) pair ceil(log2 K) times. For a single rowkey column the
// K runs are merged in ONE pass instead, the device form of a K-way merge-path partition:
//   1. every run contributes the first rowkey of each chunk of S rows as a sample; the samples are radix-sorted;
//   2. every m-th sorted sample is a splitter: bucket b holds the rows of all runs with splitter[b] <= rowkey < splitter[b + 1]
//      (lower_bound of every splitter in every run). Rowkeys are unique inside a run, so a bucket holds at most
//      (m + 2 K) S rows -- m S on average -- and all rows of one rowkey, whichever runs they come from, share a bucket;
//   3. one CTA per bucket stages the K sorted segments in shared memory, ranks every row by binary searches in the other
//      segments (equal rowkeys: newer run first, the loser tree's pop order) and writes the bucket in merged order.
// S K = 1024 and m S = 1024: buckets average 1024 rows and never exceed 3072 (48 KB of rowkeys + sources).
constexpr int kBucketMean = 1024;
constexpr int kBucketCap = 3 * kBucketMean;
constexpr int kBucketThreads = 256;
constexpr int kBucketPer = 13;   // consecutive rows per thread (odd: no shared-memory bank conflicts); 256 x 13 >= kBucketCap
constexpr int kMaxRuns = 64;

struct BucketRuns {
  const int64_t *key[kMaxRuns];
  int64_t n[kMaxRuns];
  int64_t smp_off[kMaxRuns + 1];   // first sample of run r in the sample array
  int32_t n_runs, chunk;           // chunk = S
};

__global__ void __launch_bounds__(256) bucket_sample_kernel(const __grid_constant__ BucketRuns br, int64_t n_samples, int64_t *__restrict__ smp) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_samples) return;
  int r = 0;
  while (r + 1 < br.n_runs && br.smp_off[r + 1] <= j) ++r;
  smp[j] = br.key[r][(j - br.smp_off[r]) * br.chunk];
}

// bounds[b * K + r] = first row of run r in bucket b (b = 0 .. B; bucket B is the end sentinel)
__global__ void __launch_bounds__(256) bucket_bounds_kernel(const __grid_constant__ BucketRuns br, const int64_t *__restrict__ sorted, int every,
                                                            int64_t n_buckets, int64_t *__restrict__ bounds) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int K = br.n_runs;
  if (t >= (n_buckets + 1) * K) return;
  const int64_t b = t / K;
  const int r = (int)(t % K);
  int64_t lo = 0, hi = br.n[r];
  if (b == 0) hi = 0;
  else if (b == n_buckets) lo = hi;
  else {
    const int64_t q = sorted[b * every];
    const int64_t *k = br.key[r];
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (k[mid] < q) lo = mid + 1; else hi = mid;
    }
  }
  bounds[t] = lo;
}

__global__ void __launch_bounds__(256) bucket_size_kernel(const int64_t *__restrict__ bounds, int K, int64_t n_buckets, uint32_t *__restrict__ size,
                                                          int *__restrict__ status) {
  const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_buckets) return;
  int64_t tot = 0;
  for (int r = 0; r < K; ++r) tot += bounds[(b + 1) * K + r] - bounds[b * K + r];
  if (tot > kBucketCap) {   // impossible with unique rowkeys inside every run: the input breaks the merge's contract
    atomicOr(status, ST_CORRUPT);
    tot = 0;
  }
  size[b] = (uint32_t)tot;
}

__device__ __forceinline__ int flag_of(const RunsDev &r, uint64_t src) {
  const int run = (int)(src >> kSrcShift);
  const uint8_t *f = r.flag[run];
  return f ? (int)f[src & ((1ull << kSrcShift) - 1)] : OBGPU_DF_INSERT;
}

// One CTA per bucket: stage the K sorted segments in shared memory and merge them with ceil(log2 K) PAIRWISE merge-path levels that
// never leave shared memory (a thread produces kBucketPer consecutive outputs of a level: one binary search for its diagonal, then a
// serial two-way merge; equal rowkeys: the newer run first, the loser tree's pop order). The rows travel as (rowkey, position in the
// staged bucket); the source (run, row) is rebuilt from the position at the end. Then, still in shared memory: rowkey groups (they never
// straddle buckets), emit / drop from the newest existing row of each group, the rank of every emitting head inside the bucket.
// Written once: (rowkey, source, rank-or-0xffff) per row, cnt[b] = rows the bucket emits.
constexpr uint16_t kNoEmit = 0xffffu;

__global__ void __launch_bounds__(kBucketThreads) bucket_merge_kernel(const __grid_constant__ BucketRuns br, RunsDev runs,
                                                                      const int64_t *__restrict__ bounds, const uint32_t *__restrict__ size,
                                                                      const int64_t *__restrict__ out0, int64_t *__restrict__ kout,
                                                                      uint64_t *__restrict__ sout, uint16_t *__restrict__ erank, uint32_t *__restrict__ cnt,
                                                                      unsigned long long *__restrict__ stats, int *__restrict__ status) {
  extern __shared__ __align__(16) uint8_t bk_smem[];
  int64_t *s_k0 = reinterpret_cast<int64_t *>(bk_smem);
  int64_t *s_k1 = reinterpret_cast<int64_t *>(bk_smem + (size_t)kBucketCap * 8);
  uint16_t *s_t0 = reinterpret_cast<uint16_t *>(bk_smem + (size_t)kBucketCap * 16);
  uint16_t *s_t1 = reinterpret_cast<uint16_t *>(bk_smem + (size_t)kBucketCap * 18);
  uint8_t *s_run = bk_smem + (size_t)kBucketCap * 20;
  __shared__ int s_off[kMaxRuns + 1];
  __shared__ int64_t s_lb[kMaxRuns];
  __shared__ uint32_t s_wsum[kBucketThreads / 32];
  __shared__ const uint8_t *s_flag[kMaxRuns];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, K = br.n_runs;
  const int64_t b = blockIdx.x;
  const int total = (int)size[b];
  if (total == 0) {
    if (tid == 0) cnt[b] = 0;
    return;
  }
  if (tid < 32) {   // segment offsets: a warp scans the K <= 64 segment lengths
    int acc = 0;
    for (int r0 = 0; r0 < K; r0 += 32) {
      const int r = r0 + tid;
      const int64_t lb = r < K ? bounds[b * K + r] : 0;
      const int len = r < K ? (int)(bounds[(b + 1) * K + r] - lb) : 0;
      int inc = len;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, inc, o);
        if (tid >= o) inc += u;
      }
      if (r < K) { s_off[r] = acc + inc - len; s_lb[r] = lb; s_flag[r] = runs.flag[r]; }
      acc += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (tid == 0) s_off[K] = acc;
  }
  __syncthreads();
  for (int r = 0; r < K; ++r) {
    const int o = s_off[r], len = s_off[r + 1] - o;
    const int64_t *k = br.key[r] + s_lb[r];
    for (int i = tid; i < len; i += kBucketThreads) {
      s_k0[o + i] = k[i];
      s_t0[o + i] = (uint16_t)(o + i);
      s_run[o + i] = (uint8_t)r;
    }
  }
  __syncthreads();
  int64_t *kin = s_k0, *kdst = s_k1;
  uint16_t *tin = s_t0, *tdst = s_t1;
  // every thread takes the same share of the bucket (an odd number of rows: no shared-memory bank conflicts between the lanes'
  // strided accesses): 5 rows for the average bucket, 13 for a full one -- short serial chains, all warps busy
  const int per = ((total + kBucketThreads - 1) / kBucketThreads) | 1;
  const int x_begin = tid * per < total ? tid * per : total;
  const int x_end = x_begin + per < total ? x_begin + per : total;
  for (int w = 1; w < K; w <<= 1) {
    int x = x_begin;
    while (x < x_end) {
      // the segment holding position x (segments may be empty: last one starting at or before x), then its group of 2 w segments
      int lo = 0, hi = K;
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (s_off[mid] <= x) lo = mid; else hi = mid;
      }
      const int g0 = (lo / (2 * w)) * (2 * w);
      const int a0 = s_off[g0], a1 = s_off[g0 + w < K ? g0 + w : K], b1 = s_off[g0 + 2 * w < K ? g0 + 2 * w : K];
      const int na = a1 - a0, nb = b1 - a1;
      const int d = x - a0;
      int l = d > nb ? d - nb : 0, h = d < na ? d : na;   // merge path: rows of A among the first d outputs, B first on equal rowkeys
      while (l < h) {
        const int mid = (l + h) >> 1;
        if (kin[a0 + mid] < kin[a1 + d - 1 - mid]) l = mid + 1; else h = mid;
      }
      int ia = l, ib = d - l;
      const int stop = x_end < b1 ? x_end : b1;
      for (; x < stop; ++x) {
        const bool take_b = ib < nb && (ia >= na || !(kin[a0 + ia] < kin[a1 + ib]));
        const int at = take_b ? a1 + ib : a0 + ia;
        kdst[x] = kin[at];
        tdst[x] = tin[at];
        if (take_b) ++ib; else ++ia;
      }
    }
    __syncthreads();
    int64_t *tk = kin; kin = kdst; kdst = tk;
    uint16_t *tt = tin; tin = tdst; tdst = tt;
  }
  // kin / tin: the bucket in merged order. Group heads: the newest EXISTING row of the rowkey decides (delete -> the rowkey is dropped).
  uint32_t my_emit = 0, my_mask = 0;
  for (int x = x_begin; x < x_end; ++x) {
    const int64_t key = kin[x];
    if (x == 0 || kin[x - 1] != key) {
      bool decided = false;
      for (int j = x; j < total && kin[j] == key && !decided; ++j) {
        const int p = tin[j], r = s_run[p];
        const uint8_t *fl = s_flag[r];
        const int f = fl ? (int)fl[s_lb[r] + (p - s_off[r])] : OBGPU_DF_INSERT;
        if (f == OBGPU_DF_NOT_EXIST) continue;
        decided = true;
        if (f == OBGPU_DF_DELETE) atomicAdd(&stats[0], 1ull);
        else if (f == OBGPU_DF_INSERT || f == OBGPU_DF_UPDATE) { my_mask |= 1u << (x - x_begin); ++my_emit; }
        else atomicOr(status, ST_CORRUPT);
      }
    }
  }
  // exclusive scan of the per-thread emit counts (threads own consecutive rows: the scan order is the merged order)
  uint32_t inc = my_emit;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  if (lane == 31) s_wsum[warp] = inc;
  __syncthreads();
  uint32_t woff = 0, tot = 0;
#pragma unroll
  for (int k = 0; k < kBucketThreads / 32; ++k) {
    woff += k < warp ? s_wsum[k] : 0u;
    tot += s_wsum[k];
  }
  uint32_t rank = woff + inc - my_emit;
  for (int x = x_begin; x < x_end; ++x) {   // tdst is free: the ranks go there for the coalesced write below
    const bool e = (my_mask >> (x - x_begin)) & 1u;
    tdst[x] = e ? (uint16_t)rank : kNoEmit;
    rank += e;
  }
  __syncthreads();
  const int64_t o0 = out0[b];
  for (int i = tid; i < total; i += kBucketThreads) {
    const int p = tin[i], r = s_run[p];
    kout[o0 + i] = kin[i];
    sout[o0 + i] = ((uint64_t)r << kSrcShift) | (uint64_t)(s_lb[r] + (p - s_off[r]));
    erank[o0 + i] = tdst[i];
  }
  if (tid == 0) cnt[b] = tot;
}

// Fuse of one bucket's emitting heads (the groups of a bucket are complete inside it, every head knows its rank). No CTA barriers.
// Pass 1, a thread takes kFusePer rows at a time and requests everything they need together -- rank, rowkey, source, the next
// rowkey, then every column's ext byte and value -- before the first use: a head whose rowkey lives in one run only (nine in ten in
// a major merge) is finished there; a head that shares its rowkey is appended to its warp's list instead of being fused in place
// (one lane in ten would otherwise drag the whole warp through the general fold). Pass 2: the warp fuses its listed heads, a lane
// each, newest to oldest.
constexpr int kFusePer = 4;
constexpr int kFuseListCap = 512;   // listed heads per warp before an early flush
__device__ __forceinline__ void fuse_general_row(const RunsDev &runs, const int64_t *__restrict__ keys, const uint64_t *__restrict__ src,
                                                 int64_t i, int64_t end, int64_t o, const int64_t *__restrict__ default_vals,
                                                 const uint8_t *__restrict__ default_null, int64_t *const *__restrict__ out_vals,
                                                 uint8_t *const *__restrict__ out_null) {
  const uint64_t idx_mask = (1ull << kSrcShift) - 1;
  const int n_cols = runs.n_cols;
  const int64_t key = keys[i];
  int64_t jend = i;
  bool open = true;     // no delete row met yet
  for (int64_t j = i; j < end && keys[j] == key; ++j) {
    if (open) {
      if (flag_of(runs, src[j]) == OBGPU_DF_DELETE) open = false;
      else jend = j + 1;
    }
  }
  for (int c = 0; c < n_cols; ++c) {
    int64_t v = 0;
    uint8_t st = 2;  // NOP until a cell is found
    for (int64_t j = i; j < jend && st == 2; ++j) {
      const uint64_t s = src[j];
      if (flag_of(runs, s) == OBGPU_DF_NOT_EXIST) continue;
      const int run = (int)(s >> kSrcShift);
      const int64_t at = (int64_t)(s & idx_mask);
      const uint8_t x = runs.ext[run * n_cols + c][at];
      if (x != 2) {
        st = x;
        v = x ? 0 : runs.vals[run * n_cols + c][at];
      }
    }
    if (st == 2) {  // ObMajorPartitionMergeFuser::end_fuse_row: the default row
      const bool dn = default_null ? default_null[c] != 0 : true;
      st = dn ? 1 : 0;
      v = dn ? 0 : (default_vals ? default_vals[c] : 0);
    }
    out_vals[c][o] = v;
    out_null[c][o] = st;
  }
}

__global__ void __launch_bounds__(256) fuse_bucket_kernel(const int64_t *__restrict__ keys, const uint64_t *__restrict__ src, RunsDev runs,
                                                          const uint16_t *__restrict__ erank, const int64_t *__restrict__ seg0,
                                                          const int64_t *__restrict__ out_off, const int64_t *__restrict__ default_vals,
                                                          const uint8_t *__restrict__ default_null, int64_t *__restrict__ out_key,
                                                          int64_t *const *__restrict__ out_vals, uint8_t *const *__restrict__ out_null,
                                                          unsigned long long *__restrict__ stats) {
  __shared__ uint16_t s_list[8][kFuseListCap];   // per warp: bucket-relative positions of the heads that need the general fold
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t begin = seg0[blockIdx.x], end = seg0[blockIdx.x + 1];
  const int64_t base_out = out_off[blockIdx.x];
  if (out_off[blockIdx.x + 1] == base_out) return;   // nothing to emit in this bucket
  const uint64_t idx_mask = (1ull << kSrcShift) - 1;
  const int n_cols = runs.n_cols;
  int n_list = 0;   // warp-uniform
  auto flush = [&]() {
    __syncwarp();
    for (int k = lane; k < n_list; k += 32) {
      const int64_t i = begin + s_list[warp][k];
      fuse_general_row(runs, keys, src, i, end, base_out + erank[i], default_vals, default_null, out_vals, out_null);
    }
    if (lane == 0 && n_list) atomicAdd(&stats[1], (unsigned long long)n_list);
    __syncwarp();
    n_list = 0;
  };
  for (int64_t w0 = begin + warp * 32; w0 < end; w0 += 256 * kFusePer) {   // warp-uniform trip count
    const int64_t i0 = w0 + lane;
    uint16_t rk[kFusePer];
    int64_t key[kFusePer], nkey[kFusePer];
    uint64_t ks[kFusePer];
#pragma unroll
    for (int u = 0; u < kFusePer; ++u) {
      const int64_t i = i0 + 256 * u;
      rk[u] = i < end ? erank[i] : kNoEmit;
    }
#pragma unroll
    for (int u = 0; u < kFusePer; ++u) {
      const int64_t i = i0 + 256 * u;
      if (rk[u] != kNoEmit) {
        key[u] = keys[i];
        ks[u] = src[i];
        nkey[u] = i + 1 < end ? keys[i + 1] : ~key[u];   // the bucket's last row has no successor: any value that differs
      }
    }
#pragma unroll
    for (int u = 0; u < kFusePer; ++u) {
      const int64_t i = i0 + 256 * u;
      const bool emits = rk[u] != kNoEmit;
      const bool general = emits && nkey[u] == key[u];
      const uint32_t gb = __ballot_sync(0xffffffffu, general);
      if (general) s_list[warp][n_list + __popc(gb & ((1u << lane) - 1u))] = (uint16_t)(i - begin);
      n_list += __popc(gb);
      if (emits) {
        const int64_t o = base_out + rk[u];
        out_key[o] = key[u];
        if (!general) {   // the rowkey lives in one run: that row exists (it emitted) and nothing is fused
          const int run = (int)(ks[u] >> kSrcShift);
          const int64_t at = (int64_t)(ks[u] & idx_mask);
          for (int c0 = 0; c0 < n_cols; c0 += 4) {
            uint8_t x[4];
            int64_t v[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              if (c0 + q < n_cols) {
                x[q] = runs.ext[run * n_cols + c0 + q][at];
                v[q] = runs.vals[run * n_cols + c0 + q][at];
              }
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              if (c0 + q < n_cols) {
                const int c = c0 + q;
                uint8_t st = x[q];
                int64_t val = st ? 0 : v[q];
                if (st == 2) {   // NOP everywhere: the default row (ObMajorPartitionMergeFuser::end_fuse_row)
                  const bool dn = default_null ? default_null[c] != 0 : true;
                  st = dn ? 1 : 0;
                  val = dn ? 0 : (default_vals ? default_vals[c] : 0);
                }
                out_vals[c][o] = val;
                out_null[c][o] = st;
              }
            }
          }
        }
      }
      if (n_list > kFuseListCap - 32) flush();
    }
  }
  flush();
}

// Per element: is it the head of its rowkey group, and does the group emit a row? (decided by the
// newest row that exists: delete -> dropped, insert / update -> emitted.) Writes emit[i] and the
// number of emitting heads of the tile.
__global__ void __launch_bounds__(256) head_kernel(const int64_t *__restrict__ keys, const uint64_t *__restrict__ src, int64_t n,
                                                   RunsDev runs, uint8_t *__restrict__ emit, uint32_t *__restrict__ tile_count,
                                                   unsigned long long *__restrict__ stats, int *__restrict__ status) {
  __shared__ uint32_t s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  uint32_t mine = 0;
  for (int k = 0; k < kFuseTile / 256; ++k) {
    const int64_t i = (int64_t)blockIdx.x * kFuseTile + k * 256 + threadIdx.x;
    if (i >= n) break;
    const int64_t key = keys[i];
    const uint64_t ksrc = src[i];
    uint8_t e = 0;
    if (i == 0 || !key_equal(runs, keys[i - 1], src[i - 1], key, ksrc)) {
      bool decided = false;
      for (int64_t j = i; j < n && key_equal(runs, keys[j], src[j], key, ksrc) && !decided; ++j) {
        const int f = flag_of(runs, src[j]);
        if (f == OBGPU_DF_NOT_EXIST) continue;
        decided = true;
        if (f == OBGPU_DF_DELETE) atomicAdd(&stats[0], 1ull);
        else if (f == OBGPU_DF_INSERT || f == OBGPU_DF_UPDATE) e = 1;
        else atomicOr(status, ST_CORRUPT);
      }
    }
    emit[i] = e;
    mine += e;
  }
  atomicAdd(&s_cnt, mine);
  __syncthreads();
  if (threadIdx.x == 0) tile_count[blockIdx.x] = s_cnt;
}

// Emitting heads fuse their group and write the output row at tile_off[tile] + rank inside the tile.
__global__ void __launch_bounds__(256) fuse_kernel(const int64_t *__restrict__ keys, const uint64_t *__restrict__ src, int64_t n,
                                                   RunsDev runs, const uint8_t *__restrict__ emit,
                                                   const int64_t *__restrict__ tile_off, const int64_t *__restrict__ default_vals,
                                                   const uint8_t *__restrict__ default_null, int64_t *__restrict__ out_key,
                                                   int64_t *const *__restrict__ out_vals, uint8_t *const *__restrict__ out_null,
                                                   int64_t *const *__restrict__ out_more, unsigned long long *__restrict__ stats) {
  __shared__ uint32_t s_warp[8];
  __shared__ uint32_t s_base;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_base = 0;
  __syncthreads();
  const int64_t base_out = tile_off[blockIdx.x];
  for (int k = 0; k < kFuseTile / 256; ++k) {
    const int64_t i = (int64_t)blockIdx.x * kFuseTile + k * 256 + tid;
    const uint32_t e = i < n ? emit[i] : 0u;
    // rank among the emitting heads of this 256-element slice
    const uint32_t bal = __ballot_sync(0xffffffffu, e != 0);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    uint32_t woff = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      woff += w < warp ? s_warp[w] : 0u;
      tot += s_warp[w];
    }
    const uint32_t rank = s_base + woff + __popc(bal & ((1u << lane) - 1u));
    __syncthreads();
    if (tid == 0) s_base += tot;
    if (e) {
      const int64_t o = base_out + rank;
      const int64_t key = keys[i];
      const uint64_t ksrc = src[i];
      out_key[o] = key;
      for (int c = 0; c < runs.n_more; ++c)
        out_more[c][o] = runs.more[(int)(ksrc >> kSrcShift) * runs.n_more + c][(int64_t)(ksrc & ((1ull << kSrcShift) - 1))];
      // rows of the group, newest first; the fuse stops at a delete row (final_result)
      int64_t jend = i;
      int group = 0;        // iters sharing this rowkey (minimum_iters_.count())
      bool open = true;     // no delete row met yet
      for (int64_t j = i; j < n && key_equal(runs, keys[j], src[j], key, ksrc); ++j) {
        ++group;
        if (open) {
          if (flag_of(runs, src[j]) == OBGPU_DF_DELETE) open = false;
          else jend = j + 1;
        }
      }
      const uint64_t idx_mask = (1ull << kSrcShift) - 1;
      for (int c = 0; c < runs.n_cols; ++c) {
        int64_t v = 0;
        uint8_t st = 2;  // NOP until a cell is found
        for (int64_t j = i; j < jend && st == 2; ++j) {
          const uint64_t s = src[j];
          if (flag_of(runs, s) == OBGPU_DF_NOT_EXIST) continue;
          const int run = (int)(s >> kSrcShift);
          const int64_t at = (int64_t)(s & idx_mask);
          const uint8_t x = runs.ext[run * runs.n_cols + c][at];
          if (x != 2) {
            st = x;
            v = x ? 0 : runs.vals[run * runs.n_cols + c][at];
          }
        }
        if (st == 2) {  // ObMajorPartitionMergeFuser::end_fuse_row: default row
          const bool dn = default_null ? default_null[c] != 0 : true;
          st = dn ? 1 : 0;
          v = dn ? 0 : (default_vals ? default_vals[c] : 0);
        }
        out_vals[c][o] = v;
        out_null[c][o] = st;
      }
      if (group > 1) atomicAdd(&stats[1], 1ull);
    }
    __syncthreads();
  }
}

// ---- run decode: every cell of up to kMaxDecodeCols integer columns of a batch -> (value, ext) ---------
constexpr int kMaxDecodeCols = 16;
// String-class cells are decoded to a REFERENCE into the run's page batch: (tag << 58) | (byte offset of the cell
// inside the batch image << 22) | length. The merge moves these 64-bit images like integer cells; the tag (the
// run index) tells after the merge which image a reference points into.
constexpr int kRefTagShift = 58, kRefOffShift = 22;
constexpr uint64_t kRefLenMask = (1ull << kRefOffShift) - 1, kRefOffMask = (1ull << (kRefTagShift - kRefOffShift)) - 1;

struct DecodeCols {
  int32_t n;
  uint32_t string_tag;
  int32_t col[kMaxDecodeCols];
  int64_t *vals[kMaxDecodeCols];
  uint8_t *ext[kMaxDecodeCols];
};

__global__ void __launch_bounds__(128) decode_cols_kernel(const uint8_t *__restrict__ image, const BlockRec *__restrict__ recs,
                                                          const ColDesc *__restrict__ plans, int max_cols,
                                                          const __grid_constant__ DecodeCols dc,
                                                          const int64_t *__restrict__ row_start, int *__restrict__ status) {
  __shared__ ColDesc s_d[kMaxDecodeCols];
  const int block = blockIdx.x;
  const BlockRec rec = recs[block];
  constexpr int kPieces = (int)(sizeof(ColDesc) / 16);
  for (int k = threadIdx.x; k < dc.n * kPieces; k += blockDim.x)
    reinterpret_cast<uint4 *>(s_d)[k] =
        reinterpret_cast<const uint4 *>(plans + (int64_t)block * max_cols + dc.col[k / kPieces])[k % kPieces];
  __syncthreads();
  if (rec.rows == 0) {
    if (threadIdx.x == 0) atomicOr(status, ST_CORRUPT);
    return;
  }
  BlockView b;
  const uint8_t *s = image + rec.off;
  view_from_rec(rec, s, b);
  const int64_t row0 = row_start[block];
  for (int c = 0; c < dc.n; ++c) {
    const ColDesc &d = s_d[c];
    if (!d.ok) {
      if (threadIdx.x == 0) atomicOr(status, ST_UNSUPPORTED);
      continue;
    }
    int64_t *ov = dc.vals[c] + row0;
    uint8_t *oe = dc.ext[c] + row0;
    if (d.sc == 5 || d.kind == K_VARSTR) {
      // strings -> references; var-stored integers -> value image; NULL / NOP from the stored ext value
      for (uint32_t row = threadIdx.x; row < rec.rows; row += blockDim.x) {
        uint64_t v = 0;
        uint8_t e = 0;
        bool is_null;
        if (d.sc == 5) {
          uint32_t cell, len;
          str_cell(b, d, nullptr, row, cell, len, is_null);
          if (!is_null) {
            const uint64_t off = rec.off + (uint64_t)cell;
            if (off > kRefOffMask || len > kRefLenMask) atomicOr(status, ST_UNSUPPORTED);
            v = ((uint64_t)dc.string_tag << kRefTagShift) | (off << kRefOffShift) | (uint64_t)len;
          }
        } else {
          v = int_cell(b, d, nullptr, row, is_null);
          if (d.elem_len == 4) v &= 0xffffffffull;
          else if (d.elem_len == 1) v &= 0xffull;
        }
        if (is_null) {
          e = 1;
          v = 0;
          if (is_dict_kind(d)) {
            if (ref_of(s, d, nullptr, row) > d.dict_count) e = 2;                     // ref == count + 1: NOP
          } else if (d.kind == K_VARSTR && d.var_ext_in_row) {
            const uint32_t rib = b.row_index_byte;
            const uint32_t ro = (uint32_t)ld_bytes(s, b.row_index_off + row * rib, rib);
            if (ld_bits32(s, (b.row_data_off + ro) * 8u + d.ext_index, d.ext_bit) == STORED_NOPE) e = 2;
          } else if (d.kind == K_FIXSTR && d.ext_bit && !b.is_cs) {
            if (ld_bits32(s, d.ext_bit_off + row * d.ext_bit, d.ext_bit) == STORED_NOPE) e = 2;
          }
        }
        ov[row] = (int64_t)v;
        oe[row] = e;
      }
      continue;
    }
    const bool plain = d.kind == K_BITS && d.ext_bit == 0 && !d.var_is_last && !d.sign_fix && d.elem_len == 8;
    for (uint32_t row = threadIdx.x; row < rec.rows; row += blockDim.x) {
      uint64_t v = 0;
      uint8_t e = 0;
      if (plain) {
        v = ld_bits(s, d.val_bit + row * d.stride, d.width) + d.base;
      } else if (is_dict_kind(d)) {
        const uint32_t ref = ref_of(s, d, nullptr, row);
        if (ref >= d.dict_count) e = ref == d.dict_count ? 1 : 2;
        else v = dict_int(s, d, ref);
      } else {
        if (d.ext_bit) {
          const uint32_t x = ld_bits32(s, d.ext_bit_off + ext_row(d, row) * d.ext_bit, d.ext_bit);
          e = x == STORED_NOT_EXT ? 0 : (x == STORED_NULL ? 1 : 2);
        }
        if (!e) {
          const uint64_t raw = ld_bits(s, d.val_bit + row * d.stride, d.width);
          if (null_replaced_on(d) && raw == null_replaced_raw(d)) e = 1;
          else {
            v = raw + d.base;
            if (d.sign_fix) v = sign_fix(d.int_mask, v);
          }
        }
      }
      if (d.elem_len == 4) v &= 0xffffffffull;
      else if (d.elem_len == 1) v &= 0xffull;
      ov[row] = (int64_t)v;
      oe[row] = e;
    }
  }
}

__global__ void __launch_bounds__(256) narrow_flag_kernel(const int64_t *__restrict__ v, int64_t n, uint8_t *__restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (uint8_t)v[i];
}

// ---- merged string columns: references -> bytes -------------------------------------------------------------
__global__ void __launch_bounds__(256) ref_len_kernel(const int64_t *__restrict__ refs, const uint8_t *__restrict__ nulls, int64_t n,
                                                      uint32_t *__restrict__ lens) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) lens[i] = nulls[i] ? 0u : (uint32_t)((uint64_t)refs[i] & kRefLenMask);
}
// one warp per row: copies the cell from the image its tag names to heap[off[row] ..)
__global__ void __launch_bounds__(256) ref_gather_kernel(const int64_t *__restrict__ refs, const uint8_t *__restrict__ nulls, int64_t n,
                                                         const uint8_t *const *__restrict__ images,
                                                         const uint64_t *__restrict__ image_sizes, int n_images,
                                                         const int64_t *__restrict__ off, uint8_t *__restrict__ heap,
                                                         int *__restrict__ status) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n || nulls[row]) return;
  const uint64_t r = (uint64_t)refs[row];
  const int tag = (int)(r >> kRefTagShift);
  const uint32_t len = (uint32_t)(r & kRefLenMask);
  if (tag >= n_images || images[tag] == nullptr) {
    if (lane == 0) atomicOr(status, ST_CORRUPT);
    return;
  }
  const uint64_t at = (r >> kRefOffShift) & kRefOffMask;
  if (at + len > image_sizes[tag]) {   // not a reference into that image (e.g. an integer column was asked for)
    if (lane == 0) atomicOr(status, ST_CORRUPT);
    return;
  }
  const uint8_t *src = images[tag] + at;
  uint8_t *dst = heap + off[row];
  for (uint32_t k = (uint32_t)lane; k < len; k += 32u) dst[k] = src[k];
}

}  // namespace mrg

struct obgpu_merge_result {
  obgpu_ctx *ctx = nullptr;
  void *arena = nullptr;      // pair buffers, emit flags, tables, outputs
  int32_t n_cols = 0;
  int64_t in_rows = 0;
  int64_t *d_out_key = nullptr;
  std::vector<int64_t *> out_vals;
  std::vector<uint8_t *> out_null;
  int64_t *d_tile_off = nullptr;  // n_tiles + 1
  int64_t n_tiles = 0;
  unsigned long long *d_stats = nullptr;
  int *d_status = nullptr;
  bool info_valid = false;
  obgpu_merge_info info{};
  std::vector<const int64_t *> vals_view;
  std::vector<const uint8_t *> null_view;
  std::vector<const uint8_t *> string_images;   // tag -> device image the string references point into
  std::vector<uint64_t> string_image_sizes;     // bytes of each image (bounds of a reference)
  std::vector<uint8_t> col_is_string;           // known when the runs were decoded here (obgpu_merge_runs_keys)
  std::vector<int64_t *> out_more;              // rowkey columns after the first
};

extern "C" {

int obgpu_batch_decode_columns_tagged(obgpu_batch *b, int32_t n_cols, const int32_t *cols, int32_t string_tag,
                                      int64_t *const *dev_vals, uint8_t *const *dev_ext) {
  if (!b || n_cols <= 0 || n_cols > mrg::kMaxDecodeCols || !cols || !dev_vals || !dev_ext || string_tag < 0 ||
      string_tag >= OBGPU_MERGE_MAX_RUNS)
    return OBGPU_INVALID_ARGUMENT;
  mrg::DecodeCols dc{};
  dc.n = n_cols;
  dc.string_tag = (uint32_t)string_tag;
  for (int i = 0; i < n_cols; ++i) {
    if (cols[i] < 0 || (uint32_t)cols[i] >= b->max_cols || !dev_vals[i] || !dev_ext[i]) return OBGPU_INVALID_ARGUMENT;
    dc.col[i] = cols[i];
    dc.vals[i] = dev_vals[i];
    dc.ext[i] = dev_ext[i];
  }
  obgpu_ctx *ctx = b->ctx;
  cudaSetDevice(ctx->device);
  Scratch tmp(ctx);
  CUDA_TRY(ctx, tmp.alloc(64));
  int *d_status = tmp.at<int>(0);
  CUDA_TRY(ctx, cudaMemsetAsync(d_status, 0, 4, ctx->stream));
  mrg::decode_cols_kernel<<<b->n_blocks, 128, 0, ctx->stream>>>(b->d_image, b->d_recs, b->d_plans, (int)b->max_cols, dc,
                                                                b->d_row_start, d_status);
  ctx->launches++;
  int status = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&status, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return check_status(ctx, status);
}

int obgpu_batch_decode_columns(obgpu_batch *b, int32_t n_cols, const int32_t *cols, int64_t *const *dev_vals,
                               uint8_t *const *dev_ext) {
  return obgpu_batch_decode_columns_tagged(b, n_cols, cols, 0, dev_vals, dev_ext);
}

int obgpu_batch_decode_column(obgpu_batch *b, int32_t col, int64_t *dev_vals, uint8_t *dev_ext) {
  return obgpu_batch_decode_columns(b, 1, &col, &dev_vals, &dev_ext);
}

int obgpu_merge_decoded(obgpu_ctx *ctx, const obgpu_merge_run *runs, int32_t n_runs, int32_t n_cols,
                        const int64_t *default_vals, const uint8_t *default_null, obgpu_merge_result **out) {
  if (!ctx || !runs || !out || n_runs <= 0 || n_runs > OBGPU_MERGE_MAX_RUNS || n_cols < 0 || n_cols > OBGPU_MERGE_MAX_COLS)
    return OBGPU_INVALID_ARGUMENT;
  int64_t N = 0;
  const int n_more = runs[0].n_more_keys;
  if (n_more < 0 || n_more > OBGPU_MERGE_MAX_KEY_COLS - 1) return OBGPU_INVALID_ARGUMENT;
  for (int r = 0; r < n_runs; ++r) {
    if (runs[r].n_more_keys != n_more || (n_more > 0 && runs[r].n > 0 && !runs[r].more_keys)) return OBGPU_INVALID_ARGUMENT;
    if (runs[r].n < 0 || runs[r].n >= (1ll << mrg::kSrcShift) || (runs[r].n > 0 && !runs[r].key)) return OBGPU_INVALID_ARGUMENT;
    if (n_cols > 0 && runs[r].n > 0 && (!runs[r].vals || !runs[r].ext)) return OBGPU_INVALID_ARGUMENT;
    N += runs[r].n;
  }
  cudaSetDevice(ctx->device);
  std::unique_ptr<obgpu_merge_result> owner(new (std::nothrow) obgpu_merge_result());
  obgpu_merge_result *res = owner.get();
  if (!res) return OBGPU_ALLOCATE_MEMORY_FAILED;
  res->ctx = ctx;
  res->n_cols = n_cols;
  res->in_rows = N;
  const int64_t n_tiles = (N + mrg::kFuseTile - 1) / mrg::kFuseTile;
  res->n_tiles = n_tiles;
  // ---- arena -----------------------------------------------------------------------------------------
  Scratch arena(ctx);
  // single-column rowkeys merge in one pass (bucket_merge_kernel) and need no ping-pong buffers
  const bool bucket_path = n_more == 0 && n_runs >= 2 && n_runs <= mrg::kMaxRuns && N > 0 && getenv("OBGPU_MERGE_PAIRWISE") == nullptr;
  const size_t o_k0 = arena.take(bucket_path ? 0 : (size_t)N * 8);
  const size_t o_s0 = arena.take(bucket_path ? 0 : (size_t)N * 8);
  const size_t o_k1 = arena.take((size_t)N * 8);
  const size_t o_s1 = arena.take((size_t)N * 8);
  const size_t o_emit = arena.take((size_t)N * (bucket_path ? 2 : 1));   // emit flags, or the emitting heads' ranks inside their bucket
  const size_t o_stats = arena.take(64);
  const size_t tbl_entries = (size_t)n_runs * 2 + (size_t)n_runs * n_cols * 2 + (size_t)n_cols * 2 + (size_t)n_runs * n_more + (size_t)n_more;
  const size_t o_tbl = arena.take(tbl_entries * 8);
  const size_t o_def = arena.take((size_t)n_cols * 9 + 16);
  const size_t o_pairs = arena.take(sizeof(mrg::Pair) * (size_t)(n_runs + 1) * 8);
  const size_t max_tiles = (size_t)(N / mrg::kTile) + (size_t)n_runs + 2;
  const size_t o_split = arena.take((max_tiles + 1) * 8);
  const size_t o_okey = arena.take((size_t)N * 8);
  std::vector<size_t> o_ov((size_t)n_cols), o_on((size_t)n_cols);
  for (int c = 0; c < n_cols; ++c) o_ov[(size_t)c] = arena.take((size_t)N * 8);
  for (int c = 0; c < n_cols; ++c) o_on[(size_t)c] = arena.take((size_t)N);
  std::vector<size_t> o_om((size_t)n_more);
  for (int c = 0; c < n_more; ++c) o_om[(size_t)c] = arena.take((size_t)N * 8);
  // single-pass K-way merge (single-column rowkeys, see bucket_merge_kernel): samples, splitter bounds, bucket offsets
  int bk_chunk = 1;
  while (bk_chunk * 2 * n_runs <= mrg::kBucketMean) bk_chunk *= 2;
  const int bk_every = mrg::kBucketMean / bk_chunk;
  int64_t n_samples = 0;
  mrg::BucketRuns br{};
  if (bucket_path) {
    br.n_runs = n_runs;
    br.chunk = bk_chunk;
    for (int r = 0; r < n_runs; ++r) {
      br.key[r] = runs[r].key;
      br.n[r] = runs[r].n;
      br.smp_off[r] = n_samples;
      n_samples += (runs[r].n + bk_chunk - 1) / bk_chunk;
    }
    br.smp_off[n_runs] = n_samples;
  }
  const int64_t n_buckets = bucket_path ? std::max<int64_t>(1, (n_samples + bk_every - 1) / bk_every) : 0;
  size_t sort_tmp = 0;
  if (bucket_path)
    CUDA_TRY(ctx, cub::DeviceRadixSort::SortKeys(nullptr, sort_tmp, (const int64_t *)nullptr, (int64_t *)nullptr, n_samples, 0, 64, ctx->stream));
  const size_t o_smp = arena.take((size_t)n_samples * 8);
  const size_t o_sorted = arena.take((size_t)n_samples * 8);
  const size_t o_sorttmp = arena.take(sort_tmp);
  const size_t o_bounds = arena.take((size_t)(n_buckets + 1) * (size_t)n_runs * 8);
  const size_t o_bsize = arena.take((size_t)(n_buckets + 1) * 4);
  const size_t o_bout = arena.take((size_t)(n_buckets + 2) * 8);
  const size_t n_bchunks = (size_t)((n_buckets + kPrefixChunk - 1) / kPrefixChunk);
  const size_t o_bchunk = arena.take((n_bchunks + 1) * 8);
  const int64_t n_units = bucket_path ? n_buckets : n_tiles;   // emit counts / output offsets per bucket (single pass) or per tile
  const size_t o_cnt = arena.take(((size_t)n_units + 1) * 4);
  const size_t o_off = arena.take(((size_t)n_units + 2) * 8);
  const size_t n_chunks = (size_t)((n_units + kPrefixChunk - 1) / kPrefixChunk);
  const size_t o_chunk = arena.take((n_chunks + 1) * 8);
  if (bucket_path) res->n_tiles = n_units;
  arena.take(256);   // tail slack
  CUDA_TRY(ctx, arena.alloc());
  uint8_t *a = arena.p;
  int64_t *k0 = (int64_t *)(a + o_k0), *k1 = (int64_t *)(a + o_k1);
  uint64_t *s0 = (uint64_t *)(a + o_s0), *s1 = (uint64_t *)(a + o_s1);
  uint8_t *emit = a + o_emit;
  uint32_t *tile_cnt = (uint32_t *)(a + o_cnt);
  res->d_tile_off = (int64_t *)(a + o_off);
  res->d_stats = (unsigned long long *)(a + o_stats);
  res->d_status = (int *)(a + o_stats + 32);
  res->d_out_key = (int64_t *)(a + o_okey);
  CUDA_TRY(ctx, cudaMemsetAsync(a + o_stats, 0, 64, ctx->stream));
  // ---- pointer tables (host -> device) ------------------------------------------------------------------
  std::vector<uint64_t> tbl(tbl_entries, 0);
  size_t t = 0;
  const size_t t_key = t; for (int r = 0; r < n_runs; ++r) tbl[t++] = (uint64_t)runs[r].key;
  const size_t t_flag = t; for (int r = 0; r < n_runs; ++r) tbl[t++] = (uint64_t)runs[r].flag;
  const size_t t_vals = t;
  for (int r = 0; r < n_runs; ++r) for (int c = 0; c < n_cols; ++c) tbl[t++] = runs[r].n > 0 ? (uint64_t)runs[r].vals[c] : 0;
  const size_t t_ext = t;
  for (int r = 0; r < n_runs; ++r) for (int c = 0; c < n_cols; ++c) tbl[t++] = runs[r].n > 0 ? (uint64_t)runs[r].ext[c] : 0;
  const size_t t_ov = t;
  for (int c = 0; c < n_cols; ++c) { res->out_vals.push_back((int64_t *)(a + o_ov[(size_t)c])); tbl[t++] = (uint64_t)res->out_vals.back(); }
  const size_t t_on = t;
  for (int c = 0; c < n_cols; ++c) { res->out_null.push_back(a + o_on[(size_t)c]); tbl[t++] = (uint64_t)res->out_null.back(); }
  const size_t t_more = t;
  for (int r = 0; r < n_runs; ++r) for (int c = 0; c < n_more; ++c) tbl[t++] = runs[r].n > 0 ? (uint64_t)runs[r].more_keys[c] : 0;
  const size_t t_om = t;
  for (int c = 0; c < n_more; ++c) { res->out_more.push_back((int64_t *)(a + o_om[(size_t)c])); tbl[t++] = (uint64_t)res->out_more.back(); }
  uint64_t *d_tbl = (uint64_t *)(a + o_tbl);
  // defaults: [n_cols] int64 then [n_cols] bytes
  std::vector<uint8_t> defs((size_t)n_cols * 9 + 16, 0);
  for (int c = 0; c < n_cols; ++c) {
    const int64_t v = default_vals ? default_vals[c] : 0;
    memcpy(defs.data() + (size_t)c * 8, &v, 8);
    defs[(size_t)n_cols * 8 + (size_t)c] = default_null ? default_null[c] : 1;
  }
  // merge passes (host plan)
  struct Seg { int64_t begin, end; };
  std::vector<Seg> segs;
  {
    int64_t at = 0;
    for (int r = 0; r < n_runs; ++r) { segs.push_back({at, at + runs[r].n}); at += runs[r].n; }
  }
  std::vector<std::vector<mrg::Pair>> passes;
  {
    std::vector<Seg> cur = segs;
    while (cur.size() > 1) {
      std::vector<mrg::Pair> ps;
      std::vector<Seg> next;
      int64_t tile0 = 0;
      for (size_t i = 0; i < cur.size(); i += 2) {
        mrg::Pair p{};
        p.a0 = cur[i].begin; p.a1 = cur[i].end;   // A = older group
        if (i + 1 < cur.size()) { p.b0 = cur[i + 1].begin; p.b1 = cur[i + 1].end; }
        else { p.b0 = p.b1 = cur[i].end; }
        p.out0 = p.a0;
        p.tile0 = tile0;
        const int64_t tot = (p.a1 - p.a0) + (p.b1 - p.b0);
        tile0 += (tot + mrg::kTile - 1) / mrg::kTile;
        ps.push_back(p);
        next.push_back({p.a0, p.a0 + tot});
      }
      mrg::Pair sentinel{};
      sentinel.tile0 = tile0;
      ps.push_back(sentinel);
      passes.push_back(ps);
      cur = next;
    }
  }
  std::vector<mrg::Pair> all_pairs;
  std::vector<size_t> pass_at;
  for (auto &ps : passes) { pass_at.push_back(all_pairs.size()); all_pairs.insert(all_pairs.end(), ps.begin(), ps.end()); }
  // one pinned-free upload: tables, defaults, pairs are small pageable buffers -> synchronous staging is fine
  CUDA_TRY(ctx, cudaMemcpyAsync(d_tbl, tbl.data(), tbl_entries * 8, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(a + o_def, defs.data(), defs.size(), cudaMemcpyHostToDevice, ctx->stream));
  if (!all_pairs.empty())
    CUDA_TRY(ctx, cudaMemcpyAsync(a + o_pairs, all_pairs.data(), all_pairs.size() * sizeof(mrg::Pair), cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  // ---- launches ----------------------------------------------------------------------------------------------
  std::function<void(const mrg::RunsDev &)> bk_launch;
  if (bucket_path) {
    static bool attr_set = false;   // 63 KB of dynamic shared memory per CTA
    const size_t bk_smem = (size_t)mrg::kBucketCap * 21;
    if (!attr_set) {
      CUDA_TRY(ctx, cudaFuncSetAttribute(mrg::bucket_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bk_smem));
      attr_set = true;
    }
    int64_t *smp = (int64_t *)(a + o_smp), *sorted = (int64_t *)(a + o_sorted), *bounds = (int64_t *)(a + o_bounds), *bout = (int64_t *)(a + o_bout);
    uint32_t *bsize = (uint32_t *)(a + o_bsize);
    mrg::bucket_sample_kernel<<<(unsigned)((n_samples + 255) / 256), 256, 0, ctx->stream>>>(br, n_samples, smp);
    CUDA_TRY(ctx, cub::DeviceRadixSort::SortKeys(a + o_sorttmp, sort_tmp, (const int64_t *)smp, sorted, n_samples, 0, 64, ctx->stream));
    const int64_t nb_threads = (n_buckets + 1) * n_runs;
    mrg::bucket_bounds_kernel<<<(unsigned)((nb_threads + 255) / 256), 256, 0, ctx->stream>>>(br, sorted, bk_every, n_buckets, bounds);
    mrg::bucket_size_kernel<<<(unsigned)((n_buckets + 255) / 256), 256, 0, ctx->stream>>>(bounds, n_runs, n_buckets, bsize, res->d_status);
    obgpu_prefix_local_kernel<<<(int)n_bchunks, 256, 0, ctx->stream>>>(bsize, (int)n_buckets, bout, (unsigned long long *)(a + o_bchunk));
    obgpu_prefix_fix_kernel<<<(int)n_bchunks + 1, 256, 0, ctx->stream>>>((int)n_buckets, (int)n_bchunks, bout, (const unsigned long long *)(a + o_bchunk));
    bk_launch = [=](const mrg::RunsDev &rd_) {   // after the pointer tables are described (rd below)
      mrg::bucket_merge_kernel<<<(unsigned)n_buckets, mrg::kBucketThreads, bk_smem, ctx->stream>>>(
          br, rd_, bounds, bsize, bout, k1, s1, (uint16_t *)emit, tile_cnt, res->d_stats, res->d_status);
    };
    ctx->launches += 9;
  }
  for (int r = 0; r < n_runs && !bucket_path; ++r) {
    if (runs[r].n == 0) continue;
    mrg::init_kernel<<<(unsigned)((runs[r].n + 255) / 256), 256, 0, ctx->stream>>>(runs[r].key, runs[r].n, (uint64_t)r,
                                                                                 k0 + segs[(size_t)r].begin, s0 + segs[(size_t)r].begin);
    ctx->launches++;
  }
  mrg::RunsDev rd;
  rd.key = (const int64_t *const *)(d_tbl + t_key);
  rd.flag = (const uint8_t *const *)(d_tbl + t_flag);
  rd.vals = (const int64_t *const *)(d_tbl + t_vals);
  rd.ext = (const uint8_t *const *)(d_tbl + t_ext);
  rd.more = (const int64_t *const *)(d_tbl + t_more);
  rd.n_runs = n_runs;
  rd.n_cols = n_cols;
  rd.n_more = n_more;
  int64_t *kin = k0, *kout = k1;
  uint64_t *sin = s0, *sout = s1;
  if (bucket_path) {   // already merged, in k1 / s1
    kin = k1;
    sin = s1;
  }
  for (size_t ps = 0; ps < passes.size() && !bucket_path; ++ps) {
    const int n_pairs = (int)passes[ps].size() - 1;
    const int64_t tiles = passes[ps].back().tile0;
    if (tiles > 0) {
      int64_t *split = (int64_t *)(a + o_split);
      mrg::partition_kernel<<<(unsigned)((tiles + 255) / 256), 256, 0, ctx->stream>>>(
          kin, sin, rd, (const mrg::Pair *)(a + o_pairs) + pass_at[ps], n_pairs, tiles, split);
      mrg::pass_kernel<<<(unsigned)tiles, mrg::kThreads, 0, ctx->stream>>>(
          kin, sin, kout, sout, rd, (const mrg::Pair *)(a + o_pairs) + pass_at[ps], n_pairs, split);
      ctx->launches += 2;
    }
    std::swap(kin, kout);
    std::swap(sin, sout);
  }
  if (bucket_path) {
    bk_launch(rd);
    const int nc = (int)n_chunks;
    obgpu_prefix_local_kernel<<<nc, 256, 0, ctx->stream>>>(tile_cnt, (int)n_buckets, res->d_tile_off, (unsigned long long *)(a + o_chunk));
    obgpu_prefix_fix_kernel<<<nc + 1, 256, 0, ctx->stream>>>((int)n_buckets, nc, res->d_tile_off, (const unsigned long long *)(a + o_chunk));
    mrg::fuse_bucket_kernel<<<(unsigned)n_buckets, 256, 0, ctx->stream>>>(
        kin, sin, rd, (const uint16_t *)emit, (const int64_t *)(a + o_bout), res->d_tile_off, (const int64_t *)(a + o_def),
        (const uint8_t *)(a + o_def + (size_t)n_cols * 8), res->d_out_key, (int64_t *const *)(d_tbl + t_ov), (uint8_t *const *)(d_tbl + t_on),
        res->d_stats);
    ctx->launches += 3;
  } else if (N > 0) {
    mrg::head_kernel<<<(unsigned)n_tiles, 256, 0, ctx->stream>>>(kin, sin, N, rd, emit, tile_cnt, res->d_stats, res->d_status);
    const int nc = (int)n_chunks;
    obgpu_prefix_local_kernel<<<nc, 256, 0, ctx->stream>>>(tile_cnt, (int)n_tiles, res->d_tile_off,
                                                          (unsigned long long *)(a + o_chunk));
    obgpu_prefix_fix_kernel<<<nc + 1, 256, 0, ctx->stream>>>((int)n_tiles, nc, res->d_tile_off,
                                                            (const unsigned long long *)(a + o_chunk));
    mrg::fuse_kernel<<<(unsigned)n_tiles, 256, 0, ctx->stream>>>(
        kin, sin, N, rd, emit, res->d_tile_off, (const int64_t *)(a + o_def), (const uint8_t *)(a + o_def + (size_t)n_cols * 8),
        res->d_out_key, (int64_t *const *)(d_tbl + t_ov), (uint8_t *const *)(d_tbl + t_on), (int64_t *const *)(d_tbl + t_om),
        res->d_stats);
    ctx->launches += 4;
  } else {
    CUDA_TRY(ctx, cudaMemsetAsync(res->d_tile_off, 0, 16, ctx->stream));
  }
  CUDA_TRY(ctx, cudaGetLastError());
  for (int c = 0; c < n_cols; ++c) { res->vals_view.push_back(res->out_vals[(size_t)c]); res->null_view.push_back(res->out_null[(size_t)c]); }
  res->arena = arena.release();
  *out = owner.release();
  return OBGPU_SUCCESS;
}

int obgpu_merge_runs(obgpu_ctx *ctx, obgpu_batch *const *batches, int32_t n_runs, int32_t rowkey_col, int32_t flag_col,
                     const int32_t *cols, int32_t n_cols, const int64_t *default_vals, const uint8_t *default_null,
                     obgpu_merge_result **out) {
  return obgpu_merge_runs_keys(ctx, batches, n_runs, &rowkey_col, 1, flag_col, cols, n_cols, default_vals, default_null, out);
}

int obgpu_merge_runs_keys(obgpu_ctx *ctx, obgpu_batch *const *batches, int32_t n_runs, const int32_t *rowkey_cols,
                          int32_t n_rowkey_cols, int32_t flag_col, const int32_t *cols, int32_t n_cols,
                          const int64_t *default_vals, const uint8_t *default_null, obgpu_merge_result **out) {
  if (!ctx || !batches || !out || n_runs <= 0 || n_runs > OBGPU_MERGE_MAX_RUNS || n_cols < 0 || !rowkey_cols ||
      n_rowkey_cols < 1 || n_rowkey_cols > OBGPU_MERGE_MAX_KEY_COLS ||
      n_cols + 1 + n_rowkey_cols > mrg::kMaxDecodeCols || (n_cols > 0 && !cols))
    return OBGPU_INVALID_ARGUMENT;
  const int n_more = n_rowkey_cols - 1;
  std::vector<std::vector<const int64_t *>> mores((size_t)n_runs);
  for (int r = 0; r < n_runs; ++r)
    if (!batches[r] || batches[r]->ctx != ctx) return OBGPU_INVALID_ARGUMENT;
  cudaSetDevice(ctx->device);
  std::deque<Scratch> bufs;   // freed on the stream after the merge kernels are enqueued
  std::vector<obgpu_merge_run> runs((size_t)n_runs);
  std::vector<std::vector<const int64_t *>> vals((size_t)n_runs);
  std::vector<std::vector<const uint8_t *>> exts((size_t)n_runs);
  for (int r = 0; r < n_runs; ++r) {
    obgpu_batch *b = batches[r];
    const int64_t n = b->total_rows;
    const int n_dec = n_rowkey_cols + (flag_col >= 0 ? 1 : 0) + n_cols;
    // one allocation per run: n_dec value arrays, n_dec ext arrays, the narrowed flag bytes
    Scratch &buf = bufs.emplace_back(ctx);
    size_t o_v[mrg::kMaxDecodeCols], o_e[mrg::kMaxDecodeCols];
    for (int i = 0; i < n_dec; ++i) o_v[i] = buf.take((size_t)n * 8);
    for (int i = 0; i < n_dec; ++i) o_e[i] = buf.take((size_t)n);
    const size_t o_flag = buf.take((size_t)n);
    buf.take(256);   // tail slack
    CUDA_TRY(ctx, buf.alloc());
    int32_t dcols[mrg::kMaxDecodeCols];
    int64_t *dv[mrg::kMaxDecodeCols];
    uint8_t *de[mrg::kMaxDecodeCols];
    int k = 0;
    dcols[k++] = rowkey_cols[0];
    if (flag_col >= 0) dcols[k++] = flag_col;
    for (int c = 0; c < n_cols; ++c) dcols[k++] = cols[c];
    for (int c = 0; c < n_more; ++c) dcols[k++] = rowkey_cols[1 + c];   // remaining rowkey columns last
    for (int i = 0; i < n_dec; ++i) {
      dv[i] = buf.at<int64_t>(o_v[i]);
      de[i] = buf.at<uint8_t>(o_e[i]);
    }
    uint8_t *flag8 = buf.at<uint8_t>(o_flag);
    if (n > 0) {
      const int ret = obgpu_batch_decode_columns_tagged(b, n_dec, dcols, r, dv, de);
      if (ret != OBGPU_SUCCESS) return ret;
    }
    obgpu_merge_run &run = runs[(size_t)r];
    run.n = n;
    run.key = dv[0];
    run.flag = nullptr;
    int at = 1;
    if (flag_col >= 0) {
      if (n > 0) {
        mrg::narrow_flag_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(dv[1], n, flag8);
        ctx->launches++;
      }
      run.flag = flag8;
      at = 2;
    }
    for (int c = 0; c < n_cols; ++c) {
      vals[(size_t)r].push_back(dv[at + c]);
      exts[(size_t)r].push_back(de[at + c]);
    }
    run.vals = vals[(size_t)r].data();
    run.ext = exts[(size_t)r].data();
    for (int c = 0; c < n_more; ++c) mores[(size_t)r].push_back(dv[at + n_cols + c]);
    run.more_keys = n_more > 0 ? mores[(size_t)r].data() : nullptr;
    run.n_more_keys = n_more;
  }
  const int ret = obgpu_merge_decoded(ctx, runs.data(), n_runs, n_cols, default_vals, default_null, out);
  if (ret != OBGPU_SUCCESS) return ret;
  // string references of run r carry tag r and point into that batch's image
  for (int r = 0; r < n_runs; ++r) {
    (*out)->string_images.push_back(batches[r]->d_image);
    (*out)->string_image_sizes.push_back((uint64_t)batches[r]->image_size);
  }
  for (int c = 0; c < n_cols; ++c) {
    const uint32_t col = (uint32_t)cols[c];
    const uint8_t t = col < batches[0]->col_types.size() ? batches[0]->col_types[col] : 0xff;
    (*out)->col_is_string.push_back(t != 0xff && obf::store_class_of(t) == 5);
  }
  return OBGPU_SUCCESS;
}

int obgpu_merge_result_set_string_images(obgpu_merge_result *res, const void *const *dev_images, const int64_t *image_sizes,
                                         int32_t n_images) {
  if (!res || n_images < 0 || n_images > OBGPU_MERGE_MAX_RUNS || (n_images > 0 && (!dev_images || !image_sizes)))
    return OBGPU_INVALID_ARGUMENT;
  res->string_images.clear();
  res->string_image_sizes.clear();
  for (int i = 0; i < n_images; ++i) {
    if (image_sizes[i] < 0) return OBGPU_INVALID_ARGUMENT;
    res->string_images.push_back((const uint8_t *)dev_images[i]);
    res->string_image_sizes.push_back((uint64_t)image_sizes[i]);
  }
  return OBGPU_SUCCESS;
}

int obgpu_merge_result_fetch_strings(obgpu_merge_result *res, int32_t col, int64_t row_begin, int64_t row_count,
                                     void *host_heap, int64_t heap_cap, int64_t *host_off, uint8_t *host_null,
                                     int64_t *heap_bytes) {
  if (!res || col < 0 || col >= res->n_cols || row_begin < 0 || row_count < 0 || !host_off || !heap_bytes) return OBGPU_INVALID_ARGUMENT;
  obgpu_merge_info info;
  int ret = obgpu_merge_result_info(res, &info);
  if (ret != OBGPU_SUCCESS) return ret;
  if (row_begin + row_count > info.out_rows) return OBGPU_INVALID_ARGUMENT;
  obgpu_ctx *ctx = res->ctx;
  cudaSetDevice(ctx->device);
  host_off[0] = 0;
  *heap_bytes = 0;
  if (row_count == 0) return OBGPU_SUCCESS;
  if (res->string_images.empty()) { ctx->err = "no page-batch images attached to the merge result"; return OBGPU_INVALID_ARGUMENT; }
  if (!res->col_is_string.empty() && !res->col_is_string[(size_t)col]) { ctx->err = "not a string column"; return OBGPU_INVALID_ARGUMENT; }
  const int64_t n = row_count;
  const int n_chunks = (int)((n + kPrefixChunk - 1) / kPrefixChunk);
  Scratch scratch(ctx);
  const size_t o_len = scratch.take((size_t)n * 4), o_off = scratch.take(((size_t)n + 1) * 8), o_chunk = scratch.take(((size_t)n_chunks + 2) * 8);
  const size_t o_img = scratch.take(res->string_images.size() * 8), o_isz = scratch.take(res->string_image_sizes.size() * 8);
  const size_t o_st = scratch.take(256);
  CUDA_TRY(ctx, scratch.alloc());
  uint8_t *tmp = scratch.p;
  const int64_t *refs = res->out_vals[(size_t)col] + row_begin;
  const uint8_t *nulls = res->out_null[(size_t)col] + row_begin;
  int64_t *d_off = (int64_t *)(tmp + o_off);
  CUDA_TRY(ctx, cudaMemsetAsync(tmp + o_st, 0, 4, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(tmp + o_img, res->string_images.data(), res->string_images.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(tmp + o_isz, res->string_image_sizes.data(), res->string_image_sizes.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  mrg::ref_len_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(refs, nulls, n, (uint32_t *)(tmp + o_len));
  obgpu_prefix_local_kernel<<<n_chunks, 256, 0, ctx->stream>>>((const uint32_t *)(tmp + o_len), (int)n, d_off,
                                                              (unsigned long long *)(tmp + o_chunk));
  obgpu_prefix_fix_kernel<<<n_chunks + 1, 256, 0, ctx->stream>>>((int)n, n_chunks, d_off, (const unsigned long long *)(tmp + o_chunk));
  ctx->launches += 3;
  CUDA_TRY(ctx, cudaMemcpyAsync(host_off, d_off, ((size_t)n + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (host_null) CUDA_TRY(ctx, cudaMemcpyAsync(host_null, nulls, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  const int64_t total = host_off[n];
  *heap_bytes = total;
  if (total > heap_cap || (total > 0 && !host_heap)) return OBGPU_BUF_NOT_ENOUGH;
  int status = 0;
  if (total > 0) {
    Scratch heap(ctx);
    CUDA_TRY(ctx, heap.alloc((size_t)total + 16));
    mrg::ref_gather_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, ctx->stream>>>(
        refs, nulls, n, (const uint8_t *const *)(tmp + o_img), (const uint64_t *)(tmp + o_isz), (int)res->string_images.size(), d_off,
        heap.p, (int *)(tmp + o_st));
    ctx->launches++;
    CUDA_TRY(ctx, cudaMemcpyAsync(host_heap, heap.p, (size_t)total, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(&status, tmp + o_st, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return check_status(ctx, status);
}

void obgpu_merge_result_free(obgpu_merge_result *res) {
  if (!res) return;
  cudaSetDevice(res->ctx->device);
  if (res->arena) cudaFreeAsync(res->arena, res->ctx->stream);
  delete res;
}

int obgpu_merge_result_info(obgpu_merge_result *res, obgpu_merge_info *info) {
  if (!res || !info) return OBGPU_INVALID_ARGUMENT;
  obgpu_ctx *ctx = res->ctx;
  cudaSetDevice(ctx->device);
  if (!res->info_valid) {
    unsigned long long st[2] = {0, 0};
    int64_t total = 0;
    int status = 0;
    CUDA_TRY(ctx, cudaMemcpyAsync(st, res->d_stats, 16, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(&status, res->d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(&total, res->d_tile_off + res->n_tiles, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    const int ret = check_status(ctx, status);
    if (ret != OBGPU_SUCCESS) return ret;
    res->info.in_rows = res->in_rows;
    res->info.out_rows = res->in_rows > 0 ? total : 0;
    res->info.dropped_deletes = (int64_t)st[0];
    res->info.fused_rows = (int64_t)st[1];
    res->info_valid = true;
  }
  *info = res->info;
  return OBGPU_SUCCESS;
}

int obgpu_merge_result_cols(obgpu_merge_result *res, const int64_t **key_dev, const int64_t *const **vals_dev,
                            const uint8_t *const **null_dev) {
  if (!res) return OBGPU_INVALID_ARGUMENT;
  if (key_dev) *key_dev = res->d_out_key;
  if (vals_dev) *vals_dev = res->vals_view.data();
  if (null_dev) *null_dev = res->null_view.data();
  return OBGPU_SUCCESS;
}

int obgpu_merge_result_fetch(obgpu_merge_result *res, int32_t col, int64_t row_begin, int64_t row_count,
                             int64_t *host_vals, uint8_t *host_null) {
  if (!res || col < -1 - (int32_t)res->out_more.size() || col >= res->n_cols || row_begin < 0 || row_count < 0)
    return OBGPU_INVALID_ARGUMENT;
  obgpu_merge_info info;
  const int ret = obgpu_merge_result_info(res, &info);
  if (ret != OBGPU_SUCCESS) return ret;
  if (row_begin + row_count > info.out_rows) return OBGPU_INVALID_ARGUMENT;
  obgpu_ctx *ctx = res->ctx;
  if (row_count == 0) return OBGPU_SUCCESS;
  const int64_t *src = col == -1 ? res->d_out_key : (col < -1 ? res->out_more[(size_t)(-col - 2)] : res->out_vals[(size_t)col]);
  if (host_vals) CUDA_TRY(ctx, cudaMemcpyAsync(host_vals, src + row_begin, (size_t)row_count * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (host_null) {
    if (col < 0) memset(host_null, 0, (size_t)row_count);
    else CUDA_TRY(ctx, cudaMemcpyAsync(host_null, res->out_null[(size_t)col] + row_begin, (size_t)row_count, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return OBGPU_SUCCESS;
}

}  // extern "C"
