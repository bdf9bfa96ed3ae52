// ORDER BY key, ... LIMIT k over a whole scan (obgpu_result_top_rows): the first k of the rows the scan selected, in the order of
// 1..4 sort keys, with ties broken by position (block, then row), and the output columns of those rows. Only the k rows cross PCIe.
// Every key and output cell is read through the block's decode plan (int_cell / str_cell), so any encoding the scan decodes works:
// no key table, unlike GROUP BY.
//
// A row's full sort key is read as a sequence of 64-bit ORDER WORDS, compared as unsigned numbers, first word first:
//   integer key   one word: gvals::order_key (the MIN / MAX order)
//   string key    words of 7 bytes each: bytes [7c, 7c + 7) big-endian in bits 63..8, zero-padded, and in the low byte how many
//                 bytes are left from 7c on, capped at 8 (8: more words follow). A proper prefix, or "ab" before "ab\0", then
//                 compares first; two strings are equal when every word is, and the word that ends them says so (low byte < 8).
//   DESC          the key's words complemented
//   position      the last word: block << 32 | row, unique
// NULL is no word: at a key's first word the candidates split into their NULL and non-NULL rows, placed by nulls_first.
//
// Selection (host loop, one LEVEL per word): the candidates are a list of positions, at first every selected row (list_kernel,
// a warp per block over the bitmap words). For the level's word, word_kernel materialises each candidate's word and NULL flag
// (8 + 1 bytes per candidate). A radix select of 8 passes of 8 bits (hist_kernel, one shared 256-bin histogram per CTA) finds the
// word T such that fewer than `need` non-NULL candidates are below it and at least `need` are at or below it. compact_kernel then
// moves the candidates below T to the kept list, drops those above, and keeps those equal to T as the next level's candidates
// (all of them kept instead when they fit). The next level reads the next word of those ties only: the next 7 bytes of the same
// string while T says more follow, else the next key, and after the last key the position. So a tie-heavy key costs one more
// level over its ties, not a sort of them, and the loop ends at the position word at the latest.
// Scratch: positions, next positions and words at 8 bytes and a flag byte per selected row (25 bytes a row), kept list k x 8.
//
// Set: the kept rows (at most 65 536) are gathered once into a self-contained set (SetLay: positions, and per key and output
// column NULL flags, values -- integer order keys or string offsets into the set's own heap -- and lengths), sorted by row index
// with cub::DeviceMergeSort and SetLess, which compares the stored keys and then position, and gathered again in that order.
// emit_kernel writes the fetch buffer from it. The host pipeline (obgpu_pipeline_top_rows) merges the sets of its batches with
// the same sort over at most 2k rows, k kept, after the batches have closed.
#pragma once

namespace topn {

constexpr int kMaxKeys = 4;
constexpr int kMaxOut = 16;
constexpr int64_t kMaxK = 65536;
constexpr int kThreads = 256;
enum : uint8_t { C_IN = 0, C_NEXT = 1, C_OUT = 2 };

struct Key {
  int32_t col, desc, nulls_first, str;
};

struct Cols {
  dictops::BlkArgs a;
  int n;
  int32_t col[kMaxKeys + kMaxOut];
  int32_t str[kMaxKeys + kMaxOut];
};

struct Cell {
  uint64_t v;     // integer: order key; string: image offset of the first byte
  uint32_t len;   // string bytes
  bool null;
};

// the cell of column col at row r of block b; the plan was checked by check_kernel
__device__ __forceinline__ Cell read_cell(const dictops::BlkArgs &a, int b, uint32_t r, int col, bool str) {
  const BlockRec rec = a.recs[b];
  BlockView bv;
  view_from_rec(rec, a.image + rec.off, bv);
  const ColDesc d = a.plans[(int64_t)b * a.max_cols + col];
  Cell c{0, 0, false};
  if (str) {
    uint32_t cell = 0;
    str_cell(bv, d, nullptr, r, cell, c.len, c.null);
    c.v = rec.off + cell;
  } else {
    c.v = gvals::order_key(d, int_cell(bv, d, nullptr, r, c.null));
  }
  return c;
}

// every block's plan of every key and output column decodes the column's class
__global__ void check_kernel(const __grid_constant__ Cols p, int n_blocks, int *status) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_blocks) return;
  for (int i = 0; i < p.n; ++i) {
    const ColDesc d = p.a.plans[(int64_t)b * p.a.max_cols + p.col[i]];
    if (!d.ok || (d.sc == 5) != (p.str[i] != 0)) { atomicOr(status, ST_UNSUPPORTED); return; }
  }
}

// the selected rows' positions, in no fixed order: a warp per block, one atomic per block; [0] of ctr counts them
__global__ void list_kernel(const BlockRec *recs, int n_blocks, const uint32_t *bitmap, unsigned long long *ctr, uint64_t cap,
                            uint64_t *pos, int *status) {
  const int lane = threadIdx.x & 31;
  for (int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < n_blocks; b += (gridDim.x * blockDim.x) >> 5) {
    const BlockRec rec = recs[b];
    const uint32_t rows = rec.rows;
    const auto word = [&](uint32_t r0) -> uint32_t {
      const uint32_t valid = rows - r0 >= 32u ? ~0u : (1u << (rows - r0)) - 1u;
      return bitmap ? bitmap[rec.bm_word_off + (r0 >> 5)] & valid : valid;
    };
    uint32_t n = 0;
    for (uint32_t r0 = (uint32_t)lane * 32u; r0 < rows; r0 += 32u * 32u) n += __popc(word(r0));
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(~0u, n, o);
    unsigned long long base = 0;
    if (lane == 0 && n) base = atomicAdd(ctr, (unsigned long long)n);
    base = __shfl_sync(~0u, base, 0);
    if (base + n > cap) { if (lane == 0) atomicOr(status, ST_CORRUPT); continue; }
    for (uint32_t r0 = 0; r0 < rows; r0 += 32u) {
      const uint32_t w = word(r0);
      if ((w >> lane) & 1u) pos[base + __popc(w & ((1u << lane) - 1u))] = ((uint64_t)b << 32) | (r0 + (uint32_t)lane);
      base += __popc(w);
    }
  }
}

__device__ __forceinline__ uint64_t bytes_be(const uint8_t *p, uint32_t nb) {   // nb (<= 8) bytes big-endian in the top bits
  uint64_t w = 0;
  for (uint32_t i = 0; i < nb; ++i) w |= (uint64_t)p[i] << (56 - 8 * i);
  return w;
}

// the order word of a candidate at one level: key `key` (its word `chunk` when a string), or the position when key < 0
struct WordArgs {
  dictops::BlkArgs a;
  const uint64_t *pos;
  int64_t n;
  Key key;
  int use_key;
  uint32_t chunk;
  uint64_t *words;
  uint8_t *nulls;
};

__global__ void __launch_bounds__(kThreads) word_kernel(const __grid_constant__ WordArgs p) {
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < p.n; j += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t ps = p.pos[j];
    if (!p.use_key) { p.words[j] = ps; p.nulls[j] = 0; continue; }
    const Cell c = read_cell(p.a, (int)(ps >> 32), (uint32_t)ps, p.key.col, p.key.str != 0);
    uint64_t w = c.v;
    if (p.key.str && !c.null) {
      const uint32_t at = 7u * p.chunk, left = c.len > at ? c.len - at : 0u, nb = left < 7u ? left : 7u;
      w = (bytes_be(p.a.image + c.v + at, nb) & ~0xffull) | (left < 8u ? left : 8u);
    }
    p.words[j] = c.null ? 0ull : p.key.desc ? ~w : w;
    p.nulls[j] = c.null ? 1 : 0;
  }
}

// 256-bin histogram of the byte at `shift` of the non-NULL words whose bits under `mask` equal `prefix`; hist[256]: NULL rows.
// The lanes of a warp that fall in one bin add once (a low-cardinality key puts nearly every row in one or two bins)
__global__ void __launch_bounds__(kThreads) hist_kernel(const uint64_t *words, const uint8_t *nulls, int64_t n, uint64_t prefix, uint64_t mask,
                                                        int shift, unsigned long long *hist) {
  __shared__ unsigned int h[257];
  for (int i = threadIdx.x; i < 257; i += blockDim.x) h[i] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int64_t j0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); j0 < n; j0 += (int64_t)gridDim.x * blockDim.x) {
    const int64_t j = j0 + lane;
    uint32_t bin = 257;   // none
    if (j < n) {
      const uint64_t w = words[j];
      bin = nulls[j] ? 256u : (w & mask) == prefix ? (uint32_t)((w >> shift) & 0xffu) : 257u;
    }
    const uint32_t peers = __match_any_sync(~0u, bin);
    if (bin < 257 && lane == __ffs(peers) - 1) atomicAdd(&h[bin], (unsigned)__popc(peers));
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 257; i += blockDim.x)
    if (h[i]) atomicAdd(&hist[i], (unsigned long long)h[i]);
}

// each candidate to the kept list (C_IN), the next level (C_NEXT) or nowhere, by the bits of its word under `mask` against T
// (every bit once the select has run all its passes); ctr: [kept, next]
struct CompactArgs {
  const uint64_t *pos, *words;
  const uint8_t *nulls;
  int64_t n;
  uint64_t T, mask;
  uint8_t lt, eq, gt, null;
  uint64_t *kept, *next;
  unsigned long long *ctr;
};

__global__ void __launch_bounds__(kThreads) compact_kernel(const __grid_constant__ CompactArgs p) {
  const int lane = threadIdx.x & 31;
  for (int64_t j0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); j0 < p.n; j0 += (int64_t)gridDim.x * blockDim.x) {
    const int64_t j = j0 + lane;
    uint8_t cls = C_OUT;
    if (j < p.n) {
      const uint64_t w = p.words[j] & p.mask;
      cls = p.nulls[j] ? p.null : w < p.T ? p.lt : w == p.T ? p.eq : p.gt;
    }
    for (int c = 0; c < 2; ++c) {
      const uint32_t m = __ballot_sync(~0u, cls == c);
      if (!m) continue;
      unsigned long long base = 0;
      if (lane == 0) base = atomicAdd(&p.ctr[c], (unsigned long long)__popc(m));
      base = __shfl_sync(~0u, base, 0);
      if (cls == c) (c == C_IN ? p.kept : p.next)[base + __popc(m & ((1u << lane) - 1u))] = p.pos[j];
    }
  }
}

// A SET of rows, self-contained: everything ordering, merging and fetching them reads, so that it outlives the batch it came
// from (the pipeline merges the sets of batches already closed, as gmerge does with groups). Columns 0..n_keys-1 are the sort
// keys, then the output columns; per column and row a NULL flag, a value (integer: its order key; string: offset of its bytes in
// the set's heap) and a length (string bytes, 0 for integers and NULLs). One allocation:
//   [positions: n x 8][values: cols x n x 8][lengths: cols x n x 4][NULL flags: cols x n][heap]
struct SetLay {
  size_t val, len, null, heap, end;
  SetLay(int64_t n, int n_cols, int64_t heap_bytes) {
    const auto up = [](size_t x) { return (x + 15) & ~(size_t)15; };
    val = up((size_t)n * 8);
    len = val + up((size_t)n_cols * (size_t)n * 8);
    null = len + up((size_t)n_cols * (size_t)n * 4);
    heap = null + up((size_t)n_cols * (size_t)n);
    end = heap + (size_t)heap_bytes + 16;
  }
};

struct TopSet {
  void *mem = nullptr;
  int64_t n = 0, heap = 0;
  int n_cols = 0;
};

struct SetView {
  const uint64_t *pos, *val;
  const uint32_t *len;
  const uint8_t *null, *heap;
  int64_t n;
};

static SetView view_of(const TopSet &s) {
  const SetLay l(s.n, s.n_cols, s.heap);
  const uint8_t *m = (const uint8_t *)s.mem;
  return SetView{(const uint64_t *)m, (const uint64_t *)(m + l.val), (const uint32_t *)(m + l.len), m + l.null, m + l.heap, s.n};
}

// where a gather reads its rows: the batch's cells at the kept positions, or rows of one or two sets (row r of the pair: part 0's
// row r below n0, else part 1's row r - n0, whose block gets add1) picked by idx
struct Src {
  int from_sets;
  Cols cols;                   // batch: the columns; both: n and which are strings
  const uint64_t *kept;
  SetView part[2];
  int64_t n0;
  uint64_t add1;
  const uint32_t *idx;
};

__device__ __forceinline__ Cell src_cell(const Src &s, int c, int64_t q, const uint8_t *&base, uint64_t &pos) {
  if (!s.from_sets) {
    pos = s.kept[q];
    base = s.cols.a.image;
    return read_cell(s.cols.a, (int)(pos >> 32), (uint32_t)pos, s.cols.col[c], s.cols.str[c] != 0);
  }
  const int64_t r = s.idx[q];
  const int h = r < s.n0 ? 0 : 1;
  const SetView &v = s.part[h];
  const int64_t rr = h ? r - s.n0 : r, at = (int64_t)c * v.n + rr;
  pos = v.pos[rr] + (h ? s.add1 : 0ull);
  base = v.heap;
  return Cell{v.val[at], v.len[at], v.null[at] != 0};
}

struct SetArgs {
  Src s;
  int64_t n;
  int64_t *offs;               // [cols][n] + 1: string bytes of each cell, scanned into heap offsets
  uint64_t *pos, *val;
  uint32_t *len;
  uint8_t *null, *heap;
};

// LENS: every cell's string bytes; otherwise a thread per row writes its position and a thread per (column, row) its cell, string
// bytes copied into the set's heap
template <bool LENS>
__global__ void __launch_bounds__(kThreads) set_kernel(const __grid_constant__ SetArgs p) {
  const int64_t total = (int64_t)p.s.cols.n * p.n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < (LENS ? total : total + p.n); t += (int64_t)gridDim.x * blockDim.x) {
    const bool row = t >= total;
    const int c = row ? 0 : (int)(t / p.n);
    const int64_t q = row ? t - total : t - (int64_t)c * p.n;
    const uint8_t *base;
    uint64_t pos;
    const Cell cell = src_cell(p.s, c, q, base, pos);
    const bool str = p.s.cols.str[c] != 0;
    const uint32_t len = str && !cell.null ? cell.len : 0u;
    if (LENS) { p.offs[t] = len; continue; }
    if (row) { p.pos[q] = pos; continue; }
    p.null[t] = cell.null ? 1 : 0;
    p.len[t] = len;
    p.val[t] = str ? (uint64_t)p.offs[t] : cell.null ? 0ull : cell.v;
    for (uint32_t i = 0; i < len; ++i) p.heap[p.offs[t] + i] = base[cell.v + i];
  }
}

// the full order over the rows of one or two sets: the key columns, NULLs placed per key, then position
struct SetLess {
  SetView part[2];
  int64_t n0;
  uint64_t add1;
  int n_keys;
  Key key[kMaxKeys];
  __device__ bool operator()(uint32_t x, uint32_t y) const {
    const int hx = (int64_t)x < n0 ? 0 : 1, hy = (int64_t)y < n0 ? 0 : 1;
    const SetView &vx = part[hx], &vy = part[hy];
    const int64_t rx = hx ? x - n0 : x, ry = hy ? y - n0 : y;
    for (int i = 0; i < n_keys; ++i) {
      const bool nx = vx.null[i * vx.n + rx] != 0, ny = vy.null[i * vy.n + ry] != 0;
      if (nx || ny) {
        if (nx && ny) continue;
        return nx == (key[i].nulls_first != 0);
      }
      const uint64_t ax = vx.val[i * vx.n + rx], ay = vy.val[i * vy.n + ry];
      int c = 0;
      if (!key[i].str) {
        c = ax < ay ? -1 : ax > ay ? 1 : 0;
      } else {
        const uint32_t lx = vx.len[i * vx.n + rx], ly = vy.len[i * vy.n + ry], m = lx < ly ? lx : ly;
        for (uint32_t o = 0; o < m && !c; o += 8u) {
          const uint32_t nb = m - o < 8u ? m - o : 8u;
          const uint64_t bx = bytes_be(vx.heap + ax + o, nb), by = bytes_be(vy.heap + ay + o, nb);
          c = bx < by ? -1 : bx > by ? 1 : 0;
        }
        if (!c) c = lx < ly ? -1 : lx > ly ? 1 : 0;
      }
      if (c) return key[i].desc ? c > 0 : c < 0;
    }
    return vx.pos[rx] + (hx ? add1 : 0ull) < vy.pos[ry] + (hy ? add1 : 0ull);
  }
};

// byte offsets in a fetch buffer: [blocks: int32 x n][rows: int32 x n][values: n_out x (n + 1)][NULL flags: n_out x n][heap]
struct TopBuf {
  size_t rows, vals, nulls, heap, end;
  TopBuf(int64_t n, int n_out, int64_t heap_bytes) {
    rows = (((size_t)n * 4) + 15) & ~(size_t)15;
    vals = rows + rows;
    nulls = vals + (size_t)n_out * ((size_t)n + 1) * 8;
    heap = nulls + (((size_t)n_out * (size_t)n + 15) & ~(size_t)15);
    end = heap + (size_t)heap_bytes + 16;
  }
};

struct EmitArgs {
  SetView v;
  int n_keys, n_out;
  uint32_t str_mask, sgn_mask;   // bit j: output column j is a string / has its order key's sign bit flipped
  int64_t *offs;                 // [n_out][n] + 1: string bytes, scanned into heap offsets
  int32_t *blocks, *rows;
  int64_t *vals;
  uint8_t *nulls, *heap;
};

// a sorted set -> the fetch layout (obgpu_result_fetch_group_columns'): LENS first, then positions, NULL flags, integer images,
// string offsets and bytes
template <bool LENS>
__global__ void __launch_bounds__(kThreads) emit_kernel(const __grid_constant__ EmitArgs p) {
  const int64_t n = p.v.n, total = (int64_t)p.n_out * n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < (LENS ? total : total + n); t += (int64_t)gridDim.x * blockDim.x) {
    if (t >= total) {
      const int64_t q = t - total;
      p.blocks[q] = (int32_t)(p.v.pos[q] >> 32);
      p.rows[q] = (int32_t)(uint32_t)p.v.pos[q];
      continue;
    }
    const int j = (int)(t / n);
    const int64_t q = t - (int64_t)j * n, at = (int64_t)(p.n_keys + j) * n + q;
    if (LENS) { p.offs[t] = p.v.len[at]; continue; }
    const bool null = p.v.null[at] != 0;
    int64_t *vals = p.vals + (int64_t)j * (n + 1);
    p.nulls[t] = null ? 1 : 0;
    if ((p.str_mask >> j) & 1u) {
      const int64_t o = p.offs[t], len = p.v.len[at];
      vals[q] = o;
      if (q + 1 == n) vals[n] = o + len;
      for (int64_t i = 0; i < len; ++i) p.heap[o + i] = p.v.heap[p.v.val[at] + i];
    } else {
      const uint64_t key = p.v.val[at];
      vals[q] = null ? 0 : (int64_t)((p.sgn_mask >> j) & 1u ? key ^ (1ull << 63) : key);   // the order key undone
    }
  }
}

static unsigned grid_for(const obgpu_ctx *ctx, int64_t n) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + kThreads - 1) / kThreads, (int64_t)ctx->sm_count * 8));
}

// rows [0, n) of src into a new set (out.mem allocated here on ctx's stream); one synchronisation for the heap's size
static int gather_set(obgpu_ctx *ctx, const Src &src, int64_t n, TopSet &out) {
  const int64_t cells = (int64_t)src.cols.n * n;
  Scratch sc(ctx);   // [lengths][offsets][scan temporaries]
  size_t t_scan = 0;
  CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(nullptr, t_scan, (const int64_t *)nullptr, (int64_t *)nullptr, cells + 1, ctx->stream));
  const size_t o_lens = sc.take((size_t)(cells + 1) * 8), o_offs = sc.take((size_t)(cells + 1) * 8), o_tmp = sc.take(t_scan);
  CUDA_TRY(ctx, sc.alloc());
  SetArgs a{src, n, sc.at<int64_t>(o_lens), nullptr, nullptr, nullptr, nullptr, nullptr};
  CUDA_TRY(ctx, cudaMemsetAsync(a.offs + cells, 0, 8, ctx->stream));
  if (cells > 0) {
    set_kernel<true><<<grid_for(ctx, cells), kThreads, 0, ctx->stream>>>(a);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
  }
  CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(sc.p + o_tmp, t_scan, sc.at<int64_t>(o_lens), sc.at<int64_t>(o_offs), cells + 1, ctx->stream));
  int64_t *hp = (int64_t *)ctx->h_pinned;
  CUDA_TRY(ctx, cudaMemcpyAsync(hp, sc.at<int64_t>(o_offs) + cells, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  const int64_t heap = hp[0];
  const SetLay lay(n, src.cols.n, heap);
  Scratch mem(ctx);
  CUDA_TRY(ctx, mem.alloc(lay.end));
  a.offs = sc.at<int64_t>(o_offs);
  a.pos = mem.at<uint64_t>(0);
  a.val = mem.at<uint64_t>(lay.val);
  a.len = mem.at<uint32_t>(lay.len);
  a.null = mem.at<uint8_t>(lay.null);
  a.heap = mem.at<uint8_t>(lay.heap);
  if (n > 0) {
    set_kernel<false><<<grid_for(ctx, cells + n), kThreads, 0, ctx->stream>>>(a);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
  }
  out.mem = mem.release();
  out.n = n;
  out.heap = heap;
  out.n_cols = src.cols.n;
  return OBGPU_SUCCESS;
}

static void free_set(obgpu_ctx *ctx, TopSet &s) {
  if (s.mem) cudaFreeAsync(s.mem, ctx->stream);
  s = TopSet{};
}

// the first min(k, a.n + b.n) rows of sets a and b together (b's blocks + add_b), in order, as a new set; b may be empty
static int order_sets(obgpu_ctx *ctx, const TopSet &a, const TopSet &b, uint64_t add_b, int n_keys, const Key *keys, const int32_t *col_str,
                      int64_t k, TopSet &out) {
  const int64_t n = a.n + b.n, keep = std::min(k, n);
  SetLess less{};
  less.part[0] = view_of(a);
  less.part[1] = b.mem ? view_of(b) : less.part[0];
  less.n0 = a.n;
  less.add1 = add_b << 32;
  less.n_keys = n_keys;
  for (int i = 0; i < n_keys; ++i) less.key[i] = keys[i];
  Scratch sm(ctx);   // [row indices][sort temporaries]
  size_t t_sort = 0;
  if (n > 1) CUDA_TRY(ctx, cub::DeviceMergeSort::SortKeys(nullptr, t_sort, (uint32_t *)nullptr, n, less, ctx->stream));
  const size_t o_idx = sm.take((size_t)n * 4 + 4), o_tmp = sm.take(t_sort);
  CUDA_TRY(ctx, sm.alloc());
  uint32_t *idx = sm.at<uint32_t>(o_idx);
  if (n > 0) {
    gvals::iota_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(idx, (int)n);
    ctx->launches++;
  }
  if (n > 1) CUDA_TRY(ctx, cub::DeviceMergeSort::SortKeys(sm.p + o_tmp, t_sort, idx, n, less, ctx->stream));
  Src src{};
  src.from_sets = 1;
  src.cols.n = std::max(a.n_cols, b.n_cols);   // an empty set may have no columns yet
  for (int c = 0; c < src.cols.n; ++c) src.cols.str[c] = col_str[c];
  src.part[0] = less.part[0];
  src.part[1] = less.part[1];
  src.n0 = a.n;
  src.add1 = less.add1;
  src.idx = idx;
  return gather_set(ctx, src, keep, out);
}

// a sorted set -> a new fetch buffer (*buf, allocated here); one synchronisation for the heap's size
static int emit(obgpu_ctx *ctx, const TopSet &s, int n_keys, int n_out, uint32_t str_mask, uint32_t sgn_mask, void **buf, int64_t *heap_bytes) {
  const int64_t n = s.n, cells = (int64_t)n_out * n;
  Scratch sc(ctx);
  size_t t_scan = 0;
  CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(nullptr, t_scan, (const int64_t *)nullptr, (int64_t *)nullptr, cells + 1, ctx->stream));
  const size_t o_lens = sc.take((size_t)(cells + 1) * 8), o_offs = sc.take((size_t)(cells + 1) * 8), o_tmp = sc.take(t_scan);
  CUDA_TRY(ctx, sc.alloc());
  EmitArgs e{view_of(s), n_keys, n_out, str_mask, sgn_mask, sc.at<int64_t>(o_lens), nullptr, nullptr, nullptr, nullptr, nullptr};
  CUDA_TRY(ctx, cudaMemsetAsync(e.offs + cells, 0, 8, ctx->stream));
  if (cells > 0) {
    emit_kernel<true><<<grid_for(ctx, cells), kThreads, 0, ctx->stream>>>(e);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
  }
  CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(sc.p + o_tmp, t_scan, sc.at<int64_t>(o_lens), sc.at<int64_t>(o_offs), cells + 1, ctx->stream));
  int64_t *hp = (int64_t *)ctx->h_pinned;
  CUDA_TRY(ctx, cudaMemcpyAsync(hp, sc.at<int64_t>(o_offs) + cells, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  const int64_t heap = hp[0];
  const TopBuf lay(n, n_out, heap);
  Scratch out(ctx);
  CUDA_TRY(ctx, out.alloc(lay.end));
  CUDA_TRY(ctx, cudaMemsetAsync(out.p, 0, lay.nulls, ctx->stream));   // no row or no string column: values and offsets 0
  e.offs = sc.at<int64_t>(o_offs);
  e.blocks = out.at<int32_t>(0);
  e.rows = out.at<int32_t>(lay.rows);
  e.vals = out.at<int64_t>(lay.vals);
  e.nulls = out.at<uint8_t>(lay.nulls);
  e.heap = out.at<uint8_t>(lay.heap);
  if (n > 0) {
    emit_kernel<false><<<grid_for(ctx, cells + n), kThreads, 0, ctx->stream>>>(e);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
  }
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  *buf = out.release();
  *heap_bytes = heap;
  return OBGPU_SUCCESS;
}

// a fetch buffer -> caller host arrays; one synchronisation
static int fetch(obgpu_ctx *ctx, const void *buf, int64_t n, int n_out, int64_t heap, int32_t *host_block, int32_t *host_row, int64_t *host_vals,
                 uint8_t *host_nulls, void *host_heap) {
  const TopBuf lay(n, n_out, heap);
  const uint8_t *tb = (const uint8_t *)buf;
  if (n > 0) {
    CUDA_TRY(ctx, cudaMemcpyAsync(host_block, tb, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(host_row, tb + lay.rows, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (n_out > 0) {
    CUDA_TRY(ctx, cudaMemcpyAsync(host_vals, tb + lay.vals, lay.nulls - lay.vals, cudaMemcpyDeviceToHost, ctx->stream));
    if (n > 0) CUDA_TRY(ctx, cudaMemcpyAsync(host_nulls, tb + lay.nulls, (size_t)n_out * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (heap > 0) CUDA_TRY(ctx, cudaMemcpyAsync(host_heap, tb + lay.heap, (size_t)heap, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return OBGPU_SUCCESS;
}

// drops the previous call's rows: a refused call leaves none
static void drop_rows(obgpu_result *r) {
  if (r->d_top) cudaFreeAsync(r->d_top, r->ctx->stream);
  if (r->d_tset) cudaFreeAsync(r->d_tset, r->ctx->stream);
  r->d_top = r->d_tset = nullptr;
  r->top_rows = -1;
  r->top_heap = r->tset_heap = 0;
  r->top_n_out = 0;
}

// the result's rows as a set (the pipeline merges it); the result keeps them
static TopSet set_of(const obgpu_result *r) {
  TopSet s;
  s.mem = r->d_tset;
  s.n = r->top_rows;
  s.heap = r->tset_heap;
  s.n_cols = r->tset_cols;
  return s;
}


static int top_rows(obgpu_result *r, int64_t n_sel, const obgpu_sort_key *keys, int n_keys, const int32_t *out_cols, int n_out, int64_t k,
                    int64_t *n_rows, int64_t *heap_bytes) {
  obgpu_batch *b = r->batch;
  obgpu_ctx *ctx = r->ctx;
  Cols cols{};
  cols.a = dictops::BlkArgs{b->d_image, b->d_recs, b->d_plans, (int32_t)b->max_cols};
  Key key[kMaxKeys]{};
  const auto class_of = [&](int32_t col, int32_t &str) -> bool {
    const uint8_t t = b->col_types[(size_t)col];
    const int sc = t == 0xff ? 0 : obf::store_class_of(t);
    str = sc == 5;
    return sc == 1 || sc == 2 || sc == 5;
  };
  for (int i = 0; i < n_keys + n_out; ++i) {
    const int32_t col = i < n_keys ? keys[i].col : out_cols[i - n_keys];
    if (!class_of(col, cols.str[i])) {
      ctx->err = "top-rows column is not an integer or string column in every micro block";
      return OBGPU_NOT_SUPPORTED;
    }
    cols.col[i] = col;
  }
  cols.n = n_keys + n_out;
  for (int i = 0; i < n_keys; ++i) key[i] = Key{keys[i].col, keys[i].desc ? 1 : 0, keys[i].nulls_first ? 1 : 0, cols.str[i]};
  const int nb = b->n_blocks;
  // [status][counters: listed, hist[257], kept, next][kept list][positions, next positions][words][NULL flags]
  Scratch sm(ctx);
  const size_t o_status = sm.take(64), o_ctr = sm.take(8 * 264), o_kept = sm.take((size_t)std::min(k, n_sel) * 8);
  const size_t o_pos = sm.take((size_t)n_sel * 8), o_next = sm.take((size_t)n_sel * 8), o_words = sm.take((size_t)n_sel * 8);
  const size_t o_nulls = sm.take((size_t)n_sel);
  CUDA_TRY(ctx, sm.alloc());
  int *d_status = sm.at<int>(o_status);
  unsigned long long *ctr = sm.at<unsigned long long>(o_ctr), *hist = ctr + 1, *kc = ctr + 258;
  CUDA_TRY(ctx, cudaMemsetAsync(sm.p, 0, o_kept, ctx->stream));
  if (nb > 0) {
    check_kernel<<<(unsigned)((nb + 255) / 256), 256, 0, ctx->stream>>>(cols, nb, d_status);
    list_kernel<<<grid_for(ctx, (int64_t)nb * 32), kThreads, 0, ctx->stream>>>(b->d_recs, nb, r->no_filter ? nullptr : r->d_bitmap, ctr,
                                                                              (uint64_t)n_sel, sm.at<uint64_t>(o_pos), d_status);
    ctx->launches += 2;
    CUDA_TRY(ctx, cudaGetLastError());
  }
  unsigned long long *hp = (unsigned long long *)ctx->h_pinned;
  // the device status and the counters in one copy: [status][listed, hist[257], kept, next]
  const auto read_back = [&](size_t words) -> int {
    CUDA_TRY(ctx, cudaMemcpyAsync(hp, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(hp + 1, ctr, words * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    if (const int s = (int)(uint32_t)hp[0]) return check_status(ctx, s);
    return OBGPU_SUCCESS;
  };
  if (const int ret = read_back(1); ret != OBGPU_SUCCESS) return ret;
  if ((int64_t)hp[1] != n_sel) { ctx->err = "top rows: selected rows differ from the scan's count"; return OBGPU_INVALID_DATA; }
  const int64_t m = std::min(k, n_sel);
  uint64_t *cand = sm.at<uint64_t>(o_pos), *next = sm.at<uint64_t>(o_next), *kept = sm.at<uint64_t>(o_kept);
  uint64_t *words = sm.at<uint64_t>(o_words);
  uint8_t *nulls = sm.at<uint8_t>(o_nulls);
  int64_t nc = n_sel, need = m, n_kept = 0;
  int level_key = 0;
  uint32_t chunk = 0;
  while (need > 0) {
    if (nc <= need) {   // every candidate is kept
      CUDA_TRY(ctx, cudaMemcpyAsync(kept + n_kept, cand, (size_t)nc * 8, cudaMemcpyDeviceToDevice, ctx->stream));
      n_kept += nc;
      break;
    }
    const bool use_key = level_key < n_keys;
    const Key kk = use_key ? key[level_key] : Key{};
    WordArgs wa{cols.a, cand, nc, kk, use_key ? 1 : 0, chunk, words, nulls};
    word_kernel<<<grid_for(ctx, nc), kThreads, 0, ctx->stream>>>(wa);
    ctx->launches++;
    // radix select over the non-NULL words: T, the candidates below it and those equal to it
    uint64_t prefix = 0, mask = 0;
    int64_t eq = 0, want = need;
    bool nulls_done = false;
    CompactArgs ca{cand, words, nulls, nc, 0, 0, C_IN, C_NEXT, C_OUT, C_OUT, kept + n_kept, next, kc};
    bool next_key_only = false;   // the level only splits NULL from non-NULL rows
    for (int shift = 56; shift >= 0; shift -= 8) {
      CUDA_TRY(ctx, cudaMemsetAsync(hist, 0, 257 * 8, ctx->stream));
      hist_kernel<<<grid_for(ctx, nc), kThreads, 0, ctx->stream>>>(words, nulls, nc, prefix, mask, shift, hist);
      ctx->launches++;
      CUDA_TRY(ctx, cudaGetLastError());
      if (const int ret = read_back(258); ret != OBGPU_SUCCESS) return ret;
      const unsigned long long *h = hp + 2;
      if (!nulls_done) {
        nulls_done = true;
        const int64_t n_null = (int64_t)h[256], n_val = nc - n_null;
        if (kk.nulls_first && n_null > 0) {
          if (n_null >= want) { ca.null = C_NEXT; ca.lt = ca.eq = ca.gt = C_OUT; next_key_only = true; break; }
          ca.null = C_IN;
          want -= n_null;
        } else if (!kk.nulls_first && n_null > 0 && n_val < want) {
          ca.null = C_NEXT;
          ca.lt = ca.eq = ca.gt = C_IN;
          next_key_only = true;
          break;
        }
      }
      int64_t cum = 0;
      int d = 0;
      while (d < 255 && cum + (int64_t)h[d] < want) cum += (int64_t)h[d++];
      want -= cum;
      eq = (int64_t)h[d];
      prefix |= (uint64_t)d << shift;
      mask |= 0xffull << shift;
      if (eq == want) break;          // every row under this prefix is needed: no further pass
    }
    if (!next_key_only) {
      ca.T = prefix;
      ca.mask = mask;
      if (eq == want) ca.eq = C_IN;   // every tie fits
    }
    CUDA_TRY(ctx, cudaMemsetAsync(kc, 0, 16, ctx->stream));
    compact_kernel<<<grid_for(ctx, nc), kThreads, 0, ctx->stream>>>(ca);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    if (const int ret = read_back(260); ret != OBGPU_SUCCESS) return ret;
    n_kept += (int64_t)hp[259];
    need = m - n_kept;
    nc = (int64_t)hp[260];
    std::swap(cand, next);
    if (next_key_only || !use_key) { ++level_key; chunk = 0; continue; }
    const uint64_t T = kk.desc ? ~prefix : prefix;
    if (kk.str && (T & 0xffu) == 8u) ++chunk;   // the tied strings go on past this word
    else { ++level_key; chunk = 0; }
  }
  if (n_kept != m) { ctx->err = "top rows: the selection kept a wrong number of rows"; return OBGPU_INVALID_DATA; }
  // the kept rows' cells into a set, the set in order, and the fetch buffer
  Src src{};
  src.cols = cols;
  src.kept = kept;
  TopSet u, sorted;
  if (const int ret = gather_set(ctx, src, m, u); ret != OBGPU_SUCCESS) return ret;
  const int ord = order_sets(ctx, u, TopSet{}, 0, n_keys, key, cols.str, k, sorted);
  free_set(ctx, u);
  if (ord != OBGPU_SUCCESS) return ord;
  uint32_t str_mask = 0, sgn_mask = 0;
  for (int j = 0; j < n_out; ++j) {
    const uint8_t t = b->col_types[(size_t)out_cols[j]];
    if (cols.str[n_keys + j]) str_mask |= 1u << j;
    else if (obf::store_class_of(t) == 1 || obf::datum_len_of(t) < 8) sgn_mask |= 1u << j;
  }
  void *buf = nullptr;
  int64_t heap = 0;
  if (const int ret = emit(ctx, sorted, n_keys, n_out, str_mask, sgn_mask, &buf, &heap); ret != OBGPU_SUCCESS) {
    free_set(ctx, sorted);
    return ret;
  }
  r->d_top = buf;
  r->d_tset = sorted.mem;
  r->top_rows = m;
  r->top_heap = heap;
  r->tset_heap = sorted.heap;
  r->tset_cols = sorted.n_cols;
  r->top_n_out = n_out;
  r->top_str = str_mask;
  r->top_sgn = sgn_mask;
  for (int c = 0; c < cols.n; ++c) r->tset_types[c] = b->col_types[(size_t)cols.col[c]];
  *n_rows = m;
  *heap_bytes = heap;
  return OBGPU_SUCCESS;
}

// the arguments obgpu_result_top_rows and obgpu_pipeline_top_rows check alike before any work
static int check_args(const obgpu_sort_key *keys, int32_t n_keys, const int32_t *out_cols, int32_t n_out, int64_t k, const int64_t *n_rows,
                      const int64_t *heap_bytes, uint32_t max_cols) {
  if (!keys || n_keys < 1 || n_keys > kMaxKeys || n_out < 0 || n_out > kMaxOut || (n_out > 0 && !out_cols) || k < 1 || !n_rows || !heap_bytes)
    return OBGPU_INVALID_ARGUMENT;
  for (int i = 0; i < n_keys + n_out; ++i) {
    const int32_t col = i < n_keys ? keys[i].col : out_cols[i - n_keys];
    if (col < 0 || (uint32_t)col >= max_cols) return OBGPU_INVALID_ARGUMENT;
  }
  return k > kMaxK ? OBGPU_NOT_SUPPORTED : OBGPU_SUCCESS;
}

}  // namespace topn

extern "C" {

int obgpu_result_top_rows(obgpu_result *r, const obgpu_sort_key *keys, int32_t n_keys, const int32_t *out_cols, int32_t n_out, int64_t k,
                          int64_t *n_rows, int64_t *heap_bytes) {
  if (!r) return OBGPU_INVALID_ARGUMENT;
  obgpu_result_info info;
  const int ret = obgpu_result_info_get(r, &info);
  if (ret != OBGPU_SUCCESS && ret != OBGPU_BUF_NOT_ENOUGH) return ret;
  cudaSetDevice(r->ctx->device);
  topn::drop_rows(r);
  if (const int a = topn::check_args(keys, n_keys, out_cols, n_out, k, n_rows, heap_bytes, r->batch->max_cols); a != OBGPU_SUCCESS) {
    if (a == OBGPU_NOT_SUPPORTED) r->ctx->err = "top rows: k above 65536";
    return a;
  }
  return topn::top_rows(r, info.selected_rows, keys, n_keys, out_cols, n_out, k, n_rows, heap_bytes);
}

int obgpu_result_fetch_top_rows(obgpu_result *r, int32_t *host_block, int32_t *host_row, int64_t *host_vals, uint8_t *host_nulls, void *host_heap) {
  if (!r || r->top_rows < 0 || !host_block || !host_row || (r->top_n_out > 0 && (!host_vals || !host_nulls)) || (r->top_heap > 0 && !host_heap))
    return OBGPU_INVALID_ARGUMENT;
  cudaSetDevice(r->ctx->device);
  return topn::fetch(r->ctx, r->d_top, r->top_rows, r->top_n_out, r->top_heap, host_block, host_row, host_vals, host_nulls, host_heap);
}

}  // extern "C"
