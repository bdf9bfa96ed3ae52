// Batch codes: the distinct values of a dictionary-coded filter column, numbered once for the whole page batch -- the strings of
// a VARCHAR / CHAR column (PAX DICT with variable-length entries) or the 64-bit values of a fixed-width integer K_DICT column. Every
// block repeats the column's few distinct values in its own dictionary, and a leaf used to be evaluated on each block's copy: the
// count kernel staged every block's dictionary and compared it entry by entry. With codes, the leaf is evaluated once per scan over
// the distinct values (obgpu_code_leaf_kernel: a bitset of n_codes bits), and the count kernel stages a block's refs and its slice
// of the code array instead of the column region; a row's verdict is bit code[ref] of that bitset (scan_small.cuh,
// lean_rows_coded).
//
// Built lazily by the first scan that puts a record leaf (an EQ / NE / IN leaf on a string column, a range leaf on an integer one)
// on the column with stage records, and kept until obgpu_batch_close:
//   count   one thread per block: code slice length (dictionary entries rounded to 8 codes: 16-byte TMA pieces), widest refs range
//   prefix  slice lengths -> first code of each block (16-byte units)   -- the host reads the total and checks free memory --
//   insert  one warp per block: every dictionary entry into an open-addressing table of 2^18 slots. A string's key is its first
//           inserter's image offset, length and a hash tag (a probe compares the whole bytes); an integer's key is its value as
//           the per-block leaves compare it (entry + base, sign-fixed as the block's record says) plus 1, 0 marking an empty slot:
//           the one value that wraps, 2^64 - 1, has a slot of its own past the table
//                                                                        -- the host reads the distinct count: above 65 536, no codes --
//   number  one thread per slot: occupied slots -> codes 0..n_codes-1 and the code table (a string's key, an integer's value)
//   write   one warp per block: every entry's code at its block's slice (NULL refs have no entry: ref >= dict_count)
// A column that cannot be coded (more distinct values than a uint16 code, an image past 2^37 bytes, not enough free device memory)
// keeps the region path; ColCodes::state records why.
#pragma once

namespace bcodes {

constexpr uint32_t kTableBits = 18, kTableSlots = 1u << kTableBits;
constexpr int32_t kMaxCodes = 65536;
constexpr int kWarpsPerCta = 8;

// key: image byte offset (37 bits) | length (16 bits) | hash tag (10 bits) | 1
__device__ __forceinline__ uint64_t key_of(uint64_t abs, uint32_t len, uint64_t h) {
  return (abs << 27) | ((uint64_t)len << 11) | (((h >> 40) & 0x3ffull) << 1) | 1ull;
}
__device__ __forceinline__ uint64_t key_abs(uint64_t k) { return k >> 27; }
__device__ __forceinline__ uint32_t key_len(uint64_t k) { return (uint32_t)(k >> 11) & 0xffffu; }

// nb <= 8 bytes of the image at byte offset abs + i (the image is 16-byte aligned and padded past its end)
__device__ __forceinline__ uint64_t img_bytes(const uint8_t *image, uint64_t abs, uint32_t i, uint32_t nb) {
  return ld_bits(image + (abs & ~7ull), ((uint32_t)(abs & 7ull) + i) * 8u, nb * 8u);
}

__device__ __forceinline__ uint64_t str_hash(const uint8_t *image, uint64_t abs, uint32_t len) {
  uint64_t h = 0x9E3779B97F4A7C15ull * ((uint64_t)len + 1ull);
  for (uint32_t i = 0; i < len; i += 8u) {
    h = (h ^ img_bytes(image, abs, i, len - i < 8u ? len - i : 8u)) * 0xD6E8FEB86659FD93ull;
    h ^= h >> 29;
  }
  h ^= h >> 32;
  return h * 0x9E3779B97F4A7C15ull;
}

__device__ __forceinline__ bool same_bytes(const uint8_t *image, uint64_t a, uint64_t b, uint32_t len) {
  for (uint32_t i = 0; i < len; i += 8u) {
    const uint32_t nb = len - i < 8u ? len - i : 8u;
    if (img_bytes(image, a, i, nb) != img_bytes(image, b, i, nb)) return false;
  }
  return true;
}

__device__ __forceinline__ uint64_t int_hash(uint64_t v) {
  v = (v ^ (v >> 31)) * 0xD6E8FEB86659FD93ull;
  v ^= v >> 32;
  return v * 0x9E3779B97F4A7C15ull;
}

// Slot of a dictionary entry: found, or (insert) claimed. kNoSlot when the table is full (or, not inserting, absent). STR: the string
// (abs, len); else the integer value v, whose key is v + 1 -- the value 2^64 - 1 (key 0) is slot kTableSlots, its seen flag in
// counters[3].
constexpr uint32_t kNoSlot = 0xffffffffu;
template <bool STR>
__device__ __forceinline__ uint32_t probe(const uint8_t *image, unsigned long long *table, uint64_t abs, uint32_t len, uint64_t v,
                                          bool insert, unsigned int *counters) {
  const uint64_t h = STR ? str_hash(image, abs, len) : int_hash(v), key = STR ? key_of(abs, len, h) : v + 1ull;
  if (!STR && key == 0ull) {
    if (insert && atomicCAS(&counters[3], 0u, 1u) == 0u) atomicAdd(&counters[0], 1u);
    return kTableSlots;
  }
  const uint64_t match = key & ((1ull << 27) - 1ull);   // length and tag
  uint32_t slot = (uint32_t)h & (kTableSlots - 1u);
  for (uint32_t k = 0; k < kTableSlots; ++k, slot = (slot + 1u) & (kTableSlots - 1u)) {
    unsigned long long cur = *(volatile unsigned long long *)&table[slot];
    if (cur == 0ull) {
      if (!insert) return kNoSlot;
      cur = atomicCAS(&table[slot], 0ull, (unsigned long long)key);
      if (cur == 0ull) {
        atomicAdd(&counters[0], 1u);
        return slot;
      }
    }
    if (STR ? (cur & ((1ull << 27) - 1ull)) == match && same_bytes(image, key_abs(cur), abs, len) : cur == key) return slot;
  }
  return kNoSlot;
}

// Dictionary entry e of the column's stage record sr in the block at image offset off: its string's image offset and length
// (dict_str_s over the image)
__device__ __forceinline__ void entry_of(const uint8_t *image, uint64_t off, const StageRec &sr, uint32_t e, uint64_t &abs, uint32_t &len) {
  const uint8_t *s = image + off;
  const uint32_t ib8 = sr.dict_data_size * 8u, ibit = sr.dict_payload * 8u;
  const uint32_t lo = e == 0 ? 0u : (uint32_t)ld_bits(s, ibit + (e - 1u) * ib8, ib8);
  const uint32_t hi = e + 1u == sr.dict_count ? (uint32_t)sr.last_end : (uint32_t)ld_bits(s, ibit + e * ib8, ib8);
  abs = off + sr.add + lo;
  len = hi - lo;
}

// Value of integer dictionary entry e, as dict_int_s gives it to the per-block leaves: entry + base, sign-fixed (int_mask) when the
// block's record says so
__device__ __forceinline__ uint64_t int_entry(const uint8_t *image, uint64_t off, const StageRec &sr, uint32_t e, uint64_t int_mask) {
  const uint64_t v = ld_bits(image + off, (sr.dict_payload + e * sr.dict_data_size) * 8u, sr.dict_data_size * 8u) + sr.add;
  return (sr.flags & SR_SIGN_FIX) ? sign_fix(int_mask, v) : v;
}

__global__ void __launch_bounds__(256) count_kernel(const StageRec *stage, const BlockRec *recs, int n, int max_cols, int col,
                                                    uint32_t *cnt16, unsigned int *spans) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n) return;
  const StageRec sr = stage[(int64_t)b * max_cols + col];
  const uint32_t rows = recs[b].rows, dc = rows != 0 ? sr.dict_count : 0u;
  cnt16[b] = (dc + 7u) >> 3;
  if (rows == 0) return;
  uint32_t lo, hi;
  coded_refs_range(sr, rows, lo, hi);
  atomicMax(&spans[0], hi - lo);
  atomicMax(&spans[1], ((dc + 7u) >> 3) * 16u);
}

__global__ void off16_kernel(const int64_t *off, int n, uint32_t *off16) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < n) off16[b] = (uint32_t)off[b];
}

// one warp per block, lanes over its dictionary entries: insert (codes == nullptr) or write each entry's code
template <bool STR>
__global__ void __launch_bounds__(32 * kWarpsPerCta) entries_kernel(const uint8_t *image, const StageRec *stage, const BlockRec *recs, int n,
                                                                    int max_cols, int col, uint64_t int_mask, unsigned long long *table,
                                                                    unsigned int *counters, const uint16_t *slot_code, const uint32_t *off16,
                                                                    uint16_t *codes) {
  const int b = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= n) return;
  const BlockRec rec = recs[b];
  if (rec.rows == 0) return;
  const StageRec sr = stage[(int64_t)b * max_cols + col];
  const bool insert = codes == nullptr;
  for (uint32_t e = (uint32_t)lane; e < sr.dict_count; e += 32u) {
    if (insert && *(volatile unsigned int *)&counters[0] > (unsigned int)kMaxCodes) return;   // over the cap: no codes
    uint64_t abs = 0, v = 0;
    uint32_t len = 0;
    if (STR) entry_of(image, rec.off, sr, e, abs, len);
    else v = int_entry(image, rec.off, sr, e, int_mask);
    const uint32_t slot = probe<STR>(image, table, abs, len, v, insert, counters);
    if (slot == kNoSlot) { atomicOr(&counters[1], 1u); return; }
    if (!insert) codes[(size_t)off16[b] * 8u + e] = slot_code[slot];
  }
}

// slot s < kTableSlots of the table, or (integers) s == kTableSlots: the value 2^64 - 1 when some entry held it
__global__ void number_kernel(const unsigned long long *table, bool str, unsigned int *counters, uint16_t *slot_code, uint64_t *code_table) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > kTableSlots || (s == kTableSlots ? str || counters[3] == 0u : table[s] == 0ull)) return;
  const uint32_t c = atomicAdd(&counters[2], 1u);
  slot_code[s] = (uint16_t)c;
  code_table[c] = s == kTableSlots ? ~0ull : str ? table[s] : table[s] - 1ull;
}

}  // namespace bcodes

// The leaf of filter node `node` over the code table of its column: bit c of out = the leaf on distinct value c -- the test the
// per-block leaves make: str_pred's equality test on a string, int_pred's range test on an integer (the column's store class and
// datum length from the scan; the values were sign-fixed when the codes were built). Bits at and past n_codes stay 0.
__global__ void __launch_bounds__(256) obgpu_code_leaf_kernel(const __grid_constant__ ScanParams p, int node, const uint64_t *table,
                                                              int n_codes, int words, uint32_t *out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= words * 32) return;
  const FilterNodeDev &nd = p.nodes[node];
  bool r = false;
  if (c < n_codes) {
    const uint64_t k = table[c];
    if (p.used_sc[nd.used_idx] == 5) {
      const uint64_t abs = bcodes::key_abs(k);
      r = str_pred(p, nd, p.image + (abs & ~7ull), (uint32_t)(abs & 7ull), bcodes::key_len(k));
    } else {
      RecDesc d{};
      d.sc = p.used_sc[nd.used_idx];
      d.elem_len = p.used_elem_len[nd.used_idx];
      r = int_pred(p, nd, d, k);
    }
  }
  const uint32_t w = __ballot_sync(0xffffffffu, r);
  if ((threadIdx.x & 31) == 0) out[c >> 5] = w;
}

// Codes of store column col of b, built on first use: the column's ColCodes (state 1: built; < 0: the column keeps the region path).
static const ColCodes &batch_codes(obgpu_batch *b, int col) {
  if (b->col_codes.size() != b->max_cols) b->col_codes.assign(b->max_cols, ColCodes{});
  ColCodes &sc = b->col_codes[(size_t)col];
  if (sc.state != 0) return sc;
  obgpu_ctx *ctx = b->ctx;
  const int n = b->n_blocks;
  const int store = b->col_types[(size_t)col] == 0xff ? 0 : obf::store_class_of(b->col_types[(size_t)col]);
  if (b->d_stage == nullptr || (b->col_stage_gaps[(size_t)col] & SR_NOT_FILTER) || (store != 5 && store != 1 && store != 2)) {
    sc.state = OBGPU_CODES_NOT_CODABLE;
    return sc;
  }
  const bool str = store == 5;
  const uint64_t int_mask = str ? 0ull : obf::integer_mask_of(b->col_types[(size_t)col]);
  if (b->image_size >= (int64_t)1 << 37) { sc.state = OBGPU_CODES_NOT_CODABLE; return sc; }
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventRecord(e0, ctx->stream);
  auto fail = [&](int32_t why) -> const ColCodes & {
    cudaGetLastError();   // a refused allocation leaves a (non-sticky) error behind: the scan goes on without codes
    if (sc.d_mem) cudaFreeAsync(sc.d_mem, ctx->stream);
    sc = ColCodes{};
    sc.state = why;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return sc;
  };
  // temporaries: [table: 2^18 keys][slot -> code, one more for the integer 2^64 - 1][counters][spans][slice lengths][slice offsets]
  // [prefix chunk totals]
  Scratch tmp(ctx);
  const size_t o_table = tmp.take((size_t)bcodes::kTableSlots * 8), o_slot = tmp.take((size_t)bcodes::kTableSlots * 2 + 16);
  const size_t o_ctr = tmp.take(32), o_cnt = tmp.take((size_t)n * 4), o_off = tmp.take(((size_t)n + 1) * 8);
  const size_t o_chunk = tmp.take(((size_t)n / kPrefixChunk + 2) * 8);
  if (tmp.alloc() != cudaSuccess) return fail(OBGPU_CODES_NO_MEMORY);
  unsigned long long *table = tmp.at<unsigned long long>(o_table);
  // [entries inserted, table full, codes numbered, integer 2^64 - 1 seen, refs span, codes span]
  unsigned int *ctr = tmp.at<unsigned int>(o_ctr);
  int64_t *off = tmp.at<int64_t>(o_off);
  if (cudaMemsetAsync(tmp.p, 0, o_slot, ctx->stream) != cudaSuccess || cudaMemsetAsync(ctr, 0, 32, ctx->stream) != cudaSuccess)
    return fail(OBGPU_CODES_NO_MEMORY);
  const int n_chunks = (n + kPrefixChunk - 1) / kPrefixChunk;
  bcodes::count_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(b->d_stage, b->d_recs, n, (int)b->max_cols, col, tmp.at<uint32_t>(o_cnt), ctr + 4);
  obgpu_prefix_local_kernel<<<n_chunks, 256, 0, ctx->stream>>>(tmp.at<uint32_t>(o_cnt), n, off, tmp.at<unsigned long long>(o_chunk));
  obgpu_prefix_fix_kernel<<<n_chunks + 1, 256, 0, ctx->stream>>>(n, n_chunks, off, tmp.at<const unsigned long long>(o_chunk));
  ctx->launches += 3;
  int64_t *hp = (int64_t *)ctx->h_pinned;
  if (cudaMemcpyAsync(hp, off + n, 8, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
      cudaMemcpyAsync(hp + 1, ctr + 4, 8, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
      cudaStreamSynchronize(ctx->stream) != cudaSuccess)
    return fail(OBGPU_CODES_NO_MEMORY);
  const int64_t units = hp[0];
  const uint32_t refs_span = (uint32_t)hp[1], codes_span = (uint32_t)(hp[1] >> 32);
  if (units >= ((int64_t)1 << 32)) return fail(OBGPU_CODES_NOT_CODABLE);
  // [code_off16: n][code table: kMaxCodes][codes: 16 bytes per unit], next to the image and the stage records: keep 1 GiB free
  const size_t a_off = ((size_t)n * 4 + 255) & ~(size_t)255, a_tab = (size_t)bcodes::kMaxCodes * 8;
  const size_t need = a_off + a_tab + (size_t)units * 16 + 16;
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess || need + ((size_t)1 << 30) > free_b) return fail(OBGPU_CODES_NO_MEMORY);
  if (cudaMallocAsync(&sc.d_mem, need, ctx->stream) != cudaSuccess) { sc.d_mem = nullptr; return fail(OBGPU_CODES_NO_MEMORY); }
  uint8_t *m = (uint8_t *)sc.d_mem;
  uint32_t *off16 = (uint32_t *)m;
  uint64_t *code_table = (uint64_t *)(m + a_off);
  uint16_t *codes = (uint16_t *)(m + a_off + a_tab);
  bcodes::off16_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(off, n, off16);
  const unsigned grid = (unsigned)((n + bcodes::kWarpsPerCta - 1) / bcodes::kWarpsPerCta);
  const auto entries = str ? bcodes::entries_kernel<true> : bcodes::entries_kernel<false>;
  entries<<<grid, 32 * bcodes::kWarpsPerCta, 0, ctx->stream>>>(b->d_image, b->d_stage, b->d_recs, n, (int)b->max_cols, col, int_mask, table, ctr,
                                                             nullptr, nullptr, nullptr);
  ctx->launches += 2;
  if (cudaMemcpyAsync(hp, ctr, 8, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess || cudaStreamSynchronize(ctx->stream) != cudaSuccess)
    return fail(OBGPU_CODES_NO_MEMORY);
  const uint32_t distinct = (uint32_t)hp[0], full = (uint32_t)(hp[0] >> 32);
  if (full || distinct > (uint32_t)bcodes::kMaxCodes) return fail(OBGPU_CODES_OVER_CAP);
  if (cudaMemsetAsync(codes, 0, (size_t)units * 16 + 16, ctx->stream) != cudaSuccess) return fail(OBGPU_CODES_NO_MEMORY);
  bcodes::number_kernel<<<bcodes::kTableSlots / 256 + 1, 256, 0, ctx->stream>>>(table, str, ctr, tmp.at<uint16_t>(o_slot), code_table);
  entries<<<grid, 32 * bcodes::kWarpsPerCta, 0, ctx->stream>>>(b->d_image, b->d_stage, b->d_recs, n, (int)b->max_cols, col, int_mask, table, ctr,
                                                             tmp.at<uint16_t>(o_slot), off16, codes);
  ctx->launches += 2;
  cudaEventRecord(e1, ctx->stream);
  if (cudaGetLastError() != cudaSuccess || cudaEventSynchronize(e1) != cudaSuccess) return fail(OBGPU_CODES_NO_MEMORY);
  cudaEventElapsedTime(&sc.build_ms, e0, e1);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  sc.state = 1;
  sc.n_codes = (int32_t)distinct;
  sc.refs_span = refs_span;
  sc.codes_span = codes_span;
  sc.d_off16 = off16;
  sc.d_table = code_table;
  sc.d_codes = codes;
  return sc;
}

static void batch_codes_free(obgpu_batch *b) {
  for (ColCodes &sc : b->col_codes)
    if (sc.d_mem) cudaFreeAsync(sc.d_mem, b->ctx->stream);
  b->col_codes.clear();
}

extern "C" {

int obgpu_batch_string_codes(const obgpu_batch *b, int32_t col, int32_t *state, int32_t *n_codes, float *build_ms) {
  if (!b || col < 0 || (uint32_t)col >= b->max_cols || !state) return OBGPU_INVALID_ARGUMENT;
  const ColCodes none{};
  const ColCodes &sc = (size_t)col < b->col_codes.size() ? b->col_codes[(size_t)col] : none;
  *state = sc.state;
  if (n_codes) *n_codes = sc.n_codes;
  if (build_ms) *build_ms = sc.build_ms;
  return OBGPU_SUCCESS;
}

int obgpu_ctx_count_layout(const obgpu_ctx *ctx, int32_t *pc_bytes, int32_t *ctas_per_sm, int32_t *kernel) {
  if (!ctx || !pc_bytes || !ctas_per_sm) return OBGPU_INVALID_ARGUMENT;
  *pc_bytes = ctx->last_pc_bytes;
  *ctas_per_sm = ctx->last_count_ctas;
  if (kernel) *kernel = ctx->last_count_kernel;
  return OBGPU_SUCCESS;
}

}  // extern "C"
