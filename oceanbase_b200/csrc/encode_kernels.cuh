// Phase B of the compaction on the device: merged column arrays -> PAX micro-blocks (RAW columns; AUTO below), byte for byte the
// blocks the host writer (sstable_writer.cpp: BlockBuilder::encode_raw / build / finish_header) produces for the same rows,
// plus the column checksums of the rows (K16). One kernel, one CTA per micro-block, input read once, output written once:
//
//   stats   : per column max of the stored value image + NULL count (and, fused, the column checksum of the cells); four
//             columns' loads in flight together, warp reductions through redux.sync
//   plan    : warp 0, one lane per column, lays the block out (ObRawEncoder::traverse width rules, ext bits, column stores back
//             to back by a warp scan) and publishes the aligned block size for the look-back at once
//   pack    : cells -> shared-memory image of the block (ext bits, bit-packed and byte-packed values are all "w bits at bit
//             address b": at most three shared atomicOr per cell); the second read of the cells hits L2
//   crc32c  : payload checksum in parallel -- every thread the raw CRC of an odd-word-stride chunk (slicing by 4, tables in
//             shared memory), shifted to its position by ONE carry-less multiplication with x^(32 * words after it) mod P
//             (host-built table) and XOR-reduced; leading zero words cost nothing with init 0 / no final xor
//   offset  : decoupled look-back over the aligned block sizes (tickets in scheduling order, one 64-bit flag per block), resolved
//             by thread 0 while the other warps pack
//   store   : header + checksums, then ONE bulk copy (TMA, cp.async.bulk shared -> global) of the aligned slot
//
// Columns asking for OBGPU_ENC_AUTO run the AUTO instantiation, the device form of the writer's build_int_dict +
// choose_auto_encoding (sstable_writer.cpp): per AUTO column a block-wide stable sort of (sort key, row) in shared memory
// (bitonic over the next power of two; the sort key is the store image with the sign bit flipped for the signed class, the
// writer's sorted order) gives the distinct values, their frequencies and first rows, the sorted ref of every row and the runs;
// warp 0 then evaluates the writer's estimates in the writer's order and lays out the chosen codec, and the pack writes it as
// BlockBuilder::encode_dict / encode_rle / encode_const / encode_base_diff do (re-sorting the columns that store a dictionary).
// RAW-only calls keep the RAW instantiation.
#pragma once
#include <map>
#include <mutex>

namespace enc {

constexpr int kThreads = 128;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxCols = 64;
constexpr uint32_t kCrcPoly = 0x82f63b78u;   // CRC-32C (Castagnoli), reflected
constexpr uint32_t kHeaderSize = 64u;        // MICRO_HEADER_FIXED_SIZE

struct ColSpec {
  const int64_t *vals;
  const uint8_t *nulls;
  uint64_t store_mask;     // low type_store_size bytes (ColCtx::uval)
  uint8_t obj_type, byte_only, datum_len, is_auto;
  uint8_t store_size, is_signed;   // type_store_size; store class 1 (signed)
  uint8_t cs_dict, pad1;           // CS encoder: OBGPU_ENC_CS_INT_DICT (is_auto: OBGPU_ENC_CS_AUTO)
};

struct Params {
  ColSpec col[kMaxCols];
  int32_t n_cols, rowkey_cnt, n_blocks, want_checksums;
  int64_t total_rows, rows_per_block;
  uint32_t align, slot_cap;          // slot_cap: bytes of the shared-memory block image (multiple of align)
  uint32_t lw_max, sort_cap;         // xpow32 holds (kThreads - 1) * lw_max + 1 entries; sort_cap: AUTO sort length (power of 2)
  uint8_t *image;
  int64_t *blk_off;                  // [n_blocks]
  uint32_t *blk_size;                // [n_blocks] exact bytes, 0: left to the host writer
  unsigned long long *flags;         // [n_blocks] look-back words: state << 62 | bytes
  unsigned long long *checksums;     // [n_cols]
  unsigned long long *totals;        // [0] image bytes, [1] host blocks
  int32_t *ticket;
  const uint32_t *xpow32;            // x^(32 k) mod P, reflected (x^0 = 0x80000000)
  int32_t stream_mode;               // CS encoder with stream codecs: the integer stream mode (0 detect, 2..8 that codec)
};

__device__ __forceinline__ uint32_t gf2_mulmod(uint32_t a, uint32_t b) {
  uint32_t p = 0;
#pragma unroll 8
  for (int i = 0; i < 32; ++i) {
    p ^= (a & 0x80000000u) ? b : 0u;
    a <<= 1;
    b = (b >> 1) ^ ((b & 1u) ? kCrcPoly : 0u);
  }
  return p;
}

__device__ __forceinline__ uint32_t crc_word(const uint32_t *tab, uint32_t crc, uint32_t w) {
  crc ^= w;
  return tab[768 + (crc & 0xffu)] ^ tab[512 + ((crc >> 8) & 0xffu)] ^ tab[256 + ((crc >> 16) & 0xffu)] ^ tab[crc >> 24];
}
__device__ __forceinline__ uint32_t crc_byte(const uint32_t *tab, uint32_t crc, uint32_t b) {
  return tab[(crc ^ b) & 0xffu] ^ (crc >> 8);
}

// get_packing_size (encoding/ob_encoding_util.cpp:37-73): size in bits when bit packing, else in bytes
__device__ __forceinline__ uint32_t packing_size(uint64_t v, bool enable_bp, bool &bp) {
  const uint32_t bits = v == 0 ? 1u : 64u - (uint32_t)__clzll((long long)v);
  if (!enable_bp) {
    bp = false;
    return v <= 0xffull ? 1u : v <= 0xffffull ? 2u : v <= 0xffffffffull ? 4u : 8u;
  }
  uint32_t size = bits / 8u;
  const uint32_t ext = bits % 8u;
  if (ext == 0) { bp = false; return size; }
  if (8u - ext < size / 2u + 1u) { bp = false; return size + 1u; }
  bp = true;
  return bits;
}

struct ColLayout {
  uint32_t store_off;   // byte offset of the column store inside the block
  uint32_t bits_size;   // bytes of the bit area ([ext bits][bit-packed values])
  uint8_t attr, size, bp, has_null;
};

// ---- OBGPU_ENC_AUTO ----------------------------------------------------------------------------------------------------------
// What the analysis finds in one AUTO column of a block, and the layout the plan picks for it.
struct AutoCol {
  unsigned long long kmin, kmax;   // smallest / largest sort key of the non-NULL cells
  uint32_t d;                      // distinct non-NULL values
  uint32_t fmax;                   // largest frequency of a value
  uint32_t runs, last_run;         // runs over the refs in row order (a NULL is ref d), first row of the last run
  uint32_t row_e, row_w;           // last row off the constant, for the estimate's / encode_const's constant
  uint32_t ref_w;                  // encode_const's constant: smallest sorted ref among the most frequent (d: NULL)
  uint32_t exc, len;               // CONST exceptions; the column header's length_
  uint8_t codec, size, bp, dsz, rib, refb, pad[2];   // chosen codec, its cell width (bits when bp), dict width, row-id / ref bytes
};

struct AutoScratch {
  unsigned long long *sk;   // [sort_cap] sort keys, sorted
  uint32_t *sr;             // [sort_cap] rows, sorted with the keys (0xffffffff: padding and NULL rows)
  uint32_t *hs;             // [sort_cap] scan scratch
  uint32_t *a;              // [rows] sorted ref of every row (NULL: d)
  uint32_t *b;              // [rows] 1 on the first occurrence of a value (scanned: distinct values seen up to the row)
  uint32_t *hp;             // [rows + 1] sorted position of each value's first entry; hp[d] = non-NULL rows
  uint32_t *red;            // [kWarps] reduction scratch
};

__device__ __forceinline__ uint32_t bpis(unsigned long long v) {   // get_byte_packed_int_size
  return v <= 0xffull ? 1u : v <= 0xffffull ? 2u : v <= 0xffffffffull ? 4u : 8u;
}
__device__ __forceinline__ uint32_t int_size_bytes(unsigned long long v) {   // get_int_size
  const uint32_t bits = v == 0 ? 1u : 64u - (uint32_t)__clzll((long long)v);
  return (bits + 7u) / 8u;
}

// OR the low w bits of x (w <= 64, x holds no higher bit) into the image at bit address b (the image is zeroed first)
__device__ __forceinline__ void or_bits(uint32_t *img32, uint32_t b, uint32_t w, unsigned long long x) {
  if (x == 0) return;
  const uint32_t sh = b & 31u;
  uint32_t *q = img32 + (b >> 5);
  atomicOr(q, (uint32_t)(x << sh));
  if (sh + w > 32u) atomicOr(q + 1, (uint32_t)(x >> (32u - sh)));
  if (sh + w > 64u) atomicOr(q + 2, (uint32_t)(x >> (64u - sh)));
}
__device__ __forceinline__ void put_bytes(uint32_t *img32, uint32_t at, uint32_t n, unsigned long long x) {
  or_bits(img32, at * 8u, 8u * n, n >= 8u ? x : (x & ((1ull << (8u * n)) - 1ull)));
}

__device__ __forceinline__ uint32_t blk_sum(uint32_t v, uint32_t *red) {
  v = __reduce_add_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t r = 0;
  for (int w = 0; w < kWarps; ++w) r += red[w];
  __syncthreads();
  return r;
}
__device__ __forceinline__ uint32_t blk_max(uint32_t v, uint32_t *red) {
  v = __reduce_max_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t r = 0;
  for (int w = 0; w < kWarps; ++w) r = max(r, red[w]);
  __syncthreads();
  return r;
}
__device__ __forceinline__ uint32_t blk_min(uint32_t v, uint32_t *red) {
  v = __reduce_min_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t r = 0xffffffffu;
  for (int w = 0; w < kWarps; ++w) r = min(r, red[w]);
  __syncthreads();
  return r;
}

// inclusive prefix sum of x[0, m) in place: one contiguous chunk per thread
__device__ void blk_scan(uint32_t *x, uint32_t m, uint32_t *red) {
  const uint32_t tid = threadIdx.x, lane = tid & 31u, per = (m + kThreads - 1u) / kThreads;
  const uint32_t lo = min(tid * per, m), hi = min(lo + per, m);
  uint32_t s = 0;
  for (uint32_t i = lo; i < hi; ++i) s += x[i];
  uint32_t incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= (uint32_t)o) incl += u;
  }
  if (lane == 31u) red[tid >> 5] = incl;
  __syncthreads();
  uint32_t off = incl - s;
  for (uint32_t w = 0; w < (tid >> 5); ++w) off += red[w];
  for (uint32_t i = lo; i < hi; ++i) { off += x[i]; x[i] = off; }
  __syncthreads();
}

// Stable sort of the block's non-NULL cells of one column by (sort key, row), then the sorted ref of every row (a), the
// first occurrences (b) and the first sorted position of every value (hp). Returns the distinct count. Every thread calls it.
__device__ uint32_t sort_column(const ColSpec &cs, const int64_t row0, const uint32_t n, const uint32_t nn, const uint32_t P,
                                const AutoScratch &s) {
  const uint32_t tid = threadIdx.x;
  const unsigned long long flip = cs.is_signed ? 1ull << (8u * cs.store_size - 1u) : 0ull;
  for (uint32_t i = tid; i < P; i += kThreads) {
    unsigned long long k = ~0ull;
    uint32_t r = 0xffffffffu;
    if (i < n) {
      if (!(cs.nulls && cs.nulls[row0 + i] != 0)) { k = ((unsigned long long)cs.vals[row0 + i] & cs.store_mask) ^ flip; r = i; }
      s.a[i] = 0xffffffffu;
      s.b[i] = 0u;
    }
    s.sk[i] = k;
    s.sr[i] = r;
  }
  __syncthreads();
  for (uint32_t k = 2; k <= P; k <<= 1) {   // bitonic, ascending; (key, row) pairs are unique, so the order is stable
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      for (uint32_t i = tid; i < P / 2u; i += kThreads) {
        const uint32_t lo = ((i & ~(j - 1u)) << 1) | (i & (j - 1u)), hi = lo + j;
        const unsigned long long ka = s.sk[lo], kb = s.sk[hi];
        const uint32_t ra = s.sr[lo], rb = s.sr[hi];
        const bool gt = ka > kb || (ka == kb && ra > rb);
        if (gt == ((lo & k) == 0)) { s.sk[lo] = kb; s.sk[hi] = ka; s.sr[lo] = rb; s.sr[hi] = ra; }
      }
      __syncthreads();
    }
  }
  const uint32_t m = n - nn;
  for (uint32_t i = tid; i < m; i += kThreads) s.hs[i] = (i == 0 || s.sk[i] != s.sk[i - 1]) ? 1u : 0u;
  __syncthreads();
  blk_scan(s.hs, m, s.red);
  const uint32_t d = m ? s.hs[m - 1] : 0u;
  for (uint32_t i = tid; i < m; i += kThreads) {
    const uint32_t seg = s.hs[i] - 1u, r = s.sr[i];
    s.a[r] = seg;
    if (i == 0 || s.hs[i - 1] != s.hs[i]) { s.b[r] = 1u; s.hp[seg] = i; }
  }
  if (tid == 0) s.hp[d] = m;
  __syncthreads();
  for (uint32_t r = tid; r < n; r += kThreads)
    if (s.a[r] == 0xffffffffu) s.a[r] = d;
  __syncthreads();
  return d;
}

// The analysis of one AUTO column (every thread calls it; thread 0 writes out).
__device__ void analyze_column(const ColSpec &cs, const int64_t row0, const uint32_t n, const uint32_t nn, const uint32_t P,
                               const AutoScratch &s, AutoCol &out) {
  const uint32_t tid = threadIdx.x;
  const uint32_t d = sort_column(cs, row0, n, nn, P, s);
  uint32_t f = 0;
  for (uint32_t v = tid; v < d; v += kThreads) f = max(f, s.hp[v + 1] - s.hp[v]);
  const uint32_t fmax = blk_max(f, s.red);
  // the estimate's constant: the most frequent value, ties to the earliest first occurrence; encode_const's: ties to the
  // smallest sorted ref. NULL is the constant of both only when strictly more frequent.
  uint32_t fr = 0xffffffffu, sw = 0xffffffffu;
  for (uint32_t v = tid; v < d; v += kThreads)
    if (s.hp[v + 1] - s.hp[v] == fmax) { fr = min(fr, s.sr[s.hp[v]]); sw = min(sw, v); }
  fr = blk_min(fr, s.red);
  sw = blk_min(sw, s.red);
  const bool const_null = nn > fmax;
  const uint32_t se = const_null ? d : s.a[fr], cw = const_null ? d : sw;
  uint32_t chg = 0, last = 0, re = 0, rw = 0;
  for (uint32_t r = tid; r < n; r += kThreads) {
    const uint32_t x = s.a[r];
    if (r > 0 && x != s.a[r - 1]) { ++chg; last = max(last, r); }
    if (x != se) re = max(re, r);
    if (x != cw) rw = max(rw, r);
  }
  chg = blk_sum(chg, s.red);
  last = blk_max(last, s.red);
  re = blk_max(re, s.red);
  rw = blk_max(rw, s.red);
  if (tid == 0) {
    out.kmin = n > nn ? s.sk[0] : 0ull;
    out.kmax = n > nn ? s.sk[n - nn - 1] : 0ull;
    out.d = d;
    out.fmax = fmax;
    out.runs = 1u + chg;
    out.last_run = last;
    out.row_e = re;
    out.row_w = rw;
    out.ref_w = cw;
  }
  __syncthreads();
}

__device__ __forceinline__ long long sign_extend(unsigned long long v, uint32_t ts) {
  const unsigned long long rev = ts >= 8u ? 0ull : ~((1ull << (8u * ts)) - 1ull);
  if (rev != 0 && (v & (rev >> 1))) v |= rev;
  return (long long)v;
}

// choose_auto_encoding (sstable_writer.cpp) for one integer column of the block, then the chosen codec's layout. Returns
// the column store's bytes; the RAW layout already in l / var stays when RAW is chosen. Warp 0, one lane per column.
__device__ uint32_t plan_auto(const ColSpec &cs, AutoCol &A, const uint32_t nrows, const uint32_t nnull,
                              const unsigned long long mx, const uint32_t ext_bit, ColLayout &l, bool &var, uint32_t raw_bytes) {
  const long long n = nrows, nn = nnull, ts = cs.store_size, distinct = A.d, eb = ext_bit;
  const bool ebp = cs.byte_only == 0;
  bool bp;
  // ---- RAW (ObRawEncoder::traverse + calc_size)
  long long raw_size;
  {
    long long bp_len = 0, fix_len = 0, raw_var = 0;
    bool is_var = false;
    const long long size = packing_size(mx, ebp, bp);
    if (bp) {
      if (size * nn > n * 2 * 8) { is_var = true; raw_var = (size / 8 + 1) * (n - nn); }
      else bp_len = size;
    } else {
      fix_len = size;
    }
    if (fix_len > 0 && bp_len == 0 && fix_len * nn > n * 2) { is_var = true; fix_len = 0; }
    raw_size = bp_len > 0 ? bp_len * n / 8 + 1 : (!is_var ? fix_len * n : raw_var + n * 2);
    raw_size += nn > 0 ? (n * eb + 1) / 8 : 0;   // (n * ext_bit + 1) / 8, as the writer estimates it
  }
  // ---- DICT
  const long long dsz = ebp ? int_size_bytes(mx) : bpis(mx);
  const long long dict_meta = 9 + dsz * distinct;
  const long long max_ref = nn > 0 ? distinct : distinct - 1;
  const unsigned long long ref_v = (unsigned long long)(max_ref > 0 ? max_ref : 0);
  long long dict_size;
  bool ref_bp;
  const long long ref_size = packing_size(ref_v, ebp, ref_bp);
  dict_size = dict_meta + (ref_bp ? (n * ref_size + 7) / 8 : n * ref_size);
  // ---- CONST
  const long long max_cnt = nn > (long long)A.fmax ? nn : (long long)A.fmax, exc = n - max_cnt;
  const bool const_ok = !(exc > 32 || exc > max(n * 10 / 100, 1ll));
  long long const_size = 0;
  if (exc == 0) const_size = (nn == 0 ? ts : 0) + 6;
  else const_size = 6 + dict_meta + exc * (bpis(A.row_e) + 1);
  int choose = 0 /*RAW*/;
  if (distinct <= 1 && const_ok) {
    choose = 3;
  } else {
    long long choose_size = raw_size;
    const long long acceptable = raw_size / 4;
    if (dict_size < choose_size) { choose = 1; choose_size = dict_size; }
    if (distinct <= n / 2) {
      const long long rle_size = 10 + dict_meta + (long long)A.runs * (bpis(A.last_run) + bpis(ref_v));
      if (rle_size < choose_size) { choose = 2; choose_size = rle_size; }
      if (const_ok && const_size < choose_size) { choose = 3; choose_size = const_size; }
    }
    if (choose_size > acceptable && distinct > 0) {   // ObIntegerBaseDiffEncoder (no ext-bit term in its estimate)
      unsigned long long delta, max_unsigned;
      if (cs.is_signed) {
        const long long smin = sign_extend(A.kmin ^ (1ull << (8u * ts - 1u)), (uint32_t)ts);
        const long long smax = sign_extend(A.kmax ^ (1ull << (8u * ts - 1u)), (uint32_t)ts);
        delta = smin < smax ? (unsigned long long)smax - (unsigned long long)smin : 0ull;
        max_unsigned = smin < 0 ? ~0ull : (unsigned long long)smax;
      } else {
        delta = A.kmin < A.kmax ? A.kmax - A.kmin : 0ull;
        max_unsigned = A.kmax;
      }
      if (delta != 0) {
        long long orig = packing_size(max_unsigned, true, bp);
        if (!bp) orig *= 8;
        long long dbits = packing_size(delta, true, bp);
        if (!bp) dbits *= 8;
        if ((orig - dbits) * n > (2 + ts) * 8) {
          const long long bd_size = (bp ? (n * dbits + 7) / 8 : n * (dbits / 8)) + 2 + ts;
          if (bd_size < choose_size) { choose = 4; choose_size = bd_size; }
        }
      }
    }
  }
  A.codec = (uint8_t)choose;
  if (choose == 0) return raw_bytes;
  var = false;
  l.has_null = nn != 0;
  A.dsz = (uint8_t)dsz;
  if (choose == 1) {   // encode_dict: [sorted dict meta][refs, NULL cells included, no ext bits]
    A.size = (uint8_t)ref_size;
    A.bp = ref_bp;
    A.len = (uint32_t)dict_meta;
    l.attr = (uint8_t)(0x1u | (ref_bp ? 0x4u : 0u));
    return (uint32_t)dict_size;
  }
  if (choose == 2) {   // encode_rle: [header][run rows][run refs][dict meta, first-occurrence order]
    A.rib = (uint8_t)bpis(A.last_run);
    A.refb = (uint8_t)bpis(ref_v);
    if ((long long)A.runs * A.rib > 32767) var = true;   // the writer refuses it (ObRLEDecoder's int16 bound): host block
    A.len = (uint32_t)(10 + (long long)A.runs * (A.rib + A.refb) + dict_meta);
    l.attr = 0;
    return A.len;
  }
  if (choose == 3) {   // encode_const: header [+ exceptions + sorted dict meta] or [+ the value]
    A.exc = (uint32_t)exc;
    A.rib = (uint8_t)bpis(A.row_w);
    A.len = exc == 0 ? (uint32_t)(6 + (distinct == 0 ? 0 : ts)) : (uint32_t)(6 + exc * (A.rib + 1) + dict_meta);
    l.attr = 0;
    return A.len;
  }
  // encode_base_diff: [header][base][ext bits][bit-packed deltas] or [..][byte-packed deltas]
  unsigned long long delta;
  if (cs.is_signed) {
    const unsigned long long f = 1ull << (8u * ts - 1u);
    delta = (unsigned long long)sign_extend(A.kmax ^ f, (uint32_t)ts) - (unsigned long long)sign_extend(A.kmin ^ f, (uint32_t)ts);
  } else {
    delta = A.kmax - A.kmin;
  }
  const uint32_t size = packing_size(delta, true, bp);
  A.size = (uint8_t)size;
  A.bp = bp;
  A.len = (uint32_t)(2 + ts);
  l.size = (uint8_t)size;
  l.bp = bp;
  l.attr = (uint8_t)(0x1u | (nn ? 0x2u : 0u) | (bp ? 0x4u : 0u));
  const unsigned long long bits = (nn ? (unsigned long long)ext_bit * nrows : 0ull) + (bp ? (unsigned long long)size * nrows : 0ull);
  l.bits_size = (uint32_t)((bits + 7ull) / 8ull);
  return A.len + l.bits_size + (bp ? 0u : size * nrows);
}

// DictMetaHeader {version_, row_ref_size_, count_, data_size_, attr_} + the values, dsz bytes each, at byte `at`
__device__ __forceinline__ void put_dict_header(uint32_t *img32, uint32_t at, uint32_t ref_size, uint32_t count, uint32_t dsz, uint32_t attr) {
  put_bytes(img32, at + 1u, 1u, ref_size);
  put_bytes(img32, at + 2u, 4u, count);
  put_bytes(img32, at + 6u, 2u, dsz);
  put_bytes(img32, at + 8u, 1u, attr);
}

// Pack one AUTO column whose codec is not RAW (every thread calls it).
__device__ void pack_auto(const ColSpec &cs, const AutoCol &A, const ColLayout &l, const int64_t row0, const uint32_t n,
                          const uint32_t nn, const uint32_t ext_bit, const uint32_t P, const AutoScratch &s, uint32_t *img32) {
  const uint32_t tid = threadIdx.x, o = l.store_off, dsz = A.dsz;
  const unsigned long long flip = cs.is_signed ? 1ull << (8u * cs.store_size - 1u) : 0ull;
  if (A.codec == 4) {   // INTEGER_BASE_DIFF
    const uint32_t ts = cs.store_size;
    const unsigned long long base = cs.is_signed ? (unsigned long long)sign_extend(A.kmin ^ flip, ts) : A.kmin;
    if (tid == 0) {
      put_bytes(img32, o + 1u, 1u, A.size);
      put_bytes(img32, o + 2u, ts, base);
    }
    const uint32_t bit0 = (o + 2u + ts) * 8u, val0 = bit0 + (nn ? ext_bit * n : 0u);
    const uint8_t *nl = (cs.nulls && nn) ? cs.nulls + row0 : nullptr;
    for (uint32_t r = tid; r < n; r += kThreads) {
      if (nl && nl[r] != 0) { or_bits(img32, bit0 + r * ext_bit, ext_bit, 1ull); continue; }
      const unsigned long long u = (unsigned long long)cs.vals[row0 + r] & cs.store_mask;
      const unsigned long long x = (cs.is_signed ? (unsigned long long)sign_extend(u, ts) : u) - base;
      if (A.bp) or_bits(img32, val0 + r * A.size, A.size, A.size >= 64u ? x : x & ((1ull << A.size) - 1ull));
      else put_bytes(img32, o + 2u + ts + l.bits_size + r * A.size, min((uint32_t)A.size, 8u), x);
    }
    return;
  }
  if (A.codec == 3 && A.exc == 0) {   // CONST without exceptions: the value, or const_ref_ 1 when every row is NULL
    if (tid == 0) {
      if (A.d == 0) put_bytes(img32, o + 2u, 1u, 1u);
      put_bytes(img32, o + 4u, 2u, 6u);
      if (A.d != 0) put_bytes(img32, o + 6u, cs.store_size, A.kmin ^ flip);
    }
    return;
  }
  const uint32_t d = sort_column(cs, row0, n, nn, P, s);
  if (A.codec == 1) {   // DICT: sorted dict, then the sorted ref of every row
    if (tid == 0) put_dict_header(img32, o, A.size, d, dsz, 0x1u | 0x2u);
    for (uint32_t v = tid; v < d; v += kThreads) put_bytes(img32, o + 9u + v * dsz, dsz, s.sk[s.hp[v]] ^ flip);
    const uint32_t at = o + A.len;
    for (uint32_t r = tid; r < n; r += kThreads) {
      if (A.bp) or_bits(img32, at * 8u + r * A.size, A.size, s.a[r]);
      else put_bytes(img32, at + r * A.size, A.size, s.a[r]);
    }
    return;
  }
  if (A.codec == 2) {   // RLE: refs and dict in first-occurrence order
    blk_scan(s.b, n, s.red);   // b[r]: distinct values whose first occurrence is at or before row r
    for (uint32_t r = tid; r < n; r += kThreads) s.hs[r] = (r == 0 || s.a[r] != s.a[r - 1]) ? 1u : 0u;
    __syncthreads();
    blk_scan(s.hs, n, s.red);
    const uint32_t runs = A.runs, rib = A.rib, refb = A.refb, head = 10u + runs * (rib + refb);
    if (tid == 0) {
      put_bytes(img32, o + 1u, 1u, (rib & 7u) | ((refb & 7u) << 3));
      put_bytes(img32, o + 2u, 4u, runs);
      put_bytes(img32, o + 6u, 4u, head);
      put_dict_header(img32, o + head, 0u, d, dsz, 0x1u);
    }
    for (uint32_t r = tid; r < n; r += kThreads) {
      if (!(r == 0 || s.a[r] != s.a[r - 1])) continue;
      const uint32_t k = s.hs[r] - 1u, x = s.a[r];
      const uint32_t ref = x == d ? d : s.b[s.sr[s.hp[x]]] - 1u;
      put_bytes(img32, o + 10u + k * rib, rib, r);
      put_bytes(img32, o + 10u + runs * rib + k * refb, refb, ref);
    }
    for (uint32_t v = tid; v < d; v += kThreads)
      put_bytes(img32, o + head + 9u + (s.b[s.sr[s.hp[v]]] - 1u) * dsz, dsz, s.sk[s.hp[v]] ^ flip);
    return;
  }
  // CONST with exceptions: [header][exception refs, u8][exception rows][sorted dict meta]
  const uint32_t cw = A.ref_w, exc = A.exc, rib = A.rib, head = 6u + exc * (rib + 1u);
  for (uint32_t r = tid; r < n; r += kThreads) s.hs[r] = s.a[r] != cw ? 1u : 0u;
  __syncthreads();
  blk_scan(s.hs, n, s.red);
  if (tid == 0) {
    put_bytes(img32, o + 1u, 1u, exc);
    put_bytes(img32, o + 2u, 1u, cw);
    put_bytes(img32, o + 3u, 1u, rib & 7u);
    put_bytes(img32, o + 4u, 2u, head);
    put_dict_header(img32, o + head, 0u, d, dsz, 0x1u | 0x2u);
  }
  for (uint32_t r = tid; r < n; r += kThreads) {
    if (s.a[r] == cw) continue;
    const uint32_t k = s.hs[r] - 1u;
    put_bytes(img32, o + 6u + k, 1u, s.a[r]);
    put_bytes(img32, o + 6u + exc + k * rib, rib, r);
  }
  for (uint32_t v = tid; v < d; v += kThreads) put_bytes(img32, o + head + 9u + v * dsz, dsz, s.sk[s.hp[v]] ^ flip);
}

// ---- phases both block encoders share (this kernel and the CS one in encode_cs.cuh) -----------------------------------------
// Ticket, zeroed image (cells are OR-ed in; padding up to the aligned slot must be zero) and the crc tables (slicing by 4:
// tab[k * 256 + i] = crc of byte i followed by k zero bytes). The caller reads *s_blk after its next barrier.
__device__ __forceinline__ void block_prologue(const Params &p, uint8_t *smem, uint32_t *tab, int *s_blk) {
  const int tid = threadIdx.x;
  if (tid == 0) *s_blk = atomicAdd(p.ticket, 1);
  // zero image: before anything else, under the ticket's round trip
  for (uint32_t i = (uint32_t)tid; i < p.slot_cap / 16u; i += kThreads) reinterpret_cast<uint4 *>(smem)[i] = make_uint4(0u, 0u, 0u, 0u);
  for (int i = tid; i < 256; i += kThreads) {
    uint32_t c = (uint32_t)i;
#pragma unroll
    for (int k = 0; k < 8; ++k) c = (c & 1u) ? kCrcPoly ^ (c >> 1) : c >> 1;
    tab[i] = c;
  }
  __syncthreads();
  for (int i = tid; i < 256; i += kThreads) {
    uint32_t c = tab[i];
#pragma unroll
    for (int k = 1; k < 4; ++k) {
      c = (c >> 8) ^ tab[c & 0xffu];
      tab[k * 256 + i] = c;
    }
  }
}

// ObDatum::checksum(0) of one cell: the crc32c of the 4 pack_ bytes (len_crc / null_crc), then of the value bytes. The CS stats pass
// calls it; the PAX one keeps the same steps inline (calling it there costs the PAX kernels 2 and 8 registers and a spill).
__device__ __forceinline__ uint32_t cell_crc(const uint32_t *tab, uint32_t crc, unsigned long long x, uint32_t datum_len, bool is_null) {
  if (!is_null) {
    if (datum_len == 8) {
      crc = crc_word(tab, crc, (uint32_t)x);
      crc = crc_word(tab, crc, (uint32_t)(x >> 32));
    } else if (datum_len == 4) {
      crc = crc_word(tab, crc, (uint32_t)x);
    } else {
      for (uint32_t k = 0; k < datum_len; ++k) crc = crc_byte(tab, crc, (uint32_t)(x >> (8u * k)) & 0xffu);
    }
  }
  return crc;
}

// The plan's aligned block size, published at once: the look-backs of the following blocks can pass over this one without waiting.
__device__ __forceinline__ void publish_size(const Params &p, int blk, bool host, uint32_t at) {
  if (blk > 0) {
    volatile unsigned long long *flags = p.flags;
    flags[blk] = (1ull << 62) | (host ? 0ull : (unsigned long long)((at + p.align - 1u) & ~(p.align - 1u)));
  }
}

// Output offset of the block: decoupled look-back over the aligned sizes (flag word: bits 63..62 state -- 1 aggregate, 2 inclusive
// prefix --, low 62 bits bytes). Tickets are handed out in scheduling order, so every predecessor is running or done. Thread 0.
__device__ __forceinline__ long long resolve_offset(const Params &p, int blk, uint32_t size, uint32_t slot, bool host) {
  volatile unsigned long long *flags = p.flags;
  unsigned long long excl = 0;
  if (blk > 0) {
    int j = blk - 1;
    for (;;) {
      unsigned long long f;
      do { f = flags[j]; } while ((f >> 62) == 0ull);
      excl += f & ((1ull << 62) - 1ull);
      if ((f >> 62) == 2ull) break;
      --j;
    }
  }
  flags[blk] = (2ull << 62) | (excl + slot);
  p.blk_off[blk] = (int64_t)excl;
  p.blk_size[blk] = size;
  if (blk == p.n_blocks - 1) p.totals[0] = excl + slot;
  if (host) atomicAdd(p.totals + 1, 1ull);
  return (long long)excl;
}

// Payload checksum in parallel: every thread the raw CRC of an odd-word-stride chunk, shifted to its position by one carry-less
// multiplication with x^(32 * words after it) mod P and XOR-reduced per warp into s_red. Every thread, after the pack's barrier.
__device__ __forceinline__ void payload_crc(const Params &p, const uint32_t *img32, const uint32_t *tab, uint32_t size, uint32_t *s_red) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t len = size - kHeaderSize, W = len >> 2;
  uint32_t lw = (W + kThreads - 1u) / kThreads;
  lw |= 1u;   // odd word stride between the threads' chunks: bank-conflict free
  const int padw = (int)(kThreads * lw) - (int)W;   // leading zero words of the conceptual message
  const uint32_t *pay = img32 + kHeaderSize / 4u;
  uint32_t crc = 0;
  {
    const int w0 = tid * (int)lw - padw;
    for (int w = max(w0, 0); w < w0 + (int)lw; ++w) crc = crc_word(tab, crc, pay[w]);
  }
  if (crc != 0) crc = gf2_mulmod(crc, p.xpow32[(uint32_t)(kThreads - 1 - tid) * lw]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) crc ^= __shfl_xor_sync(0xffffffffu, crc, o);
  if (lane == 0) s_red[warp] = crc;
}

// ObMicroBlockHeader (ob_micro_block_header.h:95-153) + its 16-bit checksum (ob_micro_block_header.cpp:193-233), then ONE bulk
// copy (TMA, cp.async.bulk shared -> global) of the aligned slot. Thread 0, after the barrier behind payload_crc.
__device__ __forceinline__ void finish_block(const Params &p, uint8_t *smem, const uint32_t *tab, const uint32_t *s_red, uint32_t size,
                                             uint32_t slot, uint32_t nrows, uint32_t rst, uint32_t opt, uint32_t opt2, uint32_t row_data_off,
                                             uint32_t original, long long off) {
  uint32_t *img32 = reinterpret_cast<uint32_t *>(smem);
  const uint32_t len = size - kHeaderSize;
  uint32_t crc = 0;
  for (int w = 0; w < kWarps; ++w) crc ^= s_red[w];
  for (uint32_t k = len & ~3u; k < len; ++k) crc = crc_byte(tab, crc, smem[kHeaderSize + k]);
  const uint32_t ncu = (uint32_t)p.n_cols, rk = (uint32_t)p.rowkey_cnt, flag16 = 1u << 2;   // all_lob_in_row_
  const uint16_t magic = (uint16_t)obf::MICRO_BLOCK_HEADER_MAGIC, version = (uint16_t)obf::MICRO_BLOCK_HEADER_VERSION;
  uint32_t cs = 0;
  auto f32 = [&](uint32_t x) { cs ^= (x & 0xffffu) ^ (x >> 16); };
  cs ^= magic;
  cs ^= version;
  cs ^= rst;
  cs ^= opt;
  f32(ncu); f32(rk); f32(flag16 & 1u); f32(opt2);
  f32(kHeaderSize); f32(nrows); f32(row_data_off); f32(original);
  f32(len); f32(len); f32(crc);   // 64-bit fields with a zero high half fold like 32-bit ones
  cs &= 0xffffu;
  img32[0] = (uint32_t)magic | ((uint32_t)version << 16);
  img32[1] = kHeaderSize;
  img32[2] = cs | (ncu << 16);
  img32[3] = rk | (flag16 << 16);
  img32[4] = nrows;
  img32[5] = rst | (opt << 8) | (opt2 << 16);   // row_store_type_, opt_, opt2_
  img32[6] = row_data_off;
  img32[7] = original;
  img32[8] = 0u; img32[9] = 0u;                 // max_merged_trans_version_
  img32[10] = len;                              // data_length_
  img32[11] = len;                              // data_zlength_
  img32[12] = crc; img32[13] = 0u;              // data_checksum_
  img32[14] = 0u; img32[15] = 0u;               // column_checksums_ptr_
  // the other threads made their shared-memory writes visible to the async proxy before the barrier above
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  uint8_t *dst = p.image + off;
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(smem)), "r"(slot) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

template <bool CKSUM, bool AUTO>
__global__ void __launch_bounds__(kThreads) obgpu_encode_blocks_kernel(const __grid_constant__ Params p) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint32_t *img32 = reinterpret_cast<uint32_t *>(smem);                 // block image, p.slot_cap bytes
  uint32_t *tab = reinterpret_cast<uint32_t *>(smem + p.slot_cap);      // 4 x 256 crc tables
  // per column scratch behind the tables: [kWarps][n_cols] max, [kWarps][n_cols] NULL count, [n_cols] layout
  unsigned long long *s_wmax = reinterpret_cast<unsigned long long *>(smem + p.slot_cap + 4096u);
  uint32_t *s_wnull = reinterpret_cast<uint32_t *>(s_wmax + kWarps * p.n_cols);
  ColLayout *s_lay = reinterpret_cast<ColLayout *>(s_wnull + kWarps * p.n_cols);
  // AUTO: [n_cols] AutoCol, then the sort scratch (auto_smem_bytes on the host counts the same)
  AutoCol *s_auto = nullptr;
  AutoScratch scr{};
  __shared__ uint32_t s_ared[AUTO ? kWarps : 1];
  if constexpr (AUTO) {
    uintptr_t q = (reinterpret_cast<uintptr_t>(s_lay + p.n_cols) + 15u) & ~(uintptr_t)15u;
    s_auto = reinterpret_cast<AutoCol *>(q);
    q = (q + (uintptr_t)p.n_cols * sizeof(AutoCol) + 15u) & ~(uintptr_t)15u;
    const uint32_t P = p.sort_cap, R = (uint32_t)p.rows_per_block;
    scr.sk = reinterpret_cast<unsigned long long *>(q);
    scr.sr = reinterpret_cast<uint32_t *>(scr.sk + P);
    scr.hs = scr.sr + P;
    scr.a = scr.hs + P;
    scr.b = scr.a + R;
    scr.hp = scr.b + R;
    scr.red = s_ared;
  }
  __shared__ uint32_t s_red[kWarps];
  __shared__ int s_blk;
  __shared__ uint32_t s_size, s_original, s_ext_bit, s_host;
  __shared__ long long s_off;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  block_prologue(p, smem, tab, &s_blk);
  const int blk = s_blk;
  const int64_t row0 = (int64_t)blk * p.rows_per_block;
  const uint32_t nrows = (uint32_t)min(p.rows_per_block, p.total_rows - row0);
  const int nc = p.n_cols;
  __syncthreads();

  // ---- stats (+ column checksums): four columns at a time, their loads in flight together ---------------------------------
  for (int c0 = 0; c0 < nc; c0 += 4) {
    unsigned long long mx[4] = {0, 0, 0, 0}, sum[4] = {0, 0, 0, 0};
    uint32_t nn[4] = {0, 0, 0, 0};
    // ObDatum::checksum(0) starts with the crc32c of the 4 pack_ bytes {len_:29, flag_:2, null_:1}: two values per column
    uint32_t len_crc[4] = {0, 0, 0, 0};
    const uint32_t null_crc = CKSUM ? crc_word(tab, 0u, 0x80000000u) : 0u;
    if (CKSUM) {
#pragma unroll
      for (int j = 0; j < 4; ++j) len_crc[j] = crc_word(tab, 0u, (uint32_t)p.col[min(c0 + j, nc - 1)].datum_len);
    }
    for (uint32_t r = (uint32_t)tid; r < nrows; r += kThreads) {
      unsigned long long x[4];
      uint32_t nlb[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = min(c0 + j, nc - 1);   // the tail repeats the last column (its results are dropped below)
        x[j] = (unsigned long long)p.col[c].vals[row0 + r];
        nlb[j] = p.col[c].nulls ? p.col[c].nulls[row0 + r] : 0u;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const ColSpec &cs = p.col[min(c0 + j, nc - 1)];
        const bool is_null = nlb[j] != 0;
        if (is_null) ++nn[j];
        else mx[j] = max(mx[j], x[j] & cs.store_mask);
        if (CKSUM) {   // ... then the crc of the value bytes
          uint32_t crc = is_null ? null_crc : len_crc[j];
          if (!is_null) {
            if (cs.datum_len == 8) {
              crc = crc_word(tab, crc, (uint32_t)x[j]);
              crc = crc_word(tab, crc, (uint32_t)(x[j] >> 32));
            } else if (cs.datum_len == 4) {
              crc = crc_word(tab, crc, (uint32_t)x[j]);
            } else {
              for (uint32_t k = 0; k < cs.datum_len; ++k) crc = crc_byte(tab, crc, (uint32_t)(x[j] >> (8u * k)) & 0xffu);
            }
          }
          sum[j] += crc;
        }
      }
    }
    // warp reductions through redux.sync (one instruction per 32-bit value): 64-bit max as (high word, then the low words of
    // the lanes that hold it); the checksum sum (< 2^32 * rows per lane) as 16-bit digits that cannot overflow 32 bits
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (c0 + j >= nc) break;
      const uint32_t hi = (uint32_t)(mx[j] >> 32), hmax = __reduce_max_sync(0xffffffffu, hi);
      const uint32_t lmax = __reduce_max_sync(0xffffffffu, hi == hmax ? (uint32_t)mx[j] : 0u);
      const uint32_t nsum = __reduce_add_sync(0xffffffffu, nn[j]);
      unsigned long long tot = 0;
      if (CKSUM) {
#pragma unroll
        for (int d = 0; d < 4; ++d) tot += (unsigned long long)__reduce_add_sync(0xffffffffu, (uint32_t)(sum[j] >> (16 * d)) & 0xffffu) << (16 * d);
      }
      if (lane == 0) {
        s_wmax[warp * nc + c0 + j] = ((unsigned long long)hmax << 32) | lmax;
        s_wnull[warp * nc + c0 + j] = nsum;
        if (CKSUM && tot != 0) atomicAdd(p.checksums + c0 + j, tot);
      }
    }
  }
  __syncthreads();

  if constexpr (AUTO) {   // ---- analysis of the AUTO columns, one after another, every thread --------------------------------
    for (int c = 0; c < nc; ++c) {
      if (!p.col[c].is_auto) continue;
      uint32_t nn = 0;
      for (int w = 0; w < kWarps; ++w) nn += s_wnull[w * nc + c];
      analyze_column(p.col[c], row0, nrows, nn, p.sort_cap, scr, s_auto[c]);
    }
  }

  // ---- plan: warp 0, one lane per column (two rounds for more than 32 columns) -------------------------------------------
  if (warp == 0) {
    uint32_t at = kHeaderSize + 16u * (uint32_t)nc;
    unsigned long long original = 0;
    bool host = false;
    // ext bits: 1 as soon as any column has a NULL (ob_micro_block_encoder.cpp:507-517; a major merge leaves no NOP cell)
    bool any_null = false;
    for (int c = lane; c < nc; c += 32) {
      uint32_t n = 0;
      for (int w = 0; w < kWarps; ++w) n += s_wnull[w * nc + c];
      any_null = any_null || n != 0;
    }
    const uint32_t ext_bit = __any_sync(0xffffffffu, any_null) ? 1u : 0u;
    for (int cb = 0; cb < nc; cb += 32) {
      const int c = cb + lane;
      uint32_t bytes = 0, nn = 0;
      ColLayout l{};
      bool var = false;
      if (c < nc) {
        unsigned long long mx = 0;
        for (int w = 0; w < kWarps; ++w) { mx = max(mx, s_wmax[w * nc + c]); nn += s_wnull[w * nc + c]; }
        bool bp;
        const uint32_t size = packing_size(mx, p.col[c].byte_only == 0, bp);
        // ObRawEncoder::traverse (ob_raw_encoder.cpp:106-110,150-155): NULLs dominate -> var-stored column
        var = bp ? (unsigned long long)size * nn > (unsigned long long)nrows * 16ull : (unsigned long long)size * nn > (unsigned long long)nrows * 2ull;
        l.has_null = nn != 0;
        l.bp = bp;
        l.size = (uint8_t)size;
        l.attr = (uint8_t)(0x1u /*FIX_LENGTH*/ | (nn ? 0x2u /*HAS_EXTEND_VALUE*/ : 0u) | (bp ? 0x4u /*BIT_PACKING*/ : 0u));
        const unsigned long long bits = (nn ? (unsigned long long)ext_bit * nrows : 0ull) + (bp ? (unsigned long long)size * nrows : 0ull);
        l.bits_size = (uint32_t)((bits + 7ull) / 8ull);
        bytes = l.bits_size + (bp ? 0u : size * nrows);
        if constexpr (AUTO) {
          if (p.col[c].is_auto) bytes = plan_auto(p.col[c], s_auto[c], nrows, nn, mx, ext_bit, l, var, bytes);
        }
      }
      uint32_t incl = bytes;   // column stores back to back: exclusive prefix over the columns
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
      }
      if (c < nc) {
        l.store_off = at + incl - bytes;
        s_lay[c] = l;
      }
      at += __shfl_sync(0xffffffffu, incl, 31);
      host = host || __any_sync(0xffffffffu, var);
      const uint32_t cells = c < nc ? (nrows - nn) * p.col[c].datum_len : 0u;
      original += __reduce_add_sync(0xffffffffu, cells);
    }
    // a layout above the shared-memory slot is left to the host writer, never written past the slot
    if constexpr (AUTO) host = host || at > p.slot_cap;
    if (lane == 0) {
      s_size = host ? 0u : at;
      s_original = (uint32_t)min(original, 0x7fffffffull);
      s_ext_bit = ext_bit;
      s_host = host;
      publish_size(p, blk, host, at);
    }
  }
  __syncthreads();
  const uint32_t size = s_size;
  const uint32_t slot = (size + p.align - 1u) & ~(p.align - 1u);
  if (tid == 0) s_off = resolve_offset(p, blk, size, slot, s_host);

  if (size != 0) {
    // ---- pack ------------------------------------------------------------------------------------------------------------
    const uint32_t ext_bit = s_ext_bit;   // (the image was zeroed at the start of the kernel)
    if (tid < nc) {   // ObColumnHeader: version_, type_ (RAW = 0), attr_, obj_type_, extend_value_index_, offset_ (from the meta start), length_
      const ColLayout l = s_lay[tid];
      uint32_t *h = img32 + (kHeaderSize + 16u * (uint32_t)tid) / 4u;
      h[0] = ((uint32_t)l.attr << 16) | ((uint32_t)p.col[tid].obj_type << 24);
      h[1] = 0u;
      h[2] = l.store_off - (kHeaderSize + 16u * (uint32_t)nc);
      h[3] = l.size;
      if constexpr (AUTO) {
        if (p.col[tid].is_auto && s_auto[tid].codec != 0) {   // type_ = the codec (COL_DICT 1 ... COL_INTEGER_BASE_DIFF 4)
          h[0] |= (uint32_t)s_auto[tid].codec << 8;
          h[3] = s_auto[tid].len;
        }
      }
    }
    for (int c = 0; c < nc; ++c) {
      const ColSpec &cs = p.col[c];
      const ColLayout l = s_lay[c];
      if constexpr (AUTO) {
        if (cs.is_auto && s_auto[c].codec != 0) {
          uint32_t nn = 0;
          for (int w = 0; w < kWarps; ++w) nn += s_wnull[w * nc + c];
          pack_auto(cs, s_auto[c], l, row0, nrows, nn, ext_bit, p.sort_cap, scr, img32);
          __syncthreads();
          continue;
        }
      }
      const int64_t *v = cs.vals + row0;
      const uint8_t *nl = (cs.nulls && l.has_null) ? cs.nulls + row0 : nullptr;
      const uint32_t bit0 = l.store_off * 8u;                                    // block bit address of the bit area
      const uint32_t val0 = bit0 + (l.has_null ? ext_bit * nrows : 0u);         // bit-packed values follow the ext bits
      for (uint32_t r = (uint32_t)tid; r < nrows; r += kThreads) {
        if (nl && nl[r] != 0) {
          const uint32_t b = bit0 + r * ext_bit;   // STORED_NULL = 1
          atomicOr(img32 + (b >> 5), 1u << (b & 31u));
          continue;
        }
        const unsigned long long x = (unsigned long long)v[r] & cs.store_mask;
        // bit-packed cells: size bits each behind the ext bits; byte-packed cells: 8 * size bits each behind the bit area
        const uint32_t w = l.bp ? l.size : 8u * l.size;
        const uint32_t b = (l.bp ? val0 : (l.store_off + l.bits_size) * 8u) + r * w, sh = b & 31u;
        const unsigned long long xm = w >= 64u ? x : (x & ((1ull << w) - 1ull));
        uint32_t *q = img32 + (b >> 5);
        atomicOr(q, (uint32_t)(xm << sh));
        if (sh + w > 32u) atomicOr(q + 1, (uint32_t)(xm >> (32u - sh)));
        if (sh + w > 64u) atomicOr(q + 2, (uint32_t)(xm >> (64u - sh)));
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // pack writes -> visible to the bulk copy issued by thread 0
    __syncthreads();
    payload_crc(p, img32, tab, size, s_red);   // ---- payload checksum
  }
  __syncthreads();

  if (tid == 0 && size != 0)   // header, row_data_offset_ = meta end == block end; opt_: row_index_byte 0, ext bits
    finish_block(p, smem, tab, s_red, size, slot, nrows, (uint32_t)obf::ENCODING_ROW_STORE, (s_ext_bit & 7u) << 3, 0u /*var columns*/,
                 size, s_original, s_off);
}

// Column checksums alone (ObMicroBlockChecksumHelper::cal_column_checksum over plain columns).
constexpr int kCkThreads = 256;
__global__ void __launch_bounds__(kCkThreads) obgpu_column_checksum_kernel(const __grid_constant__ Params p) {
  __shared__ uint32_t tab[1024];
  const int tid = threadIdx.x, lane = tid & 31;
  {
    uint32_t c = (uint32_t)tid;
#pragma unroll
    for (int k = 0; k < 8; ++k) c = (c & 1u) ? kCrcPoly ^ (c >> 1) : c >> 1;
    tab[tid] = c;
  }
  __syncthreads();
  {
    uint32_t c = tab[tid];
#pragma unroll
    for (int k = 1; k < 4; ++k) {
      c = (c >> 8) ^ tab[c & 0xffu];
      tab[k * 256 + tid] = c;
    }
  }
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * kCkThreads;
  for (int c = 0; c < p.n_cols; ++c) {
    const ColSpec &cs = p.col[c];
    const uint32_t len_crc = crc_word(tab, 0u, (uint32_t)cs.datum_len), null_crc = crc_word(tab, 0u, 0x80000000u);
    unsigned long long sum = 0;
    for (int64_t r = (int64_t)blockIdx.x * kCkThreads + tid; r < p.total_rows; r += stride) {
      uint32_t crc = null_crc;
      if (!(cs.nulls && cs.nulls[r] != 0)) {
        const unsigned long long x = (unsigned long long)cs.vals[r];
        crc = len_crc;
        if (cs.datum_len == 8) {
          crc = crc_word(tab, crc, (uint32_t)x);
          crc = crc_word(tab, crc, (uint32_t)(x >> 32));
        } else if (cs.datum_len == 4) {
          crc = crc_word(tab, crc, (uint32_t)x);
        } else {
          for (uint32_t k = 0; k < cs.datum_len; ++k) crc = crc_byte(tab, crc, (uint32_t)(x >> (8u * k)) & 0xffu);
        }
      }
      sum += crc;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0 && sum != 0) atomicAdd(p.checksums + c, sum);
  }
}

}  // namespace enc

struct obgpu_encoded {
  obgpu_ctx *ctx = nullptr;
  void *arena = nullptr;
  uint8_t *d_image = nullptr;
  int64_t *d_off = nullptr;
  uint32_t *d_size = nullptr;
  unsigned long long *d_checksums = nullptr, *d_totals = nullptr;
  int32_t n_cols = 0, n_blocks = 0;
  int64_t total_rows = 0;
  bool info_valid = false;
  obgpu_encoded_info info{};
};

// x^(32 k) mod P for every k a chunk shift can take (a CTA's shared memory bounds the block image), built once per device
static const uint32_t *enc_xpow_table(obgpu_ctx *ctx) {
  static std::mutex mu;
  static std::map<int, uint32_t *> tables;
  std::lock_guard<std::mutex> g(mu);
  auto it = tables.find(ctx->device);
  if (it != tables.end()) return it->second;
  const size_t lw_cap = (size_t)((ctx->max_smem_optin / 4 + enc::kThreads - 1) / enc::kThreads) | 1;
  const size_t n_pow = (size_t)(enc::kThreads - 1) * lw_cap + 1;
  std::vector<uint32_t> xpow(n_pow);
  uint32_t b = 0x80000000u;
  for (size_t k = 0; k < n_pow; ++k) {
    xpow[k] = b;
    for (int i = 0; i < 32; ++i) b = (b >> 1) ^ ((b & 1u) ? enc::kCrcPoly : 0u);
  }
  uint32_t *d = nullptr;
  if (cudaMalloc((void **)&d, n_pow * 4) != cudaSuccess) return nullptr;
  if (cudaMemcpy(d, xpow.data(), n_pow * 4, cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(d); return nullptr; }
  tables[ctx->device] = d;
  return d;
}

static int enc_fill_cols(enc::Params &p, const obgpu_encode_col *cols, int32_t n_cols) {
  for (int c = 0; c < n_cols; ++c) {
    const int sc = obf::store_class_of((uint8_t)cols[c].obj_type);
    if ((sc != 1 && sc != 2) || !cols[c].dev_vals) return sc == 5 ? OBGPU_NOT_SUPPORTED : OBGPU_INVALID_ARGUMENT;
    enc::ColSpec &s = p.col[c];
    s.vals = cols[c].dev_vals;
    s.nulls = cols[c].dev_null;
    s.store_mask = obf::low_mask((uint32_t)obf::type_store_size((uint8_t)cols[c].obj_type) * 8u);
    s.obj_type = (uint8_t)cols[c].obj_type;
    s.byte_only = cols[c].byte_packing_only ? 1 : 0;
    s.datum_len = (uint8_t)obf::datum_len_of((uint8_t)cols[c].obj_type);
    s.store_size = (uint8_t)obf::type_store_size((uint8_t)cols[c].obj_type);
    s.is_signed = sc == 1 ? 1 : 0;
  }
  p.n_cols = n_cols;
  return OBGPU_SUCCESS;
}

// The encoded handle's arena (totals, ticket, checksums, look-back flags, offsets, sizes, n_blocks slots of slot_cap bytes) and
// the one launch of a block encoder kernel over it. p: the columns and rowkey_cnt filled in.
static int enc_launch(obgpu_ctx *ctx, enc::Params &p, int64_t n_blocks64, int64_t total_rows, int64_t rows_per_block, int32_t align,
                      int64_t slot_cap, uint32_t sort_cap, size_t smem, void (*kernel)(enc::Params), obgpu_encoded **out) {
  const uint32_t lw_max = (uint32_t)(((slot_cap / 4 + enc::kThreads - 1) / enc::kThreads) | 1);
  const uint32_t *d_xpow = enc_xpow_table(ctx);
  if (!d_xpow) return OBGPU_ALLOCATE_MEMORY_FAILED;
  const int32_t n_cols = p.n_cols;
  std::unique_ptr<obgpu_encoded> e(new obgpu_encoded());
  e->ctx = ctx;
  e->n_cols = n_cols;
  e->n_blocks = (int32_t)n_blocks64;
  e->total_rows = total_rows;
  Scratch arena(ctx);
  const size_t o_ctl = arena.take(256 + (size_t)n_cols * 8);
  const size_t o_flags = arena.take((size_t)n_blocks64 * 8);
  const size_t o_off = arena.take((size_t)n_blocks64 * 8);
  const size_t o_size = arena.take((size_t)n_blocks64 * 4);
  const size_t o_img = arena.take((size_t)n_blocks64 * (size_t)slot_cap);
  CUDA_TRY(ctx, arena.alloc());
  uint8_t *a = arena.p;
  e->d_totals = (unsigned long long *)(a + o_ctl);
  e->d_checksums = (unsigned long long *)(a + o_ctl + 256);
  e->d_off = (int64_t *)(a + o_off);
  e->d_size = (uint32_t *)(a + o_size);
  e->d_image = a + o_img;
  CUDA_TRY(ctx, cudaMemsetAsync(a, 0, o_off, ctx->stream));   // totals, ticket, checksums, look-back flags
  p.n_blocks = e->n_blocks;
  p.want_checksums = 1;
  p.total_rows = total_rows;
  p.rows_per_block = rows_per_block;
  p.align = (uint32_t)align;
  p.slot_cap = (uint32_t)slot_cap;
  p.lw_max = lw_max;
  p.sort_cap = sort_cap;
  p.image = e->d_image;
  p.blk_off = e->d_off;
  p.blk_size = e->d_size;
  p.flags = (unsigned long long *)(a + o_flags);
  p.checksums = e->d_checksums;
  p.totals = e->d_totals;
  p.ticket = (int32_t *)(a + o_ctl + 128);
  p.xpow32 = d_xpow;
  CUDA_TRY(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<(unsigned)e->n_blocks, enc::kThreads, smem, ctx->stream>>>(p);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  e->arena = arena.release();
  *out = e.release();
  return OBGPU_SUCCESS;
}

extern "C" {

int obgpu_encode_columns_ex(obgpu_ctx *ctx, const obgpu_encode_col *cols, const int32_t *encodings, int32_t n_cols, int32_t rowkey_col_cnt,
                            int64_t total_rows, int64_t rows_per_block, int32_t align, obgpu_encoded **out) {
  if (!ctx || !cols || !out || n_cols <= 0 || n_cols > enc::kMaxCols || rowkey_col_cnt < 0 || rowkey_col_cnt > n_cols || total_rows <= 0 ||
      rows_per_block <= 0 || rows_per_block > (1 << 22) || align < 16 || align > 4096 || (align & (align - 1)) != 0)
    return OBGPU_INVALID_ARGUMENT;
  const int64_t n_blocks64 = (total_rows + rows_per_block - 1) / rows_per_block;
  if (n_blocks64 > 0x7fffffff) return OBGPU_NOT_SUPPORTED;
  int n_auto = 0;
  for (int c = 0; encodings && c < n_cols; ++c) {
    if (encodings[c] != OBGPU_ENC_RAW && encodings[c] != OBGPU_ENC_AUTO) return OBGPU_NOT_SUPPORTED;
    n_auto += encodings[c] == OBGPU_ENC_AUTO;
  }
  enc::Params p{};
  int rc = enc_fill_cols(p, cols, n_cols);
  if (rc != OBGPU_SUCCESS) return rc;
  for (int c = 0; encodings && c < n_cols; ++c) p.col[c].is_auto = encodings[c] == OBGPU_ENC_AUTO ? 1 : 0;
  cudaSetDevice(ctx->device);
  // the largest block: every RAW column 8 bytes wide + one ext bit per cell; an AUTO column the largest store of any codec it
  // can pick -- DICT / RLE at 12 bytes a row (8-byte values, 4-byte refs), BASE_DIFF at RAW's size + its 10-byte meta, CONST
  // below 512 bytes (at most 32 exceptions)
  const int64_t R = rows_per_block;
  const int64_t bound = (int64_t)enc::kHeaderSize + 16 * n_cols + (int64_t)(n_cols - n_auto) * (R * 8 + (R + 7) / 8 + 1) +
                        (int64_t)n_auto * (R * 12 + (R + 7) / 8 + 512);
  const int64_t slot_cap = (bound + align - 1) / align * align;
  size_t smem = (size_t)slot_cap + 4096 + (size_t)n_cols * (enc::kWarps * 12 + sizeof(enc::ColLayout)) + 16;
  uint32_t sort_cap = 1;
  while ((int64_t)sort_cap < R) sort_cap <<= 1;
  // AUTO: the AutoCol records and the sort scratch (keys, rows, scan: sort_cap each; refs, first occurrences: R each; R + 1 heads)
  if (n_auto) smem += 32 + (size_t)n_cols * sizeof(enc::AutoCol) + (size_t)sort_cap * 16 + (size_t)R * 12 + 4;
  if ((int64_t)smem > (int64_t)ctx->max_smem_optin - 8192) return OBGPU_NOT_SUPPORTED;   // block image does not fit one CTA's shared memory
  p.rowkey_cnt = rowkey_col_cnt;
  // the AUTO instantiation only when some column asks for it: RAW-only calls keep the RAW kernel
  return enc_launch(ctx, p, n_blocks64, total_rows, rows_per_block, align, slot_cap, sort_cap, smem,
                    n_auto ? enc::obgpu_encode_blocks_kernel<true, true> : enc::obgpu_encode_blocks_kernel<true, false>, out);
}

int obgpu_encoded_get_info(obgpu_encoded *e, obgpu_encoded_info *info) {
  if (!e || !info) return OBGPU_INVALID_ARGUMENT;
  obgpu_ctx *ctx = e->ctx;
  if (!e->info_valid) {
    cudaSetDevice(ctx->device);
    unsigned long long *hp = (unsigned long long *)ctx->h_pinned;
    CUDA_TRY(ctx, cudaMemcpyAsync(hp, e->d_totals, 16, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    e->info.image_size = (int64_t)hp[0];
    e->info.n_host_blocks = (int32_t)hp[1];
    e->info.n_blocks = e->n_blocks;
    e->info.total_rows = e->total_rows;
    e->info_valid = true;
  }
  *info = e->info;
  return OBGPU_SUCCESS;
}

int obgpu_encoded_fetch(obgpu_encoded *e, void *host_image, int64_t image_cap, int64_t *host_offsets, int64_t *host_sizes, int32_t blocks_cap) {
  if (!e) return OBGPU_INVALID_ARGUMENT;
  obgpu_encoded_info info;
  int rc = obgpu_encoded_get_info(e, &info);
  if (rc != OBGPU_SUCCESS) return rc;
  obgpu_ctx *ctx = e->ctx;
  if ((host_image && image_cap < info.image_size) || ((host_offsets || host_sizes) && blocks_cap < info.n_blocks)) return OBGPU_BUF_NOT_ENOUGH;
  if (host_image && info.image_size > 0) CUDA_TRY(ctx, cudaMemcpyAsync(host_image, e->d_image, (size_t)info.image_size, cudaMemcpyDeviceToHost, ctx->stream));
  if (host_offsets) CUDA_TRY(ctx, cudaMemcpyAsync(host_offsets, e->d_off, (size_t)info.n_blocks * 8, cudaMemcpyDeviceToHost, ctx->stream));
  std::vector<uint32_t> sz;
  if (host_sizes) {
    sz.resize((size_t)info.n_blocks);
    CUDA_TRY(ctx, cudaMemcpyAsync(sz.data(), e->d_size, (size_t)info.n_blocks * 4, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (host_sizes) for (int32_t i = 0; i < info.n_blocks; ++i) host_sizes[i] = sz[(size_t)i];
  return OBGPU_SUCCESS;
}

int obgpu_encoded_device_image(obgpu_encoded *e, const void **dev_image, const int64_t **dev_offsets, const uint32_t **dev_sizes) {
  if (!e) return OBGPU_INVALID_ARGUMENT;
  if (dev_image) *dev_image = e->d_image;
  if (dev_offsets) *dev_offsets = e->d_off;
  if (dev_sizes) *dev_sizes = e->d_size;
  return OBGPU_SUCCESS;
}

int obgpu_encoded_column_checksums(obgpu_encoded *e, int64_t *host_checksums) {
  if (!e || !host_checksums) return OBGPU_INVALID_ARGUMENT;
  obgpu_ctx *ctx = e->ctx;
  cudaSetDevice(ctx->device);
  CUDA_TRY(ctx, cudaMemcpyAsync(host_checksums, e->d_checksums, (size_t)e->n_cols * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return OBGPU_SUCCESS;
}

void obgpu_encoded_free(obgpu_encoded *e) {
  if (!e) return;
  if (e->arena) {
    cudaSetDevice(e->ctx->device);
    cudaFreeAsync(e->arena, e->ctx->stream);
  }
  delete e;
}

int obgpu_column_checksums(obgpu_ctx *ctx, const obgpu_encode_col *cols, int32_t n_cols, int64_t total_rows, int64_t *host_checksums) {
  if (!ctx || !cols || !host_checksums || n_cols <= 0 || n_cols > enc::kMaxCols || total_rows < 0) return OBGPU_INVALID_ARGUMENT;
  enc::Params p{};
  int rc = enc_fill_cols(p, cols, n_cols);
  if (rc != OBGPU_SUCCESS) return rc;
  cudaSetDevice(ctx->device);
  Scratch sums(ctx);
  CUDA_TRY(ctx, sums.alloc((size_t)n_cols * 8));
  unsigned long long *d = sums.at<unsigned long long>(0);
  CUDA_TRY(ctx, cudaMemsetAsync(d, 0, (size_t)n_cols * 8, ctx->stream));
  p.total_rows = total_rows;
  p.checksums = d;
  const int64_t want = (total_rows + enc::kCkThreads * 8 - 1) / (enc::kCkThreads * 8);
  const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)ctx->sm_count * 8));
  enc::obgpu_column_checksum_kernel<<<grid, enc::kCkThreads, 0, ctx->stream>>>(p);
  ctx->launches++;
  CUDA_TRY(ctx, cudaMemcpyAsync(host_checksums, d, (size_t)n_cols * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return OBGPU_SUCCESS;
}

int obgpu_encode_columns(obgpu_ctx *ctx, const obgpu_encode_col *cols, int32_t n_cols, int32_t rowkey_col_cnt, int64_t total_rows,
                         int64_t rows_per_block, int32_t align, obgpu_encoded **out) {
  return obgpu_encode_columns_ex(ctx, cols, nullptr, n_cols, rowkey_col_cnt, total_rows, rows_per_block, align, out);
}

}  // extern "C"

// The device columns of a merge result that result_cols names (-1 the rowkey, -2, -3 ...: the following rowkey columns, >= 0 a
// payload column) with obj_types, and the merged row count: what the encoder and the aggregate rows read of a column group.
static int merge_result_cols(obgpu_merge_result *res, const int32_t *result_cols, const int32_t *obj_types, int32_t n_cols,
                             std::vector<obgpu_encode_col> &cols, int64_t &rows) {
  obgpu_merge_info info;
  int rc = obgpu_merge_result_info(res, &info);
  if (rc != OBGPU_SUCCESS) return rc;
  if (info.out_rows <= 0) return OBGPU_INVALID_ARGUMENT;
  cols.assign((size_t)n_cols, obgpu_encode_col{});
  for (int i = 0; i < n_cols; ++i) {
    obgpu_encode_col &c = cols[(size_t)i];
    c.obj_type = obj_types[i];
    c.byte_packing_only = 0;
    const int32_t k = result_cols[i];
    if (k == -1) { c.dev_vals = res->d_out_key; c.dev_null = nullptr; }
    else if (k < -1) {
      const size_t m = (size_t)(-k - 2);
      if (m >= res->out_more.size()) return OBGPU_INVALID_ARGUMENT;
      c.dev_vals = res->out_more[m];
      c.dev_null = nullptr;
    } else {
      if (k >= res->n_cols) return OBGPU_INVALID_ARGUMENT;
      if (!res->col_is_string.empty() && res->col_is_string[(size_t)k]) return OBGPU_NOT_SUPPORTED;
      c.dev_vals = res->out_vals[(size_t)k];
      c.dev_null = res->out_null[(size_t)k];
    }
  }
  rows = info.out_rows;
  return OBGPU_SUCCESS;
}

extern "C" {

int obgpu_merge_result_encode_ex(obgpu_merge_result *res, const int32_t *result_cols, const int32_t *obj_types, const int32_t *encodings,
                                 int32_t n_cols, int32_t rowkey_col_cnt, int64_t rows_per_block, int32_t align, obgpu_encoded **out) {
  if (!res || !result_cols || !obj_types || n_cols <= 0 || n_cols > enc::kMaxCols || !out) return OBGPU_INVALID_ARGUMENT;
  for (int c = 0; encodings && c < n_cols; ++c)
    if (encodings[c] != OBGPU_ENC_RAW && encodings[c] != OBGPU_ENC_AUTO) return OBGPU_NOT_SUPPORTED;
  std::vector<obgpu_encode_col> cols;
  int64_t rows = 0;
  const int rc = merge_result_cols(res, result_cols, obj_types, n_cols, cols, rows);
  if (rc != OBGPU_SUCCESS) return rc;
  return obgpu_encode_columns_ex(res->ctx, cols.data(), encodings, n_cols, rowkey_col_cnt, rows, rows_per_block, align, out);
}

int obgpu_merge_result_encode(obgpu_merge_result *res, const int32_t *result_cols, const int32_t *obj_types, int32_t n_cols,
                              int32_t rowkey_col_cnt, int64_t rows_per_block, int32_t align, obgpu_encoded **out) {
  return obgpu_merge_result_encode_ex(res, result_cols, obj_types, nullptr, n_cols, rowkey_col_cnt, rows_per_block, align, out);
}

}  // extern "C"
