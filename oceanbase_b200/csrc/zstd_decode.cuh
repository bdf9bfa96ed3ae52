// One zstd frame (RFC 8878) -> exactly n_out bytes: the decoder behind stored_blocks.cuh (ObZstdCompressor_1_3_8::decompress,
// ZSTD_decompressDCtx into a buffer of data_length_ bytes, per micro-block payload in the reference).
// Self-contained and __host__ __device__: the same code runs in a warp on the device and single-threaded in a CPU build.
//   lanes   : every lane runs the serial walk (headers, bit readers, FSE states) on the same bytes, so the warp stays converged
//             and each lane holds every decoded value in registers. Shared state (the FSE / Huffman tables, their scratch)
//             is written by lane 0 alone, then the warp synchronises; the Huffman streams are decoded by lanes 0..3 (one each);
//             literal and match copies are spread over the lanes. A CPU build is the same code with one lane.
//   literals: Raw literals are read in place; RLE and Huffman literals go to the tail of the output, out[n_out - size, n_out),
//             as libzstd puts them inside dst. Safe because every sequence is checked to write only below the next unread
//             literal (op + match length + literals left <= n_out), which holds for every stream whose output fits.
//   tables  : LL / ML <= 2^9, OF <= 2^8 and Huffman <= 2^11 entries (RFC 8878 maxima); Repeat modes and Treeless literals use
//             the tables of the previous block of the same frame.
// Refused (kBad): a dictionary ID, a skippable or unknown magic, bytes after the first frame, a reserved bit or block type,
// a Frame_Content_Size != n_out, a read past a section or the input, a write past n_out, an offset outside
// 1..bytes produced, a bitstream not consumed exactly (Huffman streams, the sequence stream, FSE weight streams end at their
// last bit as RFC 8878 4.2.1.2 says), invalid FSE / Huffman descriptions, a wrong content checksum, output != n_out.
#pragma once
#include <stdint.h>

namespace zstdd {

#ifdef __CUDA_ARCH__
#define ZSTDD_SYNC() __syncwarp()
#define ZSTDD_BCAST(v) __shfl_sync(0xffffffffu, (v), 0)
#define ZSTDD_ANY(p) __any_sync(0xffffffffu, (p))
#else
#define ZSTDD_SYNC() ((void)0)
#define ZSTDD_BCAST(v) (v)
#define ZSTDD_ANY(p) (p)
#endif

constexpr int32_t kOk = 0, kBad = 2;
constexpr int64_t kBlockMax = 128 * 1024;
constexpr int kLLMaxLog = 9, kMLMaxLog = 9, kOFMaxLog = 8, kHufMaxLog = 11, kWeightMaxLog = 6;
constexpr int kLLMaxSym = 35, kMLMaxSym = 52, kOFMaxSym = 31;

struct Fse {   // FSE decoding table entry: symbol, bits to read, next state = base + those bits
  uint16_t base;
  uint8_t sym, nb;
};

// per-warp tables and scratch (shared memory on the device): 10.75 KiB
struct Work {
  Fse ll[1 << kLLMaxLog], ml[1 << kMLMaxLog], of[1 << kOFMaxLog], wt[1 << kWeightMaxLog];
  uint16_t huf[1 << kHufMaxLog];   // (symbol << 8) | bits, indexed by the next huf_log bits
  int16_t norm[256];
  uint16_t next[256];
  uint8_t w[256];
  int32_t ll_log, ml_log, of_log, huf_log;
};

__host__ __device__ __forceinline__ int highbit(uint32_t v) {   // index of the highest set bit, v > 0
#ifdef __CUDA_ARCH__
  return 31 - __clz(v);
#else
  return 31 - __builtin_clz(v);
#endif
}

__host__ __device__ __forceinline__ uint32_t ld_le(const uint8_t *p, int nbytes) {
  uint32_t v = 0;
  for (int k = 0; k < nbytes; ++k) v |= (uint32_t)p[k] << (8 * k);
  return v;
}

// k <= 32 bits of the little-endian bit string p[0, n) starting at bit `start` (>= 0); bytes past n read as zero
__host__ __device__ __forceinline__ uint32_t bits_at(const uint8_t *p, int64_t n, int64_t start, int k) {
  if (k == 0) return 0;
  const int64_t b = start >> 3;
  uint64_t v = 0;
  for (int j = 0; j < 5; ++j)
    if (b + j < n) v |= (uint64_t)p[b + j] << (8 * j);
  v >>= (start & 7);
  return (uint32_t)(v & ((1ull << k) - 1));
}

// backward bitstream (RFC 8878 4.1 / 4.2.2): read from the last byte's highest set bit toward bit 0. pos = bits left;
// a read past bit 0 returns zeros for the missing bits and leaves pos < 0 (overflow).
struct BackBits {
  const uint8_t *p;
  int64_t n, pos;
  __host__ __device__ bool init(const uint8_t *src, int64_t len) {
    p = src;
    n = len;
    if (len < 1 || src[len - 1] == 0) return false;
    pos = (len - 1) * 8 + highbit(src[len - 1]);
    return true;
  }
  __host__ __device__ __forceinline__ uint32_t peek(int k) const {
    if (k == 0) return 0;
    const int64_t s = pos - k;
    if (s >= 0) return bits_at(p, n, s, k);
    if (s + k <= 0) return 0;
    return bits_at(p, n, 0, (int)(s + k)) << (int)(-s);
  }
  __host__ __device__ __forceinline__ uint32_t read(int k) {
    const uint32_t v = peek(k);
    pos -= k;
    return v;
  }
};

// ---- FSE (RFC 8878 4.1.1) ------------------------------------------------------------------------------------------------
// Table description at src[0, n) -> norm[0, max_sym], *log. Returns the bytes used, or -1.
__host__ __device__ int64_t read_ncount(const uint8_t *src, int64_t n, int16_t *norm, int max_sym, int max_log, int32_t *log) {
  if (n < 1) return -1;
  int64_t bp = 0;
  const int al = (int)bits_at(src, n, 0, 4) + 5;
  bp = 4;
  if (al > max_log) return -1;
  int remaining = (1 << al) + 1, threshold = 1 << al, nb = al + 1, sym = 0;
  bool prev0 = false;
  for (;;) {
    if (prev0) {   // 2-bit repeat flags: r more zero counts, 3 = three and another flag
      int r;
      do {
        r = (int)bits_at(src, n, bp, 2);
        bp += 2;
        for (int k = 0; k < r; ++k, ++sym)
          if (sym <= max_sym) norm[sym] = 0;
      } while (r == 3 && sym <= max_sym);
      if (sym > max_sym) break;
    }
    const int mx = (2 * threshold - 1) - remaining;
    int count;
    const int low = (int)bits_at(src, n, bp, nb - 1);
    if (low < mx) {
      count = low;
      bp += nb - 1;
    } else {
      count = (int)bits_at(src, n, bp, nb);
      if (count >= threshold) count -= mx;
      bp += nb;
    }
    --count;
    remaining -= count < 0 ? -count : count;
    norm[sym++] = (int16_t)count;
    prev0 = count == 0;
    if (remaining < threshold) {
      if (remaining <= 1) break;
      nb = highbit((uint32_t)remaining) + 1;
      threshold = 1 << (nb - 1);
    }
    if (sym > max_sym) break;
  }
  if (remaining != 1 || sym > max_sym + 1) return -1;
  for (int s = sym; s <= max_sym; ++s) norm[s] = 0;
  const int64_t used = (bp + 7) >> 3;
  if (used > n) return -1;
  *log = al;
  return used;
}

// decoding table from normalised counts (sum of |norm| == 2^log); false when the spread does not visit every cell once
__host__ __device__ bool fse_build(Fse *t, const int16_t *norm, int nsym, int log, uint16_t *next) {
  const int size = 1 << log;
  int high = size - 1;
  for (int s = 0; s < nsym; ++s) {
    if (norm[s] == -1) {
      t[high--].sym = (uint8_t)s;
      next[s] = 1;
    } else {
      next[s] = (uint16_t)(norm[s] > 0 ? norm[s] : 0);
    }
  }
  const int step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
  int pos = 0;
  for (int s = 0; s < nsym; ++s)
    for (int i = 0; i < norm[s]; ++i) {
      t[pos].sym = (uint8_t)s;
      do pos = (pos + step) & mask; while (pos > high);
    }
  if (pos != 0) return false;
  for (int u = 0; u < size; ++u) {
    const uint32_t x = next[t[u].sym]++;
    const int nb = log - highbit(x);
    t[u].nb = (uint8_t)nb;
    t[u].base = (uint16_t)((x << nb) - size);
  }
  return true;
}

// predefined distributions (RFC 8878 3.1.1.3.2.2)
// (string literals: constant data, not per-thread arrays; 0xff stands for -1)
__host__ __device__ __forceinline__ void fse_default(Fse *t, int which, int16_t *norm, uint16_t *next, int32_t *log) {
  const char *ll = "\x04\x03\x02\x02\x02\x02\x02\x02\x02\x02\x02\x02\x02\x01\x01\x01\x02\x02\x02\x02\x02\x02\x02\x02\x02\x03\x02"
                   "\x01\x01\x01\x01\x01\xff\xff\xff\xff";
  const char *of = "\x01\x01\x01\x01\x01\x01\x02\x02\x02\x01\x01\x01\x01\x01\x01\x01\x01\x01\x01\x01\x01\x01\x01\x01\xff\xff\xff"
                   "\xff\xff";
  const int n = which == 0 ? 36 : which == 1 ? 29 : 53;
  for (int s = 0; s < n; ++s)
    norm[s] = which == 0 ? (int16_t)(int8_t)ll[s] : which == 1 ? (int16_t)(int8_t)of[s]
                                                   : (int16_t)(s == 0 ? 1 : s == 1 ? 4 : s == 2 ? 3 : s <= 8 ? 2 : s <= 45 ? 1 : -1);
  *log = which == 1 ? 5 : 6;
  fse_build(t, norm, n, *log, next);
}

// one sequence table (mode 0 predefined, 1 RLE, 2 FSE description, 3 repeat) from src[0, n); lane 0 only.
// Returns the bytes used, or -1.
__host__ __device__ int64_t seq_table(Work &w, int which, int mode, const uint8_t *src, int64_t n, bool have) {
  Fse *t = which == 0 ? w.ll : which == 1 ? w.of : w.ml;
  int32_t *log = which == 0 ? &w.ll_log : which == 1 ? &w.of_log : &w.ml_log;
  const int max_sym = which == 0 ? kLLMaxSym : which == 1 ? kOFMaxSym : kMLMaxSym;
  const int max_log = which == 0 ? kLLMaxLog : which == 1 ? kOFMaxLog : kMLMaxLog;
  if (mode == 0) {
    fse_default(t, which, w.norm, w.next, log);
    return 0;
  }
  if (mode == 1) {
    if (n < 1 || src[0] > max_sym) return -1;
    t[0].sym = src[0];
    t[0].nb = 0;
    t[0].base = 0;
    *log = 0;
    return 1;
  }
  if (mode == 3) return have ? 0 : -1;
  int32_t lg = 0;
  const int64_t used = read_ncount(src, n, w.norm, max_sym, max_log, &lg);
  if (used < 0 || !fse_build(t, w.norm, max_sym + 1, lg, w.next)) return -1;
  *log = lg;
  return used;
}

// ---- Huffman (RFC 8878 4.2.1) --------------------------------------------------------------------------------------------
// Huffman tree description at src[0, n) -> w.huf, w.huf_log; lane 0 only. Returns the bytes used, or -1.
__host__ __device__ int64_t huf_table(Work &w, const uint8_t *src, int64_t n) {
  if (n < 1) return -1;
  const int hb = src[0];
  int nw = 0;
  int64_t used;
  if (hb >= 128) {   // direct: 4-bit weights
    nw = hb - 127;
    used = 1 + (nw + 1) / 2;
    if (used > n) return -1;
    for (int i = 0; i < nw; ++i) w.w[i] = (uint8_t)((i & 1) ? src[1 + i / 2] & 15 : src[1 + i / 2] >> 4);
  } else {           // FSE-compressed weights: two interleaved states over a backward stream
    used = 1 + hb;
    if (used > n) return -1;
    int32_t lg = 0;
    const int64_t nc = read_ncount(src + 1, hb, w.norm, 255, kWeightMaxLog, &lg);
    if (nc < 0 || !fse_build(w.wt, w.norm, 256, lg, w.next)) return -1;
    BackBits br;
    if (!br.init(src + 1 + nc, hb - nc)) return -1;
    uint32_t s1 = br.read(lg), s2 = br.read(lg);
    for (;;) {
      if (nw >= 254) return -1;
      w.w[nw++] = w.wt[s1].sym;
      s1 = w.wt[s1].base + br.read(w.wt[s1].nb);
      if (br.pos < 0) { w.w[nw++] = w.wt[s2].sym; break; }
      if (nw >= 254) return -1;
      w.w[nw++] = w.wt[s2].sym;
      s2 = w.wt[s2].base + br.read(w.wt[s2].nb);
      if (br.pos < 0) { w.w[nw++] = w.wt[s1].sym; break; }
    }
  }
  uint32_t total = 0, rank1 = 0;
  for (int i = 0; i < nw; ++i) {
    if (w.w[i] > 12) return -1;
    total += (1u << w.w[i]) >> 1;
    rank1 += w.w[i] == 1;
  }
  if (total == 0) return -1;
  const int maxb = highbit(total) + 1;
  if (maxb > kHufMaxLog) return -1;
  const uint32_t rest = (1u << maxb) - total;
  if (rest != (1u << highbit(rest))) return -1;
  w.w[nw] = (uint8_t)(highbit(rest) + 1);
  rank1 += w.w[nw] == 1;
  const int nsym = nw + 1;
  if (rank1 < 2 || (rank1 & 1)) return -1;
  uint32_t pos = 0;
  for (int wt = 1; wt <= maxb; ++wt)
    for (int s = 0; s < nsym; ++s)
      if (w.w[s] == wt) {
        const uint16_t e = (uint16_t)((s << 8) | (maxb + 1 - wt));
        for (uint32_t k = 0; k < (1u << (wt - 1)); ++k) w.huf[pos + k] = e;
        pos += 1u << (wt - 1);
      }
  w.huf_log = maxb;
  return used;
}

// one Huffman stream src[0, n) -> dst[0, cnt); true when it decodes and ends exactly at its first bit
__host__ __device__ bool huf_stream(const Work &w, const uint8_t *src, int64_t n, uint8_t *dst, int64_t cnt) {
  BackBits br;
  if (!br.init(src, n)) return false;
  const int lg = w.huf_log;
  for (int64_t i = 0; i < cnt; ++i) {
    const uint16_t e = w.huf[br.peek(lg)];
    dst[i] = (uint8_t)(e >> 8);
    br.pos -= e & 0xff;
  }
  return br.pos == 0;
}

// ---- XXH64, seed 0 (the frame's Content_Checksum is its low 32 bits) -----------------------------------------------------
__host__ __device__ __forceinline__ uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__host__ __device__ __forceinline__ uint64_t ld64le(const uint8_t *p) { return (uint64_t)ld_le(p, 4) | ((uint64_t)ld_le(p + 4, 4) << 32); }
__host__ __device__ uint64_t xxh64(const uint8_t *p, int64_t len) {
  const uint64_t P1 = 11400714785074694791ull, P2 = 14029467366897019727ull, P3 = 1609587929392839161ull, P4 = 9650029242287828579ull,
                 P5 = 2870177450012600261ull;
  auto round = [&](uint64_t acc, uint64_t in) { return rotl64(acc + in * P2, 31) * P1; };
  int64_t i = 0;
  uint64_t h;
  if (len >= 32) {
    uint64_t v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0 - P1;
    for (; i + 32 <= len; i += 32) {
      v1 = round(v1, ld64le(p + i));
      v2 = round(v2, ld64le(p + i + 8));
      v3 = round(v3, ld64le(p + i + 16));
      v4 = round(v4, ld64le(p + i + 24));
    }
    h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
    h = (h ^ round(0, v1)) * P1 + P4;
    h = (h ^ round(0, v2)) * P1 + P4;
    h = (h ^ round(0, v3)) * P1 + P4;
    h = (h ^ round(0, v4)) * P1 + P4;
  } else {
    h = P5;
  }
  h += (uint64_t)len;
  for (; i + 8 <= len; i += 8) h = rotl64(h ^ round(0, ld64le(p + i)), 27) * P1 + P4;
  if (i + 4 <= len) {
    h = rotl64(h ^ ((uint64_t)ld_le(p + i, 4) * P1), 23) * P2 + P3;
    i += 4;
  }
  for (; i < len; ++i) h = rotl64(h ^ (p[i] * P5), 11) * P1;
  h ^= h >> 33;
  h *= P2;
  h ^= h >> 29;
  h *= P3;
  h ^= h >> 32;
  return h;
}

// ---- copies spread over the lanes ------------------------------------------------------------------------------------------
// dst <= src (or disjoint): a chunk is loaded by every lane before any lane stores it, so a forward overlap is safe
__host__ __device__ __forceinline__ void copy_fwd(uint8_t *dst, const uint8_t *src, int64_t n, int lane, int nl) {
  for (int64_t b = 0; b < n; b += nl) {
    const int64_t i = b + lane;
    const uint8_t v = i < n ? src[i] : 0;
    ZSTDD_SYNC();
    if (i < n) dst[i] = v;
  }
  ZSTDD_SYNC();
}

// match at distance off (1 <= off <= bytes before dst): every source byte precedes dst, out[i] = out[i - off + (i mod off)]
__host__ __device__ __forceinline__ void copy_match(uint8_t *dst, int64_t off, int64_t n, int lane, int nl) {
  const uint8_t *src = dst - off;
  for (int64_t i = lane; i < n; i += nl) dst[i] = src[i < off ? i : i % off];
  ZSTDD_SYNC();
}

// ---- blocks ----------------------------------------------------------------------------------------------------------------
struct FrameState {
  int64_t op;          // bytes produced
  uint32_t rep[3];     // repeat offsets
  bool have_huf, have_seq;
};

// Literals_Length / Match_Length codes (RFC 8878 3.1.1.3.2.1.1): baseline and extra bits. The short-code bits are packed one
// nibble per code; a baseline is the previous one plus 2^(previous bits).
__host__ __device__ __forceinline__ void ll_code(int c, uint32_t &base, int &bits) {
  if (c < 16) { base = (uint32_t)c; bits = 0; return; }
  if (c >= 25) { bits = c - 19; base = 1u << bits; return; }
  const uint64_t nb = 0x433221111ull;   // codes 16..24
  base = 16;
  for (int k = 16; k < c; ++k) base += 1u << ((nb >> (4 * (k - 16))) & 15);
  bits = (int)((nb >> (4 * (c - 16))) & 15);
}
__host__ __device__ __forceinline__ void ml_code(int c, uint32_t &base, int &bits) {
  if (c < 32) { base = (uint32_t)c + 3; bits = 0; return; }
  if (c >= 43) { bits = c - 36; base = (1u << bits) + 3; return; }
  const uint64_t nb = 0x54433221111ull;   // codes 32..42
  base = 35;
  for (int k = 32; k < c; ++k) base += 1u << ((nb >> (4 * (k - 32))) & 15);
  bits = (int)((nb >> (4 * (c - 32))) & 15);
}

// one Compressed_Block in[0, n) appending to out (frame output of n_out bytes)
__host__ __device__ int32_t compressed_block(const uint8_t *in, int64_t n, uint8_t *out, int64_t n_out, Work &w, FrameState &fs, int lane,
                                             int nl) {
  if (n < 2) return kBad;
  const int64_t room = n_out - fs.op;
  // literals section
  const uint32_t b0 = in[0];
  const int ltype = (int)(b0 & 3), sf = (int)((b0 >> 2) & 3);
  int64_t lit_size, pos;
  const uint8_t *lit;
  if (ltype <= 1) {   // Raw / RLE
    int lh = sf == 1 ? 2 : sf == 3 ? 3 : 1;
    if (lh + (ltype == 1 ? 1 : 0) > n) return kBad;
    lit_size = lh == 1 ? (b0 >> 3) : lh == 2 ? (ld_le(in, 2) >> 4) : (ld_le(in, 3) >> 4);
    if (lit_size > kBlockMax || lit_size > room) return kBad;
    if (ltype == 0) {
      if (lh + lit_size > n) return kBad;
      lit = in + lh;
      pos = lh + lit_size;
    } else {
      uint8_t *tail = out + n_out - lit_size;
      const uint8_t v = in[lh];
      for (int64_t i = lane; i < lit_size; i += nl) tail[i] = v;
      ZSTDD_SYNC();
      lit = tail;
      pos = lh + 1;
    }
  } else {            // Compressed / Treeless
    if (n < 5) return kBad;
    const int lh = sf <= 1 ? 3 : sf == 2 ? 4 : 5;
    const bool single = sf == 0;
    int64_t csize;
    if (lh == 3) {
      const uint32_t v = ld_le(in, 3);
      lit_size = (v >> 4) & 0x3ff;
      csize = (v >> 14) & 0x3ff;
    } else if (lh == 4) {
      const uint32_t v = ld_le(in, 4);
      lit_size = (v >> 4) & 0x3fff;
      csize = v >> 18;
    } else {
      const uint32_t v = ld_le(in, 4);
      lit_size = (v >> 4) & 0x3ffff;
      csize = (int64_t)(v >> 22) | ((int64_t)in[4] << 10);
    }
    if (lit_size > kBlockMax || (!single && lit_size < 6) || lh + csize > n || lit_size > room) return kBad;
    int64_t tree = 0;
    if (ltype == 2) {
      int64_t r = 0;
      if (lane == 0) r = huf_table(w, in + lh, csize);
      r = ZSTDD_BCAST(r);
      ZSTDD_SYNC();
      if (r < 0) return kBad;
      tree = r;
      fs.have_huf = true;
    } else if (!fs.have_huf) {
      return kBad;
    }
    const uint8_t *st = in + lh + tree;
    const int64_t ssz = csize - tree;
    uint8_t *tail = out + n_out - lit_size;
    bool bad = false;
    if (single) {
      if (lane == 0) bad = !huf_stream(w, st, ssz, tail, lit_size);
    } else {
      const int64_t seg = (lit_size + 3) / 4;
      if (ssz < 10) return kBad;
      const int64_t l1 = ld_le(st, 2), l2 = ld_le(st + 2, 2), l3 = ld_le(st + 4, 2), l4 = ssz - 6 - l1 - l2 - l3;
      if (l4 < 0 || 3 * seg > lit_size) return kBad;
      for (int k = lane; k < 4; k += nl) {
        const int64_t so = 6 + (k > 0 ? l1 : 0) + (k > 1 ? l2 : 0) + (k > 2 ? l3 : 0);
        const int64_t sl = k == 0 ? l1 : k == 1 ? l2 : k == 2 ? l3 : l4;
        bad = bad || !huf_stream(w, st + so, sl, tail + k * seg, k < 3 ? seg : lit_size - 3 * seg);
      }
    }
    ZSTDD_SYNC();
    if (ZSTDD_ANY(bad)) return kBad;
    lit = tail;
    pos = lh + csize;
  }
  // sequences section
  if (pos >= n) return kBad;
  int64_t nseq = in[pos++];
  if (nseq >= 128) {
    if (nseq == 255) {
      if (pos + 2 > n) return kBad;
      nseq = (int64_t)ld_le(in + pos, 2) + 0x7f00;
      pos += 2;
    } else {
      if (pos + 1 > n) return kBad;
      nseq = ((nseq - 128) << 8) + in[pos];
      pos += 1;
    }
  }
  int64_t lit_left = lit_size;
  if (nseq == 0) {
    if (pos != n) return kBad;
  } else {
    if (pos + 1 > n) return kBad;
    const uint32_t modes = in[pos++];
    if (modes & 3) return kBad;
    int64_t r = 0;
    if (lane == 0) {
      int64_t p = pos;
      for (int k = 0; k < 3 && p >= 0; ++k) {   // LL (bits 7-6), OF (5-4), ML (3-2)
        const int64_t u = seq_table(w, k, (int)((modes >> (6 - 2 * k)) & 3), in + p, n - p, fs.have_seq);
        p = u < 0 ? -1 : p + u;
      }
      r = p;
    }
    r = ZSTDD_BCAST(r);
    ZSTDD_SYNC();
    if (r < 0) return kBad;
    pos = r;
    fs.have_seq = true;
    BackBits br;
    if (!br.init(in + pos, n - pos)) return kBad;
    uint32_t sll = br.read(w.ll_log), sof = br.read(w.of_log), sml = br.read(w.ml_log);
    for (int64_t i = 0; i < nseq; ++i) {
      const Fse el = w.ll[sll], eo = w.of[sof], em = w.ml[sml];
      const uint32_t ofv = (1u << eo.sym) + br.read(eo.sym);
      uint32_t mb, lb;
      int mbits, lbits;
      ml_code(em.sym, mb, mbits);
      ll_code(el.sym, lb, lbits);
      const int64_t ml = mb + br.read(mbits), ll = lb + br.read(lbits);
      int64_t off;
      if (ofv > 3) {
        off = ofv - 3;
        fs.rep[2] = fs.rep[1];
        fs.rep[1] = fs.rep[0];
        fs.rep[0] = (uint32_t)off;
      } else {
        const int idx = (int)ofv - 1 + (ll == 0 ? 1 : 0);   // 0: rep1, 1: rep2, 2: rep3, 3: rep1 - 1
        off = idx == 3 ? (int64_t)fs.rep[0] - 1 : (int64_t)fs.rep[idx];
        if (idx != 0) {
          if (idx != 1) fs.rep[2] = fs.rep[1];
          fs.rep[1] = fs.rep[0];
          fs.rep[0] = (uint32_t)off;
        }
      }
      if (i + 1 < nseq) {
        sll = el.base + br.read(el.nb);
        sml = em.base + br.read(em.nb);
        sof = eo.base + br.read(eo.nb);
      }
      // bounds: literals available, the match ends below the next unread literal, offset inside the produced bytes
      if (ll > lit_left || fs.op + ml + lit_left > n_out || off < 1 || off > fs.op + ll) return kBad;
      copy_fwd(out + fs.op, lit, ll, lane, nl);
      lit += ll;
      lit_left -= ll;
      fs.op += ll;
      copy_match(out + fs.op, off, ml, lane, nl);
      fs.op += ml;
    }
    if (br.pos != 0) return kBad;
  }
  if (fs.op + lit_left > n_out) return kBad;
  copy_fwd(out + fs.op, lit, lit_left, lane, nl);
  fs.op += lit_left;
  return kOk;
}

// one zstd frame in[0, n_in) -> out[0, n_out); kOk only when the frame is the whole input and decodes to exactly n_out bytes
__host__ __device__ int32_t decode_frame(const uint8_t *in, int64_t n_in, uint8_t *out, int64_t n_out, Work &w, int lane, int nl) {
  if (n_in < 5 || ld_le(in, 4) != 0xFD2FB528u) return kBad;   // skippable frames and other magics included
  const uint32_t fhd = in[4];
  const int fcs_flag = (int)(fhd >> 6), did_flag = (int)(fhd & 3);
  const bool single = (fhd >> 5) & 1, cksum = (fhd >> 2) & 1;
  if (fhd & 8) return kBad;   // reserved bit
  int64_t p = 5;
  if (!single) {
    if (p + 1 > n_in) return kBad;
    if (10 + (in[p] >> 3) > 31) return kBad;   // Window_Log above ZSTD_WINDOWLOG_MAX
    ++p;
  }
  const int did_size = did_flag == 0 ? 0 : did_flag == 1 ? 1 : did_flag == 2 ? 2 : 4;
  if (p + did_size > n_in) return kBad;
  if (did_size && ld_le(in + p, did_size) != 0) return kBad;   // a dictionary is required
  p += did_size;
  const int fcs_size = fcs_flag == 0 ? (single ? 1 : 0) : fcs_flag == 1 ? 2 : fcs_flag == 2 ? 4 : 8;
  if (p + fcs_size > n_in) return kBad;
  if (fcs_size) {
    uint64_t fcs = fcs_size == 8 ? ld64le(in + p) : ld_le(in + p, fcs_size);
    if (fcs_size == 2) fcs += 256;
    if (fcs != (uint64_t)n_out) return kBad;
    p += fcs_size;
  }
  FrameState fs;
  fs.op = 0;
  fs.rep[0] = 1;
  fs.rep[1] = 4;
  fs.rep[2] = 8;
  fs.have_huf = fs.have_seq = false;
  for (;;) {
    if (p + 3 > n_in) return kBad;
    const uint32_t bh = ld_le(in + p, 3);
    p += 3;
    const int type = (int)((bh >> 1) & 3);
    const int64_t bs = bh >> 3;
    if (type == 3 || bs > kBlockMax) return kBad;
    if (type == 0) {
      if (p + bs > n_in || fs.op + bs > n_out) return kBad;
      for (int64_t i = lane; i < bs; i += nl) out[fs.op + i] = in[p + i];
      p += bs;
      fs.op += bs;
    } else if (type == 1) {
      if (p + 1 > n_in || fs.op + bs > n_out) return kBad;
      const uint8_t v = in[p];
      for (int64_t i = lane; i < bs; i += nl) out[fs.op + i] = v;
      p += 1;
      fs.op += bs;
    } else {
      if (p + bs > n_in) return kBad;
      if (compressed_block(in + p, bs, out, n_out, w, fs, lane, nl) != kOk) return kBad;
      p += bs;
    }
    ZSTDD_SYNC();
    if (bh & 1) break;
  }
  if (cksum) {
    if (p + 4 > n_in) return kBad;
    uint32_t ok = 0;
    if (lane == 0) ok = (uint32_t)xxh64(out, fs.op) == ld_le(in + p, 4) ? 1u : 0u;
    ok = ZSTDD_BCAST(ok);
    if (!ok) return kBad;
    p += 4;
  }
  return p == n_in && fs.op == n_out ? kOk : kBad;
}

}  // namespace zstdd
