// One zlib stream (RFC 1950 around RFC 1951 DEFLATE) -> exactly n_out bytes: the decoder behind stored_blocks.cuh
// (ObZlibCompressor::decompress, zlib's uncompress into a buffer of data_length_ bytes, per micro-block payload in the reference).
// Self-contained and __host__ __device__: the same code runs in a warp on the device and single-threaded in a CPU build.
//   lanes   : every lane walks the same bit stream (block headers, code lengths, symbols), so symbols are warp-uniform and
//             need no shuffles. Shared state (the code tables) is counted by lane 0 and filled by every lane, then the warp
//             synchronises. Literals: lane k keeps the k-th pending literal in a register; the run is stored with one store per
//             lane when a match or an end of block arrives or 32 literals are pending. Matches and stored blocks are copied by
//             the whole warp; the Adler-32 of the output is per-lane strided sums reduced over the warp.
//   tables  : per code, counts per length and the symbols sorted by (length, value) (zlib's inflate_table order), plus a root
//             table indexed by the next kLitRoot / kDistRoot stream bits: (length << 9) | symbol for codes that short, 0 else.
//             A longer (or missing) code is decoded canonically from the counts, one length at a time, resuming after the
//             root's lengths from a state kept with the code (about 2 % of the symbols of zlib level 1..9 micro-blocks).
// Refused (kBad), as zlib's inflate refuses: CM != 8, CINFO > 7, a header check not divisible by 31, FDICT, BTYPE 3, stored
// LEN != ~NLEN, HLIT > 286 or HDIST > 30, a code-length repeat (16) with no previous length, a code-length run past HLIT + HDIST,
// an over-subscribed code, an incomplete code (the code-length code always; a literal/length or distance code unless it is
// one code of length 1), no end-of-block code, an undecodable code, length symbols 286 / 287, distance symbols 30 / 31, a
// distance beyond the bytes produced, a wrong Adler-32. Bounds: every read inside in[0, n_in), every write inside
// out[0, n_out); the output must be exactly n_out bytes and the Adler-32 must end exactly at n_in (zlib ignores bytes after it).
#pragma once
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#define __forceinline__ inline
#endif

namespace zlibd {

#ifdef __CUDA_ARCH__
#define ZLIBD_SYNC() __syncwarp()
#define ZLIBD_BCAST(v) __shfl_sync(0xffffffffu, (v), 0)
#define ZLIBD_SUM(v) zlibd::warp_sum(v)
#else
#define ZLIBD_SYNC() ((void)0)
#define ZLIBD_BCAST(v) (v)
#define ZLIBD_SUM(v) (v)
#endif

constexpr int32_t kOk = 0, kBad = 2;
constexpr int kLitRoot = 10, kDistRoot = 8, kMaxBits = 15;
constexpr uint32_t kAdlerMod = 65521;
constexpr int64_t kMaxStream = 0x7fff0000;   // longest input and output: the bit reader's offsets stay in 32 bits

struct Code {   // canonical Huffman code: count[len], symbols sorted by (length, value)
  uint16_t count[kMaxBits + 1];
  uint16_t sym[288];
  uint16_t rfirst, rindex;   // the canonical walk's first / index after the root table's lengths (decode_long)
};

// per-warp tables (shared memory on the device): 4.6 KiB
struct Work {
  uint16_t lroot[1 << kLitRoot], droot[1 << kDistRoot];
  Code lit, dist, cl;
  uint8_t lens[288 + 32];
  int32_t fixed;   // lit / dist hold the fixed code
};

#ifdef __CUDA_ARCH__
__device__ __forceinline__ uint64_t warp_sum(uint64_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
#endif

// LSB-first bit reader over in[0, n), n <= kMaxStream: bytes past n read as zero; overrun() once more than n bytes are consumed.
// 32-bit offsets keep the whole walk in few registers.
struct Bits {
  const uint8_t *in;
  uint32_t n, p;   // p: next byte to load
  uint64_t hold;
  int nb;         // bits in hold
  __host__ __device__ __forceinline__ void refill() {
    while (nb <= 56) {
      hold |= (uint64_t)(p < n ? in[p] : 0) << nb;
      ++p;
      nb += 8;
    }
  }
  __host__ __device__ __forceinline__ uint32_t peek(int k) const { return (uint32_t)(hold & ((1ull << k) - 1)); }
  __host__ __device__ __forceinline__ void drop(int k) {
    hold >>= k;
    nb -= k;
  }
  __host__ __device__ __forceinline__ uint32_t take(int k) {   // k <= nb
    const uint32_t v = peek(k);
    drop(k);
    return v;
  }
  __host__ __device__ __forceinline__ uint32_t next_byte() const { return p - (uint32_t)(nb >> 3); }   // first byte not wholly consumed
  __host__ __device__ __forceinline__ bool overrun() const { return 8 * ((int32_t)p - (int32_t)n) > nb; }
  __host__ __device__ __forceinline__ void to_byte(uint32_t byte) {   // restart at a byte offset
    p = byte;
    hold = 0;
    nb = 0;
  }
};

// counts and sorted symbols of lens[0, n); lane 0 only. false for an over-subscribed code or an incomplete one that
// inflate_table refuses (any incomplete code-length code; else anything but one code of length 1). An empty code is
// accepted (every decode through it fails), except as the code-length code (it could only lead to a missing end-of-block).
__host__ __device__ __forceinline__ bool build_code(Code &c, const uint8_t *lens, int n, bool codes) {
  for (int l = 0; l <= kMaxBits; ++l) c.count[l] = 0;
  for (int s = 0; s < n; ++s) c.count[lens[s]]++;
  int max = kMaxBits;
  while (max > 0 && c.count[max] == 0) --max;
  if (max == 0) return !codes;
  int left = 1;
  for (int l = 1; l <= kMaxBits; ++l) {
    left = (left << 1) - c.count[l];
    if (left < 0) return false;
  }
  if (left > 0 && (codes || max != 1)) return false;
  uint16_t offs[kMaxBits + 1];
  offs[1] = 0;
  for (int l = 1; l < kMaxBits; ++l) offs[l + 1] = (uint16_t)(offs[l] + c.count[l]);
  for (int s = 0; s < n; ++s)
    if (lens[s]) c.sym[offs[lens[s]]++] = (uint16_t)s;
  return true;
}

// canonical decode of the stream bits v (LSB first) with codes of at most `maxlen` bits: (length << 9) | symbol, 0 when no code
// of at most maxlen bits is a prefix of v. The walk may start after length len0 (code, first, index: its state there).
__host__ __device__ __forceinline__ uint32_t decode_slow(const Code &c, uint32_t v, int maxlen, int len0 = 0, int code = 0, int first = 0,
                                                         int index = 0) {
  for (int len = len0 + 1; len <= maxlen; ++len) {
    code |= (int)((v >> (len - 1)) & 1u);
    const int count = c.count[len];
    if (code - count < first) return ((uint32_t)len << 9) | c.sym[index + (code - first)];
    index += count;
    first = (first + count) << 1;
    code <<= 1;
  }
  return 0;
}

// the walk's state after lengths 1..rootbits (it depends on the counts alone); lane 0
__host__ __device__ __forceinline__ void root_state(Code &c, int rootbits) {
  int first = 0, index = 0;
  for (int len = 1; len <= rootbits; ++len) {
    index += c.count[len];
    first = (first + c.count[len]) << 1;
  }
  c.rfirst = (uint16_t)first;
  c.rindex = (uint16_t)index;
}

// a code longer than rootbits (root entry 0): the walk resumes after rootbits with the bit-reversed root bits as its code
__host__ __device__ __forceinline__ uint32_t decode_long(const Code &c, uint32_t v, int rootbits) {
  uint32_t r = 0;
  for (int k = 0; k < rootbits; ++k) r |= ((v >> k) & 1u) << (rootbits - 1 - k);
  return decode_slow(c, v, kMaxBits, rootbits, (int)(r << 1), c.rfirst, c.rindex);
}

// root table of `code`: every lane fills a stride of the 2^root entries
__host__ __device__ __forceinline__ void fill_root(uint16_t *root, const Code &c, int rootbits, int lane, int nl) {
  for (int i = lane; i < (1 << rootbits); i += nl) root[i] = (uint16_t)decode_slow(c, (uint32_t)i, rootbits);
}

// one symbol through root + code (the reader holds >= 15 bits); -1 when no code matches
__host__ __device__ __forceinline__ int decode_sym(Bits &br, const uint16_t *root, int rootbits, const Code &c) {
  uint32_t e = root[br.peek(rootbits)];
  if (e == 0) {
    e = decode_long(c, br.peek(kMaxBits), rootbits);
    if (e == 0) return -1;
  }
  br.drop((int)(e >> 9));
  return (int)(e & 511u);
}

// lit / dist codes from w.lens (nlen + ndist lengths), then both root tables; false when either code is refused
__host__ __device__ __forceinline__ bool build_tables(Work &w, int nlen, int ndist, int lane, int nl) {
  int ok = 1;
  if (lane == 0) {
    ok = build_code(w.lit, w.lens, nlen, false) && build_code(w.dist, w.lens + nlen, ndist, false);
    root_state(w.lit, kLitRoot);
    root_state(w.dist, kDistRoot);
  }
  ok = ZLIBD_BCAST(ok);
  ZLIBD_SYNC();
  if (!ok) return false;
  fill_root(w.lroot, w.lit, kLitRoot, lane, nl);
  fill_root(w.droot, w.dist, kDistRoot, lane, nl);
  ZLIBD_SYNC();
  return true;
}

// dynamic block header (RFC 1951 3.2.7) -> w.lit / w.dist; false on any refusal
__host__ __device__ __forceinline__ bool dynamic_header(Bits &br, Work &w, int lane, int nl) {
  br.refill();
  const int nlen = (int)br.take(5) + 257, ndist = (int)br.take(5) + 1, ncode = (int)br.take(4) + 4;
  if (nlen > 286 || ndist > 30) return false;
  const char *order = "\x10\x11\x12\x00\x08\x07\x09\x06\x0a\x05\x0b\x04\x0c\x03\x0d\x02\x0e\x01\x0f";
  br.refill();
  if (lane == 0)   // the code-length code's lengths go to w.lens[0, 19) until w.cl is built from them
    for (int k = 0; k < 19; ++k) w.lens[k] = 0;
  ZLIBD_SYNC();
  for (int k = 0; k < ncode; ++k) {
    const uint8_t v = (uint8_t)br.take(3);
    if (lane == 0) w.lens[(int)order[k]] = v;
  }
  ZLIBD_SYNC();
  int ok = 1;
  if (lane == 0) {
    ok = build_code(w.cl, w.lens, 19, true);
    w.fixed = 0;   // w.lens and the tables are overwritten below
  }
  ok = ZLIBD_BCAST(ok);
  ZLIBD_SYNC();
  if (!ok) return false;
  int have = 0;
  while (have < nlen + ndist) {
    br.refill();
    const uint32_t e = decode_slow(w.cl, br.peek(7), 7);
    if (e == 0) return false;   // unreachable for a complete code; kept for safety
    br.drop((int)(e >> 9));
    const int sym = (int)(e & 511u);
    int len = 0, rep;
    if (sym < 16) {
      len = sym;
      rep = 1;
    } else if (sym == 16) {
      if (have == 0) return false;
      len = w.lens[have - 1];
      rep = 3 + (int)br.take(2);
    } else {
      rep = sym == 17 ? 3 + (int)br.take(3) : 11 + (int)br.take(7);
    }
    if (have + rep > nlen + ndist) return false;
    ZLIBD_SYNC();   // every lane has read lens[have - 1] before lane 0 writes
    if (lane == 0)
      for (int k = 0; k < rep; ++k) w.lens[have + k] = (uint8_t)len;
    ZLIBD_SYNC();
    have += rep;
  }
  if (w.lens[256] == 0) return false;
  ZLIBD_SYNC();
  return build_tables(w, nlen, ndist, lane, nl);
}

__host__ __device__ __forceinline__ bool fixed_tables(Work &w, int lane, int nl) {
  const int32_t have = w.fixed;
  ZLIBD_SYNC();   // every lane has read the flag before lane 0 sets it
  if (have) return true;
  if (lane == 0) {
    for (int s = 0; s < 288 + 32; ++s) w.lens[s] = (uint8_t)(s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5);
    w.fixed = 1;
  }
  ZLIBD_SYNC();
  return build_tables(w, 288, 32, lane, nl);
}

// match at distance d (1 <= d <= bytes before dst): every source byte precedes dst, dst[i] = dst[i - d + (i mod d)]
__host__ __device__ __forceinline__ void copy_match(uint8_t *dst, uint32_t d, uint32_t n, int lane, int nl) {
  const uint8_t *src = dst - d;
  for (uint32_t i = (uint32_t)lane; i < n; i += (uint32_t)nl) dst[i] = src[i < d ? i : i % d];
  ZLIBD_SYNC();
}

// Adler-32 of p[0, n): lane-strided sums of x_i and (n - i) x_i, reduced over the warp
__host__ __device__ __forceinline__ uint32_t adler32(const uint8_t *p, uint32_t n, int lane, int nl) {
  uint64_t s = 0, t = 0;
  uint32_t wgt = ((uint32_t)lane < n ? n - (uint32_t)lane : 0u) % kAdlerMod;   // (n - i) mod 65521 for i = lane
  const uint32_t step = (uint32_t)nl % kAdlerMod;
  for (uint32_t i = (uint32_t)lane; i < n; i += (uint32_t)nl) {   // t grows by < 2^24 per byte: < 2^55 for n < 2^31
    const uint32_t x = p[i];
    s += x;
    t += (uint64_t)wgt * x;
    wgt = wgt >= step ? wgt - step : wgt + kAdlerMod - step;
  }
  s %= kAdlerMod;
  t %= kAdlerMod;
  s = ZLIBD_SUM(s);
  t = ZLIBD_SUM(t);
  const uint32_t a = (uint32_t)((1 + s) % kAdlerMod), b = (uint32_t)(((uint64_t)(n % kAdlerMod) + t) % kAdlerMod);
  return (b << 16) | a;
}

// one zlib stream in[0, n_in) -> out[0, n_out); kOk only when the stream is the whole input and decodes to exactly n_out bytes
// (both at most kMaxStream)
__host__ __device__ __forceinline__ int32_t decode_stream(const uint8_t *in, int64_t n_in, uint8_t *out, int64_t n_out, Work &w, int lane, int nl) {
  if (n_in < 2 || n_in > kMaxStream || n_out > kMaxStream) return kBad;
  const uint32_t cmf = in[0], flg = in[1];
  if ((cmf & 15) != 8 || (cmf >> 4) > 7 || (cmf * 256 + flg) % 31 != 0 || (flg & 0x20)) return kBad;
  if (lane == 0) w.fixed = 0;
  ZLIBD_SYNC();
  const uint32_t nin = (uint32_t)n_in, nout = (uint32_t)n_out;
  Bits br;
  br.in = in;
  br.n = nin;
  br.to_byte(2);
  uint32_t op = 0;     // bytes stored
  int pend = 0;        // pending literals (lane k holds the k-th)
  uint32_t mylit = 0;
  bool last = false;
  while (!last) {
    br.refill();
    last = br.take(1) != 0;
    const uint32_t type = br.take(2);
    if (type == 0) {   // stored: LEN, NLEN at the next byte boundary
      br.drop(br.nb & 7);
      const uint32_t at = br.next_byte();
      if (at + 4 > nin) return kBad;
      const uint32_t len = (uint32_t)in[at] | ((uint32_t)in[at + 1] << 8), nlen = (uint32_t)in[at + 2] | ((uint32_t)in[at + 3] << 8);
      if (len != (~nlen & 0xffffu) || at + 4 + len > nin || op + len > nout) return kBad;
      for (uint32_t i = (uint32_t)lane; i < len; i += (uint32_t)nl) out[op + i] = in[at + 4 + i];
      op += len;
      br.to_byte(at + 4 + len);
      ZLIBD_SYNC();
      continue;
    }
    if (type == 3) return kBad;
    if (type == 1 ? !fixed_tables(w, lane, nl) : !dynamic_header(br, w, lane, nl)) return kBad;
    for (;;) {
      br.refill();   // >= 57 bits: a length code and its extra bits, a distance code and its extra bits
      if (br.overrun()) return kBad;
      const int sym = decode_sym(br, w.lroot, kLitRoot, w.lit);
      if (sym < 0 || sym > 285) return kBad;
      if (sym < 256) {
        if (op + (uint32_t)pend >= nout) return kBad;
        if (lane == pend) mylit = (uint32_t)sym;
        if (++pend < nl) continue;
      }
      if (pend) {   // store the pending run
        if (lane < pend) out[op + lane] = (uint8_t)mylit;
        op += (uint32_t)pend;
        pend = 0;
        ZLIBD_SYNC();
      }
      if (sym < 256) continue;
      if (sym == 256) break;
      const int c = sym - 257;
      uint32_t len;
      if (c < 8) {
        len = 3u + (uint32_t)c;
      } else if (c == 28) {
        len = 258;
      } else {
        const int e = (c >> 2) - 1;
        len = ((4u + (uint32_t)(c & 3)) << e) + 3u + br.take(e);
      }
      const int ds = decode_sym(br, w.droot, kDistRoot, w.dist);
      if (ds < 0 || ds > 29) return kBad;
      uint32_t dist;
      if (ds < 4) {
        dist = 1u + (uint32_t)ds;
      } else {
        const int e = (ds >> 1) - 1;
        dist = ((2u + (uint32_t)(ds & 1)) << e) + 1u + br.take(e);
      }
      if (dist > op || op + len > nout) return kBad;
      copy_match(out + op, dist, len, lane, nl);
      op += len;
    }
  }
  // the Adler-32 (big-endian) at the next byte boundary ends the input
  if (br.overrun()) return kBad;
  br.drop(br.nb & 7);
  const uint32_t at = br.next_byte();
  if (at + 4 != nin || op != nout) return kBad;
  ZLIBD_SYNC();
  const uint32_t want = ((uint32_t)in[at] << 24) | ((uint32_t)in[at + 1] << 16) | ((uint32_t)in[at + 2] << 8) | in[at + 3];
  return adler32(out, nout, lane, nl) == want ? kOk : kBad;
}

}  // namespace zlibd
