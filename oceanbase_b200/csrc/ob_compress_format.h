// The bytes of the micro-block payload compressors, shared by the host writer (sstable_writer.cpp: ObLZ4Compressor /
// ObZstdCompressor_1_3_8 output) and the device compressor (stored_compress.cuh), so that the two agree byte for byte:
//   - the greedy matcher's constants: 4-byte hash -> last position in a table of 64 Ki entries, offsets <= 65535, no probe
//     after n - 12, a match ends at n - 5 at the latest (lz4_Block_format.md end-of-block rules);
//   - zstd (RFC 8878): the frame / block / literals / sequences headers, the Literals_Length and Match_Length code tables,
//     the predefined normalised distributions, the FSE encoding-table build (FSE_buildCTable) and the sequence bitstream in
//     ZSTD_encodeSequences order.
// Byte sinks (`put(uint8_t)`) are the caller's: the writer appends to a vector, the device writes to a bounded buffer.
#pragma once
#include <stdint.h>

#include "ob_format.h"   // OBF_HD

#if defined(__CUDACC__)   // the tables live in device memory: what reads them is device code under nvcc
#define OBZ_TABLE __device__ constexpr
#define OBZ_HD __device__ __forceinline__
#else
#define OBZ_TABLE constexpr
#define OBZ_HD inline
#endif

namespace obz {

// ---- greedy matcher -------------------------------------------------------------------------------------------------------
constexpr uint32_t kHashMul = 2654435761u;
constexpr int kHashLog = 16;
constexpr uint32_t kHashEntries = 1u << kHashLog;
constexpr int64_t kMaxOffset = 65535, kMfLimit = 12, kLastLiterals = 5;
constexpr int64_t kZstdBlock = 128 * 1024;   // zstd matches every 128 KiB chunk on its own, with a fresh table

OBF_HD uint32_t hash4(uint32_t seq) { return (seq * kHashMul) >> (32 - kHashLog); }

OBF_HD int high_bit(uint32_t v) {   // v > 0
#if defined(__CUDA_ARCH__)
  return 31 - __clz(v);
#else
  return 31 - __builtin_clz(v);
#endif
}

// ---- zstd: Literals_Length / Match_Length codes (RFC 8878 3.1.1.3.2.1.1) ----------------------------------------------------
OBZ_TABLE uint32_t kLLBase[36] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64,
                                  128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536};
OBZ_TABLE uint32_t kMLBase[53] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28,
                                  29, 30, 31, 32, 33, 34, 35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051,
                                  4099, 8195, 16387, 32771, 65539};
OBZ_TABLE uint8_t kLLBits[36] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12,
                                 13, 14, 15, 16};
// predefined distributions (RFC 8878 3.1.1.3.2.2): accuracy logs 6 / 5 / 6
OBZ_TABLE int16_t kLLNorm[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
OBZ_TABLE int16_t kOFNorm[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
OBZ_TABLE int16_t kMLNorm[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                                 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};

OBZ_HD int ll_code(uint32_t v) {   // largest code whose baseline is <= v
  int c = 35;
  while (kLLBase[c] > v) --c;
  return c;
}
OBZ_HD int ml_code(uint32_t v) {   // v = match length (>= 3)
  int c = 52;
  while (kMLBase[c] > v) --c;
  return c;
}
OBZ_HD int ml_bits(int c) { return c < 32 ? 0 : c < 36 ? 1 : c < 38 ? 2 : c < 40 ? 3 : c < 42 ? 4 : c == 42 ? 5 : c - 36; }

// ---- FSE encoding table of one predefined distribution (FSE_buildCTable) ------------------------------------------------------
struct FseCTable {
  int32_t log;
  uint16_t state[64];
  int32_t dnb[53], dfs[53];   // per symbol: deltaNbBits, deltaFindState
};
OBZ_HD void fse_build(const int16_t *norm, int nsym, int lg, FseCTable &t) {
  const int size = 1 << lg, mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
  int sym[64], cumul[54];
  int high = size - 1;
  t.log = lg;
  cumul[0] = 0;
  for (int s = 0; s < nsym; ++s) {
    if (norm[s] == -1) {
      cumul[s + 1] = cumul[s] + 1;
      sym[high--] = s;
    } else {
      cumul[s + 1] = cumul[s] + norm[s];
    }
  }
  int pos = 0;
  for (int s = 0; s < nsym; ++s)
    for (int i = 0; i < norm[s]; ++i) {
      sym[pos] = s;
      do pos = (pos + step) & mask; while (pos > high);
    }
  for (int u = 0; u < size; ++u) t.state[cumul[sym[u]]++] = (uint16_t)(size + u);
  int total = 0;
  for (int s = 0; s < nsym; ++s) {
    const int c = norm[s];
    if (c == -1 || c == 1) {
      t.dnb[s] = (lg << 16) - size;
      t.dfs[s] = total - 1;
      ++total;
    } else if (c > 1) {
      const int max_bits_out = lg - high_bit((uint32_t)(c - 1));
      t.dnb[s] = (max_bits_out << 16) - (c << max_bits_out);
      t.dfs[s] = total - c;
      total += c;
    } else {
      t.dnb[s] = t.dfs[s] = 0;
    }
  }
}
struct FseSet { FseCTable ll, of, ml; };
OBZ_HD void fse_build_predefined(FseSet &f) {
  fse_build(kLLNorm, 36, 6, f.ll);
  fse_build(kOFNorm, 29, 5, f.of);
  fse_build(kMLNorm, 53, 6, f.ml);
}

// forward little-endian bit accumulator over a byte sink (the decoder reads the stream backward)
template <class Sink>
struct BitWriter {
  Sink &o;
  uint64_t acc = 0;
  int nb = 0;
  OBZ_HD explicit BitWriter(Sink &out) : o(out) {}
  OBZ_HD void add(uint64_t v, int k) {
    acc |= (v & ((1ull << k) - 1)) << nb;
    nb += k;
    for (; nb >= 8; nb -= 8, acc >>= 8) o.put((uint8_t)acc);
  }
  OBZ_HD void close() {   // the end mark: one 1 bit, then padding to the byte
    add(1, 1);
    if (nb) o.put((uint8_t)acc);
  }
};

struct Seq { uint32_t ll, off, ml; };   // literals before the match, match offset, match length

// Frame_Header: magic, Single_Segment descriptor, Frame_Content_Size in 1 / 2 / 4 / 8 bytes
template <class Sink>
OBZ_HD void zstd_frame_header(Sink &o, int64_t n) {
  o.put(0x28); o.put(0xb5); o.put(0x2f); o.put(0xfd);
  const int fcs_bytes = n < 256 ? 1 : n < 65536 + 256 ? 2 : n <= 0xffffffffll ? 4 : 8;
  o.put((uint8_t)(((fcs_bytes == 1 ? 0 : fcs_bytes == 2 ? 1 : fcs_bytes == 4 ? 2 : 3) << 6) | 0x20));
  const uint64_t fcs = (uint64_t)n - (fcs_bytes == 2 ? 256 : 0);
  for (int k = 0; k < fcs_bytes; ++k) o.put((uint8_t)(fcs >> (8 * k)));
}
template <class Sink>
OBZ_HD void zstd_block_header(Sink &o, bool last, bool raw, uint32_t size) {
  const uint32_t bh = (last ? 1u : 0u) | ((raw ? 0u : 2u) << 1) | (size << 3);
  o.put((uint8_t)bh); o.put((uint8_t)(bh >> 8)); o.put((uint8_t)(bh >> 16));
}
OBZ_HD int zstd_literals_header_size(uint32_t nl) { return nl < 32 ? 1 : nl < 4096 ? 2 : 3; }
template <class Sink>
OBZ_HD void zstd_literals_header(Sink &o, uint32_t nl) {   // Raw_Literals_Block
  if (nl < 32) {
    o.put((uint8_t)(nl << 3));
  } else if (nl < 4096) {
    o.put((uint8_t)((1u << 2) | ((nl & 15) << 4)));
    o.put((uint8_t)(nl >> 4));
  } else {
    o.put((uint8_t)((3u << 2) | ((nl & 15) << 4)));
    o.put((uint8_t)(nl >> 4));
    o.put((uint8_t)(nl >> 12));
  }
}
// Sequences_Section_Header (Number_of_Sequences, then Symbol_Compression_Modes = Predefined x 3) and the FSE bitstream
template <class Sink>
OBZ_HD void zstd_sequences(Sink &o, const Seq *seqs, uint32_t ns, const FseSet &f) {
  if (ns < 128) {
    o.put((uint8_t)ns);
  } else if (ns < 0x7f00) {
    o.put((uint8_t)((ns >> 8) + 128));
    o.put((uint8_t)ns);
  } else {
    o.put(255);
    o.put((uint8_t)(ns - 0x7f00));
    o.put((uint8_t)((ns - 0x7f00) >> 8));
  }
  if (ns == 0) return;
  o.put(0);
  BitWriter<Sink> bw(o);
  auto init = [](const FseCTable &t, int s) {
    const uint32_t nbo = (uint32_t)((t.dnb[s] + (1 << 15)) >> 16);
    const uint32_t v = (nbo << 16) - (uint32_t)t.dnb[s];
    return (uint32_t)t.state[(v >> nbo) + (uint32_t)t.dfs[s]];
  };
  auto encode = [&bw](const FseCTable &t, uint32_t &st, int s) {
    const uint32_t nbo = (st + (uint32_t)t.dnb[s]) >> 16;
    bw.add(st, (int)nbo);
    st = t.state[(st >> nbo) + (uint32_t)t.dfs[s]];
  };
  struct Codes { int ll, ml, of; };
  auto codes = [](const Seq &q) { return Codes{ll_code(q.ll), ml_code(q.ml), high_bit(q.off + 3)}; };   // Offset_Value = offset + 3
  auto extras = [&bw](const Seq &q, const Codes &c) {   // the baselines' low bits are zero: the extra bits are the value's low bits
    bw.add(q.ll, kLLBits[c.ll]);
    bw.add(q.ml - 3, ml_bits(c.ml));
    bw.add(q.off + 3, c.of);
  };
  Seq q = seqs[ns - 1];
  Codes c = codes(q);
  uint32_t sml = init(f.ml, c.ml), sof = init(f.of, c.of), sll = init(f.ll, c.ll);
  extras(q, c);
  for (uint32_t k = ns - 1; k-- > 0;) {
    q = seqs[k];
    c = codes(q);
    encode(f.of, sof, c.of);
    encode(f.ml, sml, c.ml);
    encode(f.ll, sll, c.ll);
    extras(q, c);
  }
  bw.add(sml, f.ml.log);
  bw.add(sof, f.of.log);
  bw.add(sll, f.ll.log);
  bw.close();
}

}  // namespace obz
