// Integer stream ENCODERS of CS_ENCODING_ROW_STORE blocks on the device: stream_codecs_host.h (the reference's codec library as
// ObIntegerStreamEncoder instantiates it, scalar packing, LSB-first bit streams) and its codec choice, restated CTA-parallel for
// one stream of a block in shared memory. Every function is called by every thread of the CTA with the same arguments; writes
// OR the codec's bits into the zeroed block image (or_bits / put_bytes), a null image only sizes the stream.
//
//   PFOR family (SIMD_FIXEDPFOR, DELTA_ZIGZAG_PFOR, DOUBLE_DELTA_ZIGZAG_PFOR, XOR_FIXED_PFOR): chunks of 128 values, one warp per
//     chunk. A chunk's transformed values need only the stream values i - 1 and i - 2, read by index, so chunks are independent:
//     the warp builds the bit-width histogram, runs find_most_fit_bx, sets the exception bitmap from ballots and numbers the
//     exceptions by prefix popcount; a CTA scan over the chunk sizes places each chunk. A tail chunk below 128 values is simple
//     bit packing with its own width byte; XOR puts its shift byte before every chunk.
//   RLE family (DELTA_ZIGZAG_RLE, DOUBLE_DELTA_ZIGZAG_RLE): every non-zero delta emits the code of the run of zero deltas before
//     it, then its own delta code; a trailing run emits its run code only. Each thread takes a contiguous slice of the stream:
//     an exclusive max-scan over the slices' last non-zero deltas gives the run entering each slice, an exclusive sum-scan over
//     the slices' bit counts places each slice's codes.
#pragma once

namespace enc {

enum : uint32_t { ST_RAW = 1, ST_DD_RLE = 2, ST_DD_PFOR = 3, ST_D_RLE = 4, ST_D_PFOR = 5, ST_FIXEDPFOR = 6, ST_XOR_PFOR = 8 };
constexpr uint32_t kCrefMax = 2u + 2u * 64u;   // values of a const-form ref stream: exceptions, constant, 64 rows, 64 refs
constexpr uint32_t kHistBins = 65u;            // bit widths 0..64

// The codec and the encoded bytes of a CS column's streams: [0] the CS_INTEGER value stream or the dictionary stream, [1] the ref
// stream. Written by the sizing phase, read by the plan and the pack.
struct CsCodec {
  uint32_t bytes[2];
  uint8_t type[2], pad[2];
};

struct StreamScratch {
  CsCodec *cod;     // [n_cols]
  uint32_t *hist;   // [kWarps][kHistBins] bit-width histogram of a PFOR chunk
  uint32_t *csz;    // [chunks of a block's longest stream] chunk sizes, then their inclusive scan
  uint32_t *cref;   // [kCrefMax] the const-form ref stream
  uint32_t *red;    // [kWarps]
};

// Stream values by index (already minus the stream base; the codecs mask them to the stream width).
struct IntVals {   // a CS_INTEGER column: the NULL replacement in NULL rows
  const int64_t *vals;
  const uint8_t *nl;
  unsigned long long mask, base, nv;
  __device__ __forceinline__ unsigned long long operator()(uint32_t i) const {
    return nl && nl[i] ? nv : ((unsigned long long)vals[i] & mask) - base;
  }
};
struct DictVals {   // the sorted dictionary of a CS_INT_DICT column (sort keys back to datums)
  const unsigned long long *sk;
  const uint32_t *hp;
  unsigned long long flip, base;
  __device__ __forceinline__ unsigned long long operator()(uint32_t i) const { return (sk[hp[i]] ^ flip) - base; }
};
struct RefVals {   // a ref stream
  const uint32_t *a;
  __device__ __forceinline__ unsigned long long operator()(uint32_t i) const { return a[i]; }
};

__device__ __forceinline__ uint32_t st_bits(unsigned long long v) { return v == 0 ? 0u : 64u - (uint32_t)__clzll((long long)v); }
__device__ __forceinline__ unsigned long long st_mask(uint32_t wb) { return wb >= 8u ? ~0ull : (1ull << (8u * wb)) - 1ull; }
__device__ __forceinline__ uint32_t pad8(uint32_t bits) { return (bits + 7u) / 8u; }
__device__ __forceinline__ unsigned long long zigzag(unsigned long long d, uint32_t wb) {
  return ((d << 1) ^ (0ull - ((d >> (8u * wb - 1u)) & 1ull))) & st_mask(wb);
}

// Exclusive scan (sum, or max when MAX) of one value per thread over the CTA; *total: the whole CTA's result.
template <bool MAX>
__device__ uint32_t thr_scan(uint32_t x, uint32_t *red, uint32_t *total) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t incl = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= (uint32_t)o) incl = MAX ? max(incl, u) : incl + u;
  }
  uint32_t excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0u) excl = 0u;
  if (lane == 31u) red[warp] = incl;
  __syncthreads();
  uint32_t before = 0, all = 0;
  for (uint32_t w = 0; w < (uint32_t)kWarps; ++w) {
    if (w == warp) before = all;
    all = MAX ? max(all, red[w]) : all + red[w];
  }
  __syncthreads();
  *total = all;
  return MAX ? max(before, excl) : before + excl;
}

// ---- PFOR family: kind 0 plain, 1 delta zigzag, 2 double delta zigzag, 3 xor --------------------------------------------------
template <class V>
__device__ __forceinline__ unsigned long long pfor_value(int kind, const V &v, uint32_t i, uint32_t wb) {
  const unsigned long long m = st_mask(wb), u = v(i) & m;
  if (kind == 0) return u;
  const unsigned long long u1 = i ? v(i - 1u) & m : 0ull;
  if (kind == 3) return u ^ u1;
  if (kind == 1) return zigzag((u - u1) & m, wb);
  const unsigned long long u2 = i > 1u ? v(i - 2u) & m : 0ull;
  return zigzag((u - u1 - (u1 - u2)) & m, wb);
}

__device__ __forceinline__ unsigned long long warp_or(unsigned long long x) {
  return ((unsigned long long)__reduce_or_sync(0xffffffffu, (uint32_t)(x >> 32)) << 32) | __reduce_or_sync(0xffffffffu, (uint32_t)x);
}

// One chunk of 128 (or, at the stream's end, fewer) values: its bytes; written at byte `at` when img32 is set. One whole warp.
template <class V>
__device__ uint32_t pfor_chunk(int kind, const V &v, uint32_t j, uint32_t count, uint32_t wb, uint32_t *hist, uint32_t *img32,
                               uint32_t at) {
  const uint32_t lane = threadIdx.x & 31u, i0 = j * 128u, n = min(128u, count - i0);
  unsigned long long t[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t i = lane + 32u * k;
    t[k] = i < n ? pfor_value(kind, v, i0 + i, wb) : 0ull;
  }
  uint32_t head = 0;
  if (kind == 3) {   // shift out the leading zeros the whole chunk shares, then bit-reverse within the width
    const uint32_t sh = 8u * wb - st_bits(warp_or(t[0] | t[1] | t[2] | t[3]));
#pragma unroll
    for (int k = 0; k < 4; ++k) t[k] = sh >= 64u ? 0ull : __brevll((t[k] << sh) & st_mask(wb)) >> (64u - 8u * wb);
    if (img32 && lane == 0) put_bytes(img32, at, 1u, sh);
    head = 1;
  }
  const uint32_t b0 = st_bits(warp_or(t[0] | t[1] | t[2] | t[3]));
  const uint32_t o = at + head;
  if (n < 128u) {   // ObSimpleBitPacking: width byte, n values of b0 bits
    if (img32) {
      if (lane == 0) put_bytes(img32, o, 1u, b0);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t i = lane + 32u * k;
        if (i < n) or_bits(img32, (o + 1u) * 8u + i * b0, b0, t[k]);
      }
    }
    return head + 1u + pad8(n * b0);
  }
  // enc_pfor_block: find_most_fit_bx over the bit-width histogram
  for (uint32_t k = lane; k < kHistBins; k += 32u) hist[k] = 0u;
  __syncwarp();
#pragma unroll
  for (int k = 0; k < 4; ++k) atomicAdd(&hist[st_bits(t[k])], 1u);
  __syncwarp();
  uint32_t b = b0, ml = 16u * b0 + 1u;
  if (lane == 0) {
    uint32_t x = hist[b0];
    for (int i = (int)b0 - 1; i >= 0; --i) {
      const uint32_t l = 18u + pad8(x * (b0 - (uint32_t)i)) + 16u * (uint32_t)i;
      x += hist[i];
      if (l < ml) { ml = l; b = (uint32_t)i; }
    }
  }
  b = __shfl_sync(0xffffffffu, b, 0);
  ml = __shfl_sync(0xffffffffu, ml, 0);
  __syncwarp();   // the histogram is free again
  if (img32) {
    const uint32_t bx = b0 - b;
    if (bx == 0) {
      if (lane == 0) put_bytes(img32, o, 1u, b);
#pragma unroll
      for (int k = 0; k < 4; ++k) or_bits(img32, (o + 1u) * 8u + (lane + 32u * k) * b, b, t[k]);
    } else {   // [0x80 | b][bx][exception bitmap, 16 bytes][exceptions' high parts, bx bits each][every low part, b bits each]
      if (lane == 0) put_bytes(img32, o, 2u, 0x80u | b | (bx << 8));
      const unsigned long long msk = (1ull << b) - 1ull;
      uint32_t xb = 0, xn = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t e = __ballot_sync(0xffffffffu, t[k] > msk);
        if (t[k] > msk) xb |= (xn + __popc(e & ((1u << lane) - 1u))) << (8 * k);   // exception numbers fit a byte
        xn += __popc(e);
      }
      const uint32_t lo_at = (o + 18u + pad8(xn * bx)) * 8u;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t i = lane + 32u * k;
        if (t[k] > msk) {
          or_bits(img32, (o + 2u) * 8u + i, 1u, 1ull);
          or_bits(img32, (o + 18u) * 8u + ((xb >> (8 * k)) & 0xffu) * bx, bx, t[k] >> b);
        }
        or_bits(img32, lo_at + i * b, b, t[k] & msk);
      }
    }
  }
  return head + ml;
}

template <class V>
__device__ uint32_t pfor_stream(int kind, const V &v, uint32_t count, uint32_t wb, const StreamScratch &s, uint32_t *img32, uint32_t at) {
  const uint32_t warp = threadIdx.x >> 5, nch = (count + 127u) / 128u;
  for (uint32_t j = warp; j < nch; j += kWarps) {
    const uint32_t sz = pfor_chunk(kind, v, j, count, wb, s.hist + warp * kHistBins, nullptr, 0u);
    if ((threadIdx.x & 31u) == 0) s.csz[j] = sz;
  }
  __syncthreads();
  blk_scan(s.csz, nch, s.red);
  const uint32_t total = s.csz[nch - 1u];
  if (img32)
    for (uint32_t j = warp; j < nch; j += kWarps) pfor_chunk(kind, v, j, count, wb, s.hist + warp * kHistBins, img32, at + (j ? s.csz[j - 1u] : 0u));
  __syncthreads();
  return total;
}

// ---- RLE family ----------------------------------------------------------------------------------------------------------------
struct RleWidths {   // encode_delta_and_repeat_cnt's tiers for the stream width
  uint32_t n2, n3, n4;
  __device__ __forceinline__ explicit RleWidths(uint32_t wb)
      : n2(wb == 1u ? 3u : 6u), n3(wb == 1u ? 5u : wb == 4u ? 10u : 12u), n4(wb == 1u ? 9u : wb == 8u ? 20u : 17u) {}
};
__device__ __forceinline__ uint32_t rle_run_bits(uint32_t r) { return r <= 18u ? r : 10u + 8u * ((st_bits(r - 18u) + 7u) >> 3); }
__device__ __forceinline__ uint32_t rle_delta_bits(unsigned long long zz, const RleWidths &w) {
  if (zz < (1ull << (w.n2 - 1u))) return w.n2 + 2u;
  if (zz < (1ull << (w.n3 - 1u))) return w.n3 + 3u;
  if (zz < (1ull << (w.n4 - 1u))) return w.n4 + 4u;
  return 7u + 8u * ((st_bits(zz) + 7u) >> 3);
}
// ObBitUtils::put<uint64_t> of a value above 45 bits: the high part first, then the low 32 bits
__device__ __forceinline__ void rle_put_wide(uint32_t *img32, uint32_t &pos, unsigned long long x, uint32_t width, bool split) {
  if (split && width > 45u) {
    or_bits(img32, pos, width - 32u, x >> 32);
    or_bits(img32, pos + width - 32u, 32u, x & 0xffffffffull);
  } else {
    or_bits(img32, pos, width, x);
  }
  pos += width;
}
__device__ __forceinline__ void rle_put_run(uint32_t *img32, uint32_t &pos, uint32_t r) {
  if (r > 18u) {
    r -= 18u;
    const uint32_t b = (st_bits(r) + 7u) >> 3;
    or_bits(img32, pos, 10u, (unsigned long long)(b - 1u) << 7);
    pos += 10u;
    rle_put_wide(img32, pos, r, 8u * b, true);
  } else {
    or_bits(img32, pos, r, (1ull << r) - 1ull);   // r one-bits
    pos += r;
  }
}
__device__ __forceinline__ void rle_put_delta(uint32_t *img32, uint32_t &pos, unsigned long long zz, const RleWidths &w, uint32_t wb) {
  if (zz < (1ull << (w.n2 - 1u))) { or_bits(img32, pos, w.n2 + 2u, (zz << 2) | 2u); pos += w.n2 + 2u; }
  else if (zz < (1ull << (w.n3 - 1u))) { or_bits(img32, pos, w.n3 + 3u, (zz << 3) | 4u); pos += w.n3 + 3u; }
  else if (zz < (1ull << (w.n4 - 1u))) { or_bits(img32, pos, w.n4 + 4u, (zz << 4) | 8u); pos += w.n4 + 4u; }
  else {
    const uint32_t b = (st_bits(zz) + 7u) >> 3;
    or_bits(img32, pos, 7u, (unsigned long long)(b - 1u) << 4);
    pos += 7u;
    rle_put_wide(img32, pos, zz, 8u * b, wb == 8u);
  }
}

template <class V>
__device__ uint32_t rle_stream(bool dbl, const V &v, uint32_t count, uint32_t wb, const StreamScratch &s, uint32_t *img32, uint32_t at) {
  const uint32_t per = (count + kThreads - 1u) / kThreads, lo = min((uint32_t)threadIdx.x * per, count), hi = min(lo + per, count);
  const unsigned long long m = st_mask(wb);
  const RleWidths w(wb);
  const unsigned long long p1 = lo ? v(lo - 1u) & m : 0ull, p2 = lo > 1u ? v(lo - 2u) & m : 0ull;
  // 1 + the index of the slice's last non-zero delta (0: none), then the same for everything before the slice
  uint32_t last = 0, total = 0;
  {
    unsigned long long u1 = p1, u2 = p2;
    for (uint32_t i = lo; i < hi; ++i) {
      const unsigned long long u = v(i) & m, d = (dbl ? u - u1 - (u1 - u2) : u - u1) & m;
      if (d) last = i + 1u;
      u2 = u1;
      u1 = u;
    }
  }
  const uint32_t enter = thr_scan<true>(last, s.red, &total);
  const bool tail = lo < hi && hi == count;   // the slice that holds the trailing run
  uint32_t bits = 0;   // of the slice's codes
  {
    uint32_t L = enter;
    unsigned long long u1 = p1, u2 = p2;
    for (uint32_t i = lo; i < hi; ++i) {
      const unsigned long long u = v(i) & m, d = (dbl ? u - u1 - (u1 - u2) : u - u1) & m;
      if (d) { bits += rle_run_bits(i - L) + rle_delta_bits(zigzag(d, wb), w); L = i + 1u; }
      u2 = u1;
      u1 = u;
    }
    if (tail && L < count) bits += rle_run_bits(count - L);
  }
  const uint32_t before = thr_scan<false>(bits, s.red, &total);
  if (img32) {
    uint32_t pos = at * 8u + before, L = enter;
    unsigned long long u1 = p1, u2 = p2;
    for (uint32_t i = lo; i < hi; ++i) {
      const unsigned long long u = v(i) & m, d = (dbl ? u - u1 - (u1 - u2) : u - u1) & m;
      if (d) { rle_put_run(img32, pos, i - L); rle_put_delta(img32, pos, zigzag(d, wb), w, wb); L = i + 1u; }
      u2 = u1;
      u1 = u;
    }
    if (tail && L < count) rle_put_run(img32, pos, count - L);
  }
  return pad8(total);
}

// The stream's bytes with codec `type` (RAW: count * wb, nothing written); its codes ORed in at byte `at` when img32 is set.
template <class V>
__device__ uint32_t codec_stream(uint32_t type, const V &v, uint32_t count, uint32_t wb, const StreamScratch &s, uint32_t *img32,
                                 uint32_t at) {
  switch (type) {
    case ST_DD_RLE: return rle_stream(true, v, count, wb, s, img32, at);
    case ST_D_RLE: return rle_stream(false, v, count, wb, s, img32, at);
    case ST_DD_PFOR: return pfor_stream(2, v, count, wb, s, img32, at);
    case ST_D_PFOR: return pfor_stream(1, v, count, wb, s, img32, at);
    case ST_FIXEDPFOR: return pfor_stream(0, v, count, wb, s, img32, at);
    case ST_XOR_PFOR: return pfor_stream(3, v, count, wb, s, img32, at);
    default: return count * wb;
  }
}

// emit_int_stream's codec for a stream under stream mode `mode` (ObIntegerStreamEncoder::choose_stream_codec / inner_encode):
//   0     detect: RAW below 4 values; every candidate encodes a prefix sample (the whole stream below 1 024 values, else
//         max(25 %, 1 024) values) in the order FIXEDPFOR, DD_RLE, DD_PFOR, D_RLE, D_PFOR, XOR (XOR skipped when the whole stream
//         does not decrease); a later candidate wins only when strictly smaller, the winner only when strictly below the RAW sample
//   2..8  that codec
// then RAW wherever the codec's full stream is larger than RAW. Returns the codec; *bytes: the stream's bytes.
template <class V>
__device__ uint32_t choose_codec(int mode, const V &v, uint32_t count, uint32_t wb, const StreamScratch &s, uint32_t *bytes) {
  uint32_t type = ST_RAW;
  if (mode == 0 && count >= 4u) {
    const uint32_t sample = count < 1024u ? count : max(count * 25u / 100u, 1024u);
    const unsigned long long m = st_mask(wb);
    uint32_t dec = 0;
    for (uint32_t i = threadIdx.x + 1u; i < count; i += kThreads) dec |= (v(i) & m) < (v(i - 1u) & m) ? 1u : 0u;
    dec = blk_max(dec, s.red);
    uint32_t best = 0xffffffffu, pick = ST_RAW;
    for (uint32_t k = 0; k < 6u; ++k) {
      const uint32_t t = (0x854326u >> (4u * k)) & 0xfu;   // FIXEDPFOR, DD_RLE, DD_PFOR, D_RLE, D_PFOR, XOR
      if (t == ST_XOR_PFOR && !dec) continue;
      const uint32_t sz = codec_stream(t, v, sample, wb, s, nullptr, 0u);
      if (sz < best) { best = sz; pick = t; }
    }
    if (best < sample * wb) type = pick;
  } else if (mode >= 2) {
    type = (uint32_t)mode;
  }
  *bytes = count * wb;
  if (type != ST_RAW) {
    const uint32_t sz = codec_stream(type, v, count, wb, s, nullptr, 0u);
    if (sz > count * wb) type = ST_RAW;
    else *bytes = sz;
  }
  return type;
}

}  // namespace enc
