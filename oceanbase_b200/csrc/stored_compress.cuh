// Plain micro-blocks -> stored form ON THE DEVICE (obgpu_compress_blocks): byte for byte what obgpu_writer_compress_blocks
// writes (ObMacroBlockWriter's per-micro-block compress in the reference). Formats and constants are ob_compress_format.h's,
// shared with the writer. One call is a fixed sequence of launches whatever the block count:
//   survey  : one thread per block -- plain framing checks, aligned plain sizes, the capacity the call needs (one reduced value
//             and a verdict copied back; nothing is written to the output before they are known)
//   stage   : prefix over the plain sizes rounded to 16 -> a staging slot per block for the compressed payload
//   match   : ONE WARP per CTA (the 64 Ki-entry hash table and the FSE tables take 137.6 KiB of shared memory), blocks
//             taken from a counter. The warp runs greedy_matches 32 positions per step: lane k hashes ip + k, lanes sharing
//             a hash find each other with __match_any_sync (a lane's candidate is the highest lower lane with its hash,
//             else the table entry), the lowest lane with a valid candidate wins, positions up to the winner are inserted
//             (the highest lane per hash), and the match is extended 32 bytes per ballot -- the serial matcher's decisions
//             and table after every step.
//             LZ4 sequences are written as they are found; zstd literals are written as they are found and the sequences are
//             listed per 128 KiB chunk, then FSE-coded by lane 0. Writes stop at data_length_: a longer payload is stored raw.
//   layout  : prefix over the stored sizes rounded up to `align` -> output offsets (the writer's layout)
//   frame   : one CTA per block -- header, stored payload, data_zlength_, data_checksum_ (crc32c of the stored bytes) and
//             the header checksum; the padding up to the next aligned offset is zeroed
// The table: 64 Ki entries of 17 bits (uint16 + one bit in a bitmap), the position modulo 2^17. An entry more than 65535
// bytes back is stale; a sweep rewrites every stale entry to a value read as 65536..131071 bytes back before any probe can
// see it wrapped (every <= 64 KiB of input), so the device accepts payloads of any length a micro-block can hold.
#pragma once
#include "ob_compress_format.h"
#include "stored_blocks.cuh"

namespace sc {

constexpr uint32_t kBadArg = 1, kBadData = 2, kTooLarge = 4;   // survey verdict bits
constexpr int64_t kMaxStored = 0x7f000000;   // larger blocks are refused (OBGPU_NOT_SUPPORTED): aligned sizes stay in uint32
constexpr int kFrameThreads = 128;

struct Work {   // device-side totals of one call
  unsigned long long cap;      // sum of align_up(size, align)
  unsigned long long stage;    // sum of align_up(size, 16)
  unsigned long long end;      // end of the last stored block
  uint32_t verdict;
  int32_t next;                // block counter of the match kernel
};

__device__ __forceinline__ void plain_fields(const uint8_t *h, int64_t &hs, int64_t &len, int64_t &zlen) {
  hs = sb::ld32u(h + 4);
  len = (int32_t)sb::ld32u(h + 40);
  zlen = (int32_t)sb::ld32u(h + 44);
}

__global__ void __launch_bounds__(256) obgpu_compress_survey_kernel(const uint8_t *image, const int64_t *off, const uint32_t *size,
                                                                    int32_t n, int64_t align, uint32_t *stage_cnt, Work *w) {
  const int32_t i = (int32_t)(blockIdx.x * blockDim.x + threadIdx.x);
  unsigned long long cap = 0, stage = 0;
  uint32_t verdict = 0;
  if (i < n) {
    const int64_t sz = size[i];
    if (sz > 0) {
      const int64_t o = off[i];
      if (o < 0 || (o & 15) != 0) {
        verdict = kBadArg;
      } else if (sz > kMaxStored) {
        verdict = kTooLarge;
      } else {
        int64_t hs = 0, len = 0, zlen = 0;
        if (sz >= 64) plain_fields(image + o, hs, len, zlen);
        if (sz < 64 || hs < 64 || len < 0 || len != zlen || hs + len != sz) verdict = kBadData;   // plain, well-framed blocks only
      }
      cap = (unsigned long long)((sz + align - 1) & ~(align - 1));
      stage = (unsigned long long)((sz + 15) & ~15ll);
    }
    stage_cnt[i] = (uint32_t)stage;
  }
  for (int o = 16; o > 0; o >>= 1) {
    cap += __shfl_xor_sync(0xffffffffu, cap, o);
    stage += __shfl_xor_sync(0xffffffffu, stage, o);
    verdict |= __shfl_xor_sync(0xffffffffu, verdict, o);
  }
  if ((threadIdx.x & 31) == 0 && (cap | stage | verdict)) {
    atomicAdd(&w->cap, cap);
    atomicAdd(&w->stage, stage);
    if (verdict) atomicOr(&w->verdict, verdict);
  }
}

// ---- the warp matcher ----------------------------------------------------------------------------------------------------
struct MatchSmem {
  uint16_t lo[obz::kHashEntries];         // entry bits 0..15
  uint32_t hi[obz::kHashEntries / 32];    // entry bit 16
  obz::FseSet fse;
};

__device__ __forceinline__ void table_reset(MatchSmem &s, int lane) {   // every entry 65536: 65536 bytes back from position 0
  uint4 *lo = reinterpret_cast<uint4 *>(s.lo);
  for (int k = lane; k < (int)(obz::kHashEntries * 2 / 16); k += 32) lo[k] = make_uint4(0, 0, 0, 0);
  for (int k = lane; k < (int)(obz::kHashEntries / 32); k += 32) s.hi[k] = 0xffffffffu;
  __syncwarp();
}

// entries read at position R whose position is more than 65535 bytes before ip -> 65536 bytes before ip
__device__ void table_sweep(MatchSmem &s, int64_t R, int64_t ip, int lane) {
  const uint32_t dead = (uint32_t)(ip - 65536) & 0x1ffffu;
  const int64_t shift = ip - R;
  for (int w = lane; w < (int)(obz::kHashEntries / 32); w += 32) {
    uint32_t hi = s.hi[w];
    for (int j = 0; j < 32; ++j) {
      const uint32_t h = (uint32_t)w * 32 + j;
      const uint32_t v = s.lo[h] | (((hi >> j) & 1u) << 16);
      const int64_t d = (int64_t)(((uint32_t)R - v) & 0x1ffffu);
      if (d + shift > obz::kMaxOffset) {
        s.lo[h] = (uint16_t)dead;
        hi = (hi & ~(1u << j)) | (((dead >> 16) & 1u) << j);
      }
    }
    s.hi[w] = hi;
  }
  __syncwarp();
}

__device__ __forceinline__ uint32_t byte_at(const uint8_t *p) { return __ldg(p); }
__device__ __forceinline__ uint32_t rd32(const uint8_t *p) {
  return byte_at(p) | (byte_at(p + 1) << 8) | (byte_at(p + 2) << 16) | (byte_at(p + 3) << 24);
}

// greedy_matches over src[0, n) by the warp: on_match(at, offset, length) is called by every lane, in order. It returns
// false to stop the parse early (the caller's output has already outgrown the payload).
template <class OnMatch>
__device__ void warp_matches(const uint8_t *src, int64_t n, MatchSmem &s, int lane, OnMatch on_match) {
  if (n <= obz::kMfLimit) return;
  table_reset(s, lane);
  const int64_t limit = n - obz::kMfLimit, mend = n - obz::kLastLiterals;
  const uint32_t below = (1u << lane) - 1u;
  int64_t ip = 0, S = 0;   // S: where the table was last swept (every entry read from there on is unambiguous)
  while (ip <= limit) {
    if (min(ip + 31, limit) - S > obz::kMaxOffset) {
      table_sweep(s, min(ip, S + obz::kMaxOffset), ip, lane);
      S = ip;
    }
    const int64_t p = ip + lane;
    const bool active = p <= limit;
    const uint32_t seq = active ? rd32(src + p) : 0u;
    const uint32_t h = obz::hash4(seq);
    const uint32_t peers = __match_any_sync(0xffffffffu, active ? h : 0x10000u + lane);
    const uint32_t lower = peers & below;
    int64_t ref;
    bool ok;
    if (lower) {
      ref = ip + (31 - __clz(lower));
      ok = true;
    } else {
      const uint32_t v = s.lo[h] | (((s.hi[h >> 5] >> (h & 31)) & 1u) << 16);
      const int64_t d = (int64_t)(((uint32_t)p - v) & 0x1ffffu);
      ok = d >= 1 && d <= obz::kMaxOffset;
      ref = p - d;
    }
    const bool valid = active && ok && rd32(src + ref) == seq;
    const uint32_t vb = __ballot_sync(0xffffffffu, valid);
    const int last = vb ? __ffs(vb) - 1 : 31;   // positions up to here were probed
    const uint32_t upto = last == 31 ? 0xffffffffu : (2u << last) - 1u;
    if (active && lane <= last && (peers & upto & ~((2u << lane) - 1u)) == 0) {   // the last writer of its hash
      const uint32_t v = (uint32_t)p & 0x1ffffu;
      s.lo[h] = (uint16_t)v;
      if (v >> 16) atomicOr(&s.hi[h >> 5], 1u << (h & 31));
      else atomicAnd(&s.hi[h >> 5], ~(1u << (h & 31)));
    }
    __syncwarp();
    if (!vb) {
      ip += 32;
      continue;
    }
    const int64_t at = ip + last;
    const int64_t mref = __shfl_sync(0xffffffffu, ref, last);
    int64_t len = 4;
    for (;;) {
      const int64_t q = at + len + lane;
      const bool same = q < mend && byte_at(src + mref + len + lane) == byte_at(src + q);
      const uint32_t diff = __ballot_sync(0xffffffffu, !same);
      if (diff) {
        len += __ffs(diff) - 1;
        break;
      }
      len += 32;
    }
    if (!on_match(at, at - mref, len)) return;
    ip = at + len;
  }
}

// warp copy of src[0, n) to dst[0, n), bytes at dst index >= cap dropped
__device__ __forceinline__ void warp_copy(uint8_t *dst, const uint8_t *src, int64_t n, int64_t cap, int lane) {
  const int64_t m = min(n, cap);
  for (int64_t i = lane; i < m; i += 32) dst[i] = byte_at(src + i);
}

struct BoundedSink {   // obz byte sink: z[pos], bytes at or beyond cap dropped
  uint8_t *z;
  int64_t pos, cap;
  __device__ void put(uint8_t b) {
    if (pos < cap) z[pos] = b;
    ++pos;
  }
};

// LZ4 block of src[0, n) into z (capacity n); returns its size (>= n: keep the payload raw)
__device__ int64_t warp_lz4(const uint8_t *src, int64_t n, uint8_t *z, MatchSmem &s, int lane) {
  int64_t o = 0, anchor = 0;
  auto sequence = [&](int64_t lit_end, int64_t offset, int64_t mlen) {   // mlen 0: the final literal-only sequence
    const int64_t lit = lit_end - anchor, ml = mlen ? mlen - 4 : 0;
    const int64_t el = lit >= 15 ? (lit - 15) / 255 + 1 : 0, em = mlen && ml >= 15 ? (ml - 15) / 255 + 1 : 0;
    const int64_t total = 1 + el + lit + (mlen ? 2 + em : 0);
    const int64_t m = min(total, n - o);
    for (int64_t i = lane; i < m; i += 32) {
      uint8_t b;
      if (i == 0) {
        b = (uint8_t)((min(lit, (int64_t)15) << 4) | min(ml, (int64_t)15));
      } else if (i < 1 + el) {
        b = i < el ? 255 : (uint8_t)((lit - 15) % 255);
      } else if (i < 1 + el + lit) {
        b = (uint8_t)byte_at(src + anchor + (i - 1 - el));
      } else {
        const int64_t k = i - (1 + el + lit);
        b = k == 0 ? (uint8_t)(offset & 0xff) : k == 1 ? (uint8_t)(offset >> 8) : k < 1 + em ? 255 : (uint8_t)((ml - 15) % 255);
      }
      z[o + i] = b;
    }
    o += total;
  };
  warp_matches(src, n, s, lane, [&](int64_t at, int64_t offset, int64_t len) {
    sequence(at, offset, len);
    anchor = at + len;
    return o < n;
  });
  if (o < n) sequence(n, 0, 0);
  return o;
}

// zstd frame of src[0, n) into z (capacity n); returns its size (>= n: keep the payload raw). seqs: room for one chunk's list.
__device__ int64_t warp_zstd(const uint8_t *src, int64_t n, uint8_t *z, obz::Seq *seqs, MatchSmem &s, int lane) {
  BoundedSink head{z, 0, n};
  if (lane == 0) obz::zstd_frame_header(head, n);
  int64_t pos = head.pos;   // every lane counts the same bytes
  if (lane != 0) {
    BoundedSink dry{nullptr, 0, 0};
    obz::zstd_frame_header(dry, n);
    pos = dry.pos;
  }
  int64_t at = 0;
  do {
    const int64_t len = min(obz::kZstdBlock, n - at);
    const uint8_t *c = src + at;
    const int64_t body = pos + 3;   // the block content, after the 3-byte block header
    int64_t csize = len;            // content size (len: Raw block)
    bool raw = true;
    if (len > 0 && body < n) {
      // literals as they are found, 3 bytes after the content start (the largest literals header); sequences listed
      uint32_t ns = 0;
      int64_t nl = 0, anchor = 0;
      auto literals = [&](int64_t end) {
        if (end > anchor) warp_copy(z + body + 3 + nl, c + anchor, end - anchor, n - (body + 3 + nl), lane);
        nl += end - anchor;
      };
      warp_matches(c, len, s, lane, [&](int64_t m_at, int64_t offset, int64_t m_len) {
        if (lane == 0) seqs[ns] = obz::Seq{(uint32_t)(m_at - anchor), (uint32_t)offset, (uint32_t)m_len};
        ++ns;
        literals(m_at);
        anchor = m_at + m_len;
        return true;
      });
      literals(len);
      __syncwarp();
      // the literals header is 1..3 bytes: move the literals down to meet it (forward, 32 bytes per step)
      const int hl = obz::zstd_literals_header_size((uint32_t)nl);
      if (hl < 3) {
        const int64_t from = body + 3, to = body + hl, m = min(nl, n - from);
        for (int64_t g = 0; g < m; g += 32) {
          const int64_t i = g + lane;
          const uint8_t b = i < m ? z[from + i] : 0;
          __syncwarp();
          if (i < m) z[to + i] = b;
          __syncwarp();
        }
      }
      int64_t end = 0;
      if (lane == 0) {
        BoundedSink o{z, body, n};
        obz::zstd_literals_header(o, (uint32_t)nl);
        o.pos += nl;
        obz::zstd_sequences(o, seqs, ns, s.fse);
        end = o.pos;
      }
      end = __shfl_sync(0xffffffffu, end, 0);
      csize = end - body;
      raw = csize >= len;
    }
    __syncwarp();
    if (raw) {
      csize = len;
      warp_copy(z + body, c, len, n - body, lane);
    }
    if (lane == 0) {
      BoundedSink o{z, pos, n};
      obz::zstd_block_header(o, at + len == n, raw, (uint32_t)csize);
    }
    pos = body + csize;
    at += len;
  } while (at < n && pos < n);
  __syncwarp();
  return at < n ? n : pos;
}

template <int32_t COMPRESSOR>
__global__ void __launch_bounds__(32, 1) obgpu_compress_match_kernel(const uint8_t *image, const int64_t *off, const uint32_t *size,
                                                                     int32_t n_blocks, const int64_t *stage_off, uint8_t *stage,
                                                                     obz::Seq *seq_scratch, uint32_t *stored, Work *w) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  MatchSmem &s = *reinterpret_cast<MatchSmem *>(smem_raw);
  const int lane = threadIdx.x;
  if (COMPRESSOR == OBGPU_COMPRESSOR_ZSTD_1_3_8 && lane == 0) obz::fse_build_predefined(s.fse);
  __syncwarp();
  obz::Seq *seqs = seq_scratch + (size_t)blockIdx.x * (obz::kZstdBlock / 4);
  for (;;) {
    int32_t b = 0;
    if (lane == 0) b = atomicAdd(&w->next, 1);
    b = __shfl_sync(0xffffffffu, b, 0);
    if (b >= n_blocks) return;
    const int64_t sz = size[b];
    if (sz == 0) {
      if (lane == 0) stored[b] = 0;
      continue;
    }
    const uint8_t *blk = image + off[b];
    int64_t hs, len, zlen;
    plain_fields(blk, hs, len, zlen);
    int64_t zn = len;   // >= len: stored raw
    if (COMPRESSOR != OBGPU_COMPRESSOR_NONE && len > 0) {
      uint8_t *z = stage + stage_off[b];
      if (COMPRESSOR == OBGPU_COMPRESSOR_ZSTD_1_3_8) zn = warp_zstd(blk + hs, len, z, seqs, s, lane);
      else zn = warp_lz4(blk + hs, len, z, s, lane);
    }
    if (lane == 0) stored[b] = (uint32_t)(zn < len ? hs + zn : sz);
  }
}

// aligned stored sizes -> the layout prefix's counts
__global__ void __launch_bounds__(256) obgpu_compress_align_kernel(const uint32_t *stored, int32_t n, uint32_t align, uint32_t *cnt) {
  const int32_t i = (int32_t)(blockIdx.x * blockDim.x + threadIdx.x);
  if (i < n) cnt[i] = (stored[i] + align - 1) & ~(align - 1);
}

__global__ void __launch_bounds__(kFrameThreads) obgpu_compress_frame_kernel(const uint8_t *image, const int64_t *off, const uint32_t *size,
                                                                             const int64_t *stage_off, const uint8_t *stage,
                                                                             const uint32_t *stored, const int64_t *dst_off, int64_t align,
                                                                             uint8_t *out, int64_t *out_off, uint32_t *out_size, Work *w) {
  __shared__ uint32_t tab[256];
  __shared__ uint32_t crc;
  const int64_t b = blockIdx.x;
  const int tid = threadIdx.x;
  const int64_t dst = dst_off[b], ss = stored[b], sz = size[b];
  if (tid == 0) {
    out_off[b] = dst;
    out_size[b] = (uint32_t)ss;
  }
  if (ss == 0) return;
  sb::build_crc_table(tab);
  const uint8_t *in = image + off[b];
  const int64_t hs = sb::ld32u(in + 4);
  const bool packed = ss != sz;
  const uint8_t *payload = packed ? stage + stage_off[b] : in + hs;
  uint8_t *d = out + dst;
  for (int64_t i = tid; i < hs; i += kFrameThreads) d[i] = __ldg(in + i);
  for (int64_t i = tid; i < ss - hs; i += kFrameThreads) d[hs + i] = __ldg(payload + i);
  const int64_t pad_end = (dst + ss + align - 1) & ~(align - 1);
  for (int64_t i = dst + ss + tid; i < pad_end; i += kFrameThreads) out[i] = 0;
  if (packed && tid < 32) {
    const uint32_t c = sb::warp_crc32c(tab, payload, ss - hs, tid);
    if (tid == 0) crc = c;
  }
  __syncthreads();
  if (tid == 0) {
    if (packed) {   // data_zlength_, data_checksum_ (crc32c of the stored bytes, zero-extended), then the header checksum
      const uint32_t zl = (uint32_t)(ss - hs);
      for (int k = 0; k < 4; ++k) d[44 + k] = (uint8_t)(zl >> (8 * k));
      for (int k = 0; k < 8; ++k) d[48 + k] = k < 4 ? (uint8_t)(crc >> (8 * k)) : 0;
      const uint16_t hc = (uint16_t)obf::micro_header_checksum(d);
      d[8] = (uint8_t)hc;
      d[9] = (uint8_t)(hc >> 8);
    }
    atomicMax(&w->end, (unsigned long long)(dst + ss));
  }
}

}  // namespace sc

extern "C" int obgpu_compress_blocks(obgpu_ctx *ctx, const void *d_image, const int64_t *d_offsets, const uint32_t *d_sizes, int32_t n_blocks,
                                     int32_t compressor, int32_t align, void *d_out, int64_t out_cap, int64_t *d_out_offsets,
                                     uint32_t *d_out_sizes, int64_t *out_size) {
  if (!ctx || !d_image || !d_offsets || !d_sizes || n_blocks <= 0 || !out_size || align < 1 || align > 4096 || (align & (align - 1)) != 0 ||
      (d_out && (!d_out_offsets || !d_out_sizes)))
    return OBGPU_INVALID_ARGUMENT;
  if (!obf::device_compressor(compressor)) {
    ctx->err = "compressor not handled by the device path";
    return OBGPU_NOT_SUPPORTED;
  }
  cudaSetDevice(ctx->device);
  const int64_t n = n_blocks;
  const int n_chunks = (int)((n + kPrefixChunk - 1) / kPrefixChunk);
  // [Work][stage_off i64 x (n + 1)][dst_off i64 x (n + 1)][chunk totals u64 x n_chunks][cnt u32 x n][stored u32 x n]
  Scratch work(ctx);
  const size_t o_w = work.take(64, 8), o_stage_off = work.take((size_t)(n + 1) * 8, 8), o_dst_off = work.take((size_t)(n + 1) * 8, 8);
  const size_t o_chunk = work.take((size_t)n_chunks * 8, 8), o_cnt = work.take((size_t)n * 4, 4), o_stored = work.take((size_t)n * 4, 4);
  CUDA_TRY(ctx, work.alloc());
  sc::Work *w = work.at<sc::Work>(o_w);
  int64_t *stage_off = work.at<int64_t>(o_stage_off), *dst_off = work.at<int64_t>(o_dst_off);
  unsigned long long *chunk_tot = work.at<unsigned long long>(o_chunk);
  uint32_t *cnt = work.at<uint32_t>(o_cnt), *stored = work.at<uint32_t>(o_stored);
  CUDA_TRY(ctx, cudaMemsetAsync(w, 0, sizeof(sc::Work), ctx->stream));
  const unsigned grid = (unsigned)((n + 255) / 256);
  sc::obgpu_compress_survey_kernel<<<grid, 256, 0, ctx->stream>>>((const uint8_t *)d_image, d_offsets, d_sizes, n_blocks, align, cnt, w);
  ctx->launches++;
  sc::Work h{};
  CUDA_TRY(ctx, cudaMemcpyAsync(&h, w, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (h.verdict & sc::kBadArg) { ctx->err = "block offsets must be non-negative multiples of 16"; return OBGPU_INVALID_ARGUMENT; }
  if (h.verdict & sc::kBadData) { ctx->err = "a block to compress is not a plain, well-framed micro-block"; return OBGPU_INVALID_DATA; }
  if (h.verdict & sc::kTooLarge) { ctx->err = "a block to compress is larger than 0x7f000000 bytes"; return OBGPU_NOT_SUPPORTED; }
  if (!d_out) {
    *out_size = (int64_t)h.cap;
    return OBGPU_SUCCESS;
  }
  if (out_cap < (int64_t)h.cap) { ctx->err = "output capacity below the sum of the aligned block sizes"; return OBGPU_BUF_NOT_ENOUGH; }
  // staging slots for the compressed payloads
  obgpu_prefix_local_kernel<<<n_chunks, 256, 0, ctx->stream>>>(cnt, n_blocks, stage_off, chunk_tot);
  obgpu_prefix_fix_kernel<<<n_chunks + 1, 256, 0, ctx->stream>>>(n_blocks, n_chunks, stage_off, chunk_tot);
  ctx->launches += 2;
  const bool packs = compressor != OBGPU_COMPRESSOR_NONE;
  Scratch stage(ctx), seqs(ctx);
  if (packs) CUDA_TRY(ctx, stage.alloc((size_t)h.stage + 16));
  const int ctas = (int)std::min<int64_t>(n, std::max(ctx->sm_count, 1));
  if (compressor == OBGPU_COMPRESSOR_ZSTD_1_3_8) CUDA_TRY(ctx, seqs.alloc((size_t)ctas * (obz::kZstdBlock / 4) * sizeof(obz::Seq)));
  decltype(&sc::obgpu_compress_match_kernel<OBGPU_COMPRESSOR_NONE>) match;
  switch (compressor) {
    case OBGPU_COMPRESSOR_LZ4: case OBGPU_COMPRESSOR_LZ4_1_9_1: match = sc::obgpu_compress_match_kernel<OBGPU_COMPRESSOR_LZ4>; break;
    case OBGPU_COMPRESSOR_ZSTD_1_3_8: match = sc::obgpu_compress_match_kernel<OBGPU_COMPRESSOR_ZSTD_1_3_8>; break;
    default: match = sc::obgpu_compress_match_kernel<OBGPU_COMPRESSOR_NONE>; break;
  }
  const int smem = packs ? (int)sizeof(sc::MatchSmem) : 0;
  if (packs) CUDA_TRY(ctx, cudaFuncSetAttribute((const void *)match, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  match<<<(unsigned)ctas, 32, smem, ctx->stream>>>((const uint8_t *)d_image, d_offsets, d_sizes, n_blocks, stage_off, stage.p,
                                                   seqs.at<obz::Seq>(0), stored, w);
  sc::obgpu_compress_align_kernel<<<grid, 256, 0, ctx->stream>>>(stored, n_blocks, (uint32_t)align, cnt);
  obgpu_prefix_local_kernel<<<n_chunks, 256, 0, ctx->stream>>>(cnt, n_blocks, dst_off, chunk_tot);
  obgpu_prefix_fix_kernel<<<n_chunks + 1, 256, 0, ctx->stream>>>(n_blocks, n_chunks, dst_off, chunk_tot);
  sc::obgpu_compress_frame_kernel<<<(unsigned)n, sc::kFrameThreads, 0, ctx->stream>>>(
      (const uint8_t *)d_image, d_offsets, d_sizes, stage_off, stage.p, stored, dst_off, align, (uint8_t *)d_out,
      d_out_offsets, d_out_sizes, w);
  ctx->launches += 5;
  CUDA_TRY(ctx, cudaGetLastError());
  CUDA_TRY(ctx, cudaMemcpyAsync(&h, w, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  *out_size = (int64_t)h.end;
  return OBGPU_SUCCESS;
}
