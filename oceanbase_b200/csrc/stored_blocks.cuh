// Micro-blocks in stored form opened ON THE DEVICE into a page batch (ObMacroBlockReader::decompress_data -> the compressor's
// decompress, one micro-block at a time on the CPU in the reference). On disk a micro-block is [ObMicroBlockHeader, plain]
// [payload compressed on its own]: data_zlength_ bytes stored, data_length_ bytes after decoding, data_checksum_ = crc32c of the
// STORED payload. A block whose payload did not shrink is stored raw (data_zlength_ == data_length_). Opening such blocks is
//   survey  : one thread per block -- magic, header_size_, header_size_ + data_zlength_ == stored size -> decoded size, raw or not
//   slots   : host prefix over the decoded sizes, 128-byte aligned slots
//   copy    : raw blocks, one CTA per block (obgpu_macro_realign_kernel): unaligned source words through funnel shifts, 16-byte
//             stores, zero padding -- one read + one write of the data, at HBM speed
//   decode  : compressed blocks, ONE WARP per block (obgpu_stored_decode_kernel, one instantiation per codec):
//             header checksum (lane 0) and payload crc32c over the stored bytes (every lane the raw CRC of a contiguous chunk,
//             shifted into place by a carry-less multiplication with x^(8 * bytes after it), XOR-reduced -- enc::gf2_mulmod /
//             enc::crc_byte of the device encoder), then the codec's decoder straight into the block's slot in global memory:
//             lz4d::warp_lz4_decode (lz4_decode.cuh; compressors 2 and 7), zstdd::decode_frame (zstd_decode.cuh, compressor 6,
//             one plain zstd frame per payload) or zlibd::decode_stream (zlib_decode.cuh, compressor 4, one zlib stream per
//             payload), with the warp's tables in shared memory. The slot's tail up to 128 bytes is zeroed.
//   open    : obgpu_batch_open(image_on_device = 1, header_view = NULL) over the decoded image, which the batch then owns
// The decoders are the boundary for bytes from outside the program: every read is checked against the stored extent, every
// write against data_length_. A failed block sets its status; the open returns OBGPU_INVALID_DATA and the ctx stays usable.
#pragma once
#include <type_traits>

#include "lz4_decode.cuh"
#include "zlib_decode.cuh"
#include "zstd_decode.cuh"

namespace sb {

constexpr int kWarps = 4;   // warps (blocks) per CTA: 4 x zstd's 10.75 KiB of tables + the crc table fit the 48 KiB static limit
constexpr int32_t kStOk = 0, kStBadHeader = 1, kStBadStream = 2, kStBadChecksum = 3;

__device__ __forceinline__ uint32_t ld32u(const uint8_t *p) {   // unaligned little-endian loads
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
__device__ __forceinline__ uint64_t ld64u(const uint8_t *p) { return (uint64_t)ld32u(p) | ((uint64_t)ld32u(p + 4) << 32); }

__device__ __forceinline__ uint32_t xpow8(uint32_t n) {   // x^(8 n) mod P, reflected (x^0 = 0x80000000)
  uint32_t r = 0x80000000u, b = 0x00800000u;               // b = x^8
  while (n) {
    if (n & 1u) r = enc::gf2_mulmod(r, b);
    b = enc::gf2_mulmod(b, b);
    n >>= 1;
  }
  return r;
}

// crc32c (seed 0, no final xor: ob_crc64_sse42) of in[0, n) by the whole warp
__device__ uint32_t warp_crc32c(const uint32_t *tab, const uint8_t *in, int64_t n, int lane) {
  const int64_t chunk = (n + 31) / 32;
  const int64_t b0 = min((int64_t)lane * chunk, n), b1 = min(b0 + chunk, n);
  uint32_t crc = 0;
  for (int64_t i = b0; i < b1; ++i) crc = enc::crc_byte(tab, crc, __ldg(in + i));
  if (crc != 0 && b1 < n) crc = enc::gf2_mulmod(crc, xpow8((uint32_t)(n - b1)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) crc ^= __shfl_xor_sync(0xffffffffu, crc, o);
  return crc;
}

__device__ __forceinline__ void build_crc_table(uint32_t *tab) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    uint32_t c = (uint32_t)i;
#pragma unroll
    for (int k = 0; k < 8; ++k) c = (c & 1u) ? enc::kCrcPoly ^ (c >> 1) : c >> 1;
    tab[i] = c;
  }
  __syncthreads();
}

// ObMicroBlockHeader::check_header_checksum (ob_micro_block_header.cpp:236-262)
__device__ bool header_checksum_ok(const uint8_t *h) {
  return (uint16_t)obf::micro_header_checksum(h) == ((uint32_t)h[8] | ((uint32_t)h[9] << 8));
}

// survey of stored micro-blocks: dsize[i] = header_size_ + data_length_, kind[i] = 1 when compressed; *status = max verdict
__global__ void obgpu_stored_survey_kernel(const uint8_t *image, const int64_t *src_off, const int64_t *zsize, int32_t n, int32_t compressor,
                                           int64_t *dsize, int32_t *kind, int32_t *status) {
  const int32_t i = (int32_t)(blockIdx.x * blockDim.x + threadIdx.x);
  if (i >= n) return;
  const uint8_t *h = image + src_off[i];
  const uint32_t magic = (uint32_t)h[0] | ((uint32_t)h[1] << 8);
  const int64_t hs = ld32u(h + 4);
  const int64_t len = (int32_t)ld32u(h + 40), zlen = (int32_t)ld32u(h + 44);
  int32_t st = kStOk;
  if (magic != 1005u || hs < 64 || len <= 0 || zlen <= 0 || hs + zlen != zsize[i] || hs + len > 0x7fffffffll) st = kStBadHeader;
  else if (zlen != len && compressor == OBGPU_COMPRESSOR_NONE) st = kStBadHeader;   // a NONE table stores every block raw
  dsize[i] = st == kStOk ? hs + len : 0;
  kind[i] = st == kStOk && zlen != len ? 1 : 0;
  if (st != kStOk) atomicMax(status, st);
}

// raw block i: image[src_off[i], + sizes[i]) -> out[dst_off[i], + sizes[i] rounded up to 128), zero padded
constexpr int kCopyThreads = 128;
__global__ void __launch_bounds__(kCopyThreads) obgpu_macro_realign_kernel(const uint8_t *image, int64_t image_size, const int64_t *src_off,
                                                                            const int64_t *sizes, const int64_t *dst_off, uint8_t *out) {
  const int64_t blk = blockIdx.x;
  const int64_t src = src_off[blk], sz = sizes[blk];
  const int64_t slot = (sz + 127) & ~127ll;
  uint4 *dst = reinterpret_cast<uint4 *>(out + dst_off[blk]);
  const uint32_t sh = (uint32_t)(src & 3) * 8u;
  const uint32_t *w = reinterpret_cast<const uint32_t *>(image + (src & ~3ll));
  const int64_t avail = image_size - (src & ~3ll);   // bytes readable from w
  const int64_t w_cap = avail >> 2;                   // whole words readable from w
  // the image may end inside a word (stored blocks lie at any byte offset): its last 1 - 3 bytes are read one by one
  uint32_t tail = 0;
  for (int b = 0; b < (int)(avail & 3); ++b) tail |= (uint32_t)(reinterpret_cast<const uint8_t *>(w + w_cap))[b] << (8 * b);
  for (int64_t j = threadIdx.x; j < slot / 16; j += kCopyThreads) {
    uint32_t v[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      const int64_t idx = j * 4 + k;
      v[k] = idx < w_cap ? __ldg(w + idx) : (idx == w_cap ? tail : 0u);
    }
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k] = __funnelshift_r(v[k], v[k + 1], sh);
    const int64_t left = sz - j * 16;   // bytes of this chunk that belong to the block
    if (left < 16) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int64_t lb = left - 4 * k;
        o[k] = lb >= 4 ? o[k] : (lb <= 0 ? 0u : (o[k] & (0xffffffffu >> (32 - 8 * (int)lb))));
      }
    }
    dst[j] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// A codec: the per-warp shared scratch its decoder needs (an empty struct: none) and decode(), kStOk only when in[0, n_in) is
// one well-formed payload of exactly n_out bytes.
struct Lz4 {
  struct Scratch {};
  static __device__ __forceinline__ int32_t decode(const uint8_t *in, int64_t n_in, uint8_t *out, int64_t n_out, Scratch *, int lane) {
    return lz4d::warp_lz4_decode(in, n_in, out, n_out, lane) ? kStOk : kStBadStream;
  }
};
struct Zstd {
  using Scratch = zstdd::Work;
  static __device__ __forceinline__ int32_t decode(const uint8_t *in, int64_t n_in, uint8_t *out, int64_t n_out, Scratch *w, int lane) {
    return zstdd::decode_frame(in, n_in, out, n_out, *w, lane, 32) == zstdd::kOk ? kStOk : kStBadStream;
  }
};
struct Zlib {
  using Scratch = zlibd::Work;
  static __device__ __forceinline__ int32_t decode(const uint8_t *in, int64_t n_in, uint8_t *out, int64_t n_out, Scratch *w, int lane) {
    return zlibd::decode_stream(in, n_in, out, n_out, *w, lane, 32) == zlibd::kOk ? kStOk : kStBadStream;
  }
};

// BLOCKS = true : micro-blocks (checksums checked, header copied, payload decoded, slot tail zeroed), tables indexed by block
// BLOCKS = false: bare payloads in[in_off, + in_len) -> out[out_off, + out_len) (obgpu_lz4_decompress, obgpu_zstd_decompress,
//                 obgpu_zlib_decompress)
template <class Codec, bool BLOCKS>
__global__ void __launch_bounds__(kWarps * 32) obgpu_stored_decode_kernel(const uint8_t *in_base, const int64_t *in_off, const int64_t *in_len,
                                                                          uint8_t *out_base, const int64_t *out_off, const int64_t *out_len,
                                                                          int32_t n, int32_t *blk_status, int32_t *any_status) {
  __shared__ uint32_t tab[256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  typename Codec::Scratch *scratch = nullptr;
  if constexpr (!std::is_empty<typename Codec::Scratch>::value) {   // an array of empty structs would still take shared memory
    __shared__ typename Codec::Scratch work[kWarps];
    scratch = work + warp;
  }
  if (BLOCKS) build_crc_table(tab);
  const int64_t blk = (int64_t)blockIdx.x * kWarps + warp;
  if (blk >= n) return;
  const uint8_t *in = in_base + in_off[blk];
  uint8_t *out = out_base + out_off[blk];
  const int64_t zn = in_len[blk], dn = out_len[blk];
  int32_t st = kStOk;
  if (BLOCKS) {
    const int64_t hs = ld32u(in + 4);   // the survey checked hs >= 64, hs + data_zlength_ == zn, hs + data_length_ == dn
    int32_t ok = 1;
    if (lane == 0) ok = header_checksum_ok(in) ? 1 : 0;
    ok = __shfl_sync(0xffffffffu, ok, 0);
    if (ok) {
      const uint32_t crc = warp_crc32c(tab, in + hs, zn - hs, lane);
      ok = (uint64_t)crc == ld64u(in + 48);
    }
    if (!ok) {
      st = kStBadChecksum;
    } else {
      for (int64_t i = lane; i < hs; i += 32) out[i] = __ldg(in + i);   // the stored header, unchanged
      st = Codec::decode(in + hs, zn - hs, out + hs, dn - hs, scratch, lane);
    }
    __syncwarp();
    const int64_t slot = (dn + 127) & ~127ll;
    for (int64_t i = (st == kStOk ? dn : 0) + lane; i < slot; i += 32) out[i] = 0;   // zero tail (whole slot on failure)
  } else {
    st = Codec::decode(in, zn, out, dn, scratch, lane);
  }
  if (lane == 0) {
    blk_status[blk] = st;
    if (st != kStOk) atomicMax(any_status, st);
  }
}

}  // namespace sb

// Launches the decode of n payloads of `compressor` (blocks: stored micro-blocks, else bare payloads) and returns what a
// malformed payload is called in ctx->err; nullptr for a compressor without a decoder (NONE: its blocks are all raw).
static const char *launch_decode(obgpu_ctx *ctx, int32_t compressor, bool blocks, const uint8_t *in, const int64_t *in_off,
                                 const int64_t *in_len, uint8_t *out, const int64_t *out_off, const int64_t *out_len, int32_t n,
                                 int32_t *blk_status, int32_t *any_status) {
  decltype(&sb::obgpu_stored_decode_kernel<sb::Lz4, true>) kernel;
  const char *malformed;
  switch (compressor) {
    case OBGPU_COMPRESSOR_LZ4:
    case OBGPU_COMPRESSOR_LZ4_1_9_1:
      kernel = blocks ? sb::obgpu_stored_decode_kernel<sb::Lz4, true> : sb::obgpu_stored_decode_kernel<sb::Lz4, false>;
      malformed = blocks ? "LZ4 payload of a micro-block is malformed" : "an LZ4 block is malformed";
      break;
    case OBGPU_COMPRESSOR_ZSTD_1_3_8:
      kernel = blocks ? sb::obgpu_stored_decode_kernel<sb::Zstd, true> : sb::obgpu_stored_decode_kernel<sb::Zstd, false>;
      malformed = blocks ? "zstd payload of a micro-block is malformed" : "a zstd frame is malformed";
      break;
    case OBGPU_COMPRESSOR_ZLIB:
      kernel = blocks ? sb::obgpu_stored_decode_kernel<sb::Zlib, true> : sb::obgpu_stored_decode_kernel<sb::Zlib, false>;
      malformed = blocks ? "zlib payload of a micro-block is malformed" : "a zlib stream is malformed";
      break;
    default:
      return nullptr;
  }
  kernel<<<(unsigned)((n + sb::kWarps - 1) / sb::kWarps), sb::kWarps * 32, 0, ctx->stream>>>(in, in_off, in_len, out, out_off, out_len, n,
                                                                                             blk_status, any_status);
  ctx->launches++;
  return malformed;
}

// The image an open reads on the device. A host image is uploaded to `copy`, freed on the ctx stream once the open is enqueued;
// a device image is read in place and must be 16-byte aligned, else `misaligned` is the error.
struct DeviceImage {
  const uint8_t *d = nullptr;
  Scratch copy;
  explicit DeviceImage(obgpu_ctx *ctx) : copy(ctx) {}
};
static int stage_image(obgpu_ctx *ctx, const void *image, int64_t image_size, int32_t image_on_device, const char *misaligned,
                       DeviceImage &img) {
  if (image_on_device) {
    if (((uintptr_t)image & 15u) != 0) {
      ctx->err = misaligned;
      return OBGPU_INVALID_ARGUMENT;
    }
    img.d = (const uint8_t *)image;
    return OBGPU_SUCCESS;
  }
  CUDA_TRY(ctx, img.copy.alloc((size_t)image_size));
  CUDA_TRY(ctx, cudaMemcpyAsync(img.copy.p, image, (size_t)image_size, cudaMemcpyHostToDevice, ctx->stream));
  img.d = img.copy.p;
  return OBGPU_SUCCESS;
}

// Stored micro-blocks d_image[d_src[i], + d_zsize[i]) (device tables) -> page batch owning the decoded, realigned image.
// The one routine behind obgpu_batch_open_macro_blocks and obgpu_batch_open_compressed.
static int open_stored_blocks(obgpu_ctx *ctx, const uint8_t *d_image, int64_t image_size, const int64_t *d_src, const int64_t *d_zsize,
                              int32_t n, int32_t compressor, obgpu_batch **out) {
  std::vector<int64_t> src((size_t)n), zsize((size_t)n), dsize((size_t)n), dst((size_t)n);
  std::vector<int32_t> kind((size_t)n);
  Scratch work(ctx);   // survey tables
  const size_t o_dsize = work.take((size_t)n * 8, 4), o_kind = work.take((size_t)n * 4, 4), o_status = work.take(64, 4);
  CUDA_TRY(ctx, work.alloc());
  int64_t *d_dsize = work.at<int64_t>(o_dsize);
  int32_t *d_kind = work.at<int32_t>(o_kind), *d_status = work.at<int32_t>(o_status);
  CUDA_TRY(ctx, cudaMemsetAsync(d_status, 0, 4, ctx->stream));
  sb::obgpu_stored_survey_kernel<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(d_image, d_src, d_zsize, n, compressor, d_dsize,
                                                                                        d_kind, d_status);
  ctx->launches++;
  int32_t st = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(dsize.data(), d_dsize, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(kind.data(), d_kind, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(&st, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(src.data(), d_src, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(zsize.data(), d_zsize, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (st != sb::kStOk) {
    ctx->err = "micro-block header of a stored block is invalid";
    return OBGPU_INVALID_DATA;
  }
  // slots + the two work lists: raw -> realign copy, compressed -> decoder
  const int64_t out_bytes = (int64_t)slot_layout(dsize.data(), n, dst.data());
  std::vector<int64_t> raw_tab, lz_tab;   // raw: [src][size][dst], compressed: [src][zsize][dst][dsize]
  std::vector<int32_t> raw_idx, lz_idx;
  for (int32_t i = 0; i < n; ++i) (kind[(size_t)i] ? lz_idx : raw_idx).push_back(i);
  const size_t nr = raw_idx.size(), nz = lz_idx.size();
  raw_tab.resize(nr * 3);
  lz_tab.resize(nz * 4);
  for (size_t k = 0; k < nr; ++k) {
    const int32_t i = raw_idx[k];
    raw_tab[k] = src[(size_t)i]; raw_tab[nr + k] = zsize[(size_t)i]; raw_tab[2 * nr + k] = dst[(size_t)i];
  }
  for (size_t k = 0; k < nz; ++k) {
    const int32_t i = lz_idx[k];
    lz_tab[k] = src[(size_t)i]; lz_tab[nz + k] = zsize[(size_t)i]; lz_tab[2 * nz + k] = dst[(size_t)i]; lz_tab[3 * nz + k] = dsize[(size_t)i];
  }
  Scratch decoded(ctx);   // the batch's image once it opens
  CUDA_TRY(ctx, decoded.alloc((size_t)out_bytes + 64));
  uint8_t *d_out = decoded.p;
  CUDA_TRY(ctx, cudaMemsetAsync(d_out + out_bytes, 0, 64, ctx->stream));
  Scratch tab(ctx);   // [raw work list][compressed work list][per-block status]
  const size_t o_raw = tab.take(nr * 24, 8), o_lz = tab.take(nz * 32, 8), o_blk_status = tab.take(nz * 4 + 64, 4);
  CUDA_TRY(ctx, tab.alloc());
  int64_t *d_raw = tab.at<int64_t>(o_raw), *d_lz = tab.at<int64_t>(o_lz);
  int32_t *d_blk_status = tab.at<int32_t>(o_blk_status);
  if (nr) CUDA_TRY(ctx, cudaMemcpyAsync(d_raw, raw_tab.data(), nr * 24, cudaMemcpyHostToDevice, ctx->stream));
  if (nz) CUDA_TRY(ctx, cudaMemcpyAsync(d_lz, lz_tab.data(), nz * 32, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaMemsetAsync(d_status, 0, 4, ctx->stream));
  if (nr) {
    sb::obgpu_macro_realign_kernel<<<(unsigned)nr, sb::kCopyThreads, 0, ctx->stream>>>(d_image, image_size, d_raw, d_raw + nr, d_raw + 2 * nr,
                                                                                       d_out);
    ctx->launches++;
  }
  const char *malformed = nullptr;
  if (nz)
    malformed = launch_decode(ctx, compressor, true, d_image, d_lz, d_lz + nz, d_out, d_lz + 2 * nz, d_lz + 3 * nz, (int32_t)nz,
                              d_blk_status, d_status);
  // the host tables were copy sources: synchronise before they go out of scope
  CUDA_TRY(ctx, cudaGetLastError());
  CUDA_TRY(ctx, cudaMemcpyAsync(&st, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (st != sb::kStOk) {
    ctx->err = st == sb::kStBadChecksum ? "checksum of a compressed micro-block does not match" : malformed;
    return OBGPU_INVALID_DATA;
  }
  obgpu_batch *b = nullptr;
  const int ret = obgpu_batch_open(ctx, d_out, out_bytes, dst.data(), dsize.data(), n, 1, nullptr, &b);
  if (ret != OBGPU_SUCCESS) return ret;
  b->own_image = true;   // the decoded image lives and dies with the batch
  decoded.release();
  *out = b;
  return OBGPU_SUCCESS;
}

// n independent payloads of one codec in device memory (obgpu_lz4_decompress, obgpu_zstd_decompress, obgpu_zlib_decompress)
static int decompress_streams(obgpu_ctx *ctx, const void *d_in, const int64_t *in_off, const int64_t *in_len, void *d_out, const int64_t *out_off,
                              const int64_t *out_len, int32_t n, int32_t *status, int32_t compressor) {
  if (!ctx || !d_in || !in_off || !in_len || !d_out || !out_off || !out_len || n <= 0 || !status) return OBGPU_INVALID_ARGUMENT;
  for (int32_t i = 0; i < n; ++i)
    if (in_off[i] < 0 || in_len[i] < 0 || out_off[i] < 0 || out_len[i] < 0) return OBGPU_INVALID_ARGUMENT;
  cudaSetDevice(ctx->device);
  std::vector<int64_t> tab((size_t)n * 4);
  memcpy(tab.data(), in_off, (size_t)n * 8);
  memcpy(tab.data() + n, in_len, (size_t)n * 8);
  memcpy(tab.data() + 2 * (size_t)n, out_off, (size_t)n * 8);
  memcpy(tab.data() + 3 * (size_t)n, out_len, (size_t)n * 8);
  Scratch t(ctx);   // [in_off][in_len][out_off][out_len][per-stream status][any status]
  const size_t o_tab = t.take((size_t)n * 32, 4), o_st = t.take((size_t)n * 4, 4), o_any = t.take(64, 4);
  CUDA_TRY(ctx, t.alloc());
  int64_t *d = t.at<int64_t>(o_tab);
  int32_t *d_st = t.at<int32_t>(o_st), *d_any = t.at<int32_t>(o_any);
  CUDA_TRY(ctx, cudaMemcpyAsync(d, tab.data(), (size_t)n * 32, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaMemsetAsync(d_any, 0, 4, ctx->stream));
  const char *malformed = launch_decode(ctx, compressor, false, (const uint8_t *)d_in, d, d + n, (uint8_t *)d_out, d + 2 * n, d + 3 * n, n,
                                        d_st, d_any);
  int32_t any = 0;
  CUDA_TRY(ctx, cudaGetLastError());
  CUDA_TRY(ctx, cudaMemcpyAsync(status, d_st, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(&any, d_any, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (any != sb::kStOk) {
    ctx->err = malformed;
    return OBGPU_INVALID_DATA;
  }
  return OBGPU_SUCCESS;
}

extern "C" {

int obgpu_batch_open_compressed(obgpu_ctx *ctx, const void *image, int64_t image_size, const int64_t *offsets, const int64_t *sizes,
                                int32_t n_blocks, int32_t image_on_device, int32_t compressor_type, obgpu_batch **out) {
  if (!ctx || !image || !offsets || !sizes || !out || n_blocks <= 0 || image_size <= 0) return OBGPU_INVALID_ARGUMENT;
  if (!obf::stored_compressor(compressor_type)) {
    ctx->err = "compressor not handled by the device path";
    return OBGPU_NOT_SUPPORTED;
  }
  for (int32_t i = 0; i < n_blocks; ++i)
    if (offsets[i] < 0 || sizes[i] < 64 || offsets[i] + sizes[i] > image_size) {
      ctx->err = "stored block outside the image";
      return OBGPU_INVALID_ARGUMENT;
    }
  cudaSetDevice(ctx->device);
  DeviceImage img(ctx);
  const int ret = stage_image(ctx, image, image_size, image_on_device, "a device-resident image must be 16-byte aligned", img);
  if (ret != OBGPU_SUCCESS) return ret;
  Scratch tabs(ctx);   // [src][zsize]
  const size_t o_src = tabs.take((size_t)n_blocks * 8, 8), o_zs = tabs.take((size_t)n_blocks * 8, 8);
  CUDA_TRY(ctx, tabs.alloc());
  int64_t *d_src = tabs.at<int64_t>(o_src), *d_zs = tabs.at<int64_t>(o_zs);
  CUDA_TRY(ctx, cudaMemcpyAsync(d_src, offsets, (size_t)n_blocks * 8, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(d_zs, sizes, (size_t)n_blocks * 8, cudaMemcpyHostToDevice, ctx->stream));
  return open_stored_blocks(ctx, img.d, image_size, d_src, d_zs, n_blocks, compressor_type, out);
}

int obgpu_batch_device_image(const obgpu_batch *batch, const void **image, int64_t *image_size) {
  if (!batch || !image || !image_size) return OBGPU_INVALID_ARGUMENT;
  *image = batch->d_image;
  *image_size = batch->image_size;
  return OBGPU_SUCCESS;
}

int obgpu_lz4_decompress(obgpu_ctx *ctx, const void *d_in, const int64_t *in_off, const int64_t *in_len, void *d_out, const int64_t *out_off,
                         const int64_t *out_len, int32_t n, int32_t *status) {
  return decompress_streams(ctx, d_in, in_off, in_len, d_out, out_off, out_len, n, status, OBGPU_COMPRESSOR_LZ4);
}

int obgpu_zstd_decompress(obgpu_ctx *ctx, const void *d_in, const int64_t *in_off, const int64_t *in_len, void *d_out, const int64_t *out_off,
                          const int64_t *out_len, int32_t n, int32_t *status) {
  return decompress_streams(ctx, d_in, in_off, in_len, d_out, out_off, out_len, n, status, OBGPU_COMPRESSOR_ZSTD_1_3_8);
}

int obgpu_zlib_decompress(obgpu_ctx *ctx, const void *d_in, const int64_t *in_off, const int64_t *in_len, void *d_out, const int64_t *out_off,
                          const int64_t *out_len, int32_t n, int32_t *status) {
  return decompress_streams(ctx, d_in, in_off, in_len, d_out, out_off, out_len, n, status, OBGPU_COMPRESSOR_ZLIB);
}

}  // extern "C"
