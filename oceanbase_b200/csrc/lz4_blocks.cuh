// LZ4-compressed micro-blocks decoded ON THE DEVICE when a page batch or a run of macro blocks is opened
// (ObMacroBlockReader::decompress_data -> ObLZ4Compressor::decompress, one micro-block at a time on the CPU in the reference).
// On disk a micro-block is [ObMicroBlockHeader, plain][payload compressed on its own]: data_zlength_ bytes stored,
// data_length_ bytes after decoding, data_checksum_ = crc32c of the STORED payload. A block whose payload did not shrink is
// stored raw (data_zlength_ == data_length_). Opening such blocks is
//   survey  : one thread per block -- magic, header_size_, header_size_ + data_zlength_ == stored size -> decoded size, raw or not
//   slots   : host prefix over the decoded sizes, 128-byte aligned slots (the layout obgpu_macro_realign_kernel produces)
//   copy    : raw blocks go through obgpu_macro_realign_kernel
//   decode  : compressed blocks, ONE WARP per block (obgpu_lz4_blocks_kernel):
//             header checksum (lane 0) and payload crc32c over the stored bytes (every lane the raw CRC of a contiguous chunk,
//             shifted into place by a carry-less multiplication with x^(8 * bytes after it), XOR-reduced -- enc::gf2_mulmod /
//             enc::crc_byte of the device encoder), then the LZ4 sequences: every lane reads the token; length extensions are
//             read 32 bytes at a time and the first byte != 255 found with a ballot; literals move 32 bytes per step; a match at
//             distance d is fully parallel even when it overlaps, out[pos + i] = out[pos - d + (i mod d)], because every source
//             byte precedes pos. The output goes straight to the block's slot in global memory (matches read it back through
//             L1); the slot's tail up to 128 bytes is zeroed.
//   open    : obgpu_batch_open(image_on_device = 1, header_view = NULL) over the decoded image, which the batch then owns
// The decoder is the boundary for bytes from outside the program: every read is checked against the stored extent, every
// write against data_length_; 1 <= offset <= bytes produced; the format's end-of-block rules (a sequence that is not the
// last leaves >= 12 output and >= 8 input bytes after its literals, a match ends >= 5 bytes before the end, >= 5 input bytes
// follow a match length); the last sequence ends exactly at data_zlength_ and the output is exactly data_length_ bytes.
// A failed block sets its status; the open returns OBGPU_INVALID_DATA and the ctx stays usable.
#pragma once

namespace lz4dev {

constexpr int kWarps = 4;   // warps (blocks) per CTA
constexpr int32_t kStOk = 0, kStBadHeader = 1, kStBadStream = 2, kStBadChecksum = 3;

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

// LZ4 length extension at in[ip]: bytes of 255 continue it. false: it runs past the input.
__device__ __forceinline__ bool read_ext(const uint8_t *in, int64_t n_in, int64_t &ip, int64_t &len, int lane) {
  for (;;) {
    const int64_t p = ip + lane;
    const bool valid = p < n_in;
    const uint32_t v = valid ? __ldg(in + p) : 0u;
    const unsigned stop = __ballot_sync(0xffffffffu, !valid || v != 255u);
    if (stop == 0u) {
      ip += 32;
      len += 255 * 32;
      continue;
    }
    const int f = __ffs(stop) - 1;
    if (ip + f >= n_in) return false;
    len += 255 * (int64_t)f + __shfl_sync(0xffffffffu, v, f);
    ip += f + 1;
    return true;
  }
}

// One LZ4 block in[0, n_in) -> out[0, n_out) by the warp; kStOk only when the stream decodes to exactly n_out bytes.
__device__ __forceinline__ int32_t warp_lz4_decode(const uint8_t *in, int64_t n_in, uint8_t *out, int64_t n_out, int lane) {
  int64_t ip = 0, op = 0;
  for (;;) {
    if (ip >= n_in) return kStBadStream;
    const uint32_t token = __ldg(in + ip);
    ++ip;
    int64_t lit = token >> 4;
    if (lit == 15 && !read_ext(in, n_in, ip, lit, lane)) return kStBadStream;
    if (lit > n_in - ip || lit > n_out - op) return kStBadStream;
    const bool last = ip + lit == n_in;
    if (!last && (op + lit > n_out - 12 || ip + lit > n_in - 8)) return kStBadStream;
    for (int64_t i = lane; i < lit; i += 32) out[op + i] = __ldg(in + ip + i);
    ip += lit;
    op += lit;
    if (last) break;
    const int64_t offset = (int64_t)__ldg(in + ip) | ((int64_t)__ldg(in + ip + 1) << 8);
    ip += 2;
    int64_t mlen = token & 15u;
    if (mlen == 15 && !read_ext(in, n_in, ip, mlen, lane)) return kStBadStream;
    mlen += 4;
    if (ip > n_in - 5) return kStBadStream;
    if (offset == 0 || offset > op || mlen > n_out - 5 - op) return kStBadStream;
    __syncwarp();   // the literals (and earlier matches) written by other lanes are visible
    const uint8_t *src = out + op - offset;
    for (int64_t i = lane; i < mlen; i += 32) out[op + i] = src[i < offset ? (uint32_t)i : (uint32_t)i % (uint32_t)offset];   // offset < 2^16, mlen < 2^31
    __syncwarp();
    op += mlen;
  }
  return op == n_out ? kStOk : kStBadStream;
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

// ObMicroBlockHeader::check_header_checksum (ob_micro_block_header.cpp:236-262): the fold including the stored checksum is 0
__device__ bool header_checksum_ok(const uint8_t *h) {
  uint32_t cs = 0;
  auto half = [&](int off) { return (uint32_t)__ldg(h + off) | ((uint32_t)__ldg(h + off + 1) << 8); };
  auto f32 = [&](uint32_t v) { cs ^= (v & 0xffffu) ^ (v >> 16); };
  auto f64 = [&](uint64_t v) { cs ^= (uint32_t)(v & 0xffffu) ^ (uint32_t)((v >> 16) & 0xffffu) ^ (uint32_t)((v >> 32) & 0xffffu) ^ (uint32_t)(v >> 48); };
  auto i32 = [&](int off) { return (uint64_t)(int64_t)(int32_t)mb::ld32u(h + off); };
  cs ^= half(0) ^ half(2) ^ half(8);
  cs ^= (uint32_t)__ldg(h + 20) ^ (uint32_t)__ldg(h + 21);
  f32(half(10)); f32(half(12)); f32(half(14) & 1u); f32(half(22));
  f64(mb::ld32u(h + 4)); f64(mb::ld32u(h + 16)); f64(mb::ld32u(h + 24)); f64(i32(28)); f64(mb::ld64u(h + 32));
  f64(i32(40)); f64(i32(44)); f64(mb::ld64u(h + 48));
  return (cs & 0xffffu) == 0u;
}

// survey of stored micro-blocks: dsize[i] = header_size_ + data_length_, kind[i] = 1 when compressed; *status = max verdict
__global__ void obgpu_lz4_survey_kernel(const uint8_t *image, const int64_t *src_off, const int64_t *zsize, int32_t n, int32_t compressor,
                                        int64_t *dsize, int32_t *kind, int32_t *status) {
  const int32_t i = (int32_t)(blockIdx.x * blockDim.x + threadIdx.x);
  if (i >= n) return;
  const uint8_t *h = image + src_off[i];
  const uint32_t magic = (uint32_t)h[0] | ((uint32_t)h[1] << 8);
  const int64_t hs = mb::ld32u(h + 4);
  const int64_t len = (int32_t)mb::ld32u(h + 40), zlen = (int32_t)mb::ld32u(h + 44);
  int32_t st = kStOk;
  if (magic != 1005u || hs < 64 || len <= 0 || zlen <= 0 || hs + zlen != zsize[i] || hs + len > 0x7fffffffll) st = kStBadHeader;
  else if (zlen != len && compressor == OBGPU_COMPRESSOR_NONE) st = kStBadHeader;   // a NONE table stores every block raw
  dsize[i] = st == kStOk ? hs + len : 0;
  kind[i] = st == kStOk && zlen != len ? 1 : 0;
  if (st != kStOk) atomicMax(status, st);
}

// BLOCKS = true : micro-blocks (header copied, checksums checked, payload decoded, slot tail zeroed), tables indexed by block
// BLOCKS = false: bare LZ4 streams in[in_off, + in_len) -> out[out_off, + out_len) (obgpu_lz4_decompress)
template <bool BLOCKS>
__global__ void __launch_bounds__(kWarps * 32) obgpu_lz4_blocks_kernel(const uint8_t *in_base, const int64_t *in_off, const int64_t *in_len,
                                                                      uint8_t *out_base, const int64_t *out_off, const int64_t *out_len,
                                                                      int32_t n, int32_t *blk_status, int32_t *any_status) {
  __shared__ uint32_t tab[256];
  if (BLOCKS) build_crc_table(tab);
  const int lane = threadIdx.x & 31;
  const int64_t blk = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (blk >= n) return;
  const uint8_t *in = in_base + in_off[blk];
  uint8_t *out = out_base + out_off[blk];
  const int64_t zn = in_len[blk], dn = out_len[blk];
  int32_t st = kStOk;
  if (BLOCKS) {
    const int64_t hs = mb::ld32u(in + 4);   // the survey checked hs >= 64, hs + data_zlength_ == zn, hs + data_length_ == dn
    int32_t ok = 1;
    if (lane == 0) ok = header_checksum_ok(in) ? 1 : 0;
    ok = __shfl_sync(0xffffffffu, ok, 0);
    if (ok) {
      const uint32_t crc = warp_crc32c(tab, in + hs, zn - hs, lane);
      ok = (uint64_t)crc == mb::ld64u(in + 48);
    }
    if (!ok) {
      st = kStBadChecksum;
    } else {
      for (int64_t i = lane; i < hs; i += 32) out[i] = __ldg(in + i);   // the stored header, unchanged
      st = warp_lz4_decode(in + hs, zn - hs, out + hs, dn - hs, lane);
    }
    const int64_t slot = (dn + 127) & ~127ll;
    for (int64_t i = (st == kStOk ? dn : 0) + lane; i < slot; i += 32) out[i] = 0;   // zero tail (whole slot on failure)
  } else {
    st = warp_lz4_decode(in, zn, out, dn, lane);
  }
  if (lane == 0) {
    blk_status[blk] = st;
    if (st != kStOk) atomicMax(any_status, st);
  }
}

}  // namespace lz4dev

static void launch_zstd_blocks(obgpu_ctx *ctx, bool blocks, const uint8_t *in, const int64_t *in_off, const int64_t *in_len, uint8_t *out,
                               const int64_t *out_off, const int64_t *out_len, int32_t n, int32_t *blk_status,
                               int32_t *any_status);   // zstd_blocks.cuh

static void launch_decode(obgpu_ctx *ctx, int32_t compressor, bool blocks, const uint8_t *in, const int64_t *in_off, const int64_t *in_len,
                          uint8_t *out, const int64_t *out_off, const int64_t *out_len, int32_t n, int32_t *blk_status, int32_t *any_status) {
  if (compressor == OBGPU_COMPRESSOR_ZSTD_1_3_8) {
    launch_zstd_blocks(ctx, blocks, in, in_off, in_len, out, out_off, out_len, n, blk_status, any_status);
    return;
  }
  const unsigned grid = (unsigned)((n + lz4dev::kWarps - 1) / lz4dev::kWarps);
  if (blocks)
    lz4dev::obgpu_lz4_blocks_kernel<true><<<grid, lz4dev::kWarps * 32, 0, ctx->stream>>>(in, in_off, in_len, out, out_off, out_len, n,
                                                                                        blk_status, any_status);
  else
    lz4dev::obgpu_lz4_blocks_kernel<false><<<grid, lz4dev::kWarps * 32, 0, ctx->stream>>>(in, in_off, in_len, out, out_off, out_len, n,
                                                                                         blk_status, any_status);
  ctx->launches++;
}

static bool device_compressor(int32_t c) {
  return c == OBGPU_COMPRESSOR_NONE || c == OBGPU_COMPRESSOR_LZ4 || c == OBGPU_COMPRESSOR_LZ4_1_9_1 || c == OBGPU_COMPRESSOR_ZSTD_1_3_8;
}

// Stored micro-blocks d_image[d_src[i], + d_zsize[i]) (device tables) -> page batch owning the decoded, realigned image.
// The one routine behind obgpu_batch_open_macro_blocks and obgpu_batch_open_compressed.
static int open_stored_blocks(obgpu_ctx *ctx, const uint8_t *d_image, int64_t image_size, const int64_t *d_src, const int64_t *d_zsize,
                              int32_t n, int32_t compressor, obgpu_batch **out) {
  int ret = OBGPU_SUCCESS;
  void *d_work = nullptr, *d_tab = nullptr, *d_out = nullptr;
  auto fail = [&](int code, const char *what) { ctx->err = what; ret = code; };
  std::vector<int64_t> src((size_t)n), zsize((size_t)n), dsize((size_t)n), dst((size_t)n);
  std::vector<int32_t> kind((size_t)n);
  do {
    // [dsize i64 x n][kind i32 x n][status i32]
    if (cudaMallocAsync(&d_work, (size_t)n * 12 + 64, ctx->stream) != cudaSuccess) { fail(OBGPU_ALLOCATE_MEMORY_FAILED, "stored-block survey tables"); break; }
    int64_t *d_dsize = (int64_t *)d_work;
    int32_t *d_kind = (int32_t *)(d_dsize + n), *d_status = d_kind + n;
    cudaMemsetAsync(d_status, 0, 4, ctx->stream);
    lz4dev::obgpu_lz4_survey_kernel<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(d_image, d_src, d_zsize, n, compressor, d_dsize,
                                                                                           d_kind, d_status);
    ctx->launches++;
    int32_t st = 0;
    if (cudaMemcpyAsync(dsize.data(), d_dsize, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
        cudaMemcpyAsync(kind.data(), d_kind, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
        cudaMemcpyAsync(&st, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
        cudaMemcpyAsync(src.data(), d_src, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
        cudaMemcpyAsync(zsize.data(), d_zsize, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
        cudaStreamSynchronize(ctx->stream) != cudaSuccess) { fail(OBGPU_ERR_SYS, "stored-block survey"); break; }
    if (st != lz4dev::kStOk) { fail(OBGPU_INVALID_DATA, "micro-block header of a stored block is invalid"); break; }
    // slots + the two work lists: raw -> realign copy, compressed -> decoder
    int64_t out_bytes = 0;
    std::vector<int64_t> raw_tab, lz_tab;   // raw: [src][size][dst], compressed: [src][zsize][dst][dsize]
    std::vector<int32_t> raw_idx, lz_idx;
    for (int32_t i = 0; i < n; ++i) {
      dst[(size_t)i] = out_bytes;
      out_bytes += (dsize[(size_t)i] + 127) & ~127ll;
      (kind[(size_t)i] ? lz_idx : raw_idx).push_back(i);
    }
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
    if (cudaMallocAsync(&d_out, (size_t)out_bytes + 64, ctx->stream) != cudaSuccess) { fail(OBGPU_ALLOCATE_MEMORY_FAILED, "decoded image"); break; }
    cudaMemsetAsync((uint8_t *)d_out + out_bytes, 0, 64, ctx->stream);
    const size_t tab_bytes = (nr * 3 + nz * 4) * 8 + nz * 4 + 64;
    if (cudaMallocAsync(&d_tab, tab_bytes, ctx->stream) != cudaSuccess) { fail(OBGPU_ALLOCATE_MEMORY_FAILED, "stored-block tables"); break; }
    int64_t *d_raw = (int64_t *)d_tab, *d_lz = d_raw + nr * 3;
    int32_t *d_blk_status = (int32_t *)(d_lz + nz * 4);
    if (nr) cudaMemcpyAsync(d_raw, raw_tab.data(), nr * 24, cudaMemcpyHostToDevice, ctx->stream);
    if (nz) cudaMemcpyAsync(d_lz, lz_tab.data(), nz * 32, cudaMemcpyHostToDevice, ctx->stream);
    cudaMemsetAsync(d_status, 0, 4, ctx->stream);
    if (nr) {
      mb::obgpu_macro_realign_kernel<<<(unsigned)nr, mb::kCopyThreads, 0, ctx->stream>>>(d_image, image_size, d_raw, d_raw + nr, d_raw + 2 * nr,
                                                                                         (uint8_t *)d_out);
      ctx->launches++;
    }
    if (nz)
      launch_decode(ctx, compressor, true, d_image, d_lz, d_lz + nz, (uint8_t *)d_out, d_lz + 2 * nz, d_lz + 3 * nz, (int32_t)nz, d_blk_status,
                    d_status);
    // the host tables were copy sources: synchronise before they go out of scope
    if (cudaGetLastError() != cudaSuccess || cudaMemcpyAsync(&st, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
        cudaStreamSynchronize(ctx->stream) != cudaSuccess) { fail(OBGPU_ERR_SYS, "stored-block decode"); break; }
    if (st != lz4dev::kStOk) {
      fail(OBGPU_INVALID_DATA, st == lz4dev::kStBadChecksum ? "checksum of a compressed micro-block does not match"
                               : compressor == OBGPU_COMPRESSOR_ZSTD_1_3_8 ? "zstd payload of a micro-block is malformed"
                                                                           : "LZ4 payload of a micro-block is malformed");
      break;
    }
    obgpu_batch *b = nullptr;
    ret = obgpu_batch_open(ctx, d_out, out_bytes, dst.data(), dsize.data(), n, 1, nullptr, &b);
    if (ret != OBGPU_SUCCESS) break;
    b->own_image = true;   // the decoded image lives and dies with the batch
    d_out = nullptr;
    *out = b;
  } while (0);
  if (d_work) cudaFreeAsync(d_work, ctx->stream);
  if (d_tab) cudaFreeAsync(d_tab, ctx->stream);
  if (d_out) cudaFreeAsync(d_out, ctx->stream);
  return ret;
}

extern "C" {

int obgpu_batch_open_compressed(obgpu_ctx *ctx, const void *image, int64_t image_size, const int64_t *offsets, const int64_t *sizes,
                                int32_t n_blocks, int32_t image_on_device, int32_t compressor_type, obgpu_batch **out) {
  if (!ctx || !image || !offsets || !sizes || !out || n_blocks <= 0 || image_size <= 0) return OBGPU_INVALID_ARGUMENT;
  if (!device_compressor(compressor_type)) {
    ctx->err = "compressor not handled by the device path";
    return OBGPU_NOT_SUPPORTED;
  }
  for (int32_t i = 0; i < n_blocks; ++i)
    if (offsets[i] < 0 || sizes[i] < 64 || offsets[i] + sizes[i] > image_size) {
      ctx->err = "stored block outside the image";
      return OBGPU_INVALID_ARGUMENT;
    }
  if (image_on_device && ((uintptr_t)image & 15u) != 0) {
    ctx->err = "a device-resident image must be 16-byte aligned";
    return OBGPU_INVALID_ARGUMENT;
  }
  cudaSetDevice(ctx->device);
  const uint8_t *d_img = (const uint8_t *)image;
  void *tmp_image = nullptr, *d_tabs = nullptr;
  int ret = OBGPU_SUCCESS;
  do {
    if (!image_on_device) {
      if (cudaMallocAsync(&tmp_image, (size_t)image_size, ctx->stream) != cudaSuccess) { ctx->err = "image copy"; ret = OBGPU_ALLOCATE_MEMORY_FAILED; break; }
      if (cudaMemcpyAsync(tmp_image, image, (size_t)image_size, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) {
        ctx->err = "image copy";
        ret = OBGPU_ERR_SYS;
        break;
      }
      d_img = (const uint8_t *)tmp_image;
    }
    if (cudaMallocAsync(&d_tabs, (size_t)n_blocks * 16, ctx->stream) != cudaSuccess) { ctx->err = "block tables"; ret = OBGPU_ALLOCATE_MEMORY_FAILED; break; }
    int64_t *d_src = (int64_t *)d_tabs, *d_zs = d_src + n_blocks;
    if (cudaMemcpyAsync(d_src, offsets, (size_t)n_blocks * 8, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess ||
        cudaMemcpyAsync(d_zs, sizes, (size_t)n_blocks * 8, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) {
      ctx->err = "block tables";
      ret = OBGPU_ERR_SYS;
      break;
    }
    ret = open_stored_blocks(ctx, d_img, image_size, d_src, d_zs, n_blocks, compressor_type, out);
  } while (0);
  if (d_tabs) cudaFreeAsync(d_tabs, ctx->stream);
  if (tmp_image) cudaFreeAsync(tmp_image, ctx->stream);
  return ret;
}

int obgpu_batch_device_image(const obgpu_batch *batch, const void **image, int64_t *image_size) {
  if (!batch || !image || !image_size) return OBGPU_INVALID_ARGUMENT;
  *image = batch->d_image;
  *image_size = batch->image_size;
  return OBGPU_SUCCESS;
}

}  // extern "C"

// n independent streams of one codec in device memory (obgpu_lz4_decompress, obgpu_zstd_decompress)
static int decompress_streams(obgpu_ctx *ctx, const void *d_in, const int64_t *in_off, const int64_t *in_len, void *d_out, const int64_t *out_off,
                              const int64_t *out_len, int32_t n, int32_t *status, int32_t compressor) {
  if (!ctx || !d_in || !in_off || !in_len || !d_out || !out_off || !out_len || n <= 0 || !status) return OBGPU_INVALID_ARGUMENT;
  for (int32_t i = 0; i < n; ++i)
    if (in_off[i] < 0 || in_len[i] < 0 || out_off[i] < 0 || out_len[i] < 0) return OBGPU_INVALID_ARGUMENT;
  cudaSetDevice(ctx->device);
  void *d_tab = nullptr;
  int ret = OBGPU_SUCCESS;
  std::vector<int64_t> tab((size_t)n * 4);
  memcpy(tab.data(), in_off, (size_t)n * 8);
  memcpy(tab.data() + n, in_len, (size_t)n * 8);
  memcpy(tab.data() + 2 * (size_t)n, out_off, (size_t)n * 8);
  memcpy(tab.data() + 3 * (size_t)n, out_len, (size_t)n * 8);
  do {
    if (cudaMallocAsync(&d_tab, (size_t)n * 36 + 64, ctx->stream) != cudaSuccess) { ctx->err = "stream tables"; ret = OBGPU_ALLOCATE_MEMORY_FAILED; break; }
    int64_t *d = (int64_t *)d_tab;
    int32_t *d_st = (int32_t *)(d + 4 * (size_t)n), *d_any = d_st + n;
    cudaMemcpyAsync(d, tab.data(), (size_t)n * 32, cudaMemcpyHostToDevice, ctx->stream);
    cudaMemsetAsync(d_any, 0, 4, ctx->stream);
    launch_decode(ctx, compressor, false, (const uint8_t *)d_in, d, d + n, (uint8_t *)d_out, d + 2 * n, d + 3 * n, n, d_st, d_any);
    int32_t any = 0;
    if (cudaGetLastError() != cudaSuccess || cudaMemcpyAsync(status, d_st, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
        cudaMemcpyAsync(&any, d_any, 4, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
        cudaStreamSynchronize(ctx->stream) != cudaSuccess) { ctx->err = "stream decode"; ret = OBGPU_ERR_SYS; break; }
    if (any != lz4dev::kStOk) {
      ctx->err = compressor == OBGPU_COMPRESSOR_ZSTD_1_3_8 ? "a zstd frame is malformed" : "an LZ4 block is malformed";
      ret = OBGPU_INVALID_DATA;
    }
  } while (0);
  if (d_tab) cudaFreeAsync(d_tab, ctx->stream);
  return ret;
}

extern "C" {

int obgpu_lz4_decompress(obgpu_ctx *ctx, const void *d_in, const int64_t *in_off, const int64_t *in_len, void *d_out, const int64_t *out_off,
                         const int64_t *out_len, int32_t n, int32_t *status) {
  return decompress_streams(ctx, d_in, in_off, in_len, d_out, out_off, out_len, n, status, OBGPU_COMPRESSOR_LZ4);
}

}  // extern "C"
