// zstd-compressed micro-blocks (ObCompressorType 6 "zstd_1.3.8": one plain zstd frame per micro-block payload, what
// ObZstdCompressor_1_3_8::decompress takes apart with ZSTD_decompressDCtx into data_length_ bytes) decoded ON THE DEVICE.
// The open is lz4_blocks.cuh's open_stored_blocks (survey, slots, raw-block realign); this file is the decode step behind it:
// ONE WARP per compressed block, the header checksum and the payload crc32c of the stored bytes first (lz4dev helpers), then
// zstdd::decode_frame (zstd_decode.cuh) with the warp's tables in shared memory. A failed block sets its status; the open
// returns OBGPU_INVALID_DATA and the ctx stays usable.
#pragma once
#include "zstd_decode.cuh"

namespace zstddev {

constexpr int kWarps = 4;   // warps (blocks) per CTA: 4 x 10.75 KiB of tables + the crc table fit the 48 KiB static limit

// BLOCKS = true : micro-blocks (header copied, checksums checked, payload decoded, slot tail zeroed), tables indexed by block
// BLOCKS = false: bare zstd frames in[in_off, + in_len) -> out[out_off, + out_len) (obgpu_zstd_decompress)
template <bool BLOCKS>
__global__ void __launch_bounds__(kWarps * 32) obgpu_zstd_blocks_kernel(const uint8_t *in_base, const int64_t *in_off, const int64_t *in_len,
                                                                       uint8_t *out_base, const int64_t *out_off, const int64_t *out_len,
                                                                       int32_t n, int32_t *blk_status, int32_t *any_status) {
  __shared__ uint32_t tab[256];
  __shared__ zstdd::Work work[kWarps];
  if (BLOCKS) lz4dev::build_crc_table(tab);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t blk = (int64_t)blockIdx.x * kWarps + warp;
  if (blk >= n) return;
  const uint8_t *in = in_base + in_off[blk];
  uint8_t *out = out_base + out_off[blk];
  const int64_t zn = in_len[blk], dn = out_len[blk];
  int32_t st = lz4dev::kStOk;
  if (BLOCKS) {
    const int64_t hs = mb::ld32u(in + 4);   // the survey checked hs >= 64, hs + data_zlength_ == zn, hs + data_length_ == dn
    int32_t ok = 1;
    if (lane == 0) ok = lz4dev::header_checksum_ok(in) ? 1 : 0;
    ok = __shfl_sync(0xffffffffu, ok, 0);
    if (ok) {
      const uint32_t crc = lz4dev::warp_crc32c(tab, in + hs, zn - hs, lane);
      ok = (uint64_t)crc == mb::ld64u(in + 48);
    }
    if (!ok) {
      st = lz4dev::kStBadChecksum;
    } else {
      for (int64_t i = lane; i < hs; i += 32) out[i] = __ldg(in + i);   // the stored header, unchanged
      st = zstdd::decode_frame(in + hs, zn - hs, out + hs, dn - hs, work[warp], lane, 32) == zstdd::kOk ? lz4dev::kStOk
                                                                                                   : lz4dev::kStBadStream;
    }
    __syncwarp();
    const int64_t slot = (dn + 127) & ~127ll;
    for (int64_t i = (st == lz4dev::kStOk ? dn : 0) + lane; i < slot; i += 32) out[i] = 0;   // zero tail (whole slot on failure)
  } else {
    st = zstdd::decode_frame(in, zn, out, dn, work[warp], lane, 32) == zstdd::kOk ? lz4dev::kStOk : lz4dev::kStBadStream;
  }
  if (lane == 0) {
    blk_status[blk] = st;
    if (st != lz4dev::kStOk) atomicMax(any_status, st);
  }
}

}  // namespace zstddev

// the decode launch of open_stored_blocks / decompress_streams for OBGPU_COMPRESSOR_ZSTD_1_3_8
static void launch_zstd_blocks(obgpu_ctx *ctx, bool blocks, const uint8_t *in, const int64_t *in_off, const int64_t *in_len, uint8_t *out,
                               const int64_t *out_off, const int64_t *out_len, int32_t n, int32_t *blk_status, int32_t *any_status) {
  const unsigned grid = (unsigned)((n + zstddev::kWarps - 1) / zstddev::kWarps);
  if (blocks)
    zstddev::obgpu_zstd_blocks_kernel<true><<<grid, zstddev::kWarps * 32, 0, ctx->stream>>>(in, in_off, in_len, out, out_off, out_len, n,
                                                                                            blk_status, any_status);
  else
    zstddev::obgpu_zstd_blocks_kernel<false><<<grid, zstddev::kWarps * 32, 0, ctx->stream>>>(in, in_off, in_len, out, out_off, out_len, n,
                                                                                             blk_status, any_status);
  ctx->launches++;
}

extern "C" int obgpu_zstd_decompress(obgpu_ctx *ctx, const void *d_in, const int64_t *in_off, const int64_t *in_len, void *d_out,
                                     const int64_t *out_off, const int64_t *out_len, int32_t n, int32_t *status) {
  return decompress_streams(ctx, d_in, in_off, in_len, d_out, out_off, out_len, n, status, OBGPU_COMPRESSOR_ZSTD_1_3_8);
}
