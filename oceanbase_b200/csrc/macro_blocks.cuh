// Disk-format bytes straight into the block cache: a run of fixed-size macro blocks (ObMacroBlock, ob_macro_block.cpp:455-520) is
// parsed ON THE DEVICE and re-laid as a page batch. Inside a macro block the micro-blocks lie back to back at arbitrary byte
// offsets; the scan kernels stage blocks with bulk copies (TMA), which need 16-byte aligned sources, so the open path is
//   survey  : one thread per macro block -- ObMacroBlockCommonHeader::check_integrity, FixedHeader::is_valid
//             (ob_macro_block_common_header.cpp:54-69, ob_sstable_macro_block_header.cpp:118-140) -> micro_block_count_
//   walk    : one thread per macro block follows the micro headers (header_size_ + data_zlength_ each) from
//             micro_block_data_offset_; the walk must end at micro_block_data_offset_ + micro_block_data_size_ with row_count_ rows
//   open    : the walk's (offset, stored size) pairs go to open_stored_blocks (stored_blocks.cuh), which copies every raw
//             micro-block to a 128-byte aligned slot of a new image (obgpu_macro_realign_kernel) and decodes the compressed ones
//             (compressor_type_ LZ4 / LZ4_1_9_1 / ZLIB / ZSTD_1_3_8) into theirs -- once per cache fill
// The survey reports each macro block's compressor, and the ones of one open must agree. 16 bytes per micro-block (offset,
// size) and 4 per macro block come back to the host for obgpu_batch_open's tables; the block bytes never touch the CPU. Other
// compressors and encrypted blocks are refused.
#pragma once

namespace mb {

constexpr int32_t kStOk = 0, kStBadCommon = 1, kStBadFixed = 2, kStBadWalk = 3, kStCompressed = 4;

using sb::ld32u;
using sb::ld64u;

struct Fixed {
  int32_t micro_count, data_off, data_size, row_count, compressor;
};

__device__ __forceinline__ int32_t parse_headers(const uint8_t *m, int64_t macro_size, Fixed &f) {
  // ObMacroBlockCommonHeader: header_size_, version_, magic_, attr_, payload_size_, payload_checksum_ (aligned: macro blocks start
  // at multiples of the macro block size)
  const int32_t *c = reinterpret_cast<const int32_t *>(m);
  if (c[0] != 24 || c[1] != 1 || c[2] != 1001 || c[3] != 1 /*SSTableData*/) return kStBadCommon;
  if (c[4] <= 0 || 24 + (int64_t)c[4] > macro_size) return kStBadCommon;
  const uint8_t *h = m + 24;
  const uint32_t version = (uint32_t)h[4] | ((uint32_t)h[5] << 8), magic = (uint32_t)h[6] | ((uint32_t)h[7] << 8);
  const uint64_t tablet = ld64u(h + 8);
  const int64_t logical = (int64_t)ld64u(h + 16);
  const int32_t column_count = (int32_t)ld32u(h + 32), rowkey_cnt = (int32_t)ld32u(h + 36), row_store_type = (int32_t)ld32u(h + 40);
  f.row_count = (int32_t)ld32u(h + 44);
  const int32_t occupy = (int32_t)ld32u(h + 48);
  f.micro_count = (int32_t)ld32u(h + 52);
  f.data_off = (int32_t)ld32u(h + 56);
  f.data_size = (int32_t)ld32u(h + 60);
  const int64_t data_checksum = (int64_t)ld64u(h + 80), encrypt_id = (int64_t)ld64u(h + 88), master_key = (int64_t)ld64u(h + 96);
  const uint32_t compressor = h[104];
  f.compressor = (int32_t)compressor;
  if (!(version >= 1 && version <= 2 && magic == 1007 && tablet != 0 && logical >= 0 && rowkey_cnt >= 0 && row_store_type >= 0 &&
        f.row_count > 0 && occupy > 0 && f.micro_count > 0 && f.data_off > 0 && f.data_size > 0 && data_checksum >= 0 && encrypt_id >= 0 &&
        master_key >= -1 && compressor > 0))
    return kStBadFixed;
  const int64_t type_cols = version == 2 ? rowkey_cnt : column_count;
  if (f.data_off != 24 + 128 + type_cols * 8 + (int64_t)column_count * 8 + 1) return kStBadFixed;
  if ((int64_t)f.data_off + f.data_size > macro_size || occupy != f.data_off + f.data_size) return kStBadFixed;
  if ((int64_t)f.micro_count * 64 > f.data_size) return kStBadFixed;   // a micro-block is at least its 64-byte header
  if (!obf::stored_compressor(f.compressor) || encrypt_id != 0) return kStCompressed;
  return kStOk;
}

__global__ void obgpu_macro_survey_kernel(const uint8_t *image, int64_t macro_size, int32_t n_macro, int32_t *counts, int32_t *comps,
                                          int32_t *status) {
  const int32_t i = (int32_t)(blockIdx.x * blockDim.x + threadIdx.x);
  if (i >= n_macro) return;
  Fixed f;
  const int32_t st = parse_headers(image + (int64_t)i * macro_size, macro_size, f);
  counts[i] = st == kStOk ? f.micro_count : 0;
  comps[i] = st == kStOk ? f.compressor : 0;
  if (st != kStOk) atomicMax(status, st);
}

// first[i]: index of macro block i's first micro-block in the output tables
__global__ void obgpu_macro_walk_kernel(const uint8_t *image, int64_t macro_size, int32_t n_macro, const int64_t *first, int64_t *src_off,
                                        int64_t *sizes, int32_t *status) {
  const int32_t i = (int32_t)(blockIdx.x * blockDim.x + threadIdx.x);
  if (i >= n_macro) return;
  const uint8_t *m = image + (int64_t)i * macro_size;
  Fixed f;
  if (parse_headers(m, macro_size, f) != kStOk) return;
  int64_t at = f.data_off, rows = 0;
  const int64_t end = (int64_t)f.data_off + f.data_size;
  bool ok = true;
  for (int32_t k = 0; k < f.micro_count; ++k) {
    if (at + 64 > end) { ok = false; break; }
    const uint8_t *h = m + at;
    const uint32_t magic = (uint32_t)h[0] | ((uint32_t)h[1] << 8);
    const int64_t sz = (int64_t)ld32u(h + 4) + (int32_t)ld32u(h + 44);   // header_size_ + data_zlength_
    if (magic != 1005u || sz < 64 || at + sz > end) { ok = false; break; }
    if (f.compressor == OBGPU_COMPRESSOR_NONE && ld32u(h + 40) != ld32u(h + 44)) { ok = false; break; }   // NONE: stored raw
    src_off[first[i] + k] = (int64_t)i * macro_size + at;
    sizes[first[i] + k] = sz;
    rows += ld32u(h + 16);
    at += sz;
  }
  if (!ok || at != end || rows != f.row_count) atomicMax(status, kStBadWalk);
}

}  // namespace mb

extern "C" {

int obgpu_batch_open_macro_blocks(obgpu_ctx *ctx, const void *macro_image, int64_t image_size, int64_t macro_block_size, int32_t n_macro_blocks,
                                  int32_t image_on_device, obgpu_batch **out, int32_t *n_micro_out) {
  if (!ctx || !macro_image || !out || n_macro_blocks <= 0 || macro_block_size < 4096 || (macro_block_size & 15) != 0 ||
      image_size < macro_block_size * (int64_t)n_macro_blocks)
    return OBGPU_INVALID_ARGUMENT;
  cudaSetDevice(ctx->device);
  DeviceImage img(ctx);
  int ret = stage_image(ctx, macro_image, image_size, image_on_device, "device-resident macro blocks must be 16-byte aligned", img);
  if (ret != OBGPU_SUCCESS) return ret;
  const uint8_t *d_macro = img.d;
  std::vector<int32_t> counts((size_t)n_macro_blocks + 1), comps((size_t)n_macro_blocks);
  std::vector<int64_t> first((size_t)n_macro_blocks + 1);
  int64_t n_micro = 0;
  // [counts i32 x n][status i32][first i64 x (n + 1), 16-byte aligned by the padding of the counts][compressor i32 x n]
  Scratch small(ctx);
  const size_t o_counts = small.take(((size_t)n_macro_blocks + 1) * 4, 16), o_first = small.take(((size_t)n_macro_blocks + 1) * 8, 8);
  const size_t o_comps = small.take((size_t)n_macro_blocks * 4 + 64, 4);
  CUDA_TRY(ctx, small.alloc());
  int32_t *d_counts = small.at<int32_t>(o_counts), *d_status = d_counts + n_macro_blocks;
  int64_t *d_first = small.at<int64_t>(o_first);
  int32_t *d_comps = small.at<int32_t>(o_comps);
  CUDA_TRY(ctx, cudaMemsetAsync(d_status, 0, 4, ctx->stream));
  mb::obgpu_macro_survey_kernel<<<(unsigned)((n_macro_blocks + 127) / 128), 128, 0, ctx->stream>>>(d_macro, macro_block_size, n_macro_blocks, d_counts,
                                                                                                   d_comps, d_status);
  ctx->launches++;
  CUDA_TRY(ctx, cudaMemcpyAsync(counts.data(), d_counts, ((size_t)n_macro_blocks + 1) * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(comps.data(), d_comps, (size_t)n_macro_blocks * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (counts[(size_t)n_macro_blocks] != mb::kStOk) {
    const bool compressed = counts[(size_t)n_macro_blocks] == mb::kStCompressed;
    ctx->err = compressed ? "compressed or encrypted macro block" : "macro block header is invalid";
    return compressed ? OBGPU_NOT_SUPPORTED : OBGPU_INVALID_DATA;
  }
  // one SSTable has one compressor: the macro blocks that are not NONE must agree (NONE ones hold raw blocks only)
  int32_t compressor = OBGPU_COMPRESSOR_NONE;
  bool mixed = false;
  for (int32_t c : comps)
    if (c != OBGPU_COMPRESSOR_NONE) {
      mixed = mixed || (compressor != OBGPU_COMPRESSOR_NONE && c != compressor);
      compressor = c;
    }
  if (mixed) {
    ctx->err = "macro blocks of one open use different compressors";
    return OBGPU_NOT_SUPPORTED;
  }
  for (int32_t i = 0; i < n_macro_blocks; ++i) { first[(size_t)i] = n_micro; n_micro += counts[(size_t)i]; }
  first[(size_t)n_macro_blocks] = n_micro;
  if (n_micro <= 0 || n_micro > 0x7fffffff) {
    ctx->err = "macro blocks hold no micro-block";
    return OBGPU_INVALID_DATA;
  }
  Scratch tab(ctx);   // [src][sizes]
  const size_t o_src = tab.take((size_t)n_micro * 8, 8), o_sizes = tab.take((size_t)n_micro * 8 + 64, 8);
  CUDA_TRY(ctx, tab.alloc());
  int64_t *d_src = tab.at<int64_t>(o_src), *d_sizes = tab.at<int64_t>(o_sizes);
  CUDA_TRY(ctx, cudaMemcpyAsync(d_first, first.data(), ((size_t)n_macro_blocks + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
  mb::obgpu_macro_walk_kernel<<<(unsigned)((n_macro_blocks + 63) / 64), 64, 0, ctx->stream>>>(d_macro, macro_block_size, n_macro_blocks, d_first, d_src, d_sizes, d_status);
  ctx->launches++;
  int32_t st = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&st, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (st != mb::kStOk) {
    ctx->err = "micro-block chain of a macro block is inconsistent";
    return OBGPU_INVALID_DATA;
  }
  // NONE macro blocks were checked by the walk (every block raw); the others admit raw and compressed blocks alike
  obgpu_batch *b = nullptr;
  ret = open_stored_blocks(ctx, d_macro, image_size, d_src, d_sizes, (int32_t)n_micro, compressor, &b);
  if (ret != OBGPU_SUCCESS) return ret;
  *out = b;
  if (n_micro_out) *n_micro_out = (int32_t)n_micro;
  return OBGPU_SUCCESS;
}

}  // extern "C"
