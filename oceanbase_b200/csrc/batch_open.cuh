// Opening a page batch (obgpu_batch_open). Every block's header passes obf::check_micro_header, read from a host view of the
// blocks or, for a device-resident image opened without one, by obgpu_survey_kernel. Two open-time rewrites then give the batch an
// image every scan kernel reads as it is:
//   cs_restate_batch      : CS blocks with non-RAW integer streams -> RAW restatement (stream_codecs.cuh)
//   pax_materialise_batch : PAX columns whose strings are rebuilt -> strings materialised behind the block (mat_codecs.cuh)
// Each rewrite is survey_fetch (per-block survey records to the host), slot_layout (128-byte slots of the new image), its own
// kernels and install_image (the batch takes the new image). open_stored_blocks (stored_blocks.cuh) lays out its decoded image
// with slot_layout and opens it here. Last, obgpu_index_kernel builds the decode plans.
// Errors return at once; obgpu_batch_open closes the batch, which owns everything allocated so far, on any failure.
#pragma once

// Header survey of a device-resident image opened without a host view: one thread per block reports
// {row count, column count | obf::check_micro_header verdict << 16}.
__global__ void __launch_bounds__(256) obgpu_survey_kernel(const uint8_t *image, const uint64_t *blk_off, const uint32_t *blk_size,
                                                           int n_blocks, uint32_t *out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_blocks) return;
  obf::MicroHeaderFacts f;
  const uint32_t verdict = obf::check_micro_header(image + blk_off[i], blk_size[i], f);
  out[2 * i] = f.rows;
  out[2 * i + 1] = f.ncol | (verdict << 16);
}

// Survey fetch: allocates `bytes` of device records and clears the first zero_bytes, enqueues `launch(d_rec)` (one per-block survey
// kernel writing them), copies out.size() records back into `out` and synchronises once.
template <class R, class Launch>
static int survey_fetch(obgpu_ctx *ctx, size_t bytes, size_t zero_bytes, std::vector<R> &out, Launch launch) {
  Scratch rec(ctx);
  CUDA_TRY(ctx, rec.alloc(bytes));
  if (zero_bytes) CUDA_TRY(ctx, cudaMemsetAsync(rec.p, 0, zero_bytes, ctx->stream));
  launch(rec.at<uint32_t>(0));
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  CUDA_TRY(ctx, cudaMemcpyAsync(out.data(), rec.p, out.size() * sizeof(R), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return OBGPU_SUCCESS;
}

// Slot layout of a rewritten image: block i at off[i], in a slot of size[i] bytes rounded up to 128. Returns the image's bytes.
template <class Size, class Off>
static uint64_t slot_layout(const Size *size, int32_t n, Off *off) {
  uint64_t pos = 0;
  for (int32_t i = 0; i < n; ++i) {
    off[i] = (Off)pos;
    pos += ((uint64_t)size[i] + 127) & ~127ull;
  }
  return pos;
}

// Install: the batch takes the allocation of `img`, a rewritten image of `bytes` bytes, with block i at off[i] and size[i] bytes
// long. Enqueues the uploads of the device block tables and frees the image the batch owned before once the stream is past it.
static int install_image(obgpu_ctx *ctx, obgpu_batch *b, Scratch &img, uint64_t bytes, const uint64_t *off, const uint32_t *size) {
  const int32_t n = b->n_blocks;
  CUDA_TRY(ctx, cudaMemcpyAsync(b->d_blk_off, off, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(b->d_blk_size, size, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
  if (b->own_image && b->d_image) cudaFreeAsync((void *)b->d_image, ctx->stream);
  b->d_image = (const uint8_t *)img.release();
  b->own_image = true;
  b->image_size = (int64_t)bytes;
  b->max_block_bytes = 0;
  for (int32_t i = 0; i < n; ++i) {
    b->offsets[(size_t)i] = (int64_t)off[i];
    b->sizes[(size_t)i] = size[i];
    b->max_block_bytes = std::max<uint32_t>(b->max_block_bytes, (size[i] + 15u) & ~15u);
  }
  return OBGPU_SUCCESS;
}

// CS blocks with non-RAW integer streams -> a RAW restatement of the batch's image (stream_codecs.cuh), in place of
// the caller's image for every later kernel. Runs on the ctx stream after the image is resident; synchronises.
static int cs_restate_batch(obgpu_ctx *ctx, obgpu_batch *b) {
  const int32_t n = b->n_blocks;
  std::vector<uint32_t> sv((size_t)n * 4);
  int ret = survey_fetch(ctx, (size_t)n * 16, 0, sv, [&](uint32_t *d_sv) {
    obcs::cs_survey_kernel<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(b->d_image, b->d_blk_off, b->d_blk_size, n, d_sv);
  });
  if (ret != OBGPU_SUCCESS) return ret;
  bool any = false;
  for (int32_t i = 0; i < n; ++i) {
    const uint32_t flags = sv[(size_t)4 * i + 2];
    if (flags & obcs::XF_CORRUPT) { ctx->err = "corrupt CS micro block (stream layout)"; return OBGPU_INVALID_DATA; }
    if (flags & obcs::XF_UNSUPPORTED) continue;   // the index kernel marks the plans of such blocks unsupported: scans say OB_NOT_SUPPORTED
    any = any || (flags & obcs::XF_NONRAW);
  }
  if (!any) return OBGPU_SUCCESS;
  // layout of the restated image and of the job / scratch tables
  std::vector<uint64_t> tab((size_t)n * 3);   // [new_off][job_base][scratch_base]
  std::vector<uint32_t> nsz((size_t)n);
  uint64_t jobs = 0, scr = 0;
  for (int32_t i = 0; i < n; ++i) {
    const bool bad = (sv[(size_t)4 * i + 2] & obcs::XF_UNSUPPORTED) != 0;
    nsz[(size_t)i] = bad ? (uint32_t)b->sizes[(size_t)i] : sv[(size_t)4 * i];
    tab[(size_t)n + i] = jobs;
    tab[(size_t)2 * n + i] = scr;
    jobs += bad ? 0 : sv[(size_t)4 * i + 1];
    scr += 4ull * sv[(size_t)4 * i + 3];
  }
  const uint64_t pos = slot_layout(nsz.data(), n, tab.data());
  Scratch img(ctx), scratch(ctx), tabs(ctx), sizes(ctx), job_list(ctx), status(ctx);
  CUDA_TRY(ctx, img.alloc((size_t)pos + 64));
  CUDA_TRY(ctx, scratch.alloc((size_t)scr + 16));
  CUDA_TRY(ctx, tabs.alloc((size_t)n * 24));
  CUDA_TRY(ctx, sizes.alloc((size_t)n * 4));
  CUDA_TRY(ctx, job_list.alloc((size_t)(jobs + 1) * sizeof(obcs::StreamJob)));
  CUDA_TRY(ctx, status.alloc(16));
  CUDA_TRY(ctx, cudaMallocAsync((void **)&b->d_xf, (size_t)n * sizeof(obcs::XformRec), ctx->stream));
  uint8_t *d_new = img.p;
  uint64_t *d_tab = tabs.at<uint64_t>(0);
  uint32_t *d_nsz = sizes.at<uint32_t>(0);
  obcs::StreamJob *d_jobs = job_list.at<obcs::StreamJob>(0);
  int *d_status = status.at<int>(0);
  CUDA_TRY(ctx, cudaMemsetAsync(d_status, 0, 16, ctx->stream));
  CUDA_TRY(ctx, cudaMemsetAsync(d_new, 0, (size_t)pos + 64, ctx->stream));   // block padding and tail slack read as zero
  CUDA_TRY(ctx, cudaMemcpyAsync(d_tab, tab.data(), (size_t)n * 24, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(d_nsz, nsz.data(), (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
  obcs::cs_rewrite_kernel<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(b->d_image, b->d_blk_off, b->d_blk_size, n, d_new, d_tab, d_nsz,
                                                                            d_tab + n, d_jobs, scratch.p, d_tab + 2 * (size_t)n, b->d_xf, d_status);
  if (jobs > 0)
    obcs::cs_decode_kernel<<<(unsigned)((jobs + 127) / 128), 128, 0, ctx->stream>>>(b->d_image, d_new, d_jobs, (int64_t)jobs, d_status);
  ctx->launches += jobs > 0 ? 2 : 1;
  CUDA_TRY(ctx, cudaGetLastError());
  int st = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&st, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
  if ((ret = install_image(ctx, b, img, pos, tab.data(), nsz.data())) != OBGPU_SUCCESS) return ret;
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (st != 0) {
    ctx->err = "CS integer stream does not decode (corrupt or unsupported codec)";
    return (st & obcs::XF_CORRUPT) ? OBGPU_INVALID_DATA : OBGPU_NOT_SUPPORTED;
  }
  return OBGPU_SUCCESS;
}

// PAX blocks with HEX_PACKING / STRING_DIFF / STRING_PREFIX columns -> a copy of the batch's image in which every such column has
// its strings materialised behind the block (mat_codecs.cuh). Runs after cs_restate_batch (the two compose: a batch may hold both
// kinds of blocks); synchronises.
static int pax_materialise_batch(obgpu_ctx *ctx, obgpu_batch *b) {
  const int32_t n = b->n_blocks;
  std::vector<uint32_t> flag(1);
  int ret = survey_fetch(ctx, 16, 16, flag, [&](uint32_t *d_flag) {
    obmat::mat_probe_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(b->d_image, b->d_blk_off, b->d_blk_size, n, d_flag);
  });
  if (ret != OBGPU_SUCCESS) return ret;
  if (!(flag[0] & obmat::MF_ANY)) return OBGPU_SUCCESS;
  std::vector<uint32_t> sv((size_t)n * 4);
  ret = survey_fetch(ctx, (size_t)n * 16, 0, sv, [&](uint32_t *d_sv) {
    obmat::mat_survey_kernel<<<(unsigned)(((int64_t)n * 32 + 127) / 128), 128, 0, ctx->stream>>>(b->d_image, b->d_blk_off, b->d_blk_size, n, d_sv);
  });
  if (ret != OBGPU_SUCCESS) return ret;
  std::vector<uint64_t> tab((size_t)n * 2);   // [new_off][job_base]
  std::vector<uint32_t> nsz((size_t)n);
  uint64_t jobs = 0;
  for (int32_t i = 0; i < n; ++i) {
    tab[(size_t)n + i] = jobs;
    nsz[(size_t)i] = sv[(size_t)4 * i];
    jobs += sv[(size_t)4 * i + 1];
  }
  if (jobs == 0) return OBGPU_SUCCESS;   // every such column was refused: the index kernel leaves them unsupported
  const uint64_t pos = slot_layout(nsz.data(), n, tab.data());
  // where the caller's image has every block (string pointers of the untouched columns keep addressing it): carried over from
  // the CS restatement when that ran
  const bool carried = b->d_xf != nullptr;
  std::vector<obcs::XformRec> xf((size_t)n);
  if (carried) {
    CUDA_TRY(ctx, cudaMemcpyAsync(xf.data(), b->d_xf, (size_t)n * sizeof(obcs::XformRec), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  } else {
    for (int32_t i = 0; i < n; ++i) { xf[(size_t)i].orig_off = (uint64_t)b->offsets[(size_t)i]; xf[(size_t)i].str_delta = 0; }
  }
  Scratch img(ctx), tabs(ctx), sizes(ctx), job_list(ctx), status(ctx);
  CUDA_TRY(ctx, img.alloc((size_t)pos + 64));
  CUDA_TRY(ctx, tabs.alloc((size_t)n * 16));
  CUDA_TRY(ctx, sizes.alloc((size_t)n * 4));
  CUDA_TRY(ctx, job_list.alloc((size_t)(jobs + 1) * sizeof(obmat::MatJob)));
  CUDA_TRY(ctx, status.alloc(16));
  if (!carried) CUDA_TRY(ctx, cudaMallocAsync((void **)&b->d_xf, (size_t)n * sizeof(obcs::XformRec), ctx->stream));
  uint8_t *d_new = img.p;
  uint64_t *d_tab = tabs.at<uint64_t>(0);
  uint32_t *d_nsz = sizes.at<uint32_t>(0);
  obmat::MatJob *d_jobs = job_list.at<obmat::MatJob>(0);
  int *d_status = status.at<int>(0);
  CUDA_TRY(ctx, cudaMemsetAsync(d_status, 0, 16, ctx->stream));
  CUDA_TRY(ctx, cudaMemsetAsync(d_new, 0, (size_t)pos + 64, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(d_tab, tab.data(), (size_t)n * 16, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(d_nsz, nsz.data(), (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
  obmat::mat_rewrite_kernel<<<(unsigned)(((int64_t)n * 32 + 127) / 128), 128, 0, ctx->stream>>>(b->d_image, b->d_blk_off, b->d_blk_size, n, d_new,
                                                                                           d_tab, d_nsz, d_tab + n, d_jobs);
  obmat::mat_decode_kernel<<<(unsigned)(((int64_t)jobs * 32 + 127) / 128), 128, 0, ctx->stream>>>(b->d_image, d_new, d_jobs, (int64_t)jobs, d_status);
  ctx->launches += 2;
  CUDA_TRY(ctx, cudaGetLastError());
  int st = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&st, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
  if ((ret = install_image(ctx, b, img, pos, tab.data(), nsz.data())) != OBGPU_SUCCESS) return ret;
  if (!carried) CUDA_TRY(ctx, cudaMemcpyAsync(b->d_xf, xf.data(), (size_t)n * sizeof(obcs::XformRec), cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (st != 0) {
    ctx->err = "HEX_PACKING / STRING_DIFF / STRING_PREFIX column does not decode (corrupt micro block)";
    return OBGPU_INVALID_DATA;
  }
  return OBGPU_SUCCESS;
}

// The body of obgpu_batch_open: fills b, which the caller closes when this fails. host: a host view of the blocks, or nullptr.
static int fill_batch(obgpu_ctx *ctx, obgpu_batch *b, const void *image, int64_t image_size, const int64_t *offsets, const int64_t *sizes,
                      int32_t n_blocks, int32_t image_on_device, const uint8_t *host) {
  b->n_blocks = n_blocks;
  b->image_size = image_size;
  b->offsets.assign(offsets, offsets + n_blocks);
  b->sizes.assign(sizes, sizes + n_blocks);
  b->row_count.resize((size_t)n_blocks);
  b->col_count.resize((size_t)n_blocks);
  b->bm_word_off.resize((size_t)n_blocks + 1);
  for (int32_t i = 0; i < n_blocks; ++i) {
    const int64_t off = offsets[i], sz = sizes[i];
    if (off < 0 || (off & 15) || sz < 64 || sz > 0x7fffffffll || off + sz > image_size) return OBGPU_INVALID_ARGUMENT;
    const int64_t padded = (sz + 15) & ~15ll;
    const int64_t limit = i + 1 < n_blocks ? offsets[i + 1] : image_size;
    if (image_on_device && off + padded > limit) {
      ctx->err = "blocks of a device-resident image must be padded to 16 bytes";
      return OBGPU_INVALID_ARGUMENT;
    }
    b->max_block_bytes = std::max<uint32_t>(b->max_block_bytes, (uint32_t)padded);
  }
  // device tables: [blk_off u64 x n][bm_word_off i64 x (n + 1)][blk_size u32 x n] ... [row_start i64 x (n + 1)]
  const size_t tb_rs = (((size_t)n_blocks * (8 + 4) + ((size_t)n_blocks + 1) * 8) + 15) & ~(size_t)15;  // row_start follows
  const size_t tb = tb_rs + ((size_t)n_blocks + 1) * 8 + 64;
  CUDA_TRY(ctx, cudaMallocAsync(&b->d_tables, tb, ctx->stream));
  uint8_t *dt = (uint8_t *)b->d_tables;
  b->d_blk_off = (uint64_t *)dt;
  b->d_bm_word_off = (int64_t *)(dt + (size_t)n_blocks * 8);
  b->d_blk_size = (uint32_t *)(dt + (size_t)n_blocks * 8 + ((size_t)n_blocks + 1) * 8);
  b->d_row_start = (int64_t *)(dt + tb_rs);
  std::vector<uint8_t> stage(tb);
  {
    uint64_t *o = (uint64_t *)stage.data();
    uint32_t *s = (uint32_t *)(stage.data() + (size_t)n_blocks * 8 + ((size_t)n_blocks + 1) * 8);
    for (int32_t i = 0; i < n_blocks; ++i) { o[i] = (uint64_t)offsets[i]; s[i] = (uint32_t)sizes[i]; }
  }
  bool any_cs = false, any_mat = false;
  if (host) {
    for (int32_t i = 0; i < n_blocks; ++i) {
      const uint8_t *p = host + offsets[i];
      obf::MicroHeaderFacts f;
      switch (obf::check_micro_header(p, (uint32_t)sizes[i], f)) {
        case obf::HDR_OK: break;
        case obf::HDR_INVALID: ctx->err = "invalid micro block header"; return OBGPU_INVALID_DATA;
        case obf::HDR_ROW_STORE: ctx->err = "row store type not handled by the device path"; return OBGPU_NOT_SUPPORTED;
        case obf::HDR_EXTENT: return OBGPU_INVALID_DATA;
        default: ctx->err = "more than 65535 rows in one micro block"; return OBGPU_NOT_SUPPORTED;
      }
      b->row_count[(size_t)i] = f.rows;
      b->col_count[(size_t)i] = (int32_t)f.ncol;
      any_cs = any_cs || f.is_cs;
      for (uint32_t c = 0; !f.is_cs && !any_mat && c < f.ncol; ++c) any_mat = obf::rebuilt_at_open(p[f.header_size + 16u * c + 1]);
    }
  } else {
    any_cs = true;   // no host view: the survey kernel of the restatement looks at every block's store type
    any_mat = true;  // ... and the probe kernel of the materialisation at every block's column types
    std::vector<uint32_t> sv((size_t)n_blocks * 2);
    CUDA_TRY(ctx, cudaMemcpyAsync(b->d_tables, stage.data(), tb_rs, cudaMemcpyHostToDevice, ctx->stream));
    const int ret = survey_fetch(ctx, (size_t)n_blocks * 8, 0, sv, [&](uint32_t *d_sv) {
      obgpu_survey_kernel<<<(unsigned)((n_blocks + 255) / 256), 256, 0, ctx->stream>>>((const uint8_t *)image, b->d_blk_off, b->d_blk_size,
                                                                                       n_blocks, d_sv);
    });
    if (ret != OBGPU_SUCCESS) return ret;
    for (int32_t i = 0; i < n_blocks; ++i) {
      const uint32_t verdict = sv[(size_t)2 * i + 1] >> 16;
      if (verdict == obf::HDR_INVALID || verdict == obf::HDR_EXTENT) { ctx->err = "invalid micro block header"; return OBGPU_INVALID_DATA; }
      if (verdict != obf::HDR_OK) { ctx->err = "micro block not handled by the device path"; return OBGPU_NOT_SUPPORTED; }
      b->row_count[(size_t)i] = sv[(size_t)2 * i];
      b->col_count[(size_t)i] = (int32_t)(sv[(size_t)2 * i + 1] & 0xffffu);
    }
  }
  int64_t words = 0;
  for (int32_t i = 0; i < n_blocks; ++i) {
    const uint32_t rows = b->row_count[(size_t)i];
    b->bm_word_off[(size_t)i] = words;
    words += (rows + 31) / 32;
    b->total_rows += rows;
    b->max_rows = std::max(b->max_rows, rows);
    b->max_cols = std::max<uint32_t>(b->max_cols, (uint32_t)b->col_count[(size_t)i]);
  }
  b->bm_word_off[(size_t)n_blocks] = words;
  b->col_max_dict.assign(b->max_cols, 0);
  b->col_types.assign(b->max_cols, 0);
  b->col_max_rle.assign(b->max_cols, 0);
  // blocks larger than a shared-memory page are fine for the batch scan (columns are then decoded straight
  // from global memory); only the one-block entry points need the block to fit
  {
    int64_t *w = (int64_t *)(stage.data() + (size_t)n_blocks * 8);
    memcpy(w, b->bm_word_off.data(), ((size_t)n_blocks + 1) * 8);
    int64_t *rs = (int64_t *)(stage.data() + tb_rs);  // first row of every block in the batch's row order
    rs[0] = 0;
    for (int32_t i = 0; i < n_blocks; ++i) rs[i + 1] = rs[i] + b->row_count[(size_t)i];
  }
  CUDA_TRY(ctx, cudaMemcpyAsync(b->d_tables, stage.data(), tb, cudaMemcpyHostToDevice, ctx->stream));
  if (image_on_device) {
    b->d_image = (const uint8_t *)image;
  } else {
    void *di = nullptr;
    CUDA_TRY(ctx, cudaMallocAsync(&di, (size_t)image_size + 64, ctx->stream));
    b->d_image = (const uint8_t *)di;
    b->own_image = true;
    CUDA_TRY(ctx, cudaMemsetAsync((uint8_t *)di + image_size, 0, 64, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(di, image, (size_t)image_size, cudaMemcpyHostToDevice, ctx->stream));
  }
  int ret;
  // CS blocks whose integer streams carry codecs are restated as RAW once, here (the reference's full_transform at cache fill)
  if (any_cs && (ret = cs_restate_batch(ctx, b)) != OBGPU_SUCCESS) return ret;
  // PAX string codecs that rebuild their values (HEX_PACKING / STRING_DIFF / STRING_PREFIX): materialised once, here
  if (any_mat && (ret = pax_materialise_batch(ctx, b)) != OBGPU_SUCCESS) return ret;
  // decode plans: one thread per (block, column)
  if (b->max_cols > 128) {
    ctx->err = "more than 128 columns in a micro block";
    return OBGPU_NOT_SUPPORTED;
  }
  const size_t plan_bytes = (size_t)n_blocks * b->max_cols * sizeof(ColDesc);
  void *dp = nullptr;
  const size_t rows_bytes = ((size_t)n_blocks * 4 + 63) & ~(size_t)63;
  const size_t rec_bytes = (size_t)n_blocks * sizeof(BlockRec);
  // stage records only where the small-block pipelined kernels can run
  const bool pipe = pipe_wanted(b->max_rows);
  const size_t stage_bytes = pipe ? (size_t)n_blocks * b->max_cols * sizeof(StageRec) : 0;
  constexpr size_t kSpanRows = 8;
  CUDA_TRY(ctx, cudaMallocAsync(&dp, plan_bytes + stage_bytes + rows_bytes + rec_bytes + (size_t)b->max_cols * 4 * kSpanRows + 64, ctx->stream));
  b->d_plans = (ColDesc *)dp;
  b->d_stage = pipe ? (StageRec *)((uint8_t *)dp + plan_bytes) : nullptr;
  b->d_rows = (uint32_t *)((uint8_t *)dp + plan_bytes + stage_bytes);
  b->d_recs = (BlockRec *)((uint8_t *)dp + plan_bytes + stage_bytes + rows_bytes);
  uint32_t *d_span = (uint32_t *)((uint8_t *)dp + plan_bytes + stage_bytes + rows_bytes + rec_bytes);
  // per-column reductions of the index kernel: [region span][dictionary size][type min][type max][RLE runs][projection span][materialised]
  // [stage record gaps: SR_NOT_FILTER | SR_NOT_FLAT]
  CUDA_TRY(ctx, cudaMemsetAsync(d_span, 0, (size_t)b->max_cols * 4 * kSpanRows, ctx->stream));
  CUDA_TRY(ctx, cudaMemsetAsync(d_span + 2 * (size_t)b->max_cols, 0xff, (size_t)b->max_cols * 4, ctx->stream));
  const int64_t nthreads = (int64_t)n_blocks * b->max_cols;
  obgpu_index_kernel<<<(unsigned)((nthreads + 255) / 256), 256, 0, ctx->stream>>>(
      b->d_image, b->d_blk_off, b->d_blk_size, b->d_bm_word_off, n_blocks, (int)b->max_cols, b->d_plans,
      b->d_rows, b->d_recs, b->d_stage, d_span);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  b->col_span.assign((size_t)b->max_cols * kSpanRows, 0);
  CUDA_TRY(ctx, cudaMemcpyAsync(b->col_span.data(), d_span, (size_t)b->max_cols * 4 * kSpanRows, cudaMemcpyDeviceToHost, ctx->stream));
  // `stage` is pageable: the copy above is staged synchronously by the runtime before returning
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  const size_t mc = b->max_cols;
  b->col_pspan.assign(b->col_span.begin() + 5 * mc, b->col_span.begin() + 6 * mc);
  b->col_stage_gaps.assign(b->col_span.begin() + 7 * mc, b->col_span.begin() + 8 * mc);
  b->col_mat.assign(mc, 0);
  for (size_t c = 0; c < mc; ++c) b->col_mat[c] = b->col_span[6 * mc + c] ? 1 : 0;
  for (size_t c = 0; c < mc; ++c) {
    b->col_max_dict[c] = b->col_span[mc + c];
    const uint32_t tmin = b->col_span[2 * mc + c], tmax = b->col_span[3 * mc + c];
    b->col_types[c] = tmin == 0xffffffffu ? 0 : (tmin == tmax ? (uint8_t)tmin : 0xff);   // 0xff: the blocks disagree
    b->col_max_rle[c] = b->col_span[4 * mc + c];
  }
  b->col_span.resize(mc);
  return OBGPU_SUCCESS;
}

extern "C" {

int obgpu_batch_open(obgpu_ctx *ctx, const void *image, int64_t image_size, const int64_t *offsets,
                     const int64_t *sizes, int32_t n_blocks, int32_t image_on_device, const void *header_view,
                     obgpu_batch **out) {
  if (!ctx || !image || !offsets || !sizes || n_blocks <= 0 || !out || image_size <= 0)
    return OBGPU_INVALID_ARGUMENT;
  if (image_on_device && ((uintptr_t)image & 15u) != 0) {
    ctx->err = "device-resident image must be 16-byte aligned (TMA bulk copies)";
    return OBGPU_INVALID_ARGUMENT;
  }
  cudaSetDevice(ctx->device);
  obgpu_batch *b = new (std::nothrow) obgpu_batch();
  if (!b) return OBGPU_ALLOCATE_MEMORY_FAILED;
  b->ctx = ctx;
  // header facts come from a host view of the blocks when there is one; a device-resident image opened without
  // a host view is surveyed on the device instead (obgpu_survey_kernel)
  const int ret = fill_batch(ctx, b, image, image_size, offsets, sizes, n_blocks, image_on_device,
                             image_on_device ? (const uint8_t *)header_view : (const uint8_t *)image);
  if (ret != OBGPU_SUCCESS) {
    obgpu_batch_close(b);
    return ret;
  }
  *out = b;
  return OBGPU_SUCCESS;
}

void obgpu_batch_close(obgpu_batch *b) {
  if (!b) return;
  cudaSetDevice(b->ctx->device);
  if (b->d_tables) cudaFreeAsync(b->d_tables, b->ctx->stream);
  if (b->d_plans) cudaFreeAsync(b->d_plans, b->ctx->stream);
  if (b->d_agg) cudaFreeAsync(b->d_agg, b->ctx->stream);
  if (b->d_agg_off) cudaFreeAsync(b->d_agg_off, b->ctx->stream);
  if (b->d_xf) cudaFreeAsync(b->d_xf, b->ctx->stream);
  if (b->own_image && b->d_image) cudaFreeAsync((void *)b->d_image, b->ctx->stream);
  delete b;
}

int obgpu_batch_block_info(const obgpu_batch *b, int32_t block, int64_t *row_count, int32_t *column_count) {
  if (!b || block < 0 || block >= b->n_blocks) return OBGPU_INVALID_ARGUMENT;
  if (row_count) *row_count = b->row_count[(size_t)block];
  if (column_count) *column_count = b->col_count[(size_t)block];
  return OBGPU_SUCCESS;
}

int obgpu_batch_total_rows(const obgpu_batch *b, int64_t *total_rows) {
  if (!b || !total_rows) return OBGPU_INVALID_ARGUMENT;
  *total_rows = b->total_rows;
  return OBGPU_SUCCESS;
}

}  // extern "C"
