// Phase B for tables whose row store is CS_ENCODING_ROW_STORE: merged integer columns -> CS micro-blocks, byte for byte the blocks
// the host writer (sstable_writer.cpp: BlockBuilder::build_cs, choose_cs_auto_encoding, put_dict_ref_stream, emit_int_stream) writes
// at the same CS stream mode (obgpu_writer_set_cs_stream_encoding): mode 1 RAW integer streams, the other modes the stream codecs of
// stream_encode.cuh (the CODEC instantiations). One kernel, one CTA per micro-block, on the phases of the
// PAX encoder (encode_kernels.cuh): ticket + decoupled look-back, stats pass with the column checksum folded in, block-wide stable
// sort, parallel crc32c, one TMA store of the aligned slot.
//
//   [header][ObAllColumnHeader][ObCSColumnHeader x ncol][per column: CS_INTEGER | CS_INT_DICT][stream offsets]
//
//   CS_INTEGER  : [NULL bitmap, MSB first, only when NULL cannot be replaced][stream meta][v - base, width bytes each]
//   CS_INT_DICT : [ObDictEncodingMeta][dictionary stream][ref stream] (an all-NULL column: the meta alone, no streams)
//   offsets     : one more RAW stream of the block-relative stream ends, width byte_packed_int_size(last end)
//
// Key domains. The writer orders and ranges a signed column on the full 8-byte datum (int64) and an unsigned one on the masked
// store image (uint64): the stats and the write's sort use that key (the full datum with bit 63 flipped / the store image), so a
// datum that is not sign-extended is written as the writer writes it. choose_cs_auto_encoding's estimate counts the distinct
// store images (build_int_dict): an AUTO column is analysed on the store image first, and re-sorted on the write's key only when
// the dictionary wins and the two keys differ (a signed column narrower than 8 bytes).
#pragma once

namespace enc {

constexpr unsigned long long kSign = 1ull << 63;
constexpr uint32_t kCsHead = kHeaderSize + 12u;   // ObAllColumnHeader behind the micro header; the column headers follow

// What one CS column of a block is written as (the plan's output, read by the pack).
struct CsCol {
  unsigned long long base, nullv;   // INTEGER: stream base and NULL replacement; INT_DICT: dictionary base
  uint32_t off, bytes;              // column start (block-relative) and bytes
  uint32_t s0;                      // INT_DICT: end of the dictionary stream, relative to the column start
  uint32_t sidx;                    // index of the column's first stream end in the stream-offsets stream
  uint32_t exc, rcnt;               // INT_DICT: exceptions of the const ref form, values in the ref stream
  uint8_t type, attrs, width, meta; // CSColType, CSColAttr, value width, bytes of the (first) stream meta
  uint8_t sattr, rwidth, cform, nstreams;   // stream attr (IS_USE_BASE / IS_REPLACE_NULL_VALUE), ref width, const ref form
};

__device__ __forceinline__ uint32_t vi_len(unsigned long long v) {   // serialization::encode_vi64 length
  uint32_t n = 1;
  while (v > 0x7full) { v >>= 7; ++n; }
  return n;
}
__device__ __forceinline__ uint32_t cs_bit_size(unsigned long long v) { return v == 0 ? 1u : 64u - (uint32_t)__clzll((long long)v); }

// INTEGER_STREAM_META_V2, attr, codec type, width tag, [vi64 base], [vi64 NULL replacement], pfor_packing_type_ 1, at byte `at`
__device__ void put_stream_meta(uint32_t *img32, uint32_t at, uint32_t attr, uint32_t width, unsigned long long base,
                                unsigned long long nullv, uint32_t type = obf::IS_RAW) {
  const uint32_t tag = width == 1u ? 0u : width == 2u ? 1u : width == 4u ? 2u : 3u;
  put_bytes(img32, at, 4u, 1u | (attr << 8) | (type << 16) | (tag << 24));
  at += 4u;
  for (int k = 0; k < 2; ++k) {
    if (!(attr & (1u << k))) continue;
    unsigned long long v = k == 0 ? base : nullv;
    while (v > 0x7full) { put_bytes(img32, at++, 1u, (v & 0x7full) | 0x80ull); v >>= 7; }
    put_bytes(img32, at++, 1u, v);
  }
  put_bytes(img32, at, 1u, 1u);
}

// build_cs's CS_INTEGER branch (ObIntegerColumnEncoder::build_signed_stream_meta_ / build_unsigned_encoder_ctx_): the range after
// the NULL replacement rules, the base, and whether NULL needs the bitmap. kmin / kmax: the write's keys of the non-NULL cells.
struct CsIntPlan {
  unsigned long long base, nullv, range;
  bool use_base, replace, bitmap;
};
__device__ __forceinline__ CsIntPlan cs_int_plan(bool sgn, uint32_t ts, unsigned long long kmin, unsigned long long kmax, bool any,
                                                 bool has_null) {
  CsIntPlan r{};
  const unsigned long long mask = obf::low_mask(8u * ts);
  if (sgn) {
    const unsigned long long rmask = ~mask;
    const long long type_min = rmask == 0 ? (long long)kSign : (long long)(rmask | (rmask >> 1)), type_max = (long long)(mask >> 1);
    long long nmin = (long long)(kmin ^ kSign), nmax = (long long)(kmax ^ kSign);
    if (has_null) {
      if (!any) nmin = nmax = 0;
      if (nmin == 0) {
        r.replace = true;
        if (nmax != type_max) { nmax += 1; r.nullv = (unsigned long long)nmax; }
        else { nmin = -1; r.nullv = (unsigned long long)nmin; }
      } else if (nmin == type_min) {
        if (nmax != type_max) { nmax += 1; r.replace = true; r.nullv = (unsigned long long)nmax; }
        else r.bitmap = true;
      } else {
        nmin -= 1; r.replace = true; r.nullv = (unsigned long long)nmin;
      }
    }
    r.use_base = nmin < 0;
    r.base = r.use_base ? (unsigned long long)nmin : 0ull;
    r.range = (unsigned long long)nmax - r.base;
  } else {
    unsigned long long nmin = kmin, nmax = kmax;
    if (has_null) {
      if (!any) nmin = nmax = 0;
      if (nmin == 0) {
        if (nmax != mask) { nmax += 1; r.replace = true; r.nullv = nmax; }
        else r.bitmap = true;
      } else {
        nmin -= 1; r.replace = true; r.nullv = nmin;
      }
    }
    r.range = nmax;
  }
  return r;
}

// choose_cs_auto_encoding for an integer column: true when the dictionary wins. A: the analysis on the store image (the estimate's
// build_int_dict: distinct images, ties of the constant to the earliest first occurrence, max_row searched from the end).
__device__ bool cs_auto_pick(const ColSpec &cs, const AutoCol &A, uint32_t nrows, uint32_t nnull, unsigned long long kmin,
                             unsigned long long kmax) {
  const long long n = nrows, nn = nnull, d = A.d;
  const uint32_t ts = cs.store_size;
  const CsIntPlan ip = cs_int_plan(cs.is_signed, ts, kmin, kmax, nn < n, nn > 0);
  const long long int_est = (long long)cs_bit_size(ip.range) * n / 8 + (ip.bitmap ? (n + 7) / 8 : 0);
  long long dict_est = 10;   // sizeof(ObDictEncodingMeta)
  if (d > 0) {
    unsigned long long range;
    if (cs.is_signed) {
      const unsigned long long f = 1ull << (8u * ts - 1u);
      const long long mn = sign_extend(A.kmin ^ f, ts), mx = sign_extend(A.kmax ^ f, ts);
      range = mn < 0 ? (unsigned long long)mx - (unsigned long long)mn : (unsigned long long)mx;
    } else {
      range = A.kmax;
    }
    long long ref_rows = n;
    unsigned long long ref_max = (unsigned long long)(nn > 0 ? d : d - 1);
    const long long max_cnt = nn > (long long)A.fmax ? nn : (long long)A.fmax, exc = n - max_cnt;
    if (exc == 0) { ref_rows = 2; ref_max = 0; }   // one value in every row: the constant is ref 0
    else if (exc <= 64 && exc < n * 10 / 100) {
      ref_rows = 2 + 2 * exc;
      ref_max = max(max((unsigned long long)exc, (unsigned long long)A.row_e), ref_max);
    }
    dict_est += (long long)cs_bit_size(range) * d / 8 + (long long)cs_bit_size(ref_max) * ref_rows / 8;
  }
  return dict_est < int_est * 70 / 100 || (dict_est < int_est && d < n * 50 / 100);
}

// The streams of a CS_INT_DICT column with d > 0 distinct values (A: the analysis on the write's key): the dictionary's base,
// width and meta, and the ref stream, plain or in the const form (put_dict_ref_stream: the constant ties to the smallest sorted
// ref, NULL only when strictly more frequent).
__device__ __forceinline__ void cs_dict_layout(const ColSpec &cs, const AutoCol &A, uint32_t nrows, uint32_t nn, CsCol &L) {
  const uint32_t d = A.d;
  const unsigned long long f = cs.is_signed ? kSign : 0ull, vmin = A.kmin ^ f, vmax = A.kmax ^ f;
  const bool use_base = cs.is_signed && (long long)vmin < 0;
  L.base = use_base ? vmin : 0ull;
  L.width = (uint8_t)bpis(vmax - L.base);
  L.sattr = use_base ? (uint8_t)obf::IS_USE_BASE : 0;
  L.meta = (uint8_t)(5u + (use_base ? vi_len(L.base) : 0u));
  const uint32_t max_ref = nn ? d : d - 1u, max_cnt = max(A.fmax, nn), exc = nrows - max_cnt;
  L.cform = exc == 0 || (exc <= 64u && exc < nrows * 10u / 100u);
  L.exc = exc;
  if (L.cform) {
    L.rcnt = 2u + 2u * exc;
    L.rwidth = (uint8_t)bpis(exc == 0 ? A.ref_w : max(max(exc, A.row_w), max_ref));
  } else {
    L.rcnt = nrows;
    L.rwidth = (uint8_t)bpis(max_ref);
  }
}

// The const-form ref stream [exceptions][constant cw][exception rows][exception refs] into cref, from the sorted refs in s.a.
// Every thread calls it.
__device__ void cs_const_refs(const AutoScratch &s, uint32_t nrows, uint32_t cw, uint32_t exc, uint32_t *cref) {
  if (threadIdx.x == 0) { cref[0] = exc; cref[1] = cw; }
  if (exc) {
    for (uint32_t r = threadIdx.x; r < nrows; r += kThreads) s.hs[r] = s.a[r] != cw ? 1u : 0u;
    __syncthreads();
    blk_scan(s.hs, nrows, s.red);
    for (uint32_t r = threadIdx.x; r < nrows; r += kThreads) {
      if (s.a[r] == cw) continue;
      const uint32_t k = s.hs[r] - 1u;
      cref[2u + k] = r;
      cref[2u + exc + k] = s.a[r];
    }
  }
  __syncthreads();
}

// SORT: some column may store a dictionary (the sort scratch); CODEC: the integer streams take the stream codecs of
// p.stream_mode (stream_encode.cuh) through a sizing phase between the analysis and the plan. <SORT, false> writes RAW streams.
template <bool SORT, bool CODEC>
__global__ void __launch_bounds__(kThreads) obgpu_encode_cs_kernel(const __grid_constant__ Params p) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint32_t *img32 = reinterpret_cast<uint32_t *>(smem);              // block image, p.slot_cap bytes
  uint32_t *tab = reinterpret_cast<uint32_t *>(smem + p.slot_cap);   // 4 x 256 crc tables
  // per column scratch behind the tables: [kWarps][n_cols] min / max key, [kWarps][n_cols] NULL count, [n_cols] CsCol
  unsigned long long *s_wmin = reinterpret_cast<unsigned long long *>(smem + p.slot_cap + 4096u);
  unsigned long long *s_wmax = s_wmin + kWarps * p.n_cols;
  uint32_t *s_wnull = reinterpret_cast<uint32_t *>(s_wmax + kWarps * p.n_cols);
  CsCol *s_cs = reinterpret_cast<CsCol *>((reinterpret_cast<uintptr_t>(s_wnull + kWarps * p.n_cols) + 15u) & ~(uintptr_t)15u);
  // INT_DICT / AUTO: [n_cols] AutoCol, then the sort scratch (cs_smem_bytes on the host counts the same)
  AutoCol *s_auto = nullptr;
  AutoScratch scr{};
  __shared__ uint32_t s_ared[SORT ? kWarps : 1];
  if constexpr (SORT) {
    uintptr_t q = (reinterpret_cast<uintptr_t>(s_cs + p.n_cols) + 15u) & ~(uintptr_t)15u;
    s_auto = reinterpret_cast<AutoCol *>(q);
    q = (q + (uintptr_t)p.n_cols * sizeof(AutoCol) + 15u) & ~(uintptr_t)15u;
    const uint32_t P = p.sort_cap, R = (uint32_t)p.rows_per_block;
    scr.sk = reinterpret_cast<unsigned long long *>(q);
    scr.sr = reinterpret_cast<uint32_t *>(scr.sk + P);
    scr.hs = scr.sr + P;
    scr.a = scr.hs + P;
    scr.b = scr.a + R;
    scr.hp = scr.b + R;
    scr.red = s_ared;
  }
  // CODEC: [n_cols] CsCodec, [kWarps][kHistBins] histograms, [chunks] chunk sizes, [kCrefMax] const-form refs behind the rest
  StreamScratch sts{};
  __shared__ uint32_t s_sred[CODEC ? kWarps : 1];
  if constexpr (CODEC) {
    uintptr_t q = SORT ? reinterpret_cast<uintptr_t>(scr.hp + p.rows_per_block + 1) : reinterpret_cast<uintptr_t>(s_cs + p.n_cols);
    q = (q + 15u) & ~(uintptr_t)15u;
    sts.cod = reinterpret_cast<CsCodec *>(q);
    sts.hist = reinterpret_cast<uint32_t *>(sts.cod + p.n_cols);
    sts.cref = sts.hist + kWarps * kHistBins;
    sts.csz = sts.cref + kCrefMax;
    sts.red = s_sred;
  }
  __shared__ uint32_t s_red[kWarps];
  __shared__ int s_blk;
  __shared__ uint32_t s_size, s_original, s_ends_at, s_swidth, s_scount, s_pick;
  __shared__ long long s_off;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  block_prologue(p, smem, tab, &s_blk);
  const int blk = s_blk;
  const int64_t row0 = (int64_t)blk * p.rows_per_block;
  const uint32_t nrows = (uint32_t)min(p.rows_per_block, p.total_rows - row0);
  const int nc = p.n_cols;
  __syncthreads();

  // ---- stats (+ column checksums): smallest / largest key and NULL count, four columns at a time --------------------------
  for (int c0 = 0; c0 < nc; c0 += 4) {
    unsigned long long mn[4] = {~0ull, ~0ull, ~0ull, ~0ull}, mx[4] = {0, 0, 0, 0}, sum[4] = {0, 0, 0, 0};
    uint32_t nn[4] = {0, 0, 0, 0}, len_crc[4];
    const uint32_t null_crc = crc_word(tab, 0u, 0x80000000u);
#pragma unroll
    for (int j = 0; j < 4; ++j) len_crc[j] = crc_word(tab, 0u, (uint32_t)p.col[min(c0 + j, nc - 1)].datum_len);
    for (uint32_t r = (uint32_t)tid; r < nrows; r += kThreads) {
      unsigned long long x[4];
      uint32_t nlb[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = min(c0 + j, nc - 1);   // the tail repeats the last column (its results are dropped below)
        x[j] = (unsigned long long)p.col[c].vals[row0 + r];
        nlb[j] = p.col[c].nulls ? p.col[c].nulls[row0 + r] : 0u;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const ColSpec &cs = p.col[min(c0 + j, nc - 1)];
        const bool is_null = nlb[j] != 0;
        const unsigned long long k = cs.is_signed ? x[j] ^ kSign : x[j] & cs.store_mask;
        if (is_null) ++nn[j];
        else { mn[j] = min(mn[j], k); mx[j] = max(mx[j], k); }
        sum[j] += cell_crc(tab, is_null ? null_crc : len_crc[j], x[j], cs.datum_len, is_null);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (c0 + j >= nc) break;
      const uint32_t hi = (uint32_t)(mx[j] >> 32), hmax = __reduce_max_sync(0xffffffffu, hi);
      const uint32_t lmax = __reduce_max_sync(0xffffffffu, hi == hmax ? (uint32_t)mx[j] : 0u);
      const uint32_t mhi = (uint32_t)(mn[j] >> 32), hmin = __reduce_min_sync(0xffffffffu, mhi);
      const uint32_t lmin = __reduce_min_sync(0xffffffffu, mhi == hmin ? (uint32_t)mn[j] : 0xffffffffu);
      const uint32_t nsum = __reduce_add_sync(0xffffffffu, nn[j]);
      unsigned long long tot = 0;
#pragma unroll
      for (int d = 0; d < 4; ++d) tot += (unsigned long long)__reduce_add_sync(0xffffffffu, (uint32_t)(sum[j] >> (16 * d)) & 0xffffu) << (16 * d);
      if (lane == 0) {
        s_wmax[warp * nc + c0 + j] = ((unsigned long long)hmax << 32) | lmax;
        s_wmin[warp * nc + c0 + j] = ((unsigned long long)hmin << 32) | lmin;
        s_wnull[warp * nc + c0 + j] = nsum;
        if (tot != 0) atomicAdd(p.checksums + c0 + j, tot);
      }
    }
  }
  __syncthreads();

  if constexpr (SORT) {   // ---- analysis of the INT_DICT / AUTO columns, one after another, every thread ---------------------
    for (int c = 0; c < nc; ++c) {
      const ColSpec &cs = p.col[c];
      bool dict = cs.cs_dict != 0;
      if (cs.is_auto || dict) {
        uint32_t nn = 0;
        unsigned long long kmin = ~0ull, kmax = 0;
        for (int w = 0; w < kWarps; ++w) {
          nn += s_wnull[w * nc + c];
          kmin = min(kmin, s_wmin[w * nc + c]);
          kmax = max(kmax, s_wmax[w * nc + c]);
        }
        ColSpec wk = cs;   // the write's sort key: the full datum of a signed column
        if (wk.is_signed) { wk.store_mask = ~0ull; wk.store_size = 8; }
        const bool same_key = !cs.is_signed || cs.store_size == 8;
        if (cs.is_auto) {
          analyze_column(cs, row0, nrows, nn, p.sort_cap, scr, s_auto[c]);
          if (tid == 0) s_pick = cs_auto_pick(cs, s_auto[c], nrows, nn, kmin, kmax) ? 1u : 0u;
          __syncthreads();
          dict = s_pick != 0;
        }
        if (dict && !(cs.is_auto && same_key)) analyze_column(wk, row0, nrows, nn, p.sort_cap, scr, s_auto[c]);
        if constexpr (CODEC) {   // the dictionary streams, while the column's sort on the write's key is in the scratch
          if (dict && s_auto[c].d > 0) {
            CsCol L{};
            cs_dict_layout(cs, s_auto[c], nrows, nn, L);
            uint32_t b0, b1;
            const uint32_t t0 = choose_codec(p.stream_mode, DictVals{scr.sk, scr.hp, cs.is_signed ? kSign : 0ull, L.base}, s_auto[c].d,
                                             L.width, sts, &b0);
            if (L.cform) cs_const_refs(scr, nrows, s_auto[c].ref_w, L.exc, sts.cref);
            const uint32_t t1 = choose_codec(p.stream_mode, RefVals{L.cform ? sts.cref : scr.a}, L.rcnt, L.rwidth, sts, &b1);
            if (tid == 0) sts.cod[c] = CsCodec{{b0, b1}, {(uint8_t)t0, (uint8_t)t1}, {0, 0}};
          }
        }
      }
      if (tid == 0) s_cs[c].type = dict ? (uint8_t)obf::CS_INT_DICT : (uint8_t)obf::CS_INTEGER;
    }
    __syncthreads();
  }

  if constexpr (CODEC) {   // ---- stream sizing of the CS_INTEGER columns (the dictionary streams were sized in the analysis) ----
    for (int c = 0; c < nc; ++c) {
      if (SORT && s_cs[c].type != obf::CS_INTEGER) continue;
      const ColSpec &cs = p.col[c];
      uint32_t nn = 0;
      unsigned long long kmin = ~0ull, kmax = 0;
      for (int w = 0; w < kWarps; ++w) {
        nn += s_wnull[w * nc + c];
        kmin = min(kmin, s_wmin[w * nc + c]);
        kmax = max(kmax, s_wmax[w * nc + c]);
      }
      const CsIntPlan ip = cs_int_plan(cs.is_signed, cs.store_size, kmin, kmax, nn < nrows, nn > 0);
      const IntVals iv{cs.vals + row0, cs.nulls ? cs.nulls + row0 : nullptr, cs.is_signed ? ~0ull : cs.store_mask, ip.base,
                       ip.replace ? ip.nullv - ip.base : 0ull};
      uint32_t b0;
      const uint32_t t0 = choose_codec(p.stream_mode, iv, nrows, bpis(ip.range), sts, &b0);
      if (tid == 0) sts.cod[c] = CsCodec{{b0, 0u}, {(uint8_t)t0, (uint8_t)ST_RAW}, {0, 0}};
    }
    __syncthreads();
  }

  // ---- plan: warp 0, one lane per column (two rounds for more than 32 columns) -------------------------------------------
  if (warp == 0) {
    uint32_t at = kCsHead + 4u * (uint32_t)nc, sbase = 0, last_end = 0;
    unsigned long long original = 0;
    for (int cb = 0; cb < nc; cb += 32) {
      const int c = cb + lane;
      uint32_t bytes = 0, ns = 0, nn = 0;
      CsCol L{};
      if (c < nc) {
        const ColSpec &cs = p.col[c];
        unsigned long long kmin = ~0ull, kmax = 0;
        for (int w = 0; w < kWarps; ++w) {
          nn += s_wnull[w * nc + c];
          kmin = min(kmin, s_wmin[w * nc + c]);
          kmax = max(kmax, s_wmax[w * nc + c]);
        }
        L.type = SORT ? s_cs[c].type : (uint8_t)obf::CS_INTEGER;
        if (L.type == obf::CS_INTEGER) {
          const CsIntPlan ip = cs_int_plan(cs.is_signed, cs.store_size, kmin, kmax, nn < nrows, nn > 0);
          L.base = ip.base;
          L.nullv = ip.nullv;
          L.width = (uint8_t)bpis(ip.range);
          L.sattr = (uint8_t)((ip.use_base ? obf::IS_USE_BASE : 0) | (ip.replace ? obf::IS_REPLACE_NULL_VALUE : 0));
          L.attrs = ip.bitmap ? (uint8_t)obf::CS_HAS_NULL_OR_NOP_BITMAP : 0;
          L.meta = (uint8_t)(5u + (ip.use_base ? vi_len(ip.base) : 0u) + (ip.replace ? vi_len(ip.nullv) : 0u));
          bytes = (ip.bitmap ? (nrows + 7u) / 8u : 0u) + L.meta + (CODEC ? sts.cod[c].bytes[0] : L.width * nrows);
          ns = 1;
        } else if (SORT) {
          const AutoCol &A = s_auto[c];
          const uint32_t d = A.d;
          bytes = 10u;   // ObDictEncodingMeta
          if (d > 0) {
            cs_dict_layout(cs, A, nrows, nn, L);
            L.s0 = 10u + L.meta + (CODEC ? sts.cod[c].bytes[0] : L.width * d);
            bytes = L.s0 + 5u + (CODEC ? sts.cod[c].bytes[1] : L.rwidth * L.rcnt);
            ns = 2;
          }
        }
      }
      uint32_t incl = bytes, sincl = ns;   // column stores back to back, their streams in column order
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o), v = __shfl_up_sync(0xffffffffu, sincl, o);
        if (lane >= o) { incl += u; sincl += v; }
      }
      if (c < nc) {
        L.off = at + incl - bytes;
        L.bytes = bytes;
        L.sidx = sbase + sincl - ns;
        L.nstreams = (uint8_t)ns;
        s_cs[c] = L;
        if (ns) last_end = L.off + bytes;
      }
      at += __shfl_sync(0xffffffffu, incl, 31);
      sbase += __shfl_sync(0xffffffffu, sincl, 31);
      const uint32_t cells = c < nc ? (nrows - nn) * p.col[c].datum_len : 0u;
      original += __reduce_add_sync(0xffffffffu, cells);
    }
    // the stream offsets: RAW, no base, at the width of the last stream end (store_stream_offsets_)
    last_end = __reduce_max_sync(0xffffffffu, last_end);
    const uint32_t sw = bpis(last_end);
    if (lane == 0) {
      s_ends_at = at;
      s_swidth = sw;
      s_scount = sbase;
      if (sbase) at += 5u + sw * sbase;
      s_size = at;
      s_original = (uint32_t)min(original, 0x7fffffffull);
      publish_size(p, blk, false, at);
    }
  }
  __syncthreads();
  const uint32_t size = s_size;
  const uint32_t slot = (size + p.align - 1u) & ~(p.align - 1u);
  if (tid == 0) s_off = resolve_offset(p, blk, size, slot, false);

  // ---- pack (the image was zeroed at the start of the kernel) ------------------------------------------------------------
  const uint32_t ends_at = s_ends_at, sw = s_swidth, scount = s_scount;
  if (tid == 0) {   // ObAllColumnHeader: version_ 0, attrs_ 0, all_string_data_length_ 0, stream_offsets_length_, stream_count_
    put_bytes(img32, kHeaderSize + 6u, 4u, scount ? 5u + sw * scount : 0u);
    put_bytes(img32, kHeaderSize + 10u, 2u, scount);
    if (scount) put_stream_meta(img32, ends_at, 0u, sw, 0ull, 0ull);
  }
  for (int c = tid; c < nc; c += kThreads) {   // ObCSColumnHeader {version_, type_, attrs_, obj_type_}, then the column's stream ends
    const CsCol L = s_cs[c];
    put_bytes(img32, kCsHead + 4u * (uint32_t)c, 4u, ((uint32_t)L.type << 8) | ((uint32_t)L.attrs << 16) | ((uint32_t)p.col[c].obj_type << 24));
    if (L.nstreams == 2) put_bytes(img32, ends_at + 5u + sw * L.sidx, sw, L.off + L.s0);
    if (L.nstreams) put_bytes(img32, ends_at + 5u + sw * (L.sidx + L.nstreams - 1u), sw, L.off + L.bytes);
  }
  for (int c = 0; c < nc; ++c) {
    const ColSpec &cs = p.col[c];
    const CsCol L = s_cs[c];
    const uint32_t o = L.off;
    const uint8_t *nl = cs.nulls ? cs.nulls + row0 : nullptr;
    if (L.type == obf::CS_INTEGER) {
      const bool bitmap = L.attrs != 0;
      const uint32_t mo = o + (bitmap ? (nrows + 7u) / 8u : 0u), v0 = mo + L.meta, w = L.width;
      const uint32_t type = CODEC ? sts.cod[c].type[0] : (uint32_t)ST_RAW;
      const bool raw = type == ST_RAW;
      if (tid == 0) put_stream_meta(img32, mo, L.sattr, w, L.base, L.nullv, type);
      const unsigned long long nv = (L.sattr & obf::IS_REPLACE_NULL_VALUE) ? L.nullv - L.base : 0ull;
      for (uint32_t r = (uint32_t)tid; r < nrows; r += kThreads) {
        if (nl && nl[r] != 0) {
          if (bitmap) or_bits(img32, (o + r / 8u) * 8u + 7u - (r & 7u), 1u, 1ull);   // MSB first
          if (raw) put_bytes(img32, v0 + r * w, w, nv);
          continue;
        }
        const unsigned long long x = (unsigned long long)cs.vals[row0 + r];
        if (raw) put_bytes(img32, v0 + r * w, w, (cs.is_signed ? x : x & cs.store_mask) - L.base);
      }
      if constexpr (CODEC)
        if (!raw) codec_stream(type, IntVals{cs.vals + row0, nl, cs.is_signed ? ~0ull : cs.store_mask, L.base, nv}, nrows, w, sts, img32, v0);
      continue;
    }
    if constexpr (SORT) {   // INT_DICT
      const uint32_t d = s_auto[c].d;
      uint32_t nn = 0;
      for (int w = 0; w < kWarps; ++w) nn += s_wnull[w * nc + c];
      if (tid == 0) {   // ObDictEncodingMeta {version_, attrs_ (IS_SORTED, HAS_NULL, CONST_ENCODING_REF), distinct_val_cnt_, ref_row_cnt_}
        put_bytes(img32, o + 1u, 1u, 0x1u | (nn ? 0x2u : 0u) | (L.cform ? 0x4u : 0u));
        put_bytes(img32, o + 2u, 4u, d);
        put_bytes(img32, o + 6u, 4u, d ? L.rcnt : nrows);
      }
      if (d == 0) continue;
      ColSpec wk = cs;
      if (wk.is_signed) { wk.store_mask = ~0ull; wk.store_size = 8; }
      sort_column(wk, row0, nrows, nn, p.sort_cap, scr);
      const unsigned long long f = cs.is_signed ? kSign : 0ull;
      const uint32_t w = L.width, rw = L.rwidth, r0 = o + L.s0 + 5u, cw = s_auto[c].ref_w, exc = L.exc;
      const uint32_t t0 = CODEC ? sts.cod[c].type[0] : (uint32_t)ST_RAW, t1 = CODEC ? sts.cod[c].type[1] : (uint32_t)ST_RAW;
      if (tid == 0) {
        put_stream_meta(img32, o + 10u, L.sattr, w, L.base, 0ull, t0);
        put_stream_meta(img32, o + L.s0, 0u, rw, 0ull, 0ull, t1);
      }
      if (t0 == ST_RAW) {
        for (uint32_t v = (uint32_t)tid; v < d; v += kThreads) put_bytes(img32, o + 10u + L.meta + v * w, w, (scr.sk[scr.hp[v]] ^ f) - L.base);
      } else if constexpr (CODEC) {
        codec_stream(t0, DictVals{scr.sk, scr.hp, f, L.base}, d, w, sts, img32, o + 10u + L.meta);
      }
      if (t1 != ST_RAW) {
        if constexpr (CODEC) {
          if (L.cform) cs_const_refs(scr, nrows, cw, exc, sts.cref);
          codec_stream(t1, RefVals{L.cform ? sts.cref : scr.a}, L.rcnt, rw, sts, img32, r0);
        }
      } else if (!L.cform) {
        for (uint32_t r = (uint32_t)tid; r < nrows; r += kThreads) put_bytes(img32, r0 + r * rw, rw, scr.a[r]);
      } else {   // [exceptions][const ref][exception rows][exception refs]
        if (tid == 0) {
          put_bytes(img32, r0, rw, exc);
          put_bytes(img32, r0 + rw, rw, cw);
        }
        if (exc) {
          for (uint32_t r = (uint32_t)tid; r < nrows; r += kThreads) scr.hs[r] = scr.a[r] != cw ? 1u : 0u;
          __syncthreads();
          blk_scan(scr.hs, nrows, scr.red);
          for (uint32_t r = (uint32_t)tid; r < nrows; r += kThreads) {
            if (scr.a[r] == cw) continue;
            const uint32_t k = scr.hs[r] - 1u;
            put_bytes(img32, r0 + (2u + k) * rw, rw, r);
            put_bytes(img32, r0 + (2u + exc + k) * rw, rw, scr.a[r]);
          }
        }
      }
      __syncthreads();
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // pack writes -> visible to the bulk copy issued by thread 0
  __syncthreads();
  payload_crc(p, img32, tab, size, s_red);
  __syncthreads();
  // opt_ 0; opt2_: compressor_type_ NONE, no row header; row_data_offset_ 0
  if (tid == 0) finish_block(p, smem, tab, s_red, size, slot, nrows, (uint32_t)obf::CS_ENCODING_ROW_STORE, 0u, (uint32_t)OBGPU_COMPRESSOR_NONE,
                             0u, s_original, s_off);
}

}  // namespace enc

static bool cs_encoding_ok(int32_t e) { return e == OBGPU_ENC_CS_INTEGER || e == OBGPU_ENC_CS_INT_DICT || e == OBGPU_ENC_CS_AUTO; }
// obgpu_writer_set_cs_stream_encoding's modes: 0 detect, 1 RAW, 2..8 one codec except 7 (UNIVERSAL_COMPRESS)
static bool cs_stream_mode_ok(int32_t m) { return m >= 0 && m <= 8 && m != 7; }

extern "C" {

int obgpu_encode_columns_cs_ex(obgpu_ctx *ctx, const obgpu_encode_col *cols, const int32_t *encodings, int32_t n_cols,
                               int32_t rowkey_col_cnt, int64_t total_rows, int64_t rows_per_block, int32_t align, int32_t stream_mode,
                               obgpu_encoded **out) {
  if (!ctx || !cols || !out || n_cols <= 0 || rowkey_col_cnt < 0 || rowkey_col_cnt > n_cols || total_rows <= 0 || rows_per_block <= 0 ||
      rows_per_block > (1 << 22) || align < 16 || align > 4096 || (align & (align - 1)) != 0 || !cs_stream_mode_ok(stream_mode))
    return OBGPU_INVALID_ARGUMENT;
  if (n_cols > enc::kMaxCols) return OBGPU_NOT_SUPPORTED;
  const int64_t n_blocks64 = (total_rows + rows_per_block - 1) / rows_per_block;
  if (n_blocks64 > 0x7fffffff) return OBGPU_NOT_SUPPORTED;
  int n_sort = 0;
  for (int c = 0; encodings && c < n_cols; ++c) {
    if (!cs_encoding_ok(encodings[c])) return OBGPU_NOT_SUPPORTED;
    n_sort += encodings[c] != OBGPU_ENC_CS_INTEGER;
  }
  enc::Params p{};
  int rc = enc_fill_cols(p, cols, n_cols);
  if (rc != OBGPU_SUCCESS) return rc;
  for (int c = 0; encodings && c < n_cols; ++c) {
    p.col[c].is_auto = encodings[c] == OBGPU_ENC_CS_AUTO ? 1 : 0;
    p.col[c].cs_dict = encodings[c] == OBGPU_ENC_CS_INT_DICT ? 1 : 0;
  }
  cudaSetDevice(ctx->device);
  // the largest block: a CS_INTEGER column 8 bytes a row + the NULL bitmap + a 25-byte stream meta; a CS_INT_DICT column an
  // 8-byte value per row + a ref stream of 2-byte refs (a block holds at most 65535 rows; the const form at most 130 values) +
  // 10 + 25 + 5 bytes of metas (AUTO: the larger of the two, the dictionary's); the stream offsets at most 4 bytes per stream
  const int64_t R = rows_per_block;
  if (R > 65535) return OBGPU_NOT_SUPPORTED;
  const int64_t int_col = R * 8 + (R + 7) / 8 + 25, dict_col = 40 + R * 8 + 2 * std::max<int64_t>(R, 130);
  const int64_t bound = (int64_t)enc::kCsHead + 4 * n_cols + (int64_t)(n_cols - n_sort) * int_col + (int64_t)n_sort * dict_col +
                        5 + 8 * n_cols;
  const int64_t slot_cap = (bound + align - 1) / align * align;
  size_t smem = (size_t)slot_cap + 4096 + (size_t)n_cols * (enc::kWarps * 20 + sizeof(enc::CsCol)) + 16;
  uint32_t sort_cap = 1;
  while ((int64_t)sort_cap < R) sort_cap <<= 1;
  // INT_DICT / AUTO: the AutoCol records and the sort scratch (keys, rows, scan: sort_cap each; refs, first occurrences: R each; R + 1 heads)
  if (n_sort) smem += 32 + (size_t)n_cols * sizeof(enc::AutoCol) + (size_t)sort_cap * 16 + (size_t)R * 12 + 4;
  // stream codecs: the CsCodec records, the chunk histograms, the const-form refs and the chunk sizes of the longest stream
  const bool codec = stream_mode != enc::ST_RAW;
  if (codec)
    smem += 16 + (size_t)n_cols * sizeof(enc::CsCodec) + 4 * (size_t)(enc::kWarps * enc::kHistBins + enc::kCrefMax) +
            4 * (size_t)((std::max<int64_t>(R, enc::kCrefMax) + 127) / 128);
  if ((int64_t)smem > (int64_t)ctx->max_smem_optin - 8192) return OBGPU_NOT_SUPPORTED;   // block image does not fit one CTA's shared memory
  p.rowkey_cnt = rowkey_col_cnt;
  p.stream_mode = stream_mode;
  // the sorting instantiations only when some column may store a dictionary: CS_INTEGER-only calls keep the lean kernel; RAW
  // streams (mode 1) keep the kernels without the stream codecs
  void (*kernel)(enc::Params) = n_sort ? (codec ? enc::obgpu_encode_cs_kernel<true, true> : enc::obgpu_encode_cs_kernel<true, false>)
                                       : (codec ? enc::obgpu_encode_cs_kernel<false, true> : enc::obgpu_encode_cs_kernel<false, false>);
  return enc_launch(ctx, p, n_blocks64, total_rows, rows_per_block, align, slot_cap, sort_cap, smem, kernel, out);
}

int obgpu_encode_columns_cs(obgpu_ctx *ctx, const obgpu_encode_col *cols, const int32_t *encodings, int32_t n_cols, int32_t rowkey_col_cnt,
                            int64_t total_rows, int64_t rows_per_block, int32_t align, obgpu_encoded **out) {
  return obgpu_encode_columns_cs_ex(ctx, cols, encodings, n_cols, rowkey_col_cnt, total_rows, rows_per_block, align, enc::ST_RAW, out);
}

int obgpu_merge_result_encode_cs_ex(obgpu_merge_result *res, const int32_t *result_cols, const int32_t *obj_types,
                                    const int32_t *encodings, int32_t n_cols, int32_t rowkey_col_cnt, int64_t rows_per_block,
                                    int32_t align, int32_t stream_mode, obgpu_encoded **out) {
  if (!res || !result_cols || !obj_types || n_cols <= 0 || !out || !cs_stream_mode_ok(stream_mode)) return OBGPU_INVALID_ARGUMENT;
  if (n_cols > enc::kMaxCols) return OBGPU_NOT_SUPPORTED;
  for (int c = 0; encodings && c < n_cols; ++c)
    if (!cs_encoding_ok(encodings[c])) return OBGPU_NOT_SUPPORTED;
  std::vector<obgpu_encode_col> cols;
  int64_t rows = 0;
  const int rc = merge_result_cols(res, result_cols, obj_types, n_cols, cols, rows);
  if (rc != OBGPU_SUCCESS) return rc;
  return obgpu_encode_columns_cs_ex(res->ctx, cols.data(), encodings, n_cols, rowkey_col_cnt, rows, rows_per_block, align, stream_mode, out);
}

int obgpu_merge_result_encode_cs(obgpu_merge_result *res, const int32_t *result_cols, const int32_t *obj_types, const int32_t *encodings,
                                 int32_t n_cols, int32_t rowkey_col_cnt, int64_t rows_per_block, int32_t align, obgpu_encoded **out) {
  return obgpu_merge_result_encode_cs_ex(res, result_cols, obj_types, encodings, n_cols, rowkey_col_cnt, rows_per_block, align, enc::ST_RAW,
                                         out);
}

}  // extern "C"
