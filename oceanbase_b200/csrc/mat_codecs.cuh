// PAX string codecs whose values do not exist in the block: HEX_PACKING, STRING_DIFF, STRING_PREFIX (SURVEY a10).
//
// Reference: ObHexStringDecoder / ObStringDiffDecoder / ObStringPrefixDecoder rebuild a cell into memory of the decoder's allocator
// every time it is read (encoding/ob_hex_string_decoder.cpp:33-127, ob_string_diff_decoder.cpp:34-120, ob_string_prefix_decoder.cpp:
// 30-110); white filters on such columns take the retro path (decode each row, compare). The device rebuilds them ONCE per page
// batch, at obgpu_batch_open, the way CS stream codecs are restated (stream_codecs.cuh): every block that has such a column is
// copied into the batch's own image with a MATERIALISED AREA appended per column,
//     [NULL bits, 1 per row, LSB first][END offset u32 x rows][the strings]
// and the column's decode plan becomes the plan of a CS STRING column (K_CSSTR: END offset per row) over that area, so count /
// project / the per-block entry points need nothing new. The codec's own header in the COPY is patched to say where the area is
// (version byte -> kMatMarker, offset_ field -> area offset); the decode reads the untouched original.
// Rebuilt strings are not part of the caller's image: a scan hands them out through obgpu_result_fetch_strings (a dense heap of the
// selected rows' bytes), the per-block entry point through obgpu_project_strings.
//
// Span columns (COLUMN_EQUAL / COLUMN_SUBSTR, ObColumnEqualDecoder / ObInterColSubStrDecoder, encoding/ob_column_equal_decoder.cpp:
// 32-133, ob_inter_column_substring_decoder.cpp:32-93) go the same way: the value of a row is the referenced column's value (the
// whole of it / a byte range of it) unless the row is in the exception list (ObBitMapMetaReader, ob_encoding_bitset.h:574-760). A
// string span column becomes the same [NULL bits][END offsets][strings] area; an integer COLUMN_EQUAL column becomes
// [NULL bits, padded to 8 bytes][8-byte value image x rows], the plan of a RAW fixed-length column (K_BITS). Their 3 / 8-byte meta
// headers have no room for the area's position, so in the COPY the 16-byte COLUMN header is patched instead: version byte ->
// kMatMarker, offset_ -> the area (from the block start), length_ -> its size. The referenced column must be an ordinary column
// with a decode plan in the original block (RAW / DICT / RLE / CONST / INTEGER_BASE_DIFF).
#pragma once

namespace obmat {

using namespace obdev;

constexpr uint8_t kMatMarker = 0xA5;
enum : uint32_t { MF_ANY = 1, MF_UNSUPPORTED = 2, MF_CORRUPT = 4 };

struct MatJob {
  uint64_t old_off;    // block in the image the batch was opened on
  uint64_t new_off;    // its copy
  uint32_t old_size;
  uint32_t col;
  uint32_t area_off;   // materialised area, relative to the copy's start
  uint32_t area_cap;
};

struct CodecHdr {
  uint32_t meta, length;      // block offset of the codec meta, its length (column header offset_ / length_)
  uint32_t pos_off, pos_len;  // the codec header's offset_ / length_ (row position of var cells, or the fixed cell length)
  uint32_t max_len;           // max_string_size / string_size
  uint32_t pos_field;         // block offset of the offset_ field inside the codec header
  uint8_t type, attr, ok;
};

// the three codec headers (ob_hex_string_encoder.h:139-152, ob_string_diff_encoder.h:27-104, ob_string_prefix_encoder.h:72-107)
__device__ __forceinline__ void read_codec_hdr(const uint8_t *s, const BlockView &b, int col, CodecHdr &h) {
  h = CodecHdr{};
  const uint32_t ch = b.header_size + 16u * (uint32_t)col;
  const uint32_t w0 = ld32(s, ch);
  h.type = (uint8_t)((w0 >> 8) & 0xff);
  h.attr = (uint8_t)((w0 >> 16) & 0xff);
  const uint8_t obj_type = (uint8_t)(w0 >> 24);
  if (h.type != COL_STRING_DIFF && h.type != COL_HEX_PACKING && h.type != COL_STRING_PREFIX) return;
  if (store_class_of(obj_type) != 5) return;
  const uint32_t offset = ld32(s, ch + 8), length = ld32(s, ch + 12);
  if (offset > b.size || b.meta_off > b.size - offset || length < 13u || b.meta_off + offset + length > b.size) return;
  h.meta = b.meta_off + offset;
  h.length = length;
  const uint8_t ver = s[h.meta];
  if (ver != 0 && ver != kMatMarker) return;
  if (h.type == COL_HEX_PACKING) {
    h.pos_field = h.meta + 1u;
    h.max_len = (uint32_t)ld_bytes(s, h.meta + 9u, 4);
  } else if (h.type == COL_STRING_DIFF) {
    h.pos_field = h.meta + 4u;
    h.max_len = (uint32_t)ld_bytes(s, h.meta + 2u, 2);
  } else {
    if (length < 15u) return;
    h.pos_field = h.meta + 2u;
    h.max_len = (uint32_t)ld_bytes(s, h.meta + 10u, 4);
  }
  h.pos_off = (uint32_t)ld_bytes(s, h.pos_field, 4);
  h.pos_len = (uint32_t)ld_bytes(s, h.pos_field + 4u, 4);
  h.ok = 1;
}

__device__ __forceinline__ uint32_t area_bytes(uint32_t rows, uint32_t max_len) {
  return (((rows + 31u) / 32u) * 4u + rows * 4u + rows * max_len + 16u + 15u) & ~15u;
}

// ---- span columns ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool is_span_type(uint32_t t) { return t == COL_COLUMN_EQUAL || t == COL_COLUMN_SUBSTR; }

struct SpanCol {
  ColDesc ref;               // plan of the referenced column, in the original block
  uint32_t meta, length;     // the span meta (column header offset_ / length_)
  uint32_t exc, exc_len;     // block offset / bytes of the exception meta (exc == 0: no exceptions)
  uint32_t rows_off;         // COLUMN_SUBSTR: per-row [start_pos][length]
  uint32_t start, flen;      // COLUMN_SUBSTR: the shared start position / length
  uint64_t int_mask;
  uint8_t type, sc, bit_packing, spb, vlb, same_pos, fix_len, ok;
};

__device__ __forceinline__ void span_col_init(const uint8_t *s, const BlockView &b, int col, SpanCol &m) {
  m.ok = 0;
  const uint32_t ch = b.header_size + 16u * (uint32_t)col;
  const uint32_t w0 = ld32(s, ch);
  if ((w0 & 0xffu) != 0) return;
  m.type = (uint8_t)((w0 >> 8) & 0xff);
  const uint8_t attr = (uint8_t)((w0 >> 16) & 0xff), obj_type = (uint8_t)(w0 >> 24);
  m.sc = (uint8_t)store_class_of(obj_type);
  m.int_mask = integer_mask_of(obj_type);
  m.bit_packing = (attr & ATTR_BIT_PACKING) != 0;
  const uint32_t hdr = m.type == COL_COLUMN_EQUAL ? 3u : 8u;
  if (m.sc == 0 || (m.type == COL_COLUMN_SUBSTR && m.sc != 5)) return;
  const uint32_t offset = ld32(s, ch + 8), length = ld32(s, ch + 12);
  if (offset > b.size || b.meta_off > b.size - offset || length < hdr || length > b.size || b.meta_off + offset + length > b.size) return;
  m.meta = b.meta_off + offset;
  m.length = length;
  if (s[m.meta] != 0) return;
  const uint32_t ref = (uint32_t)ld_bytes(s, m.meta + (m.type == COL_COLUMN_EQUAL ? 1u : 6u), 2);
  if (ref >= b.column_count || ref == (uint32_t)col) return;
  const uint32_t rw0 = ld32(s, b.header_size + 16u * ref), rt = (rw0 >> 8) & 0xffu;
  if ((rw0 >> 24) != obj_type) return;
  if (rt != COL_RAW && rt != COL_DICT && rt != COL_RLE && rt != COL_CONST && rt != COL_INTEGER_BASE_DIFF) return;
  build_col_desc(b, (int)ref, m.ref);
  if (!m.ref.ok) return;
  m.exc = length > hdr ? m.meta + hdr : 0u;
  m.exc_len = length - hdr;
  if (m.exc) {   // ObBitMapMetaHeader + the BitSet over every row must lie inside the meta
    if (m.exc_len <= 4u) return;
    const uint32_t eo = s[m.exc], io = s[m.exc + 1], dof = s[m.exc + 2], u = s[m.exc + 3];
    if (eo < (b.row_count + 63u) / 64u * 8u || io < eo || dof < io || 4u + dof > m.exc_len || u == 0) return;
  }
  m.spb = m.vlb = m.same_pos = m.fix_len = 0;
  m.start = m.flen = m.rows_off = 0;
  if (m.type == COL_COLUMN_SUBSTR) {
    const uint8_t a = s[m.meta + 1];
    m.spb = a & 3u; m.vlb = (a >> 2) & 3u; m.same_pos = (a >> 4) & 1u; m.fix_len = (a >> 5) & 1u;
    m.start = (uint32_t)ld_bytes(s, m.meta + 2u, 2);
    m.flen = (uint32_t)ld_bytes(s, m.meta + 4u, 2);
    m.rows_off = m.meta + length;
    if ((!m.same_pos && m.spb == 0) || (!m.fix_len && m.vlb == 0) || m.spb == 3 || m.vlb == 3) return;
    if ((uint64_t)m.rows_off + (uint64_t)(m.spb + m.vlb) * b.row_count > b.size) return;
  }
  m.ok = 1;
}

// BitSet::get_ref (ob_encoding_bitset.h:68-71,131-149): rank of `row` among the exception rows, -1: not an exception
__device__ __forceinline__ int span_exc_rank(const uint8_t *s, const SpanCol &m, uint32_t row) {
  if (!m.exc) return -1;
  const uint32_t words = m.exc + 4u, wi = row >> 6, bit = row & 63u;
  const uint64_t w = ld_bytes(s, words + wi * 8u, 8);
  if (!((w >> bit) & 1ull)) return -1;
  int r = __popcll(w & ((1ull << bit) - 1ull));
  for (uint32_t k = 0; k < wi; ++k) r += __popcll(ld_bytes(s, words + k * 8u, 8));
  return r;
}

// One row of a span column: integers -> (value image, NULL); strings -> (block offset, length, NULL). false: corrupt.
// ObBitMapMetaReader::read / read_exc_cell for the exception rows, the referenced column's cell otherwise.
__device__ __forceinline__ bool span_row(const uint8_t *s, const BlockView &b, const SpanCol &m, uint32_t row, bool &is_null, uint64_t &ival,
                                         uint32_t &cell, uint32_t &len) {
  is_null = false;
  ival = 0;
  cell = len = 0;
  const int rank = span_exc_rank(s, m, row);
  if (rank >= 0) {
    const uint32_t eo = s[m.exc], io = s[m.exc + 1], dof = s[m.exc + 2], u = s[m.exc + 3], base = m.exc + 4u;
    if (io > eo) {   // has_ext_val: 2 bits per exception
      if (eo * 8u + (uint32_t)rank * 2u + 2u > io * 8u) return false;
      if (ld_bits32(s, (base + eo) * 8u + (uint32_t)rank * 2u, 2) != STORED_NOT_EXT) { is_null = true; return true; }
    }
    const uint32_t data = base + dof, data_len = m.exc_len - 4u - dof;
    if (m.sc != 5) {
      if (m.bit_packing) {
        if (u > 64u || ((uint64_t)rank + 1u) * u > (uint64_t)data_len * 8u) return false;
        ival = ld_bits(s, data * 8u + (uint32_t)rank * u, u);
      } else {
        const uint32_t cl = data_len / u;   // fix_data_cnt_ exceptions
        if (cl == 0 || cl > 8u || ((uint32_t)rank + 1u) * cl > data_len) return false;
        ival = sign_fix(m.int_mask, ld_bytes(s, data + (uint32_t)rank * cl, cl));
      }
      return true;
    }
    if (dof == io) {   // fixed-length exceptions
      len = data_len / u;
      cell = data + (uint32_t)rank * len;
    } else {
      if (u != 1 && u != 2 && u != 4) return false;
      const uint32_t cnt = (dof - io) / u + 1u;
      if ((uint32_t)rank >= cnt) return false;
      const uint32_t off = rank ? (uint32_t)ld_bytes(s, base + io + ((uint32_t)rank - 1u) * u, u) : 0u;
      const uint32_t end = (uint32_t)rank == cnt - 1u ? data_len : (uint32_t)ld_bytes(s, base + io + (uint32_t)rank * u, u);
      if (end < off) return false;
      cell = data + off;
      len = end - off;
    }
    return (uint64_t)cell + len <= (uint64_t)m.meta + m.length;
  }
  if (m.sc != 5) {
    ival = int_cell(b, m.ref, nullptr, row, is_null);
    return true;
  }
  str_cell(b, m.ref, nullptr, row, cell, len, is_null);
  if (is_null) { len = 0; return true; }
  if ((uint64_t)cell + len > b.size) return false;
  if (m.type == COL_COLUMN_SUBSTR) {
    const uint32_t at = m.rows_off + row * (uint32_t)(m.spb + m.vlb);
    const uint32_t start = m.same_pos ? m.start : (uint32_t)ld_bytes(s, at, m.spb);
    const uint32_t sub = m.fix_len ? m.flen : (uint32_t)ld_bytes(s, at + m.spb, m.vlb);
    if ((uint64_t)start + sub > len) return false;
    cell += start;
    len = sub;
  }
  return true;
}

__device__ __forceinline__ uint32_t span_int_area_bytes(uint32_t rows) {
  return ((((rows + 31u) / 32u * 4u + 7u) & ~7u) + rows * 8u + 16u + 15u) & ~15u;
}
__device__ __forceinline__ uint32_t str_area_bytes(uint32_t rows, uint64_t total) {
  const uint64_t n = (((uint64_t)(rows + 31u) / 32u) * 4u + (uint64_t)rows * 4u + total + 16u + 15u) & ~15ull;
  return n > 0x7fffff00ull ? 0xffffffffu : (uint32_t)n;
}

// Bytes of the area of span column `col` (every lane of the warp calls it; 0: the column cannot be materialised)
__device__ __forceinline__ uint32_t span_area_need(const uint8_t *s, const BlockView &b, int col, int lane) {
  SpanCol m;
  span_col_init(s, b, col, m);
  if (!m.ok) return 0;
  if (m.sc != 5) return span_int_area_bytes(b.row_count);
  uint64_t total = 0;
  bool bad = false;
  for (uint32_t row = (uint32_t)lane; row < b.row_count; row += 32u) {
    bool is_null;
    uint64_t iv;
    uint32_t cell, len;
    if (!span_row(s, b, m, row, is_null, iv, cell, len)) bad = true;
    else total += len;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
  if (__any_sync(0xffffffffu, bad)) return 0;
  const uint32_t n = str_area_bytes(b.row_count, total);
  return n == 0xffffffffu ? 0u : n;
}

// Does any block of the batch carry such a column? (one flag: the detailed survey and its copy back only run when it is set)
__global__ void __launch_bounds__(256) mat_probe_kernel(const uint8_t *image, const uint64_t *blk_off, const uint32_t *blk_size, int n_blocks,
                                                        uint32_t *flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_blocks) return;
  const uint8_t *s = image + blk_off[i];
  BlockView b;
  parse_block(s, blk_size[i], b);
  if (!b.ok || b.is_cs) return;
  for (uint32_t c = 0; c < b.column_count; ++c) {
    const uint32_t t = (ld32(s, b.header_size + 16u * c) >> 8) & 0xffu;
    if (obf::rebuilt_at_open(t)) { atomicOr(flag, MF_ANY); return; }
  }
}

// out[4 i ..]: size of the copy (the block, 16-byte aligned, + the areas), jobs, flags, 0. One warp per block: the lanes share the row
// loop that sizes a span column's strings.
__global__ void __launch_bounds__(128) mat_survey_kernel(const uint8_t *image, const uint64_t *blk_off, const uint32_t *blk_size, int n_blocks,
                                                         uint32_t *out) {
  const int i = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (i >= n_blocks) return;
  const uint8_t *s = image + blk_off[i];
  const uint32_t size = blk_size[i];
  BlockView b;
  parse_block(s, size, b);
  uint32_t total = (size + 15u) & ~15u, jobs = 0, flags = 0;
  if (b.ok && !b.is_cs) {
    for (uint32_t c = 0; c < b.column_count; ++c) {
      const uint32_t w0 = ld32(s, b.header_size + 16u * c), t = (w0 >> 8) & 0xffu;
      if (!obf::rebuilt_at_open(t)) continue;
      uint64_t need;
      if (is_span_type(t)) {
        need = span_area_need(s, b, (int)c, lane);
        if (need == 0) { flags |= MF_UNSUPPORTED; continue; }
      } else {
        CodecHdr h;
        read_codec_hdr(s, b, (int)c, h);
        if (!h.ok || s[h.meta] == kMatMarker) { flags |= MF_UNSUPPORTED; continue; }   // the index kernel leaves the column unsupported
        need = (uint64_t)area_bytes(b.row_count, h.max_len);
      }
      if ((uint64_t)total + need > 0x7fffff00ull) { flags |= MF_UNSUPPORTED; continue; }
      total += (uint32_t)need;
      ++jobs;
      flags |= MF_ANY;
    }
  }
  if (lane != 0) return;
  out[4 * i] = jobs ? total : size;   // an untouched block keeps its exact size (a CS block finds its stream offsets from its end)
  out[4 * i + 1] = jobs;
  out[4 * i + 2] = flags;
  out[4 * i + 3] = 0;
}

// One warp per block: copy it, then lane 0 lays the areas out behind it, patches the codec headers of the copy and lists the jobs.
__global__ void __launch_bounds__(128) mat_rewrite_kernel(const uint8_t *image, const uint64_t *blk_off, const uint32_t *blk_size, int n_blocks,
                                                          uint8_t *new_image, const uint64_t *new_off, const uint32_t *new_size,
                                                          const uint64_t *job_base, MatJob *jobs) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n_blocks) return;
  const uint8_t *s = image + blk_off[i];
  uint8_t *d = new_image + new_off[i];
  const uint32_t size = blk_size[i], padded = (size + 15u) & ~15u;
  const uint4 *s4 = reinterpret_cast<const uint4 *>(s);
  uint4 *d4 = reinterpret_cast<uint4 *>(d);
  for (uint32_t k = (uint32_t)lane; k < padded / 16u; k += 32u) d4[k] = s4[k];   // blocks are 16-byte aligned and padded in both images
  __syncwarp();
  if (new_size[i] <= padded) return;   // nothing materialised in this block
  BlockView b;
  parse_block(s, size, b);
  uint32_t at = padded;
  uint64_t j = job_base[i];
  for (uint32_t c = 0; c < b.column_count; ++c) {
    const uint32_t ch = b.header_size + 16u * c;
    const uint32_t t = (ld32(s, ch) >> 8) & 0xffu;
    if (!obf::rebuilt_at_open(t)) continue;
    if (is_span_type(t)) {   // the column header of the copy says where the area is
      const uint32_t need = span_area_need(s, b, (int)c, lane);
      if (need == 0) continue;
      if ((uint64_t)at + need > (uint64_t)new_size[i]) break;   // cannot happen: the survey walked the same columns
      if (lane == 0) {
        d[ch] = kMatMarker;
        *reinterpret_cast<uint32_t *>(d + ch + 8) = at;
        *reinterpret_cast<uint32_t *>(d + ch + 12) = need;
        jobs[j] = MatJob{blk_off[i], new_off[i], size, c, at, need};
      }
      ++j;
      at += need;
      continue;
    }
    CodecHdr h;
    read_codec_hdr(s, b, (int)c, h);
    if (!h.ok) continue;
    const uint32_t need = area_bytes(b.row_count, h.max_len);
    if ((uint64_t)at + need > (uint64_t)new_size[i]) break;
    if (lane == 0) {
      d[h.meta] = kMatMarker;
      d[h.pos_field] = (uint8_t)at; d[h.pos_field + 1] = (uint8_t)(at >> 8); d[h.pos_field + 2] = (uint8_t)(at >> 16); d[h.pos_field + 3] = (uint8_t)(at >> 24);
      jobs[j] = MatJob{blk_off[i], new_off[i], size, c, at, need};
    }
    ++j;
    at += need;
  }
}

__device__ __forceinline__ uint8_t hex_at(const uint8_t *s, uint32_t map, uint32_t data, uint32_t pos) {
  return s[map + ((s[data + pos / 2u] >> (((pos + 1u) & 1u) * 4u)) & 0xfu)];
}

// encoded cell of a row: fixed store right behind the codec meta, var store through the row index like a RAW var cell
struct MatCol {
  CodecHdr h;
  ColDesc var;          // K_VARSTR plan of the var-stored cell (codec header's row position)
  uint32_t fix_data;    // fixed store: block offset of cell 0
  uint32_t ext_bit_off; // fixed store: bit offset of the ext values
  uint32_t hex_map;     // block offset of the alphabet (0: none)
  uint32_t descs, n_descs, common;       // STRING_DIFF
  uint32_t pfx_index, pfx_ib, pfx_count; // STRING_PREFIX
  bool fixed, has_ext;
};

__device__ __forceinline__ bool mat_col_init(const uint8_t *s, const BlockView &b, int col, MatCol &m) {
  read_codec_hdr(s, b, col, m.h);
  if (!m.h.ok) return false;
  m.fixed = (m.h.attr & ATTR_FIX_LENGTH) != 0;
  m.has_ext = (m.h.attr & ATTR_HAS_EXTEND_VALUE) != 0;
  const uint32_t col_data = m.h.meta + m.h.length;
  m.ext_bit_off = col_data * 8u;
  m.fix_data = col_data + (m.has_ext ? ((uint32_t)b.ext_bit * b.row_count + 7u) / 8u : 0u);
  m.var = ColDesc{};
  m.var.kind = K_VARSTR;
  m.var.sc = 5;
  m.var.ok = 1;
  m.var.var_ext_in_row = m.has_ext;
  m.var.ext_bit = m.has_ext ? b.ext_bit : 0;
  m.var.ext_index = ld32(s, b.header_size + 16u * (uint32_t)col + 4u);
  m.var.var_header_off = m.h.pos_off;
  m.var.var_k = m.h.pos_len;
  m.var.var_is_last = (m.h.attr & ATTR_LAST_VAR_FIELD) != 0;
  m.hex_map = m.descs = m.n_descs = m.common = m.pfx_index = m.pfx_ib = m.pfx_count = 0;
  if (m.h.type == COL_HEX_PACKING) {
    m.hex_map = m.h.meta + 13u;
  } else if (m.h.type == COL_STRING_DIFF) {
    const uint32_t hex_size = s[m.h.meta + 1u];
    m.n_descs = s[m.h.meta + 12u];
    m.descs = m.h.meta + 13u;
    m.hex_map = hex_size ? m.descs + m.n_descs : 0u;
    m.common = m.descs + m.n_descs + hex_size;
    if (m.common > m.h.meta + m.h.length) return false;
  } else {
    m.pfx_count = s[m.h.meta + 1u];
    m.pfx_ib = s[m.h.meta + 14u] & 3u;
    const uint32_t hex_size = (s[m.h.meta + 14u] >> 2) & 0x1fu;
    m.hex_map = hex_size ? m.h.meta + 15u : 0u;
    m.pfx_index = m.h.meta + 15u + hex_size;
    m.common = m.pfx_index + (m.pfx_count ? m.pfx_count - 1u : 0u) * m.pfx_ib;
    if (m.pfx_count == 0 || (m.pfx_count > 1 && m.pfx_ib != 1 && m.pfx_ib != 2) || m.common > m.h.meta + m.h.length) return false;
  }
  if (!m.fixed && b.row_index_byte == 0) return false;
  return true;
}

// (cell, cell length, NULL) of a row, then the length of the rebuilt string; false: the block is corrupt
__device__ __forceinline__ bool mat_row(const uint8_t *s, const BlockView &b, const MatCol &m, uint32_t row, uint32_t &cell, uint32_t &clen,
                                        bool &is_null, uint32_t &len) {
  is_null = false;
  len = 0;
  if (m.fixed) {
    if (m.has_ext && ld_bits32(s, m.ext_bit_off + row * b.ext_bit, b.ext_bit) != STORED_NOT_EXT) { is_null = true; return true; }
    clen = m.h.pos_len;
    cell = m.fix_data + row * clen;
  } else {
    str_cell(b, m.var, nullptr, row, cell, clen, is_null);
    if (is_null) return true;
  }
  if ((uint64_t)cell + clen > b.size) return false;
  if (m.h.type == COL_HEX_PACKING) {
    if (m.fixed) len = m.h.max_len;
    else {
      if (clen < 1u) return false;
      len = (clen - 1u) * 2u - s[cell];
    }
  } else if (m.h.type == COL_STRING_DIFF) {
    len = m.h.max_len;
  } else {
    if (clen < 3u) return false;
    const uint32_t odd = s[cell] >> 4, common = (uint32_t)s[cell + 1] | ((uint32_t)s[cell + 2] << 8);
    len = common + (m.hex_map ? (clen - 3u) * 2u - odd : clen - 3u);
  }
  return len <= m.h.max_len;
}

__device__ __forceinline__ bool mat_write(const uint8_t *s, const BlockView &b, const MatCol &m, uint32_t cell, uint32_t clen, uint32_t len,
                                          uint8_t *dst) {
  if (m.h.type == COL_HEX_PACKING) {
    const uint32_t data = m.fixed ? cell : cell + 1u;
    for (uint32_t i = 0; i < len; ++i) dst[i] = hex_at(s, m.hex_map, data, i);
    return true;
  }
  if (m.h.type == COL_STRING_DIFF) {
    uint32_t fpos = 0, cpos = 0, ppos = 0;   // position in the string, in the common bytes, in the row's part
    for (uint32_t i = 0; i < m.n_descs; ++i) {
      const uint32_t diff = s[m.descs + i] & 1u, cnt = s[m.descs + i] >> 1;
      if (fpos + cnt > len) return false;
      for (uint32_t k = 0; k < cnt; ++k, ++fpos) {
        if (!diff) dst[fpos] = s[m.common + cpos++];
        else { dst[fpos] = m.hex_map ? hex_at(s, m.hex_map, cell, ppos) : s[cell + ppos]; ++ppos; }
      }
    }
    return fpos == len && (m.hex_map ? (ppos + 1u) / 2u : ppos) <= clen;
  }
  const uint32_t ref = s[cell] & 0xfu, common = (uint32_t)s[cell + 1] | ((uint32_t)s[cell + 2] << 8);
  if (ref >= m.pfx_count) return false;
  const uint32_t poff = ref ? (uint32_t)ld_bytes(s, m.pfx_index + (ref - 1u) * m.pfx_ib, m.pfx_ib) : 0u;
  if ((uint64_t)m.common + poff + common > (uint64_t)m.h.meta + m.h.length) return false;
  for (uint32_t i = 0; i < common; ++i) dst[i] = s[m.common + poff + i];
  const uint32_t rest = len - common;
  if (m.hex_map) for (uint32_t i = 0; i < rest; ++i) dst[common + i] = hex_at(s, m.hex_map, cell + 3u, i);
  else for (uint32_t i = 0; i < rest; ++i) dst[common + i] = s[cell + 3u + i];
  return true;
}

// A span column's area, by one warp: integers -> [NULL bits][value images]; strings -> [NULL bits][END offsets][bytes]
__device__ __forceinline__ void span_decode(const uint8_t *s, const BlockView &b, const MatJob &job, uint8_t *area, int lane, int *status) {
  SpanCol m;
  span_col_init(s, b, (int)job.col, m);
  if (!m.ok) {
    if (lane == 0) atomicOr(status, (int)MF_CORRUPT);
    return;
  }
  const uint32_t rows = b.row_count, nwords = (rows + 31u) / 32u;
  uint32_t *null_words = reinterpret_cast<uint32_t *>(area);
  bool bad = false;
  if (m.sc != 5) {
    uint64_t *vals = reinterpret_cast<uint64_t *>(area + ((nwords * 4u + 7u) & ~7u));
    for (uint32_t r0 = 0; r0 < rows; r0 += 32u) {
      const uint32_t row = r0 + (uint32_t)lane;
      bool is_null = false;
      uint64_t iv = 0;
      uint32_t cell, len;
      if (row < rows && !span_row(s, b, m, row, is_null, iv, cell, len)) bad = true;
      const uint32_t nb = __ballot_sync(0xffffffffu, row < rows && is_null);
      if (lane == 0) null_words[r0 >> 5] = nb;
      if (row < rows) vals[row] = is_null ? 0ull : iv;
    }
  } else {
    uint32_t *ends = reinterpret_cast<uint32_t *>(area + nwords * 4u);
    uint8_t *bytes = area + nwords * 4u + rows * 4u;
    const uint32_t cap = job.area_cap - nwords * 4u - rows * 4u;
    uint32_t run = 0;
    for (uint32_t r0 = 0; r0 < rows; r0 += 32u) {
      const uint32_t row = r0 + (uint32_t)lane;
      bool is_null = false;
      uint64_t iv;
      uint32_t cell = 0, len = 0;
      if (row < rows && !span_row(s, b, m, row, is_null, iv, cell, len)) { bad = true; len = 0; }
      uint32_t inc = len;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += u;
      }
      const uint32_t end = run + inc;
      const uint32_t nb = __ballot_sync(0xffffffffu, row < rows && is_null);
      if (lane == 0) null_words[r0 >> 5] = nb;
      if (row < rows) {
        if (end > cap) bad = true;
        else {
          ends[row] = end;
          uint8_t *dst = bytes + (end - len);
          for (uint32_t k = 0; k < len; ++k) dst[k] = s[cell + k];
        }
      }
      run += __shfl_sync(0xffffffffu, inc, 31);
    }
  }
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(status, (int)MF_CORRUPT);
}

// One warp per (block, column): lengths -> END offsets (a warp scan per 32 rows, the running total carried), NULL bits by ballot,
// then every lane rebuilds its rows' strings at their offsets.
__global__ void __launch_bounds__(128) mat_decode_kernel(const uint8_t *image, uint8_t *new_image, const MatJob *jobs, int64_t n_jobs, int *status) {
  const int64_t j = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= n_jobs) return;
  const MatJob job = jobs[j];
  const uint8_t *s = image + job.old_off;
  BlockView b;
  parse_block(s, job.old_size, b);
  if (b.ok && !b.is_cs && job.col < b.column_count && is_span_type((ld32(s, b.header_size + 16u * job.col) >> 8) & 0xffu)) {
    span_decode(s, b, job, new_image + job.new_off + job.area_off, lane, status);
    return;
  }
  MatCol m;
  if (!b.ok || b.is_cs || !mat_col_init(s, b, (int)job.col, m)) {
    if (lane == 0) atomicOr(status, (int)MF_CORRUPT);
    return;
  }
  uint8_t *area = new_image + job.new_off + job.area_off;
  const uint32_t rows = b.row_count, nwords = (rows + 31u) / 32u;
  uint32_t *null_words = reinterpret_cast<uint32_t *>(area);
  uint32_t *ends = reinterpret_cast<uint32_t *>(area + nwords * 4u);
  uint8_t *bytes = area + nwords * 4u + rows * 4u;
  const uint32_t cap = job.area_cap - nwords * 4u - rows * 4u;
  uint32_t run = 0;
  bool bad = false;
  for (uint32_t r0 = 0; r0 < rows; r0 += 32u) {
    const uint32_t row = r0 + (uint32_t)lane;
    uint32_t cell = 0, clen = 0, len = 0;
    bool is_null = false;
    if (row < rows && !mat_row(s, b, m, row, cell, clen, is_null, len)) { bad = true; len = 0; }
    uint32_t inc = len;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += u;
    }
    const uint32_t end = run + inc;
    const uint32_t nb = __ballot_sync(0xffffffffu, row < rows && is_null);
    if (lane == 0) null_words[r0 >> 5] = nb;
    if (row < rows) {
      if (end > cap) bad = true;
      else {
        ends[row] = end;
        if (len && !is_null && !bad && !mat_write(s, b, m, cell, clen, len, bytes + (end - len))) bad = true;
      }
    }
    run += __shfl_sync(0xffffffffu, inc, 31);
  }
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(status, (int)MF_CORRUPT);
}

}  // namespace obmat
