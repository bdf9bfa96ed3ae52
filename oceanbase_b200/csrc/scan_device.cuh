// Device-side micro-block decode primitives (sm_90a).
//
// A micro-block (one "page", ~16 KiB) is staged into shared memory by one TMA bulk copy; every
// primitive below reads the block image out of shared memory with 32-bit aligned loads and
// funnel shifts. All addressing is bit-granular (byte-aligned fields are the 8*n-bit special
// case), which gives one uniform load path for bit-packed values, byte-packed values, dictionary
// references and dictionary entries.
//
// Reference loops these replace (file:line in /root/reference/src/storage/blocksstable):
//   K1 bit unpack        encoding/ob_bit_stream.h:169-283
//   K2 RAW fixed load    encoding/ob_raw_decoder.cpp:128-173,530-591
//   K3 RAW var locate    encoding/ob_raw_decoder.cpp:29-125, ob_icolumn_decoder.h:463-527
//   K5 DICT gather       encoding/ob_dict_decoder.cpp:26-120,243-314
//   K7 RLE lookup        encoding/ob_rle_decoder.cpp:25-49,528-583
//   K8 base-diff         encoding/ob_integer_base_diff_decoder.cpp:25-82, .h:140-170
//   K9 ext (NULL) bits   encoding/ob_icolumn_decoder.h:259-318
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "ob_format.h"

namespace obdev {

using namespace obf;

constexpr int kMaxUsedCols = 24;   // distinct columns referenced by one scan (filter U projection)
constexpr int kMaxNodes = 16;      // filter tree nodes
constexpr int kMaxParams = 48;     // filter constants
constexpr int kMaxProj = 24;       // projected columns
constexpr int kThreads = 128;      // threads per CTA (4 warps): many small CTAs per SM hide the per-block latency chain
constexpr int kWarps = kThreads / 32;

// status bits written by kernels
enum : int { ST_UNSUPPORTED = 1, ST_OVERFLOW = 2, ST_CORRUPT = 4 };

// white-filter ops (sql::ObWhiteFilterOperatorType) + two host-resolved constants
enum : int { OP_EQ = 0, OP_LE, OP_LT, OP_GE, OP_GT, OP_NE, OP_BT, OP_IN, OP_NU, OP_NN,
             OP_FALSE = 100, OP_TRUE = 101 };
enum : int { NODE_WHITE = 0, NODE_AND = 1, NODE_OR = 2 };

// ---- loads from the shared-memory block image ---------------------------------------------------
// `s` is 16-byte aligned and has >= 16 readable bytes of slack after the block.
__device__ __forceinline__ uint32_t ld32(const uint8_t *s, uint32_t word_byte_off) {
  return *reinterpret_cast<const uint32_t *>(s + word_byte_off);
}

// w bits (1..32) at absolute bit offset (LSB-first stream, ObBitStream::get)
__device__ __forceinline__ uint32_t ld_bits32(const uint8_t *s, uint32_t bit_off, uint32_t w) {
  const uint32_t a = (bit_off >> 5) << 2, sh = bit_off & 31u;
  const uint32_t lo = __funnelshift_r(ld32(s, a), ld32(s, a + 4), sh);
  return lo & (0xffffffffu >> (32u - w));
}

// w bits (1..64)
__device__ __forceinline__ uint64_t ld_bits(const uint8_t *s, uint32_t bit_off, uint32_t w) {
  const uint32_t a = (bit_off >> 5) << 2, sh = bit_off & 31u;
  const uint32_t w0 = ld32(s, a), w1 = ld32(s, a + 4);
  const uint32_t lo = __funnelshift_r(w0, w1, sh);
  if (w <= 32) return (uint64_t)(lo & (0xffffffffu >> (32u - w)));
  const uint32_t hi = __funnelshift_r(w1, ld32(s, a + 8), sh);
  return (((uint64_t)hi << 32) | lo) & (~0ull >> (64u - w));
}

// Same loads on shared-window addresses (bit offset = 8 * 32-bit shared address): explicit
// ld.shared keeps the compiler from re-deriving the generic->shared base inside hot loops.
extern __shared__ __align__(128) uint8_t g_smem[];
__device__ __forceinline__ uint32_t sld32(uint32_t saddr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr));
  return v;
}
__device__ __forceinline__ uint32_t sbits32(uint32_t bit_off, uint32_t w) {
  const uint32_t a = (bit_off >> 5) << 2, sh = bit_off & 31u;
  return __funnelshift_r(sld32(a), sld32(a + 4), sh) & (0xffffffffu >> (32u - w));
}
__device__ __forceinline__ uint64_t sbits(uint32_t bit_off, uint32_t w) {
  const uint32_t a = (bit_off >> 5) << 2, sh = bit_off & 31u;
  const uint32_t w0 = sld32(a), w1 = sld32(a + 4);
  const uint32_t lo = __funnelshift_r(w0, w1, sh);
  if (w <= 32) return (uint64_t)(lo & (0xffffffffu >> (32u - w)));
  const uint32_t hi = __funnelshift_r(w1, sld32(a + 8), sh);
  return (((uint64_t)hi << 32) | lo) & (~0ull >> (64u - w));
}

// n bytes (1..8) at byte offset off, zero extended
__device__ __forceinline__ uint64_t ld_bytes(const uint8_t *s, uint32_t off, uint32_t n) {
  return ld_bits(s, off * 8u, n * 8u);
}

// ---- per-column decode descriptor, built once per block per referenced column -----------------
enum ColKind : uint8_t {
  K_NONE = 0,
  K_BITS,     // value = ld_bits(val_bit + row * stride, width) [+ base] : RAW fixed/bit-packed, BASE_DIFF
  K_DICT,     // ref   = ld_bits32(val_bit + row * stride, width), then dictionary
  K_RLE,      // ref   = refs[run_of(row)], then dictionary
  K_VARSTR,   // RAW var-length string in the row data
  K_FIXSTR,   // RAW fixed-length string
  K_CONST,    // ref   = exception ref if the row is in the exception list, else const_ref; then dictionary
  K_CSSTR,    // CS STRING, variable length: END offset per row (dict_payload, dict_data_size bytes each), bytes at dict_var
};

struct alignas(16) ColDesc {
  uint8_t kind;        // ColKind
  uint8_t type;        // ColType
  uint8_t attr;        // ColAttr
  uint8_t obj_type;
  uint8_t sc;          // 1 signed int class, 2 unsigned int class, 5 string
  uint8_t elem_len;    // datum length of integer classes (8 / 4 / 1)
  uint8_t ext_bit;     // extend_value_bit if the column stores ext bits, else 0
  uint8_t ok;          // 0 => unsupported encoding / type for the device path
  uint8_t width;       // value / ref width in bits
  uint8_t sign_fix;    // apply the ObIntTC sign-extension mask after the load
  uint8_t dict_fixed;
  uint8_t var_is_last; // RAW var: LAST_VAR_FIELD
  uint32_t stride;     // bits between consecutive rows' values / refs
  uint32_t val_bit;    // bit offset of value / ref 0
  uint32_t ext_bit_off;// bit offset of ext value 0
  uint64_t base;       // BASE_DIFF base
  uint64_t int_mask;   // ~INTEGER_MASK_TABLE[type_store_size] for ObIntTC, else 0
  // dictionary (DICT / RLE)
  uint32_t dict_payload;   // block byte offset of the dict payload (after the 9-byte meta header)
  uint32_t dict_var;       // block byte offset of var data (var dict)
  uint32_t dict_end;       // block byte offset one past the dict meta (last var cell ends here)
  uint32_t dict_count;
  uint32_t dict_data_size; // fixed: bytes per entry (also RAW fixed string length); var: index_byte
  // RLE
  uint32_t rle_count;
  uint32_t rle_refs_bit;   // bit offset of ref 0
  uint32_t rle_row_ids_bit;
  uint8_t rle_row_id_bits, rle_ref_bits;
  uint8_t var_ext_in_row;  // RAW var: ext bits inside each row at bit ext_index
  int8_t rle_slot;         // run-table scratch slot (-1: none)
  // RAW var-length cells in the row data
  uint32_t var_header_off; // bytes of per-row ext bits (row_offset_)
  uint32_t var_k;          // index among the var columns
  uint32_t ext_index;
  // CONST: exception list in rle_count / rle_row_ids_bit / rle_row_id_bits / rle_refs_bit (8-bit refs)
  uint32_t const_ref;
  uint8_t dict_sorted;     // ObDictMetaHeader::IS_SORTED on a fixed-length dictionary: entries ascend in the column's order
  uint8_t pad_[3];
};
static_assert(sizeof(ColDesc) == 96, "ColDesc layout is shared by the index kernel and the scan kernels");

// K_BITS columns of CS_ENCODING_ROW_STORE blocks reuse the (otherwise RAW-var-only) fields:
//   var_ext_in_row -> XOR applied to the row index of an ext lookup (7: the CS null bitmap is MSB-first
//                     per byte, so bit `row` of it is bit `row ^ 7` of an LSB-first stream; 0 for PAX)
//   var_is_last    -> 1: NULL is a replaced value (ObIntegerStreamMeta REPLACE_NULL_VALUE)
//   var_header_off / var_k -> low / high half of the raw value that stands for NULL (null_replaced - base)
__device__ __forceinline__ uint32_t ext_row(const ColDesc &d, uint32_t row) { return row ^ (uint32_t)d.var_ext_in_row; }
__device__ __forceinline__ bool null_replaced_on(const ColDesc &d) { return d.kind == K_BITS && d.var_is_last != 0; }
__device__ __forceinline__ uint64_t null_replaced_raw(const ColDesc &d) {
  return ((uint64_t)d.var_k << 32) | (uint64_t)d.var_header_off;
}

// CS string columns (STRING / STR_DICT) keep their bytes in the block's all-string-data area, outside the
// column's own meta + streams: no single region covers them (see col_region). K_CSSTR / CS K_FIXSTR use
// var_ext_in_row like K_BITS (MSB-first NULL bitmap) and var_is_last = 1 for "a zero-length value is NULL".
__device__ __forceinline__ bool cs_bytes_outside(const ColDesc &d) { return d.type == 101 || d.type == 103; }

__device__ __forceinline__ bool is_dict_kind(const ColDesc &d) {
  return d.kind == K_DICT || d.kind == K_RLE || d.kind == K_CONST;
}

struct BlockView {
  const uint8_t *s;        // shared-memory image
  uint32_t size;
  uint32_t row_count;
  uint32_t header_size;
  uint32_t column_count;
  uint32_t meta_off;       // header + column headers
  uint32_t row_data_off;
  uint32_t row_index_off;  // start of the row index array (var row index)
  uint8_t row_index_byte, ext_bit;
  uint16_t var_col_cnt;
  uint8_t ok;
  uint8_t is_cs;           // CS_ENCODING_ROW_STORE block: the fields below replace the PAX ones
  uint16_t cs_stream_count;
  uint32_t cs_first_stream_begin;  // header + ObAllColumnHeader + ObCSColumnHeader x ncol
  uint32_t cs_off_data;            // block offset of the stream end offsets array
  uint32_t cs_off_width;           // bytes per stream end offset
};

// Per-block record written once at batch open by the index kernel: everything the scan kernels
// need to address a block and rebuild its BlockView with ONE dependent-free 48-byte load (instead
// of a chain of table lookups followed by a header parse).
struct alignas(16) BlockRec {
  uint64_t off;           // byte offset of the block in the image
  int64_t bm_word_off;    // first word of the block in the packed selection bitmap
  uint32_t size;
  uint32_t rows;          // 0: header rejected
  uint32_t row_data_off;
  uint32_t row_index_off;
  uint32_t header_size;
  uint16_t column_count;
  uint16_t var_col_cnt;
  uint8_t row_index_byte, ext_bit;
  uint8_t pad[6];
};
static_assert(sizeof(BlockRec) == 48, "BlockRec is loaded as three 16-byte pieces");

// Per (block, column) stage record, written at batch open next to the plan by the index kernel for batches that can take
// the small-block pipelined kernels (scan_small.cuh): the byte ranges a projection stages (proj_ranges) and the fields the
// lean filter leaves and the flat projection read, so those kernels copy 32 bytes per column and block instead of the
// 96-byte plan and never run col_region / proj_ranges. Offsets are block relative, as in the plan.
enum : uint8_t { SR_DICT = 1, SR_SORTED = 2, SR_SIGN_FIX = 4 };
enum : uint32_t { SR_NOT_FILTER = 1, SR_NOT_FLAT = 2 };   // per-column reduction over the blocks (index kernel)
struct alignas(16) StageRec {
  uint64_t add;           // K_BITS / integer dictionary: the plan's base; string dictionary: dict_var
  uint32_t val_bit;       // bit offset of value / ref 0
  uint32_t dict_payload;  // byte offset of dictionary entry 0 (string dictionary: END offset 0)
  uint16_t lo[2], hi[2];  // projection ranges [16 lo, 16 hi); lo[1] == hi[1]: one range. A filter stages [16 lo[0], 16 max(hi))
  uint16_t dict_count;
  uint16_t last_end;      // string dictionary: dict_end - dict_var
  uint8_t width, stride, dict_data_size, flags;   // flags: SR_DICT (else K_BITS), SR_SORTED, SR_SIGN_FIX
};
static_assert(sizeof(StageRec) == 32, "StageRec is loaded as two 16-byte pieces");

__device__ __forceinline__ void view_from_rec(const BlockRec &r, const uint8_t *s, BlockView &b) {
  b.s = s;
  b.size = r.size;
  b.row_count = r.rows;
  b.header_size = r.header_size;
  b.column_count = r.column_count;
  b.meta_off = r.header_size + 16u * r.column_count;
  b.row_data_off = r.row_data_off;
  b.row_index_off = r.row_index_off;
  b.row_index_byte = r.row_index_byte;
  b.ext_bit = r.ext_bit;
  b.var_col_cnt = r.var_col_cnt;
  b.ok = r.rows > 0;
  b.is_cs = r.pad[0];   // the scan kernels work from the plans: the CS stream tables are not needed again
  b.cs_stream_count = 0;
  b.cs_first_stream_begin = b.cs_off_data = b.cs_off_width = 0;
}

// ObIntegerStreamMeta, serialized (cs_encoding/ob_stream_encoding_struct.cpp:27-77)
struct IntStreamMeta {
  uint32_t width;      // bytes
  uint32_t meta_len;
  uint64_t base, null_replaced;
  uint8_t use_base, replace_null, ok;
};
__device__ __forceinline__ bool rd_vi64(const uint8_t *s, uint32_t &pos, uint32_t end, uint64_t &v) {
  uint64_t r = 0;
  int shift = 0;
  while (pos < end && shift <= 63) {
    const uint8_t c = s[pos++];
    r |= (uint64_t)(c & 0x7f) << shift;
    if (!(c & 0x80)) { v = r; return true; }
    shift += 7;
  }
  return false;
}
__device__ __forceinline__ void parse_int_stream_meta(const uint8_t *s, uint32_t at, uint32_t end, IntStreamMeta &m) {
  m = IntStreamMeta{};
  if (at + 4u > end) return;
  const uint8_t version = s[at], attr = s[at + 1], type = s[at + 2], wtag = s[at + 3];
  uint32_t pos = at + 4u;
  m.use_base = attr & IS_USE_BASE;
  m.replace_null = (attr & IS_REPLACE_NULL_VALUE) != 0;
  if (m.use_base && !rd_vi64(s, pos, end, m.base)) return;
  if (m.replace_null && !rd_vi64(s, pos, end, m.null_replaced)) return;
  if (attr & IS_DECIMAL_INT) return;
  if (version > 0) { if (pos >= end) return; ++pos; }
  if (wtag > 3 || type != IS_RAW) return;   // the other stream codecs need the CPU transformer
  m.width = 1u << wtag;
  m.meta_len = pos - at;
  m.ok = 1;
}

// ObStringStreamMeta, serialized (ob_stream_encoding_struct.cpp:255-283): version, attr (1 zero length is NULL,
// 2 fixed length), vi32 uncompressed_len, [vi32 fixed_len]
struct StrStreamMeta {
  uint32_t uncompressed_len, fixed_len;
  uint8_t zero_len_null, fixed, ok;
};
__device__ __forceinline__ void parse_str_stream_meta(const uint8_t *s, uint32_t at, uint32_t end, StrStreamMeta &m) {
  m = StrStreamMeta{};
  if (at + 3u > end || s[at] != 0) return;
  uint32_t pos = at + 2u;
  uint64_t v = 0;
  m.zero_len_null = s[at + 1] & 0x1;
  m.fixed = (s[at + 1] & 0x2) != 0;
  if (!rd_vi64(s, pos, end, v) || v > 0xffffffffull) return;
  m.uncompressed_len = (uint32_t)v;
  if (m.fixed) {
    if (!rd_vi64(s, pos, end, v) || v > 0xffffull) return;
    m.fixed_len = (uint32_t)v;
  }
  m.ok = 1;
}

// CS block: ObCSMicroBlockTransformer::init / decode_stream_offsets_ (ob_cs_micro_block_transformer.cpp:106-202)
__device__ __forceinline__ void parse_cs_block(const uint8_t *s, uint32_t size, int16_t magic, int16_t version, BlockView &b) {
  b.is_cs = 1;
  b.ok = 0;
  b.row_index_off = 0;
  b.row_index_byte = b.ext_bit = 0;
  b.var_col_cnt = 0;
  b.row_data_off = size;
  if (magic != MICRO_BLOCK_HEADER_MAGIC || version < 1 || version > 3 || b.header_size < 64 || b.row_count == 0) return;
  const uint32_t ah = b.header_size;
  b.meta_off = ah + 12u + 4u * b.column_count;   // ObAllColumnHeader + ObCSColumnHeader x ncol
  if (b.meta_off > size) return;
  if (s[ah] != 0 || (s[ah + 1] & 0x3)) return;  // transformed / compressed string data: not handled
  const uint32_t all_string_len = (uint32_t)ld_bytes(s, ah + 2, 4);
  const uint32_t offsets_len = (uint32_t)ld_bytes(s, ah + 6, 4);
  b.cs_stream_count = (uint16_t)ld_bytes(s, ah + 10, 2);
  b.cs_first_stream_begin = b.meta_off;
  if (offsets_len > size - b.meta_off || all_string_len > size - b.meta_off - offsets_len) return;
  b.row_data_off = size - offsets_len - all_string_len;   // CS: start of the all-string-data area
  if (b.cs_stream_count > 0) {
    IntStreamMeta m;
    parse_int_stream_meta(s, size - offsets_len, size, m);
    if (!m.ok || m.use_base || m.width > 4) return;
    if (m.meta_len + m.width * b.cs_stream_count != offsets_len) return;
    b.cs_off_data = size - offsets_len + m.meta_len;
    b.cs_off_width = m.width;
  }
  b.ok = 1;
}

__device__ __forceinline__ void parse_block(const uint8_t *s, uint32_t size, BlockView &b) {
  b.s = s;
  b.size = size;
  const uint32_t w0 = ld32(s, 0);
  const int16_t magic = (int16_t)(w0 & 0xffff), version = (int16_t)(w0 >> 16);
  b.header_size = ld32(s, 4);
  b.column_count = ld32(s, 8) >> 16;
  b.row_count = ld32(s, 16);
  const uint32_t w5 = ld32(s, 20);
  const uint32_t row_store_type = w5 & 0xff, opt = (w5 >> 8) & 0xff;
  b.var_col_cnt = (uint16_t)(w5 >> 16);
  b.row_index_byte = opt & 7;
  b.ext_bit = (opt >> 3) & 7;
  b.row_data_off = ld32(s, 24);
  b.meta_off = b.header_size + 16u * b.column_count;
  b.is_cs = 0;
  b.cs_stream_count = 0;
  b.cs_first_stream_begin = b.cs_off_data = b.cs_off_width = 0;
  if (row_store_type == CS_ENCODING_ROW_STORE) {
    parse_cs_block(s, size, magic, version, b);
    return;
  }
  b.ok = magic == MICRO_BLOCK_HEADER_MAGIC && version >= 1 && version <= 3 &&
         (row_store_type == ENCODING_ROW_STORE || row_store_type == SELECTIVE_ENCODING_ROW_STORE) &&
         b.meta_off <= size && b.row_data_off <= size && b.header_size >= 64 && b.row_count > 0;
  b.row_index_off = 0;
  if (b.ok && b.row_index_byte > 0) {
    const uint32_t need = (uint32_t)b.row_index_byte * (b.row_count + 1);
    // the row index closes the block PROPER, header_size_ + data_length_ bytes; a page batch's own copy of a block may carry
    // materialised string areas behind it (mat_codecs.cuh), so `size` can be larger than that
    uint32_t end = size;
    const uint32_t logical = b.header_size + ld32(s, 40);
    if (logical < size && logical >= b.row_data_off) end = logical;
    if (need > end - b.row_data_off) b.ok = 0;
    else b.row_index_off = end - need;
  }
}

// Const-encoded dictionary refs (ObDictColumnEncoder::do_store_dict_ref_, cs_encoding/ob_dict_column_encoder.h:65-116;
// ObConstEncodingRefDesc, ob_dict_column_decoder.h:73-95): the ref stream holds
// [exception count][const ref][exception row ids x count][exception refs x count] instead of one ref per row.
// It is the PAX CONST codec's shape: a K_CONST plan over the column's dictionary.
__device__ __forceinline__ bool cs_const_ref_plan(const uint8_t *s, uint32_t data, uint32_t end, uint32_t width, uint32_t ref_cnt,
                                                  uint32_t row_count, ColDesc &d) {
  if (ref_cnt < 2 || data + width * ref_cnt != end) return false;
  const uint32_t exc = (uint32_t)ld_bytes(s, data, width);
  if (ref_cnt != 2u + 2u * exc || exc > row_count) return false;
  d.kind = K_CONST;
  d.const_ref = (uint32_t)ld_bytes(s, data + width, width);
  d.rle_count = exc;
  d.rle_row_id_bits = (uint8_t)(width * 8u);
  d.rle_ref_bits = (uint8_t)(width * 8u);
  d.rle_row_ids_bit = (data + 2u * width) * 8u;
  d.rle_refs_bit = (data + 2u * width + exc * width) * 8u;
  return true;
}

// CS STRING / STR_DICT column (cs_encoding/ob_string_column_decoder.cpp, ob_dict_column_decoder.cpp:158-326).
// pos: the column's meta (NULL bitmap or ObDictEncodingMeta), str_at: its bytes in the all-string-data area,
// send: end of the string stream (= start of the next stream of this column), next_stream: index of that stream.
__device__ __forceinline__ void build_cs_str_col_desc(const BlockView &b, uint32_t w, uint32_t pos, uint32_t str_at, uint32_t send,
                                                      int next_stream, const StrStreamMeta &sm, ColDesc &d) {
  const uint8_t *s = b.s;
  const uint32_t type = (w >> 8) & 0xff, attrs = (w >> 16) & 0xff;
  d.type = (uint8_t)(100 + type);
  d.attr = (uint8_t)attrs;
  d.obj_type = (uint8_t)(w >> 24);
  if (store_class_of(d.obj_type) != 5 || (attrs & (CS_HAS_NOP_BITMAP | CS_HAS_NOP | CS_OUT_ROW))) return;
  d.sc = 5;
  if (sm.fixed != ((attrs & CS_IS_FIXED_LENGTH) != 0)) return;
  const uint32_t count = type == CS_STRING ? b.row_count : (uint32_t)ld_bytes(s, pos + 2, 4);
  uint32_t at = send;
  uint32_t off_data = 0, off_w = 0;
  if (sm.fixed) {
    if ((uint64_t)sm.fixed_len * count != sm.uncompressed_len) return;
  } else {  // END offset per value: RAW integer stream, no base
    if (next_stream >= (int)b.cs_stream_count) return;
    const uint32_t oend = (uint32_t)ld_bytes(s, b.cs_off_data + (uint32_t)next_stream * b.cs_off_width, b.cs_off_width);
    if (oend < at || oend > b.size) return;
    IntStreamMeta m;
    parse_int_stream_meta(s, at, oend, m);
    if (!m.ok || m.use_base || m.replace_null || m.width > 4) return;
    if (at + m.meta_len + m.width * count != oend) return;
    off_data = at + m.meta_len;
    off_w = m.width;
    at = oend;
    ++next_stream;
  }
  if (type == CS_STRING) {
    if (attrs & CS_HAS_NULL_OR_NOP_BITMAP) {
      d.ext_bit = 1;
      d.ext_bit_off = pos * 8u;
      d.var_ext_in_row = 7;
    }
    d.var_is_last = sm.zero_len_null;
    if (sm.fixed) {
      d.kind = K_FIXSTR;
      d.dict_data_size = sm.fixed_len;
      d.val_bit = str_at;
    } else {
      d.kind = K_CSSTR;
      d.dict_count = count;
      d.dict_payload = off_data;
      d.dict_data_size = off_w;
      d.dict_var = str_at;
      d.dict_end = str_at + sm.uncompressed_len;
    }
    d.ok = 1;
    return;
  }
  // STR_DICT: [ObDictEncodingMeta][string stream meta][END offsets x distinct (variable)][refs x rows]
  if (s[pos] != 0) return;
  const bool const_refs = (s[pos + 1] & 0x4) != 0;   // ObDictEncodingMeta::CONST_ENCODING_REF
  if (next_stream >= (int)b.cs_stream_count) return;
  const uint32_t rend = (uint32_t)ld_bytes(s, b.cs_off_data + (uint32_t)next_stream * b.cs_off_width, b.cs_off_width);
  if (rend < at || rend > b.size) return;
  IntStreamMeta m;
  parse_int_stream_meta(s, at, rend, m);
  if (!m.ok || m.use_base || m.replace_null || m.width > 4) return;
  d.kind = K_DICT;
  d.dict_count = count;
  if (const_refs) {
    if (!cs_const_ref_plan(s, at + m.meta_len, rend, m.width, (uint32_t)ld_bytes(s, pos + 6, 4), b.row_count, d)) return;
  } else {
    if (at + m.meta_len + m.width * b.row_count != rend) return;
    d.width = (uint8_t)(m.width * 8u);
    d.stride = m.width * 8u;
    d.val_bit = (at + m.meta_len) * 8u;
  }
  if (sm.fixed) {
    d.dict_fixed = 1;
    d.dict_data_size = sm.fixed_len;
    d.dict_payload = str_at;
    d.dict_end = str_at + sm.uncompressed_len;
  } else {
    d.dict_fixed = 0;
    d.dict_payload = off_data;
    d.dict_data_size = off_w;
    d.dict_var = str_at;
    d.dict_end = str_at + sm.uncompressed_len;
  }
  d.ok = 1;
}

// CS INTEGER column -> K_BITS plan. Walks the column headers like
// ObCSMicroBlockTransformer::build_original_transform_desc_ (ob_cs_micro_block_transformer.cpp:216-380)
// to find the column's meta and first stream; value = raw + base (ConvertUintToDatum_T,
// ob_integer_stream_decoder.cpp:37-350); NULL by MSB-first bitmap or by replaced value.
__device__ __forceinline__ void build_cs_col_desc(const BlockView &b, int col, ColDesc &d) {
  const uint8_t *s = b.s;
  const uint32_t bitmap_bytes = (b.row_count + 7u) >> 3;
  const uint32_t hdrs = b.header_size + 12u;
  uint32_t pos = b.cs_first_stream_begin;
  uint32_t str_at = b.row_data_off;   // running position inside the all-string-data area
  int stream_idx = -1;
  for (int i = 0; i <= col; ++i) {
    const uint32_t w = ld32(s, hdrs + 4u * (uint32_t)i);
    const uint32_t type = (w >> 8) & 0xff, attrs = (w >> 16) & 0xff;
    if ((w & 0xff) != 0) return;
    int n_streams;
    uint32_t meta_len = 0;
    if (type == CS_INTEGER) {
      n_streams = 1;
      meta_len = ((attrs & CS_HAS_NULL_OR_NOP_BITMAP) ? bitmap_bytes : 0u) + ((attrs & CS_HAS_NOP_BITMAP) ? bitmap_bytes : 0u);
    } else if (type == CS_STRING) {
      n_streams = (attrs & CS_IS_FIXED_LENGTH) ? 1 : 2;
      meta_len = ((attrs & CS_HAS_NULL_OR_NOP_BITMAP) ? bitmap_bytes : 0u) + ((attrs & CS_HAS_NOP_BITMAP) ? bitmap_bytes : 0u);
    } else if (type == CS_INT_DICT || type == CS_STR_DICT) {
      if (pos + 10u > b.size) return;
      const uint32_t distinct = (uint32_t)ld_bytes(s, pos + 2, 4);
      meta_len = 10u + ((attrs & CS_HAS_NOP_BITMAP) ? bitmap_bytes : 0u);
      n_streams = distinct == 0 ? 0 : (type == CS_INT_DICT ? 2 : ((attrs & CS_IS_FIXED_LENGTH) ? 2 : 3));
    } else {
      return;
    }
    if ((type == CS_STRING || type == CS_STR_DICT) && n_streams > 0) {
      // the column's first stream is its string stream: the meta stays here, the bytes are the next
      // uncompressed_len bytes of the all-string-data area (stream order)
      if (stream_idx + 1 >= (int)b.cs_stream_count) return;
      const uint32_t send = (uint32_t)ld_bytes(s, b.cs_off_data + (uint32_t)(stream_idx + 1) * b.cs_off_width, b.cs_off_width);
      if (pos + meta_len > send || send > b.size) return;
      StrStreamMeta sm;
      parse_str_stream_meta(s, pos + meta_len, send, sm);
      if (!sm.ok || sm.uncompressed_len > b.size - str_at) return;
      if (i == col) {
        build_cs_str_col_desc(b, w, pos, str_at, send, stream_idx + 2, sm, d);
        return;
      }
      str_at += sm.uncompressed_len;
    }
    if (i == col) {
      d.type = (uint8_t)(100 + type);
      d.attr = (uint8_t)attrs;
      d.obj_type = (uint8_t)(w >> 24);
      const int sc = store_class_of(d.obj_type);
      if (type == CS_STR_DICT && sc == 5 && !(attrs & (CS_HAS_NOP_BITMAP | CS_HAS_NOP | CS_OUT_ROW))) {
        d.sc = 5;                     // no streams: every row NULL (CONST plan with an empty dictionary)
        d.kind = K_CONST;
        d.ok = 1;
        return;
      }
      if ((type != CS_INTEGER && type != CS_INT_DICT) || (sc != 1 && sc != 2)) return;
      if (type == CS_INT_DICT) {
        // [ObDictEncodingMeta 10 B][dict value stream][ref stream] -> K_DICT plan (ref == distinct count: NULL,
        // value = dict[ref] + base, ob_int_dict_column_decoder.cpp:25-60)
        if (attrs & (CS_HAS_NOP_BITMAP | CS_HAS_NOP | CS_OUT_ROW)) return;
        if (s[pos] != 0) return;
        const bool const_refs = (s[pos + 1] & 0x4) != 0;   // ObDictEncodingMeta::CONST_ENCODING_REF
        const uint32_t ref_cnt = (uint32_t)ld_bytes(s, pos + 6, 4);
        const uint32_t distinct = (uint32_t)ld_bytes(s, pos + 2, 4);
        d.sc = (uint8_t)sc;
        d.elem_len = (uint8_t)datum_len_of(d.obj_type);
        d.int_mask = 0;
        d.sign_fix = 0;
        d.dict_fixed = 1;
        if (distinct == 0) {  // every row NULL: a CONST plan with an empty dictionary reads no memory
          d.kind = K_CONST;
          d.ok = 1;
          return;
        }
        if (stream_idx + 2 >= (int)b.cs_stream_count) return;
        const uint32_t end0 = (uint32_t)ld_bytes(s, b.cs_off_data + (uint32_t)(stream_idx + 1) * b.cs_off_width, b.cs_off_width);
        const uint32_t end1 = (uint32_t)ld_bytes(s, b.cs_off_data + (uint32_t)(stream_idx + 2) * b.cs_off_width, b.cs_off_width);
        if (pos + meta_len > end0 || end0 > end1 || end1 > b.size) return;
        IntStreamMeta m;
        parse_int_stream_meta(s, pos + meta_len, end0, m);
        if (!m.ok || m.replace_null) return;
        const uint32_t dict = pos + meta_len + m.meta_len;
        if (dict + m.width * distinct != end0) return;
        d.kind = K_DICT;
        d.dict_count = distinct;
        d.dict_data_size = m.width;
        d.dict_payload = dict;
        d.dict_end = end0;
        d.base = m.use_base ? m.base : 0;
        parse_int_stream_meta(s, end0, end1, m);
        if (!m.ok || m.use_base || m.replace_null || m.width > 4) return;
        const uint32_t refs = end0 + m.meta_len;
        if (const_refs) {
          if (!cs_const_ref_plan(s, refs, end1, m.width, ref_cnt, b.row_count, d)) return;
        } else {
          if (refs + m.width * b.row_count != end1) return;
          d.width = (uint8_t)(m.width * 8u);
          d.stride = m.width * 8u;
          d.val_bit = refs * 8u;
        }
        d.ok = 1;
        return;
      }
      if (attrs & (CS_HAS_NOP_BITMAP | CS_HAS_NOP | CS_OUT_ROW)) return;
      if (stream_idx + 1 >= (int)b.cs_stream_count) return;
      const uint32_t end = (uint32_t)ld_bytes(s, b.cs_off_data + (uint32_t)(stream_idx + 1) * b.cs_off_width, b.cs_off_width);
      if (end > b.size || pos + meta_len > end) return;
      IntStreamMeta m;
      parse_int_stream_meta(s, pos + meta_len, end, m);
      if (!m.ok) return;
      const uint32_t data = pos + meta_len + m.meta_len;
      if (data + m.width * b.row_count != end) return;
      d.sc = (uint8_t)sc;
      d.elem_len = (uint8_t)datum_len_of(d.obj_type);
      d.int_mask = 0;
      d.kind = K_BITS;
      d.width = (uint8_t)(m.width * 8u);
      d.stride = m.width * 8u;
      d.val_bit = data * 8u;
      d.base = m.use_base ? m.base : 0;
      d.sign_fix = 0;
      if (attrs & CS_HAS_NULL_OR_NOP_BITMAP) {
        d.ext_bit = 1;
        d.ext_bit_off = pos * 8u;
        d.var_ext_in_row = 7;   // MSB-first bitmap (see ext_row)
      } else if (m.replace_null) {
        uint64_t raw = m.null_replaced - d.base;
        if (m.width < 8) raw &= low_mask(m.width * 8u);
        d.var_is_last = 1;
        d.var_header_off = (uint32_t)raw;
        d.var_k = (uint32_t)(raw >> 32);
      }
      d.ok = 1;
      return;
    }
    if (n_streams == 0) pos += meta_len;
    else {
      stream_idx += n_streams;
      if (stream_idx >= (int)b.cs_stream_count) return;
      pos = (uint32_t)ld_bytes(s, b.cs_off_data + (uint32_t)stream_idx * b.cs_off_width, b.cs_off_width);
    }
  }
}

// Builds the descriptor of column `col`. Mirrors the decoder init of each codec.
__device__ __forceinline__ void build_col_desc(const BlockView &b, int col, ColDesc &d) {
  const uint8_t *s = b.s;
  d = ColDesc{};
  d.rle_slot = -1;
  if (col < 0 || (uint32_t)col >= b.column_count) return;
  if (b.is_cs) {
    build_cs_col_desc(b, col, d);
    return;
  }
  const uint32_t ch = b.header_size + 16u * (uint32_t)col;
  const uint32_t w0 = ld32(s, ch);
  d.type = (uint8_t)((w0 >> 8) & 0xff);
  const bool span_area = (w0 & 0xff) == 0xA5 && (d.type == COL_COLUMN_EQUAL || d.type == COL_COLUMN_SUBSTR);
  if ((w0 & 0xff) != 0 && !span_area) return;  // version
  d.attr = (uint8_t)((w0 >> 16) & 0xff);
  d.obj_type = (uint8_t)(w0 >> 24);
  d.ext_index = ld32(s, ch + 4);
  const uint32_t offset = ld32(s, ch + 8), length = ld32(s, ch + 12);
  const int sc = store_class_of(d.obj_type);
  if (sc == 0) return;
  d.sc = (uint8_t)sc;
  d.elem_len = (uint8_t)datum_len_of(d.obj_type);
  d.int_mask = integer_mask_of(d.obj_type);
  if (span_area) {
    // A span column (COLUMN_EQUAL / COLUMN_SUBSTR) whose values the page batch rebuilt at open (mat_codecs.cuh): in the batch's copy
    // of the block the column header (version byte 0xA5) points at the area, offset_ from the block start, length_ bytes.
    const uint32_t area = offset, rows = b.row_count, nwords = (rows + 31u) / 32u;
    if ((area & 15u) || area > b.size || length > b.size - area || rows == 0) return;
    d.ext_bit = 1;
    d.ext_bit_off = area * 8u;
    if (sc == 5) {   // [NULL bits][END offset u32 x rows][strings]: the plan of a CS STRING column
      if ((uint64_t)nwords * 4u + (uint64_t)rows * 4u > length) return;
      d.kind = K_CSSTR;
      d.dict_payload = area + nwords * 4u;
      d.dict_data_size = 4;
      d.dict_var = d.dict_payload + rows * 4u;
      d.dict_end = d.dict_var + (uint32_t)ld_bytes(s, d.dict_payload + (rows - 1u) * 4u, 4);
      if (d.dict_end > area + length || d.dict_end < d.dict_var) return;
    } else {         // [NULL bits, padded to 8 bytes][8-byte value image x rows]: the plan of a RAW fixed-length column
      const uint32_t vals = area + ((nwords * 4u + 7u) & ~7u);
      if ((uint64_t)(vals - area) + (uint64_t)rows * 8u > length || (uint64_t)vals * 8u + (uint64_t)rows * 64u > 0xffffffffull) return;
      d.kind = K_BITS;
      d.width = 64;
      d.stride = 64;
      d.val_bit = vals * 8u;
    }
    d.ok = 1;
    return;
  }
  if (offset > b.size || b.meta_off > b.size - offset) return;   // untrusted: no wrap-around in meta_off + offset
  const uint32_t meta = b.meta_off + offset;
  const bool has_ext = d.attr & ATTR_HAS_EXTEND_VALUE;
  const bool fixed = d.attr & ATTR_FIX_LENGTH, bp = d.attr & ATTR_BIT_PACKING;
  switch (d.type) {
    case COL_RAW: {
      if (fixed || bp) {
        if (meta > b.size) return;
        d.ext_bit = has_ext ? b.ext_bit : 0;
        d.ext_bit_off = meta * 8u;
        const uint32_t ext_bits = (uint32_t)d.ext_bit * b.row_count;
        if (bp) {
          if (sc == 5 || length == 0 || length > 64) return;
          d.kind = K_BITS;
          d.width = (uint8_t)length;
          d.stride = length;
          d.val_bit = meta * 8u + ext_bits;
        } else {
          const uint32_t data = meta + (ext_bits + 7u) / 8u;
          if (sc == 5) {
            if (length == 0 || length > 0xffff) return;
            d.kind = K_FIXSTR;
            d.dict_data_size = length;
            d.val_bit = data;  // byte offset of cell 0
          } else {
            if (length == 0 || length > 8) return;
            d.kind = K_BITS;
            d.width = (uint8_t)(length * 8u);
            d.stride = length * 8u;
            d.val_bit = data * 8u;
            d.sign_fix = d.int_mask != 0;
          }
        }
      } else {
        // var-stored cells in the row data: strings, and integer columns the encoder turned into var-stored ones
        // because NULLs dominate (ObRawEncoder::traverse, ob_raw_encoder.cpp:106-110,150-155: a non-NULL cell
        // holds the low fix_data_size_ bytes of the datum, a NULL cell nothing)
        if (b.row_index_byte == 0) return;
        d.sign_fix = sc != 5 && d.int_mask != 0;
        d.kind = K_VARSTR;
        d.var_ext_in_row = has_ext;
        d.ext_bit = has_ext ? b.ext_bit : 0;
        d.var_header_off = offset;
        d.var_k = length;
        d.var_is_last = (d.attr & ATTR_LAST_VAR_FIELD) != 0;
      }
      d.ok = 1;
      return;
    }
    case COL_INTEGER_BASE_DIFF: {
      if (sc == 5 || meta + length > b.size) return;
      const int ts = type_store_size(d.obj_type);
      const uint32_t dl = s[meta + 1];
      if (dl == 0) return;
      uint64_t base = ld_bytes(s, meta + 2, (uint32_t)ts);
      const uint64_t mask = ~low_mask((uint32_t)ts * 8u);
      if (sc == 1 && mask != 0 && (base & (mask >> 1))) base |= mask;
      d.base = base;
      const uint32_t data = meta + length;
      d.ext_bit = has_ext ? b.ext_bit : 0;
      d.ext_bit_off = data * 8u;
      const uint32_t ext_bits = (uint32_t)d.ext_bit * b.row_count;
      d.kind = K_BITS;
      if (bp) {
        if (dl > 64) return;
        d.width = (uint8_t)dl;
        d.stride = dl;
        d.val_bit = data * 8u + ext_bits;
      } else {
        if (dl > 8) return;
        d.width = (uint8_t)(dl * 8u);
        d.stride = dl * 8u;
        d.val_bit = (data + (ext_bits + 7u) / 8u) * 8u;
      }
      d.ok = 1;
      return;
    }
    case COL_DICT:
    case COL_RLE: {
      uint32_t dm = meta;
      uint32_t dict_len = length;
      if (d.type == COL_RLE) {
        if (meta + 10 > b.size) return;
        const uint8_t a = s[meta + 1];
        const uint32_t rib = a & 7, rfb = (a >> 3) & 7;
        d.rle_count = (uint32_t)ld_bytes(s, meta + 2, 4);
        const uint32_t doff = (uint32_t)ld_bytes(s, meta + 6, 4);
        if (d.rle_count == 0 || rib == 0 || rfb == 0 || rib > 4 || rfb > 4 || doff > length || length > b.size - meta) return;
        // run-start ids and refs lie between the 10-byte header and the dictionary meta
        if (10ull + (uint64_t)d.rle_count * (rib + rfb) > doff) return;
        // the reference keeps count*row_id_byte in an int16 (ob_rle_decoder.h:193)
        if (d.rle_count * rib > 32767u) return;
        d.rle_row_id_bits = (uint8_t)(rib * 8u);
        d.rle_ref_bits = (uint8_t)(rfb * 8u);
        d.rle_row_ids_bit = (meta + 10u) * 8u;
        d.rle_refs_bit = (meta + 10u + d.rle_count * rib) * 8u;
        dm = meta + doff;
        dict_len = length - doff;
        d.kind = K_RLE;
      } else {
        d.kind = K_DICT;
      }
      if (dm + 9 > b.size || dm + dict_len > b.size) return;
      const uint32_t ref_size = s[dm + 1];  // row_ref_size
      d.dict_count = (uint32_t)ld_bytes(s, dm + 2, 4);
      d.dict_data_size = (uint32_t)ld_bytes(s, dm + 6, 2);
      const uint8_t dattr = s[dm + 8];
      d.dict_fixed = dattr & DICT_FIX_LENGTH;
      d.dict_sorted = (dattr & DICT_IS_SORTED) && d.dict_fixed;
      d.dict_payload = dm + 9;
      d.dict_end = dm + dict_len;
      if (!d.dict_fixed) {
        if (d.dict_data_size != 1 && d.dict_data_size != 2 && d.dict_data_size != 4) return;
        d.dict_var = d.dict_payload + (d.dict_count ? d.dict_count - 1 : 0) * d.dict_data_size;
        if (sc != 5) return;  // var dict of integers does not occur
      } else if (sc != 5 && (d.dict_data_size == 0 || d.dict_data_size > 8)) {
        return;
      }
      d.sign_fix = d.int_mask != 0;
      if (d.type == COL_DICT) {
        const uint32_t data = meta + length;  // refs follow the dict meta
        if (bp) {
          if (ref_size == 0 || ref_size > 32) return;
          d.width = (uint8_t)ref_size;
          d.stride = ref_size;
        } else {
          if (ref_size == 0 || ref_size > 4) return;
          d.width = (uint8_t)(ref_size * 8u);
          d.stride = ref_size * 8u;
        }
        d.val_bit = data * 8u;
      }
      d.ok = 1;
      return;
    }
    case COL_CONST: {
      // ObConstDecoder (ob_const_decoder.cpp:25-137): header {version, count, const_ref, row_id_byte:3,
      // offset u16}; count == 0: value image after the header (const_ref 0) or NULL / NOP (1 / 2);
      // count > 0: [count x u8 ref][count x row_id_byte row ids][dict meta at offset]
      if (length < 6 || meta + length > b.size || s[meta] != 0) return;
      const uint32_t count = s[meta + 1], cref = s[meta + 2], rib = s[meta + 3] & 7u;
      const uint32_t doff = (uint32_t)ld_bytes(s, meta + 4, 2);
      d.kind = K_CONST;
      d.sign_fix = d.int_mask != 0;
      d.dict_fixed = 1;
      if (count == 0) {
        if (cref > 2) return;
        if (cref == 0) {  // a one-entry dictionary whose payload is the stored value
          d.dict_count = 1;
          d.dict_data_size = length - 6u;
          d.dict_payload = meta + 6u;
          d.dict_end = meta + length;
          if (sc != 5 && d.dict_data_size != (uint32_t)type_store_size(d.obj_type)) return;
        }  // else dict_count = 0: ref 0 >= count reads as NULL
        d.ok = 1;
        return;
      }
      if (rib != 1 && rib != 2 && rib != 4) return;
      if (doff < 6u + count * (rib + 1u) || doff + 9u > length) return;   // exception refs + row ids end before the dict meta
      d.rle_count = count;
      d.const_ref = cref;
      d.rle_ref_bits = 8;
      d.rle_row_id_bits = (uint8_t)(rib * 8u);
      d.rle_refs_bit = (meta + 6u) * 8u;
      d.rle_row_ids_bit = (meta + 6u + count) * 8u;
      const uint32_t dm = meta + doff;
      d.dict_count = (uint32_t)ld_bytes(s, dm + 2, 4);
      d.dict_data_size = (uint32_t)ld_bytes(s, dm + 6, 2);
      d.dict_fixed = s[dm + 8] & DICT_FIX_LENGTH;
      d.dict_sorted = (s[dm + 8] & DICT_IS_SORTED) && d.dict_fixed;
      d.dict_payload = dm + 9;
      d.dict_end = meta + length;
      if (!d.dict_fixed) {
        if (d.dict_data_size != 1 && d.dict_data_size != 2 && d.dict_data_size != 4) return;
        d.dict_var = d.dict_payload + (d.dict_count ? d.dict_count - 1 : 0) * d.dict_data_size;
        if (sc != 5) return;
      } else if (sc != 5 && (d.dict_data_size == 0 || d.dict_data_size > 8)) {
        return;
      }
      d.ok = 1;
      return;
    }
    case COL_STRING_DIFF:
    case COL_HEX_PACKING:
    case COL_STRING_PREFIX: {
      // Values these codecs rebuild are materialised once per page batch (mat_codecs.cuh): in the batch's copy of the block the
      // codec header says where the column's area [NULL bits][END offset u32 x rows][strings] lies. Without that marker (a block
      // opened some other way) the column stays unsupported and the caller falls back.
      if (sc != 5 || length < 13 || meta + length > b.size || s[meta] != 0xA5) return;
      const uint32_t pf = meta + (d.type == COL_HEX_PACKING ? 1u : (d.type == COL_STRING_DIFF ? 4u : 2u));
      const uint32_t area = (uint32_t)ld_bytes(s, pf, 4), rows = b.row_count, nwords = (rows + 31u) / 32u;
      if ((area & 15u) || area < meta + length || (uint64_t)area + nwords * 4ull + rows * 4ull > b.size) return;
      d.kind = K_CSSTR;
      d.ext_bit = 1;
      d.ext_bit_off = area * 8u;
      d.dict_payload = area + nwords * 4u;
      d.dict_data_size = 4;
      d.dict_var = d.dict_payload + rows * 4u;
      d.dict_end = d.dict_var + (uint32_t)ld_bytes(s, d.dict_payload + (rows - 1u) * 4u, 4);
      if (d.dict_end > b.size || d.dict_end < d.dict_var) return;
      d.ok = 1;
      return;
    }
    default:
      return;  // span columns (COLUMN_EQUAL / COLUMN_SUBSTR): caller falls back
  }
}

// Byte range [lo, hi) of the block that a scan of column d touches (lo 16-byte aligned, hi padded by
// 16 for the funnel-shift over-read). Everything a fixed / bit-packed / DICT / RLE / CONST column
// needs -- ext bits, values or refs, run arrays, dictionary -- lies inside its column region; RAW
// var-length strings need the row data + row index instead.
__device__ __forceinline__ bool col_region(const ColDesc &d, const BlockView &bv, uint32_t &lo, uint32_t &hi) {
  const uint32_t rows = bv.row_count;
  uint32_t a, b;
  if (cs_bytes_outside(d) && d.kind != K_CONST) return false;   // meta here, bytes in the all-string-data area
  switch (d.kind) {
    case K_VARSTR:  // cells live in the row data, addressed through the row index at the block tail
      a = bv.row_data_off;
      b = bv.size;
      break;
    case K_BITS:
      a = (d.ext_bit ? (d.ext_bit_off < d.val_bit ? d.ext_bit_off : d.val_bit) : d.val_bit) >> 3;
      b = (d.val_bit + rows * d.stride + 7u) >> 3;
      break;
    case K_FIXSTR:
      a = d.ext_bit ? d.ext_bit_off >> 3 : d.val_bit;
      b = d.val_bit + rows * d.dict_data_size;
      break;
    case K_DICT:
      a = d.dict_payload;
      b = (d.val_bit + rows * d.stride + 7u) >> 3;
      if (b < d.dict_end) b = d.dict_end;
      break;
    case K_RLE:
      a = d.rle_row_ids_bit >> 3;
      b = d.dict_end;
      break;
    case K_CSSTR:   // a materialised PAX string column: NULL bits, END offsets and strings are one contiguous area (mat_codecs.cuh)
      a = d.ext_bit_off >> 3;
      b = d.dict_end;
      break;
    case K_CONST: {
      // dictionary + exception lists (PAX: refs, row ids, dictionary in this order; CS: dictionary stream, then
      // the ref stream holding row ids and refs)
      a = 0xffffffffu;
      b = 0;
      if (d.dict_count) { a = d.dict_payload; b = d.dict_end; }
      if (d.rle_count) {
        const uint32_t r0 = d.rle_refs_bit >> 3, r1 = (d.rle_refs_bit + d.rle_count * d.rle_ref_bits + 7u) >> 3;
        const uint32_t i0 = d.rle_row_ids_bit >> 3, i1 = (d.rle_row_ids_bit + d.rle_count * d.rle_row_id_bits + 7u) >> 3;
        a = min(a, min(r0, i0));
        b = max(b, max(r1, i1));
      }
      if (a > b) { a = 0; b = 0; }
      break;
    }
    default:
      return false;
  }
  lo = a & ~15u;
  hi = ((b + 16u + 15u) & ~15u);
  return true;
}

// Byte ranges of the block a PROJECTION of column d reads (r = {lo0, hi0, lo1, hi1}, 16-byte aligned, padded for the
// funnel-shift over-read). Returns the number of ranges: 0 = no bounded range (the caller reports it), 1, or 2 for a
// var-length string dictionary whose offset array and refs are staged without the string bytes between them.
__device__ __forceinline__ int proj_ranges(const ColDesc &d, const BlockView &bv, uint32_t r[4]) {
  if (d.kind == K_DICT && d.sc == 5) {
    const uint32_t ref_lo = (d.val_bit >> 3) & ~15u;
    const uint32_t ref_hi = (((d.val_bit + bv.row_count * d.stride + 7u) >> 3) + 16u + 15u) & ~15u;
    if (d.dict_fixed) { r[0] = ref_lo; r[1] = ref_hi; return 1; }   // cell address is arithmetic: refs only
    const uint32_t idx_lo = d.dict_payload & ~15u;
    const uint32_t idx_hi = (d.dict_payload + d.dict_count * d.dict_data_size + 16u + 15u) & ~15u;
    if (idx_hi < ref_lo) { r[0] = idx_lo; r[1] = idx_hi; r[2] = ref_lo; r[3] = ref_hi; return 2; }
    if (ref_hi < idx_lo) { r[0] = ref_lo; r[1] = ref_hi; r[2] = idx_lo; r[3] = idx_hi; return 2; }
    r[0] = min(idx_lo, ref_lo);
    r[1] = max(idx_hi, ref_hi);
    return 1;
  }
  uint32_t lo, hi;
  if (!col_region(d, bv, lo, hi) || hi <= lo) return 0;
  r[0] = lo;
  r[1] = hi;
  return 1;
}
// "Flat" projected column (scan_small.cuh, project_flat): a row's output is one ref / value load plus at most two dictionary loads
__device__ __forceinline__ bool flat_kind(const ColDesc &d) {
  if (d.kind == K_BITS) return d.sc != 5 && d.ext_bit == 0 && !d.sign_fix && !d.var_is_last;
  if (d.kind == K_DICT) return d.sc == 5 ? !d.dict_fixed : d.dict_data_size <= 8u;
  return false;
}
__device__ __forceinline__ uint32_t proj_ranges_bytes(const ColDesc &d, const BlockView &bv) {
  uint32_t r[4];
  const int n = proj_ranges(d, bv, r);
  if (n == 0) return 0xffffffffu;
  return (r[1] - r[0]) + (n == 2 ? r[3] - r[2] : 0u);
}

// ---- RLE run table (per block, per RLE column, in shared memory) -------------------------------
// mask: one bit per row, set where a run starts; pre[g]: number of run starts before row 32 * g.
// run(row) = rank of row among the run starts - 1: two loads + popc, no search, no divergence.
struct RleTable {
  const uint32_t *mask;
  const uint16_t *pre;
};

__device__ __forceinline__ uint32_t rle_run_of(const RleTable &t, uint32_t row) {
  const uint32_t w = row >> 5;
  const uint32_t r = (uint32_t)t.pre[w] + (uint32_t)__popc(t.mask[w] & (0xffffffffu >> (31u - (row & 31u))));
  return r ? r - 1u : 0u;
}

__device__ __forceinline__ uint32_t rle_ref_slow(const uint8_t *s, const ColDesc &d, uint32_t row) {
  // upper_bound over the run starts, then refs[pos - 1] (no table: one-off lookups)
  uint32_t lo = 0, hi = d.rle_count;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    const uint32_t v = ld_bits32(s, d.rle_row_ids_bit + mid * d.rle_row_id_bits, d.rle_row_id_bits);
    if (v <= row) lo = mid + 1; else hi = mid;
  }
  const uint32_t pos = lo > 0 ? lo - 1 : 0;
  return ld_bits32(s, d.rle_refs_bit + pos * d.rle_ref_bits, d.rle_ref_bits);
}

// row -> dictionary reference (DICT / RLE). `rt` may be null for RLE (slow path).
__device__ __forceinline__ uint32_t ref_of(const uint8_t *s, const ColDesc &d, const RleTable *rt, uint32_t row) {
  if (d.kind == K_RLE) {
    if (rt == nullptr) return rle_ref_slow(s, d, row);
    return ld_bits32(s, d.rle_refs_bit + rle_run_of(*rt, row) * d.rle_ref_bits, d.rle_ref_bits);
  }
  if (d.kind == K_CONST) {
    // lower_bound over the (sorted, <= 255) exception row ids (ob_const_decoder.cpp:93-121)
    uint32_t lo = 0, hi = d.rle_count;
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (ld_bits32(s, d.rle_row_ids_bit + mid * d.rle_row_id_bits, d.rle_row_id_bits) < row) lo = mid + 1;
      else hi = mid;
    }
    if (lo < d.rle_count && ld_bits32(s, d.rle_row_ids_bit + lo * d.rle_row_id_bits, d.rle_row_id_bits) == row)
      return ld_bits32(s, d.rle_refs_bit + lo * d.rle_ref_bits, d.rle_ref_bits);   // 8-bit refs in PAX CONST, stream width in CS
    return d.const_ref;
  }
  return ld_bits32(s, d.val_bit + row * d.stride, d.width);
}

__device__ __forceinline__ uint64_t sign_fix(uint64_t int_mask, uint64_t v) {
  // load_data_to_datum: if (mask && (v & (mask >> 1))) v |= mask   (ob_encoding_util.h:505-509)
  if (int_mask != 0 && (v & (int_mask >> 1))) v |= int_mask;
  return v;
}

__device__ __forceinline__ uint64_t dict_int(const uint8_t *s, const ColDesc &d, uint32_t ref) {
  const uint64_t v = ld_bits(s, (d.dict_payload + ref * d.dict_data_size) * 8u, d.dict_data_size * 8u) + d.base;
  return d.sign_fix ? sign_fix(d.int_mask, v) : v;   // base: CS INT_DICT value streams (0 for PAX dictionaries)
}

// dictionary string cell -> (block offset, length)
__device__ __forceinline__ void dict_str(const uint8_t *s, const ColDesc &d, uint32_t ref,
                                         uint32_t &cell, uint32_t &len) {
  if (d.dict_fixed) {
    cell = d.dict_payload + ref * d.dict_data_size;
    len = d.dict_data_size;
    return;
  }
  const uint32_t ib = d.dict_data_size;
  const uint32_t off = ref == 0 ? 0u : (uint32_t)ld_bytes(s, d.dict_payload + (ref - 1) * ib, ib);
  cell = d.dict_var + off;
  len = ref == d.dict_count - 1 ? d.dict_end - cell
                                : (uint32_t)ld_bytes(s, d.dict_payload + ref * ib, ib) - off;
}

// Shared-window twins of dict_int / dict_str: `sbit` is 8 * the shared-window address of the staged block (or of the
// staged column region, shifted so block offsets resolve into it). D is a ColDesc or a descriptor with the same field names.
template <class D>
__device__ __forceinline__ uint64_t dict_int_s(uint32_t sbit, const D &d, uint32_t ref) {
  const uint32_t dbits = d.dict_data_size * 8u, at = sbit + d.dict_payload * 8u + ref * dbits;
  const uint64_t v = (dbits <= 32u ? (uint64_t)sbits32(at, dbits) : sbits(at, dbits)) + d.base;
  return d.sign_fix ? sign_fix(d.int_mask, v) : v;
}
template <class D>
__device__ __forceinline__ void dict_str_s(uint32_t sbit, const D &d, uint32_t ref, uint32_t &cell, uint32_t &len) {
  if (d.dict_fixed) {
    len = d.dict_data_size;
    cell = d.dict_payload + ref * len;
    return;
  }
  const uint32_t ib8 = d.dict_data_size * 8u, ibit = sbit + d.dict_payload * 8u;
  const uint32_t off = ref == 0 ? 0u : sbits32(ibit + (ref - 1u) * ib8, ib8);
  const uint32_t end = ref == d.dict_count - 1u ? d.dict_end - d.dict_var : sbits32(ibit + ref * ib8, ib8);
  cell = d.dict_var + off;
  len = end - off;
}

// ---- integer-class cell (generic path) -----------------------------------------------------------
// Returns the 64-bit value image the reference would MEMCPY into the datum (low elem_len bytes
// significant); is_null set for NULL (and NOP) cells.
__device__ __forceinline__ void str_cell(const BlockView &b, const ColDesc &d, const RleTable *rt, uint32_t row,
                                         uint32_t &cell, uint32_t &len, bool &is_null);

__device__ __forceinline__ uint64_t int_cell(const BlockView &b, const ColDesc &d, const RleTable *rt,
                                             uint32_t row, bool &is_null) {
  const uint8_t *s = b.s;
  is_null = false;
  if (d.kind == K_VARSTR) {  // var-stored integer: the cell's bytes are the low bytes of the datum
    uint32_t cell, len;
    str_cell(b, d, rt, row, cell, len, is_null);
    if (is_null) return 0;
    const uint64_t v = len ? ld_bytes(s, cell, len < 8u ? len : 8u) : 0ull;
    return d.sign_fix ? sign_fix(d.int_mask, v) : v;
  }
  if (is_dict_kind(d)) {
    const uint32_t ref = ref_of(s, d, rt, row);
    if (ref >= d.dict_count) { is_null = true; return 0; }
    return dict_int(s, d, ref);
  }
  if (d.ext_bit && ld_bits32(s, d.ext_bit_off + ext_row(d, row) * d.ext_bit, d.ext_bit) != STORED_NOT_EXT) {
    is_null = true;
    return 0;
  }
  const uint64_t raw = ld_bits(s, d.val_bit + row * d.stride, d.width);
  if (null_replaced_on(d) && raw == null_replaced_raw(d)) {
    is_null = true;
    return 0;
  }
  const uint64_t v = raw + d.base;
  return d.sign_fix ? sign_fix(d.int_mask, v) : v;
}

// value used for comparisons: sign-extended from the datum length for signed classes
template <class D>
__device__ __forceinline__ int64_t cmp_image(const D &d, uint64_t v) {
  if (d.elem_len == 4) return d.sc == 1 ? (int64_t)(int32_t)(uint32_t)v : (int64_t)(uint32_t)v;
  if (d.elem_len == 1) return (int64_t)(uint8_t)v;
  return (int64_t)v;
}

// ---- string-class cell -------------------------------------------------------------------------
__device__ __forceinline__ void str_cell(const BlockView &b, const ColDesc &d, const RleTable *rt, uint32_t row,
                                         uint32_t &cell, uint32_t &len, bool &is_null) {
  const uint8_t *s = b.s;
  is_null = false;
  cell = 0;
  len = 0;
  if (is_dict_kind(d)) {
    const uint32_t ref = ref_of(s, d, rt, row);
    if (ref >= d.dict_count) { is_null = true; return; }
    dict_str(s, d, ref, cell, len);
    return;
  }
  if (d.kind == K_FIXSTR) {
    if (d.ext_bit && ld_bits32(s, d.ext_bit_off + ext_row(d, row) * d.ext_bit, d.ext_bit) != STORED_NOT_EXT) {
      is_null = true;
      return;
    }
    len = d.dict_data_size;
    cell = d.val_bit + row * len;
    return;
  }
  if (d.kind == K_CSSTR) {  // END offset per row; NULL by bitmap or as a zero-length value
    if (d.ext_bit && ld_bits32(s, d.ext_bit_off + ext_row(d, row) * d.ext_bit, d.ext_bit) != STORED_NOT_EXT) {
      is_null = true;
      return;
    }
    const uint32_t ib = d.dict_data_size;
    const uint32_t off = row == 0 ? 0u : (uint32_t)ld_bytes(s, d.dict_payload + (row - 1) * ib, ib);
    cell = d.dict_var + off;
    len = (uint32_t)ld_bytes(s, d.dict_payload + row * ib, ib) - off;
    if (d.var_is_last && len == 0) is_null = true;
    return;
  }
  // RAW var-length: row = [ext bits][col_idx_byte][idx x (nvar-1)][cells]
  const uint32_t rib = b.row_index_byte;
  const uint32_t ro = (uint32_t)ld_bytes(s, b.row_index_off + row * rib, rib);
  const uint32_t re = (uint32_t)ld_bytes(s, b.row_index_off + (row + 1) * rib, rib);
  const uint32_t rowp = b.row_data_off + ro;
  const uint32_t row_len = re - ro;
  if (d.var_ext_in_row && ld_bits32(s, rowp * 8u + d.ext_index, d.ext_bit) != STORED_NOT_EXT) {
    is_null = true;
    return;
  }
  if (b.var_col_cnt == 1) {
    cell = rowp + d.var_header_off;
    len = row_len - d.var_header_off;
    return;
  }
  const uint32_t ib = s[rowp + d.var_header_off];
  const uint32_t idx = rowp + d.var_header_off + 1;
  const uint32_t var = idx + ib * (b.var_col_cnt - 1u);
  const uint32_t col_off = d.var_k == 0 ? 0u : (uint32_t)ld_bytes(s, idx + (d.var_k - 1) * ib, ib);
  len = d.var_is_last ? row_len - col_off - (var - rowp)
                      : (uint32_t)ld_bytes(s, idx + d.var_k * ib, ib) - col_off;
  cell = var + col_off;
}

// memcmp-then-length order of a cell against a constant, 8 bytes per step. `c` is 8-byte aligned and
// readable up to the next multiple of 8 past clen (the host pads the constant heap).
__device__ __forceinline__ int str_cmp(const uint8_t *s, uint32_t cell, uint32_t len,
                                       const uint8_t *c, uint32_t clen) {
  const uint32_t m = len < clen ? len : clen;
  for (uint32_t i = 0; i < m; i += 8u) {
    const uint32_t nb = m - i < 8u ? m - i : 8u;
    const uint64_t a = ld_bits(s, (cell + i) * 8u, nb * 8u);   // little endian: first byte in the low bits
    const uint64_t b = *reinterpret_cast<const uint64_t *>(c + i) & (~0ull >> (64u - nb * 8u));
    if (a != b) {
      const int k = (__ffsll((long long)(a ^ b)) - 1) & ~7;      // first differing byte
      return ((a >> k) & 0xffull) < ((b >> k) & 0xffull) ? -1 : 1;
    }
  }
  return len < clen ? -1 : (len > clen ? 1 : 0);
}

__device__ __forceinline__ bool cmp_to_bool(int op, int c) {
  switch (op) {
    case OP_EQ: return c == 0;
    case OP_LE: return c <= 0;
    case OP_LT: return c < 0;
    case OP_GE: return c >= 0;
    case OP_GT: return c > 0;
    case OP_NE: return c != 0;
    default: return false;
  }
}

}  // namespace obdev
