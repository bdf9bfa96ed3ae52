// Host-side PAX ("ENCODING_ROW_STORE") micro-block writer.
//
// Produces reference-format micro-blocks for a forced per-column encoding, following the byte
// layout the reference's encoder emits (this file is a fresh implementation written against that
// layout, not a translation of the encoder's control flow):
//   block assembly      encoding/ob_micro_block_encoder.cpp:499-721 (build_block,
//                       store_encoding_meta_and_fix_cols), :724-931 (set_row_data_pos, fill_row_data)
//   fixed column store  encoding/ob_icolumn_encoder.h:122-275 (calc_fix_data_size, store_fix_bits,
//                       fill_column_store): [ext bits][bit-packed values] as ONE bit stream, then
//                       byte-aligned fixed-width values
//   RAW                 encoding/ob_raw_encoder.cpp:96-188 (width choice), :271-291
//   DICT                encoding/ob_dict_encoder.cpp:84-133,187-276,380-400 (sorted dict, refs)
//   RLE                 encoding/ob_rle_encoder.cpp:68-120,137-196 (run starts + refs + dict)
//   INTEGER_BASE_DIFF   encoding/ob_integer_base_diff_encoder.cpp:154-245,267-287
//   width rules         encoding/ob_encoding_util.cpp:37-97 (get_packing_size, get_int_size,
//                       get_byte_packed_int_size)
//   header finalisation blocksstable/ob_imicro_block_writer.cpp:169-204, ob_micro_block_header.cpp:203-233
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/obgpu_writer.h"
#include "ob_agg_row_format.h"
#include "ob_compress_format.h"
#include "ob_format.h"
#include "stream_codecs_host.h"

namespace {

using namespace obf;

// ---- width rules -------------------------------------------------------------------------------
int bit_width_of(uint64_t v) { return v == 0 ? 1 : 64 - __builtin_clzll(v); }

// Returns size in bits when *bit_packing, else in bytes.
int64_t packing_size(bool *bit_packing, uint64_t v, bool enable_bit_packing) {
  int64_t size = 0;
  if (enable_bit_packing) {
    const int64_t bit_size = bit_width_of(v);
    size = bit_size / 8;
    const int64_t ext = bit_size % 8;
    if (ext == 0) {
      *bit_packing = false;
    } else if (8 - ext < size / 2 + 1) {
      size++;
      *bit_packing = false;
    } else {
      *bit_packing = true;
      size = bit_size;
    }
  } else {
    *bit_packing = false;
    size = v <= 0xffull ? 1 : v <= 0xffffull ? 2 : v <= 0xffffffffull ? 4 : 8;
  }
  return size;
}
int64_t int_size_bytes(uint64_t v) { return (bit_width_of(v) + 7) / 8; }
int64_t byte_packed_int_size(uint64_t v) {
  return v <= 0xffull ? 1 : v <= 0xffffull ? 2 : v <= 0xffffffffull ? 4 : 8;
}

// ---- LSB-first bit writer over a zeroed buffer -----------------------------------------------
inline void put_bits(uint8_t *buf, int64_t pos, int len, uint64_t v) {
  int64_t done = 0;
  while (done < len) {
    const int64_t byte = (pos + done) >> 3;
    const int off = (pos + done) & 7;
    const int take = (int)std::min<int64_t>(len - done, 8 - off);
    buf[byte] |= (uint8_t)(((v >> done) & ((1u << take) - 1u)) << off);
    done += take;
  }
}

struct Buf {
  std::vector<uint8_t> d;
  size_t size() const { return d.size(); }
  uint8_t *grow(size_t n) {
    const size_t o = d.size();
    d.resize(o + n, 0);
    return d.data() + o;
  }
};

struct StrRef {
  const char *p;
  int64_t len;
};
inline int str_cmp(const StrRef &a, const StrRef &b) {
  const int64_t m = std::min(a.len, b.len);
  const int c = m > 0 ? memcmp(a.p, b.p, (size_t)m) : 0;
  if (c != 0) return c;
  return a.len < b.len ? -1 : (a.len > b.len ? 1 : 0);
}
struct StrHash {
  size_t operator()(const StrRef &s) const {
    uint64_t h = 1469598103934665603ull;
    for (int64_t i = 0; i < s.len; ++i) h = (h ^ (uint8_t)s.p[i]) * 1099511628211ull;
    return (size_t)h;
  }
};
struct StrEq {
  bool operator()(const StrRef &a, const StrRef &b) const {
    return a.len == b.len && (a.len == 0 || memcmp(a.p, b.p, (size_t)a.len) == 0);
  }
};

struct ColCtx {
  const obgpu_col_input *in;
  int sc;  // store class 1 int / 2 uint / 5 string
  int64_t row_begin, nrows;
  int64_t null_cnt = 0;
  bool enable_bp = true;
  // is_null[] : 0 value, 1 NULL, 2 NOP (ObStoredExtValue, ob_encoding_util.h:279-285); "null" below
  // means "stored as an extend value"
  bool is_null(int64_t r) const { return in->is_null && in->is_null[row_begin + r]; }
  uint64_t ext_val(int64_t r) const { return in->is_null[row_begin + r] == 2 ? STORED_NOPE : STORED_NULL; }
  int64_t nope_cnt = 0;
  int64_t ival(int64_t r) const { return in->i64[row_begin + r]; }
  StrRef sval(int64_t r) const {
    const int64_t a = in->str_off[row_begin + r], b = in->str_off[row_begin + r + 1];
    return StrRef{in->str_heap + a, b - a};
  }
  // value image the reference stores: datum.get_uint64() & INTEGER_MASK_TABLE[type_store_size]
  uint64_t uval(int64_t r) const {
    const int ts = type_store_size((uint8_t)in->obj_type);
    return (uint64_t)ival(r) & low_mask(ts * 8);
  }
};

// What a column contributes to the block.
struct ColOut {
  ColumnHeader hdr{};
  bool is_var = false;          // var-length cells live in the row data
  int var_int_size = 0;         // integer column turned into a var-stored one: bytes per non-NULL cell
  bool need_ext_in_row = false; // var column with NULLs: ext bits inside each row
  // string codecs with their own meta header (HEX_PACKING / STRING_DIFF / STRING_PREFIX): the column header keeps the meta's
  // position; a var-stored column's row position goes into the codec header's offset_ / length_ fields (set_data_pos), and its
  // cells are encoded bytes (cell_off[r] .. cell_off[r + 1] of cell_heap), not the strings themselves
  bool own_meta = false;
  size_t pos_field_at = 0;      // offset inside `meta` of the codec header's offset_ field (length_ follows it)
  std::vector<uint8_t> cell_heap;
  std::vector<int64_t> cell_off;
};

// ObHexStringMap / ObHexStringPacker (encoding/ob_hex_string_encoder.h:26-107): at most 16 distinct bytes, two per stored byte,
// the first one in the high nibble; indexes are assigned in byte order (build_index, ob_hex_string_encoder.cpp:30-43).
struct HexMap {
  int size = 0;
  uint8_t map[256] = {0};
  void mark(uint8_t c) { if (size <= 16 && map[c] == 0) map[c] = (uint8_t)++size; }
  bool can_packing() const { return size <= 16; }
  void build_index(uint8_t *arr) {
    int idx = 0;
    for (int i = 0; i < 256 && idx < size; ++i)
      if (map[i]) { map[i] = (uint8_t)idx; arr[idx++] = (uint8_t)i; }
  }
};
struct HexPacker {
  const HexMap &m;
  std::vector<uint8_t> &out;
  size_t base;
  uint64_t pos = 0;
  HexPacker(const HexMap &m_, std::vector<uint8_t> &o) : m(m_), out(o), base(o.size()) {}
  void pack(uint8_t c) {
    if (base + pos / 2 >= out.size()) out.push_back(0);
    out[base + pos / 2] = (uint8_t)(out[base + pos / 2] | (m.map[c] << (((pos + 1) % 2) * 4)));
    ++pos;
  }
};

// Fixed column store: [ext bits][bit packed] then byte aligned fixed values.
//   bp_len > 0  : value_of(row) packed bp_len bits;  fix_len > 0 : fix_len bytes per row.
template <typename ValueOf>
void fill_column_store(Buf &meta, const ColCtx &c, bool need_ext, int ext_bit, int bp_len,
                       int fix_len, bool include_null_cells, ValueOf value_of) {
  const int64_t n = c.nrows;
  int64_t bits = 0;
  if (need_ext) bits += (int64_t)ext_bit * n;
  bits += (int64_t)bp_len * n;
  const int64_t bits_size = (bits + 7) / 8;
  uint8_t *buf = meta.grow((size_t)(bits_size + (int64_t)fix_len * n));
  int64_t pos = 0;
  if (need_ext) {
    for (int64_t r = 0; r < n; ++r) {
      if (c.is_null(r)) put_bits(buf, pos, ext_bit, c.ext_val(r));
      pos += ext_bit;
    }
  }
  if (bp_len > 0) {
    for (int64_t r = 0; r < n; ++r) {
      if (include_null_cells || !c.is_null(r)) put_bits(buf, pos, bp_len, value_of(r) & low_mask(bp_len));
      pos += bp_len;
    }
  }
  if (fix_len > 0) {
    uint8_t *p = buf + bits_size;
    for (int64_t r = 0; r < n; ++r) {
      if (include_null_cells || !c.is_null(r)) {
        const uint64_t v = value_of(r);
        memcpy(p, &v, (size_t)std::min(fix_len, 8));
      }
      p += fix_len;
    }
  }
}

// ---- dictionary builders ---------------------------------------------------------------------
struct IntDict {
  std::vector<uint64_t> values;  // dict order
  std::vector<uint32_t> refs;    // per row (null -> count)
  uint64_t max_integer = 0;
};

void build_int_dict(const ColCtx &c, bool sorted, IntDict &d) {
  std::unordered_map<uint64_t, uint32_t> first;
  first.reserve((size_t)std::min<int64_t>(c.nrows, 1 << 16));
  d.refs.resize((size_t)c.nrows);
  for (int64_t r = 0; r < c.nrows; ++r) {
    if (c.is_null(r)) continue;
    const uint64_t v = c.uval(r);
    auto it = first.find(v);
    if (it == first.end()) {
      first.emplace(v, (uint32_t)d.values.size());
      d.values.push_back(v);
      d.max_integer = std::max(d.max_integer, v);
    }
  }
  if (sorted) {
    const uint8_t t = (uint8_t)c.in->obj_type;
    const int ts = type_store_size(t);
    if (c.sc == 1) {
      const uint64_t sign = 1ull << (ts * 8 - 1);
      std::sort(d.values.begin(), d.values.end(),
                [sign](uint64_t a, uint64_t b) { return (a ^ sign) < (b ^ sign); });
    } else {
      std::sort(d.values.begin(), d.values.end());
    }
    for (uint32_t i = 0; i < d.values.size(); ++i) first[d.values[i]] = i;
  }
  const uint32_t cnt = (uint32_t)d.values.size();
  for (int64_t r = 0; r < c.nrows; ++r)
    d.refs[(size_t)r] = c.is_null(r) ? (c.ext_val(r) == STORED_NOPE ? cnt + 1 : cnt) : first[c.uval(r)];
}

struct StrDict {
  std::vector<StrRef> values;
  std::vector<uint32_t> refs;
  int64_t var_data_size = 0;  // sum of distinct lengths
  int64_t fix_len = -1;       // >= 0 when every distinct value has the same length
};

void build_str_dict(const ColCtx &c, bool sorted, StrDict &d) {
  std::unordered_map<StrRef, uint32_t, StrHash, StrEq> first;
  d.refs.resize((size_t)c.nrows);
  bool var = false;
  for (int64_t r = 0; r < c.nrows; ++r) {
    if (c.is_null(r)) continue;
    const StrRef s = c.sval(r);
    if (first.find(s) == first.end()) {
      first.emplace(s, (uint32_t)d.values.size());
      d.values.push_back(s);
      d.var_data_size += s.len;
      if (!var) {
        if (d.fix_len < 0) d.fix_len = s.len;
        else if (d.fix_len != s.len) { d.fix_len = -1; var = true; }
      }
    }
  }
  if (sorted) {
    std::sort(d.values.begin(), d.values.end(),
              [](const StrRef &a, const StrRef &b) { return str_cmp(a, b) < 0; });
    for (uint32_t i = 0; i < d.values.size(); ++i) first[d.values[i]] = i;
  }
  const uint32_t cnt = (uint32_t)d.values.size();
  for (int64_t r = 0; r < c.nrows; ++r)
    d.refs[(size_t)r] = c.is_null(r) ? (c.ext_val(r) == STORED_NOPE ? cnt + 1 : cnt) : first[c.sval(r)];
}

// Writes ObDictMetaHeader + payload; returns pointer offset of the header inside meta.
size_t store_int_dict_meta(Buf &meta, const ColCtx &c, const IntDict &d, bool sorted) {
  const int64_t data_size = c.enable_bp ? int_size_bytes(d.max_integer) : byte_packed_int_size(d.max_integer);
  const size_t at = meta.size();
  uint8_t *p = meta.grow(sizeof(DictMetaHeader) + (size_t)data_size * d.values.size());
  DictMetaHeader h{};
  h.count_ = (uint32_t)d.values.size();
  h.data_size_ = (uint16_t)data_size;
  h.attr_ = DICT_FIX_LENGTH | (sorted ? DICT_IS_SORTED : 0);
  memcpy(p, &h, sizeof(h));
  p += sizeof(h);
  for (uint64_t v : d.values) {
    memcpy(p, &v, (size_t)data_size);
    p += data_size;
  }
  return at;
}

size_t store_str_dict_meta(Buf &meta, const StrDict &d) {
  const size_t at = meta.size();
  const size_t cnt = d.values.size();
  DictMetaHeader h{};
  h.count_ = (uint32_t)cnt;
  const bool var = d.fix_len < 0 || d.fix_len > 0xffff;
  if (!var) {
    uint8_t *p = meta.grow(sizeof(h) + (size_t)d.fix_len * cnt);
    h.data_size_ = (uint16_t)d.fix_len;
    h.attr_ = DICT_FIX_LENGTH | DICT_IS_SORTED;  // need_sort_ => sorted attr on the fixed path
    memcpy(p, &h, sizeof(h));
    p += sizeof(h);
    for (const StrRef &s : d.values) {
      memcpy(p, s.p, (size_t)s.len);
      p += s.len;
    }
  } else {
    const int idx_byte = d.var_data_size <= 0xff ? 1 : (d.var_data_size <= 0xffff ? 2 : 4);
    const size_t idx_bytes = cnt > 0 ? (cnt - 1) * (size_t)idx_byte : 0;
    uint8_t *p = meta.grow(sizeof(h) + idx_bytes + (size_t)d.var_data_size);
    h.data_size_ = (uint16_t)idx_byte;  // index_byte_
    h.attr_ = 0;                        // var dict of strings: stored sorted, attr not set
    memcpy(p, &h, sizeof(h));
    uint8_t *idx = p + sizeof(h);
    uint8_t *data = idx + idx_bytes;
    int64_t off = 0;
    for (size_t i = 0; i < cnt; ++i) {
      if (i > 0) {
        const uint64_t o = (uint64_t)off;
        memcpy(idx + (i - 1) * (size_t)idx_byte, &o, (size_t)idx_byte);
      }
      memcpy(data + off, d.values[i].p, (size_t)d.values[i].len);
      off += d.values[i].len;
    }
  }
  return at;
}

// CRC-32C (Castagnoli) continued from c over p[0, len): ob_crc64_sse42 with seed 0 and no final xor
uint32_t crc32c_update(uint32_t c, const uint8_t *p, size_t len) {
  static uint32_t tab[256];
  static std::atomic<int> ready{0};
  if (!ready.load(std::memory_order_acquire)) {
    uint32_t t[256];
    for (uint32_t n = 0; n < 256; ++n) {
      uint32_t cc = n;
      for (int k = 0; k < 8; ++k) cc = (cc & 1) ? 0x82f63b78u ^ (cc >> 1) : cc >> 1;
      t[n] = cc;
    }
    memcpy(tab, t, sizeof(t));
    ready.store(1, std::memory_order_release);
  }
  for (size_t k = 0; k < len; ++k) c = tab[(c ^ p[k]) & 0xff] ^ (c >> 8);
  return c;
}

// Fills the 64-byte micro block header in front of the finished payload: CRC-32C payload checksum
// (ob_crc64_sse42, seed 0, no final xor) and the 16-bit header checksum (ob_micro_block_header.cpp:193-224).
void finish_header(std::vector<uint8_t> &block, uint32_t header_size, int32_t ncol, int32_t rowkey_cnt, int64_t nrows,
                   uint8_t row_store_type, uint8_t opt, uint16_t opt2, uint32_t row_offset, int64_t original) {
  uint8_t *b = block.data();
  const size_t total = block.size();
  MicroBlockHeader h{};
  h.magic_ = MICRO_BLOCK_HEADER_MAGIC;
  h.version_ = MICRO_BLOCK_HEADER_VERSION;
  h.header_size_ = header_size;
  h.column_count_ = (uint16_t)ncol;
  h.rowkey_column_count_ = (uint16_t)rowkey_cnt;
  h.flag16_ = (uint16_t)(1u << 2);  // all_lob_in_row_ = 1, no column checksum
  h.row_count_ = (uint32_t)nrows;
  h.row_store_type_ = row_store_type;
  h.opt_ = opt;
  h.opt2_ = opt2;
  h.row_data_offset_ = row_offset;
  h.original_length_ = (int32_t)std::min<int64_t>(original, INT32_MAX);
  h.max_merged_trans_version_ = 0;
  h.data_length_ = (int32_t)(total - header_size);
  h.data_zlength_ = h.data_length_;
  h.data_checksum_ = (int64_t)(uint64_t)crc32c_update(0, b + header_size, total - header_size);
  h.column_checksums_ptr_ = 0;
  memcpy(b, &h, sizeof(h));
  const int16_t hc = micro_header_checksum(b);
  memcpy(b + 8, &hc, 2);
}

struct BlockBuilder {
  const obgpu_col_input *cols;
  int32_t ncol;
  int32_t rowkey_cnt;
  int64_t row_begin, nrows;
  std::vector<ColCtx> ctx;
  std::vector<ColOut> out;
  Buf meta;
  int ext_bit = 0;

  int encode_raw(int i);
  int encode_dict(int i);
  int encode_rle(int i);
  int encode_base_diff(int i);
  int encode_const(int i);
  int encode_hex(int i);
  int encode_string_diff(int i);
  int encode_string_prefix(int i);
  int encode_column_equal(int i);
  int encode_column_substr(int i);
  int span_ref_of(int i) const;
  void store_ext_then_fixed_cells(int i, int64_t cell_len);
  int build_cs(std::vector<uint8_t> &block, int64_t original);
  int build(std::vector<uint8_t> &block);
};

int BlockBuilder::encode_raw(int i) {
  ColCtx &c = ctx[i];
  ColOut &o = out[i];
  o.hdr.type_ = COL_RAW;
  const bool has_null = c.null_cnt > 0;
  if (c.sc == 1 || c.sc == 2) {
    uint64_t max_integer = 0;
    for (int64_t r = 0; r < nrows; ++r)
      if (!c.is_null(r)) max_integer = std::max(max_integer, c.uval(r));
    bool bp = false;
    const int64_t size = packing_size(&bp, max_integer, c.enable_bp);
    // The reference turns the column into a var-stored one when NULLs dominate (ObRawEncoder::traverse,
    // ob_raw_encoder.cpp:106-110,150-155): every non-NULL cell then takes fix_data_size_ bytes of the row data
    // (size / 8 + 1 for a bit-packing width, else the byte width; get_var_length :194-234, store_data
    // ob_raw_encoder.h:84-122), a NULL cell none.
    if (bp ? size * c.null_cnt > nrows * 2 * 8 : size * c.null_cnt > nrows * 2) {
      o.is_var = true;
      o.var_int_size = (int)(bp ? size / 8 + 1 : size);
      o.need_ext_in_row = has_null;
      if (has_null) o.hdr.attr_ |= ATTR_HAS_EXTEND_VALUE;
      return OBGPU_SUCCESS;
    }
    o.hdr.attr_ |= ATTR_FIX_LENGTH;
    if (has_null) o.hdr.attr_ |= ATTR_HAS_EXTEND_VALUE;
    if (bp) o.hdr.attr_ |= ATTR_BIT_PACKING;
    o.hdr.offset_ = (uint32_t)meta.size();
    o.hdr.length_ = (uint32_t)size;
    fill_column_store(meta, c, has_null, ext_bit, bp ? (int)size : 0, bp ? 0 : (int)size, false,
                      [&](int64_t r) { return c.uval(r); });
    return OBGPU_SUCCESS;
  }
  // string class
  int64_t fix_len = -1;
  bool var = false;
  for (int64_t r = 0; r < nrows && !var; ++r) {
    if (c.is_null(r)) continue;
    const int64_t l = c.sval(r).len;
    if (fix_len < 0) fix_len = l;
    else if (fix_len != l) var = true;
  }
  if (!var && fix_len >= 0 && fix_len * c.null_cnt > nrows * 2) var = true;
  if (fix_len < 0) var = true;  // all NULL
  if (var || fix_len == 0) {
    o.is_var = true;
    o.need_ext_in_row = has_null;
    if (has_null) o.hdr.attr_ |= ATTR_HAS_EXTEND_VALUE;
    // offset_/length_ are set when the row data layout is fixed (set_data_pos)
    return OBGPU_SUCCESS;
  }
  o.hdr.attr_ |= ATTR_FIX_LENGTH;
  if (has_null) o.hdr.attr_ |= ATTR_HAS_EXTEND_VALUE;
  o.hdr.offset_ = (uint32_t)meta.size();
  o.hdr.length_ = (uint32_t)fix_len;
  {
    const int64_t bits_size = has_null ? ((int64_t)ext_bit * nrows + 7) / 8 : 0;
    uint8_t *buf = meta.grow((size_t)(bits_size + fix_len * nrows));
    if (has_null)
      for (int64_t r = 0; r < nrows; ++r)
        if (c.is_null(r)) put_bits(buf, r * ext_bit, ext_bit, c.ext_val(r));
    uint8_t *p = buf + bits_size;
    for (int64_t r = 0; r < nrows; ++r, p += fix_len)
      if (!c.is_null(r)) memcpy(p, c.sval(r).p, (size_t)fix_len);
  }
  return OBGPU_SUCCESS;
}

int BlockBuilder::encode_dict(int i) {
  ColCtx &c = ctx[i];
  ColOut &o = out[i];
  o.hdr.type_ = COL_DICT;
  const size_t meta_at = meta.size();
  std::vector<uint32_t> *refs = nullptr;
  IntDict idict;
  StrDict sdict;
  uint32_t cnt = 0;
  if (c.sc == 5) {
    build_str_dict(c, /*sorted=*/true, sdict);
    store_str_dict_meta(meta, sdict);
    refs = &sdict.refs;
    cnt = (uint32_t)sdict.values.size();
  } else {
    build_int_dict(c, /*sorted=*/true, idict);
    store_int_dict_meta(meta, c, idict, true);
    refs = &idict.refs;
    cnt = (uint32_t)idict.values.size();
  }
  if (cnt == 0) return OBGPU_NOT_SUPPORTED;  // all-NULL column: the reference picks CONST
  const uint64_t max_ref = c.nope_cnt > 0 ? cnt + 1 : (c.null_cnt > 0 ? cnt : cnt - 1);
  bool bp = false;
  const int64_t size = packing_size(&bp, max_ref, c.enable_bp);
  o.hdr.attr_ |= ATTR_FIX_LENGTH;
  if (bp) o.hdr.attr_ |= ATTR_BIT_PACKING;
  o.hdr.offset_ = (uint32_t)meta_at;
  o.hdr.length_ = (uint32_t)(meta.size() - meta_at);
  reinterpret_cast<DictMetaHeader *>(meta.d.data() + meta_at)->row_ref_size_ = (uint8_t)size;
  const std::vector<uint32_t> &rf = *refs;
  fill_column_store(meta, c, false, ext_bit, bp ? (int)size : 0, bp ? 0 : (int)size, true,
                    [&](int64_t r) { return (uint64_t)rf[(size_t)r]; });
  return OBGPU_SUCCESS;
}

int BlockBuilder::encode_rle(int i) {
  ColCtx &c = ctx[i];
  ColOut &o = out[i];
  o.hdr.type_ = COL_RLE;
  IntDict idict;
  StrDict sdict;
  const std::vector<uint32_t> *refs;
  uint32_t cnt;
  if (c.sc == 5) {
    build_str_dict(c, false, sdict);
    refs = &sdict.refs;
    cnt = (uint32_t)sdict.values.size();
  } else {
    build_int_dict(c, false, idict);
    refs = &idict.refs;
    cnt = (uint32_t)idict.values.size();
  }
  if (cnt == 0) return OBGPU_NOT_SUPPORTED;
  std::vector<uint32_t> run_row, run_ref;
  for (int64_t r = 0; r < nrows; ++r) {
    if (r == 0 || (*refs)[(size_t)r] != (*refs)[(size_t)r - 1]) {
      run_row.push_back((uint32_t)r);
      run_ref.push_back((*refs)[(size_t)r]);
    }
  }
  const uint64_t max_ref = c.nope_cnt > 0 ? cnt + 1 : (c.null_cnt > 0 ? cnt : cnt - 1);
  const int row_id_byte = (int)byte_packed_int_size(run_row.back());
  const int ref_byte = (int)byte_packed_int_size(max_ref);
  const size_t runs = run_row.size();
  // ObRLEDecoder keeps count * row_id_byte in an int16 (ob_rle_decoder.h:193): stay inside it.
  if ((int64_t)runs * row_id_byte > 32767) return OBGPU_NOT_SUPPORTED;
  const size_t meta_at = meta.size();
  const size_t head = sizeof(RLEMetaHeader) + runs * (size_t)(row_id_byte + ref_byte);
  uint8_t *p = meta.grow(head);
  RLEMetaHeader h{};
  h.attr_ = (uint8_t)((row_id_byte & 7) | ((ref_byte & 7) << 3));
  h.count_ = (uint32_t)runs;
  h.offset_ = (uint32_t)head;
  memcpy(p, &h, sizeof(h));
  uint8_t *rid = p + sizeof(h);
  uint8_t *rrf = rid + runs * (size_t)row_id_byte;
  for (size_t k = 0; k < runs; ++k) {
    memcpy(rid + k * (size_t)row_id_byte, &run_row[k], (size_t)row_id_byte);
    memcpy(rrf + k * (size_t)ref_byte, &run_ref[k], (size_t)ref_byte);
  }
  if (c.sc == 5) store_str_dict_meta(meta, sdict);
  else store_int_dict_meta(meta, c, idict, false);
  if (c.sc == 5 && !(sdict.fix_len < 0 || sdict.fix_len > 0xffff)) {
    // unsorted fixed-length string dict: clear the sorted attr set by the shared helper
    reinterpret_cast<DictMetaHeader *>(meta.d.data() + meta_at + head)->attr_ = DICT_FIX_LENGTH;
  }
  o.hdr.attr_ = 0;
  o.hdr.offset_ = (uint32_t)meta_at;
  o.hdr.length_ = (uint32_t)(meta.size() - meta_at);
  return OBGPU_SUCCESS;
}

// ---- string codecs that materialise their values (a10): HEX_PACKING, STRING_DIFF, STRING_PREFIX ----------------------------------
// Fixed store of encoded cells: [ext bits][nrows x cell_len bytes] after the codec meta (fill_column_store of these encoders).
void BlockBuilder::store_ext_then_fixed_cells(int i, int64_t cell_len) {
  ColCtx &c = ctx[(size_t)i];
  ColOut &o = out[(size_t)i];
  const bool has_null = c.null_cnt > 0;
  const int64_t bits_size = has_null ? ((int64_t)ext_bit * nrows + 7) / 8 : 0;
  uint8_t *buf = meta.grow((size_t)(bits_size + cell_len * nrows));
  if (has_null)
    for (int64_t r = 0; r < nrows; ++r)
      if (c.is_null(r)) put_bits(buf, r * ext_bit, ext_bit, c.ext_val(r));
  uint8_t *p = buf + bits_size;
  for (int64_t r = 0; r < nrows; ++r, p += cell_len)
    if (!c.is_null(r)) memcpy(p, o.cell_heap.data() + o.cell_off[(size_t)r], (size_t)cell_len);
  o.cell_heap.clear();
  o.cell_off.clear();
}

// HEX_PACKING (ObHexStringEncoder, encoding/ob_hex_string_encoder.cpp:83-262): strings over an alphabet of <= 16 bytes, two per byte.
//   meta: ObHexStringHeader {version u8, offset u32, length u32, max_string_size u32} + the alphabet (column header length = 13 + size)
//   fixed store (every value max_string_size long): (max + 1) / 2 bytes per row; var store: [odd u8][packed] in the row data
int BlockBuilder::encode_hex(int i) {
  ColCtx &c = ctx[(size_t)i];
  ColOut &o = out[(size_t)i];
  if (c.sc != 5) return OBGPU_NOT_SUPPORTED;
  o.hdr.type_ = COL_HEX_PACKING;
  o.own_meta = true;
  HexMap hm;
  int64_t min_len = INT64_MAX, max_len = -1;
  for (int64_t r = 0; r < nrows; ++r) {
    if (c.is_null(r)) continue;
    const StrRef v = c.sval(r);
    min_len = std::min(min_len, v.len);
    max_len = std::max(max_len, v.len);
    for (int64_t k = 0; k < v.len; ++k) hm.mark((uint8_t)v.p[k]);
  }
  if (!hm.can_packing() || max_len < 0) return OBGPU_NOT_SUPPORTED;   // the reference's "not suitable"
  bool fix_store = min_len == max_len;
  if (fix_store && c.null_cnt * ((max_len + 1) / 2) > (2 + 1) * nrows) fix_store = false;   // ext cells waste more than var indexes
  const bool has_null = c.null_cnt > 0;
  if (has_null) o.hdr.attr_ |= ATTR_HAS_EXTEND_VALUE;
  o.hdr.offset_ = (uint32_t)meta.size();
  o.hdr.length_ = (uint32_t)(13 + hm.size);
  uint8_t *h = meta.grow((size_t)(13 + hm.size));
  const uint32_t mx = (uint32_t)max_len;
  memcpy(h + 9, &mx, 4);
  hm.build_index(h + 13);
  o.pos_field_at = o.hdr.offset_ + 1;
  o.cell_off.assign((size_t)nrows + 1, 0);
  for (int64_t r = 0; r < nrows; ++r) {
    if (!c.is_null(r)) {
      const StrRef v = c.sval(r);
      if (!fix_store) o.cell_heap.push_back((uint8_t)(v.len % 2));   // ObVarHexCellHeader::odd_
      HexPacker pk(hm, o.cell_heap);
      for (int64_t k = 0; k < v.len; ++k) pk.pack((uint8_t)v.p[k]);
    }
    o.cell_off[(size_t)r + 1] = (int64_t)o.cell_heap.size();
  }
  if (fix_store) {
    o.hdr.attr_ |= ATTR_FIX_LENGTH;
    const uint32_t len = (uint32_t)((max_len + 1) / 2);
    memcpy(meta.d.data() + o.hdr.offset_ + 5, &len, 4);   // header_->length_ (store_fix_data)
    store_ext_then_fixed_cells(i, len);
  } else {
    o.is_var = true;
    o.need_ext_in_row = has_null;
  }
  return OBGPU_SUCCESS;
}

// STRING_DIFF (ObStringDiffEncoder, encoding/ob_string_diff_encoder.cpp:77-330): equal-length strings that share most positions.
//   meta: ObStringDiffHeader {version u8, hex_char_array_size u8, string_size u16, offset u32, length u32, diff_desc_cnt u8}
//         + DiffDesc[cnt] {diff:1, count:7} + alphabet (hex packing of the differing bytes) + the common bytes
//   per row: the differing bytes only (hex packed when <= 16 distinct bytes and more than one differs), fixed or var store
int BlockBuilder::encode_string_diff(int i) {
  ColCtx &c = ctx[(size_t)i];
  ColOut &o = out[(size_t)i];
  if (c.sc != 5) return OBGPU_NOT_SUPPORTED;
  o.hdr.type_ = COL_STRING_DIFF;
  o.own_meta = true;
  int64_t string_size = -1;
  const char *first = nullptr;
  std::vector<uint8_t> diff;
  for (int64_t r = 0; r < nrows; ++r) {
    if (c.is_null(r)) continue;
    const StrRef v = c.sval(r);
    if (string_size < 0) {
      if (v.len <= 0 || v.len >= 0xffff) return OBGPU_NOT_SUPPORTED;
      string_size = v.len;
      first = v.p;
      diff.assign((size_t)v.len, 0);
    } else if (v.len != string_size) {
      return OBGPU_NOT_SUPPORTED;
    } else {
      for (int64_t k = 0; k < string_size; ++k) if (v.p[k] != first[k]) diff[(size_t)k] = 1;
    }
  }
  if (string_size < 0 || c.null_cnt + 2 >= nrows) return OBGPU_NOT_SUPPORTED;
  HexMap hm;
  for (int64_t r = 0; r < nrows; ++r) {
    if (c.is_null(r)) continue;
    const StrRef v = c.sval(r);
    for (int64_t k = 0; k < string_size; ++k) if (diff[(size_t)k]) hm.mark((uint8_t)v.p[k]);
  }
  struct Desc { uint8_t diff, count; };
  std::vector<Desc> descs;
  int64_t common_size = 0;
  {
    int64_t begin = 0;
    uint8_t cur = diff[0];
    for (int64_t k = 0; k <= string_size; ++k) {
      if (k == string_size || diff[(size_t)k] != cur || k - begin == 0x7f) {
        descs.push_back(Desc{cur, (uint8_t)((k - begin) & 0x7f)});
        if (!cur) common_size += k - begin;
        begin = k;
        if (k < string_size) cur = diff[(size_t)k];
      }
    }
  }
  if (common_size == string_size || common_size == 0 || descs.size() > 255) return OBGPU_NOT_SUPPORTED;
  int64_t row_store = string_size - common_size;
  const bool hex = row_store > 1 && hm.can_packing();
  if (hex) row_store = (row_store + 1) / 2;
  const bool var_store = row_store * c.null_cnt > 2 * nrows;
  const bool has_null = c.null_cnt > 0;
  if (has_null) o.hdr.attr_ |= ATTR_HAS_EXTEND_VALUE;
  const size_t meta_size = 13 + descs.size() + (hex ? (size_t)hm.size : 0) + (size_t)common_size;
  o.hdr.offset_ = (uint32_t)meta.size();
  o.hdr.length_ = (uint32_t)meta_size;
  uint8_t *h = meta.grow(meta_size);
  h[1] = hex ? (uint8_t)hm.size : 0;
  const uint16_t ss = (uint16_t)string_size;
  memcpy(h + 2, &ss, 2);
  h[12] = (uint8_t)descs.size();
  for (size_t k = 0; k < descs.size(); ++k) h[13 + k] = (uint8_t)((descs[k].diff & 1) | (descs[k].count << 1));
  uint8_t *arr = h + 13 + descs.size();
  if (hex) hm.build_index(arr);
  uint8_t *common = arr + (hex ? hm.size : 0);
  for (int64_t k = 0, q = 0; k < string_size; ++k) if (!diff[(size_t)k]) common[q++] = (uint8_t)first[k];
  o.pos_field_at = o.hdr.offset_ + 4;
  o.cell_off.assign((size_t)nrows + 1, 0);
  for (int64_t r = 0; r < nrows; ++r) {
    if (!c.is_null(r)) {
      const StrRef v = c.sval(r);
      const size_t at = o.cell_heap.size();
      if (hex) {
        HexPacker pk(hm, o.cell_heap);
        for (int64_t k = 0; k < string_size; ++k) if (diff[(size_t)k]) pk.pack((uint8_t)v.p[k]);
      } else {
        for (int64_t k = 0; k < string_size; ++k) if (diff[(size_t)k]) o.cell_heap.push_back((uint8_t)v.p[k]);
      }
      o.cell_heap.resize(at + (size_t)row_store, 0);
    }
    o.cell_off[(size_t)r + 1] = (int64_t)o.cell_heap.size();
  }
  if (!var_store) {
    o.hdr.attr_ |= ATTR_FIX_LENGTH;
    const uint32_t len = (uint32_t)row_store;
    memcpy(meta.d.data() + o.hdr.offset_ + 8, &len, 4);
    store_ext_then_fixed_cells(i, row_store);
  } else {
    o.is_var = true;
    o.need_ext_in_row = has_null;
  }
  return OBGPU_SUCCESS;
}

// STRING_PREFIX (ObStringPrefixEncoder, encoding/ob_string_prefix_encoder.cpp:75-300): up to 16 shared prefixes in the meta, per row
// [ref:4 | odd:4][common length u16][rest of the string, hex packed when the rests use <= 16 distinct bytes]; always var-stored.
//   meta: ObStringPrefixMetaHeader {version u8, count u8, offset u32, length u32, max_string_size u32, {prefix_index_byte:2,
//         hex_char_array_size:5} u8} + alphabet + (count - 1) x prefix_index_byte start offsets + the prefixes
// The reference picks the prefixes with a multi-prefix tree (ob_multi_prefix_tree.cpp); any choice decodes the same way. Here: the
// longest common prefix of every group of strings that start with the same byte, the 16 largest groups.
int BlockBuilder::encode_string_prefix(int i) {
  ColCtx &c = ctx[(size_t)i];
  ColOut &o = out[(size_t)i];
  if (c.sc != 5) return OBGPU_NOT_SUPPORTED;
  o.hdr.type_ = COL_STRING_PREFIX;
  o.own_meta = true;
  struct Group { int64_t rows = 0; const char *p = nullptr; int64_t lcp = 0; };
  Group groups[256];
  int64_t max_len = 0;
  for (int64_t r = 0; r < nrows; ++r) {
    if (c.is_null(r)) continue;
    const StrRef v = c.sval(r);
    max_len = std::max(max_len, v.len);
    if (v.len == 0) continue;
    Group &g = groups[(uint8_t)v.p[0]];
    if (g.rows++ == 0) { g.p = v.p; g.lcp = std::min<int64_t>(v.len, 0xffff); }
    else {
      int64_t k = 0;
      while (k < g.lcp && k < v.len && v.p[k] == g.p[k]) ++k;
      g.lcp = k;
    }
  }
  std::vector<int> order;
  for (int b = 0; b < 256; ++b) if (groups[b].rows > 1) order.push_back(b);
  std::sort(order.begin(), order.end(), [&](int x, int y) { return groups[x].rows > groups[y].rows; });
  if (order.size() > 16) order.resize(16);
  if (order.empty()) return OBGPU_NOT_SUPPORTED;
  int ref_of_byte[256];
  for (int b = 0; b < 256; ++b) ref_of_byte[b] = -1;
  int64_t prefix_length = 0;
  for (size_t k = 0; k < order.size(); ++k) { ref_of_byte[order[k]] = (int)k; prefix_length += groups[order[k]].lcp; }
  if (prefix_length > 0xffff) return OBGPU_NOT_SUPPORTED;
  const int pib = prefix_length <= 0xff ? 1 : 2;
  // hex packing of the rests
  HexMap hm;
  for (int64_t r = 0; r < nrows; ++r) {
    if (c.is_null(r)) continue;
    const StrRef v = c.sval(r);
    const int ref = v.len ? ref_of_byte[(uint8_t)v.p[0]] : -1;
    const int64_t common = ref >= 0 ? groups[order[(size_t)ref]].lcp : 0;
    for (int64_t k = common; k < v.len; ++k) hm.mark((uint8_t)v.p[k]);
  }
  const bool hex = hm.can_packing() && hm.size > 0;
  const bool has_null = c.null_cnt > 0;
  if (has_null) o.hdr.attr_ |= ATTR_HAS_EXTEND_VALUE;
  const size_t cnt = order.size();
  const size_t meta_size = 15 + (hex ? (size_t)hm.size : 0) + (cnt - 1) * (size_t)pib + (size_t)prefix_length;
  o.hdr.offset_ = (uint32_t)meta.size();
  o.hdr.length_ = (uint32_t)meta_size;
  uint8_t *h = meta.grow(meta_size);
  h[1] = (uint8_t)cnt;
  const uint32_t mx = (uint32_t)max_len;
  memcpy(h + 10, &mx, 4);
  h[14] = (uint8_t)((pib & 3) | ((hex ? hm.size : 0) << 2));
  uint8_t *arr = h + 15;
  if (hex) hm.build_index(arr);
  uint8_t *idx = arr + (hex ? hm.size : 0);
  uint8_t *pdata = idx + (cnt - 1) * (size_t)pib;
  int64_t off = 0;
  for (size_t k = 0; k < cnt; ++k) {
    if (k > 0) { const uint32_t o32 = (uint32_t)off; memcpy(idx + (k - 1) * (size_t)pib, &o32, (size_t)pib); }
    memcpy(pdata + off, groups[order[k]].p, (size_t)groups[order[k]].lcp);
    off += groups[order[k]].lcp;
  }
  o.pos_field_at = o.hdr.offset_ + 2;
  o.cell_off.assign((size_t)nrows + 1, 0);
  for (int64_t r = 0; r < nrows; ++r) {
    if (!c.is_null(r)) {
      const StrRef v = c.sval(r);
      const int ref = v.len ? ref_of_byte[(uint8_t)v.p[0]] : -1;
      const int64_t common = ref >= 0 ? groups[order[(size_t)ref]].lcp : 0;
      const int64_t rest = v.len - common;
      const uint16_t cl = (uint16_t)common;
      o.cell_heap.push_back((uint8_t)(((ref >= 0 ? ref : 0) & 0xf) | ((hex ? (rest % 2) : 0) << 4)));
      o.cell_heap.push_back((uint8_t)(cl & 0xff));
      o.cell_heap.push_back((uint8_t)(cl >> 8));
      if (hex) {
        HexPacker pk(hm, o.cell_heap);
        for (int64_t k = common; k < v.len; ++k) pk.pack((uint8_t)v.p[k]);
      } else {
        o.cell_heap.insert(o.cell_heap.end(), (const uint8_t *)v.p + common, (const uint8_t *)v.p + v.len);
      }
    }
    o.cell_off[(size_t)r + 1] = (int64_t)o.cell_heap.size();
  }
  o.is_var = true;
  o.need_ext_in_row = has_null;
  return OBGPU_SUCCESS;
}

// ---- span columns (a10): COLUMN_EQUAL, COLUMN_SUBSTR -----------------------------------------------------------------------------
// Exception rows of a span column: ObBitMapMetaWriter (encoding/ob_encoding_bitset.h:163-557).
//   ObBitMapMetaHeader {ext_offset u8, index_offset u8, data_offset u8, {bit_packing_len | fix_data_cnt | index_byte} u8}
//   + BitSet of the exception rows (64-bit words over every row of the block) + 2 ext bits per exception (only when one of them is
//   NULL / NOP) + (count - 1) start offsets (var-length exceptions) + the exception values (bit packed / fixed / var);
//   an extend value keeps its slot in the bit-packed and fixed layouts and takes no bytes in the var layout.
// Returns false when the reference's writer calls the column "not suitable" (the three offsets are uint8).
struct ExcMeta {
  std::vector<uint8_t> bytes;
  bool bit_packing = false;
};
bool build_exc_meta(const ColCtx &c, const std::vector<int64_t> &exc, ExcMeta &m) {
  const int64_t count = (int64_t)exc.size();
  bool has_ext = false, var_store = false, bp = false;
  int64_t total = 0, fix = -1, index_byte = 0;
  uint64_t max_integer = 0;
  for (int64_t rid : exc) {
    if (c.is_null(rid)) { has_ext = true; continue; }
    if (c.sc == 5) {
      const int64_t len = c.sval(rid).len;
      total += len;
      if (!var_store) {
        if (fix < 0) fix = len;
        else if (len != fix) { fix = -1; var_store = true; }
      }
    } else {
      max_integer = std::max(max_integer, c.uval(rid));
    }
  }
  if (c.sc != 5) {   // fill_param<ObIntSC>: get_packing_size with its default enable_bit_packing
    fix = packing_size(&bp, max_integer, true);
    total = fix * count;
    if (bp) total = (total + 7) / 8;
  } else if (fix < 0) {
    index_byte = total <= 0xff ? 1 : total <= 0xffff ? 2 : total <= 0xffffffffll ? 4 : 8;
  } else {
    total = fix * count;
  }
  const int64_t ext_len = (c.nrows + 63) / 64 * 8;
  const int64_t bs_len = has_ext ? (count * 2 + 7) / 8 : 0;
  const int64_t index_len = fix < 0 ? (count - 1) * index_byte : 0;
  if (ext_len + bs_len + index_len > 0xff) return false;
  m.bit_packing = bp;
  m.bytes.assign((size_t)(4 + ext_len + bs_len + index_len + total + 8), 0);   // 8: the reference's safety bytes for bit packing
  uint8_t *h = m.bytes.data(), *buf = h + 4;
  h[0] = (uint8_t)ext_len;
  h[1] = (uint8_t)(ext_len + bs_len);
  h[2] = (uint8_t)(ext_len + bs_len + index_len);
  h[3] = (uint8_t)(bp ? fix : (fix < 0 ? index_byte : count));
  uint8_t *data = buf + h[2];
  int64_t offset = 0;
  for (int64_t ref = 0; ref < count; ++ref) {
    const int64_t rid = exc[(size_t)ref];
    buf[rid / 8] |= (uint8_t)(1u << (rid % 8));   // BitSet::set on little-endian 64-bit words
    const bool ext = c.is_null(rid);
    if (has_ext && ext) put_bits(buf + h[0], ref * 2, 2, c.ext_val(rid));
    if (c.sc != 5) {
      if (!ext) {
        if (bp) put_bits(data, offset, (int)fix, c.ival(rid) & low_mask((int)fix));
        else { const uint64_t v = (uint64_t)c.ival(rid); memcpy(data + offset, &v, (size_t)fix); }
      }
      offset += fix;
    } else if (fix < 0) {
      if (ref > 0) { const uint64_t o = (uint64_t)offset; memcpy(buf + h[1] + (ref - 1) * index_byte, &o, (size_t)index_byte); }
      if (!ext) { const StrRef v = c.sval(rid); if (v.len) memcpy(data + offset, v.p, (size_t)v.len); offset += v.len; }
    } else {
      if (!ext && fix) memcpy(data + offset, c.sval(rid).p, (size_t)fix);
      offset += fix;
    }
  }
  m.bytes.resize(m.bytes.size() - 8);
  return true;
}

// the column a span column refers to: an ordinary column of the same type
int BlockBuilder::span_ref_of(int i) const {
  const int ref = cols[i].ref_col;
  if (ref < 0 || ref >= ncol || ref == i || cols[ref].obj_type != cols[i].obj_type) return -1;
  if (cols[ref].encoding == OBGPU_ENC_COLUMN_EQUAL || cols[ref].encoding == OBGPU_ENC_COLUMN_SUBSTR) return -1;
  return ref;
}

// COLUMN_EQUAL (ObColumnEqualEncoder, encoding/ob_column_equal_encoder.cpp:84-301): the column equals column ref_col_idx in every
// row but the exception rows.  meta: ObColumnEqualMetaHeader {version u8, ref_col_idx u16} (+ the exception meta); nothing else.
// At most min(100, rows / 10 + 1) exceptions (ObSpanColumnEncoder::MAX_EXC_CNT / EXC_THRESHOLD_PCT, ob_icolumn_encoder.cpp:94-95).
int BlockBuilder::encode_column_equal(int i) {
  ColCtx &c = ctx[(size_t)i];
  ColOut &o = out[(size_t)i];
  const int ref = span_ref_of(i);
  if (ref < 0) return OBGPU_INVALID_ARGUMENT;
  const ColCtx &rc = ctx[(size_t)ref];
  std::vector<int64_t> exc;
  for (int64_t r = 0; r < nrows; ++r) {   // is_datum_equal (ob_column_equal_encoder.h:90-110)
    const int le = c.is_null(r) ? (int)c.ext_val(r) : 0, re = rc.is_null(r) ? (int)rc.ext_val(r) : 0;
    bool equal;
    if (le != re) equal = false;
    else if (le) equal = true;
    else if (c.sc != 5) equal = c.ival(r) == rc.ival(r);
    else { const StrRef a = c.sval(r), b = rc.sval(r); equal = a.len == b.len && (a.len == 0 || memcmp(a.p, b.p, (size_t)a.len) == 0); }
    if (!equal) exc.push_back(r);
  }
  if ((int64_t)exc.size() > std::min<int64_t>(100, nrows * 10 / 100 + 1)) return OBGPU_NOT_SUPPORTED;
  ExcMeta em;
  if (!exc.empty() && !build_exc_meta(c, exc, em)) return OBGPU_NOT_SUPPORTED;
  o.hdr.type_ = COL_COLUMN_EQUAL;
  o.hdr.attr_ = em.bit_packing ? ATTR_BIT_PACKING : 0;
  o.hdr.offset_ = (uint32_t)meta.size();
  o.hdr.length_ = (uint32_t)(3 + em.bytes.size());
  uint8_t *h = meta.grow(3 + em.bytes.size());
  const uint16_t r16 = (uint16_t)ref;
  memcpy(h + 1, &r16, 2);
  if (!em.bytes.empty()) memcpy(h + 3, em.bytes.data(), em.bytes.size());
  return OBGPU_SUCCESS;
}

// COLUMN_SUBSTR (ObInterColSubStrEncoder, encoding/ob_inter_column_substring_encoder.cpp:103-395): every value is a substring of
// the same row's value in column ref_col_idx (first occurrence, memmem), but the exception rows.
//   meta: ObInterColSubStrMetaHeader {version u8, {start_pos_byte:2, val_len_byte:2, is_same_start_pos:1, is_fix_length:1} u8,
//         start_pos u16, length u16, ref_col_idx u16} (+ the exception meta)
//   fixed store after the meta, no ext bits: per row [start_pos, start_pos_byte bytes][value length, val_len_byte bytes]; a field
//   every row shares lives in the header instead. Both cells NULL / NOP: start 0, length 0; exception rows: start -2.
int BlockBuilder::encode_column_substr(int i) {
  ColCtx &c = ctx[(size_t)i];
  ColOut &o = out[(size_t)i];
  const int ref = span_ref_of(i);
  if (ref < 0) return OBGPU_INVALID_ARGUMENT;
  if (c.sc != 5) return OBGPU_NOT_SUPPORTED;
  const ColCtx &rc = ctx[(size_t)ref];
  std::vector<int64_t> exc, start((size_t)nrows, 0);
  int64_t same_start = -1, fix_size = -1, max_start = 0, max_len = 0;
  bool is_same = true, var_data = false;
  for (int64_t r = 0; r < nrows; ++r) {
    const bool ce = c.is_null(r), re = rc.is_null(r);
    if (!ce) max_len = std::max(max_len, c.sval(r).len);
    if (ce && re) continue;   // EXT_START_POS: recorded as 0, excluded from the same-start / fixed-length tests
    int64_t sp = -2;          // EXCEPTION_START_POS
    if (!ce && !re) {
      const StrRef v = c.sval(r), w = rc.sval(r);
      if (v.len <= w.len) {
        const void *found = v.len == 0 ? (const void *)w.p : memmem(w.p, (size_t)w.len, v.p, (size_t)v.len);
        if (found) sp = (const char *)found - w.p;
      }
    }
    start[(size_t)r] = sp;
    if (sp < 0) { exc.push_back(r); continue; }
    max_start = std::max(max_start, sp);
    if (is_same) {
      if (same_start == -1) same_start = sp;
      else if (!(is_same = (same_start == sp))) same_start = -1;
    }
    if (!var_data) {
      const int64_t len = c.sval(r).len;
      if (fix_size < 0) fix_size = len;
      else if (len != fix_size) { fix_size = -1; var_data = true; }
    }
  }
  if (max_start >= 0xffff || max_len >= 0xffff) return OBGPU_NOT_SUPPORTED;
  if ((int64_t)exc.size() > std::min<int64_t>(100, nrows * 10 / 100 + 1)) return OBGPU_NOT_SUPPORTED;
  ExcMeta em;
  if (!exc.empty() && !build_exc_meta(c, exc, em)) return OBGPU_NOT_SUPPORTED;
  int spb = 0, vlb = 0;
  if (!(fix_size > 0 && same_start >= 0)) {
    if (same_start < 0) spb = max_start <= 0xff ? 1 : 2;
    if (fix_size < 0) vlb = max_len <= 0xff ? 1 : 2;
  }
  o.hdr.type_ = COL_COLUMN_SUBSTR;
  o.hdr.attr_ = ATTR_FIX_LENGTH;
  o.hdr.offset_ = (uint32_t)meta.size();
  o.hdr.length_ = (uint32_t)(8 + em.bytes.size());
  uint8_t *h = meta.grow(8 + em.bytes.size());
  uint8_t attr = 0;
  uint16_t sp16 = 0, len16 = 0;
  const uint16_t r16 = (uint16_t)ref;
  if (same_start >= 0) { sp16 = (uint16_t)same_start; attr |= 1u << 4; } else attr |= (uint8_t)(spb & 3);
  if (fix_size >= 0) { len16 = (uint16_t)fix_size; attr |= 1u << 5; } else attr |= (uint8_t)((vlb & 3) << 2);
  h[1] = attr;
  memcpy(h + 2, &sp16, 2);
  memcpy(h + 4, &len16, 2);
  memcpy(h + 6, &r16, 2);
  if (!em.bytes.empty()) memcpy(h + 8, em.bytes.data(), em.bytes.size());
  if (spb + vlb > 0) {
    uint8_t *p = meta.grow((size_t)((spb + vlb) * nrows));
    for (int64_t r = 0; r < nrows; ++r, p += spb + vlb) {
      if (spb) memcpy(p, &start[(size_t)r], (size_t)spb);
      const int64_t vl = c.is_null(r) ? 0 : c.sval(r).len;   // an extend value's length is forced to 0
      if (vlb) memcpy(p + spb, &vl, (size_t)vlb);
    }
  }
  return OBGPU_SUCCESS;
}

// CONST: one dominant value (or NULL) + at most 32 exception rows
// (ob_const_encoder.cpp:58-131 traverse / suitability, :154-196 no-exception meta, :296-356 meta with
// exceptions: [header][count x u8 ref][count x row_id_byte row ids][sorted dict meta]).
int BlockBuilder::encode_const(int i) {
  ColCtx &c = ctx[i];
  ColOut &o = out[i];
  o.hdr.type_ = COL_CONST;
  o.hdr.attr_ = 0;  // need_data_store_ = false, no ext bits: NULL is a dict ref
  if (c.nope_cnt > 0) return OBGPU_NOT_SUPPORTED;  // NOP cells only arise in incremental runs: RAW / DICT / RLE
  IntDict idict;
  StrDict sdict;
  const std::vector<uint32_t> *refs;
  uint32_t cnt;
  if (c.sc == 5) {
    build_str_dict(c, true, sdict);
    refs = &sdict.refs;
    cnt = (uint32_t)sdict.values.size();
  } else {
    build_int_dict(c, true, idict);
    refs = &idict.refs;
    cnt = (uint32_t)idict.values.size();
  }
  // the constant: most frequent ref; NULL (ref == cnt) wins only when strictly more frequent
  std::vector<int64_t> freq((size_t)cnt + 1, 0);
  for (int64_t r = 0; r < nrows; ++r) freq[(*refs)[(size_t)r]]++;
  uint32_t const_ref = 0;
  int64_t max_cnt = 0;
  for (uint32_t k = 0; k <= cnt; ++k)
    if (freq[k] > max_cnt) { max_cnt = freq[k]; const_ref = k; }
  const int64_t exceptions = nrows - max_cnt;
  if (exceptions > 32 || exceptions > std::max<int64_t>(nrows * 10 / 100, 1)) return OBGPU_NOT_SUPPORTED;
  const size_t meta_at = meta.size();
  ConstMetaHeader h{};
  if (exceptions == 0) {
    h.offset_ = (uint16_t)sizeof(ConstMetaHeader);
    if (cnt == 0) {  // every row NULL
      h.const_ref_ = 1;
      memcpy(meta.grow(sizeof(h)), &h, sizeof(h));
    } else if (c.sc == 5) {
      const StrRef &v = sdict.values[0];
      uint8_t *p = meta.grow(sizeof(h) + (size_t)v.len);
      memcpy(p, &h, sizeof(h));
      memcpy(p + sizeof(h), v.p, (size_t)v.len);
    } else {
      const int ts = type_store_size((uint8_t)c.in->obj_type);
      uint8_t *p = meta.grow(sizeof(h) + (size_t)ts);
      memcpy(p, &h, sizeof(h));
      memcpy(p + sizeof(h), &idict.values[0], (size_t)ts);
    }
  } else {
    if (cnt + 1 > 255) return OBGPU_NOT_SUPPORTED;
    int64_t max_row_id = 0;
    for (int64_t r = nrows - 1; r >= 0; --r)
      if ((*refs)[(size_t)r] != const_ref) { max_row_id = r; break; }
    const int row_id_byte = (int)byte_packed_int_size((uint64_t)max_row_id);
    const size_t head = sizeof(h) + (size_t)exceptions * (size_t)(row_id_byte + 1);
    if (head > 0xffff) return OBGPU_NOT_SUPPORTED;
    h.count_ = (uint8_t)exceptions;
    h.const_ref_ = (uint8_t)const_ref;
    h.row_id_byte_ = (uint8_t)(row_id_byte & 7);
    h.offset_ = (uint16_t)head;
    uint8_t *p = meta.grow(head);
    memcpy(p, &h, sizeof(h));
    uint8_t *rf = p + sizeof(h), *rid = rf + exceptions;
    int64_t k = 0;
    for (int64_t r = 0; r < nrows; ++r) {
      const uint32_t ref = (*refs)[(size_t)r];
      if (ref == const_ref) continue;
      rf[k] = (uint8_t)ref;
      const uint32_t r32 = (uint32_t)r;
      memcpy(rid + k * row_id_byte, &r32, (size_t)row_id_byte);
      ++k;
    }
    if (c.sc == 5) store_str_dict_meta(meta, sdict);
    else store_int_dict_meta(meta, c, idict, true);
  }
  o.hdr.offset_ = (uint32_t)meta_at;
  o.hdr.length_ = (uint32_t)(meta.size() - meta_at);
  return OBGPU_SUCCESS;
}

int BlockBuilder::encode_base_diff(int i) {
  ColCtx &c = ctx[i];
  ColOut &o = out[i];
  if (c.sc != 1 && c.sc != 2) return OBGPU_INVALID_ARGUMENT;
  const uint8_t t = (uint8_t)c.in->obj_type;
  const int ts = type_store_size(t);
  bool any = false;
  int64_t smin = INT64_MAX, smax = INT64_MIN;
  uint64_t umin = UINT64_MAX, umax = 0;
  auto to_signed = [&](uint64_t v) {
    const uint64_t rev = ~low_mask(ts * 8);
    if (rev != 0 && (v & (rev >> 1))) v |= rev;
    return (int64_t)v;
  };
  for (int64_t r = 0; r < nrows; ++r) {
    if (c.is_null(r)) continue;
    any = true;
    if (c.sc == 1) {
      const int64_t v = to_signed(c.uval(r));
      smin = std::min(smin, v);
      smax = std::max(smax, v);
    } else {
      const uint64_t v = c.uval(r);
      umin = std::min(umin, v);
      umax = std::max(umax, v);
    }
  }
  const uint64_t delta = !any ? 0 : (c.sc == 1 ? (uint64_t)smax - (uint64_t)smin : umax - umin);
  if (delta == 0) return encode_raw(i);  // "not suitable for integer base diff" -> RAW
  const uint64_t base = c.sc == 1 ? (uint64_t)smin : umin;
  bool bp = false;
  const int64_t size = packing_size(&bp, delta, true);
  o.hdr.type_ = COL_INTEGER_BASE_DIFF;
  o.hdr.attr_ |= ATTR_FIX_LENGTH;
  if (bp) o.hdr.attr_ |= ATTR_BIT_PACKING;
  const bool has_null = c.null_cnt > 0;
  if (has_null) o.hdr.attr_ |= ATTR_HAS_EXTEND_VALUE;
  const size_t meta_at = meta.size();
  uint8_t *p = meta.grow(sizeof(IntegerBaseDiffHeader) + (size_t)ts);
  IntegerBaseDiffHeader h{0, (uint8_t)size};
  memcpy(p, &h, sizeof(h));
  memcpy(p + sizeof(h), &base, (size_t)ts);
  o.hdr.offset_ = (uint32_t)meta_at;
  o.hdr.length_ = (uint32_t)(meta.size() - meta_at);
  fill_column_store(meta, c, has_null, ext_bit, bp ? (int)size : 0, bp ? 0 : (int)size, false,
                    [&](int64_t r) {
                      return c.sc == 1 ? (uint64_t)to_signed(c.uval(r)) - base : c.uval(r) - base;
                    });
  return OBGPU_SUCCESS;
}

// ---- encoder selection (OBGPU_ENC_AUTO) ------------------------------------------------------------------------------------------
// ObMicroBlockEncoder::encoder_detection -> fast_encoder_detect / choose_encoder (ob_micro_block_encoder.cpp:1259-1366,1603-1823) for
// the first micro-block of an SSTable (no previous-block hints, try_previous_encoder :1445-1497 has nothing to try) over the codecs
// whose size estimates depend on the column alone: RAW, DICT, RLE, CONST, INTEGER_BASE_DIFF. Span columns (COLUMN_EQUAL / SUBSTR need
// the cross-column detection) and the string transforms (STRING_DIFF / PREFIX / HEX) are only written when the caller names them.
// Every estimate is the encoder's own calc_size() over the column's ObColumnEncodingCtx (build_column_encoding_ctx,
// ob_encoding_hash_util.cpp:374-470), restated; a candidate replaces the choice only when STRICTLY smaller, in the reference's order,
// and the search stops once the choice is within a quarter of the RAW size.
int choose_auto_encoding(const ColCtx &c, int ext_bit) {
  const int64_t n = c.nrows;
  const bool is_int = c.sc == 1 || c.sc == 2;
  const int64_t ts = is_int ? type_store_size((uint8_t)c.in->obj_type) : 0;
  const int64_t null_cnt = c.null_cnt - c.nope_cnt, nope_cnt = c.nope_cnt, ext_cnt = c.null_cnt;
  // ---- ObColumnEncodingCtx: distinct values in first-occurrence order (the hash table's dict refs), per-row refs ----------------
  std::vector<uint32_t> refs;
  std::vector<int64_t> value_rows;   // rows per distinct value
  int64_t distinct = 0, fix_data_size = ts, dict_var_data_size = 0, var_data_size = 0;
  uint64_t max_integer = 0;
  if (is_int) {
    IntDict d;
    build_int_dict(c, false, d);
    refs.swap(d.refs);
    distinct = (int64_t)d.values.size();
    max_integer = d.max_integer;
  } else {
    StrDict d;
    build_str_dict(c, false, d);
    refs.swap(d.refs);
    distinct = (int64_t)d.values.size();
    fix_data_size = -1;
    bool var_store = false;
    for (const StrRef &v : d.values) {
      dict_var_data_size += v.len;
      if (!var_store) {
        if (fix_data_size < 0) fix_data_size = v.len;
        else if (v.len != fix_data_size) { fix_data_size = -1; var_store = true; }
      }
    }
    for (int64_t r = 0; r < n; ++r) if (!c.is_null(r)) var_data_size += c.sval(r).len;
  }
  value_rows.assign((size_t)distinct + 2, 0);
  for (int64_t r = 0; r < n; ++r) value_rows[refs[(size_t)r]]++;
  const int64_t ext_store = (ext_cnt > 0) ? (n * ext_bit + 1) / 8 : 0;
  // ---- ObRawEncoder::traverse + calc_size (ob_raw_encoder.cpp:88-165,256-273) -----------------------------------------------------
  int64_t raw_size;
  {
    int64_t bp_len = 0, fix_len = 0, raw_var = 0;
    bool is_var = false;
    if (is_int) {
      bool bp = false;
      const int64_t size = packing_size(&bp, max_integer, c.enable_bp);
      if (bp) {
        if (size * ext_cnt > n * 2 * 8) { is_var = true; raw_var = (size / 8 + 1) * (n - ext_cnt); }
        else bp_len = size;
      } else {
        fix_len = size;
      }
    } else if (fix_data_size < 0) {
      is_var = true;
      raw_var = var_data_size;
    } else {
      fix_len = fix_data_size;
      raw_var = var_data_size;
    }
    if (fix_len > 0 && bp_len == 0 && fix_len * ext_cnt > n * 2) { is_var = true; fix_len = 0; }   // (integers: var_data_size_ stays 0 here, :147-152)
    raw_size = bp_len > 0 ? bp_len * n / 8 + 1 : (!is_var ? fix_len * n : raw_var + n * 2);
    raw_size += ext_store;
  }
  // ---- ObDictEncoder::traverse / calc_meta_size / calc_size (ob_dict_encoder.cpp:83-133, ob_dict_encoder.h:98-125) ----------------
  int64_t dict_fix = is_int ? (c.enable_bp ? int_size_bytes(max_integer) : byte_packed_int_size(max_integer)) : fix_data_size;
  const bool var_dict = dict_fix < 0 || dict_fix > 0xffff;
  const int64_t dict_index_byte = dict_var_data_size <= 0xff ? 1 : (dict_var_data_size <= 0xffff ? 2 : 4);
  const int64_t dict_meta = 9 /*ObDictMetaHeader*/ + (var_dict ? dict_index_byte * (distinct - 1) + dict_var_data_size : dict_fix * distinct);
  int64_t dict_size;
  {
    int64_t max_ref = distinct - 1;
    if (null_cnt > 0) max_ref = distinct;
    if (nope_cnt > 0) max_ref = distinct + 1;
    bool bp = false;
    const int64_t size = packing_size(&bp, (uint64_t)std::max<int64_t>(max_ref, 0), c.enable_bp);
    dict_size = dict_meta + (bp ? (n * size + 7) / 8 : n * size);
  }
  // ---- ObConstEncoder::traverse / calc_size (ob_const_encoder.cpp:57-160): the most frequent value is the constant ---------------
  bool const_ok = true;
  int64_t const_size = 0;
  {
    int64_t max_cnt = 0, const_ref = 0;
    for (int64_t v = 0; v < distinct; ++v) if (value_rows[(size_t)v] > max_cnt) { max_cnt = value_rows[(size_t)v]; const_ref = v; }
    if (null_cnt > max_cnt) { max_cnt = null_cnt; const_ref = distinct; }
    if (nope_cnt > max_cnt) { max_cnt = nope_cnt; const_ref = distinct + 1; }
    const int64_t exc = n - max_cnt;
    if (nope_cnt - 1 > 32 + 1 || exc > 32 || exc > std::max<int64_t>(n * 10 / 100, 1)) {   // MAX_EXCEPTION_SIZE / MAX_EXCEPTION_PCT
      const_ok = false;
    } else if (exc == 0) {
      int64_t cell = 0;
      if (null_cnt == 0 && nope_cnt == 0) cell = is_int ? ts : (n > 0 ? c.sval(0).len : 0);   // get_cell_len of the constant
      const_size = cell + 6 /*ObConstMetaHeader*/;
    } else {
      int64_t max_row_id = 0;
      for (int64_t r = n - 1; r >= 0; --r) if ((int64_t)refs[(size_t)r] != const_ref) { max_row_id = r; break; }
      const_size = 6 + dict_meta + exc * (byte_packed_int_size((uint64_t)max_row_id) + 1);
    }
  }
  // ---- fast_encoder_detect (:1318-1366): at most one distinct value -> CONST when it is suitable -----------------------------------
  if (distinct <= 1 && const_ok) return OBGPU_ENC_CONST;
  int choose = OBGPU_ENC_RAW;
  int64_t choose_size = raw_size;
  const int64_t acceptable = raw_size / 4;
  if (dict_size < choose_size) { choose = OBGPU_ENC_DICT; choose_size = dict_size; }
  bool try_more = true;
  // (previous-block encodings, COLUMN_EQUAL, COLUMN_SUBSTR: nothing to try here)
  if (try_more && distinct <= n / 2) {   // "try rle and const" (:1686-1713)
    int64_t runs = n > 0 ? 1 : 0, max_rle_row_id = 0;
    for (int64_t r = 1; r < n; ++r) if (refs[(size_t)r] != refs[(size_t)r - 1]) { ++runs; max_rle_row_id = r; }
    int64_t max_ref = distinct - 1;
    if (null_cnt > 0) max_ref = distinct;
    if (nope_cnt > 0) max_ref = distinct + 1;
    const int64_t rle_size = 10 /*ObRLEMetaHeader*/ + dict_meta +
        runs * (byte_packed_int_size((uint64_t)max_rle_row_id) + byte_packed_int_size((uint64_t)std::max<int64_t>(max_ref, 0)));
    if (rle_size < choose_size) { choose = OBGPU_ENC_RLE; choose_size = rle_size; }
    if (const_ok && const_size < choose_size) { choose = OBGPU_ENC_CONST; choose_size = const_size; }
  }
  if (try_more && choose_size <= acceptable) try_more = false;
  if (try_more && is_int) {   // ObIntegerBaseDiffEncoder::traverse / calc_size (ob_integer_base_diff_encoder.cpp:163-224,254-265)
    // ObIntegerData<T>::traverse_cell / max_delta / max_unsign_value (:43-73): min / max over the stored images, sign-extended for
    // the signed class; a negative minimum makes the "original" width 64 bits
    bool any = false;
    int64_t smin = INT64_MAX, smax = INT64_MIN;
    uint64_t umin = UINT64_MAX, umax = 0;
    const uint64_t rev = ~low_mask((uint32_t)ts * 8);
    for (int64_t r = 0; r < n; ++r) {
      if (c.is_null(r)) continue;
      any = true;
      uint64_t v = c.uval(r);
      if (c.sc == 1) {
        if (rev != 0 && (v & (rev >> 1))) v |= rev;
        smin = std::min(smin, (int64_t)v);
        smax = std::max(smax, (int64_t)v);
      } else {
        umin = std::min(umin, v);
        umax = std::max(umax, v);
      }
    }
    const uint64_t delta = !any ? 0 : (c.sc == 1 ? (smin < smax ? (uint64_t)smax - (uint64_t)smin : 0) : (umin < umax ? umax - umin : 0));
    const uint64_t max_unsigned = !any ? 0 : (c.sc == 1 ? (smin < 0 ? ~0ull : (uint64_t)smax) : umax);
    if (delta != 0) {
      bool bp = false;
      int64_t orig = packing_size(&bp, max_unsigned, true);
      if (!bp) orig *= 8;
      bp = false;
      int64_t dsz = packing_size(&bp, delta, true);
      if (!bp) dsz *= 8;
      if ((orig - dsz) * n > (2 /*header*/ + ts) * 8) {
        const int64_t bd_size = (bp ? (n * dsz + 7) / 8 : n * (dsz / 8)) + 2 + ts;
        if (bd_size < choose_size) { choose = OBGPU_ENC_INTEGER_BASE_DIFF; choose_size = bd_size; }
      }
    }
  }
  return choose;
}

int BlockBuilder::build(std::vector<uint8_t> &block) {
  if (ncol <= 0 || nrows <= 0 || nrows > 0x7fffffff || rowkey_cnt < 0 || rowkey_cnt > ncol)
    return OBGPU_INVALID_ARGUMENT;
  ctx.resize((size_t)ncol);
  out.resize((size_t)ncol);
  int64_t original = 0;
  for (int i = 0; i < ncol; ++i) {
    ColCtx &c = ctx[(size_t)i];
    c.in = &cols[i];
    c.sc = store_class_of((uint8_t)cols[i].obj_type);
    c.row_begin = row_begin;
    c.nrows = nrows;
    c.enable_bp = !cols[i].byte_packing_only;
    if (c.sc == 0) return OBGPU_NOT_SUPPORTED;
    if ((c.sc == 5 && (!cols[i].str_heap || !cols[i].str_off)) || (c.sc != 5 && !cols[i].i64))
      return OBGPU_INVALID_ARGUMENT;
    for (int64_t r = 0; r < nrows; ++r) {
      if (c.is_null(r)) { c.null_cnt++; if (c.ext_val(r) == STORED_NOPE) c.nope_cnt++; }
      else original += c.sc == 5 ? c.sval(r).len : datum_len_of((uint8_t)cols[i].obj_type);
    }
    // ob_micro_block_encoder.cpp:507-517: 1 bit when only NULLs occur, 2 bits once any column has a NOP
    if (c.null_cnt > 0 && ext_bit < 1) ext_bit = 1;
    if (c.nope_cnt > 0) ext_bit = 2;
  }
  {
    int n_cs = 0;
    for (int i = 0; i < ncol; ++i) n_cs += (cols[i].encoding >= OBGPU_ENC_CS_INTEGER && cols[i].encoding <= OBGPU_ENC_CS_STR_DICT) || cols[i].encoding == OBGPU_ENC_CS_AUTO;
    if (n_cs == ncol) return build_cs(block, original);
    if (n_cs != 0) return OBGPU_INVALID_ARGUMENT;  // one row store type per block
  }
  for (int i = 0; i < ncol; ++i) {
    out[(size_t)i].hdr.obj_type_ = (uint8_t)cols[i].obj_type;
    int ret;
    const int enc = cols[i].encoding == OBGPU_ENC_AUTO ? choose_auto_encoding(ctx[(size_t)i], ext_bit) : cols[i].encoding;
    switch (enc) {
      case OBGPU_ENC_RAW: ret = encode_raw(i); break;
      case OBGPU_ENC_DICT: ret = encode_dict(i); break;
      case OBGPU_ENC_RLE: ret = encode_rle(i); break;
      case OBGPU_ENC_INTEGER_BASE_DIFF: ret = encode_base_diff(i); break;
      case OBGPU_ENC_CONST: ret = encode_const(i); break;
      case OBGPU_ENC_HEX_PACKING: ret = encode_hex(i); break;
      case OBGPU_ENC_STRING_DIFF: ret = encode_string_diff(i); break;
      case OBGPU_ENC_STRING_PREFIX: ret = encode_string_prefix(i); break;
      case OBGPU_ENC_COLUMN_EQUAL: ret = encode_column_equal(i); break;
      case OBGPU_ENC_COLUMN_SUBSTR: ret = encode_column_substr(i); break;
      default: ret = OBGPU_NOT_SUPPORTED;
    }
    if (ret != OBGPU_SUCCESS) return ret;
  }
  // ---- row data: var-stored columns (set_row_data_pos / fill_row_data) ------------------------
  std::vector<int> var_cols;
  int64_t ext_bits_in_row = 0;
  for (int i = 0; i < ncol; ++i) {
    if (!out[(size_t)i].is_var) continue;
    var_cols.push_back(i);
    if (out[(size_t)i].need_ext_in_row) {
      out[(size_t)i].hdr.extend_value_index_ = (uint32_t)ext_bits_in_row;
      ext_bits_in_row += ext_bit;
    }
  }
  const int64_t fix_data_size = (ext_bits_in_row + 7) / 8;
  for (size_t k = 0; k < var_cols.size(); ++k) {
    ColOut &vo = out[(size_t)var_cols[k]];
    const uint32_t row_off = (uint32_t)fix_data_size, var_idx = (uint32_t)k;   // set_data_pos(fix_data_size, i)
    if (vo.own_meta) {   // the codec's own header carries the row position; the column header keeps pointing at the meta
      memcpy(meta.d.data() + vo.pos_field_at, &row_off, 4);
      memcpy(meta.d.data() + vo.pos_field_at + 4, &var_idx, 4);
    } else {
      vo.hdr.offset_ = row_off;   // row_offset_
      vo.hdr.length_ = var_idx;   // index among the var columns
    }
  }
  if (!var_cols.empty()) out[(size_t)var_cols.back()].hdr.attr_ |= ATTR_LAST_VAR_FIELD;

  const uint32_t header_size = MICRO_HEADER_FIXED_SIZE;
  const size_t col_hdr_size = sizeof(ColumnHeader) * (size_t)ncol;
  const size_t meta_off = header_size + col_hdr_size;
  const size_t row_data_off = meta_off + meta.size();
  Buf rows;
  std::vector<uint64_t> row_index;
  if (!var_cols.empty()) {
    const size_t nv = var_cols.size();
    row_index.push_back(0);
    std::vector<int64_t> lens(nv);
    for (int64_t r = 0; r < nrows; ++r) {
      int64_t var_size = 0;
      int col_idx_byte = 0;
      for (size_t k = 0; k < nv; ++k) {
        const ColCtx &c = ctx[(size_t)var_cols[k]];
        const int vis = out[(size_t)var_cols[k]].var_int_size;
        const ColOut &vo = out[(size_t)var_cols[k]];
        lens[k] = c.is_null(r) ? 0 : (vo.own_meta ? vo.cell_off[(size_t)r + 1] - vo.cell_off[(size_t)r] : (vis > 0 ? (int64_t)vis : c.sval(r).len));
        if (k > 0 && k == nv - 1) col_idx_byte = var_size <= 0xff ? 1 : (var_size <= 0xffff ? 2 : 4);
        var_size += lens[k];
      }
      const int64_t row_size = fix_data_size + var_size + (col_idx_byte > 0 ? 1 : 0) +
                               (int64_t)col_idx_byte * (int64_t)(nv - 1);
      uint8_t *data = rows.grow((size_t)row_size);
      uint8_t *var = data + fix_data_size;
      uint8_t *idx = nullptr;
      if (col_idx_byte > 0) {
        *var = (uint8_t)col_idx_byte;
        idx = var + 1;
        var += 1 + (size_t)col_idx_byte * (nv - 1);
      }
      int64_t off = 0;
      for (size_t k = 0; k < nv; ++k) {
        const ColCtx &c = ctx[(size_t)var_cols[k]];
        if (k > 0) {
          const uint64_t o = (uint64_t)off;
          memcpy(idx + (k - 1) * (size_t)col_idx_byte, &o, (size_t)col_idx_byte);
        }
        if (c.is_null(r)) {
          put_bits(data, out[(size_t)var_cols[k]].hdr.extend_value_index_, ext_bit, c.ext_val(r));
        } else if (out[(size_t)var_cols[k]].var_int_size > 0) {
          const uint64_t v = c.uval(r);   // low bytes of the datum (MEMCPY(buf, datum.ptr_, len))
          memcpy(var + off, &v, (size_t)std::min<int64_t>(lens[k], 8));
        } else if (out[(size_t)var_cols[k]].own_meta) {
          const ColOut &vo = out[(size_t)var_cols[k]];
          if (lens[k] > 0) memcpy(var + off, vo.cell_heap.data() + vo.cell_off[(size_t)r], (size_t)lens[k]);
        } else if (lens[k] > 0) {
          memcpy(var + off, c.sval(r).p, (size_t)lens[k]);
        }
        off += lens[k];
      }
      row_index.push_back((uint64_t)rows.size());
    }
  }
  int row_index_byte = 0;
  if (!var_cols.empty()) row_index_byte = row_index.back() > 0xffff ? 4 : 2;
  const size_t total = row_data_off + rows.size() + row_index.size() * (size_t)row_index_byte;
  block.assign(total, 0);
  uint8_t *b = block.data();
  for (int i = 0; i < ncol; ++i)
    memcpy(b + header_size + sizeof(ColumnHeader) * (size_t)i, &out[(size_t)i].hdr, sizeof(ColumnHeader));
  if (meta.size()) memcpy(b + meta_off, meta.d.data(), meta.size());
  if (rows.size()) memcpy(b + row_data_off, rows.d.data(), rows.size());
  for (size_t k = 0; k < row_index.size(); ++k)
    memcpy(b + row_data_off + rows.size() + k * (size_t)row_index_byte, &row_index[k], (size_t)row_index_byte);

  finish_header(block, header_size, ncol, rowkey_cnt, nrows, ENCODING_ROW_STORE,
                (uint8_t)((row_index_byte & 7) | ((ext_bit & 7) << 3)), (uint16_t)var_cols.size(), (uint32_t)row_data_off,
                original);
  return OBGPU_SUCCESS;
}

// ---- CS_ENCODING_ROW_STORE block (ObMicroBlockCSEncoder::build_block, cs_encoding/ob_micro_block_cs_encoder.cpp:1394):
//   [header][ObAllColumnHeader][ObCSColumnHeader x ncol][per column: meta (null bitmap) + integer streams]
//   [all string data (none here)][stream offsets = one more integer stream]
// Integer streams are written RAW (serialized ObIntegerStreamMeta + width-byte array); the width / base / null
// replacement rules follow ObIntegerColumnEncoder::build_signed_stream_meta_ / build_unsigned_encoder_ctx_
// (cs_encoding/ob_integer_column_encoder.cpp:177-287) and ObIntegerStreamEncoderCtx::build_*_stream_meta
// (ob_stream_encoding_struct.cpp:101-190). Stream end offsets are relative to the block start.
static void put_vi64(Buf &b, uint64_t v) {  // serialization::encode_vi64
  while (v > 0x7f) { *b.grow(1) = (uint8_t)(v | 0x80); v >>= 7; }
  *b.grow(1) = (uint8_t)(v & 0x7f);
}
static uint8_t width_tag(int bytes) { return bytes == 1 ? 0 : (bytes == 2 ? 1 : (bytes == 4 ? 2 : 3)); }

struct IntStreamPlan {
  int width = 1;
  bool use_base = false, replace_null = false;
  uint64_t base = 0, null_replaced = 0;
};
// Stream codec choice for the integer streams of CS blocks (obgpu_writer_set_cs_stream_encoding): 1 = RAW (default),
// 0 = detect per stream like ObIntegerStreamEncoder::choose_stream_codec, 2..8 = that ObIntegerStream::EncodingType
// wherever it is not larger than RAW. The stream-offsets stream stays RAW.
static std::atomic<int> g_cs_stream_mode{1};

static void put_stream_meta(Buf &b, const IntStreamPlan &sp, int type = IS_RAW) {
  uint8_t *p = b.grow(4);
  p[0] = INTEGER_STREAM_META_V2;
  p[1] = (uint8_t)((sp.use_base ? IS_USE_BASE : 0) | (sp.replace_null ? IS_REPLACE_NULL_VALUE : 0));
  p[2] = (uint8_t)type;
  p[3] = width_tag(sp.width);
  if (sp.use_base) put_vi64(b, sp.base);
  if (sp.replace_null) put_vi64(b, sp.null_replaced);
  *b.grow(1) = 1;  // pfor_packing_type_: CPU_ARCH_INDEPENDANT_SCALAR
}

// ObStringStreamMeta, serialized: version u8, attr u8 (USE_ZERO_LEN_AS_NULL 0x1, IS_FIXED_LEN_STRING 0x2),
// vi32 uncompressed_len, [vi32 fixed_str_len] (cs_encoding/ob_stream_encoding_struct.cpp:255-268)
static void put_string_stream_meta(Buf &b, bool zero_len_null, int64_t fixed_len, uint32_t uncompressed_len) {
  uint8_t *p = b.grow(2);
  p[0] = 0;
  p[1] = (uint8_t)((zero_len_null ? 0x1 : 0) | (fixed_len >= 0 ? 0x2 : 0));
  put_vi64(b, uncompressed_len);
  if (fixed_len >= 0) put_vi64(b, (uint64_t)fixed_len);
}
// One integer stream: serialized ObIntegerStreamMeta + the codec's bytes for `vals` (already minus the base).
// ObIntegerStreamEncoder::inner_encode (cs_encoding/ob_integer_stream_encoder.h:224-290): the chosen codec, RAW when
// its output is larger than the raw array.
static void emit_int_stream(Buf &body, const IntStreamPlan &sp, const std::vector<uint64_t> &vals, bool allow_codecs = true) {
  const int mode = allow_codecs ? g_cs_stream_mode.load(std::memory_order_relaxed) : 1;
  const uint32_t wb = (uint32_t)sp.width;
  int type = obstream::T_RAW;
  if (mode == 0) {
    bool mono = true;
    const uint64_t m = obstream::mask_of(wb);
    for (size_t k = 1; k < vals.size() && mono; ++k) mono = (vals[k] & m) >= (vals[k - 1] & m);
    type = obstream::detect(wb, vals.data(), vals.size(), mono);
  } else if (mode >= 2 && mode <= 8 && mode != obstream::T_UNIVERSAL) {
    type = mode;
  }
  std::vector<uint8_t> enc;
  if (type != obstream::T_RAW) {
    obstream::encode(type, wb, vals.data(), vals.size(), enc);
    if (enc.size() > vals.size() * (size_t)wb) type = obstream::T_RAW;
  }
  put_stream_meta(body, sp, type);
  if (type == obstream::T_RAW) {
    uint8_t *d = body.grow((size_t)wb * vals.size());
    for (size_t k = 0; k < vals.size(); ++k) memcpy(d + k * (size_t)wb, &vals[k], (size_t)wb);
  } else if (!enc.empty()) {
    memcpy(body.grow(enc.size()), enc.data(), enc.size());
  }
}
static void put_raw_stream(Buf &body, const std::vector<uint64_t> &vals, uint64_t max_value) {
  IntStreamPlan sp;
  sp.width = (int)byte_packed_int_size(max_value);
  emit_int_stream(body, sp, vals);
}

// ObStringColumnEncoder::do_init_ (cs_encoding/ob_string_column_encoder.cpp:59-139) decides fixed length / NULL
// bitmap / zero-length-as-NULL; the bytes go to the block's all-string-data area, the column keeps the
// serialized string stream meta and, for variable length, one END offset per row.
static int cs_string_column(const ColCtx &c, CSColumnHeader &ch, Buf &body, Buf &all_string, std::vector<uint32_t> &stream_end,
                            uint32_t header_size) {
  const int64_t n = c.nrows;
  ch.type_ = CS_STRING;
  bool has_zero = false;
  int64_t fix = -1, var_size = 0;
  bool var = false;
  for (int64_t r = 0; r < n; ++r) {
    if (c.is_null(r)) continue;
    const int64_t l = c.sval(r).len;
    var_size += l;
    has_zero = has_zero || l == 0;
    if (fix < 0 && !var) fix = l;
    else if (fix != l) { var = true; fix = -1; }
  }
  if (var) fix = -1;
  bool bitmap = false, zero_null = false;
  int64_t fixed_len = -1;
  if (c.null_cnt > 0) {
    if (has_zero) {
      bitmap = true;
      if (fix >= 0) fixed_len = fix;
    } else if (fix >= 0) {
      const int64_t pad = fix * c.null_cnt, bm = (n + 7) / 8;
      const int64_t off_arr = n * byte_packed_int_size((uint64_t)var_size);
      if (pad + bm < off_arr) { fixed_len = fix; bitmap = true; }
      else zero_null = true;
    } else {
      zero_null = true;
    }
  } else if (fix >= 0) {
    fixed_len = fix;
  }
  if (fixed_len >= 0) ch.attrs_ |= CS_IS_FIXED_LENGTH;
  if (bitmap) {
    ch.attrs_ |= CS_HAS_NULL_OR_NOP_BITMAP;
    uint8_t *bmp = body.grow((size_t)((n + 7) / 8));
    memset(bmp, 0, (size_t)((n + 7) / 8));
    for (int64_t r = 0; r < n; ++r)
      if (c.is_null(r)) bmp[r / 8] |= (uint8_t)(1u << (7 - r % 8));
  }
  const uint64_t total = fixed_len >= 0 ? (uint64_t)fixed_len * (uint64_t)n : (uint64_t)var_size;
  if (total > 0xffffffffull) return OBGPU_NOT_SUPPORTED;
  put_string_stream_meta(body, zero_null, fixed_len, (uint32_t)total);
  stream_end.push_back(header_size + (uint32_t)body.size());
  std::vector<uint64_t> ends;
  uint64_t pos = 0;
  uint8_t *dst = all_string.grow((size_t)total);
  for (int64_t r = 0; r < n; ++r) {
    if (c.is_null(r)) {
      if (fixed_len >= 0) { memset(dst + pos, 0, (size_t)fixed_len); pos += (uint64_t)fixed_len; }
    } else {
      const StrRef v = c.sval(r);
      memcpy(dst + pos, v.p, (size_t)v.len);
      pos += (uint64_t)v.len;
    }
    if (fixed_len < 0) ends.push_back(pos);
  }
  if (fixed_len < 0) {
    put_raw_stream(body, ends, total);
    stream_end.push_back(header_size + (uint32_t)body.size());
  }
  return OBGPU_SUCCESS;
}

// Ref stream of a CS dictionary column (ObDictColumnEncoder::try_const_encoding_ref_ / do_store_dict_ref_,
// cs_encoding/ob_dict_column_encoder.cpp:144-189, .h:65-116): when one ref (a value or NULL) covers all rows, or
// all but <= 64 rows and fewer than 10 % of them, the stream holds [exception count][const ref][exception row
// ids][exception refs] and the dict meta says CONST_ENCODING_REF with ref_row_cnt_ = 2 + 2 * exceptions.
static void put_dict_ref_stream(Buf &body, size_t dm_at, const std::vector<uint64_t> &refs, uint64_t distinct, bool has_null) {
  const int64_t n = (int64_t)refs.size();
  const uint64_t max_ref = has_null ? distinct : distinct - 1;
  std::vector<int64_t> freq((size_t)distinct + 1, 0);
  for (uint64_t r : refs) ++freq[(size_t)r];
  uint64_t const_ref = 0;
  int64_t max_cnt = 0;
  for (uint64_t k = 0; k < distinct; ++k)
    if (freq[(size_t)k] > max_cnt) { max_cnt = freq[(size_t)k]; const_ref = k; }
  if (freq[(size_t)distinct] > max_cnt) { max_cnt = freq[(size_t)distinct]; const_ref = distinct; }
  const int64_t exc = n - max_cnt;
  if (exc == 0 || (exc <= 64 && exc < n * 10 / 100)) {
    std::vector<uint64_t> st;
    st.push_back((uint64_t)exc);
    st.push_back(const_ref);
    uint64_t max_row = 0;
    for (int64_t r = 0; r < n; ++r) if (refs[(size_t)r] != const_ref) { st.push_back((uint64_t)r); max_row = (uint64_t)r; }
    for (int64_t r = 0; r < n; ++r) if (refs[(size_t)r] != const_ref) st.push_back(refs[(size_t)r]);
    DictEncodingMeta dm;
    memcpy(&dm, body.d.data() + dm_at, sizeof(dm));
    dm.attrs_ |= 0x4;
    dm.ref_row_cnt_ = (uint32_t)(2 + 2 * exc);
    memcpy(body.d.data() + dm_at, &dm, sizeof(dm));
    put_raw_stream(body, st, exc == 0 ? std::max<uint64_t>(0, const_ref) : std::max<uint64_t>(std::max<uint64_t>((uint64_t)exc, max_row), max_ref));
    return;
  }
  put_raw_stream(body, refs, max_ref);
}

// String dictionary column: [ObDictEncodingMeta][dict bytes: string stream (+ END offsets when variable)][refs];
// ref == distinct_val_cnt is NULL (cs_encoding/ob_dict_column_decoder.cpp:158-326).
static int cs_str_dict_column(const ColCtx &c, CSColumnHeader &ch, Buf &body, Buf &all_string, std::vector<uint32_t> &stream_end,
                              uint32_t header_size) {
  const int64_t n = c.nrows;
  ch.type_ = CS_STR_DICT;
  StrDict d;
  build_str_dict(c, true, d);
  DictEncodingMeta dm{};
  dm.attrs_ = (uint8_t)(0x1 | (c.null_cnt > 0 ? 0x2 : 0));
  dm.distinct_val_cnt_ = (uint32_t)d.values.size();
  dm.ref_row_cnt_ = (uint32_t)n;
  const size_t dm_at = body.size();
  memcpy(body.grow(sizeof(dm)), &dm, sizeof(dm));
  if (d.values.empty()) return OBGPU_SUCCESS;
  const bool fixed = d.fix_len >= 0;
  if (fixed) ch.attrs_ |= CS_IS_FIXED_LENGTH;
  const uint64_t total = (uint64_t)d.var_data_size;
  put_string_stream_meta(body, false, fixed ? d.fix_len : -1, (uint32_t)total);
  stream_end.push_back(header_size + (uint32_t)body.size());
  uint8_t *dst = all_string.grow((size_t)total);
  std::vector<uint64_t> ends;
  uint64_t pos = 0;
  for (const StrRef &v : d.values) {
    memcpy(dst + pos, v.p, (size_t)v.len);
    pos += (uint64_t)v.len;
    ends.push_back(pos);
  }
  if (!fixed) {
    put_raw_stream(body, ends, total);
    stream_end.push_back(header_size + (uint32_t)body.size());
  }
  std::vector<uint64_t> refs((size_t)n);
  for (int64_t r = 0; r < n; ++r) refs[(size_t)r] = d.refs[(size_t)r];
  put_dict_ref_stream(body, dm_at, refs, d.values.size(), c.null_cnt > 0);
  stream_end.push_back(header_size + (uint32_t)body.size());
  return OBGPU_SUCCESS;
}

// ---- CS encoder selection (OBGPU_ENC_CS_AUTO): ObMicroBlockCSEncoder::choose_encoder_for_integer_ / _for_string_
// (cs_encoding/ob_micro_block_cs_encoder.cpp:2289-2375, data version > 4.3.5.0): the dictionary form is used when its estimate is
// below 70 % of the plain one, or below it with fewer than rows / 2 distinct values. Estimates: ObIntegerColumnEncoder::
// estimate_store_size (ob_integer_column_encoder.cpp:296-314: bits(range) x rows / 8 + NULL bitmap when NULL cannot be replaced),
// ObIntDictColumnEncoder / ObStrDictColumnEncoder (ob_int_dict_column_encoder.cpp:262-279, ob_str_dict_column_encoder.cpp:170-196:
// meta + dictionary + bits(max ref stream value) x ref rows / 8, the const-encoded ref form of ob_dict_column_encoder.cpp:150-186
// included), ObStringColumnEncoder (ob_string_column_encoder.cpp:195-218).
static int64_t cs_bit_size(uint64_t v) { return v == 0 ? 1 : 64 - __builtin_clzll(v); }   // ObCSEncodingUtil::get_bit_size

int choose_cs_auto_encoding(const ColCtx &c) {
  const int64_t n = c.nrows;
  const bool is_int = c.sc == 1 || c.sc == 2;
  if (!is_int && c.sc != 5) return -1;
  // dictionary refs (first occurrence order is enough: only counts and frequencies matter)
  std::vector<uint32_t> refs;
  int64_t distinct = 0;
  int64_t dict_var = 0, var_all = 0, fix_len = -1;
  uint64_t dict_range = 0;
  if (is_int) {
    IntDict d;
    build_int_dict(c, false, d);
    refs.swap(d.refs);
    distinct = (int64_t)d.values.size();
    if (distinct > 0) {   // ObIntDictColumnEncoder: the dictionary is an integer stream over [min, max] with a base when negative
      const int ts = type_store_size((uint8_t)c.in->obj_type);
      const uint64_t rev = ~low_mask((uint32_t)ts * 8);
      if (c.sc == 1) {
        int64_t mn = INT64_MAX, mx = INT64_MIN;
        for (uint64_t v : d.values) { if (rev != 0 && (v & (rev >> 1))) v |= rev; mn = std::min(mn, (int64_t)v); mx = std::max(mx, (int64_t)v); }
        dict_range = mn < 0 ? (uint64_t)mx - (uint64_t)mn : (uint64_t)mx;
      } else {
        dict_range = d.max_integer;
      }
    }
  } else {
    StrDict d;
    build_str_dict(c, false, d);
    refs.swap(d.refs);
    distinct = (int64_t)d.values.size();
    bool var = false;
    for (const StrRef &v : d.values) {
      dict_var += v.len;
      if (!var) { if (fix_len < 0) fix_len = v.len; else if (fix_len != v.len) { fix_len = -1; var = true; } }
    }
    for (int64_t r = 0; r < n; ++r) if (!c.is_null(r)) var_all += c.sval(r).len;
  }
  const bool has_null = c.null_cnt > 0;
  // ---- the ref stream of the dictionary forms (ObDictColumnEncoder::try_const_encoding_ref_, ob_dict_column_encoder.cpp:150-186) ----
  int64_t ref_rows = n;
  uint64_t ref_max = has_null ? (uint64_t)distinct : (uint64_t)std::max<int64_t>(distinct - 1, 0);
  if (distinct > 0) {
    std::vector<int64_t> freq((size_t)distinct + 2, 0);
    for (uint32_t r : refs) ++freq[r];
    int64_t max_cnt = 0, const_ref = 0;
    for (int64_t k = 0; k < distinct; ++k) if (freq[(size_t)k] > max_cnt) { max_cnt = freq[(size_t)k]; const_ref = k; }
    if (freq[(size_t)distinct] > max_cnt) { max_cnt = freq[(size_t)distinct]; const_ref = distinct; }
    const int64_t exc = n - max_cnt;
    if (exc == 0) { ref_rows = 2; ref_max = (uint64_t)std::max<int64_t>(exc, const_ref); }
    else if (exc <= 64 && exc < n * 10 / 100) {
      int64_t max_row = 0;
      for (int64_t r = n - 1; r >= 0; --r) if ((int64_t)refs[(size_t)r] != const_ref) { max_row = r; break; }
      ref_rows = 2 + 2 * exc;
      ref_max = std::max<uint64_t>(std::max<uint64_t>((uint64_t)exc, (uint64_t)max_row), ref_max);
    }
  }
  const int64_t bitmap = (n + 7) / 8;
  if (is_int) {
    // ---- plain INTEGER: range after the NULL replacement rules (build_signed / unsigned_encoder_ctx_, ob_integer_column_encoder.cpp:177-287)
    const int ts = type_store_size((uint8_t)c.in->obj_type);
    const uint64_t mask = low_mask((uint32_t)ts * 8);
    bool any = false, need_bitmap = false;
    int64_t smin = 0, smax = 0;
    uint64_t umin = 0, umax = 0;
    for (int64_t r = 0; r < n; ++r) {
      if (c.is_null(r)) continue;
      const int64_t sv = c.ival(r);
      const uint64_t uv = (uint64_t)sv & mask;
      if (!any) { smin = smax = sv; umin = umax = uv; any = true; }
      else { smin = std::min(smin, sv); smax = std::max(smax, sv); umin = std::min(umin, uv); umax = std::max(umax, uv); }
    }
    uint64_t range;
    if (c.sc == 1) {
      const uint64_t rmask = ~mask;
      const int64_t type_min = rmask == 0 ? INT64_MIN : (int64_t)(rmask | (rmask >> 1)), type_max = (int64_t)(mask >> 1);
      int64_t nmin = smin, nmax = smax;
      if (has_null) {
        if (!any) nmin = nmax = 0;
        if (nmin == 0) { if (nmax != type_max) nmax += 1; else nmin = -1; }
        else if (nmin == type_min) { if (nmax != type_max) nmax += 1; else need_bitmap = true; }
        else nmin -= 1;
      }
      range = nmin < 0 ? (uint64_t)nmax - (uint64_t)nmin : (uint64_t)nmax;
    } else {
      uint64_t nmin = umin, nmax = umax;
      if (has_null) {
        if (!any) nmin = nmax = 0;
        if (nmin == 0) { if (nmax != mask) nmax += 1; else need_bitmap = true; }
        else nmin -= 1;
      }
      (void)nmin;
      range = nmax;
    }
    const int64_t int_est = cs_bit_size(range) * n / 8 + (need_bitmap ? bitmap : 0);
    int64_t dict_est = (int64_t)sizeof(DictEncodingMeta);
    if (distinct > 0) dict_est += cs_bit_size(dict_range) * distinct / 8 + cs_bit_size(ref_max) * ref_rows / 8;
    const bool use_dict = dict_est < int_est * 70 / 100 || (dict_est < int_est && distinct < n * 50 / 100);
    return use_dict ? OBGPU_ENC_CS_INT_DICT : OBGPU_ENC_CS_INTEGER;
  }
  int64_t str_est;
  if (fix_len >= 0 && distinct > 0) str_est = fix_len * n;
  else str_est = var_all + cs_bit_size((uint64_t)(n > 0 ? var_all / n : 0)) * n / 8;
  if (has_null) str_est += bitmap;
  int64_t dict_est = (int64_t)sizeof(DictEncodingMeta);
  if (distinct > 0) {
    if (fix_len >= 0) dict_est += fix_len * distinct;
    else dict_est += dict_var + cs_bit_size((uint64_t)(dict_var / distinct)) * distinct / 8;
    dict_est += cs_bit_size(ref_max) * ref_rows / 8;
  }
  const bool use_dict = dict_est < str_est * 70 / 100 || (dict_est < str_est && distinct < n * 50 / 100);
  return use_dict ? OBGPU_ENC_CS_STR_DICT : OBGPU_ENC_CS_STRING;
}

int BlockBuilder::build_cs(std::vector<uint8_t> &block, int64_t original) {
  // OBGPU_ENC_CS_AUTO columns are resolved first; the rest of the function sees concrete column types
  std::vector<obgpu_col_input> resolved;
  for (int i = 0; i < ncol; ++i) {
    if (cols[i].encoding != OBGPU_ENC_CS_AUTO) continue;
    if (resolved.empty()) resolved.assign(cols, cols + ncol);
    const int enc = choose_cs_auto_encoding(ctx[(size_t)i]);
    if (enc < 0) return OBGPU_NOT_SUPPORTED;
    resolved[(size_t)i].encoding = enc;
  }
  if (!resolved.empty()) {
    const obgpu_col_input *saved = cols;
    cols = resolved.data();
    for (int i = 0; i < ncol; ++i) ctx[(size_t)i].in = &cols[i];
    const int ret = build_cs(block, original);
    cols = saved;
    for (int i = 0; i < ncol; ++i) ctx[(size_t)i].in = &cols[i];
    return ret;
  }
  const uint32_t header_size = (uint32_t)sizeof(MicroBlockHeader);
  Buf body;  // everything after the micro header
  body.grow(sizeof(AllColumnHeader) + sizeof(CSColumnHeader) * (size_t)ncol);
  std::vector<CSColumnHeader> chdr((size_t)ncol);
  std::vector<uint32_t> stream_end;  // relative to the block start
  Buf all_string;                    // bytes of every string stream, in stream order (store_all_string_data_)
  const size_t bitmap_bytes = (size_t)((nrows + 7) / 8);
  for (int i = 0; i < ncol; ++i) {
    ColCtx &c = ctx[(size_t)i];
    CSColumnHeader &ch = chdr[(size_t)i];
    ch = CSColumnHeader{};
    ch.obj_type_ = (uint8_t)cols[i].obj_type;
    if (c.nope_cnt > 0) return OBGPU_NOT_SUPPORTED;
    if (cols[i].encoding == OBGPU_ENC_CS_STRING || cols[i].encoding == OBGPU_ENC_CS_STR_DICT) {
      if (c.sc != 5) return OBGPU_NOT_SUPPORTED;
      const int ret = cols[i].encoding == OBGPU_ENC_CS_STRING ? cs_string_column(c, ch, body, all_string, stream_end, header_size)
                                                              : cs_str_dict_column(c, ch, body, all_string, stream_end, header_size);
      if (ret != OBGPU_SUCCESS) return ret;
      continue;
    }
    if ((cols[i].encoding != OBGPU_ENC_CS_INTEGER && cols[i].encoding != OBGPU_ENC_CS_INT_DICT) || (c.sc != 1 && c.sc != 2))
      return OBGPU_NOT_SUPPORTED;
    if (cols[i].encoding == OBGPU_ENC_CS_INT_DICT) {
      // ObIntDictColumnEncoder: [ObDictEncodingMeta][dict values: integer stream][refs: integer stream];
      // ref == distinct_val_cnt is NULL; an all-NULL column has the meta only (no streams)
      ch.type_ = CS_INT_DICT;
      const int ts = type_store_size((uint8_t)cols[i].obj_type);
      const uint64_t mask = low_mask(ts * 8);
      const bool sgn = c.sc == 1;
      std::vector<int64_t> vals;
      vals.reserve((size_t)nrows);
      for (int64_t r = 0; r < nrows; ++r)
        if (!c.is_null(r)) vals.push_back(sgn ? c.ival(r) : (int64_t)((uint64_t)c.ival(r) & mask));
      if (sgn) std::sort(vals.begin(), vals.end());
      else std::sort(vals.begin(), vals.end(), [](int64_t a, int64_t b) { return (uint64_t)a < (uint64_t)b; });
      vals.erase(std::unique(vals.begin(), vals.end()), vals.end());
      DictEncodingMeta dm{};
      dm.attrs_ = (uint8_t)(0x1 | (c.null_cnt > 0 ? 0x2 : 0));  // IS_SORTED | HAS_NULL
      dm.distinct_val_cnt_ = (uint32_t)vals.size();
      dm.ref_row_cnt_ = (uint32_t)nrows;
      const size_t dm_at = body.size();
      memcpy(body.grow(sizeof(dm)), &dm, sizeof(dm));
      if (vals.empty()) continue;
      IntStreamPlan dp;
      if (sgn && vals.front() < 0) {
        dp.use_base = true;
        dp.base = (uint64_t)vals.front();
        dp.width = (int)byte_packed_int_size((uint64_t)vals.back() - (uint64_t)vals.front());
      } else {
        dp.width = (int)byte_packed_int_size((uint64_t)vals.back());
      }
      {
        std::vector<uint64_t> dv(vals.size());
        for (size_t k = 0; k < vals.size(); ++k) dv[k] = (uint64_t)vals[k] - dp.base;
        emit_int_stream(body, dp, dv);
      }
      stream_end.push_back(header_size + (uint32_t)body.size());
      std::vector<uint64_t> refs((size_t)nrows);
      for (int64_t r = 0; r < nrows; ++r) {
        uint64_t ref;
        if (c.is_null(r)) ref = vals.size();
        else {
          const int64_t v = sgn ? c.ival(r) : (int64_t)((uint64_t)c.ival(r) & mask);
          ref = sgn ? (uint64_t)(std::lower_bound(vals.begin(), vals.end(), v) - vals.begin())
                    : (uint64_t)(std::lower_bound(vals.begin(), vals.end(), v,
                                                  [](int64_t a, int64_t b) { return (uint64_t)a < (uint64_t)b; }) - vals.begin());
        }
        refs[(size_t)r] = ref;
      }
      put_dict_ref_stream(body, dm_at, refs, vals.size(), c.null_cnt > 0);
      stream_end.push_back(header_size + (uint32_t)body.size());
      continue;
    }
    ch.type_ = CS_INTEGER;
    const int ts = type_store_size((uint8_t)cols[i].obj_type);
    const uint64_t mask = low_mask(ts * 8);
    const bool sgn = c.sc == 1;
    // value range over the non-null cells, in the column's own domain
    bool any = false;
    int64_t smin = 0, smax = 0;
    uint64_t umin = 0, umax = 0;
    for (int64_t r = 0; r < nrows; ++r) {
      if (c.is_null(r)) continue;
      const int64_t sv = c.ival(r);
      const uint64_t uv = (uint64_t)sv & mask;
      if (!any) { smin = smax = sv; umin = umax = uv; any = true; }
      else { smin = std::min(smin, sv); smax = std::max(smax, sv); umin = std::min(umin, uv); umax = std::max(umax, uv); }
    }
    IntStreamPlan sp;
    bool bitmap = false;
    if (sgn) {
      const uint64_t rmask = ~mask;
      const int64_t type_min = rmask == 0 ? INT64_MIN : (int64_t)(rmask | (rmask >> 1));
      const int64_t type_max = (int64_t)(mask >> 1);
      int64_t nmin = smin, nmax = smax;
      if (c.null_cnt > 0) {
        if (!any) { nmin = nmax = 0; }
        if (nmin == 0) {
          if (nmax != type_max) { nmax = nmax + 1; sp.replace_null = true; sp.null_replaced = (uint64_t)nmax; }
          else { nmin = -1; sp.replace_null = true; sp.null_replaced = (uint64_t)nmin; }
        } else if (nmin == type_min) {
          if (nmax != type_max) { nmax = nmax + 1; sp.replace_null = true; sp.null_replaced = (uint64_t)nmax; }
          else bitmap = true;
        } else {
          nmin = nmin - 1; sp.replace_null = true; sp.null_replaced = (uint64_t)nmin;
        }
      }
      if (nmin < 0) {
        sp.use_base = true;
        sp.base = (uint64_t)nmin;
        sp.width = (int)byte_packed_int_size((uint64_t)nmax - (uint64_t)nmin);
      } else {
        sp.width = (int)byte_packed_int_size((uint64_t)nmax);
      }
    } else {
      uint64_t nmin = umin, nmax = umax;
      if (c.null_cnt > 0) {
        if (!any) { nmin = nmax = 0; }
        if (nmin == 0) {
          if (nmax != mask) { nmax = nmax + 1; sp.replace_null = true; sp.null_replaced = nmax; }
          else bitmap = true;
        } else {
          nmin = nmin - 1; sp.replace_null = true; sp.null_replaced = nmin;
        }
      }
      sp.width = (int)byte_packed_int_size(nmax);
    }
    if (bitmap) {
      ch.attrs_ |= CS_HAS_NULL_OR_NOP_BITMAP;
      uint8_t *bm = body.grow(bitmap_bytes);
      memset(bm, 0, bitmap_bytes);
      for (int64_t r = 0; r < nrows; ++r)
        if (c.is_null(r)) bm[r / 8] |= (uint8_t)(1u << (7 - r % 8));  // MSB first (ob_icolumn_cs_encoder.cpp:100-123)
    }
    {
      std::vector<uint64_t> cv((size_t)nrows);
      for (int64_t r = 0; r < nrows; ++r) {
        if (c.is_null(r)) cv[(size_t)r] = sp.replace_null ? sp.null_replaced - sp.base : 0;
        else cv[(size_t)r] = (sgn ? (uint64_t)c.ival(r) : ((uint64_t)c.ival(r) & mask)) - sp.base;
      }
      emit_int_stream(body, sp, cv);
    }
    stream_end.push_back(header_size + (uint32_t)body.size());
  }
  // all string data (uncompressed: compressor none), then the stream offsets: an integer stream without base
  // (ObMicroBlockCSEncoder::store_all_string_data_ :1254-1309, store_stream_offsets_ :1312-1372)
  if (all_string.size()) memcpy(body.grow(all_string.size()), all_string.d.data(), all_string.size());
  const size_t offsets_at = body.size();
  if (!stream_end.empty()) {
    IntStreamPlan sp;
    sp.width = (int)byte_packed_int_size(stream_end.back());
    if (sp.width > 4) return OBGPU_NOT_SUPPORTED;
    put_stream_meta(body, sp);
    uint8_t *data = body.grow((size_t)sp.width * stream_end.size());
    for (size_t k = 0; k < stream_end.size(); ++k) memcpy(data + k * (size_t)sp.width, &stream_end[k], (size_t)sp.width);
  }
  AllColumnHeader ah{};
  ah.all_string_data_length_ = (uint32_t)all_string.size();
  ah.stream_offsets_length_ = (uint32_t)(body.size() - offsets_at);
  ah.stream_count_ = (uint16_t)stream_end.size();
  memcpy(body.d.data(), &ah, sizeof(ah));
  memcpy(body.d.data() + sizeof(ah), chdr.data(), sizeof(CSColumnHeader) * (size_t)ncol);
  block.assign(header_size + body.size(), 0);
  memcpy(block.data() + header_size, body.d.data(), body.size());
  // opt_: single_version_rows_ etc. = 0; opt2_: compressor_type_ = NONE, has_row_header_ = 0
  finish_header(block, header_size, ncol, rowkey_cnt, nrows, CS_ENCODING_ROW_STORE, 0, (uint16_t)OBGPU_COMPRESSOR_NONE, 0, original);
  return OBGPU_SUCCESS;
}

int encode_one(const obgpu_col_input *cols, int32_t ncol, int32_t rowkey_cnt, int64_t row_begin,
               int64_t nrows, std::vector<uint8_t> &block) {
  BlockBuilder bb;
  bb.cols = cols;
  bb.ncol = ncol;
  bb.rowkey_cnt = rowkey_cnt;
  bb.row_begin = row_begin;
  bb.nrows = nrows;
  return bb.build(block);
}


// ---- skip index: aggregate row (ObAggRowWriter, index_block/ob_agg_row_struct.cpp:49-300) ------------------
// [ObAggRowHeader 8 B][col idx x cnt][cell offset x cnt] then one cell per aggregated column:
// [type bitmap 1 B][prefix bitmap 1 B (version >= 2)][data offsets x (stored + 1)][data ...], offsets relative to
// the cell start, the last one being the cell end; a column without a stored aggregate has the bitmaps only.
struct AggCellIn {
  uint32_t col_idx;
  uint8_t col_type, is_null, is_prefix;
  std::string data;
};

void put_le(uint8_t *p, uint64_t v, int bytes) { memcpy(p, &v, (size_t)bytes); }

int write_agg_row(std::vector<AggCellIn> cells, int version, std::vector<uint8_t> &out) {
  if (cells.empty() || version < 1 || version > 3) return OBGPU_INVALID_ARGUMENT;
  for (const AggCellIn &c : cells)
    if (c.col_type >= OBGPU_SK_IDX_MAX_COL_TYPE || c.col_idx >= (1u << 24)) return OBGPU_INVALID_ARGUMENT;
  std::stable_sort(cells.begin(), cells.end(), [](const AggCellIn &a, const AggCellIn &b) {
    return a.col_idx != b.col_idx ? a.col_idx < b.col_idx : a.col_type < b.col_type;
  });
  const bool store_prefix = version >= 2;
  const int bitmaps = store_prefix ? 2 : 1;
  int idx_size = 0;
  for (uint32_t m = cells.back().col_idx;;) { ++idx_size; m >>= 8; if (m == 0) break; }
  int cell_off_size = 1, idx_off_size = 1;
  int64_t col_cnt = 0, data_size = 0, stored_total = 0;
  const size_t n = cells.size();
  for (size_t i = 0; i < n;) {
    size_t e = i;
    int64_t cell_size = 0, nop = 0;
    while (e < n && cells[e].col_idx == cells[i].col_idx) {
      if (cells[e].is_null) ++nop; else cell_size += (int64_t)cells[e].data.size();
      ++e;
    }
    cell_size += bitmaps;
    int64_t stored = (int64_t)(e - i) - nop;
    if (stored > 0) ++stored;  // one more offset for the cell end
    if (cell_off_size == 1 && cell_size + stored > UINT8_MAX) cell_off_size = 2;
    ++col_cnt;
    data_size += cell_size;
    stored_total += stored;
    i = e;
  }
  data_size += stored_total * cell_off_size;
  int64_t header_size = (int64_t)sizeof(AggRowHeader) + col_cnt * idx_size + col_cnt * idx_off_size;
  if (data_size + header_size > UINT8_MAX) {
    idx_off_size = 2;
    header_size = (int64_t)sizeof(AggRowHeader) + col_cnt * idx_size + col_cnt * idx_off_size;
    if (data_size + header_size > UINT16_MAX) return OBGPU_NOT_SUPPORTED;
  }
  AggRowHeader h{};
  h.version_ = (int16_t)version;
  h.length_ = (int16_t)(data_size + header_size);
  h.agg_col_cnt_ = (int16_t)col_cnt;
  h.pack_ = (uint16_t)(idx_size | (idx_off_size << 6) | (cell_off_size << 9) | (1 << 12));
  out.assign((size_t)(data_size + header_size), 0);
  uint8_t *buf = out.data();
  memcpy(buf, &h, sizeof(h));
  uint8_t *idx_arr = buf + sizeof(h), *idx_off_arr = idx_arr + col_cnt * idx_size;
  int64_t pos = header_size, k = 0;
  for (size_t i = 0; i < n; ++k) {
    size_t e = i;
    int64_t nop = 0;
    while (e < n && cells[e].col_idx == cells[i].col_idx) { nop += cells[e].is_null ? 1 : 0; ++e; }
    put_le(idx_arr + k * idx_size, cells[i].col_idx, idx_size);
    put_le(idx_off_arr + k * idx_off_size, (uint64_t)pos, idx_off_size);
    const int64_t cell = pos;
    uint8_t *bm = buf + pos;
    pos += bitmaps;
    int64_t stored = (int64_t)(e - i) - nop;
    if (stored > 0) ++stored;
    uint8_t *offs = buf + pos;
    pos += stored * cell_off_size;
    int64_t w = 0;
    for (size_t j = i; j < e; ++j) {
      const AggCellIn &c = cells[j];
      if (c.is_null) continue;
      bm[0] |= (uint8_t)(1u << c.col_type);
      if (store_prefix && c.is_prefix && (c.col_type == OBGPU_SK_IDX_MIN || c.col_type == OBGPU_SK_IDX_MAX))
        bm[1] |= (uint8_t)(1u << c.col_type);
      put_le(offs + w * cell_off_size, (uint64_t)(pos - cell), cell_off_size);
      memcpy(buf + pos, c.data.data(), c.data.size());
      pos += (int64_t)c.data.size();
      ++w;
    }
    if (stored > 0) put_le(offs + (stored - 1) * cell_off_size, (uint64_t)(pos - cell), cell_off_size);
    i = e;
  }
  return pos == (int64_t)out.size() ? OBGPU_SUCCESS : OBGPU_ERR_UNEXPECTED;
}

// MIN / MAX / NULL_COUNT of one column over a row range (ObColMinAggregator / ObColMaxAggregator /
// ObColNullCountAggregator, ob_index_block_aggregator.cpp): a NOP cell makes the column "not aggregated";
// integer classes compare on the datum image (obagg::image / obagg::key), strings bytewise (binary collation), a string
// longer than 40 bytes is kept as a 40-byte prefix with the prefix flag. img[0..1] hold the integer min / max images
// the result points at.
obagg::AggCol aggregate_column(const obgpu_col_input &in, uint32_t col_idx, int64_t row_begin, int64_t nrows, int64_t img[2]) {
  const int sc = store_class_of((uint8_t)in.obj_type);
  int64_t null_cnt = 0;
  bool any = false, nop = false;
  obagg::AggCol a{col_idx, -1, -1, nullptr, nullptr, 0, 0, 0, 0};
  if (sc == 5) {
    StrRef lo{nullptr, 0}, hi{nullptr, 0};
    for (int64_t r = row_begin; r < row_begin + nrows; ++r) {
      if (in.is_null && in.is_null[r]) { nop = nop || in.is_null[r] == 2; ++null_cnt; continue; }
      const StrRef v{in.str_heap + in.str_off[r], in.str_off[r + 1] - in.str_off[r]};
      if (!any || str_cmp(v, lo) < 0) lo = v;
      if (!any || str_cmp(v, hi) > 0) hi = v;
      any = true;
    }
    if (any) {
      const int64_t cap = OBGPU_SKIP_INDEX_MAX_COL_LENGTH;
      a.min = (const uint8_t *)lo.p;
      a.max = (const uint8_t *)hi.p;
      a.min_len = (int32_t)std::min(lo.len, cap);
      a.max_len = (int32_t)std::min(hi.len, cap);
      a.min_prefix = lo.len > cap;
      a.max_prefix = hi.len > cap;
    }
  } else {
    const int dl = datum_len_of((uint8_t)in.obj_type);
    const bool uns = obagg::unsigned_order(sc, dl);
    int64_t lo = 0, hi = 0;
    for (int64_t r = row_begin; r < row_begin + nrows; ++r) {
      if (in.is_null && in.is_null[r]) { nop = nop || in.is_null[r] == 2; ++null_cnt; continue; }
      const int64_t v = obagg::key(obagg::image(in.i64[r], sc, dl), uns);
      if (!any || v < lo) lo = v;
      if (!any || hi < v) hi = v;
      any = true;
    }
    if (any) {
      img[0] = obagg::key(lo, uns);   // key() is its own inverse
      img[1] = obagg::key(hi, uns);
      a.min = (const uint8_t *)&img[0];
      a.max = (const uint8_t *)&img[1];
      a.min_len = a.max_len = dl;
    }
  }
  if (nop) {
    a.min_len = a.max_len = -1;
  } else {
    a.has_null_count = 1;
    a.null_count = null_cnt;
  }
  return a;
}

int block_agg_row(const obgpu_col_input *cols, int32_t n_cols, const int32_t *agg_cols, int32_t n_agg_cols,
                  int64_t row_begin, int64_t nrows, std::vector<uint8_t> &out) {
  std::vector<obagg::AggCol> aggs((size_t)n_agg_cols);
  std::vector<int64_t> images(2 * (size_t)n_agg_cols);
  for (int32_t k = 0; k < n_agg_cols; ++k) {
    const int32_t c = agg_cols[k];
    if (c < 0 || c >= n_cols) return OBGPU_INVALID_ARGUMENT;
    const int sc = store_class_of((uint8_t)cols[c].obj_type);
    if (sc == 5 ? (!cols[c].str_off || !cols[c].str_heap) : !cols[c].i64) return OBGPU_INVALID_ARGUMENT;
    if (sc != 1 && sc != 2 && sc != 5) return OBGPU_NOT_SUPPORTED;
    aggs[(size_t)k] = aggregate_column(cols[c], (uint32_t)c, row_begin, nrows, &images[2 * (size_t)k]);
  }
  std::vector<int32_t> order((size_t)n_agg_cols);
  for (int32_t k = 0; k < n_agg_cols; ++k) order[(size_t)k] = k;
  std::stable_sort(order.begin(), order.end(), [&](int32_t x, int32_t y) { return aggs[(size_t)x].col_idx < aggs[(size_t)y].col_idx; });
  if (aggs[(size_t)order.back()].col_idx >= (1u << 24)) return OBGPU_INVALID_ARGUMENT;
  bool repeats = false;
  for (size_t k = 1; k < order.size(); ++k) repeats = repeats || aggs[(size_t)order[k]].col_idx == aggs[(size_t)order[k - 1]].col_idx;
  if (repeats) {   // a column named twice: its cells merge into one cell of six aggregates, which only the general path writes
    std::vector<AggCellIn> cells;
    for (const obagg::AggCol &a : aggs) {
      const bool mm = a.min_len >= 0;
      cells.push_back({a.col_idx, OBGPU_SK_IDX_MIN, !mm, a.min_prefix, mm ? std::string((const char *)a.min, (size_t)a.min_len) : ""});
      cells.push_back({a.col_idx, OBGPU_SK_IDX_MAX, !mm, a.max_prefix, mm ? std::string((const char *)a.max, (size_t)a.max_len) : ""});
      cells.push_back({a.col_idx, OBGPU_SK_IDX_NULL_COUNT, !a.has_null_count, 0,
                       a.has_null_count ? std::string((const char *)&a.null_count, 8) : ""});
    }
    return write_agg_row(std::move(cells), obagg::kVersion, out);
  }
  auto col_at = [&](int k) -> const obagg::AggCol & { return aggs[(size_t)order[(size_t)k]]; };
  obagg::Layout l;
  if (obagg::layout(n_agg_cols, col_at, l) < 0) return OBGPU_NOT_SUPPORTED;
  out.resize((size_t)l.size);
  obagg::write(n_agg_cols, col_at, l, out.data());
  return OBGPU_SUCCESS;
}

}  // namespace

extern "C" {

int64_t obgpu_writer_block_bound(const obgpu_col_input *cols, int32_t n_cols, int64_t row_begin,
                                 int64_t nrows) {
  if (!cols || n_cols <= 0 || nrows <= 0) return -1;
  int64_t b = 64 + 16 * (int64_t)n_cols + 64;
  for (int i = 0; i < n_cols; ++i) {
    if (store_class_of((uint8_t)cols[i].obj_type) == 5) {
      if (!cols[i].str_off) return -1;
      const int64_t bytes = cols[i].str_off[row_begin + nrows] - cols[i].str_off[row_begin];
      b += 2 * bytes + nrows * 16 + 64;
    } else {
      b += nrows * 21 + 64;
    }
  }
  return b;
}

int obgpu_writer_encode_block(const obgpu_col_input *cols, int32_t n_cols, int32_t rowkey_col_cnt,
                              int64_t row_begin, int64_t nrows, void *out, int64_t out_cap,
                              int64_t *out_size) {
  if (!cols || !out_size) return OBGPU_INVALID_ARGUMENT;
  std::vector<uint8_t> block;
  const int ret = encode_one(cols, n_cols, rowkey_col_cnt, row_begin, nrows, block);
  if (ret != OBGPU_SUCCESS) return ret;
  *out_size = (int64_t)block.size();
  if (!out) return OBGPU_SUCCESS;
  if ((int64_t)block.size() > out_cap) return OBGPU_BUF_NOT_ENOUGH;
  memcpy(out, block.data(), block.size());
  return OBGPU_SUCCESS;
}

struct obgpu_table_image {
  std::vector<std::vector<uint8_t>> blocks;
  std::vector<int64_t> offs;
  int64_t image_size = 0;
  int32_t align = 16;
  int nt = 1;
};

int obgpu_writer_encode_table(const obgpu_col_input *cols, int32_t n_cols, int32_t rowkey_col_cnt,
                              int64_t total_rows, int64_t rows_per_block, int32_t align,
                              int32_t n_threads, obgpu_table_image **out) {
  if (!cols || total_rows <= 0 || rows_per_block <= 0 || !out) return OBGPU_INVALID_ARGUMENT;
  if (align < 16 || (align & (align - 1)) != 0) return OBGPU_INVALID_ARGUMENT;
  const int64_t nb64 = (total_rows + rows_per_block - 1) / rows_per_block;
  if (nb64 > INT32_MAX) return OBGPU_SIZE_OVERFLOW;
  const int32_t nb = (int32_t)nb64;
  obgpu_table_image *img = new (std::nothrow) obgpu_table_image();
  if (!img) return OBGPU_ALLOCATE_MEMORY_FAILED;
  img->blocks.resize((size_t)nb);
  int nt = n_threads > 0 ? n_threads : (int)std::thread::hardware_concurrency();
  nt = std::max(1, std::min(nt, nb));
  img->nt = nt;
  img->align = align;
  std::atomic<int32_t> next{0};
  std::atomic<int> err{OBGPU_SUCCESS};
  auto work = [&]() {
    for (;;) {
      const int32_t b = next.fetch_add(1);
      if (b >= nb || err.load() != OBGPU_SUCCESS) break;
      const int64_t rb = (int64_t)b * rows_per_block;
      const int64_t n = std::min(rows_per_block, total_rows - rb);
      const int r = encode_one(cols, n_cols, rowkey_col_cnt, rb, n, img->blocks[(size_t)b]);
      if (r != OBGPU_SUCCESS) err.store(r);
    }
  };
  std::vector<std::thread> th;
  for (int t = 1; t < nt; ++t) th.emplace_back(work);
  work();
  for (auto &t : th) t.join();
  if (err.load() != OBGPU_SUCCESS) {
    delete img;
    return err.load();
  }
  int64_t pos = 0;
  img->offs.resize((size_t)nb);
  for (int32_t b = 0; b < nb; ++b) {
    img->offs[(size_t)b] = pos;
    pos += ((int64_t)img->blocks[(size_t)b].size() + align - 1) / align * align;
  }
  img->image_size = pos;
  *out = img;
  return OBGPU_SUCCESS;
}

int obgpu_table_image_info(const obgpu_table_image *img, int64_t *image_size, int32_t *n_blocks) {
  if (!img) return OBGPU_INVALID_ARGUMENT;
  if (image_size) *image_size = img->image_size;
  if (n_blocks) *n_blocks = (int32_t)img->blocks.size();
  return OBGPU_SUCCESS;
}

int obgpu_table_image_export(const obgpu_table_image *img, void *image, int64_t image_cap,
                             int64_t *offsets, int64_t *sizes, int32_t tables_cap) {
  if (!img || !image || !offsets || !sizes) return OBGPU_INVALID_ARGUMENT;
  const int32_t nb = (int32_t)img->blocks.size();
  if (image_cap < img->image_size || tables_cap < nb) return OBGPU_BUF_NOT_ENOUGH;
  const size_t align = (size_t)img->align;
  std::atomic<int32_t> nx{0};
  auto copy = [&]() {
    for (;;) {
      const int32_t b = nx.fetch_add(1);
      if (b >= nb) break;
      uint8_t *dst = (uint8_t *)image + img->offs[(size_t)b];
      const size_t sz = img->blocks[(size_t)b].size();
      memcpy(dst, img->blocks[(size_t)b].data(), sz);
      const size_t padded = (sz + align - 1) / align * align;
      if (padded > sz) memset(dst + sz, 0, padded - sz);
      offsets[b] = img->offs[(size_t)b];
      sizes[b] = (int64_t)sz;
    }
  };
  std::vector<std::thread> th2;
  for (int t = 1; t < img->nt; ++t) th2.emplace_back(copy);
  copy();
  for (auto &t : th2) t.join();
  return OBGPU_SUCCESS;
}

void obgpu_table_image_free(obgpu_table_image *img) { delete img; }

int obgpu_agg_row_write(const obgpu_agg_cell *cells, int32_t n_cells, int32_t version, void *out, int64_t out_cap,
                        int64_t *out_size) {
  if (!cells || n_cells <= 0 || !out_size) return OBGPU_INVALID_ARGUMENT;
  std::vector<AggCellIn> in;
  for (int32_t i = 0; i < n_cells; ++i) {
    AggCellIn c{cells[i].col_idx, cells[i].col_type, cells[i].is_null, cells[i].is_prefix, {}};
    if (!c.is_null) {
      if (cells[i].len < 0 || (cells[i].len > 0 && !cells[i].data)) return OBGPU_INVALID_ARGUMENT;
      c.data.assign((const char *)cells[i].data, (size_t)cells[i].len);
    }
    in.push_back(std::move(c));
  }
  std::vector<uint8_t> row;
  const int ret = write_agg_row(std::move(in), version, row);
  if (ret != OBGPU_SUCCESS) return ret;
  *out_size = (int64_t)row.size();
  if (!out) return OBGPU_SUCCESS;
  if ((int64_t)row.size() > out_cap) return OBGPU_BUF_NOT_ENOUGH;
  memcpy(out, row.data(), row.size());
  return OBGPU_SUCCESS;
}

int obgpu_writer_block_agg_row(const obgpu_col_input *cols, int32_t n_cols, const int32_t *agg_cols, int32_t n_agg_cols,
                               int64_t row_begin, int64_t nrows, void *out, int64_t out_cap, int64_t *out_size) {
  if (!cols || !agg_cols || n_agg_cols <= 0 || nrows <= 0 || row_begin < 0 || !out_size) return OBGPU_INVALID_ARGUMENT;
  std::vector<uint8_t> row;
  const int ret = block_agg_row(cols, n_cols, agg_cols, n_agg_cols, row_begin, nrows, row);
  if (ret != OBGPU_SUCCESS) return ret;
  *out_size = (int64_t)row.size();
  if (!out) return OBGPU_SUCCESS;
  if ((int64_t)row.size() > out_cap) return OBGPU_BUF_NOT_ENOUGH;
  memcpy(out, row.data(), row.size());
  return OBGPU_SUCCESS;
}

int obgpu_writer_table_agg_rows(const obgpu_col_input *cols, int32_t n_cols, const int32_t *agg_cols, int32_t n_agg_cols,
                                int64_t total_rows, int64_t rows_per_block, void *out, int64_t out_cap, int64_t *offsets,
                                int64_t *out_size) {
  if (!cols || !agg_cols || n_agg_cols <= 0 || total_rows <= 0 || rows_per_block <= 0 || !out_size) return OBGPU_INVALID_ARGUMENT;
  const int64_t nb = (total_rows + rows_per_block - 1) / rows_per_block;
  std::vector<std::vector<uint8_t>> rows((size_t)nb);
  int nt = std::max(1, std::min<int>((int)std::thread::hardware_concurrency(), (int)std::min<int64_t>(nb, 64)));
  std::atomic<int64_t> next{0};
  std::atomic<int> err{OBGPU_SUCCESS};
  auto work = [&]() {
    for (;;) {
      const int64_t b = next.fetch_add(1);
      if (b >= nb || err.load() != OBGPU_SUCCESS) break;
      const int64_t rb = b * rows_per_block;
      const int r = block_agg_row(cols, n_cols, agg_cols, n_agg_cols, rb, std::min(rows_per_block, total_rows - rb), rows[(size_t)b]);
      if (r != OBGPU_SUCCESS) err.store(r);
    }
  };
  std::vector<std::thread> th;
  for (int t = 1; t < nt; ++t) th.emplace_back(work);
  work();
  for (auto &t : th) t.join();
  if (err.load() != OBGPU_SUCCESS) return err.load();
  int64_t total = 0;
  for (const auto &r : rows) total += (int64_t)r.size();
  *out_size = total;
  if (!out) return OBGPU_SUCCESS;
  if (total > out_cap || !offsets) return OBGPU_BUF_NOT_ENOUGH;
  int64_t pos = 0;
  for (int64_t b = 0; b < nb; ++b) {
    offsets[b] = pos;
    memcpy((uint8_t *)out + pos, rows[(size_t)b].data(), rows[(size_t)b].size());
    pos += (int64_t)rows[(size_t)b].size();
  }
  offsets[nb] = pos;
  return OBGPU_SUCCESS;
}


// ---- macro blocks (ObMacroBlock: reserve_header / write_micro_block / write_macro_header, ob_macro_block.cpp:264-303,455-520) ----
namespace {
#pragma pack(push, 1)
struct MacroCommonHeader {   // ObMacroBlockCommonHeader, ob_macro_block_common_header.h:100-106
  int32_t header_size_, version_, magic_, attr_, payload_size_, payload_checksum_;
};
#pragma pack(pop)
struct MacroFixedHeader {    // ObSSTableMacroBlockHeader::FixedHeader, ob_sstable_macro_block_header.h:48-71 (natural alignment: 128 bytes)
  uint32_t header_size_;
  uint16_t version_, magic_;
  uint64_t tablet_id_;
  int64_t logical_version_, data_seq_;
  int32_t column_count_, rowkey_column_count_, row_store_type_, row_count_, occupy_size_, micro_block_count_,
      micro_block_data_offset_, micro_block_data_size_, idx_block_offset_, idx_block_size_, meta_block_offset_, meta_block_size_;
  int64_t data_checksum_, encrypt_id_, master_key_id_;
  uint8_t compressor_type_;
  char encrypt_key_[16];
};
static_assert(sizeof(MacroCommonHeader) == 24, "ObMacroBlockCommonHeader is 24 bytes");
static_assert(sizeof(MacroFixedHeader) == 128, "FixedHeader is 128 bytes");
}  // namespace

int obgpu_writer_build_macro_blocks(const void *micro_image, const int64_t *offsets, const int64_t *sizes, int32_t n_blocks,
                                    const obgpu_macro_spec *spec, void *out, int64_t out_cap, int64_t *out_size, int32_t *n_macro,
                                    int32_t *first_micro, int32_t first_micro_cap) {
  return obgpu_writer_build_macro_blocks_ex(micro_image, offsets, sizes, n_blocks, spec, out, out_cap, out_size, n_macro, first_micro,
                                            first_micro_cap, OBGPU_COMPRESSOR_NONE);
}

int obgpu_writer_build_macro_blocks_ex(const void *micro_image, const int64_t *offsets, const int64_t *sizes, int32_t n_blocks,
                                       const obgpu_macro_spec *spec, void *out, int64_t out_cap, int64_t *out_size, int32_t *n_macro,
                                       int32_t *first_micro, int32_t first_micro_cap, int32_t compressor_type) {
  if (!micro_image || !offsets || !sizes || n_blocks <= 0 || !spec || !out || !out_size || !n_macro || spec->tablet_id == 0 ||
      spec->n_cols <= 0 || spec->rowkey_col_cnt < 0 || spec->rowkey_col_cnt > spec->n_cols || !spec->col_metas ||
      (spec->header_version != 1 && spec->header_version != 2) || spec->macro_block_size < 4096 || spec->macro_block_size > 0x7fffffffll)
    return OBGPU_INVALID_ARGUMENT;
  if (!obf::stored_compressor(compressor_type)) return OBGPU_NOT_SUPPORTED;
  for (int32_t b = 0; b < n_blocks; ++b) {   // with NONE every micro-block must be stored raw
    if (sizes[b] < 64 || offsets[b] < 0) return OBGPU_INVALID_ARGUMENT;
    const uint8_t *mb = (const uint8_t *)micro_image + offsets[b];
    int32_t len, zlen;
    memcpy(&len, mb + 40, 4);
    memcpy(&zlen, mb + 44, 4);
    if (compressor_type == OBGPU_COMPRESSOR_NONE && len != zlen) return OBGPU_INVALID_ARGUMENT;
  }
  const int64_t n_type_cols = spec->header_version == 2 ? spec->rowkey_col_cnt : spec->n_cols;
  // get_serialize_size: fixed header + ObObjMeta[] + ObOrderType[] + int64 checksum per column + is_normal_cg_
  const int64_t mh_size = (int64_t)sizeof(MacroFixedHeader) + n_type_cols * 4 + n_type_cols * 4 + (int64_t)spec->n_cols * 8 + 1;
  const int64_t data_base = (int64_t)sizeof(MacroCommonHeader) + mh_size;
  const uint8_t *img = (const uint8_t *)micro_image;
  uint8_t *o = (uint8_t *)out;
  int64_t at = 0;
  int32_t nm = 0, b = 0;
  while (b < n_blocks) {
    if (at + spec->macro_block_size > out_cap) return OBGPU_BUF_NOT_ENOUGH;
    if (first_micro && nm < first_micro_cap) first_micro[nm] = b;
    uint8_t *m = o + at;
    memset(m, 0, (size_t)spec->macro_block_size);
    MacroFixedHeader fh{};
    fh.header_size_ = (uint32_t)mh_size;
    fh.version_ = (uint16_t)spec->header_version;
    fh.magic_ = 1007;   // SSTABLE_MACRO_BLOCK_HEADER_MAGIC
    fh.tablet_id_ = spec->tablet_id;
    fh.logical_version_ = spec->logical_version;
    fh.data_seq_ = spec->first_data_seq + nm;
    fh.column_count_ = spec->n_cols;
    fh.rowkey_column_count_ = spec->rowkey_col_cnt;
    fh.micro_block_data_offset_ = (int32_t)data_base;
    fh.encrypt_id_ = 0;
    fh.master_key_id_ = 0;   // the spec's store desc has no encryption (FixedHeader::reset leaves -1 only until init)
    fh.compressor_type_ = (uint8_t)compressor_type;   // ObCompressorType: the micro payloads are in stored form already
    int64_t len = data_base;
    uint64_t data_ck = 0;
    while (b < n_blocks) {
      const int64_t sz = sizes[b];
      if (sz < 64 || offsets[b] < 0) return OBGPU_INVALID_ARGUMENT;
      if (data_base + sz > spec->macro_block_size) return OBGPU_NOT_SUPPORTED;   // a micro block larger than a macro block
      if (len + sz > spec->macro_block_size) break;                              // check_micro_block: no room left
      const uint8_t *mb = img + offsets[b];
      memcpy(m + len, mb, (size_t)sz);
      len += sz;
      fh.micro_block_count_ += 1;
      uint32_t rows;
      memcpy(&rows, mb + 16, 4);
      fh.row_count_ += (int32_t)rows;
      fh.row_store_type_ = mb[20];
      data_ck = crc32c_update((uint32_t)data_ck, mb + 48, 8);   // ob_crc64_sse42(data_checksum_, &header->data_checksum_, 8)
      ++b;
    }
    fh.micro_block_data_size_ = (int32_t)(len - data_base);
    fh.occupy_size_ = (int32_t)len;
    fh.data_checksum_ = (int64_t)data_ck;
    uint8_t *p = m + sizeof(MacroCommonHeader);
    memcpy(p, &fh, sizeof(fh));
    p += sizeof(fh);
    memcpy(p, spec->col_metas, (size_t)n_type_cols * 4);
    p += n_type_cols * 4;
    for (int64_t i = 0; i < n_type_cols; ++i) {
      const int32_t ord = spec->col_orders ? spec->col_orders[i] : 0;
      memcpy(p + i * 4, &ord, 4);
    }
    p += n_type_cols * 4;
    p += (int64_t)spec->n_cols * 8;   // column checksums: "for compatibility, fill 0" (ob_sstable_macro_block_header.cpp:347-350)
    *p = spec->is_cg ? 1 : 0;
    MacroCommonHeader ch{};
    ch.header_size_ = (int32_t)sizeof(MacroCommonHeader);
    ch.version_ = 1;
    ch.magic_ = 1001;
    ch.attr_ = 1;   // SSTableData
    ch.payload_size_ = (int32_t)(len - (int64_t)sizeof(MacroCommonHeader));
    ch.payload_checksum_ = (int32_t)crc32c_update(0, m + sizeof(MacroCommonHeader), (size_t)ch.payload_size_);   // (int32_t)ob_crc64(payload)
    memcpy(m, &ch, sizeof(ch));
    at += spec->macro_block_size;
    ++nm;
  }
  if (first_micro && nm < first_micro_cap) first_micro[nm] = n_blocks;
  *out_size = at;
  *n_macro = nm;
  return OBGPU_SUCCESS;
}

int obgpu_writer_set_cs_stream_encoding(int32_t mode) {
  if (mode < 0 || mode > 8 || mode == obstream::T_UNIVERSAL) return OBGPU_INVALID_ARGUMENT;
  g_cs_stream_mode.store(mode);
  return OBGPU_SUCCESS;
}

int obgpu_writer_stream_encode(int32_t type, int32_t width_bytes, const uint64_t *vals, int64_t count, void *out, int64_t out_cap,
                               int64_t *out_len) {
  if (!vals || !out_len || count < 0 || (width_bytes != 1 && width_bytes != 2 && width_bytes != 4 && width_bytes != 8))
    return OBGPU_INVALID_ARGUMENT;
  std::vector<uint8_t> enc;
  if (type == 0) type = obstream::detect((uint32_t)width_bytes, vals, (size_t)count, false);
  if (!obstream::encode(type, (uint32_t)width_bytes, vals, (size_t)count, enc)) return OBGPU_NOT_SUPPORTED;
  *out_len = (int64_t)enc.size();
  if (!out) return OBGPU_SUCCESS;
  if ((int64_t)enc.size() > out_cap) return OBGPU_BUF_NOT_ENOUGH;
  if (!enc.empty()) memcpy(out, enc.data(), enc.size());
  return OBGPU_SUCCESS;
}

}  // extern "C"

// ---- LZ4 block format (lz4_Block_format.md): what ObLZ4Compressor::compress writes per micro-block payload -------------------
// Greedy single-pass compressor: 4-byte hash -> last position (64 Ki entries), offsets below 64 KiB, no backward extension.
// End-of-block rules of the format: the last 5 bytes are literals (a match ends at n - 5 at the latest) and the last match
// starts at least 12 bytes before the end; the block ends with a literal-only sequence. The constants, the zstd tables and
// the zstd headers / bitstream are ob_compress_format.h's, which the device compressor (stored_compress.cuh) shares.
namespace {
inline uint32_t rd32le(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }

void lz4_put_len(std::vector<uint8_t> &o, int64_t extra) {   // length extension: 255 ... 255, remainder
  for (; extra >= 255; extra -= 255) o.push_back(255);
  o.push_back((uint8_t)extra);
}

// The greedy matcher: emit(at, offset, length) for each match, in order (match length >= 4, offset <= 65535).
template <class Emit>
void greedy_matches(const uint8_t *src, int64_t n, Emit emit) {
  if (n <= obz::kMfLimit) return;
  std::vector<int32_t> table(obz::kHashEntries, -1);
  const int64_t match_end_limit = n - obz::kLastLiterals;
  int64_t ip = 0;
  while (ip <= n - obz::kMfLimit) {
    const uint32_t seq = rd32le(src + ip);
    const uint32_t h = obz::hash4(seq);
    const int64_t ref = table[h];
    table[h] = (int32_t)ip;
    if (ref >= 0 && ip - ref <= obz::kMaxOffset && rd32le(src + ref) == seq) {
      int64_t len = 4;
      while (ip + len < match_end_limit && src[ref + len] == src[ip + len]) ++len;
      emit(ip, ip - ref, len);
      ip += len;
    } else {
      ++ip;
    }
  }
}

void lz4_compress_block(const uint8_t *src, int64_t n, std::vector<uint8_t> &o) {
  o.clear();
  o.reserve((size_t)(n + n / 255 + 16));
  int64_t anchor = 0;
  auto emit = [&](int64_t lit_end, int64_t offset, int64_t mlen) {   // mlen 0: the last, literal-only sequence
    const int64_t lit = lit_end - anchor, ml = mlen ? mlen - 4 : 0;
    o.push_back((uint8_t)((std::min<int64_t>(lit, 15) << 4) | std::min<int64_t>(ml, 15)));
    if (lit >= 15) lz4_put_len(o, lit - 15);
    o.insert(o.end(), src + anchor, src + lit_end);
    if (!mlen) return;
    o.push_back((uint8_t)(offset & 0xff));
    o.push_back((uint8_t)(offset >> 8));
    if (ml >= 15) lz4_put_len(o, ml - 15);
  };
  greedy_matches(src, n, [&](int64_t at, int64_t offset, int64_t len) {
    emit(at, offset, len);
    anchor = at + len;
  });
  emit(n, 0, 0);
}

// ---- zstd frame (RFC 8878): what ObZstdCompressor_1_3_8::compress writes per micro-block payload -----------------------------
// One frame: Single_Segment, Frame_Content_Size, no checksum, no dictionary. Blocks of <= 128 KiB matched on their own by
// greedy_matches; Raw literals; sequences in Predefined mode for LL / OF / ML, FSE-coded from the RFC's default
// distributions (FSE_buildCTable / ZSTD_encodeSequences order); a block that does not shrink is a Raw block.
struct ByteSink {   // obz byte sink over a vector
  std::vector<uint8_t> &o;
  void put(uint8_t b) { o.push_back(b); }
};

// the Block_Content of one Compressed_Block for src[0, n) (n <= 128 KiB)
void zstd_compressed_block(const uint8_t *src, int64_t n, std::vector<uint8_t> &o) {
  static const obz::FseSet fse = [] { obz::FseSet f; obz::fse_build_predefined(f); return f; }();
  std::vector<obz::Seq> seqs;
  std::vector<uint8_t> lits;
  int64_t anchor = 0;
  greedy_matches(src, n, [&](int64_t at, int64_t offset, int64_t len) {
    seqs.push_back({(uint32_t)(at - anchor), (uint32_t)offset, (uint32_t)len});
    lits.insert(lits.end(), src + anchor, src + at);
    anchor = at + len;
  });
  lits.insert(lits.end(), src + anchor, src + n);
  o.clear();
  ByteSink sink{o};
  obz::zstd_literals_header(sink, (uint32_t)lits.size());
  o.insert(o.end(), lits.begin(), lits.end());
  obz::zstd_sequences(sink, seqs.data(), (uint32_t)seqs.size(), fse);
}

void zstd_compress_frame(const uint8_t *src, int64_t n, std::vector<uint8_t> &o) {
  o.clear();
  o.reserve((size_t)(n + n / obz::kZstdBlock * 3 + 32));
  ByteSink sink{o};
  obz::zstd_frame_header(sink, n);
  std::vector<uint8_t> blk;
  int64_t at = 0;
  do {
    const int64_t len = std::min<int64_t>(obz::kZstdBlock, n - at);
    if (len > 0) zstd_compressed_block(src + at, len, blk);
    const bool raw = len == 0 || (int64_t)blk.size() >= len;
    obz::zstd_block_header(sink, at + len == n, raw, (uint32_t)(raw ? len : (int64_t)blk.size()));
    if (raw) o.insert(o.end(), src + at, src + at + len);
    else o.insert(o.end(), blk.begin(), blk.end());
    at += len;
  } while (at < n);
}

// ---- zlib stream (RFC 1950 / RFC 1951): what ObZlibCompressor::compress's output decodes like per micro-block payload --------
// Header 78 01, then the payload in segments of whole symbols covering >= 32 KiB of input each (the last one shorter), each
// segment one fixed-Huffman block or, where fixed coding does not shrink it, one stored block; an Adler-32 trailer. Symbols
// come from greedy_matches: a match farther than 32768 bytes becomes literals, a longer one than 258 bytes pieces of 3..258.
struct Deflater {
  std::vector<uint8_t> &o;
  uint64_t acc = 0;
  int nb = 0;
  void put(uint32_t v, int k) {   // k <= 32 bits, LSB first
    acc |= (uint64_t)v << nb;
    nb += k;
    for (; nb >= 8; nb -= 8, acc >>= 8) o.push_back((uint8_t)acc);
  }
  void align() {
    if (nb > 0) o.push_back((uint8_t)acc);
    acc = 0;
    nb = 0;
  }
  void code(uint32_t c, int len) {   // a Huffman code goes most significant bit first
    uint32_t r = 0;
    for (int k = 0; k < len; ++k) r |= ((c >> k) & 1u) << (len - 1 - k);
    put(r, len);
  }
};

struct DeflateTok {   // len 0: literal `v`; else a match of len 3..258 at distance v 1..32768
  uint16_t len;
  uint16_t v;
};

inline int fixed_lit_bits(int s) { return s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8; }
inline void fixed_lit(Deflater &d, int s) {
  if (s < 144) d.code(0x30u + s, 8);
  else if (s < 256) d.code(0x190u + (s - 144), 9);
  else if (s < 280) d.code((uint32_t)(s - 256), 7);
  else d.code(0xc0u + (s - 280), 8);
}
// length 3..258 -> symbol 257..285 and extra bits; distance 1..32768 -> symbol 0..29 and extra bits
inline void len_code(uint32_t len, int &sym, int &ebits, uint32_t &extra) {
  if (len == 258) { sym = 285; ebits = 0; extra = 0; return; }
  if (len < 11) { sym = 257 + (int)len - 3; ebits = 0; extra = 0; return; }
  int c = 27;
  while ((((4u + (c & 3)) << ((c >> 2) - 1)) + 3u) > len) --c;
  sym = 257 + c;
  ebits = (c >> 2) - 1;
  extra = len - ((((4u + (c & 3)) << ebits)) + 3u);
}
inline void dist_code(uint32_t dist, int &sym, int &ebits, uint32_t &extra) {
  if (dist < 5) { sym = (int)dist - 1; ebits = 0; extra = 0; return; }
  int c = 29;
  while ((((2u + (c & 1)) << ((c >> 1) - 1)) + 1u) > dist) --c;
  sym = c;
  ebits = (c >> 1) - 1;
  extra = dist - (((2u + (c & 1)) << ebits) + 1u);
}

uint32_t adler32_bytes(const uint8_t *p, int64_t n) {
  uint32_t a = 1, b = 0;
  for (int64_t i = 0; i < n; ++i) {
    a = (a + p[i]) % 65521u;
    b = (b + a) % 65521u;
  }
  return (b << 16) | a;
}

void zlib_compress_stream(const uint8_t *src, int64_t n, std::vector<uint8_t> &o) {
  o.clear();
  o.reserve((size_t)(n + 5 * (n / 32768 + 1) + 8));
  std::vector<DeflateTok> toks;
  int64_t anchor = 0;
  greedy_matches(src, n, [&](int64_t at, int64_t offset, int64_t len) {
    for (; anchor < at; ++anchor) toks.push_back({0, src[anchor]});
    if (offset > 32768) return;   // its bytes stay literals: the next match or the tail emits them
    for (int64_t left = len; left > 0;) {   // pieces of 3..258 bytes
      const int64_t piece = left <= 258 ? left : (left - 258 < 3 ? left - 3 : 258);
      toks.push_back({(uint16_t)piece, (uint16_t)offset});
      left -= piece;
    }
    anchor = at + len;
  });
  for (; anchor < n; ++anchor) toks.push_back({0, src[anchor]});
  Deflater d{o};
  d.put(0x78, 8);
  d.put(0x01, 8);
  size_t t = 0;
  int64_t in_at = 0;
  do {
    const size_t t0 = t;
    const int64_t in0 = in_at;
    int64_t bits = 3 + 7;   // block header, end of block
    while (t < toks.size() && in_at - in0 < 32768) {
      const DeflateTok &k = toks[t++];
      if (k.len == 0) {
        bits += fixed_lit_bits(k.v);
        ++in_at;
      } else {
        int s, e, ds, de;
        uint32_t x;
        len_code(k.len, s, e, x);
        dist_code(k.v, ds, de, x);
        bits += fixed_lit_bits(s) + e + 5 + de;
        in_at += k.len;
      }
    }
    const bool last = t == toks.size();
    const int64_t seg = in_at - in0;
    const int64_t stored_bits = 3 + ((8 - (d.nb + 3) % 8) % 8) + 32 + 8 * seg;
    if (seg > 0 && stored_bits <= bits) {
      d.put(last ? 1u : 0u, 1);
      d.put(0, 2);
      d.align();
      d.put((uint32_t)seg, 16);
      d.put((uint32_t)~seg & 0xffffu, 16);
      o.insert(o.end(), src + in0, src + in_at);
    } else {
      d.put(last ? 1u : 0u, 1);
      d.put(1, 2);
      for (size_t j = t0; j < t; ++j) {
        const DeflateTok &k = toks[j];
        if (k.len == 0) {
          fixed_lit(d, k.v);
          continue;
        }
        int s, e, ds, de;
        uint32_t x, dx;
        len_code(k.len, s, e, x);
        dist_code(k.v, ds, de, dx);
        fixed_lit(d, s);
        if (e) d.put(x, e);
        d.code((uint32_t)ds, 5);
        if (de) d.put(dx, de);
      }
      fixed_lit(d, 256);
    }
  } while (t < toks.size());
  d.align();
  const uint32_t ad = adler32_bytes(src, n);
  for (int k = 3; k >= 0; --k) o.push_back((uint8_t)(ad >> (8 * k)));
}

}  // namespace

extern "C" {

int obgpu_writer_lz4_compress(const void *src, int64_t src_len, void *out, int64_t out_cap, int64_t *out_len) {
  if ((!src && src_len > 0) || src_len < 0 || src_len > 0x7e000000ll || !out_len) return OBGPU_INVALID_ARGUMENT;
  std::vector<uint8_t> o;
  lz4_compress_block((const uint8_t *)src, src_len, o);
  *out_len = (int64_t)o.size();
  if (!out) return OBGPU_SUCCESS;
  if ((int64_t)o.size() > out_cap) return OBGPU_BUF_NOT_ENOUGH;
  memcpy(out, o.data(), o.size());
  return OBGPU_SUCCESS;
}

int obgpu_writer_zstd_compress(const void *src, int64_t src_len, void *out, int64_t out_cap, int64_t *out_len) {
  if ((!src && src_len > 0) || src_len < 0 || src_len > 0x7e000000ll || !out_len) return OBGPU_INVALID_ARGUMENT;
  std::vector<uint8_t> o;
  zstd_compress_frame((const uint8_t *)src, src_len, o);
  *out_len = (int64_t)o.size();
  if (!out) return OBGPU_SUCCESS;
  if ((int64_t)o.size() > out_cap) return OBGPU_BUF_NOT_ENOUGH;
  memcpy(out, o.data(), o.size());
  return OBGPU_SUCCESS;
}

int obgpu_writer_zlib_compress(const void *src, int64_t src_len, void *out, int64_t out_cap, int64_t *out_len) {
  if ((!src && src_len > 0) || src_len < 0 || src_len > 0x7e000000ll || !out_len) return OBGPU_INVALID_ARGUMENT;
  std::vector<uint8_t> o;
  zlib_compress_stream((const uint8_t *)src, src_len, o);
  *out_len = (int64_t)o.size();
  if (!out) return OBGPU_SUCCESS;
  if ((int64_t)o.size() > out_cap) return OBGPU_BUF_NOT_ENOUGH;
  memcpy(out, o.data(), o.size());
  return OBGPU_SUCCESS;
}

int obgpu_writer_compress_blocks(const void *image, const int64_t *offsets, const int64_t *sizes, int32_t n_blocks, int32_t compressor,
                                 int64_t align, void *out, int64_t out_cap, int64_t *out_offsets, int64_t *out_sizes,
                                 int64_t *out_size) {
  if (!image || !offsets || !sizes || n_blocks <= 0 || !out || !out_offsets || !out_sizes || !out_size || align < 1 ||
      (align & (align - 1)) != 0)
    return OBGPU_INVALID_ARGUMENT;
  if (!obf::stored_compressor(compressor)) return OBGPU_NOT_SUPPORTED;
  const uint8_t *img = (const uint8_t *)image;
  uint8_t *o = (uint8_t *)out;
  std::vector<uint8_t> z;
  int64_t at = 0;
  for (int32_t b = 0; b < n_blocks; ++b) {
    const uint8_t *blk = img + offsets[b];
    uint32_t hs;
    int32_t len, zlen;
    if (sizes[b] < 64 || offsets[b] < 0) return OBGPU_INVALID_ARGUMENT;
    memcpy(&hs, blk + 4, 4);
    memcpy(&len, blk + 40, 4);
    memcpy(&zlen, blk + 44, 4);
    if (hs < 64 || len != zlen || (int64_t)hs + len != sizes[b]) return OBGPU_INVALID_DATA;   // plain, well-framed blocks only
    at = (at + align - 1) & ~(align - 1);
    bool keep_raw = compressor == OBGPU_COMPRESSOR_NONE;
    if (!keep_raw) {
      if (compressor == OBGPU_COMPRESSOR_ZSTD_1_3_8) zstd_compress_frame(blk + hs, len, z);
      else if (compressor == OBGPU_COMPRESSOR_ZLIB) zlib_compress_stream(blk + hs, len, z);
      else lz4_compress_block(blk + hs, len, z);
      keep_raw = (int64_t)z.size() >= len;   // a block that does not shrink is stored raw (data_zlength_ == data_length_)
    }
    const int64_t stored = keep_raw ? sizes[b] : (int64_t)hs + (int64_t)z.size();
    if (at + stored > out_cap) return OBGPU_BUF_NOT_ENOUGH;
    uint8_t *d = o + at;
    memcpy(d, blk, hs);
    if (keep_raw) {
      memcpy(d + hs, blk + hs, (size_t)len);
    } else {
      memcpy(d + hs, z.data(), z.size());
      const int32_t zl = (int32_t)z.size();
      const int64_t ck = (int64_t)crc32c_update(0, z.data(), z.size());   // data_checksum_: crc over the stored bytes
      memcpy(d + 44, &zl, 4);
      memcpy(d + 48, &ck, 8);
      const int16_t hc = obf::micro_header_checksum(d);
      memcpy(d + 8, &hc, 2);
    }
    out_offsets[b] = at;
    out_sizes[b] = stored;
    at += stored;
  }
  *out_size = at;
  return OBGPU_SUCCESS;
}

}  // extern "C"
