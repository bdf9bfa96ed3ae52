// On-disk layout of an OceanBase PAX ("ENCODING_ROW_STORE") micro-block, restated as plain
// packed PODs usable from host C++ and from device code.
//
// Layout authority (reference, read-only spec):
//   header           src/storage/blocksstable/ob_micro_block_header.h:97-153   (64-byte packed struct)
//   column header    src/storage/blocksstable/ob_block_sstable_struct.h:201-264 (16-byte packed struct)
//   block layout     src/storage/blocksstable/encoding/ob_micro_block_encoder.cpp:499-721
//                    [header][ObColumnHeader x ncol][per column: meta + fixed data][row data][row index]
//   dict meta        src/storage/blocksstable/encoding/ob_dict_encoder.h:31-58   (9 bytes)
//   rle meta         src/storage/blocksstable/encoding/ob_rle_encoder.h:27-48    (10 bytes)
//   base-diff meta   src/storage/blocksstable/encoding/ob_integer_base_diff_encoder.h:26-37 (2 bytes + base)
//   const meta       src/storage/blocksstable/encoding/ob_const_encoder.h:28-50
#pragma once
#include <stdint.h>

#include "../../include/obgpu_scan.h"   // OBGPU_COMPRESSOR_*

#if defined(__CUDACC__)
#define OBF_HD __host__ __device__ __forceinline__
#else
#define OBF_HD inline
#endif

namespace obf {

constexpr int16_t MICRO_BLOCK_HEADER_MAGIC = 1005;  // ob_block_sstable_struct.h:48
constexpr int16_t MICRO_BLOCK_HEADER_VERSION = 3;   // ob_micro_block_header.h:31
constexpr uint32_t MICRO_HEADER_FIXED_SIZE = 64;    // ob_micro_block_header.cpp:21

// common::ObRowStoreType  deps/oblib/src/common/ob_store_format.h:31-40
enum RowStoreType : uint8_t {
  FLAT_ROW_STORE = 0,
  ENCODING_ROW_STORE = 1,
  SELECTIVE_ENCODING_ROW_STORE = 2,
  CS_ENCODING_ROW_STORE = 3,
  MAX_ROW_STORE = 5,
};

#pragma pack(push, 1)
struct MicroBlockHeader {
  int16_t magic_;
  int16_t version_;
  uint32_t header_size_;
  int16_t header_checksum_;
  uint16_t column_count_;
  uint16_t rowkey_column_count_;
  uint16_t flag16_;  // bit0 has_column_checksum, bit1 has_string_out_row, bit2 all_lob_in_row, ...
  uint32_t row_count_;
  uint8_t row_store_type_;
  uint8_t opt_;   // PAX: row_index_byte:3 | extend_value_bit:3 | reserved:2
  uint16_t opt2_; // PAX: var_column_count
  uint32_t row_data_offset_;
  int32_t original_length_;
  int64_t max_merged_trans_version_;
  int32_t data_length_;
  int32_t data_zlength_;
  int64_t data_checksum_;
  int64_t column_checksums_ptr_;  // pointer slot / min_merged_trans_version

  OBF_HD uint32_t row_index_byte() const { return opt_ & 0x7u; }
  OBF_HD uint32_t extend_value_bit() const { return (opt_ >> 3) & 0x7u; }
  OBF_HD bool has_column_checksum() const { return flag16_ & 0x1u; }
  OBF_HD bool all_lob_in_row() const { return (flag16_ >> 2) & 0x1u; }
};

struct ColumnHeader {
  int8_t version_;
  int8_t type_;
  int8_t attr_;
  uint8_t obj_type_;
  uint32_t extend_value_index_;  // union with extend_value_offset_
  uint32_t offset_;
  uint32_t length_;
};

struct DictMetaHeader {
  uint8_t version_;
  uint8_t row_ref_size_;
  uint32_t count_;
  uint16_t data_size_;  // union with index_byte_
  uint8_t attr_;
};

struct RLEMetaHeader {
  uint8_t version_;
  uint8_t attr_;  // row_id_byte:3 | ref_byte:3 | reserved:2
  uint32_t count_;
  uint32_t offset_;  // offset of the dict meta from this header
};

struct IntegerBaseDiffHeader {
  uint8_t version_;
  uint8_t length_;
};

// ob_const_encoder.h:28-50
struct ConstMetaHeader {
  uint8_t version_;
  uint8_t count_;        // exception count
  uint8_t const_ref_;
  uint8_t row_id_byte_;
  uint16_t offset_;      // dict meta offset (when count_ > 0)
};
// ---- CS_ENCODING_ROW_STORE (column-store encoding) ---------------------------------------------
// cs_encoding/ob_column_encoding_struct.h:142-181
struct AllColumnHeader {
  uint8_t version_;
  uint8_t attrs_;                    // IS_FULL_TRANSFORMED 0x1 (memory only), IS_ALL_STRING_COMPRESSED 0x2
  uint32_t all_string_data_length_;
  uint32_t stream_offsets_length_;
  uint16_t stream_count_;
};
// cs_encoding/ob_column_encoding_struct.h:31-139
struct CSColumnHeader {
  uint8_t version_;
  uint8_t type_;                     // CSColType
  uint8_t attrs_;                    // CSColAttr
  uint8_t obj_type_;
};
// cs_encoding/ob_column_encoding_struct.h:183-221
struct DictEncodingMeta {
  uint8_t version_;
  uint8_t attrs_;                    // IS_SORTED 0x1, HAS_NULL 0x2, CONST_ENCODING_REF 0x4
  uint32_t distinct_val_cnt_;
  uint32_t ref_row_cnt_;
};
#pragma pack(pop)

static_assert(sizeof(AllColumnHeader) == 12, "all column header must be 12 bytes");
static_assert(sizeof(CSColumnHeader) == 4, "cs column header must be 4 bytes");
static_assert(sizeof(DictEncodingMeta) == 10, "dict encoding meta must be 10 bytes");

enum CSColType : uint8_t { CS_INTEGER = 0, CS_STRING = 1, CS_INT_DICT = 2, CS_STR_DICT = 3, CS_SEMISTRUCT = 4, CS_MAX_TYPE = 5 };
enum CSColAttr : uint8_t { CS_IS_FIXED_LENGTH = 0x01, CS_HAS_NULL_OR_NOP_BITMAP = 0x02, CS_OUT_ROW = 0x04,
                           CS_HAS_NOP_BITMAP = 0x08, CS_HAS_NOP = 0x10 };
// ObIntegerStreamMeta (cs_encoding/ob_stream_encoding_struct.h:108-290), serialized as
//   version u8, attr u8, type u8, width u8, [vi64 base], [vi64 null_replaced], [u8 decimal width], (v2:) u8 pfor type
enum IntStreamAttr : uint8_t { IS_USE_BASE = 0x1, IS_REPLACE_NULL_VALUE = 0x2, IS_DECIMAL_INT = 0x4 };
enum IntStreamType : uint8_t { IS_RAW = 1 };   // the other codecs need the CPU transformer (not handled)
constexpr uint8_t INTEGER_STREAM_META_V2 = 1;

// ObCompressorType values whose micro-blocks the library writes (host writer) and opens in stored form: NONE, and the payload
// codecs the device decodes (stored_blocks.cuh)
OBF_HD bool stored_compressor(int32_t c) {
  return c == OBGPU_COMPRESSOR_NONE || c == OBGPU_COMPRESSOR_LZ4 || c == OBGPU_COMPRESSOR_ZLIB || c == OBGPU_COMPRESSOR_ZSTD_1_3_8 ||
         c == OBGPU_COMPRESSOR_LZ4_1_9_1;
}

// The subset the device also compresses (obgpu_compress_blocks, stored_compress.cuh): zlib is decoded but not encoded there
OBF_HD bool device_compressor(int32_t c) {
  return c == OBGPU_COMPRESSOR_NONE || c == OBGPU_COMPRESSOR_LZ4 || c == OBGPU_COMPRESSOR_LZ4_1_9_1 || c == OBGPU_COMPRESSOR_ZSTD_1_3_8;
}

// ObMicroBlockHeader header checksum (ob_micro_block_header.cpp:203-233) of a 64-byte header as stored: the XOR of the 16-bit
// halves of its fields, header_checksum_ (bytes 8-9) left out; the signed 32-bit fields are sign-extended to 64 bits first.
OBF_HD int16_t micro_header_checksum(const uint8_t *h) {
  auto le = [h](int off, int bytes) {   // unaligned little-endian load
    uint64_t v = 0;
    for (int k = bytes - 1; k >= 0; --k) v = (v << 8) | h[off + k];
    return v;
  };
  auto i32 = [&](int off) { return (uint64_t)(int64_t)(int32_t)le(off, 4); };
  const uint64_t x = le(0, 2) ^ le(2, 2) ^ h[20] ^ h[21]                  // magic_, version_, row_store_type_, opt_
                     ^ le(10, 2) ^ le(12, 2) ^ (le(14, 2) & 1) ^ le(22, 2)  // column_count_, rowkey_column_count_, has_column_checksum, opt2_
                     ^ le(4, 4) ^ le(16, 4) ^ le(24, 4) ^ i32(28)          // header_size_, row_count_, row_data_offset_, original_length_
                     ^ le(32, 8) ^ i32(40) ^ i32(44) ^ le(48, 8);          // max_merged_trans_version_, data_length_, data_zlength_, data_checksum_
  return (int16_t)(uint16_t)(x ^ (x >> 16) ^ (x >> 32) ^ (x >> 48));
}

// What check_micro_header found wrong with a micro-block header
enum MicroHeaderVerdict : uint32_t { HDR_OK = 0, HDR_INVALID = 1, HDR_ROW_STORE = 2, HDR_EXTENT = 3, HDR_TOO_MANY_ROWS = 4 };
struct MicroHeaderFacts {
  uint32_t header_size, rows, ncol;
  bool is_cs;
};

// The header rules a page-batch open applies to a block of `size` bytes, first failure wins: ObMicroBlockHeader::is_valid
// (ob_micro_block_header.cpp:53-61); a row store type the device path decodes (PAX or CS); the column headers, and a PAX block's
// row data, start inside the block, which holds at least one row (get_micro_metas bounds); at most 65535 rows. The facts are read
// from the header whatever the verdict.
OBF_HD uint32_t check_micro_header(const uint8_t *h, uint32_t size, MicroHeaderFacts &f) {
  auto le = [h](int off, int bytes) {   // unaligned little-endian load
    uint32_t v = 0;
    for (int k = bytes - 1; k >= 0; --k) v = (v << 8) | h[off + k];
    return v;
  };
  const int16_t magic = (int16_t)le(0, 2), version = (int16_t)le(2, 2);
  const uint32_t nkey = le(12, 2), rst = h[20], row_data_off = le(24, 4);
  f.header_size = le(4, 4);
  f.ncol = le(10, 2);
  f.rows = le(16, 4);
  f.is_cs = rst == CS_ENCODING_ROW_STORE;
  if (magic != MICRO_BLOCK_HEADER_MAGIC || version < 1 || version > 3 || f.ncol < nkey || rst >= MAX_ROW_STORE) return HDR_INVALID;
  if (rst != ENCODING_ROW_STORE && rst != SELECTIVE_ENCODING_ROW_STORE && !f.is_cs) return HDR_ROW_STORE;
  if (f.header_size < 64 || (uint64_t)f.header_size + (f.is_cs ? 12ull + 4ull * f.ncol : 16ull * f.ncol) > size ||
      (!f.is_cs && row_data_off > size) || f.rows == 0)
    return HDR_EXTENT;
  if (f.rows > 65535u) return HDR_TOO_MANY_ROWS;
  return HDR_OK;
}

static_assert(sizeof(MicroBlockHeader) == 64, "micro header must be 64 bytes");
static_assert(sizeof(ColumnHeader) == 16, "column header must be 16 bytes");
static_assert(sizeof(DictMetaHeader) == 9, "dict meta header must be 9 bytes");
static_assert(sizeof(RLEMetaHeader) == 10, "rle meta header must be 10 bytes");
static_assert(sizeof(IntegerBaseDiffHeader) == 2, "base diff header must be 2 bytes");
static_assert(sizeof(ConstMetaHeader) == 6, "const meta header must be 6 bytes");

// ObColumnHeader::Type  ob_block_sstable_struct.h:203-216
enum ColType : int8_t {
  COL_RAW = 0,
  COL_DICT = 1,
  COL_RLE = 2,
  COL_CONST = 3,
  COL_INTEGER_BASE_DIFF = 4,
  COL_STRING_DIFF = 5,
  COL_HEX_PACKING = 6,
  COL_STRING_PREFIX = 7,
  COL_COLUMN_EQUAL = 8,
  COL_COLUMN_SUBSTR = 9,
  COL_MAX_TYPE = 10,
};

// Column types whose strings a page batch materialises at open (mat_codecs.cuh): rebuilt by the decoder (STRING_DIFF, HEX_PACKING,
// STRING_PREFIX) or taken from another column (COLUMN_EQUAL, COLUMN_SUBSTR)
OBF_HD bool rebuilt_at_open(uint32_t t) {
  return t == COL_STRING_DIFF || t == COL_HEX_PACKING || t == COL_STRING_PREFIX || t == COL_COLUMN_EQUAL || t == COL_COLUMN_SUBSTR;
}

// ObColumnHeader::Attribute  ob_block_sstable_struct.h:218-226
enum ColAttr : int8_t {
  ATTR_FIX_LENGTH = 0x1,
  ATTR_HAS_EXTEND_VALUE = 0x2,
  ATTR_BIT_PACKING = 0x4,
  ATTR_LAST_VAR_FIELD = 0x8,
};

enum DictAttr : uint8_t { DICT_FIX_LENGTH = 0x1, DICT_IS_SORTED = 0x2 };

// ObStoredExtValue  encoding/ob_encoding_util.h:279-285
enum StoredExt : uint32_t { STORED_NOT_EXT = 0, STORED_NULL = 1, STORED_NOPE = 2 };

// ObObjType values used by this path (deps/oblib/src/common/object/ob_obj_type.h; order also
// visible in encoding/ob_encoding_util.h:133-195).
enum ObjType : uint8_t {
  ObNullType = 0,
  ObTinyIntType = 1,
  ObSmallIntType = 2,
  ObMediumIntType = 3,
  ObInt32Type = 4,
  ObIntType = 5,
  ObUTinyIntType = 6,
  ObUSmallIntType = 7,
  ObUMediumIntType = 8,
  ObUInt32Type = 9,
  ObUInt64Type = 10,
  ObDateTimeType = 17,
  ObTimestampType = 18,
  ObDateType = 19,
  ObTimeType = 20,
  ObYearType = 21,
  ObVarcharType = 22,
  ObCharType = 23,
};

// Store class of an obj type restricted to what the path supports:
// 1 = signed integer class (ObIntSC), 2 = unsigned integer class (ObUIntSC), 5 = string (ObStringSC),
// 0 = unsupported here.  encoding/ob_encoding_util.h:59-130
OBF_HD int store_class_of(uint8_t t) {
  switch (t) {
    case ObTinyIntType: case ObSmallIntType: case ObMediumIntType: case ObInt32Type: case ObIntType:
    case ObDateTimeType: case ObTimestampType: case ObDateType: case ObTimeType:
      return 1;
    case ObUTinyIntType: case ObUSmallIntType: case ObUMediumIntType: case ObUInt32Type:
    case ObUInt64Type: case ObYearType:
      return 2;
    case ObVarcharType: case ObCharType:
      return 5;
    default:
      return 0;
  }
}

// get_type_size_map()  encoding/ob_encoding_util.h:133-195
OBF_HD int type_store_size(uint8_t t) {
  switch (t) {
    case ObTinyIntType: case ObUTinyIntType: case ObYearType: return 1;
    case ObSmallIntType: case ObUSmallIntType: return 2;
    case ObMediumIntType: case ObInt32Type: case ObUMediumIntType: case ObUInt32Type:
    case ObDateType: return 4;
    case ObIntType: case ObUInt64Type: case ObDateTimeType: case ObTimestampType: case ObTimeType:
      return 8;
    default: return -1;
  }
}

// ---- skip index aggregate row (index_block/ob_agg_row_struct.h:27-66) -----------------------------------------
struct AggRowHeader {
  int16_t version_;      // 1, 2 (prefix bitmap per cell), 3 (revised max prefix)
  int16_t length_;       // bytes of the whole row
  int16_t agg_col_cnt_;  // aggregated columns (cells)
  uint16_t pack_;        // agg_col_idx_size:6 | agg_col_idx_off_size:3 | cell_off_size:3 | bitmap_size:4 (== 1)
};
static_assert(sizeof(AggRowHeader) == 8, "ObAggRowHeader is 8 bytes");

// Datum length of an integer-class obj type: 4 for the 4-byte map types, 1 for year, else 8
// (ObDatum::get_obj_datum_map_type, share/datum/ob_datum.h; get_uint_data_datum_len).
OBF_HD int datum_len_of(uint8_t t) {
  switch (t) {
    case ObYearType: return 1;
    case ObDateType: return 4;
    default: return 8;
  }
}

// Sign-extension mask: ~INTEGER_MASK_TABLE[type_store_size] for ObIntTC only
// (encoding/ob_raw_decoder.h init, ob_dict_decoder.cpp:198-203, ob_encoding_util.cpp:32-35).
OBF_HD uint64_t integer_mask_of(uint8_t t) {
  switch (t) {
    case ObTinyIntType: return ~0xffull;
    case ObSmallIntType: return ~0xffffull;
    case ObMediumIntType: case ObInt32Type: return ~0xffffffffull;
    default: return 0;  // ObIntType (8 bytes) -> mask 0; non-ObIntTC -> 0
  }
}

OBF_HD uint64_t low_mask(uint32_t bits) { return bits >= 64 ? ~0ull : ((1ull << bits) - 1ull); }

}  // namespace obf
