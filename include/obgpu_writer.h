/*
 * obgpu_writer.h -- C-ABI of the host-side micro-block / aggregate-row writer (libobgpu_writer.so).
 *
 * Plain C++ (no CUDA): the synthetic-SSTable generator of the tests and benchmarks and the seed of the
 * compaction writer. It lives in its own shared library so that nothing that only WRITES blocks (the
 * reference arm of bench.py, the CPU test suite) maps the CUDA product library libobgpu_scan.so.
 * Reference: ObMicroBlockEncoder::build_block (encoding/ob_micro_block_encoder.cpp:561-721),
 * ObMicroBlockCSEncoder::build_block (cs_encoding/ob_micro_block_cs_encoder.cpp:1394-1488),
 * ObAggRowWriter (index_block/ob_agg_row_struct.cpp:49-300).
 */
#ifndef OBGPU_WRITER_H_
#define OBGPU_WRITER_H_

#include <stddef.h>
#include <stdint.h>

#include "obgpu_skip_index.h" /* constants only (OB error codes, OBGPU_ENC_*, OBGPU_OBJ_*, OBGPU_SK_IDX_*): no link dependency */

#ifdef __cplusplus
extern "C" {
#endif

/* =============================================================================================
 * Writer: host-side PAX micro-block encoder producing reference-format blocks
 * (ObMicroBlockEncoder::build_block, encoding/ob_micro_block_encoder.cpp:561-721) for a forced
 * per-column encoding.  Used to build SSTables for tests / benchmarks and by the compaction
 * writer.  Column inputs are column-major arrays over the rows of the table.
 * ============================================================================================= */
typedef struct obgpu_col_input {
  int32_t obj_type;        /* OBGPU_OBJ_*                                                      */
  int32_t encoding;        /* OBGPU_ENC_*                                                      */
  const int64_t *i64;      /* integer classes: value per row                                   */
  const uint8_t *is_null;  /* optional: 1 => NULL, 2 => NOP (cell absent in an incremental row)       */
  const char *str_heap;    /* string classes: bytes                                            */
  const int64_t *str_off;  /*   nrows + 1 offsets into str_heap                                */
  int32_t byte_packing_only; /* 1 => ObMicroBlockEncoderOpt.enable_bit_packing_ == false       */
  int32_t ref_col;         /* OBGPU_ENC_COLUMN_EQUAL / COLUMN_SUBSTR: the column this one refers to      */
} obgpu_col_input;

/* Upper bound of the encoded size of a block of nrows rows. */
int64_t obgpu_writer_block_bound(const obgpu_col_input *cols, int32_t n_cols, int64_t row_begin,
                                 int64_t nrows);
/* Encode rows [row_begin, row_begin + nrows) into one micro-block. */
int obgpu_writer_encode_block(const obgpu_col_input *cols, int32_t n_cols,
                              int32_t rowkey_col_cnt, int64_t row_begin, int64_t nrows,
                              void *out, int64_t out_cap, int64_t *out_size);
/* Encode total_rows rows as consecutive blocks of rows_per_block rows (last one shorter). The
 * encoded blocks are held by the returned handle; export packs them into one image where block i
 * starts at offsets[i] (aligned to `align`, a power of two >= 16, padding zeroed) and is sizes[i]
 * bytes long. n_threads <= 0 uses all hardware threads. */
typedef struct obgpu_table_image obgpu_table_image;
int obgpu_writer_encode_table(const obgpu_col_input *cols, int32_t n_cols, int32_t rowkey_col_cnt,
                              int64_t total_rows, int64_t rows_per_block, int32_t align,
                              int32_t n_threads, obgpu_table_image **out);
int obgpu_table_image_info(const obgpu_table_image *img, int64_t *image_size, int32_t *n_blocks);
int obgpu_table_image_export(const obgpu_table_image *img, void *image, int64_t image_cap,
                             int64_t *offsets, int64_t *sizes, int32_t tables_cap);
void obgpu_table_image_free(obgpu_table_image *img);


#define OBGPU_SKIP_INDEX_MAX_COL_LENGTH 40 /* ObSkipIndexColMeta::MAX_SKIP_INDEX_COL_LENGTH */

/* One aggregate of an aggregate row: (ObSkipIndexColMeta, ObStorageDatum, is_min_max_prefix). */
typedef struct obgpu_agg_cell {
  uint32_t col_idx;  /* column store index the aggregate refers to                      */
  uint8_t col_type;  /* OBGPU_SK_IDX_*                                                  */
  uint8_t is_null;   /* NULL / NOP datum: the aggregate is not stored                   */
  uint8_t is_prefix; /* MIN / MAX of a string longer than 40 bytes: only a prefix kept  */
  uint8_t reserved;
  int32_t len;       /* datum length in bytes                                           */
  const void *data;  /* datum bytes                                                     */
} obgpu_agg_cell;

/* ObAggRowWriter::init + write_agg_data (ob_agg_row_struct.cpp:49-300): serializes the cells (any order)
 * as one aggregate row. version: 1, 2 (prefix bitmap) or 3 (revised max prefix; the current one).
 * out == NULL: only *out_size is computed. */
int obgpu_agg_row_write(const obgpu_agg_cell *cells, int32_t n_cells, int32_t version, void *out,
                        int64_t out_cap, int64_t *out_size);

/* ObSkipIndexAggregator over rows [row_begin, row_begin + nrows) of the writer's column inputs
 * (index_block/ob_index_block_aggregator.cpp): MIN / MAX / NULL_COUNT of every column listed in agg_cols,
 * serialized as one version-3 aggregate row. Strings longer than 40 bytes keep a 40-byte prefix. */
int obgpu_writer_block_agg_row(const obgpu_col_input *cols, int32_t n_cols, const int32_t *agg_cols,
                               int32_t n_agg_cols, int64_t row_begin, int64_t nrows, void *out,
                               int64_t out_cap, int64_t *out_size);
/* One aggregate row per block of obgpu_writer_encode_table's blocking: row b occupies
 * [offsets[b], offsets[b + 1]) of `out` (n_blocks + 1 offsets). out == NULL: only *out_size. */
int obgpu_writer_table_agg_rows(const obgpu_col_input *cols, int32_t n_cols, const int32_t *agg_cols,
                                int32_t n_agg_cols, int64_t total_rows, int64_t rows_per_block, void *out,
                                int64_t out_cap, int64_t *offsets, int64_t *out_size);

/* Integer stream codecs of CS blocks (ObIntegerStream::EncodingType, cs_encoding/ob_stream_encoding_struct.h:64-76:
 * 1 RAW, 2 DOUBLE_DELTA_ZIGZAG_RLE, 3 DOUBLE_DELTA_ZIGZAG_PFOR, 4 DELTA_ZIGZAG_RLE, 5 DELTA_ZIGZAG_PFOR, 6 SIMD_FIXEDPFOR,
 * 8 XOR_FIXED_PFOR). The CS writer encodes its column streams with: mode 1 RAW (default); 0 the codec
 * ObIntegerStreamEncoder::choose_stream_codec would detect (smallest on a sample, cs_encoding/ob_integer_stream_encoder.h:
 * 195-400); 2..8 that codec wherever it is not larger than RAW. Process-wide setting. */
/* =============================================================================================
 * Macro blocks: encoded micro-blocks packed into fixed-size (2 MiB) macro blocks the way ObMacroBlock does
 *   blocksstable/ob_macro_block.cpp:455-520   reserve_header / write_macro_header: [ObMacroBlockCommonHeader (24 B)]
 *                                             [ObSSTableMacroBlockHeader: FixedHeader (128 B) + column types / orders /
 *                                             checksums + is_normal_cg_] then the micro-blocks back to back
 *   blocksstable/ob_macro_block.cpp:264-303   write_micro_block: micro header + data appended; row_count_, micro_block_count_,
 *                                             micro_block_data_size_, occupy_size_ and the running data_checksum_ (crc of the
 *                                             micro headers' data_checksum_ fields)
 *   ob_macro_block_common_header.h:20-112, ob_sstable_macro_block_header.h:30-113
 * The leaf index block and the macro meta block that follow the data in the reference (idx_block_*, meta_block_*) are not
 * written (index rows are outside the path): their fields stay 0, which FixedHeader::is_valid() accepts. Every macro block
 * occupies macro_block_size bytes of `out` (zero padded), like a block slot on disk.
 * ============================================================================================= */
typedef struct obgpu_macro_spec {
  uint64_t tablet_id;           /* != 0 */
  int64_t logical_version;
  int64_t first_data_seq;       /* data_seq_ of macro block i = first_data_seq + i */
  int32_t header_version;       /* 1: type / order arrays for every column, 2: for the rowkey columns only */
  int32_t is_cg;                /* is_normal_cg_ */
  int32_t rowkey_col_cnt;
  int32_t n_cols;
  const uint8_t *col_metas;     /* n_cols x 4 bytes (ObObjMeta: type_, cs_level_, cs_type_, scale_)              */
  const int32_t *col_orders;    /* n_cols ObOrderType values (ASC 0, DESC -1); NULL: all ASC                      */
  int64_t macro_block_size;     /* 2 MiB (OB_DEFAULT_MACRO_BLOCK_SIZE)                                            */
} obgpu_macro_spec;
/* first_micro (optional): n_macro + 1 entries, micro-blocks [first_micro[i], first_micro[i + 1]) live in macro block i. */
int obgpu_writer_build_macro_blocks(const void *micro_image, const int64_t *offsets, const int64_t *sizes, int32_t n_blocks,
                                    const obgpu_macro_spec *spec, void *out, int64_t out_cap, int64_t *out_size,
                                    int32_t *n_macro, int32_t *first_micro, int32_t first_micro_cap);
/* The same with the FixedHeader's compressor_type_ (OBGPU_COMPRESSOR_*). The micro-blocks are taken as they are, in stored
 * form (obgpu_writer_compress_blocks): a macro block records the compressor, it does not apply it. With NONE every block must
 * have data_zlength_ == data_length_ (OBGPU_INVALID_ARGUMENT otherwise); LZ4 / LZ4_1_9_1 / ZLIB / ZSTD_1_3_8 record that compressor;
 * other compressors: OBGPU_NOT_SUPPORTED. obgpu_writer_build_macro_blocks is this call with OBGPU_COMPRESSOR_NONE. */
int obgpu_writer_build_macro_blocks_ex(const void *micro_image, const int64_t *offsets, const int64_t *sizes, int32_t n_blocks,
                                       const obgpu_macro_spec *spec, void *out, int64_t out_cap, int64_t *out_size,
                                       int32_t *n_macro, int32_t *first_micro, int32_t first_micro_cap, int32_t compressor_type);

/* =============================================================================================
 * Compressed micro-blocks (ObMicroBlockWriter / ObMicroBlockEncoder::build_block -> ObMicroBlockCompressor::compress): the
 * 64-byte ObMicroBlockHeader stays plain, the payload behind it is compressed on its own, data_zlength_ is the stored
 * payload size and data_length_ the decoded one; data_checksum_ is the crc32c of the STORED payload bytes.
 * ============================================================================================= */
/* One LZ4 block (lz4 block format: no frame, no size prefix; what LZ4_compress_default's output decodes like): greedy, 64 KiB
 * window, end-of-block rules of the format kept. out == NULL: only *out_len (never more than src_len + src_len / 255 + 16). */
int obgpu_writer_lz4_compress(const void *src, int64_t src_len, void *out, int64_t out_cap, int64_t *out_len);
/* One zstd frame (RFC 8878; what ZSTD_decompressDCtx and ObZstdCompressor_1_3_8::decompress read): Single_Segment with
 * Frame_Content_Size, no checksum, no dictionary; blocks of <= 128 KiB matched by the LZ4 compressor's greedy matcher; Raw
 * literals; sequences in Predefined mode (FSE from the RFC's default distributions); a block that does not shrink is a Raw
 * block. out == NULL: only *out_len (never more than src_len + 3 * (src_len / 128 KiB + 1) + 13). */
int obgpu_writer_zstd_compress(const void *src, int64_t src_len, void *out, int64_t out_cap, int64_t *out_len);
/* One zlib stream (RFC 1950 / RFC 1951; what uncompress and ObZlibCompressor::decompress read): header 78 01, the payload in
 * segments of >= 32 KiB of input (whole symbols), each one fixed-Huffman block from the LZ4 compressor's greedy matcher
 * (matches farther than 32 KiB stay literals, longer ones than 258 bytes are split) or, where that does not shrink it, one
 * stored block; the Adler-32 trailer. out == NULL: only *out_len (never more than src_len + 5 * (src_len / 32 KiB + 1) + 7). */
int obgpu_writer_zlib_compress(const void *src, int64_t src_len, void *out, int64_t out_cap, int64_t *out_len);
/* Re-frames n plain micro-blocks (data_zlength_ == data_length_) into stored form with `compressor` (OBGPU_COMPRESSOR_LZ4 /
 * LZ4_1_9_1: an LZ4 block; ZLIB: a zlib stream, obgpu_writer_zlib_compress; ZSTD_1_3_8: a zstd frame,
 * obgpu_writer_zstd_compress; NONE copies): the payload is compressed and kept raw when that is not smaller; a compressed block gets
 * data_zlength_, data_checksum_ (crc32c of the stored bytes) and a recomputed header checksum. Block i goes to
 * out[out_offsets[i], out_offsets[i] + out_sizes[i]), offsets multiples of align (a power of two; 1: back to back).
 * out_cap >= sum over i of (sizes[i] rounded up to align) always suffices; *out_size = bytes used. */
int obgpu_writer_compress_blocks(const void *image, const int64_t *offsets, const int64_t *sizes, int32_t n_blocks, int32_t compressor,
                                 int64_t align, void *out, int64_t out_cap, int64_t *out_offsets, int64_t *out_sizes,
                                 int64_t *out_size);

int obgpu_writer_set_cs_stream_encoding(int32_t mode);
/* The codec bytes alone (no ObIntegerStreamMeta) for count values of width_bytes (low bytes of vals[i]); type 0 =
 * detect. out == NULL: only *out_len. Byte-exact with the reference encoders (ObCodec::encode). */
int obgpu_writer_stream_encode(int32_t type, int32_t width_bytes, const uint64_t *vals, int64_t count, void *out,
                               int64_t out_cap, int64_t *out_len);

#ifdef __cplusplus
}
#endif
#endif /* OBGPU_WRITER_H_ */
