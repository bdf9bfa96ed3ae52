/*
 * obgpu_scan.h -- C-ABI of the H100-native columnar-scan path (libobgpu_scan.so).
 *
 * This is the drop-in boundary for OceanBase's micro-block decode / pushed-down filter /
 * projection path.  The reference has no C plugin ABI for storage operators (SURVEY.md 8b): the
 * path sits behind C++ abstract classes.  Every entry point below therefore names the reference
 * C++ method it stands in for; the thin C++ adapter (oceanbase_b200/host/) and the binding a
 * maintainer would add inside the reference tree (INTEGRATION.md) translate 1:1.
 *
 * Conventions (match the reference, deps/oblib/src/lib/ob_errno.h):
 *   - every function returns int: 0 == OB_SUCCESS, negative OB_* codes otherwise; no exceptions;
 *   - OBGPU_NOT_SUPPORTED means "caller falls back to its retrograde path", exactly like
 *     ObMicroBlockDecoder::filter_pushdown_filter (encoding/ob_micro_block_decoder.cpp:1734-1747);
 *   - plain pointers and sizes only; output buffers are caller-owned;
 *   - handles are not thread-safe; one ctx per worker thread (one CUDA stream each), many ctxs may
 *     run concurrently (ObIMicroBlockReader: one reader per scanner per worker thread).
 *   - there is NO CPU fallback: if no CUDA device is usable every call fails with OBGPU_ERR_SYS.
 */
#ifndef OBGPU_SCAN_H_
#define OBGPU_SCAN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- error codes: values of the reference's OB_* codes (lib/ob_errno.h:27-108) ------------- */
#define OBGPU_SUCCESS 0
#define OBGPU_ERROR (-4000)
#define OBGPU_INVALID_ARGUMENT (-4002)
#define OBGPU_INIT_TWICE (-4005)
#define OBGPU_NOT_INIT (-4006)
#define OBGPU_NOT_SUPPORTED (-4007)
#define OBGPU_ITER_END (-4008)
#define OBGPU_ALLOCATE_MEMORY_FAILED (-4013)
#define OBGPU_INNER_STAT_ERROR (-4014)
#define OBGPU_ERR_SYS (-4015)
#define OBGPU_ERR_UNEXPECTED (-4016)
#define OBGPU_SIZE_OVERFLOW (-4019)
#define OBGPU_BUF_NOT_ENOUGH (-4024)
#define OBGPU_INVALID_DATA (-4070)
#define OBGPU_PHYSIC_CHECKSUM_ERROR (-4108)

/* ---- sql::ObWhiteFilterOperatorType (sql/engine/basic/ob_pushdown_filter.h:388-401) --------- */
enum {
  OBGPU_WHITE_OP_EQ = 0,
  OBGPU_WHITE_OP_LE = 1,
  OBGPU_WHITE_OP_LT = 2,
  OBGPU_WHITE_OP_GE = 3,
  OBGPU_WHITE_OP_GT = 4,
  OBGPU_WHITE_OP_NE = 5,
  OBGPU_WHITE_OP_BT = 6,
  OBGPU_WHITE_OP_IN = 7,
  OBGPU_WHITE_OP_NU = 8,
  OBGPU_WHITE_OP_NN = 9,
  OBGPU_WHITE_OP_MAX = 10
};

/* ---- ObColumnHeader::Type (blocksstable/ob_block_sstable_struct.h:203-216) ------------------ */
enum {
  OBGPU_ENC_RAW = 0,
  OBGPU_ENC_DICT = 1,
  OBGPU_ENC_RLE = 2,
  OBGPU_ENC_CONST = 3,
  OBGPU_ENC_INTEGER_BASE_DIFF = 4,
  OBGPU_ENC_STRING_DIFF = 5,
  OBGPU_ENC_HEX_PACKING = 6,
  OBGPU_ENC_STRING_PREFIX = 7,
  OBGPU_ENC_COLUMN_EQUAL = 8,   /* span columns: obgpu_col_input.ref_col names the referenced column */
  OBGPU_ENC_COLUMN_SUBSTR = 9,
  /* writer only: columns of a CS_ENCODING_ROW_STORE block (ObCSColumnHeader::Type) */
  OBGPU_ENC_CS_INTEGER = 16,
  OBGPU_ENC_CS_INT_DICT = 17,
  OBGPU_ENC_CS_STRING = 18,
  OBGPU_ENC_CS_STR_DICT = 19,
  /* writer only: the codec of the column is chosen per micro-block the way ObMicroBlockEncoder::choose_encoder does
   * (encoding/ob_micro_block_encoder.cpp:1318-1366,1603-1823) among RAW / DICT / RLE / CONST / INTEGER_BASE_DIFF */
  OBGPU_ENC_AUTO = 32,
  /* writer only, CS blocks: INTEGER vs INT_DICT / STRING vs STR_DICT per micro-block like ObMicroBlockCSEncoder::choose_encoder_
   * (cs_encoding/ob_micro_block_cs_encoder.cpp:2246-2375) from the column encoders' estimate_store_size() */
  OBGPU_ENC_CS_AUTO = 33
};

/* ---- common::ObCompressorType values the path accepts (lib/compress/ob_compress_util.h) ------
 * LZ4 ("lz4_1.0") and LZ4_1_9_1 ("lz4_1.9.1") both store the plain LZ4 block format per micro-block payload;
 * ZLIB ("zlib_1.0", OceanBase's high-ratio option) stores one zlib stream (RFC 1950 around RFC 1951 DEFLATE) per payload;
 * ZSTD_1_3_8 ("zstd_1.3.8", the default table compression of OceanBase 4.x) stores one plain zstd frame (RFC 8878) per
 * payload. ZSTD ("zstd_1.0", 5) is not accepted. */
enum {
  OBGPU_COMPRESSOR_NONE = 1,
  OBGPU_COMPRESSOR_LZ4 = 2,
  OBGPU_COMPRESSOR_ZLIB = 4,
  OBGPU_COMPRESSOR_ZSTD_1_3_8 = 6,
  OBGPU_COMPRESSOR_LZ4_1_9_1 = 7
};

/* ---- ObObjType values the path accepts (common/object/ob_obj_type.h) ------------------------ */
enum {
  OBGPU_OBJ_TINYINT = 1, OBGPU_OBJ_SMALLINT = 2, OBGPU_OBJ_MEDIUMINT = 3, OBGPU_OBJ_INT32 = 4,
  OBGPU_OBJ_INT = 5, OBGPU_OBJ_UTINYINT = 6, OBGPU_OBJ_USMALLINT = 7, OBGPU_OBJ_UMEDIUMINT = 8,
  OBGPU_OBJ_UINT32 = 9, OBGPU_OBJ_UINT64 = 10, OBGPU_OBJ_DATETIME = 17, OBGPU_OBJ_TIMESTAMP = 18,
  OBGPU_OBJ_DATE = 19, OBGPU_OBJ_TIME = 20, OBGPU_OBJ_YEAR = 21, OBGPU_OBJ_VARCHAR = 22,
  OBGPU_OBJ_CHAR = 23
};

typedef struct obgpu_ctx obgpu_ctx;       /* per worker thread: device, stream, staging arenas */
typedef struct obgpu_batch obgpu_batch;   /* a page batch: N micro-blocks resident in HBM       */
typedef struct obgpu_result obgpu_result; /* device-resident result of one fused scan           */

/* common::ObDatum (share/datum/ob_datum.h:109-177): 12 packed bytes */
#pragma pack(push, 1)
typedef struct obgpu_datum {
  uint64_t ptr;
  uint32_t pack; /* len:29 | flag:2 | null:1 */
} obgpu_datum;
#pragma pack(pop)
#define OBGPU_DATUM_NULL_BIT 0x80000000u

/* =============================================================================================
 * Context
 * ============================================================================================= */
int obgpu_ctx_create(int device, obgpu_ctx **out);
void obgpu_ctx_destroy(obgpu_ctx *ctx);
/* Use an existing CUDA stream (cudaStream_t as void*) instead of the ctx-owned one, e.g. torch's
 * current stream so that torch.cuda.Event timing sees the kernels. NULL restores the owned stream. */
int obgpu_ctx_set_stream(obgpu_ctx *ctx, void *cuda_stream);
int obgpu_ctx_synchronize(obgpu_ctx *ctx);
/* Last CUDA / validation error text for this ctx (never NULL). */
const char *obgpu_ctx_last_error(const obgpu_ctx *ctx);
/* Number of kernels this ctx has launched so far (bench.py's gpu_launches). */
int64_t obgpu_ctx_launch_count(const obgpu_ctx *ctx);
/* Kernel timing: when enabled, a CUDA event pair is recorded on the ctx stream around every
 * obgpu_scan kernel launch; obgpu_ctx_kernel_times synchronises and returns the durations (ms) of
 * the most recent launches, oldest first (ring of 256). */
int obgpu_ctx_set_profiling(obgpu_ctx *ctx, int32_t enable);
int obgpu_ctx_kernel_times(obgpu_ctx *ctx, float *ms, int32_t cap, int32_t *n);

/* =============================================================================================
 * Page batch = what ObSSTableRowScanner::open_cur_data_block hands to the reader one block at a
 * time (access/ob_sstable_row_scanner.cpp:256; ObIMicroBlockReader::init,
 * blocksstable/ob_imicro_block_reader.h:295), submitted many blocks per call.
 *
 * `image` holds n reference-format PAX micro-blocks (post-decompress ObMicroBlockData buffers);
 * block i occupies [offsets[i], offsets[i] + sizes[i]). offsets must be 16-byte aligned (the
 * blocks are moved with TMA bulk copies). image_on_device == 0: host memory (pinned for
 * asynchronous copies), copied to HBM here; != 0: already a device pointer that outlives the
 * batch (block cache resident in HBM) -- only the descriptor tables are uploaded.
 * Headers are validated on the host (magic, version, row store type, sizes) the way
 * ObMicroBlockHeader::is_valid / get_micro_metas do (ob_micro_block_header.cpp:53-61,
 * encoding/ob_micro_block_decoder.cpp:363-388); `header_view` (optional, host memory, same
 * layout as image) lets the caller keep a host copy of a device-resident image for that parse.
 * A device-resident image with header_view == NULL is validated by a header survey kernel on the
 * device instead (same checks, one small device-to-host copy of the row / column counts).
 * ============================================================================================= */
int obgpu_batch_open(obgpu_ctx *ctx, const void *image, int64_t image_size,
                     const int64_t *offsets, const int64_t *sizes, int32_t n_blocks,
                     int32_t image_on_device, const void *header_view, obgpu_batch **out);
void obgpu_batch_close(obgpu_batch *batch);
/* ObIMicroBlockReader::get_row_count / column count for block i; total over the batch. */
int obgpu_batch_block_info(const obgpu_batch *batch, int32_t block, int64_t *row_count,
                           int32_t *column_count);
int obgpu_batch_total_rows(const obgpu_batch *batch, int64_t *total_rows);
/* Disk-format bytes into the block cache: n_macro_blocks macro blocks of macro_block_size bytes each (ObMacroBlock,
 * blocksstable/ob_macro_block.cpp:455-520: ObMacroBlockCommonHeader, ObSSTableMacroBlockHeader, micro-blocks back to back) are
 * validated and walked ON THE DEVICE (ObMacroBlockCommonHeader::check_integrity ob_macro_block_common_header.cpp:54-69,
 * FixedHeader::is_valid ob_sstable_macro_block_header.cpp:118-140, the micro headers' header_size_ + data_zlength_ chain) and
 * their micro-blocks re-laid into an aligned image that the returned page batch owns -- what ObMacroBlockReader /
 * ObMicroBlockBareIterator (blocksstable/ob_micro_block_bare_iterator.cpp) do block by block on the CPU. The macro image may be
 * host memory (copied once) or device memory. Macro blocks whose compressor_type_ is OBGPU_COMPRESSOR_LZ4 / LZ4_1_9_1 /
 * ZLIB / ZSTD_1_3_8 are decoded on the device as obgpu_batch_open_compressed does (raw and compressed micro-blocks may be mixed; the
 * macro blocks of one call that are not NONE must share one compressor, as one SSTable has one, else OBGPU_NOT_SUPPORTED);
 * other compressors and encrypted macro blocks: OBGPU_NOT_SUPPORTED; broken headers, chains, checksums of compressed
 * micro-blocks, LZ4 streams, zlib streams or zstd frames: OBGPU_INVALID_DATA. The macro payload checksum is not re-computed here (the IO layer's job in the reference).
 * The batch owns its re-laid image: string pointers of a scan are string_base + offset inside THAT image
 * (obgpu_batch_device_image). */
int obgpu_batch_open_macro_blocks(obgpu_ctx *ctx, const void *macro_image, int64_t image_size, int64_t macro_block_size,
                                  int32_t n_macro_blocks, int32_t image_on_device, obgpu_batch **out, int32_t *n_micro_out);
/* Compressed micro-blocks: ObMacroBlockReader::decompress_data (blocksstable/ob_macro_block_reader.cpp) for a whole page batch,
 * on the device. Block i is [offsets[i], offsets[i] + sizes[i]) of `image` in STORED form (plain ObMicroBlockHeader, payload
 * of data_zlength_ bytes; any byte offset); compressor_type is the SSTable's (the reference takes it from the SSTable meta).
 * A block with data_zlength_ == data_length_ is stored raw and copied; the others are decoded (OBGPU_COMPRESSOR_LZ4 and
 * LZ4_1_9_1: the plain LZ4 block format; ZLIB: one zlib stream, obgpu_zlib_decompress; ZSTD_1_3_8: one zstd frame,
 * obgpu_zstd_decompress) after their header checksum and
 * payload checksum (crc32c of the stored bytes == data_checksum_) are checked. Every decoded block goes to a 128-byte aligned slot of a new device image that the
 * batch owns; the decoded copy keeps the stored header unchanged. image_on_device: as obgpu_batch_open (a device image must be
 * 16-byte aligned; a host image is copied once).
 *   OBGPU_COMPRESSOR_NONE : every block must have data_zlength_ == data_length_, else OBGPU_INVALID_DATA
 *   other compressors     : OBGPU_NOT_SUPPORTED
 *   a bad header, checksum, LZ4 stream, zlib stream or zstd frame: OBGPU_INVALID_DATA; the ctx stays usable.
 * String pointers of a scan are string_base + offset inside the batch's image (obgpu_batch_device_image). */
int obgpu_batch_open_compressed(obgpu_ctx *ctx, const void *image, int64_t image_size, const int64_t *offsets,
                                const int64_t *sizes, int32_t n_blocks, int32_t image_on_device, int32_t compressor_type,
                                obgpu_batch **out);
/* The device image the batch's blocks live in and its size. For a batch that owns its image (opened from host memory, from
 * macro blocks or from compressed blocks), scan string pointers are string_base + offset in this image: string_base = *image
 * makes them device addresses. */
int obgpu_batch_device_image(const obgpu_batch *batch, const void **image, int64_t *image_size);
/* ObLZ4Compressor::decompress (LZ4_decompress_safe into a buffer of the expected size) for n independent LZ4 blocks in device
 * memory: d_in[in_off[i], + in_len[i]) -> d_out[out_off[i], + out_len[i]) (offset / length tables in host memory). status[i]
 * (host, n entries) is 0 when block i decoded to exactly out_len[i] bytes, non-zero when its stream is malformed (reads are
 * kept inside the input extent and writes inside the output extent either way). Returns OBGPU_INVALID_DATA when some block
 * failed. */
int obgpu_lz4_decompress(obgpu_ctx *ctx, const void *d_in, const int64_t *in_off, const int64_t *in_len, void *d_out,
                         const int64_t *out_off, const int64_t *out_len, int32_t n, int32_t *status);
/* ObZstdCompressor_1_3_8::decompress (ZSTD_decompressDCtx into a buffer of the expected size) for n independent zstd frames
 * (RFC 8878) in device memory, with the contract of obgpu_lz4_decompress: status[i] == 0 when d_in[in_off[i], + in_len[i]) is
 * exactly one frame that decodes to exactly out_len[i] bytes. Refused besides malformed frames: a dictionary ID, skippable
 * frames, bytes after the first frame, reserved bits and block types (DESIGN 3.14 lists where this is stricter than
 * libzstd). */
int obgpu_zstd_decompress(obgpu_ctx *ctx, const void *d_in, const int64_t *in_off, const int64_t *in_len, void *d_out,
                          const int64_t *out_off, const int64_t *out_len, int32_t n, int32_t *status);
/* ObZlibCompressor::decompress (zlib's uncompress into a buffer of the expected size) for n independent zlib streams
 * (RFC 1950 / RFC 1951) in device memory, with the contract of obgpu_lz4_decompress: status[i] == 0 when
 * d_in[in_off[i], + in_len[i]) is exactly one zlib stream, its Adler-32 included, that decodes to exactly out_len[i] bytes.
 * Refused besides what zlib's inflate refuses: a preset dictionary (FDICT), bytes after the Adler-32, which uncompress
 * ignores, and a stream or output longer than 0x7fff0000 bytes (DESIGN 3.16). */
int obgpu_zlib_decompress(obgpu_ctx *ctx, const void *d_in, const int64_t *in_off, const int64_t *in_len, void *d_out,
                          const int64_t *out_off, const int64_t *out_len, int32_t n, int32_t *status);

/* =============================================================================================
 * Filter tree = sql::ObPushdownFilterExecutor tree flattened in post-order
 * (sql/engine/basic/ob_pushdown_filter.cpp:1551-1624): leaves are ObWhiteFilterExecutor
 * (op, one column, constants), inner nodes AND / OR over their n_children preceding sub-results.
 * ============================================================================================= */
enum { OBGPU_NODE_WHITE = 0, OBGPU_NODE_AND = 1, OBGPU_NODE_OR = 2 };

typedef struct obgpu_filter_param {
  int64_t i64;      /* integer-class constant (sign/zero extended to 64 bit by the caller)   */
  const char *ptr;  /* string-class constant                                                 */
  uint32_t len;
  int32_t is_null;  /* NULL constant => leaf is all-false unless op is NU/NN
                       (encoding/ob_micro_block_decoder.cpp:1713-1715)                       */
} obgpu_filter_param;

typedef struct obgpu_filter_node {
  int32_t kind;        /* OBGPU_NODE_*                                                        */
  int32_t op;          /* leaf: OBGPU_WHITE_OP_*                                              */
  int32_t col;         /* leaf: column store index inside the micro-block (col_offsets.at(0)) */
  int32_t param_begin; /* leaf: first constant in obgpu_filter.params                          */
  int32_t n_params;    /* leaf: 1 (cmp), 2 (BT), k (IN), 0 (NU/NN)                             */
  int32_t n_children;  /* AND/OR: >= 2                                                        */
} obgpu_filter_node;

typedef struct obgpu_filter {
  const obgpu_filter_node *nodes; /* post-order, root last */
  int32_t n_nodes;
  const obgpu_filter_param *params;
  int32_t n_params;
} obgpu_filter;

/* =============================================================================================
 * Fused scan over the whole batch: filter (ObMicroBlockDecoder::filter_pushdown_filter,
 * encoding/ob_micro_block_decoder.cpp:1680) -> selection bitmap (common::ObBitmap) -> row ids
 * (ObBitmap::get_row_ids, lib/container/ob_bitmap.cpp:540) -> projection
 * (ObMicroBlockDecoder::get_rows / decode_vector, :2473) in ONE kernel, blocks in index order,
 * rows ascending inside a block. Output is dense over the selected rows of the batch.
 * ============================================================================================= */
typedef struct obgpu_scan_spec {
  const obgpu_filter *filter;  /* NULL: no predicate, every row selected                       */
  const int32_t *proj_cols;    /* column store indexes to project                              */
  int32_t n_proj;
  int32_t want_row_ids;        /* also emit block-relative int32 row ids of the selected rows  */
  uint64_t string_base;        /* address string pointers are rebased to: ptr = string_base +
                                  byte offset of the cell inside `image` (VEC_DISCRETE ptrs_
                                  point into the caller's block buffer, rule 8c.6)             */
  int64_t max_selected_rows;   /* capacity of the dense output in rows; 0 = every row of the
                                  batch. If the filter selects more, obgpu_result_info_get
                                  returns OBGPU_BUF_NOT_ENOUGH with the needed selected_rows
                                  filled in and the caller re-runs with a larger capacity.    */
} obgpu_scan_spec;

int obgpu_scan(obgpu_batch *batch, const obgpu_scan_spec *spec, obgpu_result **out);
void obgpu_result_free(obgpu_result *res);

typedef struct obgpu_result_info {
  int64_t total_rows;     /* input rows scanned                                  */
  int64_t selected_rows;  /* rows passing the filter                             */
  int32_t n_blocks;
  int32_t n_proj;
} obgpu_result_info;

/* Synchronises the ctx stream and reads back the totals. */
int obgpu_result_info_get(obgpu_result *res, obgpu_result_info *info);

/* Column i of the projection, device pointers (valid until obgpu_result_free):
 *   integer class : data = elem_len-byte values [selected_rows] (VEC_FIXED data_), aux = NULL
 *   string class  : data = uint64 pointers [selected_rows] (VEC_DISCRETE ptrs_), aux = int32 lens_
 *   nulls         : sql::ObBitVector image, LSB-first uint64 words over the dense row index
 * For a NULL row the payload slot is zero (the reference leaves it unwritten, rule 8c.1). */
typedef struct obgpu_result_col {
  void *data;
  void *aux;
  uint64_t *nulls;
  int32_t elem_len;   /* 8 / 4 / 1 for integer classes, 8 (pointer) for strings */
  int32_t is_string;
  int32_t has_null;   /* valid after obgpu_result_info_get */
  int32_t obj_type;
} obgpu_result_col;
int obgpu_result_col_get(obgpu_result *res, int32_t i, obgpu_result_col *col);

/* Per-block prefix of selected rows: sel_offset[b] .. sel_offset[b+1] is block b's slice of the
 * dense output (n_blocks + 1 int64 entries, device pointer), plus the packed per-block selection
 * bitmap (bit r of block b at word bitmap_word_offset[b] + r/32, uint32 words, LSB first). */
int obgpu_result_block_tables(obgpu_result *res, const int64_t **sel_offset_dev,
                              const uint32_t **bitmap_words_dev,
                              const int64_t **bitmap_word_offset_dev, const int32_t **row_ids_dev);

/* Device -> host copies of a dense window [row_begin, row_begin + row_count) of column i.
 * host_aux / host_nulls may be NULL. host_nulls receives (row_count + 63) / 64 words re-based so
 * that bit 0 is row_begin. */
int obgpu_result_fetch_col(obgpu_result *res, int32_t i, int64_t row_begin, int64_t row_count,
                           void *host_data, void *host_aux, uint64_t *host_nulls);
/* Rows [row_begin, row_begin + row_count) of projected column i as ObDatum[] (datum format of the batch result):
 * formatted on the device, one copy back. Integer classes: host_slots receives 8 bytes per row (value in the low
 * datum-length bytes) and datum k points at host_slots + 8 k; strings: ptr / len as in obgpu_project_datums
 * (host_slots may be NULL). */
int obgpu_result_fetch_datums(obgpu_result *result, int32_t i, int64_t row_begin, int64_t row_count,
                              obgpu_datum *host_datums, void *host_slots);
/* Same for several columns with ONE stream synchronisation (all copies are enqueued first): cols[k]
 * goes to host_data[k] / host_aux[k] / host_nulls[k]; any of the three arrays (or entries) may be NULL. */
int obgpu_result_fetch_cols(obgpu_result *res, int32_t n_cols, const int32_t *cols, int64_t row_begin,
                            int64_t row_count, void *const *host_data, void *const *host_aux,
                            uint64_t *const *host_nulls);
int obgpu_result_fetch_sel_offsets(obgpu_result *res, int64_t *host_sel_offset /* n_blocks+1 */);
int obgpu_result_fetch_row_ids(obgpu_result *res, int64_t row_begin, int64_t row_count,
                               int32_t *host_row_ids);
/* common::ObBitmap image (one byte 0x00/0x01 per row) of block b, rows [start, start+count). */
int obgpu_result_fetch_bitmap(obgpu_result *res, int32_t block, int64_t start, int64_t count,
                              uint8_t *host_bitmap_bytes);

/* Pushed-down aggregates over the selected rows of a scan (the reference folds them batch by batch in
 * ObAggregatedStoreVec / ObPushdownAggregateVec, access/ob_aggregated_store_vec.h:143,
 * access/ob_pushdown_aggregate_vec.cpp): computed on the device from the dense projected columns,
 * exact integer arithmetic. NULL rows are skipped (a product is NULL when either side is).
 *   COUNT       : out[0] = rows where col_a is not NULL
 *   SUM         : out[0..1] = 128-bit two's-complement sum of col_a (low, high word)
 *   SUM_PRODUCT : out[0..1] = 128-bit sum of col_a * col_b (each product taken in 128 bits)
 *   MIN / MAX   : out[0] = extreme of col_a in the column's own (signed / unsigned) order,
 *                 out[1] = 1 when at least one non-NULL row exists
 * col_a / col_b index the projection list of the scan (integer-class columns). */
enum {
  OBGPU_AGG_COUNT = 0,
  OBGPU_AGG_SUM = 1,
  OBGPU_AGG_SUM_PRODUCT = 2,
  OBGPU_AGG_MIN = 3,
  OBGPU_AGG_MAX = 4
};
int obgpu_result_aggregate(obgpu_result *res, int32_t kind, int32_t col_a, int32_t col_b, int64_t out[2]);

/* =============================================================================================
 * Reference-granularity calls (one micro-block, one leaf, one <=batch-size projection). They run
 * the same device code on a one-block batch; the adapter serves them from a prefetched batch.
 * ============================================================================================= */
/* ObIMicroBlockDecoder::filter_pushdown_filter(parent, ObWhiteFilterExecutor&, pd_filter_info,
 * result_bitmap) -- encoding/ob_imicro_block_decoder.h:27-73. result_bitmap: count bytes 0/1. */
int obgpu_filter_white(obgpu_batch *batch, int32_t block, int32_t col, int32_t op,
                       const obgpu_filter_param *params, int32_t n_params, int64_t start,
                       int64_t count, uint8_t *result_bitmap);
/* ObPushdownFilterExecutor::execute over a tree (ob_pushdown_filter.cpp:1551). */
int obgpu_filter_tree(obgpu_batch *batch, int32_t block, const obgpu_filter *filter,
                      int64_t start, int64_t count, uint8_t *result_bitmap);
/* common::ObBitmap::get_row_ids(row_ids, row_count, from, to, limit, id_offset)
 * (lib/container/ob_bitmap.cpp:540-561); *from is advanced like the reference does. */
int obgpu_bitmap_to_row_ids(obgpu_ctx *ctx, const uint8_t *bitmap, int64_t bitmap_size,
                            int64_t *from, int64_t to, int64_t limit, int64_t id_offset,
                            int32_t *row_ids, int64_t *row_count);
/* ObMicroBlockDecoder::get_rows -> ObIColumnDecoder::decode_vector into a VEC_FIXED vector
 * (encoding/ob_micro_block_decoder.cpp:2473-2544): data[(vec_offset + i) * elem_len] = value of
 * row_ids[i]; nulls = ObBitVector words (bit vec_offset + i). */
int obgpu_project_fixed(obgpu_batch *batch, int32_t block, int32_t col, const int32_t *row_ids,
                        int64_t row_cap, int64_t vec_offset, void *data, int32_t elem_len,
                        uint64_t *nulls, int32_t *has_null);
/* ... into a VEC_DISCRETE vector: ptrs[vec_offset + i] = string_base + cell offset in image. */
int obgpu_project_discrete(obgpu_batch *batch, int32_t block, int32_t col, const int32_t *row_ids,
                           int64_t row_cap, int64_t vec_offset, uint64_t string_base,
                           uint64_t *ptrs, int32_t *lens, uint64_t *nulls, int32_t *has_null);

/* ---- datum format (ObMicroBlockDecoder::get_rows into ObDatum[], encoding/ob_micro_block_decoder.cpp:2100-2140,
 * get_col_datums :2201-2237): common::ObDatum is 12 packed bytes -- 8-byte pointer + {len:29, flag:2, null:1}
 * (share/datum/ob_datum.h:109-177). Integer classes: the caller's datums already point at their reserved 8-byte
 * slots (the expression's datum buffer); the value is written THROUGH datum.ptr with the datum length of the type
 * (8 / 4 / 1) like load_data_to_datum. Strings: ptr = string_base + offset of the cell in the caller's image, len set.
 * NULL: ObDatum::set_null() (len 0, null 1; ptr untouched). */
int obgpu_project_datums(obgpu_batch *batch, int32_t block, int32_t col, const int32_t *row_ids,
                         int64_t row_cap, int64_t datum_offset, uint64_t string_base, obgpu_datum *datums);

/* =============================================================================================
 * Dictionary surface of one micro-block (pushdown GROUP BY, black filter on one dictionary column).
 * A column is "dictionary coded" in a block when its encoding is DICT / RLE / CONST (PAX) or INT_DICT / STR_DICT (CS);
 * otherwise the calls return OBGPU_NOT_SUPPORTED, the condition under which the reference falls back too
 * (ObIMicroBlockReader::can_apply_black, ob_micro_block_decoder.h:332-337; ObAggGroupByDecoder: group by needs
 * ObDictDecoder, ob_pushdown_aggregate.cpp check_column_can_group_by).
 * ============================================================================================= */
/* Column `col` (store index) of the batch: its ObObjType as the column headers carry it (0xff when the blocks of the batch
 * disagree) and the datum length of its class: 8 / 4 / 1 for integer classes, 0 for strings (the length is per cell). */
int obgpu_batch_column_type(const obgpu_batch *batch, int32_t col, int32_t *obj_type, int32_t *datum_len);
/* ObIMicroBlockReader::get_distinct_count(group_by_col, distinct_cnt) (ob_micro_block_decoder.cpp:2263-2278,
 * ObDictDecoder::get_distinct_count ob_dict_decoder.cpp:1681-1686). */
int obgpu_block_distinct_count(obgpu_batch *batch, int32_t block, int32_t col, int64_t *count);
/* ObIMicroBlockReader::read_distinct (ob_micro_block_decoder.cpp:2280-2304; ObDictDecoder::batch_read_distinct
 * ob_dict_decoder.cpp:1708-1790): entry i of the dictionary in dictionary order. Integer classes: vals[i] = value image
 * (low datum-length bytes significant); strings: vals[i] = string_base + offset of the cell in the caller's image,
 * lens[i] its length. *count is always set; OBGPU_BUF_NOT_ENOUGH when it exceeds cap. */
int obgpu_block_read_distinct(obgpu_batch *batch, int32_t block, int32_t col, uint64_t string_base, uint64_t *vals,
                              int32_t *lens, int64_t cap, int64_t *count);
/* ObIMicroBlockReader::read_reference (ob_micro_block_decoder.cpp:2306-2330; ObDictDecoder::read_reference
 * ob_dict_decoder.cpp:1792-1830): refs[i] = dictionary reference of row row_ids[i]; NULL rows give the distinct count
 * (the reference's "ref == dict count means NULL"). */
int obgpu_block_read_reference(obgpu_batch *batch, int32_t block, int32_t col, const int32_t *row_ids, int64_t row_cap,
                               uint32_t *refs);
/* ObMicroBlockDecoder::filter_black_filter_batch on a single dictionary column (ob_micro_block_decoder.cpp:1822-1859
 * -> ObDictDecoder::pushdown_operator for ObBlackFilterExecutor): the caller evaluates its expression once per distinct
 * value (obgpu_block_read_distinct) and passes the verdicts; rows [start, start + count) whose ref passes get
 * result_bitmap[i] = 1, NULL rows get null_pass. n_entries must equal the block's distinct count. */
int obgpu_filter_dict_pass(obgpu_batch *batch, int32_t block, int32_t col, const uint8_t *entry_pass, int64_t n_entries,
                           int32_t null_pass, int64_t start, int64_t count, uint8_t *result_bitmap);
/* Pushdown GROUP BY (ObIMicroBlockReader::get_group_by_aggregate_result, ob_micro_block_decoder.cpp:2332-2400;
 * ObGroupByCell::eval_batch): rows are grouped by the ref of group_col (group g = dictionary entry g of the block,
 * group == distinct count: the NULL group) and every aggregate is folded per group.
 *   kind COUNT with col < 0: COUNT(*); COUNT(col): non-NULL rows; SUM / MIN / MAX as obgpu_result_aggregate.
 * host_out is [n_aggs][groups][2] int64 (pairs as obgpu_result_aggregate's out[2]); cols are STORE indexes of
 * integer-class columns. */
typedef struct obgpu_group_agg {
  int32_t kind; /* OBGPU_AGG_COUNT / SUM / MIN / MAX */
  int32_t col;
} obgpu_group_agg;
/* one block, the rows of row_ids (the reference call shape); *n_groups = distinct count + 1 */
int obgpu_block_group_by(obgpu_batch *batch, int32_t block, int32_t group_col, const obgpu_group_agg *aggs, int32_t n_aggs,
                         const int32_t *row_ids, int64_t row_cap, int64_t *host_out, int64_t out_cap_groups,
                         int64_t *n_groups);
/* every block of a scan, the rows its filter selected, ONE launch: block b's groups are
 * [host_group_off[b], host_group_off[b + 1]) of the group axis (host_group_off: n_blocks + 1 entries, may be NULL). */
int obgpu_result_group_by(obgpu_result *res, int32_t group_col, const obgpu_group_agg *aggs, int32_t n_aggs,
                          int64_t *host_group_off, int64_t *host_out, int64_t out_cap_groups, int64_t *total_groups);

/* =============================================================================================
 * String cells as BYTES. HEX_PACKING / STRING_DIFF / STRING_PREFIX columns rebuild their values (ObHexStringDecoder,
 * ObStringDiffDecoder, ObStringPrefixDecoder decode into allocator memory, encoding/ob_hex_string_decoder.cpp:33-127 ...): such a
 * value is not part of the caller's block, so the (pointer, length) outputs of obgpu_scan / obgpu_project_discrete cannot address
 * it. The device rebuilds these columns once per page batch (at obgpu_batch_open); filters and aggregates over them work like on
 * any string column; their BYTES come back through the two calls below (which work for every string column).
 * ============================================================================================= */
/* 1 when some block of the batch holds column `col` in one of those codecs (its projected pointers are then not usable). */
int obgpu_batch_column_materialised(const obgpu_batch *batch, int32_t col, int32_t *materialised);
/* Rows [row_begin, row_begin + row_count) of projected string column i of a scan: host_off[k] .. host_off[k + 1] of host_heap are the
 * bytes of row k (NULL rows: empty; the NULL bits come from obgpu_result_fetch_col). *heap_bytes is always set; OBGPU_BUF_NOT_ENOUGH
 * when it exceeds heap_cap (host_off is valid then: call again with a larger heap). */
int obgpu_result_fetch_strings(obgpu_result *res, int32_t i, int64_t row_begin, int64_t row_count, void *host_heap,
                               int64_t heap_cap, int64_t *host_off, int64_t *heap_bytes);
/* Bytes the cells of rows [row_begin, row_begin + row_count) of projected string columns cols[0..n) take: bytes[j] for column
 * cols[j]. NULL rows take 0. Keeps the per-row offsets on the device with the result for the next call. Three kernel launches and
 * one synchronisation, whatever n and row_count. */
int obgpu_result_string_bytes(obgpu_result *res, int32_t n, const int32_t *cols, int64_t row_begin, int64_t row_count,
                              int64_t *bytes);
/* The previous call's rows and columns: the bytes of column cols[j] go to host_heap[j] (exactly bytes[j] bytes).
 * host_ptrs[j][k] is set to the host address of row k's bytes inside host_heap[j], or 0 for a NULL row (an empty string gets
 * an address). host_ptrs and its entries may be NULL. Another (cols, rows) than the last obgpu_result_string_bytes call:
 * OBGPU_INVALID_ARGUMENT. One kernel launch (the device writes the host addresses), then one copy of heap bytes and one of
 * pointers per column. */
int obgpu_result_fetch_string_heap(obgpu_result *res, int32_t n, const int32_t *cols, int64_t row_begin, int64_t row_count,
                                   void *const *host_heap, uint64_t *const *host_ptrs);
/* One block, the rows of row_ids (the reference call shape of a VEC_DISCRETE / VEC_CONTINUOUS decode): same outputs + the
 * ObBitVector NULL image (host_nulls, has_null may be NULL). */
int obgpu_project_strings(obgpu_batch *batch, int32_t block, int32_t col, const int32_t *row_ids, int64_t row_cap,
                          void *host_heap, int64_t heap_cap, int64_t *host_off, uint64_t *host_nulls, int32_t *has_null,
                          int64_t *heap_bytes);

/* =============================================================================================
 * Column groups (column-store tables: every column group is its own SSTable with its own micro-blocks). The reference evaluates
 * each pushed-down filter on ITS column group (ObCGScanner::apply_filter, column_store/ob_cg_scanner.cpp:273), combines the groups'
 * results in an ObCGBitmap over the row range (column_store/ob_cg_bitmap.h: bit_and / bit_or / set_bitmap at start_row_id
 * offsets) and projects the other groups by that bitmap (ObCGRowScanner::get_next_rows(count, capacity, bitmap), :614).
 * obgpu_cg_bitmap is that range bitmap, device resident; page batches of different groups (any block boundaries) meet in it.
 * All objects of one flow live on one ctx (stream).
 * ============================================================================================= */
typedef struct obgpu_cg_bitmap obgpu_cg_bitmap;
int obgpu_cg_bitmap_create(obgpu_ctx *ctx, int64_t n_rows, int32_t all_true, obgpu_cg_bitmap **out);
void obgpu_cg_bitmap_free(obgpu_cg_bitmap *bm);
enum { OBGPU_CG_SET = 0, OBGPU_CG_AND = 1, OBGPU_CG_OR = 2 };
/* The selection of a (filter) scan -> rows [row_offset, row_offset + rows of the result's batch) of the range bitmap. */
int obgpu_cg_bitmap_apply_result(obgpu_cg_bitmap *bm, obgpu_result *filter_result, int64_t row_offset, int32_t op);
int obgpu_cg_bitmap_popcnt(obgpu_cg_bitmap *bm, int64_t from, int64_t to, int64_t *count);
/* rows [from, from + count) as ObBitmap bytes (0x00 / 0x01) */
int obgpu_cg_bitmap_fetch(obgpu_cg_bitmap *bm, int64_t from, int64_t count, uint8_t *host_bitmap_bytes);
/* obgpu_scan whose selection is the range bitmap (spec->filter must be NULL): row r of the batch is selected when bit
 * row_offset + r of the bitmap is set. Results, per-block tables, aggregates, GROUP BY work as after a filter scan. */
int obgpu_scan_bitmap(obgpu_batch *batch, const obgpu_cg_bitmap *bm, int64_t row_offset, const obgpu_scan_spec *spec,
                      obgpu_result **out);

/* Library self-description (build id, arch) for logs. */
const char *obgpu_version(void);

#ifdef __cplusplus
}
#endif
#endif /* OBGPU_SCAN_H_ */
