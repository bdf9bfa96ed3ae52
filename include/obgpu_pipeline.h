/*
 * obgpu_pipeline.h -- host-buffer scan: micro-blocks in HOST memory in, vectors in HOST memory out.
 *
 * What ObSSTableRowScanner does per micro-block (open_cur_data_block -> ObIMicroBlockReader::init ->
 * filter -> get_rows, access/ob_sstable_row_scanner.cpp:256,553,594) happens here per PAGE BATCH of consecutive
 * blocks, pipelined over n_streams CUDA streams so that the host->device copy of batch i + 1, the kernels of batch i
 * and the device->host copy of batch i - 1 overlap in both PCIe directions. The C++ adapter
 * (oceanbase_b200/host/ObGpuSSTableBatchScanner) and bench.py's e2e leg call this entry.
 *
 * Outputs: the caller owns one buffer per projected column (+ lens for strings, + NULL words); page batch b gets the
 * rows [batch_row_begin[b], batch_row_begin[b] + batch_rows[b]) of each (its slice is sized by the selectivity
 * hint; results are dense inside a batch, batches in block order). Pushed-down aggregates (COUNT / SUM /
 * SUM(a*b) / MIN / MAX over projected columns) are folded on the device per batch and summed here: with
 * no_row_output only 16 bytes per aggregate and batch come back.
 */
#ifndef OBGPU_PIPELINE_H_
#define OBGPU_PIPELINE_H_

#include "obgpu_scan.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct obgpu_pipeline obgpu_pipeline;

typedef struct obgpu_host_agg {
  int32_t kind;   /* OBGPU_AGG_* */
  int32_t col_a;  /* index into proj_cols */
  int32_t col_b;  /* SUM_PRODUCT: second operand, else -1 */
} obgpu_host_agg;

typedef struct obgpu_host_scan_spec {
  const void *image;          /* host memory (pinned for full copy overlap), blocks 16-byte aligned (compressor_type 0) */
  int64_t image_size;
  const int64_t *offsets;     /* [n_blocks] */
  const int64_t *sizes;       /* [n_blocks] */
  int32_t n_blocks;
  const obgpu_filter *filter;
  const int32_t *proj_cols;
  int32_t n_proj;
  int32_t blocks_per_batch;   /* page batch size in blocks; 0: n_blocks / 12 */
  int32_t ramp;               /* the first `ramp` batches are 1/2^ramp .. 1/2 of a full one (results start flowing early) */
  double selectivity_hint;    /* expected selected / total rows (sizes each batch's output slice); <= 0: 1.0 */
  uint64_t string_base;       /* VEC_DISCRETE pointers = string_base + offset of the cell in `image` */
  const void *agg_rows;       /* optional skip index: serialized aggregate rows of the blocks ... */
  const int64_t *agg_off;     /* ... block b = agg_rows[agg_off[b], agg_off[b + 1]) */
  /* outputs (caller-owned, host; pinned for speed). May be NULL per column when no_row_output. */
  void *const *out_data;      /* [n_proj] elem_len-byte values, or uint64 string pointers */
  int32_t *const *out_lens;   /* [n_proj] string columns: int32 lengths (NULL entries for integer columns) */
  uint64_t *const *out_nulls; /* [n_proj] NULL words per BATCH SLICE: slice b starts at word batch_row_begin[b] / 64 (slices are 64-row aligned);
                               * the bits after the batch's last row in its last word are 0 */
  int64_t out_cap_rows;       /* rows each output buffer holds */
  int32_t *out_row_ids;       /* optional [out_cap_rows]: block-relative row id of every output row (ObBitmap::get_row_ids); placed in
                               * the batch slices as the columns are, with no_row_output or n_proj 0 too */
  int64_t *out_block_begin;   /* optional [n_blocks]: output row where block i's selected rows start ... */
  int64_t *out_block_count;   /* optional [n_blocks]: ... and how many there are */
  int32_t no_row_output;      /* 1: only aggregates (and counts) come back */
  const obgpu_host_agg *aggs;
  int32_t n_aggs;
  /* 1: do not stage the image in HBM. `image` must be pinned, device-accessible host memory (cudaHostAlloc / cudaHostRegister: with
   * unified addressing the same pointer is valid on the device); the kernels then pull only what they reference -- headers, the
   * filter columns' regions, the projected columns' regions -- straight over PCIe, instead of the library copying every byte of every
   * block first. Pays off when the scan references a fraction of the columns; CS blocks with encoded streams and HEX / STRING_DIFF /
   * STRING_PREFIX columns are still read in full once (their restatement at open). */
  int32_t zero_copy;
  /* 0: plain blocks, 16-byte aligned (as above). OBGPU_COMPRESSOR_NONE / LZ4 / LZ4_1_9_1 / ZLIB / ZSTD_1_3_8: the blocks are in
   * STORED form (plain ObMicroBlockHeader, payload of data_zlength_ bytes) at any byte offset, as they come from the IO buffers;
   * every page batch is opened by obgpu_batch_open_compressed (header and payload checksums checked, decoded in HBM). Projected
   * string columns then need a heap (out_heap): their decoded bytes exist only on the device. Other values and zero_copy with a
   * compressor: OBGPU_NOT_SUPPORTED before any batch is opened. */
  int32_t compressor_type;
  /* optional [n_proj]: string column c's bytes go to out_heap[c]; its out_data slots then hold host pointers into out_heap[c]
   * (0 for NULL rows) instead of pointers into `image`. Lifts the HEX_PACKING / STRING_DIFF / STRING_PREFIX refusal for that
   * column. NULL array or NULL entries: pointer mode. */
  void *const *out_heap;
  const int64_t *out_heap_cap; /* [n_proj] bytes each heap holds; a heap that overflows: OBGPU_BUF_NOT_ENOUGH */
  int64_t *out_heap_used;      /* optional [n_proj] out: bytes used (after OBGPU_BUF_NOT_ENOUGH: bytes claimed so far, a lower bound) */
} obgpu_host_scan_spec;

typedef struct obgpu_host_scan_result {
  int64_t total_rows, selected_rows;
  int32_t n_batches;
  int64_t *batch_row_begin;   /* caller array [n_batches_cap]: first output row of every batch (multiple of 64) */
  int64_t *batch_rows;        /* caller array [n_batches_cap]: selected rows of every batch */
  int32_t *batch_block_begin; /* caller array [n_batches_cap + 1] or NULL */
  int32_t n_batches_cap;
  int64_t agg_out[16][2];     /* per aggregate: SUM / SUM_PRODUCT 128-bit (lo, hi), COUNT (lo), MIN / MAX (value, seen) */
  int64_t h2d_bytes, d2h_bytes, kernel_launches;
} obgpu_host_scan_result;

int obgpu_pipeline_create(int device, int32_t n_streams, obgpu_pipeline **out);
void obgpu_pipeline_destroy(obgpu_pipeline *p);
const char *obgpu_pipeline_last_error(const obgpu_pipeline *p);
/* Number of page batches (and their first blocks) a spec is cut into: lets the caller size the result arrays. */
int obgpu_pipeline_plan(const obgpu_host_scan_spec *spec, int32_t *n_batches, int64_t *rows_cap_needed_hint);
int obgpu_pipeline_scan(obgpu_pipeline *p, const obgpu_host_scan_spec *spec, obgpu_host_scan_result *result);
/* GROUP BY group_cols (1..4 store indexes) over every row of the spec's table that its filter selects, with the groups of every
 * page batch merged on the device: each worker opens its batch as obgpu_pipeline_scan does, scans it with nothing projected,
 * groups it with obgpu_result_group_by_columns and adds the groups to one accumulator on the pipeline's first ctx (adds are
 * serialised). Only the groups reach the host, through *out (obgpu_groups_fetch), which the caller frees before destroying
 * the pipeline. The groups are those of obgpu_result_group_by_columns over the whole table as one batch.
 *   From spec: image, offsets, sizes, n_blocks, filter, blocks_per_batch, ramp, compressor_type, zero_copy, agg_rows / agg_off.
 *   It asks for no rows: no_row_output must be 1, out_row_ids, out_block_begin and out_block_count NULL, n_aggs 0; otherwise
 *   OBGPU_INVALID_ARGUMENT. result is filled as obgpu_pipeline_scan fills it, with batch_row_begin all 0, no aggregates and
 *   d2h_bytes 0.
 *   The 65 536-value cap of obgpu_result_group_by_values applies PER PAGE BATCH: a table whose dictionaries hold more distinct
 *   values in all is grouped as long as no batch's dictionaries do.
 *   The first refusal of any batch (a column not dictionary coded, more than 65 536 values in one batch's dictionaries, an
 *   over-long string key, a mismatch between batches' column types, ...) is returned, with its text in
 *   obgpu_pipeline_last_error; *out is then NULL and the pipeline stays usable. */
int obgpu_pipeline_group_by(obgpu_pipeline *p, const obgpu_host_scan_spec *spec, const int32_t *group_cols, int32_t n_group_cols,
                            const obgpu_group_agg *aggs, int32_t n_aggs, obgpu_host_scan_result *result, obgpu_groups **out);
/* GROUP BY as obgpu_pipeline_group_by, with each page batch grouped by obgpu_result_group_by_any: group columns of any
 * encoding, each batch on the path its blocks allow, and the groups of both paths merged into one accumulator. Spec, result,
 * *out and the spec refusals are obgpu_pipeline_group_by's; a batch refusal is obgpu_result_group_by_any's. The groups are those
 * of obgpu_result_group_by_any over the whole table as one batch. *cells_batches (may be NULL): how many batches took
 * OBGPU_GROUP_PATH_CELLS (0 after a failure). */
int obgpu_pipeline_group_by_any(obgpu_pipeline *p, const obgpu_host_scan_spec *spec, const int32_t *group_cols, int32_t n_group_cols,
                                const obgpu_group_agg *aggs, int32_t n_aggs, obgpu_host_scan_result *result, obgpu_groups **out,
                                int32_t *cells_batches);
/* ORDER BY keys LIMIT k over every row of the spec's table that its filter selects: each worker opens its batch as
 * obgpu_pipeline_group_by does, scans it with nothing projected, takes its rows with obgpu_result_top_rows and merges them, under
 * the pipeline's mutex, into one device-resident set of at most k rows (at most 2k rows ordered per merge, k kept). Positions are
 * made table-wide: a row's block is the index into the spec's block list. The rows are byte for byte those of
 * obgpu_result_top_rows over the whole table opened as one batch, whatever the batch cut, ramp or worker count. *n_rows and
 * *heap_bytes are set; obgpu_pipeline_fetch_top_rows copies the rows out in obgpu_result_fetch_top_rows' layout, and they stay
 * with the pipeline until its next obgpu_pipeline_top_rows or obgpu_pipeline_destroy.
 *   Spec and result as obgpu_pipeline_group_by: no_row_output 1, no row ids, block tables or scalar aggregates
 *   (OBGPU_INVALID_ARGUMENT otherwise). Arguments as obgpu_result_top_rows. The first refusal of any batch (including a key or
 *   output column whose obj_type differs between batches) is returned with its text in obgpu_pipeline_last_error; the
 *   pipeline then holds no rows and stays usable. */
int obgpu_pipeline_top_rows(obgpu_pipeline *p, const obgpu_host_scan_spec *spec, const obgpu_sort_key *keys, int32_t n_keys,
                            const int32_t *out_cols, int32_t n_out, int64_t k, obgpu_host_scan_result *result, int64_t *n_rows,
                            int64_t *heap_bytes);
int obgpu_pipeline_fetch_top_rows(obgpu_pipeline *p, int32_t *host_block, int32_t *host_row, int64_t *host_vals, uint8_t *host_nulls,
                                  void *host_heap);

#ifdef __cplusplus
}
#endif
#endif /* OBGPU_PIPELINE_H_ */
