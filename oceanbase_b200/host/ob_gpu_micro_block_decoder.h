// C++ host adapter over the C-ABI (include/obgpu_scan.h), mirroring the reference's reader surface
// for the scan path: same class / method names, argument meaning and error behaviour as
//   blocksstable::ObIMicroBlockReader / ObIMicroBlockDecoder   (ob_imicro_block_reader.h:295-614,
//                                                               encoding/ob_imicro_block_decoder.h:27-73)
//   sql::ObPushdownFilterExecutor / ObWhiteFilterExecutor      (sql/engine/basic/ob_pushdown_filter.h:690-1259)
//   common::ObBitmap                                           (deps/oblib/src/lib/container/ob_bitmap.h:64-171)
//   storage::ObIStoreRowIterator::get_next_rows                (access/ob_store_row_iterator.h:34-185)
// The reference headers do not compile outside its clang-17 build (DESIGN.md 5), so the few value
// types the interface needs are restated here in the same namespaces with the same member names;
// inside the reference tree the adapter derives from the real classes instead (INTEGRATION.md).
#pragma once
#include <stdint.h>

#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

extern "C" {
#include "../../include/obgpu_scan.h"
#include "../../include/obgpu_pipeline.h"
#include "../../include/obgpu_skip_index.h"
}

namespace oceanbase {
namespace common {

constexpr int OB_SUCCESS = 0;
constexpr int OB_INVALID_ARGUMENT = -4002;
constexpr int OB_INIT_TWICE = -4005;
constexpr int OB_NOT_INIT = -4006;
constexpr int OB_NOT_SUPPORTED = -4007;
constexpr int OB_ITER_END = -4008;
constexpr int OB_ERR_UNEXPECTED = -4016;
constexpr int OB_BUF_NOT_ENOUGH = -4024;

// Byte-per-row selection vector (0x00 / 0x01), the subset of common::ObBitmap the path uses.
class ObBitmap {
public:
  int init(const int64_t valid_bytes, const bool is_all_true = false) {
    data_.assign((size_t)valid_bytes, is_all_true ? 1 : 0);
    return OB_SUCCESS;
  }
  void reuse(const bool is_all_true = false) { std::fill(data_.begin(), data_.end(), is_all_true ? 1 : 0); }
  int64_t size() const { return (int64_t)data_.size(); }
  uint8_t *get_data() { return data_.data(); }
  const uint8_t *get_data() const { return data_.data(); }
  bool test(const int64_t pos) const { return data_[(size_t)pos] != 0; }
  uint64_t popcnt() const { uint64_t c = 0; for (uint8_t b : data_) c += b; return c; }
  bool is_all_false() const { return popcnt() == 0; }
  bool is_all_true() const { return popcnt() == data_.size(); }
  int bit_and(const ObBitmap &r) {
    if (r.size() != size()) return OB_INVALID_ARGUMENT;
    for (size_t i = 0; i < data_.size(); ++i) data_[i] &= r.data_[i];
    return OB_SUCCESS;
  }
  int bit_or(const ObBitmap &r) {
    if (r.size() != size()) return OB_INVALID_ARGUMENT;
    for (size_t i = 0; i < data_.size(); ++i) data_[i] |= r.data_[i];
    return OB_SUCCESS;
  }
  int bit_not() { for (uint8_t &b : data_) b ^= 1; return OB_SUCCESS; }
private:
  std::vector<uint8_t> data_;
};

// blocksstable::ObStorageDatum (a datum with its own value buffer, storage/blocksstable/ob_datum_row.h): what a white
// filter's constants are held in; the scan path only needs their value / NULL.
struct ObStorageDatum {
  const char *ptr_ = nullptr;
  uint32_t len_ = 0;
  bool null_ = false;
  int64_t int_ = 0;  // integer classes: value
  bool is_null() const { return null_; }
  void set_null() { null_ = true; len_ = 0; ptr_ = nullptr; }
  void set_int(int64_t v) { null_ = false; int_ = v; len_ = 8; ptr_ = reinterpret_cast<const char *>(&int_); }
  void set_string(const char *p, uint32_t l) { null_ = false; ptr_ = p; len_ = l; }
  int64_t get_int() const { return int_; }
};

// common::ObDatum (share/datum/ob_datum.h:109-197): 8-byte pointer + {len:29, flag:2, null:1}, 12 packed bytes. Same
// layout as obgpu_datum, so an ObDatum array is handed to the C-ABI as is.
struct ObDatum {
  const char *ptr_ = nullptr;
  union {
    struct {
      uint32_t len_ : 29;
      uint32_t flag_ : 2;
      uint32_t null_ : 1;
    };
    uint32_t pack_;
  };
  ObDatum() : pack_(0) {}
  bool is_null() const { return null_ == 1; }
  void set_null() { len_ = 0; null_ = 1; flag_ = 0; }
  int64_t get_int() const { int64_t v = 0; memcpy(&v, ptr_, len_ < 8 ? len_ : 8); if (len_ == 4) v = (int32_t)v; return v; }
} __attribute__((packed));
static_assert(sizeof(ObDatum) == 12 && sizeof(ObDatum) == sizeof(obgpu_datum), "ObDatum is 12 packed bytes");
}  // namespace common

namespace sql {

enum ObWhiteFilterOperatorType {  // ob_pushdown_filter.h:388-401
  WHITE_OP_EQ = 0, WHITE_OP_LE, WHITE_OP_LT, WHITE_OP_GE, WHITE_OP_GT, WHITE_OP_NE, WHITE_OP_BT,
  WHITE_OP_IN, WHITE_OP_NU, WHITE_OP_NN, WHITE_OP_MAX
};

struct PushdownFilterInfo {  // ob_pushdown_filter.h (start_/count_ window of one micro block)
  int64_t start_ = 0;
  int64_t count_ = 0;
};

enum PushdownExecutorType { WHITE_FILTER_EXECUTOR, AND_FILTER_EXECUTOR, OR_FILTER_EXECUTOR, BLACK_FILTER_EXECUTOR };

class ObPushdownFilterExecutor {
public:
  explicit ObPushdownFilterExecutor(PushdownExecutorType t) : type_(t) {}
  virtual ~ObPushdownFilterExecutor() = default;
  bool is_filter_node() const { return type_ == WHITE_FILTER_EXECUTOR; }
  bool is_logic_and_node() const { return type_ == AND_FILTER_EXECUTOR; }
  bool is_logic_or_node() const { return type_ == OR_FILTER_EXECUTOR; }
  uint32_t get_child_count() const { return (uint32_t)childs_.size(); }
  ObPushdownFilterExecutor **get_childs() { return childs_.data(); }
  void add_child(ObPushdownFilterExecutor *c) { childs_.push_back(c); }
  common::ObBitmap *get_result() { return &filter_bitmap_; }
  int init_bitmap(const int64_t row_count, common::ObBitmap *&bitmap) {
    bitmap = &filter_bitmap_;
    return filter_bitmap_.init(row_count, is_logic_and_node());
  }
protected:
  PushdownExecutorType type_;
  std::vector<ObPushdownFilterExecutor *> childs_;
  common::ObBitmap filter_bitmap_;
};

class ObWhiteFilterExecutor : public ObPushdownFilterExecutor {
public:
  ObWhiteFilterExecutor(int32_t col_offset, ObWhiteFilterOperatorType op)
      : ObPushdownFilterExecutor(WHITE_FILTER_EXECUTOR), col_offset_(col_offset), op_type_(op) {}
  ObWhiteFilterOperatorType get_op_type() const { return op_type_; }
  int32_t get_col_offset() const { return col_offset_; }  // get_col_offsets(is_pd_to_cg).at(0)
  const std::vector<common::ObStorageDatum> &get_datums() const { return datum_params_; }
  std::vector<common::ObStorageDatum> &get_datums() { return datum_params_; }
  bool null_param_contained() const {
    for (const auto &d : datum_params_) if (d.is_null()) return true;
    return false;
  }
private:
  int32_t col_offset_;
  ObWhiteFilterOperatorType op_type_;
  std::vector<common::ObStorageDatum> datum_params_;
};

// sql::ObBlackFilterExecutor (ob_pushdown_filter.h): an arbitrary SQL expression over the filter's columns. Only its
// owner can evaluate it, one datum at a time: filter(datum, filtered) as ObBlackFilterExecutor::filter(ObStorageDatum &,
// skip_bit, bool &filtered) (ob_pushdown_filter.cpp:2579-2582); filtered == true drops the row.
class ObBlackFilterExecutor : public ObPushdownFilterExecutor {
public:
  explicit ObBlackFilterExecutor(std::vector<int32_t> col_offsets)
      : ObPushdownFilterExecutor(BLACK_FILTER_EXECUTOR), col_offsets_(std::move(col_offsets)) {}
  const std::vector<int32_t> &get_col_offsets() const { return col_offsets_; }
  virtual int filter(const common::ObDatum &datum, bool &filtered) = 0;
private:
  std::vector<int32_t> col_offsets_;
};

class ObAndFilterExecutor : public ObPushdownFilterExecutor {
public:
  ObAndFilterExecutor() : ObPushdownFilterExecutor(AND_FILTER_EXECUTOR) {}
};
class ObOrFilterExecutor : public ObPushdownFilterExecutor {
public:
  ObOrFilterExecutor() : ObPushdownFilterExecutor(OR_FILTER_EXECUTOR) {}
};

}  // namespace sql

namespace blocksstable {

struct ObMicroBlockData {  // blocksstable/ob_micro_block_info.h (buf_/size_ of a decompressed block)
  const char *buf_ = nullptr;
  int64_t size_ = 0;
  const char *get_buf() const { return buf_; }
  int64_t get_buf_size() const { return size_; }
};

// The vectors ObMicroBlockDecoder::get_rows fills (share/vector): VEC_FIXED and VEC_DISCRETE.
struct ObFixedLengthVector {
  int32_t len_ = 8;
  std::vector<char> data_;
  std::vector<uint64_t> nulls_;  // sql::ObBitVector words
  bool has_null_ = false;
  void reserve_rows(int64_t n) { data_.assign((size_t)n * len_, 0); nulls_.assign((size_t)(n + 63) / 64, 0); has_null_ = false; }
  bool is_null(int64_t i) const { return (nulls_[(size_t)i / 64] >> (i % 64)) & 1; }
  int64_t get_int(int64_t i) const { int64_t v = 0; memcpy(&v, data_.data() + i * len_, (size_t)len_); return v; }
};
struct ObDiscreteVector {
  std::vector<char *> ptrs_;
  std::vector<int32_t> lens_;
  std::vector<uint64_t> nulls_;
  bool has_null_ = false;
  void reserve_rows(int64_t n) { ptrs_.assign((size_t)n, nullptr); lens_.assign((size_t)n, 0); nulls_.assign((size_t)(n + 63) / 64, 0); has_null_ = false; }
  bool is_null(int64_t i) const { return (nulls_[(size_t)i / 64] >> (i % 64)) & 1; }
};

// Per worker thread: device + stream (obgpu_ctx).
class ObGpuScanRuntime {
public:
  explicit ObGpuScanRuntime(int device = 0);
  ~ObGpuScanRuntime();
  bool is_valid() const { return ctx_ != nullptr; }
  obgpu_ctx *ctx() { return ctx_; }
  const char *last_error() const { return obgpu_ctx_last_error(ctx_); }
private:
  obgpu_ctx *ctx_ = nullptr;
};

// ObIMicroBlockDecoder over ONE micro block (reference granularity).
class ObGpuMicroBlockDecoder {
public:
  explicit ObGpuMicroBlockDecoder(ObGpuScanRuntime &rt) : rt_(rt) {}
  ~ObGpuMicroBlockDecoder() { reset(); }
  // ObIMicroBlockReader::init -- re-entrant ("can be init twice")
  int init(const ObMicroBlockData &block_data);
  void reset();
  int get_row_count(int64_t &row_count) const;
  int get_column_count(int64_t &column_count) const;
  // ObIMicroBlockDecoder::filter_pushdown_filter(parent, white filter, pd_filter_info, result_bitmap)
  int filter_pushdown_filter(const sql::ObPushdownFilterExecutor *parent, sql::ObWhiteFilterExecutor &filter,
                             const sql::PushdownFilterInfo &pd_filter_info, common::ObBitmap &result_bitmap);
  // ObMicroBlockDecoder::get_rows (rich format): one call per projected column kind
  int get_rows(const int32_t col, const int32_t *row_ids, const int64_t row_cap, const int64_t vec_offset,
               ObFixedLengthVector &vec);
  int get_rows(const int32_t col, const int32_t *row_ids, const int64_t row_cap, const int64_t vec_offset,
               ObDiscreteVector &vec);
  // ObMicroBlockDecoder::get_rows, datum format (get_col_datums, encoding/ob_micro_block_decoder.cpp:2100-2140,2201-2237):
  // integer datums point at the caller's reserved slots and are written through, string datums point into the block
  int get_rows(const int32_t col, const int32_t *row_ids, const int64_t row_cap, const int64_t datum_offset,
               common::ObDatum *col_datums);
  // ObMicroBlockDecoder::filter_black_filter_batch (encoding/ob_micro_block_decoder.cpp:1822-1859): a black filter over ONE
  // dictionary-coded column is evaluated once per distinct value, rows test their ref on the device. filter_applied
  // stays false (bitmap untouched) when the filter has several columns or the column is not dictionary coded here: the
  // caller then falls back to its row-wise path, as in the reference.
  int filter_black_filter_batch(const sql::ObPushdownFilterExecutor *parent, sql::ObBlackFilterExecutor &filter,
                                const sql::PushdownFilterInfo &pd_filter_info, common::ObBitmap &result_bitmap,
                                bool &filter_applied);
  // Pushdown GROUP BY surface (encoding/ob_micro_block_decoder.cpp:2263-2330): distinct values in dictionary order
  // (integer datums are written through their reserved slots like get_rows; strings point into the block) and the ref of
  // every listed row; a NULL row's ref is the distinct count.
  int get_distinct_count(const int32_t group_by_col, int64_t &distinct_cnt) const;
  int read_distinct(const int32_t group_by_col, common::ObDatum *datums, const int64_t cap, int64_t &distinct_cnt) const;
  int read_reference(const int32_t group_by_col, const int32_t *row_ids, const int64_t row_cap, uint32_t *refs) const;
  obgpu_batch *batch() { return batch_; }
private:
  ObGpuScanRuntime &rt_;
  obgpu_batch *batch_ = nullptr;
  std::vector<char> padded_;  // block copy padded to the 16-byte TMA granularity
  std::vector<std::vector<char>> str_arena_;  // strings a codec rebuilt (HEX_PACKING / STRING_DIFF / STRING_PREFIX), one chunk per get_rows
  const char *host_buf_ = nullptr;
  int64_t row_count_ = 0, column_count_ = 0;
};

// ObPushdownFilterExecutor::execute (ob_pushdown_filter.cpp:1551-1624) driving the decoder leaf by
// leaf with bit_and / bit_or and the reference's early-outs.
int execute_pushdown_filter(sql::ObPushdownFilterExecutor *filter, sql::ObPushdownFilterExecutor *parent,
                            const sql::PushdownFilterInfo &pd_filter_info, ObGpuMicroBlockDecoder &decoder);

// The slice of blocksstable::ObMicroIndexInfo (index_block/ob_index_block_row_struct.h) the skip index needs: the
// serialized aggregate row of the micro block's index row and the verdict check_range leaves on it.
struct ObMicroIndexInfo {
  const char *agg_row_buf_ = nullptr;
  int64_t agg_buf_size_ = 0;
  uint8_t filter_constant_type_ = OBGPU_BOOL_MASK_UNCERTAIN;   // sql::ObBoolMaskType
  bool has_agg_data() const { return agg_row_buf_ != nullptr && agg_buf_size_ > 0; }
  bool is_filter_always_false() const { return filter_constant_type_ == OBGPU_BOOL_MASK_ALWAYS_FALSE; }
  bool is_filter_always_true() const { return filter_constant_type_ == OBGPU_BOOL_MASK_ALWAYS_TRUE; }
  bool is_filter_uncertain() const { return filter_constant_type_ == OBGPU_BOOL_MASK_UNCERTAIN; }
  void set_filter_constant_type(uint8_t t) { filter_constant_type_ = t; }
};

// Page-batch scanner with the ObIStoreRowIterator batch contract: open many micro blocks, one fused
// device scan, then get_next_rows() hands out <= batch_size rows at a time, block by block, rows
// ascending, OB_ITER_END after the last row (access/ob_store_row_iterator.h, ob_sstable_row_scanner.cpp:553).
class ObGpuSSTableBatchScanner {
public:
  explicit ObGpuSSTableBatchScanner(ObGpuScanRuntime &rt) : rt_(rt) {}
  ~ObGpuSSTableBatchScanner() { reset(); }
  // image: consecutive micro blocks (16-byte aligned starts); filter may be null; proj: column store idxs
  int init(const void *image, int64_t image_size, const int64_t *offsets, const int64_t *sizes, int32_t n_blocks,
           sql::ObPushdownFilterExecutor *filter, const std::vector<int32_t> &proj, int64_t batch_size = 256);
  void reset();
  // Skip index (storage::ObSSTableIndexFilter::check_range, access/ob_sstable_index_filter.cpp:56-108): hand over the
  // micro blocks' index infos BEFORE init; the fused scan then prunes with their aggregate rows, and after init
  // every info carries the verdict (set_filter_constant_type) of the whole pushed-down filter on its block.
  int set_index_infos(ObMicroIndexInfo *infos, int32_t n_blocks);
  // Reverse scan (is_reverse_scan_ / step_ == -1 of the row scanners): call before the first get_next_rows; batches then
  // come blocks last to first, rows descending inside a block.
  void set_reverse_scan(bool reverse) { reverse_ = reverse; }
  // Pipelined open (include/obgpu_pipeline.h): init cuts the blocks into page batches and overlaps their host->device
  // copies, kernels and device->host copies on n_streams streams; get_next_rows then serves every batch from host
  // memory. Call before init. (With index infos attached the single-batch path is used: the verdicts come from it.)
  void set_pipelined(int32_t n_streams, int32_t blocks_per_batch = 0) { pipe_streams_ = n_streams; pipe_bpb_ = blocks_per_batch; }
  // Stored micro-blocks (ObMacroBlockReader's IO buffers before decompress_data): the blocks handed to init are in stored form
  // with this common::ObCompressorType (OBGPU_COMPRESSOR_*) and are decoded on the device; 0 (the default): plain blocks. String
  // cells then come back as bytes in scanner-owned buffers that str_ptrs point into. Call before init.
  void set_compressor(int32_t compressor_type) { compressor_ = compressor_type; }
  // LIMIT / OFFSET pushed down to the scan (ObTableAccessContext::limit_param_): every batch is trimmed the way
  // ObBlockBatchedRowStore::get_row_ids does (access/ob_block_batched_row_store.cpp:163-186) -- the first `offset`
  // selected rows are dropped, OB_ITER_END follows the batch that reaches `limit` (limit < 0: none).
  void set_limit(int64_t offset, int64_t limit) { limit_offset_ = offset < 0 ? 0 : offset; limit_ = limit; out_cnt_ = 0; limit_end_ = false; }
  int64_t skipped_blocks() const { return skip_false_; }       // always-false: never read
  int64_t unfiltered_blocks() const { return skip_true_; }     // always-true: no filter evaluation
  // Next batch: count rows of block `block_idx`, row ids ascending. Integer columns are returned as
  // int64 values + null flags (per projected column), string columns as (ptr into image, len).
  struct Batch {
    int32_t block_idx = -1;
    int64_t count = 0;
    std::vector<int32_t> row_ids;
    std::vector<std::vector<int64_t>> ints;          // [proj][count] (integer columns)
    std::vector<std::vector<const char *>> str_ptrs; // [proj][count] (string columns)
    std::vector<std::vector<int32_t>> str_lens;
    std::vector<std::vector<uint8_t>> is_null;       // [proj][count]
  };
  int get_next_rows(Batch &batch);
  int64_t total_selected() const { return selected_; }
private:
  int flatten(sql::ObPushdownFilterExecutor *f, std::vector<obgpu_filter_node> &nodes,
              std::vector<obgpu_filter_param> &params);
  int fetch_window(int32_t block, int64_t row_begin, int64_t n, Batch &out);
  int get_next_rows_reverse(Batch &out);
  int next_window(Batch &out);
  void trim(Batch &out, int64_t start, int64_t end);
  bool reverse_ = false, rev_started_ = false;
  int64_t limit_offset_ = 0, limit_ = -1, out_cnt_ = 0;
  bool limit_end_ = false;
  // pipelined mode: the whole result lives in host memory
  int32_t pipe_streams_ = 0, pipe_bpb_ = 0;
  obgpu_pipeline *pipe_ = nullptr;
  bool host_mode_ = false;
  std::vector<std::vector<char>> h_data_;
  std::vector<std::vector<int32_t>> h_lens_;
  std::vector<std::vector<uint64_t>> h_nulls_;
  std::vector<std::vector<char>> h_heap_;   // pipelined, stored blocks: string bytes per projected column
  std::vector<std::vector<char>> win_heap_; // single batch, stored blocks: the current window's string bytes per projected column
  int32_t compressor_ = 0;
  std::vector<int32_t> h_row_ids_;
  std::vector<int64_t> h_block_begin_;   // output row where a block's selected rows start
  ObGpuScanRuntime &rt_;
  obgpu_batch *batch_ = nullptr;
  obgpu_result *result_ = nullptr;
  const char *image_ = nullptr;
  int32_t n_blocks_ = 0;
  int64_t batch_size_ = 256, selected_ = 0;
  std::vector<int32_t> proj_;
  std::vector<int64_t> sel_offset_;
  std::vector<obgpu_result_col> cols_;
  int32_t cur_block_ = 0;
  int64_t cur_row_ = 0;  // dense row cursor
  ObMicroIndexInfo *index_infos_ = nullptr;
  int32_t n_index_infos_ = 0;
  int64_t skip_false_ = 0, skip_true_ = 0;
};

// blocksstable::ObDatumRow (storage/blocksstable/ob_datum_row.h), the slice a row iterator hands out: one storage datum per
// projected column.
struct ObDatumRow {
  std::vector<common::ObStorageDatum> storage_datums_;
  int64_t count_ = 0;
  int64_t get_column_count() const { return count_; }
};

// storage::ObIStoreRowIterator / ObStoreRowIterator (access/ob_store_row_iterator.h:34-185) over the page-batch scanner: the
// row-at-a-time contract the merge layer (ObMultipleMerge) and the compaction iterators pull through --
// get_next_row(const ObDatumRow *&) until OB_ITER_END, reuse() to rescan, reset() to release. The row handed out stays valid until
// the next call, string datums point into the scanned image (or the scanner's host buffers in pipelined mode or with stored blocks).
class ObGpuStoreRowIterator {
public:
  explicit ObGpuStoreRowIterator(ObGpuScanRuntime &rt) : scanner_(rt) {}
  int init(const void *image, int64_t image_size, const int64_t *offsets, const int64_t *sizes, int32_t n_blocks,
           sql::ObPushdownFilterExecutor *filter, const std::vector<int32_t> &proj, int64_t batch_size = 256) {
    image_ = image; image_size_ = image_size; offsets_ = offsets; sizes_ = sizes; n_blocks_ = n_blocks; filter_ = filter; proj_ = proj;
    batch_size_ = batch_size;
    row_.storage_datums_.assign(proj.size(), common::ObStorageDatum());
    row_.count_ = (int64_t)proj.size();
    at_ = 0;
    batch_ = ObGpuSSTableBatchScanner::Batch();
    inited_ = true;
    return scanner_.init(image, image_size, offsets, sizes, n_blocks, filter, proj, batch_size);
  }
  ObGpuSSTableBatchScanner &scanner() { return scanner_; }   // set_reverse_scan / set_limit / set_index_infos / set_pipelined before init
  bool can_blockscan() const { return true; }
  bool can_batch_scan() const { return true; }
  bool is_sstable_iter() const { return true; }
  int get_next_row(const ObDatumRow *&row) {
    if (!inited_) return common::OB_NOT_INIT;
    while (at_ >= batch_.count) {
      const int ret = scanner_.get_next_rows(batch_);
      if (ret != common::OB_SUCCESS) return ret;   // OB_ITER_END after the last row
      at_ = 0;
    }
    for (size_t c = 0; c < proj_.size(); ++c) {
      common::ObStorageDatum &d = row_.storage_datums_[c];
      if (batch_.is_null[c][(size_t)at_]) d.set_null();
      else if (!batch_.str_ptrs[c].empty()) d.set_string(batch_.str_ptrs[c][(size_t)at_], (uint32_t)batch_.str_lens[c][(size_t)at_]);
      else d.set_int(batch_.ints[c][(size_t)at_]);
    }
    ++at_;
    row = &row_;
    return common::OB_SUCCESS;
  }
  // ObStoreRowIterator::reuse: the same scan again from its first row
  int reuse() {
    if (!inited_) return common::OB_NOT_INIT;
    scanner_.reset();
    at_ = 0;
    batch_ = ObGpuSSTableBatchScanner::Batch();
    return scanner_.init(image_, image_size_, offsets_, sizes_, n_blocks_, filter_, proj_, batch_size_);
  }
  void reset() { scanner_.reset(); inited_ = false; at_ = 0; batch_ = ObGpuSSTableBatchScanner::Batch(); }
private:
  ObGpuSSTableBatchScanner scanner_;
  ObGpuSSTableBatchScanner::Batch batch_;
  ObDatumRow row_;
  int64_t at_ = 0;
  bool inited_ = false;
  const void *image_ = nullptr;
  int64_t image_size_ = 0, batch_size_ = 256;
  const int64_t *offsets_ = nullptr, *sizes_ = nullptr;
  int32_t n_blocks_ = 0;
  sql::ObPushdownFilterExecutor *filter_ = nullptr;
  std::vector<int32_t> proj_;
};

}  // namespace blocksstable
}  // namespace oceanbase
