// See ob_gpu_micro_block_decoder.h. Host glue only: every data-parallel step happens in
// libobgpu_scan.so (sm_90a kernels); this file never decodes a cell itself.
#include "ob_gpu_micro_block_decoder.h"

#include <algorithm>
#include <cstring>

namespace oceanbase {
using namespace common;
namespace blocksstable {

ObGpuScanRuntime::ObGpuScanRuntime(int device) {
  if (obgpu_ctx_create(device, &ctx_) != OBGPU_SUCCESS) ctx_ = nullptr;
}
ObGpuScanRuntime::~ObGpuScanRuntime() {
  if (ctx_) obgpu_ctx_destroy(ctx_);
}

// ---- ObGpuMicroBlockDecoder ------------------------------------------------------------------------
void ObGpuMicroBlockDecoder::reset() {
  str_arena_.clear();
  if (batch_) obgpu_batch_close(batch_);
  batch_ = nullptr;
  row_count_ = column_count_ = 0;
}

int ObGpuMicroBlockDecoder::init(const ObMicroBlockData &block_data) {
  if (!rt_.is_valid()) return OB_NOT_INIT;
  if (block_data.get_buf() == nullptr || block_data.get_buf_size() <= 0) return OB_INVALID_ARGUMENT;
  reset();  // can be init twice
  const int64_t size = block_data.get_buf_size();
  padded_.assign((size_t)((size + 15) & ~15ll) + 64, 0);
  memcpy(padded_.data(), block_data.get_buf(), (size_t)size);
  host_buf_ = block_data.get_buf();
  const int64_t off = 0;
  int ret = obgpu_batch_open(rt_.ctx(), padded_.data(), (int64_t)padded_.size(), &off, &size, 1, 0, nullptr, &batch_);
  if (ret != OBGPU_SUCCESS) return ret;
  int32_t cols = 0;
  ret = obgpu_batch_block_info(batch_, 0, &row_count_, &cols);
  column_count_ = cols;
  return ret;
}

int ObGpuMicroBlockDecoder::get_row_count(int64_t &row_count) const {
  if (!batch_) return OB_NOT_INIT;
  row_count = row_count_;
  return OB_SUCCESS;
}

int ObGpuMicroBlockDecoder::get_column_count(int64_t &column_count) const {
  if (!batch_) return OB_NOT_INIT;
  column_count = column_count_;
  return OB_SUCCESS;
}

static void to_params(const sql::ObWhiteFilterExecutor &filter, std::vector<obgpu_filter_param> &params) {
  for (const ObStorageDatum &d : filter.get_datums()) {
    obgpu_filter_param p{};
    p.is_null = d.is_null() ? 1 : 0;
    if (!d.is_null()) {
      p.i64 = d.get_int();
      p.ptr = d.ptr_;
      p.len = d.len_;
    }
    params.push_back(p);
  }
}

int ObGpuMicroBlockDecoder::filter_pushdown_filter(const sql::ObPushdownFilterExecutor *parent,
                                                   sql::ObWhiteFilterExecutor &filter,
                                                   const sql::PushdownFilterInfo &pd_filter_info,
                                                   ObBitmap &result_bitmap) {
  (void)parent;  // can_skip_filter is an optimisation of the CPU path; the result bitmap is the same
  if (!batch_) return OB_NOT_INIT;
  if (pd_filter_info.start_ < 0 || pd_filter_info.start_ + pd_filter_info.count_ > row_count_ ||
      result_bitmap.size() != pd_filter_info.count_)
    return OB_INVALID_ARGUMENT;
  std::vector<obgpu_filter_param> params;
  to_params(filter, params);
  return obgpu_filter_white(batch_, 0, filter.get_col_offset(), (int32_t)filter.get_op_type(), params.data(),
                            (int32_t)params.size(), pd_filter_info.start_, pd_filter_info.count_,
                            result_bitmap.get_data());
}

int ObGpuMicroBlockDecoder::get_rows(const int32_t col, const int32_t *row_ids, const int64_t row_cap,
                                     const int64_t vec_offset, ObFixedLengthVector &vec) {
  if (!batch_) return OB_NOT_INIT;
  if ((int64_t)vec.data_.size() < (vec_offset + row_cap) * vec.len_) return OB_BUF_NOT_ENOUGH;
  int32_t has_null = 0;
  const int ret = obgpu_project_fixed(batch_, 0, col, row_ids, row_cap, vec_offset, vec.data_.data(), vec.len_,
                                      vec.nulls_.data(), &has_null);
  if (has_null) vec.has_null_ = true;
  return ret;
}

int ObGpuMicroBlockDecoder::get_rows(const int32_t col, const int32_t *row_ids, const int64_t row_cap,
                                     const int64_t vec_offset, ObDiscreteVector &vec) {
  if (!batch_) return OB_NOT_INIT;
  if ((int64_t)vec.ptrs_.size() < vec_offset + row_cap) return OB_BUF_NOT_ENOUGH;
  int32_t has_null = 0;
  int32_t rebuilt = 0;
  if (obgpu_batch_column_materialised(batch_, col, &rebuilt) == OB_SUCCESS && rebuilt) {
    // HEX_PACKING / STRING_DIFF / STRING_PREFIX: the values do not exist in the block. The reference decodes them into memory of the
    // decoder's allocator (ob_hex_string_decoder.cpp:87-93); here they land in an arena this decoder owns until its next init / reset.
    std::vector<int64_t> off((size_t)row_cap + 1);
    std::vector<uint64_t> nulls((size_t)(row_cap + 63) / 64, 0);
    int64_t need = 0;
    int ret = obgpu_project_strings(batch_, 0, col, row_ids, row_cap, nullptr, 0, off.data(), nulls.data(), &has_null, &need);
    if (ret == OB_BUF_NOT_ENOUGH) {
      str_arena_.emplace_back((size_t)need + 1);
      ret = obgpu_project_strings(batch_, 0, col, row_ids, row_cap, str_arena_.back().data(), need, off.data(), nulls.data(), &has_null, &need);
    }
    if (ret != OB_SUCCESS) return ret;
    char *heap = str_arena_.empty() ? nullptr : str_arena_.back().data();
    for (int64_t i = 0; i < row_cap; ++i) {
      const int64_t at = vec_offset + i;
      if ((nulls[(size_t)i / 64] >> (i % 64)) & 1) { vec.nulls_[(size_t)at / 64] |= 1ull << (at % 64); continue; }   // slot left as it was
      vec.ptrs_[(size_t)at] = heap + off[(size_t)i];
      vec.lens_[(size_t)at] = (int32_t)(off[(size_t)i + 1] - off[(size_t)i]);
    }
    if (has_null) vec.has_null_ = true;
    return OB_SUCCESS;
  }
  // string pointers land in the CALLER's block buffer (zero-copy like the reference, rule 8c.6)
  const int ret = obgpu_project_discrete(batch_, 0, col, row_ids, row_cap, vec_offset, (uint64_t)(uintptr_t)host_buf_,
                                         reinterpret_cast<uint64_t *>(vec.ptrs_.data()), vec.lens_.data(),
                                         vec.nulls_.data(), &has_null);
  if (has_null) vec.has_null_ = true;
  return ret;
}

int ObGpuMicroBlockDecoder::get_rows(const int32_t col, const int32_t *row_ids, const int64_t row_cap, const int64_t datum_offset,
                                     common::ObDatum *col_datums) {
  if (!batch_) return OB_NOT_INIT;
  if (!row_ids || !col_datums) return OB_INVALID_ARGUMENT;
  // string datums point into the caller's block buffer (host_buf_), like the reference's shallow string datums
  return obgpu_project_datums(batch_, 0, col, row_ids, row_cap, datum_offset, (uint64_t)(uintptr_t)host_buf_,
                              reinterpret_cast<obgpu_datum *>(col_datums));
}

// ---- dictionary surface ----------------------------------------------------------------------------------
int ObGpuMicroBlockDecoder::get_distinct_count(const int32_t group_by_col, int64_t &distinct_cnt) const {
  if (!batch_) return OB_NOT_INIT;
  return obgpu_block_distinct_count(batch_, 0, group_by_col, &distinct_cnt);
}

int ObGpuMicroBlockDecoder::read_distinct(const int32_t group_by_col, common::ObDatum *datums, const int64_t cap,
                                          int64_t &distinct_cnt) const {
  if (!batch_) return OB_NOT_INIT;
  if (!datums || cap < 0) return OB_INVALID_ARGUMENT;
  int ret = obgpu_block_distinct_count(batch_, 0, group_by_col, &distinct_cnt);
  if (ret != OB_SUCCESS) return ret;
  if (distinct_cnt > cap) return OB_BUF_NOT_ENOUGH;
  std::vector<uint64_t> vals((size_t)distinct_cnt + 1);
  std::vector<int32_t> lens((size_t)distinct_cnt + 1, -1);
  ret = obgpu_block_read_distinct(batch_, 0, group_by_col, (uint64_t)(uintptr_t)host_buf_, vals.data(), lens.data(), distinct_cnt,
                                  &distinct_cnt);
  if (ret != OB_SUCCESS) return ret;
  int32_t el = 0;
  if ((ret = obgpu_batch_column_type(batch_, group_by_col, nullptr, &el)) != OB_SUCCESS) return ret;
  for (int64_t i = 0; i < distinct_cnt; ++i) {
    ObDatum &d = datums[i];
    if (el == 0) {   // string: shallow datum into the block
      d.ptr_ = reinterpret_cast<const char *>((uintptr_t)vals[(size_t)i]);
      d.pack_ = (uint32_t)lens[(size_t)i] & 0x1fffffffu;
    } else {
      if (d.ptr_ == nullptr) return OB_INVALID_ARGUMENT;
      memcpy(const_cast<char *>(d.ptr_), &vals[(size_t)i], (size_t)el);
      d.pack_ = (uint32_t)el;
    }
  }
  return OB_SUCCESS;
}

int ObGpuMicroBlockDecoder::read_reference(const int32_t group_by_col, const int32_t *row_ids, const int64_t row_cap,
                                           uint32_t *refs) const {
  if (!batch_) return OB_NOT_INIT;
  return obgpu_block_read_reference(batch_, 0, group_by_col, row_ids, row_cap, refs);
}

int ObGpuMicroBlockDecoder::filter_black_filter_batch(const sql::ObPushdownFilterExecutor *parent, sql::ObBlackFilterExecutor &filter,
                                                      const sql::PushdownFilterInfo &pd_filter_info, ObBitmap &result_bitmap,
                                                      bool &filter_applied) {
  (void)parent;
  filter_applied = false;
  if (!batch_) return OB_NOT_INIT;
  if (pd_filter_info.start_ < 0 || pd_filter_info.start_ + pd_filter_info.count_ > row_count_ ||
      result_bitmap.size() != pd_filter_info.count_)
    return OB_INVALID_ARGUMENT;
  if (filter.get_col_offsets().size() != 1) return OB_SUCCESS;
  const int32_t col = filter.get_col_offsets()[0];
  int64_t cnt = 0;
  int ret = obgpu_block_distinct_count(batch_, 0, col, &cnt);
  if (ret == OB_NOT_SUPPORTED) return OB_SUCCESS;   // not dictionary coded: the caller's row-wise path
  if (ret != OB_SUCCESS) return ret;
  std::vector<uint64_t> slots((size_t)cnt + 1);
  std::vector<ObDatum> datums((size_t)cnt + 1);
  for (int64_t i = 0; i <= cnt; ++i) datums[(size_t)i].ptr_ = reinterpret_cast<const char *>(&slots[(size_t)i]);
  if ((ret = read_distinct(col, datums.data(), cnt, cnt)) != OB_SUCCESS) return ret;
  std::vector<uint8_t> pass((size_t)cnt + 1, 0);
  for (int64_t i = 0; i < cnt; ++i) {
    bool filtered = false;
    if ((ret = filter.filter(datums[(size_t)i], filtered)) != OB_SUCCESS) return ret;
    pass[(size_t)i] = filtered ? 0 : 1;
  }
  ObDatum null_datum;
  null_datum.set_null();
  bool null_filtered = false;
  if ((ret = filter.filter(null_datum, null_filtered)) != OB_SUCCESS) return ret;
  ret = obgpu_filter_dict_pass(batch_, 0, col, pass.data(), cnt, null_filtered ? 0 : 1, pd_filter_info.start_, pd_filter_info.count_,
                               result_bitmap.get_data());
  if (ret == OB_SUCCESS) filter_applied = true;
  return ret;
}

// ---- ObPushdownFilterExecutor::execute ----------------------------------------------------------------
int execute_pushdown_filter(sql::ObPushdownFilterExecutor *filter, sql::ObPushdownFilterExecutor *parent,
                            const sql::PushdownFilterInfo &pd, ObGpuMicroBlockDecoder &decoder) {
  int ret = OB_SUCCESS;
  ObBitmap *result = nullptr;
  if (filter == nullptr || pd.start_ < 0 || pd.count_ <= 0) return OB_INVALID_ARGUMENT;
  if ((ret = filter->init_bitmap(pd.count_, result)) != OB_SUCCESS) return ret;
  if (filter->is_filter_node()) {
    result->reuse(false);
    return decoder.filter_pushdown_filter(parent, *static_cast<sql::ObWhiteFilterExecutor *>(filter), pd, *result);
  }
  if (filter->get_child_count() < 2) return OB_ERR_UNEXPECTED;
  sql::ObPushdownFilterExecutor **children = filter->get_childs();
  for (uint32_t i = 0; ret == OB_SUCCESS && i < filter->get_child_count(); ++i) {
    if ((ret = execute_pushdown_filter(children[i], filter, pd, decoder)) != OB_SUCCESS) break;
    const ObBitmap *child = children[i]->get_result();
    if (filter->is_logic_and_node()) {
      if ((ret = result->bit_and(*child)) == OB_SUCCESS && result->is_all_false()) break;
    } else {
      if ((ret = result->bit_or(*child)) == OB_SUCCESS && result->is_all_true()) break;
    }
  }
  return ret;
}

// ---- ObGpuSSTableBatchScanner -------------------------------------------------------------------------
void ObGpuSSTableBatchScanner::reset() {
  if (result_) obgpu_result_free(result_);
  if (batch_) obgpu_batch_close(batch_);
  if (pipe_) obgpu_pipeline_destroy(pipe_);
  pipe_ = nullptr;
  host_mode_ = false;
  result_ = nullptr;
  batch_ = nullptr;
  cur_block_ = 0;
  cur_row_ = 0;
  selected_ = 0;
  rev_started_ = false;
}

int ObGpuSSTableBatchScanner::flatten(sql::ObPushdownFilterExecutor *f, std::vector<obgpu_filter_node> &nodes,
                                      std::vector<obgpu_filter_param> &params) {
  obgpu_filter_node nd{};
  if (f->is_filter_node()) {
    auto *w = static_cast<sql::ObWhiteFilterExecutor *>(f);
    nd.kind = OBGPU_NODE_WHITE;
    nd.op = (int32_t)w->get_op_type();
    nd.col = w->get_col_offset();
    nd.param_begin = (int32_t)params.size();
    to_params(*w, params);
    nd.n_params = (int32_t)params.size() - nd.param_begin;
  } else {
    for (uint32_t i = 0; i < f->get_child_count(); ++i) {
      const int ret = flatten(f->get_childs()[i], nodes, params);
      if (ret != OB_SUCCESS) return ret;
    }
    nd.kind = f->is_logic_and_node() ? OBGPU_NODE_AND : OBGPU_NODE_OR;
    nd.n_children = (int32_t)f->get_child_count();
  }
  nodes.push_back(nd);
  return OB_SUCCESS;
}

int ObGpuSSTableBatchScanner::set_index_infos(ObMicroIndexInfo *infos, int32_t n_blocks) {
  if (batch_) return OB_INIT_TWICE;   // the aggregate rows travel with the batch: before init only
  if ((infos == nullptr) != (n_blocks == 0) || n_blocks < 0) return OB_INVALID_ARGUMENT;
  index_infos_ = infos;
  n_index_infos_ = n_blocks;
  return OB_SUCCESS;
}

int ObGpuSSTableBatchScanner::init(const void *image, int64_t image_size, const int64_t *offsets, const int64_t *sizes,
                                   int32_t n_blocks, sql::ObPushdownFilterExecutor *filter,
                                   const std::vector<int32_t> &proj, int64_t batch_size) {
  if (!rt_.is_valid()) return OB_NOT_INIT;
  if (batch_size <= 0) return OB_INVALID_ARGUMENT;
  reset();
  image_ = static_cast<const char *>(image);
  n_blocks_ = n_blocks;
  batch_size_ = batch_size;
  proj_ = proj;
  int ret = OB_SUCCESS;
  std::vector<obgpu_filter_node> nodes;
  std::vector<obgpu_filter_param> params;
  obgpu_filter flt{};
  if (filter) {
    if ((ret = flatten(filter, nodes, params)) != OB_SUCCESS) return ret;
    flt.nodes = nodes.data();
    flt.n_nodes = (int32_t)nodes.size();
    flt.params = params.data();
    flt.n_params = (int32_t)params.size();
  }
  const bool use_index = filter && index_infos_ != nullptr;
  if (pipe_streams_ > 0 && !use_index) {
    // ---- pipelined open: every page batch's H2D, kernels and D2H overlap; the result ends up in host memory ----
    if ((ret = obgpu_pipeline_create(0, pipe_streams_, &pipe_)) != OBGPU_SUCCESS) return ret;
    obgpu_host_scan_spec hs{};
    hs.image = image;
    hs.image_size = image_size;
    hs.offsets = offsets;
    hs.sizes = sizes;
    hs.n_blocks = n_blocks;
    hs.filter = filter ? &flt : nullptr;
    hs.proj_cols = proj_.data();
    hs.n_proj = (int32_t)proj_.size();
    hs.blocks_per_batch = pipe_bpb_;
    hs.selectivity_hint = 1.0;                 // slices hold every row of their batch: no overflow handling needed
    hs.string_base = (uint64_t)(uintptr_t)image;
    int32_t nb = 0;
    int64_t cap = 0;
    if ((ret = obgpu_pipeline_plan(&hs, &nb, &cap)) != OBGPU_SUCCESS) return ret;
    // column shapes from the first block's headers through a one-block batch (types are per SSTable)
    {
      obgpu_batch *probe = nullptr;
      const int64_t zero = 0;
      ret = compressor_ ? obgpu_batch_open_compressed(rt_.ctx(), (const char *)image + offsets[0], sizes[0], &zero, sizes, 1, 0, compressor_, &probe)
                        : obgpu_batch_open(rt_.ctx(), (const char *)image + offsets[0], sizes[0], &zero, sizes, 1, 0, nullptr, &probe);
      if (ret != OBGPU_SUCCESS) return ret;
      obgpu_scan_spec ps{};
      ps.proj_cols = proj_.data();
      ps.n_proj = (int32_t)proj_.size();
      ps.max_selected_rows = 1;
      obgpu_result *pr = nullptr;
      ret = obgpu_scan(probe, &ps, &pr);
      cols_.resize(proj_.size());
      for (size_t c = 0; ret == OBGPU_SUCCESS && c < proj_.size(); ++c) ret = obgpu_result_col_get(pr, (int32_t)c, &cols_[c]);
      if (pr) obgpu_result_free(pr);
      obgpu_batch_close(probe);
      if (ret != OBGPU_SUCCESS) return ret;
    }
    const size_t np = proj_.size();
    h_data_.assign(np, {});
    h_lens_.assign(np, {});
    h_nulls_.assign(np, {});
    std::vector<void *> od(np);
    std::vector<int32_t *> ol(np);
    std::vector<uint64_t *> on(np);
    for (size_t c = 0; c < np; ++c) {
      h_data_[c].assign((size_t)cap * (cols_[c].is_string ? 8 : (size_t)cols_[c].elem_len) + 64, 0);
      if (cols_[c].is_string) h_lens_[c].assign((size_t)cap + 16, 0);
      h_nulls_[c].assign((size_t)cap / 64 + 2, 0);
      od[c] = h_data_[c].data();
      ol[c] = cols_[c].is_string ? h_lens_[c].data() : nullptr;
      on[c] = h_nulls_[c].data();
    }
    h_row_ids_.assign((size_t)cap + 16, 0);
    h_block_begin_.assign((size_t)n_blocks, 0);
    std::vector<int64_t> block_count((size_t)n_blocks, 0), row_begin((size_t)nb + 1), rows((size_t)nb + 1);
    // stored blocks: the decoded string bytes exist only on the device, so every string column gets a heap. The first size is
    // the blocks' decoded payload (data_length_); rebuilt columns may need more: grow and rescan
    std::vector<void *> oh(np, nullptr);
    std::vector<int64_t> heap_cap(np, 0), heap_used(np, 0);
    h_heap_.assign(np, {});
    if (compressor_) {
      int64_t payload = 64;
      for (int32_t b = 0; b < n_blocks; ++b) {
        int32_t dl = 0;
        memcpy(&dl, (const char *)image + offsets[b] + 40, 4);   // ObMicroBlockHeader::data_length_
        payload += dl;
      }
      for (size_t c = 0; c < np; ++c)
        if (cols_[c].is_string) heap_cap[c] = payload;
      hs.compressor_type = compressor_;
      hs.out_heap = oh.data();
      hs.out_heap_cap = heap_cap.data();
      hs.out_heap_used = heap_used.data();
    }
    hs.out_data = od.data();
    hs.out_lens = ol.data();
    hs.out_nulls = on.data();
    hs.out_cap_rows = cap;
    hs.out_row_ids = h_row_ids_.data();
    hs.out_block_begin = h_block_begin_.data();
    hs.out_block_count = block_count.data();
    obgpu_host_scan_result hr{};
    hr.batch_row_begin = row_begin.data();
    hr.batch_rows = rows.data();
    hr.n_batches_cap = nb;
    for (int attempt = 0;; ++attempt) {
      for (size_t c = 0; c < np; ++c)
        if (heap_cap[c] > 0) {
          h_heap_[c].assign((size_t)heap_cap[c], 0);
          oh[c] = h_heap_[c].data();
        }
      ret = obgpu_pipeline_scan(pipe_, &hs, &hr);
      bool grow = false;
      for (size_t c = 0; c < np; ++c)
        if (heap_used[c] > heap_cap[c]) {
          heap_cap[c] = std::max(2 * heap_cap[c], 2 * heap_used[c]);
          grow = true;
        }
      if (ret != OBGPU_BUF_NOT_ENOUGH || !grow || attempt == 8) break;
    }
    if (ret != OBGPU_SUCCESS) return ret;
    selected_ = hr.selected_rows;
    sel_offset_.assign((size_t)n_blocks + 1, 0);
    for (int32_t b = 0; b < n_blocks; ++b) sel_offset_[(size_t)b + 1] = sel_offset_[(size_t)b] + block_count[(size_t)b];
    host_mode_ = true;
    return OB_SUCCESS;
  }
  ret = compressor_ ? obgpu_batch_open_compressed(rt_.ctx(), image, image_size, offsets, sizes, n_blocks, 0, compressor_, &batch_)
                    : obgpu_batch_open(rt_.ctx(), image, image_size, offsets, sizes, n_blocks, 0, nullptr, &batch_);
  if (ret != OBGPU_SUCCESS) return ret;
  if (use_index) {
    if (n_index_infos_ != n_blocks) return OB_INVALID_ARGUMENT;
    std::vector<char> rows;
    std::vector<int64_t> off((size_t)n_blocks + 1, 0);
    for (int32_t b = 0; b < n_blocks; ++b) {
      if (index_infos_[b].has_agg_data())
        rows.insert(rows.end(), index_infos_[b].agg_row_buf_, index_infos_[b].agg_row_buf_ + index_infos_[b].agg_buf_size_);
      off[(size_t)b + 1] = (int64_t)rows.size();
    }
    rows.push_back(0);
    if ((ret = obgpu_batch_set_agg_rows(batch_, rows.data(), off.data())) != OBGPU_SUCCESS) return ret;
    std::vector<uint8_t> verdicts((size_t)n_blocks, 0);
    if ((ret = obgpu_batch_skip_index_filter(batch_, &flt, verdicts.data())) != OBGPU_SUCCESS) return ret;
    for (int32_t b = 0; b < n_blocks; ++b) index_infos_[b].set_filter_constant_type(verdicts[(size_t)b]);
  }
  obgpu_scan_spec spec{};
  spec.filter = filter ? &flt : nullptr;
  spec.proj_cols = proj_.data();
  spec.n_proj = (int32_t)proj_.size();
  spec.want_row_ids = 1;
  spec.string_base = (uint64_t)(uintptr_t)image;
  spec.max_selected_rows = 0;
  if ((ret = obgpu_scan(batch_, &spec, &result_)) != OBGPU_SUCCESS) return ret;
  obgpu_result_info info{};
  if ((ret = obgpu_result_info_get(result_, &info)) != OBGPU_SUCCESS) return ret;
  selected_ = info.selected_rows;
  if (use_index && (ret = obgpu_result_skip_info(result_, &skip_false_, &skip_true_)) != OBGPU_SUCCESS) return ret;
  sel_offset_.assign((size_t)n_blocks + 1, 0);
  if ((ret = obgpu_result_fetch_sel_offsets(result_, sel_offset_.data())) != OBGPU_SUCCESS) return ret;
  cols_.resize(proj_.size());
  for (size_t c = 0; c < proj_.size(); ++c)
    if ((ret = obgpu_result_col_get(result_, (int32_t)c, &cols_[c])) != OBGPU_SUCCESS) return ret;
  return OB_SUCCESS;
}

// get_next_rows with the reference's per-batch LIMIT / OFFSET arithmetic (ObBlockBatchedRowStore::get_row_ids,
// access/ob_block_batched_row_store.cpp:163-186): out_cnt_ counts the selected rows seen so far; a batch keeps rows
// [start, end) where start skips what is left of the offset and end stops at offset + limit.
int ObGpuSSTableBatchScanner::get_next_rows(Batch &out) {
  if (!result_ && !host_mode_) return OB_NOT_INIT;
  for (;;) {
    if (limit_end_) return OB_ITER_END;               // IterEndState::LIMIT_ITER_END
    const int ret = next_window(out);
    if (ret != OB_SUCCESS) return ret;
    if (limit_offset_ == 0 && limit_ < 0) return OB_SUCCESS;
    const int64_t row_count = out.count;
    int64_t start = 0, end = row_count;
    if (limit_offset_ > out_cnt_) start = std::min(limit_offset_ - out_cnt_, row_count);
    if (limit_ >= 0 && out_cnt_ + row_count - limit_offset_ >= limit_) {
      limit_end_ = true;
      end = limit_ - out_cnt_ + limit_offset_;
    }
    out_cnt_ += end;
    if (end < start) end = start;
    trim(out, start, end);
    if (out.count > 0) return OB_SUCCESS;
  }
}

void ObGpuSSTableBatchScanner::trim(Batch &out, int64_t start, int64_t end) {
  if (start == 0 && end == out.count) return;
  auto cut = [&](auto &v) { if (!v.empty()) { v.erase(v.begin() + end, v.end()); v.erase(v.begin(), v.begin() + start); } };
  cut(out.row_ids);
  for (size_t c = 0; c < proj_.size(); ++c) {
    cut(out.ints[c]);
    cut(out.str_ptrs[c]);
    cut(out.str_lens[c]);
    cut(out.is_null[c]);
  }
  out.count = end - start;
}

int ObGpuSSTableBatchScanner::next_window(Batch &out) {
  if (reverse_) return get_next_rows_reverse(out);
  // skip blocks without (remaining) selected rows
  while (cur_block_ < n_blocks_ && cur_row_ >= sel_offset_[(size_t)cur_block_ + 1]) ++cur_block_;
  if (cur_block_ >= n_blocks_) return OB_ITER_END;
  const int64_t end = sel_offset_[(size_t)cur_block_ + 1];
  const int64_t n = std::min<int64_t>(batch_size_, end - cur_row_);
  const int ret = fetch_window(cur_block_, cur_row_, n, out);
  cur_row_ += n;
  return ret;
}

// Reverse scan (ObIMicroBlockRowScanner with step_ == -1, blocksstable/ob_micro_block_row_scanner.cpp:167-260: blocks
// last to first, rows descending): the dense result is walked from its end, every window is handed out reversed.
int ObGpuSSTableBatchScanner::get_next_rows_reverse(Batch &out) {
  if (!rev_started_) {
    rev_started_ = true;
    cur_block_ = n_blocks_ - 1;
    cur_row_ = selected_;      // one past the next row to hand out
  }
  while (cur_block_ >= 0 && cur_row_ <= sel_offset_[(size_t)cur_block_]) --cur_block_;
  if (cur_block_ < 0) return OB_ITER_END;
  const int64_t begin = sel_offset_[(size_t)cur_block_];
  const int64_t n = std::min<int64_t>(batch_size_, cur_row_ - begin);
  const int ret = fetch_window(cur_block_, cur_row_ - n, n, out);
  if (ret == OB_SUCCESS) {
    std::reverse(out.row_ids.begin(), out.row_ids.end());
    for (size_t c = 0; c < proj_.size(); ++c) {
      std::reverse(out.ints[c].begin(), out.ints[c].end());
      std::reverse(out.str_ptrs[c].begin(), out.str_ptrs[c].end());
      std::reverse(out.str_lens[c].begin(), out.str_lens[c].end());
      std::reverse(out.is_null[c].begin(), out.is_null[c].end());
    }
  }
  cur_row_ -= n;
  return ret;
}

// rows [row_begin, row_begin + n) of the dense result (all inside block `block`) -> Batch
int ObGpuSSTableBatchScanner::fetch_window(int32_t block, int64_t row_begin, int64_t n, Batch &out) {
  out.block_idx = block;
  out.count = n;
  out.row_ids.resize((size_t)n);
  if (host_mode_) {   // the pipelined open left everything in host memory: a window is a handful of memcpys
    const int64_t h0 = h_block_begin_[(size_t)block] + (row_begin - sel_offset_[(size_t)block]);
    memcpy(out.row_ids.data(), h_row_ids_.data() + h0, (size_t)n * 4);
    const size_t np = proj_.size();
    out.ints.assign(np, {});
    out.str_ptrs.assign(np, {});
    out.str_lens.assign(np, {});
    out.is_null.assign(np, {});
    for (size_t c = 0; c < np; ++c) {
      out.is_null[c].resize((size_t)n);
      for (int64_t i = 0; i < n; ++i) out.is_null[c][(size_t)i] = (h_nulls_[c][(size_t)(h0 + i) / 64] >> ((h0 + i) % 64)) & 1;
      if (cols_[c].is_string) {
        out.str_ptrs[c].resize((size_t)n);
        out.str_lens[c].assign(h_lens_[c].begin() + h0, h_lens_[c].begin() + h0 + n);
        for (int64_t i = 0; i < n; ++i) {
          uint64_t ptr;
          memcpy(&ptr, h_data_[c].data() + (size_t)(h0 + i) * 8, 8);
          out.str_ptrs[c][(size_t)i] = reinterpret_cast<const char *>((uintptr_t)ptr);
        }
      } else {
        const int el = cols_[c].elem_len;
        out.ints[c].resize((size_t)n);
        for (int64_t i = 0; i < n; ++i) {
          int64_t v = 0;
          memcpy(&v, h_data_[c].data() + (size_t)(h0 + i) * (size_t)el, (size_t)el);
          if (el == 4) v = (int32_t)v;
          out.ints[c][(size_t)i] = v;
        }
      }
    }
    return OB_SUCCESS;
  }
  int ret = obgpu_result_fetch_row_ids(result_, row_begin, n, out.row_ids.data());
  const size_t np = proj_.size();
  out.ints.assign(np, {});
  out.str_ptrs.assign(np, {});
  out.str_lens.assign(np, {});
  out.is_null.assign(np, {});
  std::vector<uint64_t> nulls((size_t)(n + 63) / 64 + 1);
  std::vector<int32_t> heap_cols;   // stored blocks: string cells come back as bytes in win_heap_
  std::vector<std::vector<uint64_t>> heap_ptrs;
  for (size_t c = 0; ret == OBGPU_SUCCESS && c < np; ++c) {
    out.is_null[c].assign((size_t)n, 0);
    if (cols_[c].is_string) {
      std::vector<uint64_t> ptrs((size_t)n);
      out.str_lens[c].resize((size_t)n);
      ret = obgpu_result_fetch_col(result_, (int32_t)c, row_begin, n, compressor_ ? nullptr : ptrs.data(), out.str_lens[c].data(), nulls.data());
      out.str_ptrs[c].resize((size_t)n);
      if (compressor_) {
        heap_cols.push_back((int32_t)c);
        heap_ptrs.push_back(std::move(ptrs));
      } else {
        for (int64_t i = 0; i < n; ++i) out.str_ptrs[c][(size_t)i] = reinterpret_cast<const char *>((uintptr_t)ptrs[(size_t)i]);
      }
    } else {
      const int el = cols_[c].elem_len;
      std::vector<char> raw((size_t)n * el);
      ret = obgpu_result_fetch_col(result_, (int32_t)c, row_begin, n, raw.data(), nullptr, nulls.data());
      out.ints[c].resize((size_t)n);
      for (int64_t i = 0; i < n; ++i) {
        int64_t v = 0;
        memcpy(&v, raw.data() + i * el, (size_t)el);
        if (el == 4) v = (int32_t)v;
        out.ints[c][(size_t)i] = v;
      }
    }
    for (int64_t i = 0; i < n; ++i) out.is_null[c][(size_t)i] = (nulls[(size_t)i / 64] >> (i % 64)) & 1;
  }
  if (ret == OBGPU_SUCCESS && !heap_cols.empty() && n > 0) {
    const int32_t nh = (int32_t)heap_cols.size();
    std::vector<int64_t> bytes((size_t)nh);
    ret = obgpu_result_string_bytes(result_, nh, heap_cols.data(), row_begin, n, bytes.data());
    std::vector<void *> heaps((size_t)nh);
    std::vector<uint64_t *> ptrs((size_t)nh);
    win_heap_.resize(proj_.size());
    for (int32_t j = 0; ret == OBGPU_SUCCESS && j < nh; ++j) {
      std::vector<char> &h = win_heap_[(size_t)heap_cols[(size_t)j]];
      h.resize((size_t)bytes[(size_t)j] + 1);
      heaps[(size_t)j] = h.data();
      ptrs[(size_t)j] = heap_ptrs[(size_t)j].data();
    }
    if (ret == OBGPU_SUCCESS) ret = obgpu_result_fetch_string_heap(result_, nh, heap_cols.data(), row_begin, n, heaps.data(), ptrs.data());
    for (int32_t j = 0; ret == OBGPU_SUCCESS && j < nh; ++j)
      for (int64_t i = 0; i < n; ++i)
        out.str_ptrs[(size_t)heap_cols[(size_t)j]][(size_t)i] = reinterpret_cast<const char *>((uintptr_t)heap_ptrs[(size_t)j][(size_t)i]);
  }
  return ret;
}

}  // namespace blocksstable
}  // namespace oceanbase
