// C++ test of ObGpuColumnGroup::skip_index_cols_: the merged stream of two runs, one of whose payload columns is NULL-dominated
// (the device leaves those blocks to the host writer, which the adapter splices in), is written into column groups that name
// skip-index columns. Every group's aggregate rows must be obgpu_writer_table_agg_rows over the group's rows (fetched back
// with get_next_rows): the same offsets and bytes for every block, host-spliced blocks included; a group without
// skip_index_cols_ comes back without rows. Without a device: exit 77.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../oceanbase_b200/host/ob_gpu_partition_merger.h"
extern "C" {
#include "../../include/obgpu_writer.h"
}

using namespace oceanbase;
using namespace oceanbase::common;
using namespace oceanbase::compaction;

static int g_fail = 0;
#define ASSERT_EQ(a, b)                                                                           \
  do {                                                                                            \
    const long long va__ = (long long)(a), vb__ = (long long)(b);                                 \
    if (va__ != vb__) {                                                                           \
      printf("FAIL %s:%d  %s = %lld, expected %lld\n", __FILE__, __LINE__, #a, va__, vb__);       \
      ++g_fail;                                                                                   \
    }                                                                                             \
  } while (0)

static uint64_t mix(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

struct Run {
  std::vector<int64_t> key, flag;
  std::vector<std::vector<int64_t>> vals;   // [3]
  std::vector<std::vector<uint8_t>> nulls;  // [3]
  std::vector<uint8_t> image;
  std::vector<int64_t> offsets, sizes;
};

int main() {
  {  // device available?
    obgpu_ctx *probe = nullptr;
    if (obgpu_ctx_create(0, &probe) != 0) { printf("no CUDA device: the adapter refuses (no CPU fallback)\n"); return 77; }
    obgpu_ctx_destroy(probe);
  }
  // two runs with disjoint rowkeys; payload 0: small signed values, payload 1: 60-bit values NULL in 60 % of the rows of every
  // fourth stretch (ObRawEncoder stores it as var-length cells: host-written blocks), payload 2: a slow counter
  std::vector<Run> runs(2);
  for (int r = 0; r < 2; ++r) {
    Run &run = runs[r];
    run.vals.assign(3, {});
    run.nulls.assign(3, {});
    for (int64_t i = 0; i < 12000; ++i) {
      const uint64_t h = mix((uint64_t)i * 131u + (uint64_t)r);
      if (h % 3 == 0) continue;
      run.key.push_back(500 + i * 2 + r);
      run.flag.push_back(OBGPU_DF_INSERT);
      const uint8_t n1 = (i / 900) % 4 == 1 && mix(h + 7) % 100 < 60 ? 1 : 0;
      run.vals[0].push_back((int64_t)(h % 17) - 8);
      run.nulls[0].push_back(0);
      run.vals[1].push_back(n1 ? 0 : (int64_t)(mix(h + 977) >> 4));
      run.nulls[1].push_back(n1);
      run.vals[2].push_back(i / 50);
      run.nulls[2].push_back(0);
    }
    obgpu_col_input cols[5];
    memset(cols, 0, sizeof(cols));
    cols[0].obj_type = OBGPU_OBJ_INT; cols[0].encoding = OBGPU_ENC_RAW; cols[0].i64 = run.key.data();
    cols[1].obj_type = OBGPU_OBJ_TINYINT; cols[1].encoding = OBGPU_ENC_RAW; cols[1].i64 = run.flag.data();
    for (int c = 0; c < 3; ++c) {
      cols[2 + c].obj_type = OBGPU_OBJ_INT; cols[2 + c].encoding = OBGPU_ENC_RAW;
      cols[2 + c].i64 = run.vals[c].data(); cols[2 + c].is_null = run.nulls[c].data();
    }
    obgpu_table_image *img = nullptr;
    if (obgpu_writer_encode_table(cols, 5, 1, (int64_t)run.key.size(), 1000, 128, 2, &img) != 0) { printf("encode failed\n"); return 2; }
    int64_t size = 0;
    int32_t nb = 0;
    obgpu_table_image_info(img, &size, &nb);
    run.image.assign((size_t)size + 64, 0);
    run.offsets.resize((size_t)nb);
    run.sizes.resize((size_t)nb);
    obgpu_table_image_export(img, run.image.data(), size, run.offsets.data(), run.sizes.data(), nb);
    obgpu_table_image_free(img);
  }
  std::vector<ObGpuMergeTable> tables;
  for (Run &r : runs) {
    ObGpuMergeTable t;
    t.image_ = r.image.data(); t.image_size_ = (int64_t)r.image.size() - 64;
    t.offsets_ = r.offsets.data(); t.sizes_ = r.sizes.data(); t.block_count_ = (int32_t)r.offsets.size();
    tables.push_back(t);
  }
  ObGpuMergeSchema schema;
  schema.rowkey_col_ = 0; schema.flag_col_ = 1; schema.payload_cols_ = {2, 3, 4};
  ObGpuPartitionMajorMerger merger;
  ASSERT_EQ(merger.init(0, tables, schema), OB_SUCCESS);
  ASSERT_EQ(merger.merge_partition(), OB_SUCCESS);
  ObGpuMergedRows rows;
  ASSERT_EQ(merger.get_next_rows(merger.get_output_row_count(), rows), OB_SUCCESS);
  std::vector<ObGpuColumnGroup> groups(4);
  groups[0].cols_ = {-1, 0, 1, 2}; groups[0].obj_types_ = {OBGPU_OBJ_INT, OBGPU_OBJ_INT, OBGPU_OBJ_INT, OBGPU_OBJ_UINT64};
  groups[0].rowkey_col_cnt_ = 1; groups[0].skip_index_cols_ = {2, 0, 3};                                  // all columns
  groups[1].cols_ = {1}; groups[1].obj_types_ = {OBGPU_OBJ_INT}; groups[1].skip_index_cols_ = {0};      // NULL-dominated
  groups[2].cols_ = {2, 0}; groups[2].obj_types_ = {OBGPU_OBJ_INT32, OBGPU_OBJ_INT};
  groups[2].encodings_ = {OBGPU_ENC_AUTO, OBGPU_ENC_AUTO}; groups[2].skip_index_cols_ = {1};
  groups[3].cols_ = {0}; groups[3].obj_types_ = {OBGPU_OBJ_INT};                                         // no skip index
  const int64_t rpb = 600;
  for (int32_t comp : {OBGPU_COMPRESSOR_NONE, OBGPU_COMPRESSOR_LZ4}) {
    std::vector<ObGpuEncodedColumnGroup> got;
    ASSERT_EQ(merger.write_column_groups(groups, rpb, 128, got, comp), OB_SUCCESS);
    ASSERT_EQ((long long)got.size(), (long long)groups.size());
    int host_blocks = 0;
    for (const ObGpuEncodedColumnGroup &g : got) host_blocks += g.host_encoded_blocks_;
    if (host_blocks == 0) { printf("FAIL: no block was left to the host writer\n"); ++g_fail; }
    for (size_t g = 0; g < got.size() && g_fail < 10; ++g) {
      const ObGpuColumnGroup &cg = groups[g];
      const ObGpuEncodedColumnGroup &o = got[g];
      if (cg.skip_index_cols_.empty()) {
        ASSERT_EQ((long long)o.agg_rows_.size(), 0);
        ASSERT_EQ((long long)o.agg_row_offsets_.size(), 0);
        continue;
      }
      const size_t nc = cg.cols_.size();
      std::vector<obgpu_col_input> in(nc);
      for (size_t c = 0; c < nc; ++c) {
        in[c] = obgpu_col_input{};
        in[c].obj_type = cg.obj_types_[c];
        in[c].encoding = OBGPU_ENC_RAW;
        const int32_t k = cg.cols_[c];
        in[c].i64 = k == -1 ? rows.rowkeys_.data() : rows.values_[(size_t)k].data();
        in[c].is_null = k == -1 ? nullptr : rows.nulls_[(size_t)k].data();
      }
      const int64_t n = rows.row_count_, nb = (n + rpb - 1) / rpb;
      int64_t size = 0;
      ASSERT_EQ(obgpu_writer_table_agg_rows(in.data(), (int32_t)nc, cg.skip_index_cols_.data(), (int32_t)cg.skip_index_cols_.size(), n,
                                            rpb, nullptr, 0, nullptr, &size), 0);
      std::vector<uint8_t> want((size_t)size);
      std::vector<int64_t> woff((size_t)nb + 1);
      ASSERT_EQ(obgpu_writer_table_agg_rows(in.data(), (int32_t)nc, cg.skip_index_cols_.data(), (int32_t)cg.skip_index_cols_.size(), n,
                                            rpb, want.data(), size, woff.data(), &size), 0);
      ASSERT_EQ((long long)o.agg_row_offsets_.size(), nb + 1);
      ASSERT_EQ((long long)o.agg_rows_.size(), size);
      ASSERT_EQ((long long)o.offsets_.size(), nb);
      if (o.agg_row_offsets_ != woff || o.agg_rows_ != want) { printf("FAIL: group %zu aggregate rows differ from the writer's\n", g); ++g_fail; }
    }
  }
  std::vector<ObGpuColumnGroup> dup(1, groups[0]);
  dup[0].skip_index_cols_ = {1, 1};
  std::vector<ObGpuEncodedColumnGroup> none;
  ASSERT_EQ(merger.write_column_groups(dup, rpb, 128, none), OB_INVALID_ARGUMENT);   // a column named twice
  if (g_fail) { printf("%d failures\n", g_fail); return 1; }
  printf("partition merger agg rows tests passed\n");
  return 0;
}
