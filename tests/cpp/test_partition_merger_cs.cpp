// C++ test of ObGpuColumnGroup::row_store_type_ = OB_GPU_CS_ENCODING_ROW_STORE in ObGpuPartitionMajorMerger::write_column_groups:
// the merged stream of two runs is written into a rowkey group and two pure column groups as CS blocks, every column
// OBGPU_ENC_CS_INTEGER, CS_INT_DICT or CS_AUTO, plain and with LZ4 / zstd_1.3.8 / LZ4_1_9_1. Every group must equal
// obgpu_writer_encode_table with the same encodings over the merged rows (RAW integer streams; compressed:
// obgpu_writer_compress_blocks of that image): same offsets, sizes and bytes. No block goes through the host writer, and the
// aggregate rows of the rowkey group equal those of the same group written as PAX blocks. Without a device: exit 77.
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

struct Image {
  std::vector<uint8_t> image;
  std::vector<int64_t> offsets, sizes;
};

// obgpu_writer_encode_table over the merged rows of one group with the group's encodings
static Image writer_group(const ObGpuMergedRows &rows, const ObGpuColumnGroup &cg, int64_t rpb, int32_t align) {
  const size_t nc = cg.cols_.size();
  std::vector<obgpu_col_input> in(nc);
  for (size_t c = 0; c < nc; ++c) {
    in[c] = obgpu_col_input{};
    in[c].obj_type = cg.obj_types_[c];
    in[c].encoding = cg.encodings_[c];
    if (cg.cols_[c] == -1) {
      in[c].i64 = rows.rowkeys_.data();
    } else {
      in[c].i64 = rows.values_[(size_t)cg.cols_[c]].data();
      in[c].is_null = rows.nulls_[(size_t)cg.cols_[c]].data();
    }
  }
  Image out;
  obgpu_table_image *img = nullptr;
  if (obgpu_writer_encode_table(in.data(), (int32_t)nc, cg.rowkey_col_cnt_, rows.row_count_, rpb, align, 2, &img) != 0) {
    printf("FAIL: writer encode\n");
    ++g_fail;
    return out;
  }
  int64_t size = 0;
  int32_t nb = 0;
  obgpu_table_image_info(img, &size, &nb);
  out.image.assign((size_t)size, 0);
  out.offsets.resize((size_t)nb);
  out.sizes.resize((size_t)nb);
  obgpu_table_image_export(img, out.image.data(), size, out.offsets.data(), out.sizes.data(), nb);
  obgpu_table_image_free(img);
  return out;
}

static void expect_same(const ObGpuEncodedColumnGroup &got, const Image &want, size_t g, int32_t comp) {
  ASSERT_EQ((long long)got.offsets_.size(), (long long)want.offsets.size());
  for (size_t b = 0; b < got.offsets_.size() && b < want.offsets.size() && g_fail < 10; ++b) {
    ASSERT_EQ(got.offsets_[b], want.offsets[b]);
    ASSERT_EQ(got.sizes_[b], want.sizes[b]);
    if (got.offsets_[b] == want.offsets[b] && got.sizes_[b] == want.sizes[b] && want.offsets[b] + want.sizes[b] <= (int64_t)got.image_.size()) {
      if (memcmp(got.image_.data() + want.offsets[b], want.image.data() + want.offsets[b], (size_t)want.sizes[b]) != 0) {
        printf("FAIL: group %zu block %zu bytes differ (compressor %d)\n", g, b, comp);
        ++g_fail;
      }
    } else {
      ++g_fail;
    }
  }
}

int main() {
  {  // device available?
    obgpu_ctx *probe = nullptr;
    if (obgpu_ctx_create(0, &probe) != 0) { printf("no CUDA device: the adapter refuses (no CPU fallback)\n"); return 77; }
    obgpu_ctx_destroy(probe);
  }
  // payload 0: 17 values (DICT), payload 1: random 64-bit values, NULL-dominated in every fourth stretch (RAW, var-stored
  // there: host-written blocks), payload 2: a slow counter (RLE / BASE_DIFF)
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
      run.vals[0].push_back((int64_t)(h % 17));
      run.nulls[0].push_back(0);
      run.vals[1].push_back(n1 ? 0 : (int64_t)mix(h + 977));
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
  ASSERT_EQ(rows.row_count_, merger.get_output_row_count());
  std::vector<ObGpuColumnGroup> groups(3);
  groups[0].cols_ = {-1, 0, 1, 2}; groups[0].obj_types_.assign(4, OBGPU_OBJ_INT); groups[0].rowkey_col_cnt_ = 1;   // all columns
  groups[0].encodings_ = {OBGPU_ENC_CS_INTEGER, OBGPU_ENC_CS_INT_DICT, OBGPU_ENC_CS_AUTO, OBGPU_ENC_CS_AUTO};
  groups[0].skip_index_cols_ = {0, 1, 2, 3};
  groups[1].cols_ = {1}; groups[1].obj_types_ = {OBGPU_OBJ_INT}; groups[1].encodings_ = {OBGPU_ENC_CS_INTEGER};   // NULL-dominated
  groups[2].cols_ = {2, 0}; groups[2].obj_types_.assign(2, OBGPU_OBJ_INT); groups[2].encodings_ = {OBGPU_ENC_CS_AUTO, OBGPU_ENC_CS_INT_DICT};
  for (ObGpuColumnGroup &g : groups) g.row_store_type_ = OB_GPU_CS_ENCODING_ROW_STORE;
  ASSERT_EQ(obgpu_writer_set_cs_stream_encoding(1), 0);   // the device writes RAW integer streams
  const int64_t rpb = 600;
  const int32_t align = 128;
  std::vector<Image> want;
  for (const ObGpuColumnGroup &g : groups) want.push_back(writer_group(rows, g, rpb, align));
  std::vector<ObGpuEncodedColumnGroup> plain;
  ASSERT_EQ(merger.write_column_groups(groups, rpb, align, plain), OB_SUCCESS);
  ASSERT_EQ((long long)plain.size(), 3);
  for (size_t g = 0; g < plain.size() && g < want.size(); ++g) {
    ASSERT_EQ(plain[g].host_encoded_blocks_, 0);
    ASSERT_EQ(plain[g].row_count_, rows.row_count_);
    expect_same(plain[g], want[g], g, OBGPU_COMPRESSOR_NONE);
  }
  {  // the aggregate rows depend on the rows alone: the PAX form of the rowkey group gives the same
    std::vector<ObGpuColumnGroup> pax(1, groups[0]);
    pax[0].row_store_type_ = OB_GPU_ENCODING_ROW_STORE;
    pax[0].encodings_.clear();
    std::vector<ObGpuEncodedColumnGroup> p;
    ASSERT_EQ(merger.write_column_groups(pax, rpb, align, p), OB_SUCCESS);
    if (p.size() != 1 || plain.empty() || p[0].agg_rows_.empty() || p[0].agg_rows_ != plain[0].agg_rows_ ||
        p[0].agg_row_offsets_ != plain[0].agg_row_offsets_) {
      printf("FAIL: aggregate rows of the CS group differ from the PAX group's\n");
      ++g_fail;
    }
  }
  for (int32_t comp : {OBGPU_COMPRESSOR_LZ4, OBGPU_COMPRESSOR_ZSTD_1_3_8, OBGPU_COMPRESSOR_LZ4_1_9_1}) {
    std::vector<ObGpuEncodedColumnGroup> got;
    ASSERT_EQ(merger.write_column_groups(groups, rpb, align, got, comp), OB_SUCCESS);
    ASSERT_EQ((long long)got.size(), 3);
    for (size_t g = 0; g < got.size() && g < want.size() && g_fail < 10; ++g) {
      const Image &p = want[g];
      const int32_t nb = (int32_t)p.offsets.size();
      Image z;
      z.image.assign(p.image.size() + (size_t)nb * align + align, 0);
      z.offsets.resize((size_t)nb);
      z.sizes.resize((size_t)nb);
      int64_t used = 0;
      ASSERT_EQ(obgpu_writer_compress_blocks(p.image.data(), p.offsets.data(), p.sizes.data(), nb, comp, align, z.image.data(),
                                             (int64_t)z.image.size(), z.offsets.data(), z.sizes.data(), &used), 0);
      ASSERT_EQ(got[g].host_encoded_blocks_, 0);
      expect_same(got[g], z, g, comp);
    }
  }
  if (g_fail) { printf("%d failures\n", g_fail); return 1; }
  printf("partition merger cs tests passed\n");
  return 0;
}
