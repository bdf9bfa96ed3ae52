// C++ test of the compressor argument of ObGpuPartitionMajorMerger::write_column_groups: the merged stream of two runs, one of
// whose payload columns is NULL-dominated (the device leaves those blocks to the host writer, which the adapter splices in), is
// written into three column groups with OBGPU_COMPRESSOR_NONE and with LZ4 / zstd_1.3.8. Every compressed group must be
// obgpu_writer_compress_blocks over the NONE group's blocks: same offsets, sizes and bytes. Without a device: exit 77.
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
  // two runs with disjoint rowkeys; payload 0: small repeating values (compressible), payload 1: 60-bit values NULL in 60 % of
  // the rows (ObRawEncoder stores it as var-length cells: host-written blocks), payload 2: a slow counter
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
      const uint8_t n1 = (i / 900) % 4 == 1 && mix(h + 7) % 100 < 60 ? 1 : 0;   // NULL-dominated in every fourth stretch
      run.vals[0].push_back((int64_t)(h % 17));
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
  std::vector<ObGpuColumnGroup> groups(3);
  groups[0].cols_ = {-1, 0, 1, 2}; groups[0].obj_types_.assign(4, OBGPU_OBJ_INT); groups[0].rowkey_col_cnt_ = 1;   // all columns
  groups[1].cols_ = {1}; groups[1].obj_types_ = {OBGPU_OBJ_INT};                                                  // NULL-dominated
  groups[2].cols_ = {2, 0}; groups[2].obj_types_.assign(2, OBGPU_OBJ_INT);
  const int64_t rpb = 600;
  const int32_t align = 128;
  std::vector<ObGpuEncodedColumnGroup> plain;
  ASSERT_EQ(merger.write_column_groups(groups, rpb, align, plain), OB_SUCCESS);
  ASSERT_EQ((long long)plain.size(), 3);
  int host_blocks = 0;
  for (const ObGpuEncodedColumnGroup &g : plain) host_blocks += g.host_encoded_blocks_;
  if (host_blocks == 0) { printf("FAIL: no block was left to the host writer\n"); ++g_fail; }
  for (int32_t comp : {OBGPU_COMPRESSOR_LZ4, OBGPU_COMPRESSOR_ZSTD_1_3_8, OBGPU_COMPRESSOR_LZ4_1_9_1}) {
    std::vector<ObGpuEncodedColumnGroup> got;
    ASSERT_EQ(merger.write_column_groups(groups, rpb, align, got, comp), OB_SUCCESS);
    ASSERT_EQ((long long)got.size(), 3);
    for (size_t g = 0; g < got.size() && g < plain.size() && g_fail < 10; ++g) {
      const ObGpuEncodedColumnGroup &p = plain[g], &c = got[g];
      const int32_t nb = (int32_t)p.offsets_.size();
      std::vector<uint8_t> want(p.image_.size() + (size_t)nb * align + align, 0);
      std::vector<int64_t> woff((size_t)nb), wsz((size_t)nb);
      int64_t used = 0;
      ASSERT_EQ(obgpu_writer_compress_blocks(p.image_.data(), p.offsets_.data(), p.sizes_.data(), nb, comp, align, want.data(),
                                             (int64_t)want.size(), woff.data(), wsz.data(), &used), 0);
      ASSERT_EQ(c.row_count_, p.row_count_);
      ASSERT_EQ(c.host_encoded_blocks_, p.host_encoded_blocks_);
      for (size_t k = 0; k < p.column_checksums_.size(); ++k) ASSERT_EQ(c.column_checksums_[k], p.column_checksums_[k]);
      ASSERT_EQ((long long)c.offsets_.size(), nb);
      int64_t stored = 0, plain_bytes = 0;
      for (int32_t b = 0; b < nb && b < (int32_t)c.offsets_.size() && g_fail < 10; ++b) {
        ASSERT_EQ(c.offsets_[(size_t)b], woff[(size_t)b]);
        ASSERT_EQ(c.sizes_[(size_t)b], wsz[(size_t)b]);
        if (c.offsets_[(size_t)b] == woff[(size_t)b] && c.sizes_[(size_t)b] == wsz[(size_t)b] &&
            woff[(size_t)b] + wsz[(size_t)b] <= (int64_t)c.image_.size())
          ASSERT_EQ(memcmp(c.image_.data() + woff[(size_t)b], want.data() + woff[(size_t)b], (size_t)wsz[(size_t)b]), 0);
        else
          ++g_fail;
        stored += wsz[(size_t)b];
        plain_bytes += p.sizes_[(size_t)b];
      }
      if (g != 1 && stored >= plain_bytes) { printf("FAIL: group %zu did not shrink with compressor %d\n", g, comp); ++g_fail; }
    }
  }
  std::vector<ObGpuEncodedColumnGroup> none;
  ASSERT_EQ(merger.write_column_groups(groups, rpb, align, none, 5), OB_NOT_SUPPORTED);   // zstd_1.0: not compressed on the device
  if (g_fail) { printf("%d failures\n", g_fail); return 1; }
  printf("partition merger compress tests passed\n");
  return 0;
}
