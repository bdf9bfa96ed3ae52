// Stored (compressed) micro-blocks through the C++ adapter: ObGpuSSTableBatchScanner with set_compressor, single-batch and
// pipelined, forward and reverse, LIMIT / OFFSET, skip-index infos, and ObGpuStoreRowIterator, must hand out what the same scan
// of the plain image hands out -- VARCHAR cells compared as bytes. A DICT column of long cells, whose decoded bytes outgrow the
// stored payload, makes the pipelined path's first heap too small: it must recover by growing the heap and rescanning.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../oceanbase_b200/host/ob_gpu_micro_block_decoder.h"
extern "C" {
#include "../../include/obgpu_writer.h"
}

using namespace oceanbase;
using namespace oceanbase::common;
using namespace oceanbase::blocksstable;

static int g_fail = 0;
#define ASSERT_EQ(a, b)                                                                           \
  do {                                                                                            \
    const long long va__ = (long long)(a), vb__ = (long long)(b);                                 \
    if (va__ != vb__) {                                                                           \
      printf("FAIL %s:%d  %s = %lld, expected %lld\n", __FILE__, __LINE__, #a, va__, vb__);       \
      ++g_fail;                                                                                   \
    }                                                                                             \
  } while (0)

struct Table {
  std::vector<uint8_t> image;
  std::vector<int64_t> offs, sizes;
  int32_t nb = 0;
};

// every row a scan hands out, in order: block, row id, then per column "N" (NULL) / the integer / the string bytes
static std::vector<std::string> drain(ObGpuSSTableBatchScanner &s) {
  std::vector<std::string> rows;
  ObGpuSSTableBatchScanner::Batch b;
  int ret;
  while ((ret = s.get_next_rows(b)) == OB_SUCCESS) {
    for (int64_t i = 0; i < b.count; ++i) {
      std::string r = std::to_string(b.block_idx) + "/" + std::to_string(b.row_ids[(size_t)i]);
      for (size_t c = 0; c < b.is_null.size(); ++c) {
        r += "|";
        if (b.is_null[c][(size_t)i]) r += "N";
        else if (!b.str_ptrs[c].empty()) r += std::string(b.str_ptrs[c][(size_t)i], (size_t)b.str_lens[c][(size_t)i]);
        else r += std::to_string(b.ints[c][(size_t)i]);
      }
      rows.push_back(r);
    }
  }
  ASSERT_EQ(OB_ITER_END, ret);
  return rows;
}

static std::vector<std::string> drain_iter(ObGpuStoreRowIterator &it, const std::vector<bool> &is_str) {
  std::vector<std::string> rows;
  const ObDatumRow *row = nullptr;
  int ret;
  while ((ret = it.get_next_row(row)) == OB_SUCCESS) {
    std::string r;
    for (int64_t c = 0; c < row->get_column_count(); ++c) {
      const ObStorageDatum &d = row->storage_datums_[(size_t)c];
      r += "|";
      if (d.is_null()) r += "N";
      else if (is_str[(size_t)c]) r += std::string(d.ptr_, d.len_);
      else r += std::to_string(d.get_int());
    }
    rows.push_back(r);
  }
  ASSERT_EQ(OB_ITER_END, ret);
  return rows;
}

static bool same(const std::vector<std::string> &a, const std::vector<std::string> &b) {
  ASSERT_EQ(a.size(), b.size());
  return a == b;
}

int main() {
  ObGpuScanRuntime rt(0);
  if (!rt.is_valid()) {
    printf("no CUDA device: the adapter has no CPU fallback (expected on a CPU-only box)\n");
    return 77;
  }
  // 30 000 rows in blocks of 700: key, a nullable integer, a DICT VARCHAR, a RAW VARCHAR (random bytes in the first blocks,
  // which then stay raw), a DICT VARCHAR of four distinct 200-byte cells
  const int64_t n = 30000, rpb = 700;
  std::vector<int64_t> key(n), a(n);
  std::vector<uint8_t> nulls(n, 0);
  std::string h_dict, h_raw, h_diff;
  std::vector<int64_t> o_dict(n + 1, 0), o_raw(n + 1, 0), o_diff(n + 1, 0);
  uint64_t x = 88172645463325252ull;
  for (int64_t i = 0; i < n; ++i) {
    x ^= x << 13; x ^= x >> 7; x ^= x << 17;
    key[i] = i;
    a[i] = (int64_t)(x % 1000);
    nulls[i] = (x >> 20) % 13 == 0;
    h_dict += "k" + std::to_string((x >> 32) % 9);
    o_dict[i + 1] = (int64_t)h_dict.size();
    if (i < 2 * rpb) for (int k = 0; k < 120; ++k) { x ^= x << 13; x ^= x >> 7; x ^= x << 17; h_raw.push_back((char)(x >> 40)); }
    else h_raw += (i % 4) ? "" : "r" + std::to_string(i % 11);
    o_raw[i + 1] = (int64_t)h_raw.size();
    std::string d(200, 'p');
    d[90] = (char)('0' + (x >> 8) % 4);
    h_diff += d;
    o_diff[i + 1] = (int64_t)h_diff.size();
  }
  h_dict.push_back('\0'); h_raw.push_back('\0'); h_diff.push_back('\0');
  obgpu_col_input cols[5];
  memset(cols, 0, sizeof(cols));
  cols[0].obj_type = OBGPU_OBJ_INT; cols[0].encoding = OBGPU_ENC_INTEGER_BASE_DIFF; cols[0].i64 = key.data();
  cols[1].obj_type = OBGPU_OBJ_INT; cols[1].encoding = OBGPU_ENC_RAW; cols[1].i64 = a.data(); cols[1].is_null = nulls.data();
  cols[2].obj_type = OBGPU_OBJ_VARCHAR; cols[2].encoding = OBGPU_ENC_DICT; cols[2].str_heap = h_dict.data(); cols[2].str_off = o_dict.data();
  cols[3].obj_type = OBGPU_OBJ_VARCHAR; cols[3].encoding = OBGPU_ENC_RAW; cols[3].str_heap = h_raw.data(); cols[3].str_off = o_raw.data();
  cols[3].is_null = nulls.data();
  cols[4].obj_type = OBGPU_OBJ_VARCHAR; cols[4].encoding = OBGPU_ENC_DICT; cols[4].str_heap = h_diff.data(); cols[4].str_off = o_diff.data();
  Table plain;
  int64_t plain_size = 0;
  {
    obgpu_table_image *img = nullptr;
    ASSERT_EQ(0, obgpu_writer_encode_table(cols, 5, 1, n, rpb, 128, 2, &img));
    int64_t size = 0;
    obgpu_table_image_info(img, &size, &plain.nb);
    plain.image.assign((size_t)size + 64, 0);
    plain.offs.resize((size_t)plain.nb);
    plain.sizes.resize((size_t)plain.nb);
    ASSERT_EQ(0, obgpu_table_image_export(img, plain.image.data(), size, plain.offs.data(), plain.sizes.data(), plain.nb));
    obgpu_table_image_free(img);
    plain_size = size;
  }
  const int32_t nb = plain.nb;
  int32_t agg_cols[1] = {0};
  int64_t agg_size = 0;
  std::vector<int64_t> agg_off((size_t)nb + 1);
  ASSERT_EQ(0, obgpu_writer_table_agg_rows(cols, 5, agg_cols, 1, n, rpb, nullptr, 0, nullptr, &agg_size));
  std::vector<char> agg((size_t)agg_size);
  ASSERT_EQ(0, obgpu_writer_table_agg_rows(cols, 5, agg_cols, 1, n, rpb, agg.data(), agg_size, agg_off.data(), &agg_size));

  sql::ObWhiteFilterExecutor lt(1, sql::WHITE_OP_LT), bt(0, sql::WHITE_OP_BT);
  ObStorageDatum d;
  d.set_int(400); lt.get_datums().push_back(d);
  d.set_int(3 * rpb + 5); bt.get_datums().push_back(d);
  d.set_int(9 * rpb - 1); bt.get_datums().push_back(d);
  sql::ObAndFilterExecutor andf; andf.add_child(&bt); andf.add_child(&lt);
  const std::vector<int32_t> proj = {0, 2, 3, 1};

  for (int32_t comp : {OBGPU_COMPRESSOR_LZ4, OBGPU_COMPRESSOR_ZSTD_1_3_8, OBGPU_COMPRESSOR_ZLIB}) {
    Table st;
    st.nb = nb;
    st.image.assign(plain.image.size() + 64, 0);
    st.offs.resize((size_t)nb);
    st.sizes.resize((size_t)nb);
    int64_t used = 0;
    ASSERT_EQ(0, obgpu_writer_compress_blocks(plain.image.data(), plain.offs.data(), plain.sizes.data(), nb, comp, 1, st.image.data(),
                                              (int64_t)st.image.size(), st.offs.data(), st.sizes.data(), &used));
    int raw = 0;
    for (int32_t b = 0; b < nb; ++b) {
      int32_t len = 0, zlen = 0;
      memcpy(&len, st.image.data() + st.offs[(size_t)b] + 40, 4);
      memcpy(&zlen, st.image.data() + st.offs[(size_t)b] + 44, 4);
      raw += len == zlen;
    }
    ASSERT_EQ(1, raw < nb);
    for (int pipelined = 0; pipelined < 2; ++pipelined)
      for (int reverse = 0; reverse < 2; ++reverse)
        for (sql::ObPushdownFilterExecutor *f : {(sql::ObPushdownFilterExecutor *)&lt, (sql::ObPushdownFilterExecutor *)nullptr}) {
          ObGpuSSTableBatchScanner p(rt), s(rt);
          for (ObGpuSSTableBatchScanner *sc : {&p, &s}) {
            if (pipelined) sc->set_pipelined(3, 5);
            sc->set_reverse_scan(reverse == 1);
          }
          s.set_compressor(comp);
          ASSERT_EQ(OB_SUCCESS, p.init(plain.image.data(), plain_size, plain.offs.data(), plain.sizes.data(), nb, f, proj, 256));
          ASSERT_EQ(OB_SUCCESS, s.init(st.image.data(), used, st.offs.data(), st.sizes.data(), nb, f, proj, 256));
          const std::vector<std::string> rp = drain(p), rs = drain(s);
          ASSERT_EQ(1, !rp.empty() && same(rp, rs));
        }
    // LIMIT / OFFSET
    for (int pipelined = 0; pipelined < 2; ++pipelined) {
      ObGpuSSTableBatchScanner p(rt), s(rt);
      for (ObGpuSSTableBatchScanner *sc : {&p, &s}) {
        if (pipelined) sc->set_pipelined(2, 4);
        sc->set_limit(1000, 777);
      }
      s.set_compressor(comp);
      ASSERT_EQ(OB_SUCCESS, p.init(plain.image.data(), plain_size, plain.offs.data(), plain.sizes.data(), nb, &lt, proj, 100));
      ASSERT_EQ(OB_SUCCESS, s.init(st.image.data(), used, st.offs.data(), st.sizes.data(), nb, &lt, proj, 100));
      const std::vector<std::string> rp = drain(p), rs = drain(s);
      ASSERT_EQ(777, rs.size());
      ASSERT_EQ(1, same(rp, rs));
    }
    // skip-index infos: the same verdicts and the same pruned rows
    {
      std::vector<ObMicroIndexInfo> ip((size_t)nb), is((size_t)nb);
      for (int32_t i = 0; i < nb; ++i) {
        ip[(size_t)i].agg_row_buf_ = is[(size_t)i].agg_row_buf_ = agg.data() + agg_off[(size_t)i];
        ip[(size_t)i].agg_buf_size_ = is[(size_t)i].agg_buf_size_ = agg_off[(size_t)i + 1] - agg_off[(size_t)i];
      }
      ObGpuSSTableBatchScanner p(rt), s(rt);
      ASSERT_EQ(OB_SUCCESS, p.set_index_infos(ip.data(), nb));
      ASSERT_EQ(OB_SUCCESS, s.set_index_infos(is.data(), nb));
      s.set_compressor(comp);
      ASSERT_EQ(OB_SUCCESS, p.init(plain.image.data(), plain_size, plain.offs.data(), plain.sizes.data(), nb, &andf, proj, 256));
      ASSERT_EQ(OB_SUCCESS, s.init(st.image.data(), used, st.offs.data(), st.sizes.data(), nb, &andf, proj, 256));
      ASSERT_EQ(p.skipped_blocks(), s.skipped_blocks());
      ASSERT_EQ(p.unfiltered_blocks(), s.unfiltered_blocks());
      ASSERT_EQ(1, p.skipped_blocks() > 0);
      for (int32_t i = 0; i < nb; ++i) ASSERT_EQ(ip[(size_t)i].filter_constant_type_, is[(size_t)i].filter_constant_type_);
      ASSERT_EQ(1, same(drain(p), drain(s)));
    }
    // the row iterator, single batch and pipelined, and reuse()
    for (int pipelined = 0; pipelined < 2; ++pipelined) {
      ObGpuStoreRowIterator ip(rt), is(rt);
      if (pipelined) { ip.scanner().set_pipelined(3, 6); is.scanner().set_pipelined(3, 6); }
      is.scanner().set_compressor(comp);
      ASSERT_EQ(OB_SUCCESS, ip.init(plain.image.data(), plain_size, plain.offs.data(), plain.sizes.data(), nb, &lt, {1, 2, 3, 0}, 128));
      ASSERT_EQ(OB_SUCCESS, is.init(st.image.data(), used, st.offs.data(), st.sizes.data(), nb, &lt, {1, 2, 3, 0}, 128));
      const std::vector<bool> is_str = {false, true, true, false};
      const std::vector<std::string> rp = drain_iter(ip, is_str);
      ASSERT_EQ(1, !rp.empty() && same(rp, drain_iter(is, is_str)));
      ASSERT_EQ(OB_SUCCESS, is.reuse());
      ASSERT_EQ(1, same(rp, drain_iter(is, is_str)));
    }
    // the long DICT column three times, no filter: 600 decoded bytes per row against a payload of a few bytes per row, so the
    // pipelined path's first heap (the blocks' data_length_ sum) is too small and must grow; single batch and pipelined give the
    // generated cells
    for (int pipelined = 0; pipelined < 2; ++pipelined) {
      ObGpuSSTableBatchScanner s(rt);
      if (pipelined) s.set_pipelined(3, 5);
      s.set_compressor(comp);
      int64_t payload = 0;
      for (int32_t b = 0; b < nb; ++b) {
        int32_t len = 0;
        memcpy(&len, st.image.data() + st.offs[(size_t)b] + 40, 4);
        payload += len;
      }
      ASSERT_EQ(1, payload < n * 200);
      ASSERT_EQ(OB_SUCCESS, s.init(st.image.data(), used, st.offs.data(), st.sizes.data(), nb, nullptr, {4, 4, 4}, 512));
      const std::vector<std::string> rs = drain(s);
      ASSERT_EQ(n, rs.size());
      int bad = 0;
      for (int64_t i = 0; i < n && i < (int64_t)rs.size(); ++i) {
        const std::string cell = h_diff.substr((size_t)o_diff[i], 200);
        bad += rs[(size_t)i] != std::to_string(i / rpb) + "/" + std::to_string(i % rpb) + "|" + cell + "|" + cell + "|" + cell;
      }
      ASSERT_EQ(0, bad);
    }
  }
  if (g_fail) { printf("%d assertion(s) failed\n", g_fail); return 1; }
  printf("compressed host adapter tests passed\n");
  return 0;
}
