// The skip-index aggregate row of one micro-block as ObSkipIndexAggregator leaves it for MIN / MAX / NULL_COUNT
// (ObAggRowWriter, index_block/ob_agg_row_struct.cpp:49-300, version 3), shared by the host writer (sstable_writer.cpp:
// block_agg_row) and the device (agg_rows.cuh), so that the two agree byte for byte:
//   [ObAggRowHeader 8 B][col idx x cnt][cell offset x cnt] then one cell per aggregated column, in ascending column index:
//   [type bitmap 1 B][prefix bitmap 1 B][data offsets x (stored + 1)][MIN][MAX][NULL_COUNT 8 B], offsets relative to the cell
//   start, the last one being the cell end; a column without a stored aggregate has the two bitmaps only.
// The format is the writer's restatement of ObAggRowWriter; it is not pinned to the reference's bytes. obgpu_agg_row_write
// (arbitrary cells, versions 1-3) keeps the writer's general path.
#pragma once
#include <stdint.h>
#include <string.h>

#include "ob_format.h"   // OBF_HD, AggRowHeader

namespace obagg {

constexpr int kVersion = 3;          // what block_agg_row writes: prefix bitmap present
constexpr int kBitmaps = 2;          // type bitmap + prefix bitmap
constexpr int64_t kMaxRowSize = 65535;   // ObAggRowHeader::length_ is 16 bits: a longer row is OBGPU_NOT_SUPPORTED
enum : uint8_t { kMin = 0, kMax = 1, kNullCount = 2 };   // ObSkipIndexColType (OBGPU_SK_IDX_*)

// One aggregated column of a MIN / MAX / NULL_COUNT row. MIN and MAX are stored when min_len >= 0 (some cell is neither NULL
// nor NOP), NULL_COUNT when has_null_count (no NOP cell: a NOP makes the column "not aggregated", and then nothing is stored).
struct AggCol {
  uint32_t col_idx;
  int32_t min_len, max_len;   // -1: not stored
  const uint8_t *min, *max;   // images of min_len / max_len bytes
  uint8_t min_prefix, max_prefix;   // the image is a prefix of the value (strings longer than the skip index keeps)
  uint8_t has_null_count;
  int64_t null_count;
};

struct Layout {
  int idx_size, idx_off_size, cell_off_size;
  int64_t header_size, size;
};

OBF_HD int stored_cells(const AggCol &c) { return (c.min_len >= 0 ? 2 : 0) + (c.has_null_count ? 1 : 0); }

OBF_HD int64_t cell_bytes(const AggCol &c) {   // bitmaps + data, without the offsets
  return kBitmaps + (c.min_len >= 0 ? (int64_t)c.min_len + c.max_len : 0) + (c.has_null_count ? 8 : 0);
}

OBF_HD void put_le(uint8_t *p, uint64_t v, int bytes) {
  for (int k = 0; k < bytes; ++k) p[k] = (uint8_t)(v >> (8 * k));
}

// Sizes the row of n columns, col_at(k) being the k-th in ascending col_idx (no repeats). Returns the row's bytes, or -1
// when they exceed kMaxRowSize.
template <class ColAt>
OBF_HD int64_t layout(int n, const ColAt &col_at, Layout &l) {
  l.idx_size = 0;
  for (uint32_t m = col_at(n - 1).col_idx;;) { ++l.idx_size; m >>= 8; if (m == 0) break; }
  l.cell_off_size = 1;
  int64_t data = 0, offsets = 0;
  for (int k = 0; k < n; ++k) {
    const AggCol c = col_at(k);
    const int s = stored_cells(c);
    const int64_t stored = s > 0 ? s + 1 : 0;   // one more offset for the cell end
    const int64_t cell = cell_bytes(c);
    if (cell + stored > 255) l.cell_off_size = 2;
    data += cell;
    offsets += stored;
  }
  data += offsets * l.cell_off_size;
  l.idx_off_size = 1;
  l.header_size = (int64_t)sizeof(obf::AggRowHeader) + (int64_t)n * (l.idx_size + 1);
  if (data + l.header_size > 255) {
    l.idx_off_size = 2;
    l.header_size = (int64_t)sizeof(obf::AggRowHeader) + (int64_t)n * (l.idx_size + 2);
  }
  l.size = data + l.header_size;
  return l.size > kMaxRowSize ? -1 : l.size;
}

// Writes the row layout() sized into out[0, l.size): every byte is written.
template <class ColAt>
OBF_HD void write(int n, const ColAt &col_at, const Layout &l, uint8_t *out) {
  put_le(out + 0, (uint16_t)kVersion, 2);
  put_le(out + 2, (uint16_t)l.size, 2);
  put_le(out + 4, (uint16_t)n, 2);
  put_le(out + 6, (uint16_t)(l.idx_size | (l.idx_off_size << 6) | (l.cell_off_size << 9) | (1 << 12)), 2);
  uint8_t *idx_arr = out + sizeof(obf::AggRowHeader), *idx_off_arr = idx_arr + (int64_t)n * l.idx_size;
  int64_t pos = l.header_size;
  for (int k = 0; k < n; ++k) {
    const AggCol c = col_at(k);
    put_le(idx_arr + (int64_t)k * l.idx_size, c.col_idx, l.idx_size);
    put_le(idx_off_arr + (int64_t)k * l.idx_off_size, (uint64_t)pos, l.idx_off_size);
    const int64_t cell = pos;
    const int s = stored_cells(c);
    const bool mm = c.min_len >= 0;
    out[pos] = (uint8_t)((mm ? (1u << kMin) | (1u << kMax) : 0u) | (c.has_null_count ? 1u << kNullCount : 0u));
    out[pos + 1] = (uint8_t)(mm ? (c.min_prefix ? 1u << kMin : 0u) | (c.max_prefix ? 1u << kMax : 0u) : 0u);
    pos += kBitmaps;
    uint8_t *offs = out + pos;
    pos += (int64_t)(s > 0 ? s + 1 : 0) * l.cell_off_size;
    int w = 0;
    if (mm) {
      put_le(offs + (w++) * l.cell_off_size, (uint64_t)(pos - cell), l.cell_off_size);
      for (int32_t i = 0; i < c.min_len; ++i) out[pos + i] = c.min[i];
      pos += c.min_len;
      put_le(offs + (w++) * l.cell_off_size, (uint64_t)(pos - cell), l.cell_off_size);
      for (int32_t i = 0; i < c.max_len; ++i) out[pos + i] = c.max[i];
      pos += c.max_len;
    }
    if (c.has_null_count) {
      put_le(offs + (w++) * l.cell_off_size, (uint64_t)(pos - cell), l.cell_off_size);
      put_le(out + pos, (uint64_t)c.null_count, 8);
      pos += 8;
    }
    if (s > 0) put_le(offs + w * l.cell_off_size, (uint64_t)(pos - cell), l.cell_off_size);
  }
}

// Compare image of an integer-class datum (the writer's aggregate_column rule): the low datum_len bytes, sign-extended for
// signed classes; unsigned 8-byte values compare unsigned, every other image signed. key() maps an image to a signed key of
// the same order, so that min / max reduce as plain int64.
OBF_HD int64_t image(int64_t v, int store_class, int datum_len) {
  if (datum_len == 4) return store_class == 1 ? (int64_t)(int32_t)(uint32_t)v : (int64_t)(uint32_t)v;
  if (datum_len == 1) return (int64_t)(uint8_t)v;
  return v;
}
OBF_HD bool unsigned_order(int store_class, int datum_len) { return !(store_class == 1 || datum_len < 8); }
OBF_HD int64_t key(int64_t image, bool unsigned_cmp) {
  return unsigned_cmp ? (int64_t)((uint64_t)image ^ 0x8000000000000000ull) : image;
}

}  // namespace obagg
