// Small micro-blocks (a 16 KiB block of a wide dictionary-coded table holds ~130 rows): per block there are only a
// few hundred bytes to filter and a dozen rows to project, so a scan is bound by the per-block chain of dependent
// global round trips (record -> plans -> column bytes), not by bandwidth. These two kernels keep ONE WARP per block
// but run it as a software pipeline over the blocks it owns (persistent grid, blocks strided over the warps):
//
//     iteration b:   wait   regions(b), meta(b + 1)          (issued one / two iterations ago)
//                    issue  regions(b + 1)   <- needs meta(b + 1): block offset, decode plans -> column byte ranges
//                    issue  meta(b + 2)      <- block record, decode plans (and the two prefix entries)
//                    work   on block b from shared memory
//
// so a block's three round trips overlap the work on the two blocks before it. Meta copies are cp.async (LDGSTS: no
// registers), completed by cp.async.wait_group + __syncwarp; region copies are TMA bulk copies completing on one mbarrier per
// region slot. warp_pipeline owns that loop, its rings and its waits; each kernel gives it three steps -- issue a block's meta,
// issue its regions, work on it -- and reads each column's meta entry (a plan, or a stage record) through one set of helpers:
// issue_meta, staged_ranges, lean_leaf / flat_fill.
//   obgpu_count_pipe_kernel   : stages every filter column's region of the block at once, then the same leaf loops
//                               as obgpu_count_kernel (K4 / K6 / K9 / K14)
//   obgpu_project_pipe_kernel : stages the block's bitmap words and the projected columns' byte ranges; a projected
//                               VARCHAR dictionary column needs only its refs and its offset array (VEC_DISCRETE
//                               output is pointers into the caller's block: the dictionary's bytes are never read).
//                               "Flat" columns (project_flat) are decoded in one pass over (column, selected row)
//                               items, the others column after column
#pragma once

#include <type_traits>

__device__ __forceinline__ void cp_async16(uint32_t saddr, const void *g) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(saddr), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async8(uint32_t saddr, const void *g) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(saddr), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t saddr, const void *g) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(saddr), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// Where a warp's pipeline iteration goes (tools/scan_kernel_split.py builds a separate library with -DOBGPU_PIPE_CLOCKS; the
// product library never carries the stamps): per kernel, summed over the warps in clock64 cycles,
// [wait for regions(b) / meta(b + 1) | issue regions(b + 1) + meta(b + 2) | everything, loop start to end].
#ifdef OBGPU_PIPE_CLOCKS
__device__ unsigned long long g_pipe_clocks[2][3];
#define PIPE_CLOCK_START() const long long pclk_t0 = clock64(); long long pclk_wait = 0, pclk_issue = 0, pclk_a = 0, pclk_b = 0
#define PIPE_CLOCK_AT(v) v = clock64()
#define PIPE_CLOCK_ADD(acc, from) acc += clock64() - (from)
#define PIPE_CLOCK_STOP(k)                                                                   \
  if (lane == 0) {                                                                           \
    atomicAdd(&g_pipe_clocks[k][0], (unsigned long long)pclk_wait);                          \
    atomicAdd(&g_pipe_clocks[k][1], (unsigned long long)pclk_issue);                         \
    atomicAdd(&g_pipe_clocks[k][2], (unsigned long long)(clock64() - pclk_t0));              \
  }
#else
#define PIPE_CLOCK_START()
#define PIPE_CLOCK_AT(v)
#define PIPE_CLOCK_ADD(acc, from)
#define PIPE_CLOCK_STOP(k)
#endif

constexpr int kPipeMaxFilterCols = 8;
constexpr uint32_t kCountHdrBytes = 64u;   // count region slot: deltas + flags | regions
// meta slot: [block record | project: sel_offset[b], sel_offset[b + 1] | decode plans], copied in 16-byte pieces
// (the two sel_offset entries in 8-byte ones)
constexpr int kRecPieces = (int)(sizeof(BlockRec) / 16);
constexpr uint32_t kMetaSel = (uint32_t)sizeof(BlockRec), kMetaPlans = kMetaSel + 2u * (uint32_t)sizeof(int64_t);
static_assert(kMetaPlans % 16u == 0u, "decode plans are copied in 16-byte pieces");

// ---- lean leaf pieces for blocks of at most 1024 rows (bitmap in registers, lane g owns word g) ----------------------
// Range leaf over the fixed-width integer dictionary of a K_DICT column -> predicate bitset (bit count = NULL: never set).
template <class D>
__device__ __forceinline__ void lean_bitset_int_range(const D &d, const FilterNodeDev &nd, uint32_t sbit, uint32_t *bits, int lane) {
  const uint32_t n = d.dict_count;
  const uint64_t lo = nd.lo, span = nd.span;
  const bool neg = nd.negate != 0;
  for (uint32_t b0 = 0; b0 < n + 2u; b0 += 32u) {
    const uint32_t idx = b0 + (uint32_t)lane;
    bool r = false;
    if (idx < n) r = (((uint64_t)cmp_image(d, dict_int_s(sbit, d, idx)) - lo) <= span) != neg;
    const uint32_t word = __ballot_sync(0xffffffffu, r);
    if (lane == 0) bits[b0 >> 5] = word;
  }
}

// Rows of a K_DICT column against a predicate over refs -- a bitset in shared memory (BITSET) or a ref interval
// [a, e), complemented inside [0, count) when neg (sorted dictionary). Lane g collects word g; returns the lane's
// updated bitmap word.
template <bool BITSET, class D>
__device__ __forceinline__ uint32_t lean_rows(const D &d, uint32_t sbit, const uint32_t *bits, uint32_t a, uint32_t e, bool neg,
                                              uint32_t mybm, uint32_t myvalid, uint32_t nwords, bool and_mode, int lane) {
  const uint32_t step = 32u * d.stride, width = d.width, dcount = d.dict_count, cntp1 = dcount + 1u, span = e - a;
  uint32_t bit = sbit + d.val_bit + (uint32_t)lane * d.stride, acc = 0;
  for (uint32_t g = 0; g < nwords; ++g, bit += step) {
    // lanes past the last row read a few refs beyond the column (inside the warp's shared memory): masked by myvalid
    const uint32_t ref = sbits32(bit, width);
    bool hit;
    if (BITSET) {
      const uint32_t rr = min(ref, cntp1);
      hit = (bits[rr >> 5] >> (rr & 31u)) & 1u;
    } else {
      hit = ((ref - a) < span) != (neg && ref < dcount);
    }
    const uint32_t w = __ballot_sync(0xffffffffu, hit);
    if ((uint32_t)lane == g) acc = w;
  }
  acc &= myvalid;
  return and_mode ? (mybm & acc) : (mybm | acc);
}

// Sorted fixed-width integer dictionary and a range leaf: the matching refs are [a, e) = [#entries below the range,
// #entries not above it) (the reference binary-searches the bounds, ob_dict_decoder.cpp:967-988,1085-1176).
template <class D>
__device__ __forceinline__ void lean_interval_sorted_int(const D &d, const FilterNodeDev &nd, uint32_t sbit, int lane,
                                                         uint32_t &a, uint32_t &e) {
  const uint32_t n = d.dict_count;
  const uint64_t lo = nd.lo, hi = nd.lo + nd.span;
  const bool sg = d.sc == 1;
  uint32_t below = 0, not_above = 0;
  for (uint32_t b0 = 0; b0 < n; b0 += 32u) {
    const uint32_t idx = b0 + (uint32_t)lane;
    bool lt = false, le = false;
    if (idx < n) {
      const uint64_t v = (uint64_t)cmp_image(d, dict_int_s(sbit, d, idx));
      lt = sg ? (int64_t)v < (int64_t)lo : v < lo;
      le = sg ? (int64_t)v <= (int64_t)hi : v <= hi;
    }
    below += __popc(__ballot_sync(0xffffffffu, lt));
    not_above += __popc(__ballot_sync(0xffffffffu, le));
  }
  a = below;
  e = not_above < below ? below : not_above;
}

// Equality screen of an EQ / NE / IN leaf for the string of `len` bytes at block offset `cell`, built on the host:
// does any constant have this length (most strings stop here), then either the hash slot of (length, first 8 bytes)
// -- it names the only constant the string can equal -- or the first-byte screen + the whole list. Returns the first
// 8 bytes; the constants left to compare are [k0, k1).
__device__ __forceinline__ uint64_t str_eq_screen(const FilterNodeDev &nd, uint32_t sbit, uint32_t cell, uint32_t len, int &k0, int &k1) {
  const uint32_t pl = len < 8u ? len : 8u;
  const uint64_t pre = pl ? sbits(sbit + cell * 8u, pl * 8u) : 0ull;
  k0 = k1 = 0;
  if ((nd.lo >> (len & 63u)) & 1ull) {
    if (nd.pad) {   // 0: first-byte screen + constant list; m + 1: hash slots under multiplier m
      const uint32_t h = str_eq_slot(pre, len, nd.pad - 1);
      if ((nd.span >> h) & 1ull) { k0 = __popcll(nd.span & ((1ull << h) - 1ull)); k1 = k0 + 1; }
    } else if (len == 0u || ((nd.span >> (pre & 63ull)) & 1ull)) {
      k1 = nd.n_params;
    }
  }
  return pre;
}

// EQ / NE / IN leaf over the string dictionary of a K_DICT column -> predicate bitset. Every entry is screened by
// (length, first 8 bytes) against the constants; only the (few) entries that pass compare their tails, 8 bytes at a
// time, out of shared memory.
template <class D>
__device__ __forceinline__ void lean_bitset_str_eq(const ScanParams &p, const FilterNodeDev &nd, const D &d, uint32_t sbit,
                                                   uint32_t *bits, int lane) {
  const uint32_t n = d.dict_count;
  const bool ne = nd.op == OP_NE;
  for (uint32_t b0 = 0; b0 < n + 2u; b0 += 32u) {
    const uint32_t idx = b0 + (uint32_t)lane;
    bool r = false;
    if (idx < n) {
      uint32_t cell, len;
      dict_str_s(sbit, d, idx, cell, len);
      int k0, k1;
      const uint64_t pre = str_eq_screen(nd, sbit, cell, len, k0, k1);
      for (int k = k0; k < k1 && !r; ++k) {
        const ParamDev &pp = p.params[nd.param_begin + k];
        if (pp.len != len || (uint64_t)pp.i64 != pre) continue;
        bool same = true;
        for (uint32_t i = 8u; i < len && same; i += 8u) {
          const uint32_t nb = len - i < 8u ? len - i : 8u;
          const uint64_t a = sbits(sbit + (cell + i) * 8u, nb * 8u);
          const uint64_t c = *reinterpret_cast<const uint64_t *>(p.param_heap + pp.heap_off + i) & (~0ull >> (64u - nb * 8u));
          same = a == c;
        }
        r = same;
      }
      r = r != ne;
    }
    const uint32_t word = __ballot_sync(0xffffffffu, r);
    if (lane == 0) bits[b0 >> 5] = word;
  }
}

// AND leaf on a string K_DICT column when few rows are still alive: evaluate the leaf on the survivors' own
// dictionary entries (one pass over <= alive rows) instead of on every dictionary entry.
template <class D>
__device__ __forceinline__ uint32_t lean_survivor_str(const ScanParams &p, const FilterNodeDev &nd, const D &d, uint32_t sbit,
                                                      const uint8_t *rs_generic, uint32_t mybm, uint32_t nwords, uint32_t alive,
                                                      uint32_t *bm, int lane) {
  // survivor list (ascending rows) in the spilled-bitmap scratch: uint16 rows after the 32 bitmap words
  uint16_t *list = reinterpret_cast<uint16_t *>(bm + 32);
  warp_select_group(mybm, nwords, 0u, 0u, list, lane);
  bm[lane] = mybm;
  __syncwarp();
  const uint32_t vbit = sbit + d.val_bit, stride = d.stride, width = d.width, dcount = d.dict_count;
  const int op = nd.op;
  const uint8_t *s = rs_generic;   // generic pointer for the (rare) full string compare
  for (uint32_t j = (uint32_t)lane; j < alive; j += 32u) {
    const uint32_t row = list[j];
    const uint32_t ref = sbits32(vbit + row * stride, width);
    bool pass;
    if (ref >= dcount) pass = op == OP_NU;
    else if (op == OP_NU) pass = false;
    else if (op == OP_NN) pass = true;
    else {
      uint32_t cell, len;
      dict_str_s(sbit, d, ref, cell, len);
      if (op == OP_EQ || op == OP_NE || op == OP_IN) {
        int k0, k1;
        const uint64_t pre = str_eq_screen(nd, sbit, cell, len, k0, k1);
        bool hit = false;
        for (int k = k0; k < k1 && !hit; ++k) {
          const ParamDev &pp = p.params[nd.param_begin + k];
          hit = pp.len == len && (uint64_t)pp.i64 == pre && (len <= 8u || str_cmp(s, cell, len, p.param_heap + pp.heap_off, pp.len) == 0);
        }
        pass = hit != (op == OP_NE);
      } else {
        pass = str_pred(p, nd, s, cell, len);
      }
    }
    if (!pass) atomicAnd(&bm[row >> 5], ~(1u << (row & 31u)));
  }
  __syncwarp();
  return (uint32_t)lane < nwords ? bm[lane] : 0u;
}

// A stage record (scan_device.cuh) in a meta slot read under the plan's field names, with the column's type facts of the
// scan (store class, datum length, sign-fix mask: the same for every block of a column whose blocks agree on its type): the
// lean leaves and flat_fill take either a plan or this. desc_of gives used column `used`'s descriptor from its meta-slot entry.
struct RecDesc {
  uint64_t base, int_mask;
  uint32_t val_bit, stride, width, dict_count, dict_payload, dict_data_size, dict_var, dict_end;
  uint8_t kind, sc, elem_len, sign_fix, dict_sorted, dict_fixed;
};
__device__ __forceinline__ const ColDesc &desc_of(const ScanParams &, const ColDesc &d, int) { return d; }
__device__ __forceinline__ RecDesc desc_of(const ScanParams &p, const StageRec &r, int used) {
  RecDesc d;
  d.sc = p.used_sc[used];
  d.elem_len = p.used_elem_len[used];
  d.kind = (r.flags & SR_DICT) ? K_DICT : K_BITS;
  d.sign_fix = (r.flags & SR_SIGN_FIX) != 0;
  d.int_mask = d.sign_fix ? p.used_int_mask[used] : 0ull;
  const bool str = d.kind == K_DICT && d.sc == 5;
  d.base = str ? 0ull : r.add;
  d.dict_var = str ? (uint32_t)r.add : 0u;
  d.dict_end = d.dict_var + r.last_end;
  d.val_bit = r.val_bit;
  d.stride = r.stride;
  d.width = r.width;
  d.dict_count = r.dict_count;
  d.dict_payload = r.dict_payload;
  d.dict_data_size = r.dict_data_size;
  d.dict_sorted = (r.flags & SR_SORTED) != 0;
  d.dict_fixed = 0;   // string dictionaries with records have variable-length entries (stage_rec_of)
  return d;
}
// Meta-slot entry of a column: its plan, or its stage record (count) / its stage record with room for the FlatCol entry
// flat_fill writes over it (projection).
template <bool REC> using MetaEnt = typename std::conditional<REC, StageRec, ColDesc>::type;
template <bool REC> constexpr uint32_t kCountEnt = (uint32_t)sizeof(MetaEnt<REC>);
template <bool REC> constexpr uint32_t kProjEnt = REC ? 64u : (uint32_t)sizeof(ColDesc);

// One lean leaf on the K_DICT column of descriptor d (width <= 32) staged at sbit (generic address rs_col): returns the lane's
// bitmap word. A plan's leaf that is neither an integer range nor a string EQ / NE / IN falls back to the generic dictionary bitset
// (build_dict_bitset, over bv pointed at the staged column); layout_pipe gives a scan records only when no leaf needs it.
template <class D>
__device__ __forceinline__ uint32_t lean_leaf(const ScanParams &p, const FilterNodeDev &nd, const D &d, uint32_t sbit, const uint8_t *rs_col,
                                              uint32_t *bits, uint32_t *bm, uint32_t mybm, uint32_t myvalid, uint32_t nwords,
                                              bool and_mode, BlockView &bv, const Team &t, int lane) {
  constexpr bool kPlan = std::is_same<D, ColDesc>::value;
  const bool is_str = d.sc == 5;
  if (is_str && and_mode) {
    // few surviving rows and a larger dictionary: test the survivors' own entries instead of every entry
    const uint32_t alive = warp_sum_u32(__popc(mybm));
    if (alive * 4u <= d.dict_count) return lean_survivor_str(p, nd, d, sbit, rs_col, mybm, nwords, alive, bm, lane);
  }
  if (!is_str && nd.range_ok && d.dict_sorted) {
    uint32_t a, e;
    lean_interval_sorted_int(d, nd, sbit, lane, a, e);
    return lean_rows<false>(d, sbit, nullptr, a, e, nd.negate != 0, mybm, myvalid, nwords, and_mode, lane);
  }
  if (!is_str && nd.range_ok) {
    lean_bitset_int_range(d, nd, sbit, bits, lane);
  } else if (!kPlan || (is_str && (nd.op == OP_EQ || nd.op == OP_NE || nd.op == OP_IN))) {
    lean_bitset_str_eq(p, nd, d, sbit, bits, lane);
  } else if constexpr (kPlan) {
    bv.s = rs_col;
    build_dict_bitset(p, bv, d, nd, bits, t);
  }
  __syncwarp();
  return lean_rows<true>(d, sbit, bits, 0u, 0u, false, mybm, myvalid, nwords, and_mode, lane);
}

// Issues block b's meta slot at shared address sa: the block record, for the projection (SEL) the two sel_offset entries, then n
// entries from the block's plans or (REC) stage records, entry i taken from column col(i) into kEnt bytes at kMetaPlans + i kEnt.
template <bool REC, bool SEL, uint32_t kEnt, class Col>
__device__ __forceinline__ void issue_meta(const ScanParams &p, int b, uint32_t sa, int n, Col col, int lane) {
  constexpr uint32_t kSrc = (uint32_t)sizeof(MetaEnt<REC>);
  constexpr int kSrcPieces = (int)(kSrc / 16u), kHead = kRecPieces + (SEL ? 2 : 0);
  const uint8_t *rec = reinterpret_cast<const uint8_t *>(p.recs + b);
  const uint8_t *src = REC ? reinterpret_cast<const uint8_t *>(p.stage + (int64_t)b * p.max_cols)
                           : reinterpret_cast<const uint8_t *>(p.plans + (int64_t)b * p.max_cols);
  for (int q = lane; q < kHead + n * kSrcPieces; q += 32) {
    if (q < kRecPieces) cp_async16(sa + (uint32_t)q * 16u, rec + q * 16);
    else if (q < kHead) cp_async8(sa + kMetaSel + (uint32_t)(q - kRecPieces) * 8u, p.sel_offset + b + (q - kRecPieces));
    else {
      const int i = (q - kHead) / kSrcPieces, piece = (q - kHead) % kSrcPieces;
      cp_async16(sa + kMetaPlans + (uint32_t)i * kEnt + (uint32_t)piece * 16u, src + (size_t)col(i) * kSrc + piece * 16);
    }
  }
}

// Byte ranges r = {lo0, hi0, lo1, hi1} of block rec that a kernel stages for the column of meta-slot entry ent: its filter
// region (FILTER: [16 lo[0], 16 max(hi)) of a record, col_region of a plan) or its projection ranges (the record's, or
// proj_ranges). Returns how many (1, or 2 for a string dictionary's refs and END offsets), or 0 -- r all zero -- when the column has
// no bounded range, or its ranges exceed the column's budget or run past the block's padded end.
template <bool REC, bool FILTER>
__device__ __forceinline__ int staged_ranges(const BlockRec &rec, const uint8_t *ent, uint32_t budget, uint32_t r[4]) {
  int nr;
  if constexpr (REC) {
    const StageRec &sr = *reinterpret_cast<const StageRec *>(ent);
    r[0] = (uint32_t)sr.lo[0] * 16u;
    r[1] = (uint32_t)(FILTER ? max(sr.hi[0], sr.hi[1]) : sr.hi[0]) * 16u;
    r[2] = FILTER ? 0u : (uint32_t)sr.lo[1] * 16u;
    r[3] = FILTER ? 0u : (uint32_t)sr.hi[1] * 16u;
    nr = r[3] != r[2] ? 2 : 1;
  } else {
    BlockView bv;
    view_from_rec(rec, nullptr, bv);
    const ColDesc &d = *reinterpret_cast<const ColDesc *>(ent);
    if (FILTER) nr = d.ok && col_region(d, bv, r[0], r[1]) ? 1 : 0;
    else nr = d.ok ? proj_ranges(d, bv, r) : 0;
  }
  const uint32_t lim = ((rec.size + 15u) & ~15u) + 32u;
  if (nr > 0 && ((r[1] - r[0]) + (nr == 2 ? r[3] - r[2] : 0u) > budget || r[1] > lim || (nr == 2 && r[3] > lim))) nr = 0;
  if (nr == 0) r[0] = r[1] = r[2] = r[3] = 0;
  return nr;
}

// Staged bit addresses of a string dictionary's refs (rbit) and END offsets (ibit) from the slot deltas d0, d1 of its projection
// ranges: with two ranges they are ordered by block offset (proj_ranges); with one (d0 == d1) both are in it.
template <class D>
__device__ __forceinline__ void str_dict_bits(const D &d, uint32_t rs_addr, int32_t d0, int32_t d1, uint32_t &rbit, uint32_t &ibit) {
  const uint32_t s0 = (rs_addr + (uint32_t)d0) * 8u, s1 = (rs_addr + (uint32_t)d1) * 8u;
  const bool refs_first = (d.val_bit >> 3) < d.dict_payload;
  rbit = refs_first ? s0 : s1;
  ibit = refs_first ? s1 : s0;
}

// The warp pipeline of both kernels. Warp w of the persistent grid takes blocks w, w + W, w + 2W, ... (W: every warp of the grid)
// through a meta ring of 3 slots and a region ring of 2 slots, with one mbarrier per region slot at bars. The kernel owns the slots'
// layout and gives three steps, each called with the ring slots it is to use:
//   meta(b, ms)              issue the cp.async copies of block b's meta into meta slot ms
//   regions(b, ms, rsl)      from block b's landed meta slot ms, issue its region slot rsl (one mbar_expect_tx on bars[rsl], even
//                            with nothing to copy, so the slot's phase completes)
//   work(b, ms, rsl)         block b, with both of its slots landed
// meta and regions are also called one and two blocks past the warp's last block and then return at once (the test sits in them:
// in this loop it costs the plan kernels spills). K names the kernel's PIPE_CLOCK counters.
template <int K, class Meta, class Regions, class Work>
__device__ __forceinline__ void warp_pipeline(int n_blocks, uint64_t *bars, int lane, Meta meta, Regions regions, Work work) {
  const int stride = (int)gridDim.x * kWarps;
  int blk = (int)blockIdx.x * kWarps + (int)(threadIdx.x >> 5);
  if (blk >= n_blocks) return;
  if (lane == 0) {
    mbar_init(bars, 1);
    mbar_init(bars + 1, 1);
    fence_barrier_init();
  }
  __syncwarp();
  // prologue: meta(b0), then regions(b0) + meta(b1)
  meta(blk, 0);
  cp_async_commit();
  cp_async_wait_all();
  __syncwarp();
  regions(blk, 0, 0);
  cp_async_commit();
  meta(blk + stride, 1);
  cp_async_commit();
  int it = 0;
  PIPE_CLOCK_START();
  for (; blk < n_blocks; blk += stride, ++it) {
    const int rsl = it & 1;
    PIPE_CLOCK_AT(pclk_a);
    cp_async_wait_all();
    mbar_wait(bars + rsl, (uint32_t)(it >> 1) & 1u);
    __syncwarp();
    PIPE_CLOCK_ADD(pclk_wait, pclk_a);
    PIPE_CLOCK_AT(pclk_b);
    regions(blk + stride, (it + 1) % 3, rsl ^ 1);
    cp_async_commit();
    meta(blk + 2 * stride, (it + 2) % 3);
    cp_async_commit();
    PIPE_CLOCK_ADD(pclk_issue, pclk_b);
    work(blk, it % 3, rsl);
    __syncwarp();   // every lane is done with this iteration's slots before the next iteration refills them
  }
  PIPE_CLOCK_STOP(K);
  cp_async_wait_all();
}

// =================================================================================================
// Count, pipelined. Per warp: meta ring (3 slots: block record + the filter columns' plans, or their stage records when
// REC), region ring (2 slots: header with the per-column deltas + the filter columns' regions), bitmap words, predicate bitsets.
// =================================================================================================
template <bool REC>
__global__ void __launch_bounds__(kThreads) obgpu_count_pipe_kernel(const __grid_constant__ ScanParams p) {
  constexpr uint32_t kEnt = kCountEnt<REC>;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t *wr = g_smem + (uint32_t)warp * p.pc_bytes;
  uint32_t *bm = reinterpret_cast<uint32_t *>(wr + p.pc_bm);
  uint32_t *bitsets = reinterpret_cast<uint32_t *>(wr + p.pc_bitset);
  const int nf = p.pf_n;
  const Team t = warp_team(lane);
  // skip-index verdict of the block whose meta was issued last: fetched two blocks ahead of the block's work, it decides whether
  // regions() stages the block and travels to work() in the region slot's header
  uint32_t verdict = 0;

  uint8_t *meta0 = wr + p.pc_meta, *reg0 = wr + p.pc_region;
  uint64_t *bars = reinterpret_cast<uint64_t *>(wr + p.pc_bar);
  auto meta = [&](int b, int ms) {
    if (b >= p.n_blocks) return;
    uint8_t *m = meta0 + (uint32_t)ms * p.pc_meta_bytes;
    if (p.blk_const != nullptr) verdict = p.blk_const[b];
    issue_meta<REC, false, kEnt>(p, b, smem_u32(m), nf, [&](int i) { return p.used_col[i]; }, lane);
  };
  // region slot: [int32 delta[kPipeMaxFilterCols] | declined mask | verdict] (64 bytes) then the regions at p.pf_off[i]
  auto regions = [&](int b, int ms, int rsl) {
    if (b >= p.n_blocks) return;
    const uint8_t *m = meta0 + (uint32_t)ms * p.pc_meta_bytes;
    uint8_t *rs = reg0 + (uint32_t)rsl * p.pc_region_bytes;
    uint64_t *bar = bars + rsl;
    const BlockRec &rec = *reinterpret_cast<const BlockRec *>(m);
    int32_t *hdr = reinterpret_cast<int32_t *>(rs);
    uint32_t r[4] = {0, 0, 0, 0};
    bool bad = false;
    if (lane < nf && rec.rows != 0 && verdict == 0) {
      bad = staged_ranges<REC, true>(rec, m + kMetaPlans + (uint32_t)lane * kEnt, p.pf_span[lane], r) == 0;
      hdr[lane] = (int32_t)(kCountHdrBytes + p.pf_off[lane]) - (int32_t)r[0];
    }
    const uint32_t badmask = __ballot_sync(0xffffffffu, bad);
    if (lane == 0) {
      hdr[kPipeMaxFilterCols] = (int32_t)badmask;
      hdr[kPipeMaxFilterCols + 1] = (int32_t)verdict;
    }
    // one bulk copy (TMA) per filter column, all completing on the slot's mbarrier
    const uint32_t total = warp_sum_u32(r[1] - r[0]);
    if (lane == 0) mbar_expect_tx(bar, total);
    __syncwarp();
    if (r[1] > r[0]) tma_bulk_g2s(rs + kCountHdrBytes + p.pf_off[lane], p.image + rec.off + r[0], r[1] - r[0], bar);
  };

  auto work = [&](int blk, int ms, int rsl) {
    const uint8_t *m = meta0 + (uint32_t)ms * p.pc_meta_bytes;
    uint8_t *rs = reg0 + (uint32_t)rsl * p.pc_region_bytes;
    const BlockRec rec = *reinterpret_cast<const BlockRec *>(m);
    const int32_t *hdr = reinterpret_cast<const int32_t *>(rs);
    const uint32_t rows = rec.rows;
    uint32_t *gbm = p.bitmap_words + rec.bm_word_off;
    const uint32_t nwords = (rows + 31u) >> 5;
    if (count_block_settled(p, blk, rows, gbm, (uint32_t)hdr[kPipeMaxFilterCols + 1], hdr[kPipeMaxFilterCols] != 0, lane)) return;
    const MetaEnt<REC> *ents = reinterpret_cast<const MetaEnt<REC> *>(m + kMetaPlans);
    BlockCtx c;
    view_from_rec(rec, nullptr, c.b);
    c.descs = reinterpret_cast<const ColDesc *>(ents);
    c.bitsets = bitsets;
    c.rle_base = nullptr;
    c.rle_slot_bytes = c.rle_starts_bytes = 0;
    const bool and_mode = p.simple_shape == 1;
    const int n_leaves = p.n_nodes == 1 ? 1 : p.n_nodes - 1;
    // every filter column is staged: block-relative offsets of a leaf's column resolve into its region
    auto staged_at = [&](const FilterNodeDev &nd, const ColDesc &, BlockCtx &cs) {
      if (nd.op != OP_FALSE && nd.op != OP_TRUE) {
        cs.b.s = rs + hdr[nd.used_idx];
        cs.sbit = (smem_u32(rs) + (uint32_t)hdr[nd.used_idx]) * 8u;
      }
      return true;
    };
    uint32_t cnt = 0;
    if (REC || nwords <= 32u) {
      // ---- lean path (with records every block has at most 1024 rows: layout_pipe): the block's bitmap lives in registers
      // (lane g owns word g); dictionary-coded leaves run through explicit shared-memory loads, everything else (plans only)
      // through the generic leaf code on a spilled bitmap
      const uint32_t myvalid = (uint32_t)lane < nwords ? valid_mask_of(rows, (uint32_t)lane) : 0u;
      uint32_t mybm = and_mode ? myvalid : 0u;
      for (int i = 0; i < n_leaves; ++i) {
        const FilterNodeDev &nd = p.nodes[i];
        if (p.leaf_const != nullptr && p.leaf_const[(int64_t)blk * p.n_nodes + i] != 0) continue;
        const auto &d = desc_of(p, ents[nd.used_idx], nd.used_idx);
        // with records every leaf is lean (layout_pipe)
        if (REC || (d.kind == K_DICT && nd.slot >= 0 && nd.op != OP_FALSE && nd.op != OP_TRUE && d.width <= 32u)) {
          mybm = lean_leaf(p, nd, d, (smem_u32(rs) + (uint32_t)hdr[nd.used_idx]) * 8u, rs + hdr[nd.used_idx],
                           bitsets + nd.slot * p.bitset_words, bm, mybm, myvalid, nwords, and_mode, c.b, t, lane);
        } else {
          bm[lane] = mybm;   // words_cap >= 32 words are reserved for the spilled bitmap
          __syncwarp();
          bool inited = true;
          leaf_step(p, c, c, nd, false, inited, bm, rows, nwords, and_mode, t, staged_at);
          mybm = (uint32_t)lane < nwords ? bm[lane] : 0u;
        }
        if (i + 1 < n_leaves && !__any_sync(0xffffffffu, and_mode ? mybm != 0u : mybm != myvalid)) break;   // early-out
      }
      if ((uint32_t)lane < nwords) gbm[lane] = mybm;
      cnt = __popc(mybm);
    } else {
      // leaf_list_over_words written out: at 64 registers the shared loop costs this kernel 4 bytes of spills
      bool inited = false;
      for (int i = 0; i < n_leaves; ++i) {
        const FilterNodeDev &nd = p.nodes[i];
        if (p.leaf_const != nullptr && p.leaf_const[(int64_t)blk * p.n_nodes + i] != 0) continue;
        if (nd.op != OP_FALSE && nd.op != OP_TRUE) {
          c.b.s = rs + hdr[nd.used_idx];
          c.sbit = (smem_u32(rs) + (uint32_t)hdr[nd.used_idx]) * 8u;
        }
        const ColDesc &d = c.descs[nd.used_idx];
        if (nd.slot >= 0 && is_dict_kind(d)) {
          build_dict_bitset(p, c.b, d, nd, bitsets + nd.slot * p.bitset_words, t);
          __syncwarp();
        }
        if (i == 0 && leaf_first_fast<false>(p, c, nd, bm, rows, nwords, t)) {
          inited = true;
          __syncwarp();
          continue;
        }
        if (!inited) {
          for (uint32_t g = (uint32_t)lane; g < nwords; g += 32u) bm[g] = and_mode ? valid_mask_of(rows, g) : 0u;
          inited = true;
          __syncwarp();
        }
        leaf_over_words<false>(p, c, nd, bm, rows, nwords, and_mode, t);
        __syncwarp();
        if (i + 1 < n_leaves) {
          bool undecided = false;
          for (uint32_t g = (uint32_t)lane; g < nwords; g += 32u)
            undecided = undecided || (and_mode ? bm[g] != 0u : bm[g] != valid_mask_of(rows, g));
          if (!__any_sync(0xffffffffu, undecided)) break;
        }
      }
      if (!inited) {
        for (uint32_t g = (uint32_t)lane; g < nwords; g += 32u) bm[g] = and_mode ? valid_mask_of(rows, g) : 0u;
        __syncwarp();
      }
      for (uint32_t g = (uint32_t)lane; g < nwords; g += 32u) {
        const uint32_t w = bm[g];
        gbm[g] = w;
        cnt += __popc(w);
      }
    }
    cnt = warp_sum_u32(cnt);
    if (lane == 0) p.counts[blk] = cnt;
  };

  warp_pipeline<0>(p.n_blocks, bars, lane, meta, regions, work);
}

// =================================================================================================
// Projection, pipelined. Meta slot: [record | sel_offset pair | n_proj plans] (kMetaSel, kMetaPlans); region slot:
// [header: per column {delta0, delta1} + flags | bitmap words | column byte ranges at p.pp_off[pc]].
// =================================================================================================
#define ROW(j) (IDENT ? (uint32_t)(j) : (uint32_t)sel[j])
template <bool IDENT>
__device__ __forceinline__ void project_str_dict_shallow(const ScanParams &p, const ColDesc &d, int pc, const uint16_t *sel,
                                                         uint32_t cnt, int64_t base_row, uint64_t blk_addr, uint32_t ref_sbit,
                                                         uint32_t idx_sbit, int lane) {
  uint64_t *optr = reinterpret_cast<uint64_t *>(p.out_data[pc]) + base_row;
  int32_t *olen = p.out_lens[pc] + base_row;
  const uint32_t vbit = ref_sbit + d.val_bit, stride = d.stride, width = d.width, dcount = d.dict_count;
  bool saw_null = false;
  for (uint32_t j = (uint32_t)lane; j < cnt; j += 32u) {
    const uint32_t ref = sbits32(vbit + ROW(j) * stride, width);
    uint32_t cell = 0, len = 0;
    const bool is_null = ref >= dcount;
    if (!is_null) dict_str_s(idx_sbit, d, ref, cell, len);
    __stcs(&optr[j], is_null ? 0ull : blk_addr + cell);
    __stcs(&olen[j], is_null ? 0 : (int32_t)len);
    if (is_null) {
      const int64_t o = base_row + (int64_t)j;
      atomicOr(&p.out_nulls[pc][o >> 5], 1u << (o & 31));
      saw_null = true;
    }
  }
  if (saw_null) p.has_null[pc] = 1;
}
#undef ROW

// "Flat" projected columns: a row's output is one ref / value load plus at most two dictionary loads, with no per-block
// table to build first -- K_BITS without ext bits, sign fix or replaced NULLs, K_DICT over a fixed-width integer
// dictionary, K_DICT over a variable-length string dictionary (pointer + length, as project_str_dict_shallow). Lane pc turns
// the column's plan into a FlatCol entry once per block, written over the plan itself in the block's meta slot (no extra
// shared memory: a table of its own per warp made the kernel slower, fewer warps fit an SM); the list of flat columns goes over the
// block record at the slot's start, already copied to registers. Then the lanes walk all (column, selected row) items together.
enum : uint8_t { FLAT_BITS = 0, FLAT_INT_DICT = 1, FLAT_STR_DICT = 2 };
struct FlatCol {
  uint64_t add;        // K_BITS / integer dictionary: the plan's base; string dictionary: string address of its var data
  uint64_t mask;       // integer dictionary with sign fix: int_mask, else 0
  uint8_t *out;        // output at the block's first selected row
  int32_t *olen;       // string dictionary: lengths at the block's first selected row
  uint32_t vbit, width, stride;   // value / ref of row r at staged bit vbit + r * stride, width bits
  uint32_t dcount, dbit, dbits;   // dictionary: entries, staged bit of entry 0 (string: END offsets), bits per entry
  uint32_t last_end;   // string dictionary: END of the last entry, relative to the var data
  uint8_t kind, elem_len, pc, pad_;
};
static_assert(sizeof(FlatCol) <= sizeof(ColDesc) && sizeof(FlatCol) <= kProjEnt<true>, "a flat entry replaces its column's plan or record");
static_assert(kMetaPlans >= kMaxProj, "the flat column list (one byte per column) fits before the plans");

// Entry of projected column pc (flat_kind) from its plan or stage record and its staged byte ranges (slot deltas d0, d1). Not
// inlined: once per block, and inlined into obgpu_project_pipe_kernel it costs the kernel spills at 64 registers.
// dst overlays src: the entry is built in registers and stored with memcpy, whose byte stores may alias any type, so
// no load of src can move past them.
template <class S>
__device__ __noinline__ void flat_fill(const ScanParams &p, const S &src, int pc, uint32_t rs_addr, int32_t d0, int32_t d1,
                                       int64_t base, uint64_t blk_addr, void *dst) {
  const auto &d = desc_of(p, src, p.proj_used[pc]);
  FlatCol f;
  uint32_t rbit = (rs_addr + (uint32_t)d0) * 8u, ibit = rbit;
  f.kind = d.kind == K_BITS ? FLAT_BITS : d.sc == 5 ? FLAT_STR_DICT : FLAT_INT_DICT;
  if (f.kind == FLAT_STR_DICT) str_dict_bits(d, rs_addr, d0, d1, rbit, ibit);
  f.elem_len = f.kind == FLAT_STR_DICT ? 8u : d.elem_len;
  f.pc = (uint8_t)pc;
  f.pad_ = 0;
  f.out = reinterpret_cast<uint8_t *>(p.out_data[pc]) + base * (int64_t)f.elem_len;
  f.olen = f.kind == FLAT_STR_DICT ? p.out_lens[pc] + base : nullptr;
  f.vbit = rbit + d.val_bit;
  f.width = d.width;
  f.stride = d.stride;
  f.dcount = d.dict_count;
  f.dbit = ibit + d.dict_payload * 8u;
  f.dbits = d.dict_data_size * 8u;
  f.last_end = d.dict_end - d.dict_var;
  f.add = f.kind == FLAT_STR_DICT ? blk_addr + d.dict_var : d.base;
  f.mask = f.kind == FLAT_INT_DICT && d.sign_fix ? d.int_mask : 0ull;
  memcpy(dst, &f, sizeof(FlatCol));
}

// Item k = f * cnt + j (flat column f, selected row j); lane l starts at item l and steps by 32.
// Flat column f is the entry over meta-slot entry cols[f] of `ents` (kEnt bytes each).
template <uint32_t kEnt>
__device__ __forceinline__ void project_flat(const ScanParams &p, const uint8_t *ents, const uint8_t *cols, uint32_t nflat,
                                             const uint16_t *sel, uint32_t cnt, int64_t base, bool all_rows, int lane) {
  const uint32_t qf = 32u / cnt, qj = 32u % cnt;
  uint32_t f = (uint32_t)lane / cnt, j = (uint32_t)lane % cnt;
  for (; f < nflat; f += qf, j += qj) {
    if (j >= cnt) { j -= cnt; ++f; if (f >= nflat) break; }
    const FlatCol &c = *reinterpret_cast<const FlatCol *>(ents + (uint32_t)cols[f] * kEnt);
    const uint32_t row = all_rows ? j : (uint32_t)sel[j];
    const uint32_t at = c.vbit + row * c.stride, width = c.width;
    bool is_null = false;
    uint64_t v;
    if (c.kind == FLAT_BITS) {
      v = (width <= 32u ? (uint64_t)sbits32(at, width) : sbits(at, width)) + c.add;
    } else {
      const uint32_t ref = sbits32(at, width), dbits = c.dbits;
      is_null = ref >= c.dcount;
      if (c.kind == FLAT_STR_DICT) {
        uint32_t off = 0, end = 0;
        if (!is_null) {
          off = ref == 0 ? 0u : sbits32(c.dbit + (ref - 1u) * dbits, dbits);
          end = ref == c.dcount - 1u ? c.last_end : sbits32(c.dbit + ref * dbits, dbits);
        }
        __stcs(&c.olen[j], is_null ? 0 : (int32_t)(end - off));
        v = is_null ? 0ull : c.add + off;
      } else if (is_null) {
        v = 0;
      } else {
        const uint32_t e = c.dbit + ref * dbits;
        v = (dbits <= 32u ? (uint64_t)sbits32(e, dbits) : sbits(e, dbits)) + c.add;
        v = sign_fix(c.mask, v);
      }
    }
    const uint32_t el = c.elem_len;
    if (el == 8u) __stcs(reinterpret_cast<uint64_t *>(c.out) + j, v);
    else if (el == 4u) __stcs(reinterpret_cast<uint32_t *>(c.out) + j, (uint32_t)v);
    else __stcs(reinterpret_cast<uint8_t *>(c.out) + j, (uint8_t)v);
    if (is_null) {
      const int pc = c.pc;
      const int64_t o = base + (int64_t)j;
      atomicOr(&p.out_nulls[pc][o >> 5], 1u << (o & 31));
      p.has_null[pc] = 1;
    }
  }
}

template <bool REC>
__global__ void __launch_bounds__(kThreads) obgpu_project_pipe_kernel(const __grid_constant__ ScanParams p) {
  constexpr uint32_t kEnt = kProjEnt<REC>;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t *wr = g_smem + (uint32_t)warp * p.pp_bytes;
  uint16_t *sel = reinterpret_cast<uint16_t *>(wr + p.pp_sel);
  uint8_t *wscr = wr + p.pp_wscr;
  const int np = p.n_proj;
  const uint32_t hdr_bytes = p.pp_hdr_bytes, bm_bytes = p.pp_bm_bytes;
  const Team t = warp_team(lane);

  uint8_t *meta0 = wr + p.pp_meta, *reg0 = wr + p.pp_region;
  uint64_t *bars = reinterpret_cast<uint64_t *>(wr + p.pp_bar);
  auto meta = [&](int b, int ms) {
    if (b >= p.n_blocks) return;
    uint8_t *m = meta0 + (uint32_t)ms * p.pp_meta_bytes;
    issue_meta<REC, true, kEnt>(p, b, smem_u32(m), np, [&](int i) { return p.used_col[p.proj_used[i]]; }, lane);
  };
  // what a block needs beyond its meta: nothing (no selected row / overflow / corrupt), or bitmap words + column ranges
  auto regions = [&](int b, int ms, int rsl) {
    if (b >= p.n_blocks) return;
    const uint8_t *m = meta0 + (uint32_t)ms * p.pp_meta_bytes;
    uint8_t *rs = reg0 + (uint32_t)rsl * p.pp_region_bytes;
    uint64_t *bar = bars + rsl;
    const BlockRec &rec = *reinterpret_cast<const BlockRec *>(m);
    const int64_t base = *reinterpret_cast<const int64_t *>(m + kMetaSel);
    const uint32_t cnt = (uint32_t)(*reinterpret_cast<const int64_t *>(m + kMetaSel + 8u) - base);
    const uint32_t rows = rec.rows;
    if (rows == 0 || cnt == 0 || base + (int64_t)cnt > p.out_cap) {
      if (lane == 0) mbar_expect_tx(bar, 0u);   // nothing to stage: the slot's phase still completes
      return;
    }
    if (cnt != rows) {
      const uint32_t nwords = (rows + 31u) >> 5;
      const uint32_t *gbm = p.bitmap_words + rec.bm_word_off;
      for (uint32_t g = (uint32_t)lane; g < nwords; g += 32u) cp_async4(smem_u32(rs) + hdr_bytes + g * 4u, gbm + g);
    }
    int32_t *hdr = reinterpret_cast<int32_t *>(rs);
    uint32_t r[4] = {0, 0, 0, 0};
    int nr = 0;
    if (lane < np) {
      nr = staged_ranges<REC, false>(rec, m + kMetaPlans + (uint32_t)lane * kEnt, p.pp_span[lane], r);
      const uint32_t o0 = hdr_bytes + bm_bytes + p.pp_off[lane], o1 = o0 + (r[1] - r[0]);
      hdr[2 * lane] = (int32_t)o0 - (int32_t)r[0];
      hdr[2 * lane + 1] = nr == 2 ? (int32_t)o1 - (int32_t)r[2] : (int32_t)o0 - (int32_t)r[0];
    }
    const uint32_t badmask = __ballot_sync(0xffffffffu, lane < np && nr == 0);
    if (lane == 0) hdr[2 * kMaxProj] = (int32_t)badmask;
    // one bulk copy (TMA) per byte range, all completing on the slot's mbarrier
    const uint32_t len0 = r[1] - r[0], len1 = nr == 2 ? r[3] - r[2] : 0u;
    const uint32_t total = warp_sum_u32(len0 + len1);
    if (lane == 0) mbar_expect_tx(bar, total);
    __syncwarp();
    if (lane < np && nr >= 1) {
      uint8_t *dst0 = rs + hdr_bytes + bm_bytes + p.pp_off[lane];
      const uint8_t *gblk = p.image + rec.off;
      tma_bulk_g2s(dst0, gblk + r[0], len0, bar);
      if (nr == 2) tma_bulk_g2s(dst0 + len0, gblk + r[2], len1, bar);
    }
  };

  auto work = [&](int blk, int ms, int rsl) {
    uint8_t *m = meta0 + (uint32_t)ms * p.pp_meta_bytes;
    uint8_t *rs = reg0 + (uint32_t)rsl * p.pp_region_bytes;
    const BlockRec rec = *reinterpret_cast<const BlockRec *>(m);
    const int64_t base = *reinterpret_cast<const int64_t *>(m + kMetaSel);
    const uint32_t cnt = (uint32_t)(*reinterpret_cast<const int64_t *>(m + kMetaSel + 8u) - base);
    const uint32_t rows = rec.rows;
    if (rows == 0 || cnt == 0 || base + (int64_t)cnt > p.out_cap) {
      if (lane == 0 && rows == 0) atomicOr(p.status, ST_CORRUPT);
      if (lane == 0 && rows != 0 && cnt != 0) atomicOr(p.status, ST_OVERFLOW);
      return;
    }
    uint8_t *ents = m + kMetaPlans;
    ColDesc *plans = reinterpret_cast<ColDesc *>(ents);
    const int32_t *hdr = reinterpret_cast<const int32_t *>(rs);
    const uint32_t badmask = (uint32_t)hdr[2 * kMaxProj];
    const bool all_rows = cnt == rows;
    if (!all_rows) {
      // bitmap words -> ascending selected-row list: lane g owns word g of each group of 32 words
      const uint32_t *bmw = reinterpret_cast<const uint32_t *>(rs + hdr_bytes);
      const uint32_t nwords = (rows + 31u) >> 5;
      for (uint32_t base_w = 0, running = 0; base_w < nwords; base_w += 32u) {
        const uint32_t w = base_w + (uint32_t)lane;
        running += warp_select_group(w < nwords ? bmw[w] : 0u, min(32u, nwords - base_w), base_w * 32u, running, sel, lane);
      }
      __syncwarp();
    }
    if (p.want_row_ids) {
      int32_t *rid = p.row_ids + base;
      if (all_rows) for (uint32_t j = (uint32_t)lane; j < cnt; j += 32u) rid[j] = (int32_t)j;
      else for (uint32_t j = (uint32_t)lane; j < cnt; j += 32u) rid[j] = (int32_t)sel[j];
    }
    BlockCtx c;
    view_from_rec(rec, nullptr, c.b);
    c.bitsets = nullptr;
    c.descs = plans;
    c.rle_base = wscr + p.pw_rle;
    c.rle_slot_bytes = 0;
    c.rle_starts_bytes = p.words_cap * 4u;
    const uint64_t blk_addr = block_string_addr(p, blk, rec.off);
    // with records every projected column is flat in every block (layout_pipe)
    const bool flat = lane < np && !((badmask >> lane) & 1u) && (REC || (plans[lane].ok && flat_kind(plans[lane])));
    const uint32_t flatmask = __ballot_sync(0xffffffffu, flat);
    if (flatmask != 0u) {
      if (flat) {
        uint8_t *ent = ents + (uint32_t)lane * kEnt;
        flat_fill(p, *reinterpret_cast<const MetaEnt<REC> *>(ent), lane, smem_u32(rs), hdr[2 * lane], hdr[2 * lane + 1], base, blk_addr, ent);
        m[__popc(flatmask & ((1u << lane) - 1u))] = (uint8_t)lane;
      }
      __syncwarp();
      project_flat<kEnt>(p, ents, m, (uint32_t)__popc(flatmask), sel, cnt, base, all_rows, lane);
    }
    for (int pc = 0; pc < np; ++pc) {
      if ((flatmask >> pc) & 1u) continue;
      ColDesc *wdesc = plans + pc;
      if (REC || !wdesc->ok || ((badmask >> pc) & 1u)) {
        if (lane == 0) atomicOr(p.status, ST_UNSUPPORTED);
        continue;
      }
      const int32_t d0 = hdr[2 * pc], d1 = hdr[2 * pc + 1];
      if (wdesc->kind == K_DICT && wdesc->sc == 5) {
        uint32_t rbit, ibit;
        str_dict_bits(*wdesc, smem_u32(rs), d0, d1, rbit, ibit);
        if (all_rows) project_str_dict_shallow<true>(p, *wdesc, pc, sel, cnt, base, blk_addr, rbit, ibit, lane);
        else project_str_dict_shallow<false>(p, *wdesc, pc, sel, cnt, base, blk_addr, rbit, ibit, lane);
        __syncwarp();
        continue;
      }
      c.b.s = rs + d0;
      c.sbit = (smem_u32(rs) + (uint32_t)d0) * 8u;
      project_column_staged(p, c, wdesc, pc, sel, cnt, base, blk_addr, all_rows, rows, wscr, t);
      __syncwarp();
    }
  };

  warp_pipeline<1>(p.n_blocks, bars, lane, meta, regions, work);
}
