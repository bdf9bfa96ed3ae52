// Small micro-blocks (a 16 KiB block of a wide dictionary-coded table holds ~130 rows): per block there are only a
// few hundred bytes to filter and a dozen rows to project, so a scan is bound by the per-block chain of dependent
// global round trips (record -> plans -> column bytes), not by bandwidth. These two kernels keep ONE WARP per block
// but run it as a software pipeline over the blocks it owns (persistent grid, blocks strided over the warps):
//
//     iteration b:   wait   regions(b), meta(b + 1)          (cp.async groups, issued one / two iterations ago)
//                    issue  regions(b + 1)   <- needs meta(b + 1): block offset, decode plans -> column byte ranges
//                    issue  meta(b + 2)      <- block record, decode plans (and the two prefix entries)
//                    work   on block b from shared memory
//
// so a block's three round trips overlap the work on the two blocks before it. All copies are 16-byte cp.async
// (LDGSTS: no registers, no mbarrier), completion is cp.async.wait_group + __syncwarp.
//   obgpu_count_pipe_kernel   : stages every filter column's region of the block at once, then the same leaf loops
//                               as obgpu_count_kernel (K4 / K6 / K9 / K14)
//   obgpu_project_pipe_kernel : stages the block's bitmap words and the projected columns' byte ranges; a projected
//                               VARCHAR dictionary column needs only its refs and its offset array (VEC_DISCRETE
//                               output is pointers into the caller's block: the dictionary's bytes are never read).
//                               "Flat" columns (project_flat) are decoded in one pass over (column, selected row)
//                               items, the others column after column
#pragma once

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
constexpr int kRecPieces = (int)(sizeof(BlockRec) / 16), kPlanPieces = (int)(sizeof(ColDesc) / 16);
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
// lean leaves and flat_fill take either a plan or this.
struct RecDesc {
  uint64_t base, int_mask;
  uint32_t val_bit, stride, width, dict_count, dict_payload, dict_data_size, dict_var, dict_end;
  uint8_t kind, sc, elem_len, sign_fix, dict_sorted, dict_fixed;
};
__device__ __forceinline__ RecDesc rec_desc(const ScanParams &p, const StageRec &r, int used) {
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
template <bool REC> constexpr uint32_t kCountEnt = REC ? (uint32_t)sizeof(StageRec) : (uint32_t)sizeof(ColDesc);
template <bool REC> constexpr uint32_t kProjEnt = REC ? 64u : (uint32_t)sizeof(ColDesc);

// One lean leaf on the K_DICT column of stage record d (width <= 32) staged at sbit (generic address rs_col): returns the lane's
// bitmap word. The plan path of obgpu_count_pipe_kernel writes the same steps out with a fall-back to the generic dictionary
// bitset (build_dict_bitset); layout_pipe gives a scan records only when no leaf needs that fall-back.
__device__ __forceinline__ uint32_t lean_leaf(const ScanParams &p, const FilterNodeDev &nd, const RecDesc &d, uint32_t sbit, const uint8_t *rs_col,
                                              uint32_t *bits, uint32_t *bm, uint32_t mybm, uint32_t myvalid, uint32_t nwords,
                                              bool and_mode, int lane) {
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
  if (!is_str && nd.range_ok) lean_bitset_int_range(d, nd, sbit, bits, lane);
  else lean_bitset_str_eq(p, nd, d, sbit, bits, lane);
  __syncwarp();
  return lean_rows<true>(d, sbit, bits, 0u, 0u, false, mybm, myvalid, nwords, and_mode, lane);
}

// =================================================================================================
// Count, pipelined. Per warp: meta ring (3 slots: block record + the filter columns' plans, or their stage records when
// REC), region ring (2 slots: header with the per-column deltas + the filter columns' regions), bitmap words, predicate bitsets.
// =================================================================================================
template <bool REC>
__global__ void __launch_bounds__(kThreads) obgpu_count_pipe_kernel(const __grid_constant__ ScanParams p) {
  constexpr uint32_t kEnt = kCountEnt<REC>;
  constexpr int kEntPieces = (int)(kEnt / 16u);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nwarps_total = (int)gridDim.x * kWarps;
  int blk = (int)blockIdx.x * kWarps + warp;
  if (blk >= p.n_blocks) return;
  uint8_t *wr = g_smem + (uint32_t)warp * p.pc_bytes;
  uint8_t *meta0 = wr + p.pc_meta, *reg0 = wr + p.pc_region;
  uint32_t *bm = reinterpret_cast<uint32_t *>(wr + p.pc_bm);
  uint32_t *bitsets = reinterpret_cast<uint32_t *>(wr + p.pc_bitset);
  uint64_t *bars = reinterpret_cast<uint64_t *>(wr + p.pc_bar);   // one mbarrier per region slot
  const int nf = p.pf_n;
  const Team t = warp_team(lane);
  if (lane == 0) {
    mbar_init(bars, 1);
    mbar_init(bars + 1, 1);
    fence_barrier_init();
  }
  __syncwarp();

  auto issue_meta = [&](int b, int slot) {
    if (b >= p.n_blocks) return;
    const uint32_t sa = smem_u32(meta0 + (uint32_t)slot * p.pc_meta_bytes);
    const uint8_t *rec = reinterpret_cast<const uint8_t *>(p.recs + b);
    const uint8_t *ents = REC ? reinterpret_cast<const uint8_t *>(p.stage + (int64_t)b * p.max_cols)
                              : reinterpret_cast<const uint8_t *>(p.plans + (int64_t)b * p.max_cols);
    for (int q = lane; q < kRecPieces + nf * kEntPieces; q += 32) {
      if (q < kRecPieces) cp_async16(sa + (uint32_t)q * 16u, rec + q * 16);
      else {
        const int i = (q - kRecPieces) / kEntPieces, piece = (q - kRecPieces) % kEntPieces;
        cp_async16(sa + kMetaPlans + (uint32_t)i * kEnt + (uint32_t)piece * 16u, ents + (size_t)p.used_col[i] * kEnt + piece * 16);
      }
    }
  };
  // region slot: [int32 delta[kPipeMaxFilterCols] | uint32 flags] (64 bytes) then the regions at p.pf_off[i]
  auto issue_regions = [&](int b, int mslot, int rslot, uint32_t verdict) {
    if (b >= p.n_blocks) return;
    const uint8_t *m = meta0 + (uint32_t)mslot * p.pc_meta_bytes;
    uint8_t *rs = reg0 + (uint32_t)rslot * p.pc_region_bytes;
    const BlockRec &rec = *reinterpret_cast<const BlockRec *>(m);
    const ColDesc *descs = reinterpret_cast<const ColDesc *>(m + kMetaPlans);
    int32_t *hdr = reinterpret_cast<int32_t *>(rs);
    uint32_t lo = 0, hi = 0;
    bool bad = false;
    if (lane < nf && rec.rows != 0 && verdict == 0) {
      if constexpr (REC) {
        const StageRec &r = reinterpret_cast<const StageRec *>(m + kMetaPlans)[lane];
        lo = (uint32_t)r.lo[0] * 16u;
        hi = (uint32_t)max(r.hi[0], r.hi[1]) * 16u;
        if (hi - lo > p.pf_span[lane] || hi > ((rec.size + 15u) & ~15u) + 32u) { bad = true; lo = hi = 0; }
      } else {
        BlockView bv;
        view_from_rec(rec, nullptr, bv);
        const ColDesc &d = descs[lane];
        if (!d.ok || !col_region(d, bv, lo, hi) || hi - lo > p.pf_span[lane] || hi > ((rec.size + 15u) & ~15u) + 32u) { bad = true; lo = hi = 0; }
      }
      hdr[lane] = (int32_t)(kCountHdrBytes + p.pf_off[lane]) - (int32_t)lo;
    }
    const uint32_t badmask = __ballot_sync(0xffffffffu, bad);
    if (lane == 0) hdr[kPipeMaxFilterCols] = (int32_t)badmask;
    // one bulk copy (TMA) per filter column, all completing on the slot's mbarrier
    const uint32_t total = warp_sum_u32(hi - lo);
    uint64_t *bar = bars + rslot;
    if (lane == 0) mbar_expect_tx(bar, total);
    __syncwarp();
    if (hi > lo) tma_bulk_g2s(rs + kCountHdrBytes + p.pf_off[lane], p.image + rec.off + lo, hi - lo, bar);
  };

  // prologue: meta(b0), then regions(b0) + meta(b1)
  uint32_t v_cur = 0, v_next = 0, v_next2 = 0;   // skip-index verdicts, fetched two blocks ahead
  if (p.blk_const != nullptr) {
    v_cur = p.blk_const[blk];
    if (blk + nwarps_total < p.n_blocks) v_next = p.blk_const[blk + nwarps_total];
  }
  issue_meta(blk, 0);
  cp_async_commit();
  cp_async_wait_all();
  __syncwarp();
  issue_regions(blk, 0, 0, v_cur);
  cp_async_commit();
  issue_meta(blk + nwarps_total, 1);
  cp_async_commit();
  int it = 0;
  PIPE_CLOCK_START();
  for (; blk < p.n_blocks; blk += nwarps_total, ++it) {
    const int ms = it % 3, rsl = it & 1;
    PIPE_CLOCK_AT(pclk_a);
    cp_async_wait_all();
    mbar_wait(bars + rsl, (uint32_t)(it >> 1) & 1u);
    __syncwarp();
    PIPE_CLOCK_ADD(pclk_wait, pclk_a);
    PIPE_CLOCK_AT(pclk_b);
    const int b2 = blk + 2 * nwarps_total;
    if (p.blk_const != nullptr && b2 < p.n_blocks) v_next2 = p.blk_const[b2];
    issue_regions(blk + nwarps_total, (it + 1) % 3, rsl ^ 1, v_next);
    cp_async_commit();
    issue_meta(b2, (it + 2) % 3);
    cp_async_commit();
    PIPE_CLOCK_ADD(pclk_issue, pclk_b);

    // ---- block `blk` from shared memory -------------------------------------------------------------------------
    const uint8_t *m = meta0 + (uint32_t)ms * p.pc_meta_bytes;
    uint8_t *rs = reg0 + (uint32_t)rsl * p.pc_region_bytes;
    const BlockRec rec = *reinterpret_cast<const BlockRec *>(m);
    const int32_t *hdr = reinterpret_cast<const int32_t *>(rs);
    const uint32_t rows = rec.rows;
    uint32_t *gbm = p.bitmap_words + rec.bm_word_off;
    const uint32_t nwords = (rows + 31u) >> 5;
    const uint32_t verdict = v_cur;
    v_cur = v_next;
    v_next = v_next2;
    if (count_block_settled(p, blk, rows, gbm, verdict, hdr[kPipeMaxFilterCols] != 0, lane)) {
      __syncwarp();
      continue;
    }
    uint32_t cnt = 0;
    if constexpr (REC) {
      // stage records: every block has at most 1024 rows (bitmap in registers) and every leaf is lean (layout_pipe)
      const bool and_mode = p.simple_shape == 1;
      const int n_leaves = p.n_nodes == 1 ? 1 : p.n_nodes - 1;
      const uint32_t myvalid = (uint32_t)lane < nwords ? valid_mask_of(rows, (uint32_t)lane) : 0u;
      uint32_t mybm = and_mode ? myvalid : 0u;
      for (int i = 0; i < n_leaves; ++i) {
        const FilterNodeDev &nd = p.nodes[i];
        if (p.leaf_const != nullptr && p.leaf_const[(int64_t)blk * p.n_nodes + i] != 0) continue;
        const RecDesc d = rec_desc(p, reinterpret_cast<const StageRec *>(m + kMetaPlans)[nd.used_idx], nd.used_idx);
        mybm = lean_leaf(p, nd, d, (smem_u32(rs) + (uint32_t)hdr[nd.used_idx]) * 8u, rs + hdr[nd.used_idx],
                         bitsets + nd.slot * p.bitset_words, bm, mybm, myvalid, nwords, and_mode, lane);
        if (i + 1 < n_leaves && !__any_sync(0xffffffffu, and_mode ? mybm != 0u : mybm != myvalid)) break;   // early-out
      }
      if ((uint32_t)lane < nwords) gbm[lane] = mybm;
      cnt = __popc(mybm);
    } else {
      const ColDesc *descs = reinterpret_cast<const ColDesc *>(m + kMetaPlans);
      BlockCtx c;
      view_from_rec(rec, nullptr, c.b);
      c.descs = descs;
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
      if (nwords <= 32u) {
        // ---- lean path: the block's bitmap lives in registers (lane g owns word g); dictionary-coded leaves run
        // through explicit shared-memory loads, everything else through the generic leaf code on a spilled bitmap
        const uint32_t myvalid = (uint32_t)lane < nwords ? valid_mask_of(rows, (uint32_t)lane) : 0u;
        uint32_t mybm = and_mode ? myvalid : 0u;
        for (int i = 0; i < n_leaves; ++i) {
          const FilterNodeDev &nd = p.nodes[i];
          if (p.leaf_const != nullptr && p.leaf_const[(int64_t)blk * p.n_nodes + i] != 0) continue;
          const ColDesc &d = descs[nd.used_idx];
          const uint32_t sbit = (smem_u32(rs) + (uint32_t)hdr[nd.used_idx]) * 8u;
          if (d.kind == K_DICT && nd.slot >= 0 && nd.op != OP_FALSE && nd.op != OP_TRUE && d.width <= 32u) {
            uint32_t *bits = bitsets + nd.slot * p.bitset_words;
            const bool is_str = d.sc == 5;
            if (is_str && and_mode) {
              // few surviving rows and a larger dictionary: test the survivors' own entries instead of every entry
              const uint32_t alive = warp_sum_u32(__popc(mybm));
              if (alive * 4u <= d.dict_count) {
                mybm = lean_survivor_str(p, nd, d, sbit, rs + hdr[nd.used_idx], mybm, nwords, alive, bm, lane);
                continue;
              }
            }
            if (!is_str && nd.range_ok && d.dict_sorted) {
              uint32_t a, e;
              lean_interval_sorted_int(d, nd, sbit, lane, a, e);
              mybm = lean_rows<false>(d, sbit, nullptr, a, e, nd.negate != 0, mybm, myvalid, nwords, and_mode, lane);
              goto leaf_done;
            }
            if (!is_str && nd.range_ok) lean_bitset_int_range(d, nd, sbit, bits, lane);
            else if (is_str && (nd.op == OP_EQ || nd.op == OP_NE || nd.op == OP_IN)) lean_bitset_str_eq(p, nd, d, sbit, bits, lane);
            else {
              c.b.s = rs + hdr[nd.used_idx];
              c.sbit = sbit;
              build_dict_bitset(p, c.b, d, nd, bits, t);
            }
            __syncwarp();
            mybm = lean_rows<true>(d, sbit, bits, 0u, 0u, false, mybm, myvalid, nwords, and_mode, lane);
          } else {
            bm[lane] = mybm;   // words_cap >= 32 words are reserved for the spilled bitmap
            __syncwarp();
            bool inited = true;
            leaf_step(p, c, c, nd, false, inited, bm, rows, nwords, and_mode, t, staged_at);
            mybm = (uint32_t)lane < nwords ? bm[lane] : 0u;
          }
        leaf_done:
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
          const ColDesc &d = descs[nd.used_idx];
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
    }
    cnt = warp_sum_u32(cnt);
    if (lane == 0) p.counts[blk] = cnt;
    __syncwarp();   // every lane is done with this iteration's slots before the next iteration refills them
  }
  PIPE_CLOCK_STOP(0);
  cp_async_wait_all();
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

__device__ __forceinline__ const ColDesc &flat_desc(const ScanParams &, const ColDesc &d, int) { return d; }
__device__ __forceinline__ RecDesc flat_desc(const ScanParams &p, const StageRec &r, int pc) { return rec_desc(p, r, p.proj_used[pc]); }

// Entry of projected column pc (flat_kind) from its plan or stage record and its staged byte ranges (slot deltas d0, d1). Not
// inlined: once per block, and inlined into obgpu_project_pipe_kernel it costs the kernel spills at 64 registers.
// dst overlays src: the entry is built in registers and stored with memcpy, whose byte stores may alias any type, so
// no load of src can move past them.
template <class S>
__device__ __noinline__ void flat_fill(const ScanParams &p, const S &src, int pc, uint32_t rs_addr, int32_t d0, int32_t d1,
                                       int64_t base, uint64_t blk_addr, void *dst) {
  const auto &d = flat_desc(p, src, pc);
  FlatCol f;
  const uint32_t s0 = (rs_addr + (uint32_t)d0) * 8u;
  uint32_t rbit = s0, ibit = s0;
  f.kind = d.kind == K_BITS ? FLAT_BITS : d.sc == 5 ? FLAT_STR_DICT : FLAT_INT_DICT;
  if (f.kind == FLAT_STR_DICT && d0 != d1) {
    // which delta belongs to the refs: with two ranges they are ordered by block offset (proj_ranges)
    const uint32_t s1 = (rs_addr + (uint32_t)d1) * 8u;
    if ((d.val_bit >> 3) < d.dict_payload) ibit = s1;
    else rbit = s1;
  }
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
  constexpr uint32_t kEnt = kProjEnt<REC>, kSrc = REC ? (uint32_t)sizeof(StageRec) : (uint32_t)sizeof(ColDesc);
  constexpr int kSrcPieces = (int)(kSrc / 16u);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nwarps_total = (int)gridDim.x * kWarps;
  int blk = (int)blockIdx.x * kWarps + warp;
  if (blk >= p.n_blocks) return;
  uint8_t *wr = g_smem + (uint32_t)warp * p.pp_bytes;
  uint8_t *meta0 = wr + p.pp_meta, *reg0 = wr + p.pp_region;
  uint16_t *sel = reinterpret_cast<uint16_t *>(wr + p.pp_sel);
  uint8_t *wscr = wr + p.pp_wscr;
  uint64_t *bars = reinterpret_cast<uint64_t *>(wr + p.pp_bar);   // one mbarrier per region slot
  if (lane == 0) {
    mbar_init(bars, 1);
    mbar_init(bars + 1, 1);
    fence_barrier_init();
  }
  __syncwarp();
  const int np = p.n_proj;
  const uint32_t hdr_bytes = p.pp_hdr_bytes, bm_bytes = p.pp_bm_bytes;
  const Team t = warp_team(lane);

  auto issue_meta = [&](int b, int slot) {
    if (b >= p.n_blocks) return;
    const uint32_t sa = smem_u32(meta0 + (uint32_t)slot * p.pp_meta_bytes);
    const uint8_t *rec = reinterpret_cast<const uint8_t *>(p.recs + b);
    const uint8_t *ents = REC ? reinterpret_cast<const uint8_t *>(p.stage + (int64_t)b * p.max_cols)
                              : reinterpret_cast<const uint8_t *>(p.plans + (int64_t)b * p.max_cols);
    constexpr int kHead = kRecPieces + 2;   // the record, then the two sel_offset entries
    for (int q = lane; q < kHead + np * kSrcPieces; q += 32) {
      if (q < kRecPieces) cp_async16(sa + (uint32_t)q * 16u, rec + q * 16);
      else if (q < kHead) cp_async8(sa + kMetaSel + (uint32_t)(q - kRecPieces) * 8u, p.sel_offset + b + (q - kRecPieces));
      else {
        const int i = (q - kHead) / kSrcPieces, piece = (q - kHead) % kSrcPieces;
        cp_async16(sa + kMetaPlans + (uint32_t)i * kEnt + (uint32_t)piece * 16u,
                   ents + (size_t)p.used_col[p.proj_used[i]] * kSrc + piece * 16);
      }
    }
  };
  // what a block needs beyond its meta: nothing (no selected row / overflow / corrupt), or bitmap words + column ranges
  auto issue_regions = [&](int b, int mslot, int rslot) {
    if (b >= p.n_blocks) return;
    const uint8_t *m = meta0 + (uint32_t)mslot * p.pp_meta_bytes;
    uint8_t *rs = reg0 + (uint32_t)rslot * p.pp_region_bytes;
    const BlockRec &rec = *reinterpret_cast<const BlockRec *>(m);
    const int64_t base = *reinterpret_cast<const int64_t *>(m + kMetaSel);
    const uint32_t cnt = (uint32_t)(*reinterpret_cast<const int64_t *>(m + kMetaSel + 8u) - base);
    const uint32_t rows = rec.rows;
    if (rows == 0 || cnt == 0 || base + (int64_t)cnt > p.out_cap) {
      if (lane == 0) mbar_expect_tx(bars + rslot, 0u);   // nothing to stage: the slot's phase still completes
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
      if constexpr (REC) {
        const StageRec &sr = *reinterpret_cast<const StageRec *>(m + kMetaPlans + (uint32_t)lane * kEnt);
        r[0] = (uint32_t)sr.lo[0] * 16u;
        r[1] = (uint32_t)sr.hi[0] * 16u;
        r[2] = (uint32_t)sr.lo[1] * 16u;
        r[3] = (uint32_t)sr.hi[1] * 16u;
        nr = r[3] != r[2] ? 2 : 1;
      } else {
        BlockView bv;
        view_from_rec(rec, nullptr, bv);
        const ColDesc &d = reinterpret_cast<const ColDesc *>(m + kMetaPlans)[lane];
        nr = d.ok ? proj_ranges(d, bv, r) : 0;
      }
      const uint32_t lim = ((rec.size + 15u) & ~15u) + 32u;
      if (nr > 0 && ((r[1] - r[0]) + (nr == 2 ? r[3] - r[2] : 0u) > p.pp_span[lane] || r[1] > lim || (nr == 2 && r[3] > lim))) nr = 0;
      if (nr == 0) r[0] = r[1] = r[2] = r[3] = 0;
      const uint32_t o0 = hdr_bytes + bm_bytes + p.pp_off[lane], o1 = o0 + (r[1] - r[0]);
      hdr[2 * lane] = (int32_t)o0 - (int32_t)r[0];
      hdr[2 * lane + 1] = nr == 2 ? (int32_t)o1 - (int32_t)r[2] : (int32_t)o0 - (int32_t)r[0];
    }
    const uint32_t badmask = __ballot_sync(0xffffffffu, lane < np && nr == 0);
    if (lane == 0) hdr[2 * kMaxProj] = (int32_t)badmask;
    // one bulk copy (TMA) per byte range, all completing on the slot's mbarrier
    const uint32_t len0 = r[1] - r[0], len1 = nr == 2 ? r[3] - r[2] : 0u;
    const uint32_t total = warp_sum_u32(len0 + len1);
    uint64_t *bar = bars + rslot;
    if (lane == 0) mbar_expect_tx(bar, total);
    __syncwarp();
    if (lane < np && nr >= 1) {
      uint8_t *dst0 = rs + hdr_bytes + bm_bytes + p.pp_off[lane];
      const uint8_t *gblk = p.image + rec.off;
      tma_bulk_g2s(dst0, gblk + r[0], len0, bar);
      if (nr == 2) tma_bulk_g2s(dst0 + len0, gblk + r[2], len1, bar);
    }
  };

  issue_meta(blk, 0);
  cp_async_commit();
  cp_async_wait_all();
  __syncwarp();
  issue_regions(blk, 0, 0);
  cp_async_commit();
  issue_meta(blk + nwarps_total, 1);
  cp_async_commit();
  int it = 0;
  PIPE_CLOCK_START();
  for (; blk < p.n_blocks; blk += nwarps_total, ++it) {
    const int ms = it % 3, rsl = it & 1;
    PIPE_CLOCK_AT(pclk_a);
    cp_async_wait_all();
    mbar_wait(bars + rsl, (uint32_t)(it >> 1) & 1u);
    __syncwarp();
    PIPE_CLOCK_ADD(pclk_wait, pclk_a);
    PIPE_CLOCK_AT(pclk_b);
    issue_regions(blk + nwarps_total, (it + 1) % 3, rsl ^ 1);
    cp_async_commit();
    issue_meta(blk + 2 * nwarps_total, (it + 2) % 3);
    cp_async_commit();
    PIPE_CLOCK_ADD(pclk_issue, pclk_b);

    uint8_t *m = meta0 + (uint32_t)ms * p.pp_meta_bytes;
    uint8_t *rs = reg0 + (uint32_t)rsl * p.pp_region_bytes;
    const BlockRec rec = *reinterpret_cast<const BlockRec *>(m);
    const int64_t base = *reinterpret_cast<const int64_t *>(m + kMetaSel);
    const uint32_t cnt = (uint32_t)(*reinterpret_cast<const int64_t *>(m + kMetaSel + 8u) - base);
    const uint32_t rows = rec.rows;
    if (rows == 0 || cnt == 0 || base + (int64_t)cnt > p.out_cap) {
      if (lane == 0 && rows == 0) atomicOr(p.status, ST_CORRUPT);
      if (lane == 0 && rows != 0 && cnt != 0) atomicOr(p.status, ST_OVERFLOW);
      __syncwarp();
      continue;
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
        if constexpr (REC) flat_fill(p, *reinterpret_cast<const StageRec *>(ent), lane, smem_u32(rs), hdr[2 * lane], hdr[2 * lane + 1], base, blk_addr, ent);
        else flat_fill(p, *reinterpret_cast<const ColDesc *>(ent), lane, smem_u32(rs), hdr[2 * lane], hdr[2 * lane + 1], base, blk_addr, ent);
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
        const uint32_t idx_sbit = (smem_u32(rs) + (uint32_t)d0) * 8u, ref_sbit = (smem_u32(rs) + (uint32_t)d1) * 8u;
        // which delta belongs to the refs: with two ranges they are ordered by block offset (proj_ranges)
        uint32_t rbit = ref_sbit, ibit = idx_sbit;
        if (d0 == d1) rbit = ibit = idx_sbit;
        else if ((wdesc->val_bit >> 3) < wdesc->dict_payload) { rbit = idx_sbit; ibit = ref_sbit; }
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
    __syncwarp();
  }
  PIPE_CLOCK_STOP(1);
  cp_async_wait_all();
}
