"""Every kernel choice of the scan planner (plan_scan, obgpu_scan.cu) at both sides of each of its limits, read back through
obgpu_ctx_scan_plan, and every output of each scan against the oracle (assert_scan_matches). The cases and their tables live in
test_scan_plan_shapes.py, which checks without a device that each table sits where its case says.

Every reachable (count kernel, projection kernel) pair runs at least once (pair_* cases on 400-row blocks):

    count \\ projection | NONE | CTA | CTA_SPARSE | PIPE_PLANS | PIPE_RECORDS
    NONE               |  x   |  x  |     -      |     x      |      x
    BITMAP             |  x   |  x  |     x      |     x      |      x
    CTA                |  x   |  x  |     x      |     x      |      x
    PIPE_PLANS         |  x   |  x  |     x      |     x      |      x
    PIPE_RECORDS       |  x   |  x  |     x      |     x      |      x
    PIPE_CODED         |  x   |  x  |     x      |     x      |      x

Branches obgpu_scan cannot reach, and so not forced here:
- NONE with CTA_SPARSE: without a filter no row is dropped, and the sparse split needs a selecting count kernel.
- the "filter column after a non-filter column" check of layout_count_pipe: build_filter registers every filter column
  before the projected ones.
- dropping `rec &&` from all_coded: batch codes are only taken when rec holds, so the coded mask is empty otherwise.
- a count-only scan whose CTA projection layout does not fit: with no_stage the CTA projection layout is a row list and two
  bitmaps, at most about 150 KB at 65536 rows per block, so it fits every device with 227 KB.
- a pipelined count scan whose CTA count layout would not fit: the pipelined layout holds the same bitsets twice over and must
  fit two CTAs per SM.
- a projected column at exactly the 16384-byte span cap on the pipelined projection kernel: its two region slots alone are over
  the two-CTA fit of a 227 KB device (proj_span_cap is skipped there; proj_span_over still runs).
"""
import ctypes as C

import pytest

import oracle_binding as ora
import test_scan_plan_shapes as S
from test_gpu_scan import assert_scan_matches

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def ctx(ob):
    c = ob.ScanContext(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def max_smem():
    import torch
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin - S.SMEM_HEADROOM


@pytest.fixture(scope="module")
def tables():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = S.TABLES[name]()
        return cache[name]
    return get


class W:
    def __init__(self, table, flt, proj):
        self.table, self.filter, self.proj = table, flt, list(proj)
        self.proj_is_string = [_is_string(table, c) for c in self.proj]
        self.proj_elem_len = [8] * len(self.proj)


def _is_string(table, col):
    s = bytes(table.block(0))
    if s[20] == 3:
        return col == 1          # cs_table: column 1 is the CS string column
    return s[int.from_bytes(s[4:8], "little") + 16 * col + 3] in (22, 23)


def count_layout(ob, ctx):
    pcb, ctas, kern = C.c_int32(-1), C.c_int32(-1), C.c_int32(-1)
    assert ob.capi.lib.obgpu_ctx_count_layout(ctx._h, C.byref(pcb), C.byref(ctas), C.byref(kern)) == 0
    return pcb.value, ctas.value, kern.value


def codes_state(ob, batch, col):
    st, n = C.c_int32(0), C.c_int32(0)
    assert ob.capi.lib.obgpu_batch_string_codes(batch._h, col, C.byref(st), C.byref(n), None) == 0
    return st.value


def filter_bitmap(ob, ctx, table, flt):
    """a CGBitmap of the rows flt selects, written by folding a scan of the same table"""
    b = ctx.open_batch(table)
    r = b.scan(flt, [])
    bm = ob.CGBitmap(ctx, table.total_rows)
    bm.apply(r, 0, "set")
    r.free()
    b.close()
    return bm


class Scans:
    """What assert_scan_matches needs of a ctx (open_batch), with the batch it opens kept open until close() here, so its
    batch codes can be read after the scan; with a bitmap, the batch's scan is scan_bitmap over it in place of the filter."""

    def __init__(self, ctx, table, bitmap=None):
        self.batch, self.bitmap = ctx.open_batch(table), bitmap

    def open_batch(self, table):
        return self

    def scan(self, flt, proj, **kw):
        if self.bitmap is not None:
            return self.batch.scan_bitmap(self.bitmap, proj, **kw)
        return self.batch.scan(flt, proj, **kw)

    def close(self):
        pass                     # assert_scan_matches is done with the batch; run_case closes it


def run_case(ob, ctx, tables, case, monkeypatch, batch_check=None):
    for k, v in case.knobs.items():
        monkeypatch.setenv(k, v)
    table, words = tables(case.table)
    flt = case.filter(ob, words) if case.filter else None
    w = W(table, flt, case.proj)
    cap = case.max_selected(table.total_rows)
    bm = filter_bitmap(ob, ctx, table, flt) if case.bitmap else None
    scans = Scans(ctx, table, bm)
    batch = scans.batch
    try:
        if case.overflow:
            res = batch.scan(flt, w.proj, want_row_ids=case.row_ids, max_selected_rows=cap)
            plan = ctx.last_plan()
            with pytest.raises(ob.ObGpuError) as ei:
                res.info()
            assert ei.value.code == ob.OB_BUF_NOT_ENOUGH
            assert res._info.selected_rows == ora.scan_table(table, flt, [], [], [])["selected"] > cap
            res.free()
        else:
            assert_scan_matches(scans, w, want_row_ids=case.row_ids, max_selected_rows=cap)
            plan = ctx.last_plan()
        assert plan == case.expect, f"{case.name}: plan {plan}, expected {case.expect}"
        pcb, ctas, kern = count_layout(ob, ctx)
        if plan[0] in (S.PLANS, S.RECORDS, S.CODED):
            assert kern == plan[0] and ctas >= 2 and pcb > 0
        else:
            assert (pcb, ctas, kern) == (0, 0, 0)
        if batch_check:
            batch_check(batch, table)
    finally:
        batch.close()
        if bm is not None:
            bm.free()
    return table


PLAIN = [c.name for c in S.CASES if c.name not in ("count_fit_in", "count_fit_out", "proj_fit_in", "proj_fit_out",
                                                    "proj_span_cap", "no_stage", "codes_four", "codes_fifth", "codes_off")]


@pytest.mark.parametrize("name", PLAIN)
def test_plan(ob, ctx, tables, monkeypatch, name):
    run_case(ob, ctx, tables, S.CASE[name], monkeypatch)


@pytest.mark.parametrize("name,coded", [("codes_four", [0, 4, 5, 1]), ("codes_fifth", [0, 4, 5, 6]), ("codes_off", [])])
def test_batch_codes(ob, ctx, tables, monkeypatch, name, coded):
    # the count kernel builds batch codes for its first four filter columns only; with codes off for none
    def check(batch, table):
        for col in (0, 1, 4, 5, 6):
            assert codes_state(ob, batch, col) == (1 if col in coded else 0), col
    run_case(ob, ctx, tables, S.CASE[name], monkeypatch, check)


def test_count_fit(ob, ctx, tables, monkeypatch, max_smem):
    f = S.facts("cfit")
    inside, outside = S.count_pipe_bytes(f, [0, 1], S.CFIT_LEAVES), S.count_pipe_bytes(f, [0, 1], S.CFIT_LEAVES + 1)
    if not (S.two_ctas(inside, max_smem) and not S.two_ctas(outside, max_smem)):
        pytest.skip(f"the count-fit pair ({inside}, {outside} bytes per warp) does not straddle this device's {max_smem} bytes")
    run_case(ob, ctx, tables, S.CASE["count_fit_in"], monkeypatch)
    assert count_layout(ob, ctx)[0] == inside
    run_case(ob, ctx, tables, S.CASE["count_fit_out"], monkeypatch)


def test_proj_fit(ob, ctx, tables, monkeypatch, max_smem):
    f = S.facts("pfit")
    inside, outside = S.proj_pipe_bytes(f, S.PFIT_IN, True), S.proj_pipe_bytes(f, S.PFIT_IN + [6], True)
    if not (S.two_ctas(inside, max_smem) and not S.two_ctas(outside, max_smem)):
        pytest.skip(f"the projection-fit pair ({inside}, {outside} bytes per warp) does not straddle this device's {max_smem} bytes")
    run_case(ob, ctx, tables, S.CASE["proj_fit_in"], monkeypatch)
    run_case(ob, ctx, tables, S.CASE["proj_fit_out"], monkeypatch)


def test_proj_span_cap(ob, ctx, tables, monkeypatch, max_smem):
    need = S.proj_pipe_bytes(S.facts("pspan_in"), [0], False)
    if not S.two_ctas(need, max_smem):
        pytest.skip(f"a column at the 16384-byte span cap needs {need} bytes per warp: over the two-CTA fit of {max_smem} bytes")
    run_case(ob, ctx, tables, S.CASE["proj_span_cap"], monkeypatch)


def test_no_stage(ob, ctx, tables, monkeypatch, max_smem):
    if S.facts("no_stage").block_bytes <= max_smem:
        pytest.skip(f"the table's blocks fit this device's {max_smem} bytes of shared memory")
    run_case(ob, ctx, tables, S.CASE["no_stage"], monkeypatch)


def test_filter_working_set_over_shared_memory(ob, ctx, tables, monkeypatch, max_smem):
    f = S.facts("big_dict")
    if S.count_cta_bytes(f, [1, 0], 14) * S.WARPS <= max_smem:
        pytest.skip("the filter's working set fits this device's shared memory")
    table, words = tables("big_dict")
    batch = ctx.open_batch(table)
    try:
        with pytest.raises(ob.ObGpuError) as ei:
            batch.scan(S.BIG_FILTER(ob, words), [])
        assert ei.value.code == ob.OB_NOT_SUPPORTED
        assert "filter working set" in ctx.last_error()
        assert ctx.last_plan() == (0, 0, 0) and count_layout(ob, ctx) == (0, 0, 0)
    finally:
        batch.close()
    run_case(ob, ctx, tables, S.CASE["pair_plans_records"], monkeypatch)      # the ctx still scans


def test_read_out_follows_each_scan(ob, ctx, tables, monkeypatch):
    # a pipelined count, then a scan with no filter and a bitmap scan: neither may report the pipelined kernel
    run_case(ob, ctx, tables, S.CASE["pair_coded_records"], monkeypatch)
    assert count_layout(ob, ctx)[2] == S.CODED
    run_case(ob, ctx, tables, S.CASE["pair_none_records"], monkeypatch)
    run_case(ob, ctx, tables, S.CASE["pair_coded_records"], monkeypatch)
    run_case(ob, ctx, tables, S.CASE["pair_bitmap_records"], monkeypatch)
    assert ctx.last_plan()[0] == S.BITMAP and count_layout(ob, ctx) == (0, 0, 0)
