"""String filters, string projection and string skip-index verdicts on the device against the Python bytes model of
tests/test_string_filter_exact.py (not against the oracle): every string codec, VARCHAR and CHAR, 0 / 10 / 100 % NULL, every operator
over edge constants (bytes >= 0x80 and NUL, equal first 8 bytes, lengths and first bytes aliasing mod 64, IN lists on the hash-slot
and on the first-byte screen, duplicate / NULL / empty constants), trees that reach the survivor path, and the constant limits.

Paths: the fused scan at 1, 133, 1024 and 1025 rows per block with OBGPU_PIPE=0 (the general kernels: str_pred, the dictionary
bitsets of build_dict_bitset / build_dict_bitset_sorted) and OBGPU_PIPE=1 (the pipelined small-block kernels). With OBGPU_PIPE=1 the
count kernel takes stage records only when every block has at most 1024 rows and every leaf is an EQ / NE / IN or an integer range
on a DICT column with a record (var-length string dictionaries, integer dictionaries): here the PAX dict_var tables under EQ / NE /
IN leaves, and the trees of such a leaf and an integer leaf on the DICT-coded 0..99 column. So the survivor trees reach
lean_survivor_str with records there, and with plans on fixed-length dictionaries and under NU / NN / LT leaves
(test_survivor_trees_run_on_records_and_plans reads the choice back). Every other PAX case with OBGPU_PIPE=1 runs the pipelined
kernels on plans; CS batches keep the general kernels under either setting. Also: the per-block calls (filter_white / filter_tree
over row windows, project_strings); batches opened from a host image, from a device image, and CS batches whose streams are
restated at open; the skip index's verdicts and a scan pruned by it."""
import numpy as np
import pytest

from test_string_filter_exact import (K, MATRIX, MATRIX_IDS, RPB, S, TCOL, assert_headers, hand_filters, hand_rows, leaf, leaves, model,
                                      over_limits, selected, skip_cases, skip_filters, skip_sound, spec_of, table_of, trees)

pytestmark = pytest.mark.gpu

PROJ = [K, S, TCOL]


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def ctx(ob):
    c = ob.ScanContext(0)
    yield c
    c.close()


def projected(res, i):
    """column i of a scan result as bytes / None per selected row"""
    _, _, nulls = res.fetch_col(i)
    heap, off = res.fetch_strings(i)
    return [None if (int(nulls[j // 64]) >> (j % 64)) & 1 else bytes(heap[off[j]:off[j + 1]]) for j in range(len(off) - 1)]


def check_scan(batch, spec, name, f, with_strings, want=None):
    want = selected(spec, f) if want is None else want
    res = batch.scan(f, PROJ)
    assert res.selected_rows == len(want), name
    if want:
        assert [int(x) for x in res.fetch_col(0)[0]] == want, name
        if with_strings:
            assert projected(res, 1) == [spec.truth[S][i] for i in want], name
            assert projected(res, 2) == [spec.truth[TCOL][i] for i in want], name
    res.free()


def check_table(ob, batch, spec, pipes, monkeypatch, thin=1):
    """every leaf (every `thin`-th comparison leaf; every IN list and tree always) and tree under each OBGPU_PIPE setting, the
    model's rows computed once"""
    cases = [(n, f) for j, (n, f) in enumerate(leaves(spec)) if j % thin == 0 or n.startswith("in")] + trees(spec)
    wants = [selected(spec, f) for _, f in cases]
    for pipe in pipes:
        monkeypatch.setenv("OBGPU_PIPE", pipe)
        for j, ((name, f), want) in enumerate(zip(cases, wants)):
            check_scan(batch, spec, (pipe, name), f, j % 7 == 0 or name.startswith(("and", "or", "in")), want)
        for name, f, _ in over_limits(spec):    # beyond kMaxParams / kParamHeap: refused, never a wrong answer
            with pytest.raises(ob.ObGpuError) as e:
                batch.scan(f, PROJ).info()
            assert e.value.code == ob.capi.OB_NOT_SUPPORTED, name


@pytest.mark.parametrize("codec,tname,nname", MATRIX, ids=MATRIX_IDS)
def test_scan_matrix(ob, ctx, monkeypatch, codec, tname, nname):
    spec = spec_of(codec, tname, nname)
    batch = ctx.open_batch(table_of(codec, tname, nname))
    try:
        # CHAR columns take the same device string paths as VARCHAR: half the comparison leaves; all-NULL columns: a quarter
        check_table(ob, batch, spec, ("1", "0"), monkeypatch, thin=4 if nname == "n100" else (2 if tname == "char" else 1))
    finally:
        batch.close()


def kernels_run(fn):
    """names of the CUDA kernels fn() launched (torch.profiler, template arguments kept)"""
    import torch
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.key for e in prof.key_averages() if e.device_time_total > 0}


@pytest.mark.parametrize("codec,rec", [("dict_var", True), ("dict_fix", False), ("cs_str_dict_var", None)])
def test_survivor_trees_run_on_records_and_plans(ob, ctx, monkeypatch, codec, rec):
    # the count kernel the survivor trees run: the pipelined one on stage records (<true>) for a var-length string dictionary, on
    # plans (<false>) for a fixed-length one; a CS batch keeps the general count kernel
    monkeypatch.setenv("OBGPU_PIPE", "1")
    spec = spec_of(codec, "varchar", "n10")
    batch = ctx.open_batch(table_of(codec, "varchar", "n10"))
    try:
        for name, f in trees(spec):
            if name not in ("and_m_eq", "and_m_in", "and_m_ne"):     # NU / NN and range leaves on strings take plans
                continue
            batch.scan(f, PROJ).free()
            # two scans in the window: a profiling session can miss the first launch after it starts
            names = kernels_run(lambda: [batch.scan(f, PROJ).free() for _ in range(2)])
            if rec is None:
                assert any(k.startswith("obgpu_count_kernel") for k in names) and not any("count_pipe" in k for k in names), names
                check_scan(batch, spec, name, f, True)
                continue
            assert any("obgpu_count_pipe_kernel<%s>" % ("true" if rec else "false") in k for k in names), (name, names)
            assert not any("obgpu_count_pipe_kernel<%s>" % ("false" if rec else "true") in k for k in names), (name, names)
            check_scan(batch, spec, name, f, True)
    finally:
        batch.close()


# ---- rows per block: 1, 133, 1024 (stage records allowed) and 1025 (records refused: more than 1024 rows) -------------------
@pytest.fixture(params=["1", "0"], ids=["pipe", "no_pipe"])
def pipe(request, monkeypatch):
    monkeypatch.setenv("OBGPU_PIPE", request.param)
    return request.param


@pytest.mark.parametrize("rpb", [1, 133, 1024, 1025])
@pytest.mark.parametrize("codec", ["dict_var", "raw_var", "cs_str_dict_var", "dict_fix"])
def test_rows_per_block(ob, ctx, pipe, monkeypatch, rpb, codec):
    # a one-row block whose only cell is NULL cannot be dictionary coded (the writer refuses it): no NULLs at one row per block
    nname = "n0" if rpb == 1 else "n10"
    spec = spec_of(codec, "varchar", nname, n=300 if rpb == 1 else 3 * rpb + 5)
    table = ob.encode_table(spec.cols, rpb)
    # a one-row block holds one value, so its store is fixed-length whatever the codec's store elsewhere: the codec only there
    assert_headers(codec, nname, spec, table, store=rpb > 1)
    batch = ctx.open_batch(table)
    try:
        check_table(ob, batch, spec, (pipe,), monkeypatch)
        # a capacity-overflowed scan reports OB_BUF_NOT_ENOUGH; the re-run without the cap returns the right rows
        f = trees(spec)[6][1]
        want = selected(spec, f)
        res = batch.scan(f, PROJ, max_selected_rows=max(len(want) // 2, 1))
        with pytest.raises(ob.ObGpuError) as e:
            res.info()
        assert e.value.code == ob.OB_BUF_NOT_ENOUGH
        res.free()
        check_scan(batch, spec, "rerun", f, True)
    finally:
        batch.close()


# ---- per-block entry points -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("codec", ["dict_var", "dict_fix", "raw_var", "rle", "hex", "string_diff", "string_prefix", "column_equal",
                                   "cs_string_var", "cs_str_dict_fix"])
def test_per_block_calls(ob, ctx, codec):
    spec = spec_of(codec, "varchar", "n10")
    table = table_of(codec, "varchar", "n10")
    batch = ctx.open_batch(table)
    flts = [f for _, f in leaves(spec)[::3]] + [f for _, f in trees(spec)]
    try:
        for b in range(table.n_blocks):
            r0 = b * RPB
            rows = batch.block_info(b)[0]
            cols = {c: spec.truth[c][r0:r0 + rows] for c in range(4)}
            for start, count in ((0, rows), (3, rows - 7)):
                for f in flts:
                    want = model(f, cols)[start:start + count]
                    if hasattr(f, "children"):
                        got = batch.filter_tree(b, f, start, count)
                    else:
                        got = batch.filter_white(b, f.col, f.op, f.params, start, count)
                    assert got.astype(bool).tolist() == want, (b, start, f)
            rid = [r for r in range(rows) if r % 3 != 1]
            heap, off, nulls = batch.project_strings(b, S, rid)
            got = [None if (int(nulls[j // 64]) >> (j % 64)) & 1 else bytes(heap[off[j]:off[j + 1]]) for j in range(len(rid))]
            assert got == [cols[S][r] for r in rid], b
    finally:
        batch.close()


# ---- host vs device open; CS streams restated at open ----------------------------------------------------------------------
@pytest.mark.parametrize("codec", ["dict_var", "raw_var", "hex", "cs_str_dict_var", "cs_string_fix"])
def test_device_image_open(ob, ctx, monkeypatch, codec):
    import torch
    spec = spec_of(codec, "varchar", "n10")
    table = table_of(codec, "varchar", "n10")
    img = torch.from_numpy(table.image).cuda()
    torch.cuda.synchronize()
    batch = ob.PageBatch(ctx, table, device_image_ptr=img.data_ptr(), image_size=table.image.size, host_view=False)
    try:
        check_table(ob, batch, spec, ("1", "0"), monkeypatch)
    finally:
        batch.close()


@pytest.mark.parametrize("codec", ["cs_string_var", "cs_str_dict_var", "cs_str_dict_fix_constref"])
def test_cs_stream_codecs_restated_at_open(ob, ctx, monkeypatch, codec):
    spec = spec_of(codec, "varchar", "n10")
    plain = table_of(codec, "varchar", "n10")
    ob.capi.lib.obgpu_writer_set_cs_stream_encoding(0)      # detect: the sorted row-number column takes a delta codec
    try:
        table = ob.encode_table(spec.cols, RPB)
    finally:
        ob.capi.lib.obgpu_writer_set_cs_stream_encoding(1)
    assert table.image.size < plain.image.size               # some stream really is coded
    assert_headers(codec, "n10", spec, table)
    batch = ctx.open_batch(table)
    try:
        check_table(ob, batch, spec, ("1", "0"), monkeypatch)
    finally:
        batch.close()


# ---- skip index --------------------------------------------------------------------------------------------------------------
def test_skip_index_verdicts_and_pruned_scans(ob, ctx, monkeypatch):
    monkeypatch.delenv("OBGPU_PIPE", raising=False)
    decided = 0
    for key, spec, rows, offs in skip_cases():
        table = ob.encode_table(spec.cols, RPB)
        batch = ctx.open_batch(table)
        try:
            batch.set_agg_rows(rows, offs)
            for f in skip_filters(spec):
                got = batch.skip_index_filter(f)
                for b, v in enumerate(got.tolist()):
                    cells = spec.truth[S][b * RPB:(b + 1) * RPB]
                    assert skip_sound(v, leaf(f.op, cells, tuple(f.params))), (key, b, f)
                    decided += v != 0
            for f in [f for _, f in trees(spec)] + skip_filters(spec)[::5]:
                check_scan(batch, spec, key, f, False)      # the same rows as the model with the aggregate rows attached
        finally:
            batch.close()
    assert decided > 100
    # hand-built rows whose stored minimum / maximum is a prefix of, equal to, or longer than the constant
    cases = hand_rows()
    cells = [c for cs, _ in cases for c in cs]
    n = len(cells)
    cols = [ob.Column(5, 0, np.arange(n, dtype=np.int64)), ob.Column(5, 0, np.zeros(n, dtype=np.int64)),
            ob.Column(22, 0, [c or b"" for c in cells], nulls=np.array([c is None for c in cells], dtype=np.uint8)),
            ob.Column(22, 0, [b"t"] * n)]
    per = len(cases[0][0])
    table = ob.encode_table(cols, per)
    rows = np.concatenate([r for _, r in cases])
    offs = np.cumsum([0] + [len(r) for _, r in cases]).astype(np.int64)
    batch = ctx.open_batch(table)
    try:
        batch.set_agg_rows(rows, offs)
        for f in hand_filters():
            for b, v in enumerate(batch.skip_index_filter(f).tolist()):
                assert skip_sound(v, leaf(f.op, cells[b * per:(b + 1) * per], tuple(f.params))), (b, f)
    finally:
        batch.close()

