"""Stage records (the 32-byte per block and column entries the index kernel writes next to the plans) against the oracle:
the pipelined kernels read them instead of the plans when every block of a referenced column is lean (filter) or flat
(projection). Selected rows, row ids, projected values, lengths and NULLs must match the oracle with the pipelined
kernels forced on and off, for the columns that take records and for scans that fall back to plans."""
import numpy as np
import pytest

import oracle_binding as ora
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


@pytest.fixture(params=["1", "0"], ids=["pipe", "no_pipe"])
def pipe(request, monkeypatch):
    monkeypatch.setenv("OBGPU_PIPE", request.param)
    return request.param


class W:
    def __init__(self, table, flt, proj, is_str, elem):
        self.table, self.filter, self.proj, self.proj_is_string, self.proj_elem_len = table, flt, proj, is_str, elem


def test_config3_shape_ragged(ob, ctx, pipe):
    from oceanbase_b200.synth import make_config3_like
    w = make_config3_like(rows=133 * 60 + 71, rows_per_block=133, seed=11)   # last block: 71 rows
    assert assert_scan_matches(ctx, w) > 0


def mixed_table(ob, n, rpb, seed, rowkey_cnt=0):
    """c0 sorted INT DICT, c1 INT DICT over multiples of 3, c2 VARCHAR DICT with NULLs,
    c3 TINYINT DICT with negative values (sign fix), c4 INT BASE_DIFF, c5 INT under ENC_AUTO: runs of one value in
    some blocks (RLE / CONST) and many values in others (DICT)."""
    from oceanbase_b200 import capi
    rng = np.random.default_rng(seed)
    c0 = rng.integers(-40, 40, size=n, dtype=np.int64) * 1_000_003
    words = [b"k%04d" % i + b"z" * (i % 11) for i in range(300)]
    s2 = [words[i] for i in rng.integers(0, len(words), size=n)]
    n2 = (rng.random(n) < 0.04).astype(np.uint8)
    c3 = rng.integers(-100, 100, size=n, dtype=np.int64)
    c4 = np.cumsum(rng.integers(0, 9, size=n, dtype=np.int64)) + 10**12
    c5 = rng.integers(0, 50, size=n, dtype=np.int64)
    for b0 in range(0, n, 2 * rpb):                     # every other block holds one value
        c5[b0:b0 + rpb] = 7
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_DICT, c0), ob.Column(ob.OBJ_INT, ob.ENC_DICT, rng.integers(0, 90, size=n, dtype=np.int64) * 3),
            ob.Column(ob.OBJ_VARCHAR, ob.ENC_DICT, s2, nulls=n2), ob.Column(ob.OBJ_TINYINT, ob.ENC_DICT, c3),
            ob.Column(ob.OBJ_INT, ob.ENC_INTEGER_BASE_DIFF, c4), ob.Column(ob.OBJ_INT, capi.ENC_AUTO, c5)]
    return ob.encode_table(cols, rpb, rowkey_cnt=rowkey_cnt), words


def mixed_filters(ob, words):
    Wt = ob.White
    return {
        "records": ob.And([Wt(0, ob.WHITE_OP_GE, (-30 * 1_000_003,)), Wt(3, ob.WHITE_OP_LT, (20,)),
                           Wt(2, ob.WHITE_OP_IN, tuple(words[k] for k in range(0, 300, 8)))]),
        "unsorted_int": Wt(1, ob.WHITE_OP_BT, (30, 150)),
        "sign_fixed_ne": Wt(3, ob.WHITE_OP_NE, (-5,)),
        "auto_column": ob.And([Wt(5, ob.WHITE_OP_LE, (20,)), Wt(0, ob.WHITE_OP_LT, (0,))]),
        "str_gt_plans": Wt(2, ob.WHITE_OP_GT, (words[150],)),
    }


@pytest.mark.parametrize("rpb,n", [(133, 133 * 40 + 17), (400, 9_000), (512, 10_000), (2000, 12_000)])
@pytest.mark.parametrize("case", ["records", "unsorted_int", "sign_fixed_ne", "auto_column", "str_gt_plans"])
def test_record_and_plan_columns(ob, ctx, pipe, rpb, n, case):
    table, words = mixed_table(ob, n, rpb, seed=rpb)
    flt = mixed_filters(ob, words)[case]
    # flat columns only (records), then with the AUTO column (plans wherever a block is RLE / CONST)
    assert_scan_matches(ctx, W(table, flt, [0, 1, 2, 3, 4], [False, False, True, False, False], [8] * 5))
    assert_scan_matches(ctx, W(table, flt, [2, 5, 3], [True, False, False], [8] * 3))


def _scan_equal(ctx, batch, table, flt, proj, is_str, elem):
    base = 0x10_0000_0000
    res = batch.scan(flt, proj, want_row_ids=True, string_base=base)
    want = ora.scan_table(table, flt, proj, is_str, elem, string_base=base)
    assert res.selected_rows == want["selected"]
    assert np.array_equal(res.fetch_row_ids(), want["row_ids"])
    for i in range(len(proj)):
        data, lens, nulls = res.fetch_col(i)
        assert np.array_equal(nulls, want["nulls"][i])
        if is_str[i]:
            assert np.array_equal(lens, want["lens"][i])
        else:
            assert np.array_equal(data, want["data"][i])
    res.free()


@pytest.mark.parametrize("how", ["lz4", "macro", "device_no_view"])
def test_open_paths(ob, ctx, pipe, how):
    # every open path reaches the one index launch that writes the records: stored (LZ4) blocks, macro blocks, and a
    # device-resident image whose headers the survey kernel reads
    import torch
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import build_macro_blocks, compress_table
    table, words = mixed_table(ob, 133 * 30 + 5, 133, seed=3, rowkey_cnt=1 if how == "macro" else 0)
    keep = None
    if how == "lz4":
        batch = ob.PageBatch(ctx, compress_table(table, capi.COMPRESSOR_LZ4), compressor=capi.COMPRESSOR_LZ4)
    elif how == "macro":
        types = [capi.OBJ_INT, capi.OBJ_INT, capi.OBJ_VARCHAR, capi.OBJ_TINYINT, capi.OBJ_INT, capi.OBJ_INT]
        mi = build_macro_blocks(table, types, 1, macro_block_size=64 << 10)
        batch = ob.PageBatch.from_macro_blocks(ctx, mi.image, 64 << 10, mi.n_macro)
    else:
        keep = torch.from_numpy(table.image).cuda()
        batch = ob.PageBatch(ctx, table, device_image_ptr=keep.data_ptr(), image_size=table.image.size, host_view=False)
    try:
        for case in ("records", "auto_column"):
            _scan_equal(ctx, batch, table, mixed_filters(ob, words)[case], [0, 2, 3, 4], [False, True, False, False], [8] * 4)
            _scan_equal(ctx, batch, table, mixed_filters(ob, words)[case], [2, 5], [True, False], [8] * 2)
    finally:
        batch.close()


def test_cs_dictionaries(ob, ctx, pipe):
    # CS INT_DICT / STR_DICT: the dictionary and ref streams are laid out differently from PAX dictionaries
    rng = np.random.default_rng(4)
    n = 133 * 25 + 9
    k = rng.integers(0, 300, size=n, dtype=np.int64) * 7 - 900
    s = [b"cs%03d" % x + b"q" * (x % 9) for x in rng.integers(0, 60, size=n)]
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_CS_INT_DICT, k), ob.Column(ob.OBJ_VARCHAR, ob.ENC_CS_STR_DICT, s)]
    table = ob.encode_table(cols, 133)
    for flt in (ob.White(0, ob.WHITE_OP_LT, (500,)), ob.White(1, ob.WHITE_OP_IN, (b"cs007qqqqqqq", b"cs040qqqq"))):
        assert_scan_matches(ctx, W(table, flt, [1, 0], [True, False], [8, 8]))


def kernels_run(fn):
    """Names of the CUDA kernels fn() launched (torch.profiler, template arguments kept)."""
    import torch
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.key for e in prof.key_averages() if e.device_time_total > 0}


def scan_kernels(ctx, table, flt, proj):
    batch = ctx.open_batch(table)
    try:
        def run():
            batch.scan(flt, proj, want_row_ids=True).free()
        run()
        return kernels_run(run)
    finally:
        batch.close()


def ran(names, kernel, rec):
    return any(kernel + ("<true>" if rec else "<false>") in k for k in names)


def test_records_are_chosen(ob, ctx, monkeypatch):
    # which instantiation of each pipelined kernel a scan runs: records where every referenced column's blocks allow them
    monkeypatch.delenv("OBGPU_PIPE", raising=False)
    from oceanbase_b200.synth import make_config3_like
    w = make_config3_like(rows=133 * 60, rows_per_block=133, seed=11)
    k = scan_kernels(ctx, w.table, w.filter, w.proj)
    assert ran(k, "obgpu_count_pipe_kernel", True) and ran(k, "obgpu_project_pipe_kernel", True), k
    table, words = mixed_table(ob, 133 * 40 + 17, 133, seed=133)
    f = mixed_filters(ob, words)
    k = scan_kernels(ctx, table, f["records"], [0, 1, 2, 3, 4])
    assert ran(k, "obgpu_count_pipe_kernel", True) and ran(k, "obgpu_project_pipe_kernel", True), k
    k = scan_kernels(ctx, table, f["records"], [2, 5, 3])        # the AUTO column is RLE / CONST in some blocks
    assert ran(k, "obgpu_count_pipe_kernel", True) and ran(k, "obgpu_project_pipe_kernel", False), k
    k = scan_kernels(ctx, table, f["str_gt_plans"], [0, 1])      # a string range leaf needs the plan's dictionary bitset
    assert ran(k, "obgpu_count_pipe_kernel", False) and ran(k, "obgpu_project_pipe_kernel", True), k
    monkeypatch.setenv("OBGPU_PIPE", "1")
    table, words = mixed_table(ob, 12_000, 2000, seed=2000)      # > 1024 rows per block: the count kernel keeps the plans
    k = scan_kernels(ctx, table, mixed_filters(ob, words)["records"], [0, 1, 2, 3, 4])
    assert ran(k, "obgpu_count_pipe_kernel", False) and not ran(k, "obgpu_count_pipe_kernel", True), k
