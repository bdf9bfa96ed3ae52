"""Opening a page batch: what every open path does before the first scan. Malformed micro-block headers are refused with the same
OB code and ctx error whether the headers are read from a host view or surveyed on the device; each kind of batch (plain PAX with
and without a host view, CS blocks with coded integer streams, PAX blocks whose strings are rebuilt at open, both in one batch,
LZ4 / zstd stored blocks, macro blocks) costs a fixed number of kernel launches, ends in a device image of a fixed size, reports
every block's row and column count, and scans like the plain table it was made from."""
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, RPB = 6000, 500


def _columns(kind):
    from oceanbase_b200 import capi as T
    from oceanbase_b200.sstable import Column
    rng = np.random.default_rng(11)
    key = np.arange(N, dtype=np.int64) * 2 + 5
    small = rng.integers(0, 40, size=N, dtype=np.int64)
    nl = (rng.random(N) < 0.07).astype(np.uint8)
    strs = [b"order-%05d-x" % ((i * 7) % 997) for i in range(N)]   # one length, shared prefix and suffix: STRING_DIFF applies
    if kind == "cs":
        return [Column(T.OBJ_INT, T.ENC_CS_INTEGER, key), Column(T.OBJ_INT, T.ENC_CS_INTEGER, small, nulls=nl),
                Column(T.OBJ_INT, T.ENC_CS_INT_DICT, small), Column(T.OBJ_VARCHAR, T.ENC_CS_STRING, strs)]
    str_enc = T.ENC_STRING_DIFF if kind == "diff" else T.ENC_RAW
    return [Column(T.OBJ_INT, T.ENC_RAW, key), Column(T.OBJ_INT, T.ENC_RAW, small, nulls=nl),
            Column(T.OBJ_INT, T.ENC_DICT, small), Column(T.OBJ_VARCHAR, str_enc, strs)]


@functools.lru_cache(maxsize=None)
def tables():
    """name -> (table, the plain table it scans like)"""
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import TableImage, build_macro_blocks, compress_table, encode_table
    pax = encode_table(_columns("pax"), RPB, rowkey_cnt=1)
    cs_raw = encode_table(_columns("cs"), RPB, rowkey_cnt=1)
    capi.lib.obgpu_writer_set_cs_stream_encoding(0)      # detect: the sorted key column takes a delta codec
    try:
        cs = encode_table(_columns("cs"), RPB, rowkey_cnt=1)
    finally:
        capi.lib.obgpu_writer_set_cs_stream_encoding(1)
    assert cs.image.size < cs_raw.image.size
    diff = encode_table(_columns("diff"), RPB, rowkey_cnt=1)
    types = [capi.OBJ_INT, capi.OBJ_INT, capi.OBJ_INT, capi.OBJ_VARCHAR]
    return {"pax": (pax, pax), "cs": (cs, cs_raw), "diff": (diff, pax), "both": (TableImage.concat([diff, cs]), TableImage.concat([pax, cs_raw])),
            "lz4": (compress_table(pax, capi.COMPRESSOR_LZ4), pax), "zstd": (compress_table(pax, capi.COMPRESSOR_ZSTD_1_3_8), pax),
            "macro": (build_macro_blocks(pax, types, 1, macro_block_size=64 << 10), pax)}


# kind -> (table, how it is opened)
KINDS = {
    "pax_host_image": ("pax", "host"),
    "pax_device_image_host_view": ("pax", "device_view"),
    "pax_device_image_no_view": ("pax", "device"),
    "cs_coded_streams": ("cs", "host"),
    "pax_string_diff": ("diff", "host"),
    "cs_and_string_diff": ("both", "host"),
    "cs_and_string_diff_no_view": ("both", "device"),
    "lz4_host_image": ("lz4", "host"),
    "zstd_device_image": ("zstd", "device"),
    "macro_blocks": ("macro", "host"),
}

# kind -> (kernel launches of one open, bytes of the device image the opened batch reads)
OPEN_COST = {
    "pax_host_image": (1, 100096),
    "pax_device_image_host_view": (1, 100096),
    "pax_device_image_no_view": (4, 100096),
    "cs_coded_streams": (4, 104448),
    "pax_string_diff": (5, 137600),
    "cs_and_string_diff": (8, 242048),
    "cs_and_string_diff_no_view": (9, 242048),
    "lz4_host_image": (6, 100096),
    "zstd_device_image": (6, 100096),
    "macro_blocks": (8, 100096),
}


def open_kind(ctx, kind):
    """(batch, device buffer the batch reads or None, plain table)"""
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi
    name, how = KINDS[kind]
    table, plain = tables()[name]
    keep = None
    if name == "macro":
        batch = ob.PageBatch.from_macro_blocks(ctx, table.image, table.macro_block_size, table.n_macro)
    else:
        comp = {"lz4": capi.COMPRESSOR_LZ4, "zstd": capi.COMPRESSOR_ZSTD_1_3_8}.get(name)
        if how == "host":
            batch = ob.PageBatch(ctx, table, compressor=comp)
        else:
            keep = torch.from_numpy(table.image).cuda()
            batch = ob.PageBatch(ctx, table, device_image_ptr=keep.data_ptr(), image_size=table.image.size, host_view=how == "device_view",
                                 compressor=comp)
    return batch, keep, plain


def measure(ctx, kind):
    """(launches of the open, device image bytes) of one open of `kind`"""
    before = ctx.launch_count
    batch, keep, _ = open_kind(ctx, kind)
    ctx.synchronize()
    launches = ctx.launch_count - before
    image_bytes = batch.device_image()[1]
    batch.close()
    del keep
    return launches, image_bytes


def header_facts(table):
    """(row count, column count) of every block, from its header"""
    out = []
    for i in range(table.n_blocks):
        blk = table.block(i)
        out.append((int(blk[16:20].view(np.uint32)[0]), int(blk[10:12].view(np.uint16)[0])))
    return out


@pytest.mark.parametrize("kind", list(KINDS))
def test_open_launches_image_and_blocks(kind):
    import oceanbase_b200 as ob
    ctx = ob.ScanContext(0)
    assert measure(ctx, kind) == OPEN_COST[kind]
    batch, keep, plain = open_kind(ctx, kind)
    assert batch.n_blocks == plain.n_blocks and batch.total_rows == plain.total_rows
    assert [batch.block_info(i) for i in range(batch.n_blocks)] == header_facts(plain)
    ref = ob.PageBatch(ctx, plain)
    f = ob.And([ob.White(1, ob.WHITE_OP_LT, [30]), ob.White(2, ob.WHITE_OP_NE, [7])])
    r1, r2 = batch.scan(f, [0, 1, 2, 3], want_row_ids=True), ref.scan(f, [0, 1, 2, 3], want_row_ids=True)
    assert r1.selected_rows == r2.selected_rows > 0
    assert np.array_equal(r1.fetch_row_ids(), r2.fetch_row_ids())
    for i in range(3):
        d1, _, n1 = r1.fetch_col(i)
        d2, _, n2 = r2.fetch_col(i)
        assert np.array_equal(d1, d2) and np.array_equal(n1, n2)
    h1, o1 = r1.fetch_strings(3)
    h2, o2 = r2.fetch_strings(3)
    assert np.array_equal(o1, o2) and np.array_equal(h1, h2)
    r1.free()
    r2.free()
    ref.close()
    batch.close()
    del keep
    ctx.close()


def _put(blk, off, fmt, value):
    blk[off:off + np.dtype(fmt).itemsize] = np.array([value], dtype=fmt).view(np.uint8)


# name -> (patch of the block's bytes, host-view verdict, device-survey verdict); a verdict is (OB code name, ctx error or None:
# the error the ctx had before)
BAD_HEADERS = {
    "bad_magic": (lambda b: _put(b, 0, "<i2", 1006), ("OB_INVALID_DATA", "invalid micro block header"),
                  ("OB_INVALID_DATA", "invalid micro block header")),
    "version_0": (lambda b: _put(b, 2, "<i2", 0), ("OB_INVALID_DATA", "invalid micro block header"),
                  ("OB_INVALID_DATA", "invalid micro block header")),
    "version_4": (lambda b: _put(b, 2, "<i2", 4), ("OB_INVALID_DATA", "invalid micro block header"),
                  ("OB_INVALID_DATA", "invalid micro block header")),
    "ncol_below_nkey": (lambda b: _put(b, 12, "<u2", int(b[10:12].view(np.uint16)[0]) + 1), ("OB_INVALID_DATA", "invalid micro block header"),
                        ("OB_INVALID_DATA", "invalid micro block header")),
    "row_store_0": (lambda b: _put(b, 20, "<u1", 0), ("OB_NOT_SUPPORTED", "row store type not handled by the device path"),
                    ("OB_NOT_SUPPORTED", "micro block not handled by the device path")),
    "row_store_4": (lambda b: _put(b, 20, "<u1", 4), ("OB_NOT_SUPPORTED", "row store type not handled by the device path"),
                    ("OB_NOT_SUPPORTED", "micro block not handled by the device path")),
    "row_store_5": (lambda b: _put(b, 20, "<u1", 5), ("OB_INVALID_DATA", "invalid micro block header"),
                    ("OB_INVALID_DATA", "invalid micro block header")),
    "column_headers_past_block": (lambda b: _put(b, 4, "<u4", b.size - 8), ("OB_INVALID_DATA", None),
                                  ("OB_INVALID_DATA", "invalid micro block header")),
    "zero_rows": (lambda b: _put(b, 16, "<u4", 0), ("OB_INVALID_DATA", None), ("OB_INVALID_DATA", "invalid micro block header")),
    "rows_70000": (lambda b: _put(b, 16, "<u4", 70000), ("OB_NOT_SUPPORTED", "more than 65535 rows in one micro block"),
                   ("OB_NOT_SUPPORTED", "micro block not handled by the device path")),
}


@pytest.mark.parametrize("name", list(BAD_HEADERS))
def test_malformed_header_is_refused_alike_with_and_without_host_view(name):
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import TableImage
    pax = tables()["pax"][0]
    patch, host_verdict, device_verdict = BAD_HEADERS[name]
    image = pax.image.copy()
    patch(image[pax.offsets[1]:pax.offsets[1] + pax.sizes[1]])   # the second block: the first one opens
    bad = TableImage(image, pax.offsets, pax.sizes, pax.total_rows, pax.n_cols)
    ctx = ob.ScanContext(0)
    keep = torch.from_numpy(image).cuda()
    for verdict, opener in ((host_verdict, lambda: ob.PageBatch(ctx, bad)),
                            (device_verdict, lambda: ob.PageBatch(ctx, bad, device_image_ptr=keep.data_ptr(), image_size=image.size,
                                                                  host_view=False))):
        before = ctx.last_error()
        with pytest.raises(capi.ObGpuError) as ei:
            opener()
        assert ei.value.code == getattr(capi, verdict[0])
        assert ctx.last_error() == (before if verdict[1] is None else verdict[1])
    # the ctx stays usable
    good = ob.PageBatch(ctx, pax)
    assert good.total_rows == N
    good.close()
    del keep
    ctx.close()
