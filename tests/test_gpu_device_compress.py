"""Micro-blocks compressed on the device (obgpu_compress_blocks): byte for byte what the host writer's
obgpu_writer_compress_blocks writes for the same plain blocks, with LZ4 (2, 7), zstd_1.3.8 (6) and NONE, at every alignment;
the output opens and scans like the plain blocks; phase B (merge -> encode -> compress) frames into the same macro blocks as
the host path; malformed calls return their codes and leave the ctx usable; the launches of a call do not grow with the
number of blocks."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_lz4_blocks import _table, scans_equal

pytestmark = pytest.mark.gpu

COMPRESSORS = (1, 2, 6, 7)   # NONE, LZ4, zstd_1.3.8, LZ4_1_9_1


def _frame(payloads):
    """Plain micro-blocks around arbitrary payloads (the writer checks only the framing), 16-byte aligned offsets."""
    from oceanbase_b200.sstable import TableImage
    blocks, offs, pos = [], [], 0
    for p in payloads:
        h = np.zeros(64, dtype=np.uint8)
        h[0:2] = np.frombuffer(np.int16(1005).tobytes(), np.uint8)
        h[2:4] = np.frombuffer(np.int16(3).tobytes(), np.uint8)
        h[4:8] = np.frombuffer(np.uint32(64).tobytes(), np.uint8)
        h[40:44] = np.frombuffer(np.int32(len(p)).tobytes(), np.uint8)
        h[44:48] = np.frombuffer(np.int32(len(p)).tobytes(), np.uint8)
        b = np.concatenate([h, np.asarray(p, dtype=np.uint8)])
        offs.append(pos)
        pad = (-b.size) % 16
        blocks += [b, np.zeros(pad, np.uint8)]
        pos += b.size + pad
    img = np.concatenate(blocks)
    return TableImage(img, np.array(offs, np.int64), np.array([64 + len(p) for p in payloads], np.int64), 0, 0)


def payload_shapes(seed=11):
    rng = np.random.default_rng(seed)
    P = [rng.integers(0, 4, n, dtype=np.uint8) for n in (0, 1, 5, 11, 12, 13, 17, 40)]   # 12 bytes or less, and just above
    P += [np.zeros(n, np.uint8) for n in (100, 5000, 70_000, 200_000)]                    # offset-1 overlapping matches
    for per in (65534, 65535, 65536, 65537):                                            # periods around the largest offset
        base = rng.integers(0, 256, per, dtype=np.uint8)
        P.append(np.concatenate([base, base, base[:3000]]))
    w = rng.integers(0, 256, 300_000, dtype=np.uint8)   # a word again 65536 and 131072 bytes later: stale entries that collide
    for k in range(0, 160_000, 997):
        w[k + 65536:k + 65544] = w[k:k + 8]
        w[k + 131072:k + 131080] = w[k:k + 8]
    P.append(w)
    P += [rng.integers(0, 256, n, dtype=np.uint8) for n in (300, 70_000, 140_000)]     # incompressible: kept raw
    P += [rng.integers(0, 3, n, dtype=np.uint8) for n in (150_000, 262_145)]
    t = np.arange(100_000, dtype=np.int64)
    P.append(((t * 7) % 251).astype(np.uint8))
    for nl in (31, 32, 33, 4095, 4096, 4097, 20_000):   # literal counts across the literals-header sizes, then a long match
        P.append(np.concatenate([rng.integers(0, 256, nl, dtype=np.uint8), np.zeros(600, np.uint8)]))
    for k in (120, 127, 128, 129, 200, 5000):           # sequence counts across the 1 / 2-byte Number_of_Sequences
        s = [rng.integers(0, 256, 4096, dtype=np.uint8)]
        for o in rng.integers(0, 4000, k):
            s += [rng.integers(0, 256, 3, dtype=np.uint8), s[0][o:o + 9]]
        P.append(np.concatenate(s))
    P.append(np.frombuffer(np.repeat(rng.integers(0, 1 << 20, 30000).astype(np.int64), 3).tobytes(), np.uint8))
    P.append(many_sequences())
    return P


def many_sequences():
    """One 131 040-byte zstd chunk of >= 0x7f00 sequences (the 3-byte Number_of_Sequences, and close to the 32 Ki-entry
    sequence list of a chunk): 200 four-byte words with distinct first bytes and distinct hashes in de Bruijn order 2, so
    that every word after the first occurrences matches its previous occurrence for exactly 4 bytes."""
    rng = np.random.default_rng(3)
    words, hashes = [], set()
    while len(words) < 200:
        w = np.concatenate([[len(words)], rng.integers(0, 256, 3)]).astype(np.uint8)
        h = ((int(w.view(np.uint32)[0]) * 2654435761) & 0xffffffff) >> 16
        if h not in hashes:
            hashes.add(h)
            words.append(w)
    k, a, seq = 200, [0] * 4, []   # de Bruijn B(200, 2), Fredricksen-Kessler-Maiorana

    def db(t, p):
        if t > 2:
            if 2 % p == 0:
                seq.extend(a[1:p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)
    db(1, 1)
    return np.concatenate([words[i] for i in seq[:32760]])


def _on_device(table):
    import torch
    img = torch.from_numpy(np.ascontiguousarray(table.image)).cuda()
    off = torch.from_numpy(np.ascontiguousarray(table.offsets, dtype=np.int64)).cuda()
    sz = torch.from_numpy(np.ascontiguousarray(table.sizes).astype(np.uint32).view(np.int32)).cuda()
    return img, off, sz


def _host_compress(table, compressor, align):
    """obgpu_writer_compress_blocks over the blocks of size > 0 (size 0: a block left to the host writer, passed through)."""
    from oceanbase_b200.sstable import TableImage, compress_table
    keep = np.nonzero(np.asarray(table.sizes) > 0)[0]
    sub = TableImage(table.image, np.asarray(table.offsets)[keep], np.asarray(table.sizes)[keep], 0, 0)
    st = compress_table(sub, compressor, align=align)
    off = np.zeros(table.n_blocks, np.int64)
    sz = np.zeros(table.n_blocks, np.int64)
    sz[keep] = st.sizes
    pos = 0
    for b in range(table.n_blocks):   # the writer's layout: every block at align_up(end of the previous one)
        pos = (pos + align - 1) // align * align
        off[b] = pos
        pos += sz[b]
    assert np.array_equal(off[keep], st.offsets)
    return np.asarray(st.image), off, sz


def assert_device_equals_writer(ctx, table, compressor, align):
    from oceanbase_b200 import compaction
    img, off, sz = _on_device(table)
    out = compaction.compress_blocks(ctx, img.data_ptr(), off.data_ptr(), sz.data_ptr(), table.n_blocks, compressor, align)
    d_img, d_off, d_sz = out.fetch()
    w_img, w_off, w_sz = _host_compress(table, compressor, align)
    assert np.array_equal(d_off, w_off), "offsets differ"
    assert np.array_equal(d_sz, w_sz), ("sizes differ", np.nonzero(d_sz != w_sz)[0][:5])
    assert d_img.size == w_img.size
    if not np.array_equal(d_img, w_img):
        bad = int(np.nonzero(d_img != w_img)[0][0])
        blk = int(np.searchsorted(d_off, bad, side="right") - 1)
        raise AssertionError(f"first differing byte {bad} (block {blk}, byte {bad - d_off[blk]} of {d_sz[blk]})")
    return out


@pytest.fixture(scope="module")
def ctx():
    import oceanbase_b200 as ob
    c = ob.ScanContext(0)
    yield c
    c.close()


def _writer_tables():
    from oceanbase_b200.sstable import TableImage
    from test_gpu_lz4_blocks import _table as t
    return TableImage.concat([t(cs=False, n=20_000)[0], t(cs=True, n=20_000)[0]])


@pytest.mark.parametrize("compressor", COMPRESSORS)
@pytest.mark.parametrize("align", [1, 16, 128, 4096])
def test_payload_shapes_equal_the_writer(ctx, compressor, align):
    assert_device_equals_writer(ctx, _frame(payload_shapes()), compressor, align)


@pytest.mark.parametrize("compressor", COMPRESSORS)
@pytest.mark.parametrize("align", [1, 16, 128, 4096])
def test_writer_tables_equal_the_writer(ctx, compressor, align):
    assert_device_equals_writer(ctx, _writer_tables(), compressor, align)


def test_every_codec_table_equals_the_writer(ctx):
    """Writer tables of every PAX codec and every CS column type, strings included."""
    from oceanbase_b200 import capi as T
    from oceanbase_b200.sstable import Column, TableImage, encode_table
    rng = np.random.default_rng(21)
    n = 12_000
    key = np.arange(n, dtype=np.int64)
    small = rng.integers(0, 30, n, dtype=np.int64)
    runs = np.repeat(rng.integers(0, 9, n // 100 + 1, dtype=np.int64), 100)[:n]
    strs = [b"s-%05d" % (i % 377) for i in range(n)]
    nl = (rng.random(n) < 0.1).astype(np.uint8)
    const = np.where(rng.random(n) < 0.02, small, 5)
    parts = []
    for enc in ("ENC_RAW", "ENC_DICT", "ENC_RLE", "ENC_CONST", "ENC_INTEGER_BASE_DIFF", "ENC_AUTO"):
        v = {"ENC_RLE": runs, "ENC_CONST": const}.get(enc, small)
        parts.append(encode_table([Column(T.OBJ_INT, T.ENC_RAW, key), Column(T.OBJ_INT, getattr(T, enc), v),
                                   Column(T.OBJ_INT, T.ENC_RAW, small, nulls=nl)], 1000, rowkey_cnt=1))
    for enc in ("ENC_CS_INTEGER", "ENC_CS_INT_DICT", "ENC_CS_AUTO"):
        parts.append(encode_table([Column(T.OBJ_INT, T.ENC_CS_INTEGER, key), Column(T.OBJ_INT, getattr(T, enc), small, nulls=nl)],
                                  1000, rowkey_cnt=1))
    for enc in ("ENC_RAW", "ENC_DICT", "ENC_STRING_DIFF", "ENC_HEX_PACKING", "ENC_STRING_PREFIX"):
        vals = [b"%08x" % (i * 7919 % 4096) for i in range(n)] if enc == "ENC_HEX_PACKING" else strs
        parts.append(encode_table([Column(T.OBJ_INT, T.ENC_RAW, key), Column(T.OBJ_VARCHAR, getattr(T, enc), vals)], 1000, rowkey_cnt=1))
    # span columns: COLUMN_EQUAL (a copy of column 1 with exceptions), COLUMN_SUBSTR (the span-column tests' shapes)
    eq = np.where(rng.random(n) < 0.05, small + 1, small)
    parts.append(encode_table([Column(T.OBJ_INT, T.ENC_RAW, key), Column(T.OBJ_INT, T.ENC_RAW, small),
                               Column(T.OBJ_INT, T.ENC_COLUMN_EQUAL, eq, ref_col=1)], 1000, rowkey_cnt=1))
    from test_span_columns import SUB
    for _, rv, rn, v, vn in SUB:
        parts.append(encode_table([Column(T.OBJ_VARCHAR, T.ENC_RAW, rv, nulls=rn), Column(T.OBJ_INT, T.ENC_RAW, np.arange(len(v))),
                                   Column(T.OBJ_VARCHAR, T.ENC_COLUMN_SUBSTR, v, nulls=vn, ref_col=0)], 190))
    for enc in ("ENC_CS_STRING", "ENC_CS_STR_DICT"):
        parts.append(encode_table([Column(T.OBJ_INT, T.ENC_CS_INTEGER, key), Column(T.OBJ_VARCHAR, getattr(T, enc), strs)],
                                  1000, rowkey_cnt=1))
    table = TableImage.concat(parts)
    for c in COMPRESSORS:
        assert_device_equals_writer(ctx, table, c, 128)


def test_device_encoder_image_with_host_blocks(ctx):
    """A device-encoder image with a NULL-dominated column: its size-0 block passes through as size 0."""
    from test_gpu_device_encoder import device_encode, make_columns
    from oceanbase_b200.sstable import TableImage
    rng = np.random.default_rng(6)
    n, rpb = 4_000, 500
    cols = make_columns(rng, n, [(5, 30, 0.0, False), (5, 60, 0.0, False)])
    nl = np.zeros(n, dtype=np.uint8)
    nl[1500:2000:2] = 1
    cols[1] = (cols[1][0], cols[1][1], nl, False)
    enc, _ = device_encode(ctx, cols, rpb, 1)
    img, off, sz = enc.fetch()
    assert sz[3] == 0
    for c in COMPRESSORS:
        out = enc.compress(c, align=128)
        d_img, d_off, d_sz = out.fetch()
        assert d_sz[3] == 0
        w_img, w_off, w_sz = _host_compress(TableImage(img, off, sz, n, 2), c, 128)
        assert np.array_equal(d_off, w_off) and np.array_equal(d_sz, w_sz) and np.array_equal(d_img, w_img)
    enc.free()


def test_twenty_thousand_blocks(ctx):
    table, _ = _table(n=20_000 * 40, rpb=40, seed=4)
    assert table.n_blocks >= 20_000
    for c in (2, 6):
        assert_device_equals_writer(ctx, table, c, 16)


@pytest.mark.parametrize("cs", [False, True])
@pytest.mark.parametrize("compressor", [2, 6, 7])
def test_round_trip_opens_and_scans_like_the_plain_batch(ctx, cs, compressor):
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import TableImage
    table, _ = _table(cs=cs)
    img, off, sz = _on_device(table)
    from oceanbase_b200 import compaction
    out = compaction.compress_blocks(ctx, img.data_ptr(), off.data_ptr(), sz.data_ptr(), table.n_blocks, compressor)
    d_img, d_off, d_sz = out.fetch()
    st = TableImage(d_img, d_off, d_sz, table.total_rows, table.n_cols)
    plain = ob.PageBatch(ctx, table)
    cb = ob.PageBatch(ctx, st, device_image_ptr=out.image.data_ptr(), image_size=out.image_size, compressor=compressor)
    scans_equal(plain, cb)
    cb.close()
    plain.close()


def test_phase_b_end_to_end(ctx):
    """merge -> encode_merge_result -> Encoded.compress -> open scans like the plain image; the fetched blocks frame into the
    macro blocks build_macro_blocks makes from the plain image, and those open."""
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi, compaction
    from oceanbase_b200.sstable import Column, MacroImage, TableImage, build_macro_blocks, encode_table
    rng = np.random.default_rng(12)
    runs = []
    for r in range(3):
        n = 30_000
        key = np.sort(rng.choice(200_000, n, replace=False)).astype(np.int64)
        runs.append(encode_table([Column(capi.OBJ_INT, capi.ENC_RAW, key),
                                  Column(capi.OBJ_INT, capi.ENC_RAW, rng.integers(0, 50, n, dtype=np.int64)),
                                  Column(capi.OBJ_INT, capi.ENC_RAW, rng.integers(0, 1 << 40, n, dtype=np.int64))], 1000, rowkey_cnt=1))
    batches = [ob.PageBatch(ctx, t) for t in runs]
    res = compaction.merge_batches(ctx, batches, 0, None, [1, 2])
    enc = compaction.encode_merge_result(res, [-1, 0, 1], [capi.OBJ_INT] * 3, 1000)
    p_img, p_off, p_sz = enc.fetch()
    ck = enc.column_checksums()
    plain_t = TableImage(p_img, p_off, p_sz, int(enc.info().total_rows), 3)
    types = [capi.OBJ_INT] * 3
    for c in (2, 6):
        out = enc.compress(c)
        d_img, d_off, d_sz = out.fetch()
        assert np.array_equal(enc.column_checksums(), ck)
        st = TableImage(d_img, d_off, d_sz, 0, 3)
        pb = ob.PageBatch(ctx, TableImage(p_img, p_off, p_sz, 0, 3))
        cb = ob.PageBatch(ctx, st, device_image_ptr=out.image.data_ptr(), image_size=out.image_size, compressor=c)
        assert cb.total_rows == pb.total_rows and cb.n_blocks == pb.n_blocks
        for col in range(3):
            r1, r2 = pb.scan(None, [col]), cb.scan(None, [col])
            assert np.array_equal(r1.fetch_col(0)[0], r2.fetch_col(0)[0])
            r1.free()
            r2.free()
        cb.close()
        pb.close()
        want = build_macro_blocks(plain_t, types, 1, macro_block_size=256 << 10, compressor=c)
        got = _macro_from_stored(st, types, 256 << 10, c)
        assert got.n_macro == want.n_macro and np.array_equal(got.image, want.image)
        mb = ob.PageBatch.from_macro_blocks(ctx, got.image, got.macro_block_size, got.n_macro)
        assert mb.total_rows == res.info().out_rows
        mb.close()
    enc.free()
    for b in batches:
        b.close()


def _macro_from_stored(st, types, macro_size, compressor):
    """obgpu_writer_build_macro_blocks_ex over blocks already in stored form (the macro headers record `compressor`)."""
    from oceanbase_b200 import capi
    from oceanbase_b200.capi import lib, check
    from oceanbase_b200.sstable import MacroImage
    n_cols = len(types)
    metas = np.zeros((n_cols, 4), dtype=np.uint8)
    metas[:, 0] = types
    orders = np.zeros(n_cols, dtype=np.int32)
    spec = capi.MacroSpec(200001, 1, 0, 1, 0, 1, n_cols, metas.ctypes.data, orders.ctypes.data, macro_size)
    img, off, sz = np.ascontiguousarray(st.image), np.ascontiguousarray(st.offsets), np.ascontiguousarray(st.sizes)
    out = np.zeros(st.n_blocks * macro_size, dtype=np.uint8)
    first = np.zeros(st.n_blocks + 1, dtype=np.int32)
    size, nm = C.c_int64(0), C.c_int32(0)
    check(lib.obgpu_writer_build_macro_blocks_ex(img.ctypes.data, off.ctypes.data, sz.ctypes.data, st.n_blocks, C.byref(spec),
                                                 out.ctypes.data, out.size, C.byref(size), C.byref(nm), first.ctypes.data, first.size,
                                                 compressor), "obgpu_writer_build_macro_blocks_ex")
    return MacroImage(out[:size.value], macro_size, nm.value, first[:nm.value + 1].copy())


def _raw_call(ctx, img, off, sz, n, compressor, align, out, cap):
    from oceanbase_b200.capi import lib
    o_off = __import__("torch").zeros(n, dtype=__import__("torch").int64, device="cuda")
    o_sz = __import__("torch").zeros(n, dtype=__import__("torch").int32, device="cuda")
    size = C.c_int64(-1)
    code = lib.obgpu_compress_blocks(ctx._h, img, off, sz, n, compressor, align, out, cap, o_off.data_ptr(), o_sz.data_ptr(),
                                     C.byref(size))
    return code, size.value


def test_errors_leave_the_ctx_usable(ctx):
    import torch
    import oceanbase_b200 as ob
    table = _frame(payload_shapes()[:20])
    img, off, sz = _on_device(table)
    n = table.n_blocks
    cap = int(((np.asarray(table.sizes) + 127) // 128 * 128).sum())
    out = torch.full((cap + 64,), 0xAB, dtype=torch.uint8, device="cuda")
    # the size query
    code, q = _raw_call(ctx, img.data_ptr(), off.data_ptr(), sz.data_ptr(), n, 2, 128, None, 0)
    assert code == ob.OB_SUCCESS and q == cap
    for comp in (5, 0, 3, 4, 8, 99, -1):
        assert _raw_call(ctx, img.data_ptr(), off.data_ptr(), sz.data_ptr(), n, comp, 128, out.data_ptr(), cap)[0] == ob.OB_NOT_SUPPORTED
    for align in (0, 3, 8192, -16):
        assert _raw_call(ctx, img.data_ptr(), off.data_ptr(), sz.data_ptr(), n, 2, align, out.data_ptr(), cap)[0] == ob.OB_INVALID_ARGUMENT
    assert _raw_call(ctx, img.data_ptr(), off.data_ptr(), sz.data_ptr(), 0, 2, 128, out.data_ptr(), cap)[0] == ob.OB_INVALID_ARGUMENT
    # one byte short: nothing written
    assert _raw_call(ctx, img.data_ptr(), off.data_ptr(), sz.data_ptr(), n, 2, 128, out.data_ptr(), cap - 1)[0] == ob.OB_BUF_NOT_ENOUGH
    assert bool((out == 0xAB).all())
    # a block above 0x7f000000 bytes: refused before its header is read
    big = sz.clone()
    big[2] = 0x7f000010
    assert _raw_call(ctx, img.data_ptr(), off.data_ptr(), big.data_ptr(), n, 2, 128, out.data_ptr(), cap)[0] == ob.OB_NOT_SUPPORTED
    # misaligned offsets
    bad_off = off.clone()
    bad_off[3] += 8
    assert _raw_call(ctx, img.data_ptr(), bad_off.data_ptr(), sz.data_ptr(), n, 6, 128, out.data_ptr(), cap)[0] == ob.OB_INVALID_ARGUMENT
    # a stored (data_zlength_ != data_length_) block
    bad = img.clone()
    o5 = int(table.offsets[5])
    bad[o5 + 44] ^= 1
    assert _raw_call(ctx, bad.data_ptr(), off.data_ptr(), sz.data_ptr(), n, 6, 128, out.data_ptr(), cap)[0] == ob.OB_INVALID_DATA
    assert bool((out == 0xAB).all())
    for c in COMPRESSORS:
        assert_device_equals_writer(ctx, table, c, 128)


def test_launches_do_not_grow_with_the_block_count(ctx):
    from oceanbase_b200 import compaction
    counts = []
    for nb in (10, 20_000):
        table = _frame([np.tile(np.arange(50, dtype=np.uint8), 20)] * nb)
        img, off, sz = _on_device(table)
        for c in (2, 6):
            before = ctx.launch_count
            compaction.compress_blocks(ctx, img.data_ptr(), off.data_ptr(), sz.data_ptr(), nb, c, 128)
            counts.append((c, ctx.launch_count - before))
    assert counts[:2] == counts[2:], counts
