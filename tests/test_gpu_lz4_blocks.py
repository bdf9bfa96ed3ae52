"""LZ4-compressed micro-blocks decoded on the device: obgpu_lz4_decompress against the checker decoder (tests/lz4_ref.py) on the
committed liblz4 vectors and on malformed streams; page batches opened from stored-form blocks (obgpu_batch_open_compressed)
and from compressed macro blocks scan bit for bit like the plain batch; corrupt input is refused with OBGPU_INVALID_DATA
and the ctx keeps working; string pointers rebased on obgpu_batch_device_image address the right device bytes."""
import ctypes as C

import numpy as np
import pytest

import lz4_ref
import oracle_binding as ora
from test_lz4_blocks import liblz4, malformed, vectors, SPEC_VECTORS

pytestmark = pytest.mark.gpu


def _table(cs=False, n=60_000, rpb=900, seed=3):
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import Column, encode_table
    rng = np.random.default_rng(seed)
    key = np.arange(n, dtype=np.int64) * 2 + 5
    small = rng.integers(0, 40, size=n, dtype=np.int64)
    nl = (rng.random(n) < 0.07).astype(np.uint8)
    strs = [b"name-%04d" % (i % 211) for i in range(n)]
    T = capi
    if cs:
        cols = [Column(T.OBJ_INT, T.ENC_CS_INTEGER, key), Column(T.OBJ_INT, T.ENC_CS_INTEGER, small, nulls=nl),
                Column(T.OBJ_INT, T.ENC_CS_INT_DICT, small), Column(T.OBJ_VARCHAR, T.ENC_CS_STRING, strs)]
    else:
        cols = [Column(T.OBJ_INT, T.ENC_RAW, key), Column(T.OBJ_INT, T.ENC_RAW, small, nulls=nl),
                Column(T.OBJ_INT, T.ENC_DICT, small), Column(T.OBJ_VARCHAR, T.ENC_RAW, strs)]
    return encode_table(cols, rpb, rowkey_cnt=1), [T.OBJ_INT, T.OBJ_INT, T.OBJ_INT, T.OBJ_VARCHAR]


def scans_equal(b1, b2):
    """Selection, sel_offsets, row ids, every projected column (strings as bytes), aggregates and GROUP BY."""
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi
    f = ob.And([ob.White(1, ob.WHITE_OP_LT, [30]), ob.White(2, ob.WHITE_OP_NE, [7])])
    for flt in (f, None):
        r1 = b1.scan(flt, [0, 1, 2, 3], want_row_ids=True)
        r2 = b2.scan(flt, [0, 1, 2, 3], want_row_ids=True)
        assert r1.selected_rows == r2.selected_rows > 0
        assert np.array_equal(r1.fetch_sel_offsets(), r2.fetch_sel_offsets())
        assert np.array_equal(r1.fetch_row_ids(), r2.fetch_row_ids())
        for i in range(3):
            d1, _, n1 = r1.fetch_col(i)
            d2, _, n2 = r2.fetch_col(i)
            assert np.array_equal(d1, d2) and np.array_equal(n1, n2)
        h1, o1 = r1.fetch_strings(3)
        h2, o2 = r2.fetch_strings(3)
        assert np.array_equal(o1, o2) and np.array_equal(h1, h2)
        for kind in (capi.AGG_COUNT, capi.AGG_SUM, capi.AGG_MIN, capi.AGG_MAX):
            assert r1.aggregate(kind, 1) == r2.aggregate(kind, 1)
        if flt is not None:
            aggs = [(capi.AGG_COUNT, -1), (capi.AGG_SUM, 1)]
            g1, g2 = r1.group_by(2, aggs), r2.group_by(2, aggs)
            for a, b in zip(g1, g2):
                assert np.array_equal(a, b)
        r1.free()
        r2.free()


def test_lz4_decompress_vectors_and_malformed_streams():
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200.capi import lib
    cases = [(s, p, True) for s, p, _ in vectors()] + [(s, w, True) for s, w in SPEC_VECTORS if w]
    cases += [(s, b"\0" * n, False) for _, s, n in malformed() if s]
    ins = [np.frombuffer(s, dtype=np.uint8) for s, _, _ in cases]
    in_len = np.array([len(s) for s, _, _ in cases], dtype=np.int64)
    in_off = np.concatenate([[0], np.cumsum(in_len)[:-1]]).astype(np.int64)
    out_len = np.array([len(p) for _, p, _ in cases], dtype=np.int64)
    out_off = np.concatenate([[0], np.cumsum(out_len)[:-1]]).astype(np.int64)
    d_in = torch.from_numpy(np.concatenate(ins)).cuda()
    d_out = torch.zeros(int(out_len.sum()), dtype=torch.uint8, device="cuda")
    status = np.full(len(cases), -1, dtype=np.int32)
    ctx = ob.ScanContext(0)
    code = lib.obgpu_lz4_decompress(ctx._h, C.c_void_p(d_in.data_ptr()), in_off.ctypes.data, in_len.ctypes.data,
                                    C.c_void_p(d_out.data_ptr()), out_off.ctypes.data, out_len.ctypes.data, len(cases), status.ctypes.data)
    assert code == ob.OB_INVALID_DATA   # the malformed streams are in the batch
    out = d_out.cpu().numpy()
    for k, (s, p, good) in enumerate(cases):
        try:
            want = lz4_ref.lz4_decompress(s, len(p))
        except lz4_ref.Lz4Error:
            want = None
        assert (want is not None) == good, k
        assert (status[k] == 0) == good, (k, status[k])
        if good:
            assert out[out_off[k]:out_off[k] + out_len[k]].tobytes() == want, k
    # the ctx stays usable after the refusals: the valid vectors alone decode with status 0
    ok = [k for k, c in enumerate(cases) if c[2]]
    st2 = np.full(len(ok), -1, dtype=np.int32)
    assert lib.obgpu_lz4_decompress(ctx._h, C.c_void_p(d_in.data_ptr()), in_off[ok].copy().ctypes.data, in_len[ok].copy().ctypes.data,
                                    C.c_void_p(d_out.data_ptr()), out_off[ok].copy().ctypes.data, out_len[ok].copy().ctypes.data,
                                    len(ok), st2.ctypes.data) == 0
    assert (st2 == 0).all()
    ctx.close()


@pytest.mark.parametrize("cs", [False, True])
@pytest.mark.parametrize("compressor,on_device", [(2, False), (7, True)])
def test_compressed_batch_scans_like_the_plain_batch(cs, compressor, on_device):
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import compress_table
    table, _ = _table(cs=cs)
    st = compress_table(table, compressor)
    n_comp = int((np.array([lz4_ref.header_fields(st.block(i))[2] for i in range(st.n_blocks)]) <
                  np.array([lz4_ref.header_fields(st.block(i))[1] for i in range(st.n_blocks)])).sum())
    assert n_comp >= 0.9 * st.n_blocks
    ctx = ob.ScanContext(0)
    plain = ob.PageBatch(ctx, table)
    keep = None
    if on_device:
        keep = torch.from_numpy(st.image).cuda()
        cb = ob.PageBatch(ctx, st, device_image_ptr=keep.data_ptr(), image_size=st.image.size, compressor=compressor)
    else:
        cb = ob.PageBatch(ctx, st, compressor=compressor)
    assert cb.n_blocks == table.n_blocks and cb.total_rows == table.total_rows
    scans_equal(plain, cb)
    cb.close()
    plain.close()
    ctx.close()


def test_mixed_raw_and_compressed_blocks_and_edge_sizes():
    """Raw and compressed blocks in one batch, a 1-row block and a block larger than 16 KiB, opened with LZ4 and with NONE
    (which must refuse the compressed blocks)."""
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import Column, TableImage, compress_table, encode_table
    rng = np.random.default_rng(9)
    t1, _ = _table(n=9000, rpb=900)
    noise = encode_table([Column(capi.OBJ_INT, capi.ENC_RAW, rng.integers(-(1 << 62), 1 << 62, size=2700, dtype=np.int64)),
                          Column(capi.OBJ_INT, capi.ENC_RAW, rng.integers(0, 40, size=2700, dtype=np.int64)),
                          Column(capi.OBJ_INT, capi.ENC_DICT, rng.integers(0, 40, size=2700, dtype=np.int64)),
                          Column(capi.OBJ_VARCHAR, capi.ENC_RAW, [rng.bytes(12) for _ in range(2700)])], 900, rowkey_cnt=1)
    one, _ = _table(n=1, rpb=1)
    big, _ = _table(n=6000, rpb=6000)
    assert big.sizes.max() > 16384
    table = TableImage.concat([t1, noise, one, big])
    st = compress_table(table, capi.COMPRESSOR_LZ4)
    kinds = [lz4_ref.header_fields(st.block(i)) for i in range(st.n_blocks)]
    assert any(z == l for _, l, z in kinds) and any(z < l for _, l, z in kinds)
    ctx = ob.ScanContext(0)
    plain = ob.PageBatch(ctx, table)
    cb = ob.PageBatch(ctx, st, compressor=capi.COMPRESSOR_LZ4)
    scans_equal(plain, cb)
    cb.close()
    with pytest.raises(ob.ObGpuError) as e:
        ob.PageBatch(ctx, st, compressor=capi.COMPRESSOR_NONE)
    assert e.value.code == ob.OB_INVALID_DATA
    with pytest.raises(ob.ObGpuError) as e:
        ob.PageBatch(ctx, st, compressor=5)   # zstd
    assert e.value.code == ob.OB_NOT_SUPPORTED
    plain.close()
    ctx.close()


def test_twenty_thousand_block_batch():
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import compress_table
    table, _ = _table(n=20_000 * 40, rpb=40, seed=4)
    assert table.n_blocks >= 20_000
    st = compress_table(table, 7)
    ctx = ob.ScanContext(0)
    plain, cb = ob.PageBatch(ctx, table), ob.PageBatch(ctx, st, compressor=7)
    scans_equal(plain, cb)
    cb.close()
    plain.close()
    ctx.close()


def _reframe_with(table, compress):
    """Stored-form blocks whose payloads come from `compress` (bytes -> bytes); kept raw when not smaller."""
    from oceanbase_b200.sstable import TableImage
    crc = lambda a: int(ora.oracle().ora_crc64_sse42(0, a.ctypes.data, a.size))
    out = []
    for i in range(table.n_blocks):
        b = table.block(i).copy()
        hs, ln, _ = lz4_ref.header_fields(b)
        z = np.frombuffer(compress(b[hs:].tobytes()), dtype=np.uint8)
        if z.size >= ln:
            out.append(b)
            continue
        nb = np.concatenate([b[:hs], z])
        nb[44:48] = np.frombuffer(np.int32(z.size).tobytes(), np.uint8)
        nb[48:56] = np.frombuffer(np.uint64(crc(np.ascontiguousarray(z))).tobytes(), np.uint8)
        nb[8:10] = 0
        nb[8:10] = np.frombuffer(np.uint16(lz4_ref.header_checksum_fold(nb)).tobytes(), np.uint8)
        out.append(nb)
    offs = np.concatenate([[0], np.cumsum([len(x) for x in out])[:-1]]).astype(np.int64)
    return TableImage(np.concatenate(out), offs, np.array([len(x) for x in out], dtype=np.int64), table.total_rows, table.n_cols)


@pytest.mark.parametrize("kind", ["default", "fast8", "hc9"])
def test_payloads_from_liblz4(kind):
    lz = liblz4()
    if lz is None:
        pytest.skip("liblz4.so.1 not present")
    import oceanbase_b200 as ob
    lz.LZ4_compressBound.argtypes = [C.c_int]
    lz.LZ4_compress_default.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int]
    lz.LZ4_compress_fast.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    lz.LZ4_compress_HC.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int]

    def comp(p):
        cap = lz.LZ4_compressBound(len(p))
        buf = C.create_string_buffer(cap)
        n = (lz.LZ4_compress_default(p, buf, len(p), cap) if kind == "default" else
             lz.LZ4_compress_fast(p, buf, len(p), cap, 8) if kind == "fast8" else lz.LZ4_compress_HC(p, buf, len(p), cap, 9))
        return buf.raw[:n]
    for cs in (False, True):
        table, _ = _table(cs=cs, n=20_000)
        st = _reframe_with(table, comp)
        ctx = ob.ScanContext(0)
        plain, cb = ob.PageBatch(ctx, table), ob.PageBatch(ctx, st, compressor=2)
        scans_equal(plain, cb)
        cb.close()
        plain.close()
        ctx.close()


@pytest.mark.parametrize("macro_size,on_device,compressor", [(2 << 20, False, 2), (256 << 10, True, 7), (64 << 10, False, 7)])
def test_compressed_macro_blocks_scan_like_the_plain_image(macro_size, on_device, compressor):
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import build_macro_blocks
    for cs in (False, True):
        table, types = _table(cs=cs)
        mi = build_macro_blocks(table, types, 1, macro_block_size=macro_size, compressor=compressor)
        ctx = ob.ScanContext(0)
        plain = ob.PageBatch(ctx, table)
        keep = None
        if on_device:
            keep = torch.from_numpy(mi.image).cuda()
            mb = ob.PageBatch.from_macro_blocks(ctx, None, macro_size, mi.n_macro, device_ptr=keep.data_ptr())
        else:
            mb = ob.PageBatch.from_macro_blocks(ctx, mi.image, macro_size, mi.n_macro)
        assert mb.n_blocks == table.n_blocks and mb.total_rows == table.total_rows
        scans_equal(plain, mb)
        mb.close()
        plain.close()
        ctx.close()


def test_corrupt_input_is_refused_and_the_ctx_keeps_working():
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import compress_table
    table, _ = _table(n=9000)
    st = compress_table(table, 2)
    crc = lambda a: int(ora.oracle().ora_crc64_sse42(0, a.ctypes.data, a.size))
    hs, ln, zl = lz4_ref.header_fields(st.block(3))
    assert zl < ln
    ctx = ob.ScanContext(0)
    # a flipped payload byte: the checker's checksum verifier refuses it, and so does the device (checksum)
    bad = st.image.copy()
    bad[st.offsets[3] + hs + zl // 2] ^= 0x20
    blk = bad[st.offsets[3]:st.offsets[3] + st.sizes[3]]
    assert not lz4_ref.stored_checksums_ok(blk, crc)
    with pytest.raises(ob.ObGpuError) as e:
        ob.PageBatch(ctx, type(st)(bad, st.offsets, st.sizes, st.total_rows, st.n_cols), compressor=2)
    assert e.value.code == ob.OB_INVALID_DATA
    # a malformed stream under a correct checksum: the first match offset points before the block (decoder bounds)
    bad = st.image.copy()
    b = bad[st.offsets[3]:st.offsets[3] + st.sizes[3]]
    pay = b[hs:]
    tok = int(pay[0])
    lit = tok >> 4
    p = 1
    if lit == 15:
        while pay[p] == 255:
            lit += 255
            p += 1
        lit += int(pay[p])
        p += 1
    at = p + lit                                  # offset of the first match
    pay[at], pay[at + 1] = 0xff, 0xff             # 65535 > bytes produced so far
    b[48:56] = np.frombuffer(np.uint64(crc(np.ascontiguousarray(pay))).tobytes(), np.uint8)
    b[8:10] = 0
    b[8:10] = np.frombuffer(np.uint16(lz4_ref.header_checksum_fold(b)).tobytes(), np.uint8)
    assert lz4_ref.stored_checksums_ok(b, crc)
    with pytest.raises(lz4_ref.Lz4Error):
        lz4_ref.micro_block_decompress(b, 2)
    with pytest.raises(ob.ObGpuError) as e:
        ob.PageBatch(ctx, type(st)(bad, st.offsets, st.sizes, st.total_rows, st.n_cols), compressor=2)
    assert e.value.code == ob.OB_INVALID_DATA
    # afterwards a good open and scan still succeed
    plain, cb = ob.PageBatch(ctx, table), ob.PageBatch(ctx, st, compressor=2)
    scans_equal(plain, cb)
    cb.close()
    plain.close()
    ctx.close()


def test_string_pointers_address_the_device_image():
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import compress_table
    table, _ = _table(n=9000)
    st = compress_table(table, 2)
    ctx = ob.ScanContext(0)
    cb = ob.PageBatch(ctx, st, compressor=2)
    base, size = cb.device_image()
    assert base != 0 and size >= table.sizes.sum()
    r = cb.scan(ob.White(1, ob.WHITE_OP_LT, [10]), [3], string_base=base)
    ptrs, lens, _ = r.fetch_col(0)
    h, o = r.fetch_strings(0)
    class DeviceBytes:   # the batch's device image, gathered by torch through the CUDA array interface
        __cuda_array_interface__ = {"shape": (size,), "typestr": "|u1", "data": (base, False), "version": 3}
    dev = torch.as_tensor(DeviceBytes(), device="cuda").cpu().numpy()
    ptrs = ptrs.astype(np.uint64)
    rows = np.arange(len(ptrs))
    for k in rows[:: max(len(rows) // 500, 1)]:
        rel = int(ptrs[k]) - base
        assert 0 <= rel and rel + int(lens[k]) <= size
        assert dev[rel:rel + int(lens[k])].tobytes() == h[o[k]:o[k + 1]].tobytes()
    r.free()
    cb.close()
    ctx.close()
