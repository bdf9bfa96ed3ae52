"""zstd-compressed micro-blocks (compressor 6, zstd_1.3.8) on the CPU side: the committed libzstd vectors are self-consistent and
their feature census covers every decoder branch; when the system libzstd loads, it reproduces the recorded verdicts, decodes
the writer's frames and the stored-form tables written with compressor 6 (mostly compressed, checksums valid, decoded blocks
equal to the source blocks, oracle scans unchanged); compressor-6 macro blocks parse and walk in the oracle."""
import ctypes as C
import hashlib
import os
import sys

import numpy as np
import pytest

import lz4_ref
import oracle_binding as ora
from test_lz4_blocks import compressible_tables, crc32c, oracle_scan

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_zstd_golden as golden  # noqa: E402

ZSTD = 6


def zstd():
    z = golden.libzstd()
    return golden.Zstd(z) if z is not None else None


def vectors():
    """(frames [(frame, payload)], malformed [(stream, payload length, libzstd accepts, sha256 of its output, strict reason)],
    census (frames x features), census names)."""
    z = np.load(os.path.join(HERE, "golden", "zstd_vectors.npz"))
    po, fo, bo = z["payload_off"], z["frame_off"], z["bad_off"]
    pay = lambda i: z["payloads"][po[i]:po[i + 1]].tobytes()
    frames = [(z["frames"][fo[k]:fo[k + 1]].tobytes(), pay(i)) for k, i in enumerate(z["frame_payload"])]
    names = [str(s) for s in z["strict_names"]]
    bad = [(z["bad"][bo[k]:bo[k + 1]].tobytes(), len(pay(i)), bool(z["bad_libzstd_ok"][k]), z["bad_libzstd_sha256"][k].tobytes(),
            names[int(z["bad_strict"][k])]) for k, i in enumerate(z["bad_payload"])]
    return frames, bad, z["census"], [str(s) for s in z["census_names"]]


def test_vectors_are_self_consistent_and_cover_every_branch():
    frames, bad, census, names = vectors()
    assert len(frames) >= 150 and len(bad) >= 500 and census.shape == (len(frames), len(names))
    assert names == golden.CENSUS
    for k, (fr, _) in enumerate(frames):   # the recorded census is the walker's
        assert {names[j] for j in np.nonzero(census[k])[0]} == golden.walk(fr)[0]
    missing = [n for j, n in enumerate(names) if not census[:, j].any()]
    assert not missing, missing
    strict = {s for *_, s in bad}
    assert strict <= set(golden.STRICT) and {"trailing_frame", "skippable_frame", "modes_reserved"} <= strict
    zs = zstd()
    if zs is None:
        pytest.skip("libzstd.so.1 not present: verdicts not re-checked")
    for fr, p in frames:
        assert zs.decompress(fr, len(p)) == p
    for s, n, ok, digest, _ in bad:
        out = zs.decompress(s, n)
        assert (out is not None) == ok
        if ok:
            assert hashlib.sha256(out).digest() == digest


def test_writer_frames_decode_with_libzstd():
    from oceanbase_b200.sstable import zstd_compress
    zs = zstd()
    if zs is None:
        pytest.skip("libzstd.so.1 not present")
    frames, _, _, _ = vectors()
    rng = np.random.default_rng(5)
    pays = sorted({p for _, p in frames}, key=len)
    pays += [rng.integers(0, 4, size=n, dtype=np.uint8).tobytes() for n in (1, 12, 13, 100, 4097, 131072, 131073, 300_001)]
    for p in pays:
        z = zstd_compress(p).tobytes()
        assert len(z) <= len(p) + 3 * (len(p) // (128 << 10) + 1) + 13
        assert zs.decompress(z, len(p)) == p, len(p)
        feats = golden.walk(z)[0]
        assert "checksum" not in feats and "single_segment" in feats
        assert feats <= {"single_segment", "fcs1", "fcs2", "fcs4", "block_raw", "block_compressed", "multi_block", "lit_raw",
                         "no_sequences", "ll_predefined", "of_predefined", "ml_predefined"}


def test_compress_table_zstd_decodes_to_the_source_blocks():
    from oceanbase_b200.sstable import TableImage, compress_table
    zs = zstd()
    for name, table, proj in compressible_tables():
        st = compress_table(table, ZSTD)
        hdr = [lz4_ref.header_fields(st.block(i)) for i in range(st.n_blocks)]
        n_comp = sum(1 for _, ln, zl in hdr if zl < ln)
        assert n_comp >= 0.9 * st.n_blocks, (name, n_comp, st.n_blocks)
        if zs is None:
            pytest.skip("libzstd.so.1 not present: stored blocks not decoded")
        dec = []
        for i in range(st.n_blocks):
            blk = st.block(i)
            assert lz4_ref.stored_checksums_ok(blk, crc32c), (name, i)
            hs, ln, zl = hdr[i]
            src = table.block(i)
            d = blk.copy() if zl == ln else np.concatenate([blk[:hs], np.frombuffer(zs.decompress(blk[hs:].tobytes(), ln), np.uint8)])
            # the decoded copy keeps the stored header: only header_checksum_, data_zlength_ and data_checksum_ differ
            assert np.array_equal(d[64:], src[64:]) and np.array_equal(d[:8], src[:8]) and np.array_equal(d[10:44], src[10:44]), (name, i)
            assert np.array_equal(d[56:64], src[56:64]), (name, i)
            dec.append(d)
        offs = np.concatenate([[0], np.cumsum([len(d) for d in dec])[:-1]]).astype(np.int64)
        decoded = TableImage(np.concatenate(dec), offs, np.array([len(d) for d in dec], dtype=np.int64), table.total_rows, table.n_cols)
        w1, w2 = oracle_scan(table, proj), oracle_scan(decoded, proj)
        assert w1["selected"] == w2["selected"] > 0 and np.array_equal(w1["row_ids"], w2["row_ids"])
        assert np.array_equal(w1["sel_offset"], w2["sel_offset"])
        for c in range(len(proj)):
            if w1["lens"][c] is not None:
                assert np.array_equal(w1["lens"][c], w2["lens"][c])
            else:
                assert np.array_equal(w1["data"][c], w2["data"][c])
            assert np.array_equal(w1["nulls"][c], w2["nulls"][c])


def test_zstd_macro_blocks_parse_and_walk_in_the_oracle():
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import build_macro_blocks, compress_table
    _, table, _ = compressible_tables()[0]
    types = [capi.OBJ_INT, capi.OBJ_INT, capi.OBJ_VARCHAR, capi.OBJ_INT, capi.OBJ_INT, capi.OBJ_INT, capi.OBJ_VARCHAR, capi.OBJ_VARCHAR]
    ms = 64 << 10
    mi = build_macro_blocks(table, types, 1, macro_block_size=ms, compressor=capi.COMPRESSOR_ZSTD_1_3_8)
    stored = compress_table(table, ZSTD)
    O = ora.oracle()
    O.ora_macro_block_micro_blocks.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_int32]
    O.ora_macro_block_parse.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32]
    k = 0
    for m in range(mi.n_macro):
        blk = np.ascontiguousarray(mi.image[m * ms:(m + 1) * ms])
        f = np.zeros(28, dtype=np.int64)
        assert O.ora_macro_block_parse(blk.ctypes.data, blk.size, f.ctypes.data, 1) == 0
        assert f[25] == ZSTD
        offs, szs, cnt = np.zeros(4096, dtype=np.int64), np.zeros(4096, dtype=np.int64), C.c_int32(0)
        assert O.ora_macro_block_micro_blocks(blk.ctypes.data, blk.size, offs.ctypes.data, szs.ctypes.data, 4096, C.byref(cnt), 1) == 0
        for j in range(cnt.value):
            assert np.array_equal(blk[offs[j]:offs[j] + szs[j]], stored.block(k))
            k += 1
    assert k == table.n_blocks


def test_writer_refuses_compressed_blocks_with_zstd():
    from oceanbase_b200 import capi
    from oceanbase_b200.capi import lib
    from oceanbase_b200.sstable import compress_table
    _, table, _ = compressible_tables()[1]
    st = compress_table(table, ZSTD)
    off, sz = st.offsets.copy(), st.sizes.copy()
    o = np.zeros(st.image.size * 2, dtype=np.uint8)
    oo, osz, used = np.zeros(st.n_blocks, np.int64), np.zeros(st.n_blocks, np.int64), C.c_int64(0)
    assert lib.obgpu_writer_compress_blocks(st.image.ctypes.data, off.ctypes.data, sz.ctypes.data, st.n_blocks, ZSTD, 1,
                                            o.ctypes.data, o.size, oo.ctypes.data, osz.ctypes.data, C.byref(used)) == capi.OB_INVALID_DATA
