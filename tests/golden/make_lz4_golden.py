"""Writes tests/golden/lz4_vectors.npz: LZ4 block-format known answers produced by the system liblz4 (liblz4.so.1, loaded with
ctypes; 1.9.4 when the vectors were made). Every payload is compressed with LZ4_compress_default, LZ4_compress_fast at
acceleration 1, 8 and 64, and LZ4_compress_HC (level 9); payloads above 16 KiB with LZ4_compress_default only. The payloads cover literal-only blocks (1..12 bytes), all-zero,
random and text data, repeats at offsets 1, 2, 3, 31, 32, 33, 4096 and 65535, and literal and match lengths around the
15-nibble boundary (14, 15, 16), the first 255 extension boundary (269, 270, 271) and ~70 000.

  python tests/golden/make_lz4_golden.py
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
KINDS = ["default", "fast1", "fast8", "fast64", "hc9"]


def payloads():
    rng = np.random.default_rng(20261015)
    rnd = lambda n: rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()
    out = [rnd(n) for n in range(1, 13)]                                        # literals only
    out += [bytes(1000), bytes(70_000), rnd(2000)]
    words = [b"micro", b"block", b"header", b"column", b"scan", b"offset", b"the", b"of", b"lz4", b"sstable"]
    out.append(b" ".join(words[i] for i in rng.integers(0, len(words), size=4000)))   # text
    for d in (1, 2, 3, 31, 32, 33, 4096):                                      # repeats at distance d
        pat = rnd(d)
        out.append(rnd(20) + pat * (3 + 600 // d) + rnd(20))
    head = rnd(65535)
    out.append(head + head[:1000] + rnd(20))                                   # offset 65535
    for lit in (14, 15, 16, 269, 270, 271, 70_000):                            # literal run of length ~lit, then a match
        seed = rnd(16)
        out.append(seed + rnd(lit) + seed * 4 + rnd(8))
    for m in (14, 15, 16, 269, 270, 271, 70_000):                              # match of length ~m
        base = rnd(100)
        rep = (base * (m // 100 + 1))[:m]
        out.append(base + rep + rnd(24))
    return out


def main():
    lz = C.CDLL("liblz4.so.1")
    lz.LZ4_compressBound.argtypes = [C.c_int]
    for f in ("LZ4_compress_default",):
        getattr(lz, f).argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int]
    lz.LZ4_compress_fast.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    lz.LZ4_compress_HC.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    lz.LZ4_versionString.restype = C.c_char_p
    pays = payloads()
    streams, p_idx, kind = [], [], []
    for i, p in enumerate(pays):
        cap = lz.LZ4_compressBound(len(p))
        for k, name in enumerate(KINDS):
            if len(p) > 16384 and name != "default":   # long payloads: one stream each keeps the file small
                continue
            buf = C.create_string_buffer(cap)
            if name == "default":
                n = lz.LZ4_compress_default(p, buf, len(p), cap)
            elif name.startswith("fast"):
                n = lz.LZ4_compress_fast(p, buf, len(p), cap, int(name[4:]))
            else:
                n = lz.LZ4_compress_HC(p, buf, len(p), cap, 9)
            assert n > 0, (i, name)
            streams.append(buf.raw[:n])
            p_idx.append(i)
            kind.append(k)
    cat = lambda bs: (np.frombuffer(b"".join(bs), dtype=np.uint8),
                      np.concatenate([[0], np.cumsum([len(b) for b in bs])]).astype(np.int64))
    pay, pay_off = cat(pays)
    st, st_off = cat(streams)
    np.savez_compressed(os.path.join(HERE, "lz4_vectors.npz"), payloads=pay, payload_off=pay_off, streams=st, stream_off=st_off,
                        payload_index=np.array(p_idx, dtype=np.int32), kind=np.array(kind, dtype=np.int32),
                        kinds=np.array(KINDS), lz4_version=np.array(lz.LZ4_versionString().decode()))
    print(f"{len(pays)} payloads, {len(streams)} streams, liblz4 {lz.LZ4_versionString().decode()}")


if __name__ == "__main__":
    main()
