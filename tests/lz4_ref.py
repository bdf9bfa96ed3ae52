"""Plain-Python checker for compressed micro-blocks: an LZ4 block decoder (lz4_Block_format.md) with exactly the acceptance
rules of the device decoder (oceanbase_b200/csrc/lz4_blocks.cuh), the stored-form micro-block decode the reference's
ObMacroBlockReader::decompress_data does, and the checksum check of a stored block. Independent of the product: it shares no
code with the writer's compressor or the device decoder.

Acceptance rules (a stream that breaks one is refused):
  - every read stays inside the input, every write inside the expected output;
  - match offset: 1 <= offset <= bytes produced so far (the format: "a 0 offset value denotes an invalid block");
  - end-of-block rules of the format: a sequence that is not the last leaves >= 12 output bytes and >= 8 input bytes after
    its literals, a match ends >= 5 bytes before the end of the output, >= 5 input bytes follow a match length;
  - the last sequence (literals only) ends exactly at the end of the input and the output is exactly the expected size.
"""
import numpy as np

MAGIC = 1005
COMPRESSOR_NONE, COMPRESSOR_LZ4, COMPRESSOR_LZ4_1_9_1 = 1, 2, 7


class Lz4Error(ValueError):
    pass


def _ext(src, ip):
    total = 0
    while True:
        if ip >= len(src):
            raise Lz4Error("length extension runs past the input")
        b = src[ip]
        ip += 1
        total += b
        if b != 255:
            return total, ip


def lz4_decompress(src, out_len: int) -> bytes:
    """LZ4 block -> exactly out_len bytes, or Lz4Error."""
    src = bytes(src)
    n_in = len(src)
    out = bytearray()
    ip = 0
    while True:
        if ip >= n_in:
            raise Lz4Error("no token")
        token = src[ip]
        ip += 1
        lit = token >> 4
        if lit == 15:
            e, ip = _ext(src, ip)
            lit += e
        op = len(out)
        if lit > n_in - ip or lit > out_len - op:
            raise Lz4Error("literal run past the input or the output")
        last = ip + lit == n_in
        if not last and (op + lit > out_len - 12 or ip + lit > n_in - 8):
            raise Lz4Error("end-of-block rule: a sequence ends too close to the end")
        out += src[ip:ip + lit]
        ip += lit
        if last:
            break
        offset = src[ip] | (src[ip + 1] << 8)
        ip += 2
        mlen = token & 15
        if mlen == 15:
            e, ip = _ext(src, ip)
            mlen += e
        mlen += 4
        if ip > n_in - 5:
            raise Lz4Error("end-of-block rule: too few input bytes after a match")
        op = len(out)
        if offset == 0 or offset > op:
            raise Lz4Error("match offset %d with %d bytes produced" % (offset, op))
        if mlen > out_len - 5 - op:
            raise Lz4Error("end-of-block rule: a match reaches into the last 5 bytes")
        start = op - offset
        if offset >= mlen:
            out += out[start:start + mlen]
        else:
            pat = bytes(out[start:op])
            out += (pat * (mlen // offset + 1))[:mlen]
    if len(out) != out_len:
        raise Lz4Error("decoded %d bytes, expected %d" % (len(out), out_len))
    return bytes(out)


def header_fields(block):
    b = np.asarray(block, dtype=np.uint8)
    hs = int(b[4:8].view(np.uint32)[0])
    length = int(b[40:44].view(np.int32)[0])
    zlength = int(b[44:48].view(np.int32)[0])
    return hs, length, zlength


def micro_block_decompress(block, compressor: int) -> np.ndarray:
    """A micro-block in stored form -> the decoded block (header unchanged), as ObMacroBlockReader::decompress_data."""
    b = np.ascontiguousarray(block, dtype=np.uint8)
    hs, length, zlength = header_fields(b)
    if int(b[0:2].view(np.uint16)[0]) != MAGIC or hs < 64 or hs + zlength != b.size:
        raise Lz4Error("bad micro-block header")
    if zlength == length:
        return b.copy()
    if compressor == COMPRESSOR_NONE:
        raise Lz4Error("compressed block in a NONE table")
    if compressor not in (COMPRESSOR_LZ4, COMPRESSOR_LZ4_1_9_1):
        raise NotImplementedError(compressor)
    payload = lz4_decompress(b[hs:].tobytes(), length)
    return np.concatenate([b[:hs], np.frombuffer(payload, dtype=np.uint8)])


def header_checksum_fold(block) -> int:
    """ObMicroBlockHeader::check_header_checksum: the 16-bit fold including the stored header_checksum_ (0 when valid)."""
    b = np.ascontiguousarray(block[:64], dtype=np.uint8)
    u16 = lambda o: int(b[o:o + 2].view(np.uint16)[0])
    u32 = lambda o: int(b[o:o + 4].view(np.uint32)[0])
    i32 = lambda o: int(b[o:o + 4].view(np.int32)[0])
    i64 = lambda o: int(b[o:o + 8].view(np.int64)[0])
    cs = u16(0) ^ u16(2) ^ u16(8) ^ int(b[20]) ^ int(b[21])

    def fold(v):
        v &= (1 << 64) - 1
        return (v ^ (v >> 16) ^ (v >> 32) ^ (v >> 48)) & 0xFFFF
    for v in (u16(10), u16(12), u16(14) & 1, u16(22), u32(4), u32(16), u32(24), i32(28), i64(32), i32(40), i32(44), i64(48)):
        cs ^= fold(v)
    return cs & 0xFFFF


def stored_checksums_ok(block, crc32c) -> bool:
    """Header checksum and payload checksum (crc32c of the STORED payload == data_checksum_) of a stored block;
    crc32c(bytes_array) -> int is the checker's crc (the oracle's ob_crc64_sse42)."""
    b = np.ascontiguousarray(block, dtype=np.uint8)
    hs, _, zlength = header_fields(b)
    if header_checksum_fold(b) != 0 or hs + zlength != b.size:
        return False
    return crc32c(b[hs:]) == int(b[48:56].view(np.uint64)[0])
