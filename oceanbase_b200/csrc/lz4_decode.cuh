// One LZ4 block (the plain block format of ObCompressorType 2 "lz4_1.0" and 7 "lz4_1.9.1", what LZ4_decompress_safe takes
// apart into data_length_ bytes) -> exactly n_out bytes, by one warp: the LZ4 counterpart of zstd_decode.cuh.
//   every lane reads the token; length extensions are read 32 bytes at a time and the first byte != 255 found with a ballot;
//   literals move 32 bytes per step; a match at distance d is fully parallel even when it overlaps,
//   out[pos + i] = out[pos - d + (i mod d)], because every source byte precedes pos. The output goes straight to global memory
//   (matches read it back through L1).
// Refused (false): a read past n_in, a write past n_out, an offset outside 1..bytes produced, a break of the format's
// end-of-block rules (a sequence that is not the last leaves >= 12 output and >= 8 input bytes after its literals, a match ends
// >= 5 bytes before the end, >= 5 input bytes follow a match length), a last sequence that does not end exactly at n_in,
// output != n_out.
#pragma once

namespace lz4d {

// LZ4 length extension at in[ip]: bytes of 255 continue it. false: it runs past the input.
__device__ __forceinline__ bool read_ext(const uint8_t *in, int64_t n_in, int64_t &ip, int64_t &len, int lane) {
  for (;;) {
    const int64_t p = ip + lane;
    const bool valid = p < n_in;
    const uint32_t v = valid ? __ldg(in + p) : 0u;
    const unsigned stop = __ballot_sync(0xffffffffu, !valid || v != 255u);
    if (stop == 0u) {
      ip += 32;
      len += 255 * 32;
      continue;
    }
    const int f = __ffs(stop) - 1;
    if (ip + f >= n_in) return false;
    len += 255 * (int64_t)f + __shfl_sync(0xffffffffu, v, f);
    ip += f + 1;
    return true;
  }
}

// One LZ4 block in[0, n_in) -> out[0, n_out) by the warp; true only when the stream decodes to exactly n_out bytes.
__device__ __forceinline__ bool warp_lz4_decode(const uint8_t *in, int64_t n_in, uint8_t *out, int64_t n_out, int lane) {
  int64_t ip = 0, op = 0;
  for (;;) {
    if (ip >= n_in) return false;
    const uint32_t token = __ldg(in + ip);
    ++ip;
    int64_t lit = token >> 4;
    if (lit == 15 && !read_ext(in, n_in, ip, lit, lane)) return false;
    if (lit > n_in - ip || lit > n_out - op) return false;
    const bool last = ip + lit == n_in;
    if (!last && (op + lit > n_out - 12 || ip + lit > n_in - 8)) return false;
    for (int64_t i = lane; i < lit; i += 32) out[op + i] = __ldg(in + ip + i);
    ip += lit;
    op += lit;
    if (last) break;
    const int64_t offset = (int64_t)__ldg(in + ip) | ((int64_t)__ldg(in + ip + 1) << 8);
    ip += 2;
    int64_t mlen = token & 15u;
    if (mlen == 15 && !read_ext(in, n_in, ip, mlen, lane)) return false;
    mlen += 4;
    if (ip > n_in - 5) return false;
    if (offset == 0 || offset > op || mlen > n_out - 5 - op) return false;
    __syncwarp();   // the literals (and earlier matches) written by other lanes are visible
    const uint8_t *src = out + op - offset;
    for (int64_t i = lane; i < mlen; i += 32) out[op + i] = src[i < offset ? (uint32_t)i : (uint32_t)i % (uint32_t)offset];   // offset < 2^16, mlen < 2^31
    __syncwarp();
    op += mlen;
  }
  return op == n_out;
}

}  // namespace lz4d
