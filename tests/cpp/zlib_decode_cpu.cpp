// zlibd::decode_stream (oceanbase_b200/csrc/zlib_decode.cuh) built for the CPU with one lane.
// stdin : records [int64 n_in][int64 n_out][n_in stream bytes]
// stdout: per record [int32 status][n_out output bytes, only when status == 0]
// Every stream is copied to a buffer of exactly n_in bytes and decoded into one of exactly n_out bytes, so a read or write
// outside them is caught by AddressSanitizer.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../oceanbase_b200/csrc/zlib_decode.cuh"

int main() {
  static zlibd::Work w;
  int64_t hdr[2];
  while (fread(hdr, 8, 2, stdin) == 2) {
    const int64_t n_in = hdr[0], n_out = hdr[1];
    uint8_t *in = (uint8_t *)malloc((size_t)(n_in > 0 ? n_in : 1)), *out = (uint8_t *)malloc((size_t)(n_out > 0 ? n_out : 1));
    if (!in || !out || (n_in > 0 && fread(in, 1, (size_t)n_in, stdin) != (size_t)n_in)) return 2;
    memset(&w, 0xa5, sizeof(w));   // no state carries over from the previous stream
    const int32_t st = zlibd::decode_stream(in, n_in, out, n_out, w, 0, 1);
    fwrite(&st, 4, 1, stdout);
    if (st == zlibd::kOk && n_out > 0) fwrite(out, 1, (size_t)n_out, stdout);
    free(in);
    free(out);
  }
  return 0;
}
