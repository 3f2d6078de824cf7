/* Plain-C consumer of ag_parquet_lz4_raw_decompress: two LZ4_RAW pages (one literal-only sequence "hello"; a sequence of
 * the literals "ab" and an overlapping 10-byte match at offset 2, then an empty final sequence) decompressed in one
 * batch, given in the reverse order of their bytes.  Exit code 0 = checks passed on a GPU, 77 = no usable device (the
 * call is refused with AG_ERR_CUDA). */
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "arrowgpu.h"

int main(void) {
  const uint8_t data[] = {0x50, 0x68, 0x65, 0x6c, 0x6c, 0x6f, 0x26, 0x61, 0x62, 0x02, 0x00, 0x00};
  /* page 0: bytes 6..11 -> dst 5..16; page 1: bytes 0..5 -> dst 0..4 */
  const ag_pq_compressed pages[2] = {{6, 6, 5, 12}, {0, 6, 0, 5}};
  const char* want = "helloabababababab";
  uint8_t out[24];
  int64_t written[2] = {0, 0};
  memset(out, 0xA5, sizeof out);
  ag_status st = ag_parquet_lz4_raw_decompress(data, pages, 2, out, written);
  if (st == AG_ERR_CUDA) { printf("no device: refused with AG_ERR_CUDA\n"); return 77; }
  if (st != AG_OK) {
    char msg[256];
    ag_last_error(msg, sizeof msg);
    fprintf(stderr, "lz4_raw_decompress: status %d: %s\n", st, msg);
    return 1;
  }
  if (memcmp(out, want, 17) != 0) { fprintf(stderr, "output %.17s\n", (const char*)out); return 1; }
  for (int i = 17; i < 24; ++i)
    if (out[i] != 0xA5) { fprintf(stderr, "byte %d past the output changed\n", i); return 1; }
  if (written[0] != 12 || written[1] != 5) { fprintf(stderr, "written %lld %lld\n", (long long)written[0], (long long)written[1]); return 1; }
  printf("pq_lz4_smoke ok\n");
  return 0;
}
