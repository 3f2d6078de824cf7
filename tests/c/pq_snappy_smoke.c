/* Plain-C consumer of ag_parquet_snappy_decompress: two raw Snappy pages ("abc" then an overlapping copy-1 of offset 3;
 * a 10-byte literal then a copy-1 of offset 10) decompressed in one batch, given in the reverse order of their bytes.
 * Exit code 0 = checks passed on a GPU, 77 = no usable device (the call is refused with AG_ERR_CUDA). */
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "arrowgpu.h"

int main(void) {
  const uint8_t data[] = {12, 0x08, 'a', 'b', 'c', 0x15, 3,
                          20, 0x24, '0', '1', '2', '3', '4', '5', '6', '7', '8', '9', 0x19, 10};
  /* page 0: bytes 7..20 -> dst 12..31; page 1: bytes 0..6 -> dst 0..11 */
  const ag_pq_compressed pages[2] = {{7, 14, 12, 20}, {0, 7, 0, 12}};
  const char* want = "abcabcabcabc01234567890123456789";
  uint8_t out[40];
  int64_t written[2] = {0, 0};
  memset(out, 0xA5, sizeof out);
  ag_status st = ag_parquet_snappy_decompress(data, pages, 2, out, written);
  if (st == AG_ERR_CUDA) { printf("no device: refused with AG_ERR_CUDA\n"); return 77; }
  if (st != AG_OK) {
    char msg[256];
    ag_last_error(msg, sizeof msg);
    fprintf(stderr, "snappy_decompress: status %d: %s\n", st, msg);
    return 1;
  }
  if (memcmp(out, want, 32) != 0) { fprintf(stderr, "output %.32s\n", (const char*)out); return 1; }
  for (int i = 32; i < 40; ++i)
    if (out[i] != 0xA5) { fprintf(stderr, "byte %d past the output changed\n", i); return 1; }
  if (written[0] != 20 || written[1] != 12) { fprintf(stderr, "written %lld %lld\n", (long long)written[0], (long long)written[1]); return 1; }
  printf("pq_snappy_smoke ok\n");
  return 0;
}
