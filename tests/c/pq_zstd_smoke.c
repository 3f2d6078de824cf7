/* Plain-C consumer of ag_parquet_zstd_decompress: two ZSTD pages (a frame with one raw zstd block "hello"; a frame with
 * one RLE zstd block of 12 'z') decompressed in one batch, given in the reverse order of their bytes.
 * Exit code 0 = checks passed on a GPU, 77 = no usable device (the call is refused with AG_ERR_CUDA). */
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "arrowgpu.h"

int main(void) {
  const uint8_t data[] = {0x28, 0xb5, 0x2f, 0xfd, 0x20, 5, 0x29, 0, 0, 'h', 'e', 'l', 'l', 'o',
                          0x28, 0xb5, 0x2f, 0xfd, 0x20, 12, 0x63, 0, 0, 'z'};
  /* page 0: bytes 14..23 -> dst 5..16; page 1: bytes 0..13 -> dst 0..4 */
  const ag_pq_compressed pages[2] = {{14, 10, 5, 12}, {0, 14, 0, 5}};
  const char* want = "hellozzzzzzzzzzzz";
  uint8_t out[24];
  int64_t written[2] = {0, 0};
  memset(out, 0xA5, sizeof out);
  ag_status st = ag_parquet_zstd_decompress(data, pages, 2, out, written);
  if (st == AG_ERR_CUDA) { printf("no device: refused with AG_ERR_CUDA\n"); return 77; }
  if (st != AG_OK) {
    char msg[256];
    ag_last_error(msg, sizeof msg);
    fprintf(stderr, "zstd_decompress: status %d: %s\n", st, msg);
    return 1;
  }
  if (memcmp(out, want, 17) != 0) { fprintf(stderr, "output %.17s\n", (const char*)out); return 1; }
  for (int i = 17; i < 24; ++i)
    if (out[i] != 0xA5) { fprintf(stderr, "byte %d past the output changed\n", i); return 1; }
  if (written[0] != 12 || written[1] != 5) { fprintf(stderr, "written %lld %lld\n", (long long)written[0], (long long)written[1]); return 1; }
  printf("pq_zstd_smoke ok\n");
  return 0;
}
