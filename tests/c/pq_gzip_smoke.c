/* Plain-C consumer of ag_parquet_gzip_decompress: two GZIP pages (a member with one stored block "hello"; a member with
 * one fixed-Huffman block of 12 'z', a literal and a copy) decompressed in one batch, given in the reverse order of their
 * bytes.  Exit code 0 = checks passed on a GPU, 77 = no usable device (the call is refused with AG_ERR_CUDA). */
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "arrowgpu.h"

int main(void) {
  const uint8_t data[] = {0x1f, 0x8b, 0x08, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0xff, 0x01, 0x05, 0x00, 0xfa,
                          0xff, 0x68, 0x65, 0x6c, 0x6c, 0x6f, 0x86, 0xa6, 0x10, 0x36, 0x05, 0x00, 0x00, 0x00,
                          0x1f, 0x8b, 0x08, 0x00, 0x00, 0x00, 0x00, 0x00, 0x02, 0x03, 0xab, 0xaa, 0x42, 0x00,
                          0x00, 0x43, 0x89, 0x74, 0x79, 0x0c, 0x00, 0x00, 0x00};
  /* page 0: bytes 28..50 -> dst 5..16; page 1: bytes 0..27 -> dst 0..4 */
  const ag_pq_compressed pages[2] = {{28, 23, 5, 12}, {0, 28, 0, 5}};
  const char* want = "hellozzzzzzzzzzzz";
  uint8_t out[24];
  int64_t written[2] = {0, 0};
  memset(out, 0xA5, sizeof out);
  ag_status st = ag_parquet_gzip_decompress(data, pages, 2, out, written);
  if (st == AG_ERR_CUDA) { printf("no device: refused with AG_ERR_CUDA\n"); return 77; }
  if (st != AG_OK) {
    char msg[256];
    ag_last_error(msg, sizeof msg);
    fprintf(stderr, "gzip_decompress: status %d: %s\n", st, msg);
    return 1;
  }
  if (memcmp(out, want, 17) != 0) { fprintf(stderr, "output %.17s\n", (const char*)out); return 1; }
  for (int i = 17; i < 24; ++i)
    if (out[i] != 0xA5) { fprintf(stderr, "byte %d past the output changed\n", i); return 1; }
  if (written[0] != 12 || written[1] != 5) { fprintf(stderr, "written %lld %lld\n", (long long)written[0], (long long)written[1]); return 1; }
  printf("pq_gzip_smoke ok\n");
  return 0;
}
