/* Plain-C consumer of ag_parquet_byte_array_decode: two PLAIN BYTE_ARRAY pages ("ab", "", "cde" and "xyz") decoded in one
 * batch, the second page first in the table, into int32 offsets with slot 1 null.  Exit code 0 = checks passed on a
 * GPU, 77 = no usable device (the call is refused with AG_ERR_CUDA). */
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "arrowgpu.h"

int main(void) {
  const uint8_t data[] = {3, 0, 0, 0, 'x', 'y', 'z',
                          2, 0, 0, 0, 'a', 'b', 3, 0, 0, 0, 'c', 'd', 'e'};
  /* page 0: bytes 7..19 -> slots 0..2 (slot 1 null); page 1: bytes 0..6 -> slot 3 */
  const ag_pq_page pages[2] = {{0, 7, 1, 3}, {7, 13, 3, 0}};
  const uint8_t valid[1] = {0x0D};
  const int32_t want_off[5] = {0, 2, 2, 5, 8};
  int32_t offsets[5] = {0};
  uint8_t out[16];
  int64_t total = -1, decoded[2] = {0}, bad = 0;
  memset(out, 0, sizeof out);
  ag_status st = ag_parquet_byte_array_decode(AG_PQ_ENC_PLAIN, 4, data, pages, 2, 4, valid, NULL, NULL, 0, 0, offsets, out,
                                              sizeof out, &total, decoded, &bad);
  if (st == AG_ERR_CUDA) { printf("no device: refused with AG_ERR_CUDA\n"); return 77; }
  if (st != AG_OK) {
    char msg[256];
    ag_last_error(msg, sizeof msg);
    fprintf(stderr, "byte_array_decode: status %d: %s\n", st, msg);
    return 1;
  }
  for (int i = 0; i < 5; ++i)
    if (offsets[i] != want_off[i]) { fprintf(stderr, "offset %d: %d != %d\n", i, offsets[i], want_off[i]); return 1; }
  if (total != 8 || memcmp(out, "abcdexyz", 8) != 0) { fprintf(stderr, "data or total %lld wrong\n", (long long)total); return 1; }
  if (decoded[0] != 1 || decoded[1] != 3) { fprintf(stderr, "counts %lld %lld\n", (long long)decoded[0], (long long)decoded[1]); return 1; }
  printf("pq_bytearray_smoke ok\n");
  return 0;
}
