/* Plain-C consumer of ag_parquet_delta_decode: two DELTA_BINARY_PACKED INT64 pages (the reference's encoder output
 * for 1..5 and for 7,5,3,1,2,3,4,5), decoded in one batch whose validity bitmap marks two slots of the second page
 * null.  Exit code 0 =
 * checks passed on a GPU, 77 = no usable device (the call is refused with AG_ERR_CUDA). */
#include <stdint.h>
#include <stdio.h>

#include "arrowgpu.h"

int main(void) {
  const uint8_t data[] = {128, 1, 4, 5, 2, 2, 0, 0, 0, 0,
                          128, 1, 4, 8, 14, 3, 2, 0, 0, 0, 192, 63, 0, 0, 0, 0, 0, 0};
  /* page 0: bytes 10..27 -> slots 5..14 (10 slots, 8 valid); page 1: bytes 0..9 -> slots 0..4 */
  const ag_pq_page pages[2] = {{10, 18, 10, 5}, {0, 10, 5, 0}};
  const uint8_t valid[2] = {0xBF, 0xFE}; /* every slot valid except 6 and 8 */
  const int64_t want[15] = {1, 2, 3, 4, 5, 7, 0, 5, 0, 3, 1, 2, 3, 4, 5};
  int64_t out[16] = {0}, decoded[2] = {0};
  ag_status st = ag_parquet_delta_decode(8, data, pages, 2, valid, out, decoded);
  if (st == AG_ERR_CUDA) { printf("no device: refused with AG_ERR_CUDA\n"); return 77; }
  if (st != AG_OK) {
    char msg[256];
    ag_last_error(msg, sizeof msg);
    fprintf(stderr, "delta_decode: status %d: %s\n", st, msg);
    return 1;
  }
  for (int i = 0; i < 15; ++i)
    if (out[i] != want[i]) { fprintf(stderr, "slot %d: %lld != %lld\n", i, (long long)out[i], (long long)want[i]); return 1; }
  if (decoded[0] != 10 || decoded[1] != 5) { fprintf(stderr, "counts %lld %lld\n", (long long)decoded[0], (long long)decoded[1]); return 1; }
  printf("pq_delta_smoke ok\n");
  return 0;
}
