/* Plain-C consumer of the Parquet page decode entry points: a two-page batch of dictionary indices (one repeated run,
 * one literal run) decoded through ag_parquet_dict_decode.  Exit code 0 = checks passed on a GPU, 77 = no usable
 * device (the call is refused with AG_ERR_CUDA). */
#include <stdint.h>
#include <stdio.h>

#include "arrowgpu.h"

int main(void) {
  /* page 0: bit width 2, repeated run of 5 x index 3; page 1: bit width 2, literal run 0,1,2,3,0,1,2,3 */
  const uint8_t data[] = {2, 10, 3, 2, 3, 0xE4, 0xE4};
  const ag_pq_page pages[2] = {{3, 4, 8, 0}, {0, 3, 5, 8}};
  const int64_t dict[4] = {10, 20, 30, 40};
  const int64_t want[13] = {10, 20, 30, 40, 10, 20, 30, 40, 40, 40, 40, 40, 40};
  int64_t out[13] = {0}, decoded[2] = {0}, bad = 0;
  /* pages[0] describes bytes 3..6 (literal), pages[1] bytes 0..2 (repeated): out of order on purpose */
  ag_status st = ag_parquet_dict_decode(8, dict, 4, data, pages, 2, NULL, out, decoded, &bad);
  if (st == AG_ERR_CUDA) { printf("no device: refused with AG_ERR_CUDA\n"); return 77; }
  if (st != AG_OK) {
    char msg[256];
    ag_last_error(msg, sizeof msg);
    fprintf(stderr, "dict_decode: status %d: %s\n", st, msg);
    return 1;
  }
  for (int i = 0; i < 13; ++i)
    if (out[i] != want[i]) { fprintf(stderr, "slot %d: %lld != %lld\n", i, (long long)out[i], (long long)want[i]); return 1; }
  if (decoded[0] != 8 || decoded[1] != 5 || bad != AG_NO_ERROR_POS) { fprintf(stderr, "counts\n"); return 1; }
  printf("pq_smoke ok\n");
  return 0;
}
