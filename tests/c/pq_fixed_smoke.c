/* Plain-C consumer of ag_parquet_bool_decode and ag_parquet_fixed_decode: two PLAIN BOOLEAN pages that share a byte of
 * the output bitmap, decoded in one batch around sentinel bits, and one BYTE_STREAM_SPLIT FIXED_LEN_BYTE_ARRAY(3) page
 * decoded spaced with slot 1 null.  Exit code 0 = checks passed on a GPU, 77 = no usable device (both calls are refused
 * with AG_ERR_CUDA). */
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "arrowgpu.h"

static int fail(const char* what, ag_status st) {
  char msg[256];
  ag_last_error(msg, sizeof msg);
  fprintf(stderr, "%s: status %d: %s\n", what, st, msg);
  return 1;
}

int main(void) {
  /* booleans: page 0 = 1,0,1,1,0 into bits 3..7; page 1 = 1,0,0,1 into bits 9..12; every other bit is a sentinel */
  const uint8_t bits[] = {0x0D, 0x09};
  const ag_pq_page bpages[2] = {{1, 1, 4, 9}, {0, 1, 5, 3}};
  uint8_t bitmap[2] = {0x00, 0xFF};
  int64_t bdec[2] = {0};
  ag_status st = ag_parquet_bool_decode(AG_PQ_ENC_PLAIN, bits, bpages, 2, NULL, bitmap, bdec);

  /* FIXED_LEN_BYTE_ARRAY(3) BYTE_STREAM_SPLIT: "abc", "def", "ghi" as three streams, into slots 0, 2, 3 */
  const uint8_t bss[] = {'a', 'd', 'g', 'b', 'e', 'h', 'c', 'f', 'i'};
  const ag_pq_page fpages[1] = {{0, 9, 4, 0}};
  const uint8_t valid[1] = {0x0D};
  uint8_t out[12];
  int64_t fdec[1] = {0}, bad = 0;
  memset(out, 0x5A, sizeof out);
  ag_status st2 = ag_parquet_fixed_decode(AG_PQ_TYPE_FIXED_LEN_BYTE_ARRAY, 3, AG_PQ_ENC_BYTE_STREAM_SPLIT, bss, fpages, 1, valid, NULL, 0,
                                          out, fdec, &bad);
  if (st == AG_ERR_CUDA || st2 == AG_ERR_CUDA) {
    if (st != AG_ERR_CUDA || st2 != AG_ERR_CUDA) { fprintf(stderr, "only one call was refused: %d %d\n", st, st2); return 1; }
    if (bitmap[0] != 0x00 || bitmap[1] != 0xFF || out[0] != 0x5A) { fprintf(stderr, "a refused call wrote its output\n"); return 1; }
    printf("no device: refused with AG_ERR_CUDA\n");
    return 77;
  }
  if (st != AG_OK) return fail("bool_decode", st);
  if (st2 != AG_OK) return fail("fixed_decode", st2);
  if (bitmap[0] != 0x68 || bitmap[1] != 0xF3) { fprintf(stderr, "bitmap %02x %02x\n", bitmap[0], bitmap[1]); return 1; }
  if (bdec[0] != 4 || bdec[1] != 5) { fprintf(stderr, "bool counts %lld %lld\n", (long long)bdec[0], (long long)bdec[1]); return 1; }
  if (memcmp(out, "abc\0\0\0defghi", 12) != 0 || fdec[0] != 4 || bad != AG_NO_ERROR_POS) {
    fprintf(stderr, "fixed output or count %lld wrong\n", (long long)fdec[0]);
    return 1;
  }
  printf("pq_fixed_smoke ok\n");
  return 0;
}
