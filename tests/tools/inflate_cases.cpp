/* Runs the host build of mashmap_b200/csrc/mm_inflate.h over a file of cases, each in buffers of exactly its sizes, so
 * that a sanitizer build reports any read or write outside them (tests/test_bgzf_cpu.py). A case is
 * [u32 comp_len][u32 out_len][comp_len bytes]; one line per case goes to stdout: "<mmi_status> <crc32 or 0>". */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <vector>

#include "mm_inflate.h"

int main(int argc, char **argv)
{
  if (argc != 2) return 2;
  FILE *f = fopen(argv[1], "rb");
  if (!f) return 2;
  uint32_t tab[256];
  mmi_crc_table(tab, 0, 1);
  std::unique_ptr<mmi_tables> t(new mmi_tables());
  uint32_t hdr[2];
  while (fread(hdr, 4, 2, f) == 2) {
    uint8_t *comp = (uint8_t *)malloc(hdr[0] ? hdr[0] : 1), *out = (uint8_t *)malloc(hdr[1] ? hdr[1] : 1);
    if (hdr[0] && fread(comp, 1, hdr[0], f) != hdr[0]) return 2;
    const int rc = mmi_inflate(comp, hdr[0], out, hdr[1], *t, 0, 1);
    const uint32_t crc = rc == MMI_OK ? mmi_crc_finish(mmi_crc_share(tab, out, hdr[1], 0, 1), hdr[1]) : 0;
    printf("%d %u\n", rc, crc);
    free(comp);
    free(out);
  }
  fclose(f);
  return 0;
}
