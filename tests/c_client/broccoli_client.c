/* Splices brotli files with the Broccoli C ABI (include/broccoli.h) through 3-byte input and output buffers, the way the
 * reference's c/catbrotli.c drives it.  Usage: broccoli_client OUT IN...  Exit status: 0, or the failing BroccoliResult. */
#include <stdio.h>
#include <string.h>

#include "broccoli.h"

static int drain(FILE* out, const uint8_t* buf, size_t n) { return fwrite(buf, 1, n, out) == n ? 0 : 1; }

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  FILE* out = fopen(argv[1], "wb");
  if (!out) return 2;
  BroccoliState state = BroccoliCreateInstance();
  uint8_t ibuf[3], obuf[3];
  for (int f = 2; f < argc; ++f) {
    FILE* in = fopen(argv[f], "rb");
    if (!in) return 2;
    BroccoliNewBrotliFile(&state);
    size_t got;
    while ((got = fread(ibuf, 1, sizeof(ibuf), in)) > 0) {
      const uint8_t* next_in = ibuf;
      size_t avail_in = got;
      for (;;) {
        uint8_t* next_out = obuf;
        size_t avail_out = sizeof(obuf);
        BroccoliResult r = BroccoliConcatStream(&state, &avail_in, &next_in, &avail_out, &next_out);
        if (drain(out, obuf, sizeof(obuf) - avail_out)) return 2;
        if (r == BroccoliNeedsMoreOutput) continue;
        if (r == BroccoliNeedsMoreInput) break;
        fprintf(stderr, "%s: %d\n", argv[f], (int)r);
        return (int)r;
      }
    }
    fclose(in);
  }
  for (;;) {
    size_t avail_out = sizeof(obuf);
    BroccoliResult r = BroccoliConcatFinished(&state, &avail_out, obuf);
    if (drain(out, obuf, sizeof(obuf) - avail_out)) return 2;
    if (r == BroccoliSuccess) break;
    if (r != BroccoliNeedsMoreOutput) return (int)r;
  }
  BroccoliDestroyInstance(state);
  return fclose(out) == 0 ? 0 : 2;
}
