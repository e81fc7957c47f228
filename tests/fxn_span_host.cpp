// Host-side checks of span_copy (csrc/mplx_span.cuh), run by tests/test_fxn_span_cpu.py (no device needed):
// for the element sizes of the staged outputs (112-byte records, 8-byte keys and costs, 4-byte actions), every
// base offset inside a line and every CTA span length up to 256 slots, against a literal byte-by-byte
// statement — the five parts cover every byte of the span exactly once and in order, the bulk parts start and
// end on 16-byte boundaries, the body starts on a 128-byte line and is whole lines, the head does not cross a
// line, and lead and trail are shorter than 16 bytes unless the span holds no 16-byte aligned range at all.
#include <cstdio>
#include <vector>

#define __host__
#define __device__
#include "../motion_primitive_library_b200/csrc/mplx_span.cuh"

static int fails = 0;
#define CHECK(c)                                              \
  do {                                                        \
    if (!(c)) {                                               \
      std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); \
      fails++;                                                \
    }                                                         \
  } while (0)

int main() {
  long spans = 0;
  const unsigned elems[3] = {112, 8, 4};
  for (unsigned elem : elems) {
    const unsigned step = elem == 4 ? 4 : 8;
    for (unsigned off = 0; off < 128; off += step) {
      // a few line-aligned bases far from 0, so that the address arithmetic is 64-bit
      for (uint64_t line : {(uint64_t)0, (uint64_t)1 << 12, (uint64_t)0x7f12345600ull}) {
        const uint64_t base = line * 128 + off;
        for (unsigned n = 1; n <= 256; n++, spans++) {
          const mplx::SpanCopy c = mplx::span_copy(base, elem, n);
          const unsigned bytes = elem * n;
          const unsigned part[5] = {c.lead, c.head, c.body, c.tail, c.trail};
          // literal statement: byte i of the span belongs to exactly one part, the parts in order
          std::vector<int> owner(bytes, -1);
          unsigned at = 0;
          for (int p = 0; p < 5; p++)
            for (unsigned k = 0; k < part[p]; k++, at++)
              if (at < bytes) {
                CHECK(owner[at] == -1);
                owner[at] = p;
              }
          CHECK(at == bytes);
          for (unsigned i = 0; i < bytes; i++) CHECK(owner[i] >= 0);
          const uint64_t head0 = base + c.lead, body0 = head0 + c.head, tail0 = body0 + c.body, trail0 = tail0 + c.tail;
          const bool bulk = c.head + c.body + c.tail > 0;
          if (bulk) {
            CHECK(head0 % 16 == 0 && trail0 % 16 == 0);
            CHECK(c.head % 16 == 0 && c.tail % 16 == 0 && c.body % 128 == 0);
            CHECK(c.lead < 16 && c.trail < 16);
            CHECK(c.head > 0 || c.body > 0);
            if (c.body) CHECK(body0 % 128 == 0 && c.head < 128 && c.tail < 128);
            // the head stays inside one line unless there is no whole line at all
            if (c.body) CHECK(c.head == 0 || (head0 / 128) == ((body0 - 1) / 128));
            else CHECK(c.tail == 0 && (base + 127) / 128 * 128 + 128 > base + bytes);  // no whole line in the span
          } else {
            // no 16-byte aligned range inside the span: all of it is stored plainly
            CHECK(c.lead == bytes && (base + 15) / 16 * 16 >= (base + bytes) / 16 * 16);
          }
          // every whole 16-byte granule of the span is covered by a bulk part
          for (uint64_t g = (base + 15) / 16 * 16; g + 16 <= base + bytes; g += 16) CHECK(g >= head0 && g + 16 <= trail0);
          // the stored edges are whole elements when elem divides 16 and the base is aligned to it
          if (16 % elem == 0) CHECK(c.lead % elem == 0 && c.trail % elem == 0);
        }
      }
    }
  }
  std::printf("fxn span: %ld spans checked\n", spans);
  std::printf("fxn_span_host fails %d\n", fails);
  return fails ? 1 : 0;
}
