// mplx_span.cuh — how a CTA's slice of an output array leaves shared memory (expand_fxn_kernel).
// A CTA's successor slots are one contiguous span, [node0·nU, (node0+npb)·nU), in every output array.  The
// bulk-copy engine (cp.async.bulk) needs 16-byte aligned addresses and sizes, so the span splits into
//   lead   the bytes before the first 16-byte boundary        (plain stores)
//   head   from there to the first 128-byte line               (one bulk copy)
//   body   whole 128-byte lines                                (one bulk copy)
//   tail   from the last line boundary to the last 16-byte one (one bulk copy)
//   trail  the bytes after that                                (plain stores)
// in this order, summing to the span.  A span too short to hold a 16-byte boundary pair is all lead; one
// without a whole line is lead + head + trail.  tests/fxn_span_host.cpp checks it byte by byte.
#pragma once
#include <stdint.h>

namespace mplx {

struct SpanCopy {
  unsigned lead, head, body, tail, trail;  // bytes
};

// n elements of elem bytes starting at address base
__host__ __device__ inline SpanCopy span_copy(uint64_t base, unsigned elem, unsigned n) {
  const unsigned bytes = elem * n;
  const uint64_t end = base + bytes;
  const uint64_t a = (base + 15) & ~(uint64_t)15, b = end & ~(uint64_t)15;
  SpanCopy c = {bytes, 0u, 0u, 0u, 0u};
  if (a >= b) return c;
  const uint64_t l = (base + 127) & ~(uint64_t)127, r = end & ~(uint64_t)127;
  c.lead = (unsigned)(a - base);
  c.trail = (unsigned)(end - b);
  if (l >= r) {
    c.head = (unsigned)(b - a);
  } else {
    c.head = (unsigned)(l - a);
    c.body = (unsigned)(r - l);
    c.tail = (unsigned)(b - r);
  }
  return c;
}

}  // namespace mplx
