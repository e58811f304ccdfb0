// Device side of PgGradRS (launch.h): where does an element of the local flat gradient buffer live after the
// data-parallel reduce-scatter, and the red.global.add that puts a contribution there (local L2 atomics for the
// owned slice, NVLink peer atomics for the others — fire-and-forget, nothing waits for them inside the kernel).
#pragma once
#include "launch.h"
#include "ptx.cuh"

namespace pg {

// owner slice of element `off` (relative to g.start), clamped to [0, world): compares instead of a 64-bit division,
// which compiles to a subroutine call
PG_DEVICE int grs_owner(const PgGradRS& g, long long off) {
  int k = 0;
#pragma unroll
  for (int i = 1; i < PG_MAX_PEERS; ++i)
    if (i < g.world && off >= i * g.seg) k = i;
  return k;
}

PG_DEVICE float* grs_target(const PgGradRS& g, const float* local_ptr) {
  const long long off = local_ptr - g.local;
  return g.peer[grs_owner(g, off - g.start)] + off;
}

PG_DEVICE void grs_add4_at(const PgGradRS& g, float* target, float4 v) {
  if (g.scalar_red) {
    red_add_f32(target, v.x);
    red_add_f32(target + 1, v.y);
    red_add_f32(target + 2, v.z);
    red_add_f32(target + 3, v.w);
  } else {
    red_add_v4_f32(target, v);
  }
}

// 16-byte aligned group of four floats (a group never straddles two owners: start and seg are multiples of 4)
PG_DEVICE void grs_add4(const PgGradRS& g, const float* local_ptr, float4 v) { grs_add4_at(g, grs_target(g, local_ptr), v); }

}  // namespace pg
