// Thin inline-PTX wrappers for the sm_90a primitives used by every kernel in this
// tree: mbarrier, TMA (cp.async.bulk.tensor), named barriers, system-scope
// acquire/release flag traffic for cross-GPU protocols, and vector global
// loads/stores (wgmma lives in wgmma.cuh).  No CUTLASS dependency: the bit layouts
// follow the PTX ISA.
#pragma once
#include <cstdio>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pg {

#define PG_DEVICE __device__ __forceinline__

PG_DEVICE uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

PG_DEVICE uint32_t lane_id() {
  uint32_t l;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
  return l;
}

PG_DEVICE bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------
PG_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
PG_DEVICE void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
PG_DEVICE void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
PG_DEVICE void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
PG_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
PG_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
PG_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------
PG_DEVICE void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tiled load global -> shared, completion signalled on an mbarrier (complete_tx).
PG_DEVICE void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0,
                           int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
PG_DEVICE void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0,
                           int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// 2-D tiled store shared -> global (bulk group completion).
PG_DEVICE void tma_store_2d(const CUtensorMap* m, const void* smem_src, int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(m)),
      "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
      : "memory");
}
// 3-D tiled reduce-add shared -> global (bulk group completion, same commit / wait as the store).  The element type
// of the map selects the add (fp32 for an fp32 map); elements outside the tensor are skipped.
PG_DEVICE void tma_reduce_add_3d(const CUtensorMap* m, const void* smem_src, int32_t c0, int32_t c1, int32_t c2) {
  asm volatile(
      "cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(m)),
      "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
PG_DEVICE void tma_reduce_add_2d(const CUtensorMap* m, const void* smem_src, int32_t c0, int32_t c1) {
  asm volatile(
      "cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(m)),
      "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
      : "memory");
}
PG_DEVICE void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
PG_DEVICE void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
PG_DEVICE void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// 1-D bulk copy global -> shared (no tensor map; 16-byte aligned, size multiple of 16).
PG_DEVICE void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
PG_DEVICE void bulk_store_1d(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(
                   reinterpret_cast<uint64_t>(gdst)),
               "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}

// shared-memory access by 32-bit shared address (a generic pointer into dynamic shared memory can compile to a
// generic LD / ST with 64-bit addresses).  volatile: never moved across the barrier waits around them.
PG_DEVICE void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
PG_DEVICE void st_shared_v2_f32(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
PG_DEVICE void st_shared_s32(uint32_t addr, int v) { asm volatile("st.shared.s32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
PG_DEVICE int ld_shared_s32(uint32_t addr) {
  int v;
  asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
PG_DEVICE float2 ld_shared_v2_f32(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}

// named barrier over `count` threads (a multiple of 32) of the CTA; id 0 is __syncthreads
PG_DEVICE void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ----------------------------------------------------------------------------------
// system-scope flags for cross-GPU protocols over NVLink peer mappings
// ----------------------------------------------------------------------------------
PG_DEVICE void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
PG_DEVICE uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
PG_DEVICE uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
PG_DEVICE void red_add_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
PG_DEVICE void fence_acq_rel_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }

// Register re-balancing between the warpgroups (4 consecutive warps) of a CTA: a kernel launched with a small per-thread
// register count (so that other CTAs fit next to it on the SM) lets its light warpgroups give registers back and its
// heavy ones take them.  Must be executed by all four warps of a warpgroup.
template <int N>
PG_DEVICE void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
PG_DEVICE void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

// Bounded spin on a monotonic flag / counter written by another CTA or another GPU (system-scope acquire).  A flag
// that never arrives (a peer that died, a protocol bug) must not hang the node silently: after ~30 s of SM clocks
// the waiting thread prints where it waited and what it saw, and traps — the host sees a launch failure with a
// diagnostic instead of a wedged GPU.  `site` identifies the wait in the source (see the table in DESIGN.md).
#ifndef PG_SPIN_BUDGET_CYCLES
#define PG_SPIN_BUDGET_CYCLES 60000000000ll
#endif
PG_DEVICE void spin_until_ge(const uint32_t* p, uint32_t want, int site) {
  if (ld_acquire_sys(p) >= want) return;
  const long long t0 = clock64();
  uint32_t seen;
  while ((seen = ld_acquire_sys(p)) < want) {
    if (clock64() - t0 > PG_SPIN_BUDGET_CYCLES) {
      printf("pipegoose_b200: spin timeout at site %d: flag %p holds %u, waiting for >= %u (block %d thread %d)\n", site,
             (const void*)p, seen, want, (int)blockIdx.x, (int)threadIdx.x);
      __trap();
    }
  }
}
// The same wait without the diagnostic printf, for kernels that issue wgmma: a printf (an ABI call) anywhere in such a
// kernel makes ptxas serialise every wgmma of it (C7510), even when the call sits in another warp role.  A flag that
// never arrives still traps after the budget: the host sees a launch failure instead of a wedged GPU, without the site.
PG_DEVICE void spin_until_ge_quiet(const uint32_t* p, uint32_t want) {
  if (ld_acquire_sys(p) >= want) return;
  const long long t0 = clock64();
  while (ld_acquire_sys(p) < want) {
    if (clock64() - t0 > PG_SPIN_BUDGET_CYCLES) __trap();
  }
}
// generic-proxy writes (peer flags / data) -> later async-proxy (TMA) reads of global memory
PG_DEVICE void fence_proxy_async_global() {
  asm volatile("fence.proxy.async.global;" ::: "memory");
}

// ----------------------------------------------------------------------------------
// programmatic dependent launch (PDL): the next kernel of the stream may start its prologue (smem carve-up,
// barrier init, tensor-map prefetch) while this one is still running; it blocks in pdl_wait()
// until every predecessor has completed and its memory operations are visible.  Both are no-ops for kernels
// that were not launched with the programmatic-stream-serialization attribute.
// ----------------------------------------------------------------------------------
PG_DEVICE void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
PG_DEVICE void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ----------------------------------------------------------------------------------
// vector global access
// ----------------------------------------------------------------------------------
PG_DEVICE uint4 ld_global_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
PG_DEVICE uint4 ld_global_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
PG_DEVICE void st_global_v4(void* p, uint4 v) {
  asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}
PG_DEVICE void st_global_na_v4(void* p, uint4 v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

PG_DEVICE void red_add_v4_f32(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

// ----------------------------------------------------------------------------------
// NVLS: loads / stores on a multicast address are executed by the NVSwitch on every replica bound to the multicast
// object — ld_reduce returns the SUM over the replicas (reduced inside the switch: one response crosses the link
// instead of one per peer), st writes all replicas with one request.
// ----------------------------------------------------------------------------------
PG_DEVICE float4 multimem_ld_reduce_add_v4_f32(const float* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
PG_DEVICE void multimem_st_v4_f32(float* mc, float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}
// eight bf16 values summed over the replicas with fp32 accumulation inside the switch
PG_DEVICE uint4 multimem_ld_reduce_add_v4_bf16x2(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
PG_DEVICE void multimem_st_v4_b32(void* mc, uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.bf16x2 [%0], {%1, %2, %3, %4};" ::"l"(mc), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}

PG_DEVICE void red_add_f32(float* p, float v) { asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory"); }

PG_DEVICE uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
PG_DEVICE float2 unpack_bf16x2(uint32_t v) {
  __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&v);
  return __bfloat1622float2(t);
}

PG_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
PG_DEVICE float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace pg
