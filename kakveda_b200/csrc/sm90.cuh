// Hopper (sm_90a) building blocks shared by the tensor-core kernels (K1b-B in bound_kernel.cuh, K2 in dense_index.cu):
// shared-memory addressing, mbarriers, 2-D TMA loads and the wgmma descriptor / fences, plus the host-side encoder of
// the tensor maps those TMA loads read (defined in kv_common.cpp).
#pragma once
#include <cuda.h>
#include <cstdint>

__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Bytes from the dynamic shared array to its first 1024-byte boundary (where 128-byte-swizzled TMA / wgmma tiles must
// start).  Kernels align by adding this OFFSET to the shared array, not by rounding a generic pointer: the compiler then
// keeps the shared address space, so every access is LDS/STS/ATOMS instead of a generic load / store / atomic.
__device__ __forceinline__ uint32_t smem_align1024(const void *smem_raw) {
  return (1024u - (smem_addr(smem_raw) & 1023u)) & 1023u;
}

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_addr(bar)),
      "r"(parity)
      : "memory");
}

// box (c0 = column, c1 = row) of a 2-D tensor map -> shared memory, completion counted in bytes on `bar`
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_addr(dst)),
      "l"((uint64_t)map), "r"(smem_addr(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// wgmma shared-memory matrix descriptor: K-major, 128-byte swizzle, 8-row groups 1024 bytes apart (the operand tile
// starts on a 1024-byte boundary, so the base offset is 0).  Advancing the start address by 32 bytes selects the next
// K = 16 step inside the swizzled 128-byte row.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(const void *smem) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr(smem) & 0x3FFFF) >> 4);  // start address
  d |= (uint64_t)1 << 16;                              // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;                    // stride byte offset
  d |= (uint64_t)1 << 62;                              // SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of an accumulator register across an asynchronous wgmma
__device__ __forceinline__ void wgmma_reg_fence(float &r) { asm volatile("" : "+f"(r)::"memory"); }

// Tensor map of a row-major matrix [rows][cols] of 2-byte elements (dtype: CU_TENSOR_MAP_DATA_TYPE_FLOAT16 or
// _BFLOAT16): boxes of 64 columns (one 128-byte swizzle row) x box_rows rows, 128-byte swizzle, L2 promotion 256 B.
// Returns KV_OK or a KV_ERR_CUDA failure (kv_last_error).
int make_map_2d(CUtensorMap *map, CUtensorMapDataType dtype, const void *base, int64_t rows, int64_t cols, int box_rows);
