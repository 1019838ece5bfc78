// wgmma / TMA / mbarrier building blocks shared by the tensor-core kernels of this library (sm_90a).
#pragma once
#include <cuda.h>
#include "formats.cuh"

namespace anyloc {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  long long t0 = 0;
  for (uint32_t it = 0; !done; ++it) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (!done && (it & 0x3ff) == 0x3ff) {              // watchdog: never hang the GPU (try_wait itself
      long long now = clock64();                        // suspends for a HW-bounded time per call)
      if (t0 == 0) t0 = now;
      else if (now - t0 > 8000000000LL) __trap();      // ~4 s
    }
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}

// TMA store of a box from shared memory (bulk-group completion), and the bulk-group bookkeeping around it
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(map), "r"(src), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every committed bulk group but the newest N has finished reading its shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// every committed bulk group but the newest N has completed (its global writes performed)
template <int N>
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// orders this thread's generic-proxy shared-memory accesses before later async-proxy (TMA) accesses
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier ID over `count` threads (id 0 is __syncthreads')
template <int ID>
__device__ __forceinline__ void named_bar_sync(int count) {
  asm volatile("bar.sync %0, %1;" ::"n"(ID), "r"(count) : "memory");
}

// wgmma matrix descriptor: K-major, 128B swizzle (8-row x 128 B atoms, 1024 B apart = SBO; LBO unused for swizzled
// K-major operands), layout type 1 = SWIZZLE_128B.  A k-step of 32 bytes inside the atom advances the start address.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma boundary
template <int R>
__device__ __forceinline__ void fence_regs(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define ANYLOC_WG_D64                                                                                               \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),       \
      "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),        \
      "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),       \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),       \
      "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),       \
      "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),       \
      "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),       \
      "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define ANYLOC_WG_D64_STR                                                                                           \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
  "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "  \
  "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define ANYLOC_WG_M64N128(SHAPE_TYPES, TAIL)                                                                        \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                                 \
               "wgmma.mma_async.sync.aligned.m64n128" SHAPE_TYPES " " ANYLOC_WG_D64_STR ", %64, %65, p, 1, 1" TAIL     \
               ";\n\t}"                                                                                              \
               : ANYLOC_WG_D64 : "l"(adesc), "l"(bdesc), "r"(scale_d))

// D[64 x 128] (+)= A[64 x K] . B[128 x K]^T of FMT operands, both K-major in shared memory; 32 bytes of K per
// instruction: K = 8 (tf32), 16 (fp16, bf16, either pairs' halves) or 32 (e4m3).
// Accumulator layout (per warpgroup thread t, warp w = t / 32, lane l): d[4j + {0,1}] = row 16w + l/4, columns
// 8j + 2(l%4) + {0,1}; d[4j + {2,3}] = row 16w + l/4 + 8, same columns.
template <int FMT>
__device__ __forceinline__ void wgmma_m64n128(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  if constexpr (FMT == ANYLOC_PAIR_TF32) ANYLOC_WG_M64N128("k8.f32.tf32.tf32", "");
  else if constexpr (FMT == ANYLOC_PAIR_FP8) ANYLOC_WG_M64N128("k32.f32.e4m3.e4m3", "");
  else if constexpr (FMT == ANYLOC_PAIR_BF16 || FMT == ANYLOC_PAIR_BF16X3) ANYLOC_WG_M64N128("k16.f32.bf16.bf16", ", 0, 0");
  else ANYLOC_WG_M64N128("k16.f32.f16.f16", ", 0, 0");     // fp16 pairs, single fp16
}
#undef ANYLOC_WG_M64N128
#undef ANYLOC_WG_D64
#undef ANYLOC_WG_D64_STR

__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

// setmaxnreg: hand registers from the producer warpgroup to the consumers (every warp of a warpgroup executes it)
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// wgmma matrix descriptor of an MN-major 16-bit operand with 128B swizzle: rows of 128 B (64 elements of N) are
// consecutive k, 8-row atoms 1024 B apart.  With N = 64 the operand is one atom wide, so only the stride between the
// 8-row groups along K matters (SBO); LBO (the stride between atoms along N) is given the same value.  A k16 step
// advances the start address by 2 atoms (2048 B).
__device__ __forceinline__ uint64_t make_desc_mn(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)(1024 >> 4) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

#define ANYLOC_WG_D32                                                                                               \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),       \
      "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),        \
      "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),       \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
#define ANYLOC_WG_D32_STR                                                                                           \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
  "%24, %25, %26, %27, %28, %29, %30, %31}"

// D[64 x 64] (+)= A[64 x 16] . B[64 x 16]^T, A and B K-major in shared memory (SS form); the 16-bit operands of FMT.
// Accumulator layout as wgmma_m64n128's: d[4j + {0,1}] = row 16w + l/4, columns 8j + 2(l%4) + {0,1}; d[4j + {2,3}] =
// row 16w + l/4 + 8.
template <int FMT>
__device__ __forceinline__ void wgmma_m64n64_ss(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  if constexpr (FMT == ANYLOC_PAIR_BF16 || FMT == ANYLOC_PAIR_BF16X3)
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " ANYLOC_WG_D32_STR ", %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : ANYLOC_WG_D32 : "l"(adesc), "l"(bdesc), "r"(scale_d));
  else
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " ANYLOC_WG_D32_STR ", %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : ANYLOC_WG_D32 : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

// D[64 x 64] (+)= A[64 x 16] . B[16 x 64], A from registers (RS form), B MN-major in shared memory (transposed B, 16-bit
// types only), the operands of FMT.  The A fragment of warp w is mma.sync m16n8k16's for rows [16w, 16w + 16): a[0] =
// (row l/4, k 2(l%4) + {0,1}), a[1] = row + 8, a[2] = k + 8, a[3] = both -- which is the accumulator layout of a 16-bit
// wgmma, two n8 column groups per k16 step.
template <int FMT>
__device__ __forceinline__ void wgmma_m64n64_rs_tb(float* d, const uint32_t* a, uint64_t bdesc, uint32_t scale_d) {
  if constexpr (FMT == ANYLOC_PAIR_BF16 || FMT == ANYLOC_PAIR_BF16X3)
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " ANYLOC_WG_D32_STR
                 ", {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
                 : ANYLOC_WG_D32 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
  else
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " ANYLOC_WG_D32_STR
                 ", {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
                 : ANYLOC_WG_D32 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}
#undef ANYLOC_WG_D32
#undef ANYLOC_WG_D32_STR

// host: 2-D tiled tensor map over a row-major [rows, K] matrix of fmt's elements (row pitch ld elements), box = 128
// bytes of K x box_rows rows, 128B swizzle (defined in gemm_tc.cu)
int make_map(CUtensorMap* map, const void* ptr, int rows, int K, int ld, int box_rows, int fmt);
// host: 3-D tiled tensor map over imgs row-major [rows, cols] matrices of fmt's 2-byte elements laid end to end, box =
// 64 columns (128 B) x box_rows rows x 1 matrix, 128B swizzle; boxes past `rows` of a matrix read zeros
int make_map_3d16(CUtensorMap* map, const void* ptr, int imgs, int rows, int cols, int box_rows, int fmt);

}  // namespace tc
}  // namespace anyloc
