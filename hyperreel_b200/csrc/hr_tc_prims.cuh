// wgmma / mbarrier / bulk-copy primitives of the tensor-core sample-net kernel (sm_90a).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace hr {
namespace tc {

constexpr int BM = 128;  // rays per tile: two wgmma M = 64 row blocks

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(bar), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier over one warpgroup (ids 1.. ; 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
// one-way signal between two warpgroups over named barrier `id`: the signalling warpgroup arrives, the other one waits
__device__ __forceinline__ void pair_arrive(int id) { asm volatile("bar.arrive %0, 256;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void pair_wait(int id) { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }

// K-major, no-swizzle wgmma shared-memory matrix descriptor: [0,14) start>>4 | [16,30) leading byte offset>>4 (between the
// two 8-wide k core matrices of a 16-wide k-step) | [32,46) stride byte offset>>4 (between 8-row groups) | layout type 0.
// A core matrix is 8 rows x 16 bytes, rows 16 bytes apart.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across a wgmma fence or wait
template <int N>
__device__ __forceinline__ void acc_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// per-warpgroup register budget (all warps of the warpgroup execute it)
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, N = 64 or 128, bf16 operands (fp16 with F16) from shared memory, fp32
// accumulators in registers.  Accumulator d[i] of thread t (warp w = t / 32 of the warpgroup, lane l): row
// 16 w + l / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (l % 4) + i % 2.
#define HR_WGMMA_N64(TY)                                                                                                   \
  asm volatile(                                                                                                            \
      "{\n\t"                                                                                                               \
      ".reg .pred p;\n\t"                                                                                                  \
      "setp.ne.b32 p, %34, 0;\n\t"                                                                                         \
      "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " "                                                           \
      "{"                                                                                                                  \
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "          \
      "%23, %24, %25, %26, %27, %28, %29, %30, %31"                                                                        \
      "}, %32, %33, p, 1, 1, 0, 0;\n\t"                                                                                    \
      "}"                                                                                                                  \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),                    \
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),              \
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),            \
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])             \
      : "l"(adesc), "l"(bdesc), "r"(accumulate))

#define HR_WGMMA_N128(TY)                                                                                                  \
  asm volatile(                                                                                                            \
      "{\n\t"                                                                                                               \
      ".reg .pred p;\n\t"                                                                                                  \
      "setp.ne.b32 p, %66, 0;\n\t"                                                                                         \
      "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " "                                                          \
      "{"                                                                                                                  \
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "          \
      "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "          \
      "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"                 \
      "}, %64, %65, p, 1, 1, 0, 0;\n\t"                                                                                    \
      "}"                                                                                                                  \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),                    \
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),              \
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),            \
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),            \
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),            \
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),            \
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),            \
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])             \
      : "l"(adesc), "l"(bdesc), "r"(accumulate))

template <bool F16 = false>
__device__ __forceinline__ void wgmma_ss(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if constexpr (F16) HR_WGMMA_N64("f16"); else HR_WGMMA_N64("bf16");
}
template <bool F16 = false>
__device__ __forceinline__ void wgmma_ss(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if constexpr (F16) HR_WGMMA_N128("f16"); else HR_WGMMA_N128("bf16");
}
#undef HR_WGMMA_N64
#undef HR_WGMMA_N128

// Four 8x8 b16 matrices from their mma fragments (r[i]: row t / 4, columns 2 (t % 4) and + 1 of matrix i) to shared memory;
// lane t gives the address of row t % 8 of matrix t / 8 (16 contiguous bytes).
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]),
               "r"(r[3])
               : "memory");
}

// Offset (bytes) of the 16-byte slot holding k-group kg (0/1) of row `row` inside a 128-row x 16-k k-step image.
__device__ __forceinline__ uint32_t ks_slot(int row, int kg) { return (uint32_t)((kg * 16 + (row >> 3)) * 128 + (row & 7) * 16); }

// fp32 pair -> bf16 hi = rn(x) and lo = rn(x - hi), packed two per 32-bit word
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 hh = __floats2bfloat162_rn(x0, x1);
  __nv_bfloat162 ll = __floats2bfloat162_rn(x0 - __low2float(hh), x1 - __high2float(hh));
  hi = *reinterpret_cast<uint32_t*>(&hh);
  lo = *reinterpret_cast<uint32_t*>(&ll);
}

// fp32 -> the nearest fp16 value (overflow gives inf), as fp32
__device__ __forceinline__ float rn16(float x) { return __half2float(__float2half_rn(x)); }
// fp32 pair -> fp16 rn(x0), rn(x1), packed two per 32-bit word
__device__ __forceinline__ uint32_t pack_half2(float x0, float x1) {
  __half2 hh = __floats2half2_rn(x0, x1);
  return *reinterpret_cast<uint32_t*>(&hh);
}

}  // namespace tc

// host helper defined in hr_tc_pack.cu
void launch_pack_tc_pass(const float* W, const float* b, uint8_t* dst, float* bias_dst, int n, int first_chunk, int n_chunks,
                         int in_src, int mlp_in, int is_skip, int in_chunks, int out_rows, int perm_S, int perm_stride,
                         int out_col0, int f16, cudaStream_t st);
}  // namespace hr
