// Host helper of the tensor-core sample net (hr_mlp_tc2.cu): weight images.
//
// Weight images: every fp32 weight w of the reference's nn.Linear (nlf/nets/mlp.py:127-154) is split into bf16
// hi = rn(w), lo = rn(w - hi) and laid out the way wgmma reads its B operand from shared memory: K-major,
// no swizzle, core matrices of 8 rows x 16 bytes (LBO = N * 16 B between the two 8-wide k-groups of a 16-wide k-step,
// SBO = 128 B between 8-row groups).  One image = one k-step of one pass = N x 16 bf16 hi followed by N x 16 bf16 lo;
// images are concatenated in consumption order so a producer warp streams them with cp.async.bulk (pack_mlp_tc2 packs
// each column half of a pass as a pass of its own, one stream per half).
//
// fp16 net (HR_MLP_FP16_TC, f16 != 0): one image per k-step, N x 16 fp16 rn(w), in the same layout and order, and the bias
// rounded to fp16 (kept as fp32): the operands CUDA autocast gives F.linear.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "hr_tc_prims.cuh"

namespace hr {

// A pass consumes `n_chunks` 32-wide k-chunks starting at chunk `first_chunk`; chunks [0, in_chunks) are the encoded
// input (zero padded past mlp_in), chunks in_chunks.. the hidden activations.  The skip layer's weight is
// [out, mlp_in + W] with the input columns first (mlp.py:167-168: cat([input_x, x])).
__global__ void pack_tc_pass(const float* __restrict__ W, const float* __restrict__ b, uint8_t* __restrict__ dst,
                             float* __restrict__ bias_dst, int n, int first_chunk, int n_chunks, int in_src, int mlp_in,
                             int is_skip, int in_chunks, int out_rows, int perm_S, int perm_stride, int out_col0, int f16) {
  // one thread per (image, n, kk)
  const long long total = (long long)n_chunks * 2 * n * 16;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total + n; i += (long long)gridDim.x * blockDim.x) {
    if (i >= total) {
      int nn = (int)(i - total);
      int ncol = out_col0 + nn;  // output column (channel-major for the last layer)
      float v = 0.0f;
      if (ncol < out_rows) {
        int ns = perm_S > 0 ? (ncol % perm_S) * perm_stride + (ncol / perm_S) : ncol;
        v = b[ns];
      }
      bias_dst[nn] = f16 ? __half2float(__float2half_rn(v)) : v;
      continue;
    }
    int kk = (int)(i % 16);
    int nn = (int)((i / 16) % n);
    int img = (int)(i / (16LL * n));
    int c = first_chunk + img / 2, ks = img % 2;
    int kc = ks * 16 + kk;  // k inside the chunk
    // source column of the reference weight
    int ksrc = -1;
    if (c < in_chunks) {
      const int kin = c * 32 + kc;
      if (kin < mlp_in) ksrc = kin;  // encoded input (first layer, or the input part of the skip layer)
    } else {
      int hcol = (c - in_chunks) * 32 + kc;
      ksrc = is_skip ? mlp_in + hcol : hcol;
    }
    int ncol = out_col0 + nn;
    float w = 0.0f;
    if (ncol < out_rows && ksrc >= 0 && ksrc < in_src) {
      int ns = perm_S > 0 ? (ncol % perm_S) * perm_stride + (ncol / perm_S) : ncol;
      w = W[(long long)ns * in_src + ksrc];
    }
    size_t slot = (size_t)(((kk >> 3) * (n >> 3) + (nn >> 3)) * 128 + (nn & 7) * 16 + (kk & 7) * 2);
    if (f16) {
      *reinterpret_cast<__half*>(dst + (size_t)img * n * 32 + slot) = __float2half_rn(w);
      continue;
    }
    __nv_bfloat16 hi = __float2bfloat16_rn(w);
    __nv_bfloat16 lo = __float2bfloat16_rn(w - __bfloat162float(hi));
    size_t img_off = (size_t)img * n * 64;
    *reinterpret_cast<__nv_bfloat16*>(dst + img_off + slot) = hi;
    *reinterpret_cast<__nv_bfloat16*>(dst + img_off + (size_t)n * 32 + slot) = lo;
  }
}

void launch_pack_tc_pass(const float* W, const float* b, uint8_t* dst, float* bias_dst, int n, int first_chunk, int n_chunks,
                         int in_src, int mlp_in, int is_skip, int in_chunks, int out_rows, int perm_S, int perm_stride,
                         int out_col0, int f16, cudaStream_t st) {
  long long total = (long long)n_chunks * 2 * n * 16 + n;
  int grid = (int)((total + 255) / 256);
  if (grid > 4096) grid = 4096;
  pack_tc_pass<<<grid, 256, 0, st>>>(W, b, dst, bias_dst, n, first_chunk, n_chunks, in_src, mlp_in, is_skip, in_chunks, out_rows,
                                     perm_S, perm_stride, out_col0, f16);
}

}  // namespace hr
