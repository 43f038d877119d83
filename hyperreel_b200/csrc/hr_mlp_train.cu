// Backward pass of the sample net on the Hopper tensor cores (hr_train_net_backward), wgmma.
//
// Every GEMM uses the inference net's bf16x3 split (hr_mlp_tc2.cu): fp32 operands are split on load into bf16
// hi = rn(x), lo = rn(x - hi), and D = A_hi*B_hi + A_lo*B_hi + A_hi*B_lo with fp32 accumulation in registers.
// Per layer l, walking back from the last (dY_{L-1} = d heads, channel-major like the packed weights):
//   dW / db   dW_l = dY_l^T X_l over K = rays, split-K across CTAs into fp32 partial tiles, then a fixed-order sum
//             (no float atomics: the gradients are bit-reproducible); db_l = the column sums of dY_l, taken in the same
//             pass from the fp32 values the A loader holds;
//   dX        dY_{l-1} = (dY_l W_l) * leaky'(a_{l-1}) over the hidden input columns only (the encoded-input columns of
//             the first and the skip layer are dropped: rays are not parameters).  The LeakyReLU side comes from the
//             saved activation's sign (the slope is > 0, so it is the pre-activation's).
// X_l is the saved encoded input and / or a_{l-1} (mlp.py:167-168: the skip layer reads cat([input, hidden])); W_l is read
// from the fp32 CUDA-core pack Wt[k][n] = W[n][k] that hr_upload keeps for every net, so no extra weight image exists.
//
// Kernel layout (train_gemm_kernel): one 128 x 128 output tile per CTA, two consumer warpgroups of 64 rows (wgmma
// m64n128k16), K in blocks of 32.  All 256 threads load the next block's fp32 operands into registers while the wgmmas of
// the current block run, then split them into a double-buffered shared-memory stage (K-major, no swizzle, the layout of
// hr_tc_prims.cuh).  dX reads both operands K-contiguous (rows of dY_l, rows of Wt), dW reads both MN-contiguous (dY_l and
// X_l are ray-major); each loader's thread mapping keeps its shared-memory stores free of bank conflicts.
#include <cuda.h>
#include <cuda_bf16.h>

#include "hr_mlp.cuh"
#include "hr_tc_prims.cuh"

namespace hr {

namespace tg {
using namespace tc;
constexpr int BN = 128;                         // output columns per CTA
constexpr int BK = 32;                          // k per block: two k-step images
constexpr int NT = 256;                         // two consumer warpgroups
constexpr int OP_BYTES = (BK / 16) * 4096;      // one operand half (hi or lo): 2 k-step images of 128 rows x 16 k bf16
constexpr int STAGE_BYTES = 4 * OP_BYTES;       // A hi, A lo, B hi, B lo
constexpr int SMEM_BYTES = 2 * STAGE_BYTES;     // double buffered: 64 KB

struct Gemm {
  const float* a; long long lda;  // dX: A[m][k] = a[m * lda + k];  dW: A[m][k] = a[k * lda + m]
  const float* b; long long ldb;  // dX: B[n][k] = b[n * ldb + k];  dW: B[n][k] = b[k * ldb + n]
  long long m_rows;               // rows of A read (others are 0): dX rays, dW output units (multiple of 4)
  int n_rows;                     // rows of B read: dX hidden units, dW input features (multiple of 4)
  long long k_len;                // dX: output units of the layer (multiple of 4), dW: rays
  long long k_split;              // dW: K range of one blockIdx.z (multiple of BK)
  const float* act; float* out; int ld_out; float slope;  // dX epilogue
  float* part; float* dbpart; int m_pad, n_pad;           // dW epilogue: [z][m_pad][n_pad] tiles, [z][m_pad] column sums
};

__device__ __forceinline__ float4 ld4(const float* p, bool ok) {
  return ok ? __ldg(reinterpret_cast<const float4*>(p)) : make_float4(0.f, 0.f, 0.f, 0.f);
}

// K-contiguous source, 128 rows x 32 k: element group i of this thread is 4 consecutive k of one row.  Within a warp,
// lanes 0-7 take 8 consecutive rows and lanes 8-31 the four 4-k quarters of a k-step, so each half warp's 8-byte stores
// fill 128 distinct bytes.
__device__ __forceinline__ void kc_coord(int idx, int& row, int& k) {
  row = (idx >> 6) * 8 + (idx & 7);
  k = ((idx >> 5) & 1) * 16 + ((idx >> 4) & 1) * 8 + ((idx >> 3) & 1) * 4;
}
__device__ __forceinline__ void load_kc(float4 (&v)[4], const float* src, long long ld, long long r0, long long rows,
                                        long long k0, long long k_end) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int row, k;
    kc_coord(threadIdx.x + NT * i, row, k);
    v[i] = ld4(src + (r0 + row) * ld + k0 + k, r0 + row < rows && k0 + k < k_end);
  }
}
__device__ __forceinline__ void store_kc(const float4 (&v)[4], uint8_t* hi, uint8_t* lo) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int row, k;
    kc_coord(threadIdx.x + NT * i, row, k);
    const uint32_t off = (uint32_t)(k >> 4) * 4096u + ks_slot(row, (k >> 3) & 1) + (uint32_t)(k & 7) * 2u;
    uint32_t h0, l0, h1, l1;
    split2(v[i].x, v[i].y, h0, l0);
    split2(v[i].z, v[i].w, h1, l1);
    *reinterpret_cast<uint2*>(hi + off) = make_uint2(h0, h1);
    *reinterpret_cast<uint2*>(lo + off) = make_uint2(l0, l1);
  }
}

// MN-contiguous source, 32 k x 128 rows: item i of this thread is k pair (2 kp, 2 kp + 1) x rows 4 q .. 4 q + 3, loaded as
// two float4 and stored as four bf16 pairs.  Lanes: kp & 3 = lane & 3, q & 7 = lane >> 2; the four rows are visited in a
// lane-rotated order so that every store instruction of a warp hits 32 different banks.  The rows of a thread are the same
// for both items (the dW column sums rely on it).
__device__ __forceinline__ void mn_coord(int i, int& row, int& kp) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, combo = warp * 2 + i;
  kp = (lane & 3) + 4 * (combo & 3);
  row = 4 * ((lane >> 2) + 8 * (combo >> 2));
}
__device__ __forceinline__ void load_mn(float4 (&v)[4], const float* src, long long ld, long long r0, long long rows,
                                        long long k0, long long k_end) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    int row, kp;
    mn_coord(i, row, kp);
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const long long k = k0 + 2 * kp + t;
      v[2 * i + t] = ld4(src + k * ld + r0 + row, k < k_end && r0 + row < rows);
    }
  }
}
__device__ __forceinline__ float comp(const float4& v, int j) { return j == 0 ? v.x : j == 1 ? v.y : j == 2 ? v.z : v.w; }
template <bool SUM>
__device__ __forceinline__ void store_mn(const float4 (&v)[4], uint8_t* hi, uint8_t* lo, float (&sum)[4]) {
  const int rot = (threadIdx.x >> 3) & 3;  // (lane >> 2) >> 1
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    int row, kp;
    mn_coord(i, row, kp);
    const int k = 2 * kp;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = (jj + rot) & 3;
      const float x0 = comp(v[2 * i], j), x1 = comp(v[2 * i + 1], j);
      uint32_t h, l;
      split2(x0, x1, h, l);
      const uint32_t off = (uint32_t)(k >> 4) * 4096u + ks_slot(row + j, (k >> 3) & 1) + (uint32_t)(k & 7) * 2u;
      *reinterpret_cast<uint32_t*>(hi + off) = h;
      *reinterpret_cast<uint32_t*>(lo + off) = l;
    }
    if (SUM) {
#pragma unroll
      for (int j = 0; j < 4; ++j) sum[j] += comp(v[2 * i], j) + comp(v[2 * i + 1], j);
    }
  }
}

}  // namespace tg

template <bool DW>
__global__ void __launch_bounds__(tg::NT, 1) train_gemm_kernel(const __grid_constant__ tg::Gemm g) {
  using namespace tg;
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const long long m0 = (long long)blockIdx.x * 128;
  const int n0 = blockIdx.y * BN;
  long long k0 = 0, k1 = g.k_len;
  if (DW) {
    k0 = (long long)blockIdx.z * g.k_split;
    k1 = k0 + g.k_split < g.k_len ? k0 + g.k_split : g.k_len;
  }
  const int nkb = k1 > k0 ? (int)((k1 - k0 + BK - 1) / BK) : 0;
  const bool col_sums = DW && blockIdx.y == 0;

  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.0f;
  float dbs[4] = {0.f, 0.f, 0.f, 0.f};
  float4 va[4], vb[4];
  auto load = [&](long long kb0) {
    if (DW) {
      load_mn(va, g.a, g.lda, m0, g.m_rows, kb0, k1);
      load_mn(vb, g.b, g.ldb, n0, g.n_rows, kb0, k1);
    } else {
      load_kc(va, g.a, g.lda, m0, g.m_rows, kb0, k1);
      load_kc(vb, g.b, g.ldb, n0, g.n_rows, kb0, k1);
    }
  };
  if (nkb > 0) load(k0);
  for (int kb = 0; kb < nkb; ++kb) {
    // the stage written here was last read by the wgmmas of block kb - 2, which both warpgroups waited for before the
    // __syncthreads of block kb - 1
    uint8_t* st = smem + (kb & 1) * STAGE_BYTES;
    if (DW) {
      if (col_sums) store_mn<true>(va, st, st + OP_BYTES, dbs);
      else store_mn<false>(va, st, st + OP_BYTES, dbs);
      store_mn<false>(vb, st + 2 * OP_BYTES, st + 3 * OP_BYTES, dbs);
    } else {
      store_kc(va, st, st + OP_BYTES);
      store_kc(vb, st + 2 * OP_BYTES, st + 3 * OP_BYTES);
    }
    fence_async_smem();
    __syncthreads();
    if (kb + 1 < nkb) load(k0 + (long long)(kb + 1) * BK);  // in flight under this block's wgmmas
    wgmma_fence();
    acc_fence(acc);
    const uint32_t s = smem_u32(st);
#pragma unroll
    for (int ks = 0; ks < BK / 16; ++ks) {
      const uint32_t a = s + ks * 4096 + wg * 1024, b = s + 2 * OP_BYTES + ks * 4096;
      const uint64_t ah = gmma_desc(a, 2048, 128), al = gmma_desc(a + OP_BYTES, 2048, 128);
      const uint64_t bh = gmma_desc(b, 2048, 128), bl = gmma_desc(b + OP_BYTES, 2048, 128);
      wgmma_ss(acc, ah, bh, 1u);
      wgmma_ss(acc, al, bh, 1u);
      wgmma_ss(acc, ah, bl, 1u);
    }
    wgmma_commit();
    acc_fence(acc);
    wgmma_wait<0>();
    acc_fence(acc);
  }

  // accumulator d[i]: row 16 (warp % 4) + lane / 4 + 8 ((i / 2) % 2) of this warpgroup's 64, column 8 (i / 4) + 2 (lane % 4) + i % 2
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), q2 = (lane & 3) * 2;
  if (!DW) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long r = m0 + row0 + 8 * h;
      if (r >= g.m_rows) continue;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const long long o = r * g.ld_out + n0 + 8 * j + q2;
        const float2 a = *reinterpret_cast<const float2*>(g.act + o);
        *reinterpret_cast<float2*>(g.out + o) =
            make_float2(acc[4 * j + 2 * h] * (a.x > 0.0f ? 1.0f : g.slope), acc[4 * j + 2 * h + 1] * (a.y > 0.0f ? 1.0f : g.slope));
      }
    }
    return;
  }
  float* p = g.part + ((long long)blockIdx.z * g.m_pad + m0) * g.n_pad + n0;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < 16; ++j)
      *reinterpret_cast<float2*>(p + (long long)(row0 + 8 * h) * g.n_pad + 8 * j + q2) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
  if (col_sums) {
    // 8 threads hold partial sums of the same 4 rows (store_mn): add them in a fixed order
    __syncthreads();  // every warpgroup's wgmmas have retired: the stages are free
    float* red = reinterpret_cast<float*>(smem);  // [8][128]
    int row, kp;
    mn_coord(0, row, kp);
    const int slot = (warp & 1) * 4 + (lane & 3);
#pragma unroll
    for (int j = 0; j < 4; ++j) red[slot * 128 + row + j] = dbs[j];
    __syncthreads();
    if (tid < 128) {
      float s = 0.0f;
#pragma unroll
      for (int i = 0; i < 8; ++i) s += red[i * 128 + tid];
      g.dbpart[(long long)blockIdx.z * g.m_pad + m0 + tid] = s;
    }
  }
}

// dw[perm(m)][col0 + c] = sum over z (ascending) of part[z][m][c]; db[perm(m)] likewise from dbpart.  perm maps the packed
// last layer's channel-major row c*S+s back to the reference's s*stride+c.
__global__ void train_dw_reduce(const float* __restrict__ part, const float* __restrict__ dbpart, int splits, int m_pad, int n_pad,
                                int m_rows, int n_valid, float* __restrict__ dw, int ld_dw, int col0, float* __restrict__ db, int perm_S,
                                int perm_stride) {
  const long long total = (long long)m_rows * n_valid, all = total + (db ? m_rows : 0);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < all; i += (long long)gridDim.x * blockDim.x) {
    const bool is_db = i >= total;
    const int m = is_db ? (int)(i - total) : (int)(i / n_valid), c = is_db ? 0 : (int)(i % n_valid);
    float s = 0.0f;
    for (int z = 0; z < splits; ++z) s += is_db ? dbpart[(long long)z * m_pad + m] : part[((long long)z * m_pad + m) * n_pad + c];
    const int ms = perm_S > 0 ? (m % perm_S) * perm_stride + m / perm_S : m;
    if (is_db) db[ms] = s;
    else dw[(long long)ms * ld_dw + col0 + c] = s;
  }
}

namespace {
size_t seg(long long floats) { return (size_t)((floats * 4 + 255) / 256 * 256); }
int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }
}  // namespace

TrainNetLayout train_net_layout(const hr_config& c, long long n, int num_sms) {
  TrainNetLayout t{};
  const long long W = c.mlp_width;
  t.ld_enc = (c.mlp_in + 15) / 16 * 16;
  size_t off = 0;
  t.enc = off; off += seg(n * t.ld_enc);
  t.act = off; t.act_stride = seg(n * W) / 4; off += (size_t)(c.mlp_layers - 1) * seg(n * W);
  t.ld_dlast = (c.mlp_out + 3) / 4 * 4;
  t.dlast = off; off += seg(n * t.ld_dlast);
  t.dy[0] = off; off += seg(n * W);
  t.dy[1] = off; off += seg(n * W);
  // split-K: at most 2 CTAs per SM of 128 x 128 partial tiles (train_net_backward picks the split count)
  t.part = off; off += seg(2LL * num_sms * 128 * 128);
  t.dbpart = off; off += seg(2LL * num_sms * 128);
  t.total = off;
  return t;
}

cudaError_t train_net_backward(const hr_config& c, const MlpSimtPack& simt, long long n, float* const* weight,
                               float* const* bias, uint8_t* ws, int num_sms, cudaStream_t st) {
  using namespace tg;
  const TrainNetLayout t = train_net_layout(c, n, num_sms);
  const int L = c.mlp_layers, W = c.mlp_width;
  auto fp = [&](size_t off) { return reinterpret_cast<float*>(ws + off); };
  float* act = fp(t.act);
  cudaError_t e = cudaFuncSetAttribute(train_gemm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(train_gemm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  if (e != cudaSuccess) return e;

  // dW[rows of dy][col0 .. col0 + n_valid) += dy^T x over all rays, dy [n][ld_dy] (out_l rows of dW, then zero pad columns up
  // to ld_dy, a multiple of 4: the GEMM computes their rows too, the reduction writes back the out_l real ones), x [n][ldx]
  // with ldx >= n_rows
  auto dw_gemm = [&](const float* dy, int out_l, int ld_dy, const float* x, int ldx, int n_valid, float* dw, int ld_dw, int col0,
                     float* db, int perm_S) -> cudaError_t {
    Gemm g{};
    g.a = dy; g.lda = ld_dy; g.m_rows = ld_dy;
    g.b = x; g.ldb = ldx; g.n_rows = ldx;
    g.k_len = n;
    const int tm = cdiv(ld_dy, 128), tn = cdiv(ldx, BN), kbs = cdiv(n, BK);
    int splits = (2 * num_sms) / (tm * tn);
    if (splits < 1) splits = 1;
    if (splits > kbs) splits = kbs > 0 ? kbs : 1;
    g.k_split = (long long)cdiv(kbs, splits) * BK;
    splits = n > 0 ? cdiv(n, g.k_split) : 1;
    g.part = fp(t.part); g.dbpart = fp(t.dbpart); g.m_pad = tm * 128; g.n_pad = tn * BN;
    train_gemm_kernel<true><<<dim3(tm, tn, splits), NT, SMEM_BYTES, st>>>(g);
    const long long work = (long long)out_l * n_valid + (db ? out_l : 0);
    train_dw_reduce<<<cdiv(work, 256) < 4096 ? cdiv(work, 256) : 4096, 256, 0, st>>>(
        g.part, g.dbpart, splits, g.m_pad, g.n_pad, out_l, n_valid, dw, ld_dw, col0, db, perm_S, c.head_stride);
    return cudaGetLastError();
  };

  for (int l = L - 1; l >= 0; --l) {
    const bool last = (l == L - 1), skip = (l == c.mlp_skip);
    const int out_l = last ? c.mlp_out : W, ld_dy = last ? t.ld_dlast : W;
    const float* dy = last ? fp(t.dlast) : fp(t.dy[(L - 2 - l) & 1]);
    const int in_l = l == 0 ? c.mlp_in : (skip ? c.mlp_in + W : W);
    const int perm_S = last ? c.n_samples : 0;
    if (l == 0 || skip) {  // encoded-input columns (and db)
      e = dw_gemm(dy, out_l, ld_dy, fp(t.enc), t.ld_enc, c.mlp_in, weight[l], in_l, 0, bias[l], perm_S);
      if (e != cudaSuccess) return e;
    }
    if (l > 0) {
      const float* a_prev = act + (size_t)(l - 1) * t.act_stride;
      e = dw_gemm(dy, out_l, ld_dy, a_prev, W, W, weight[l], in_l, skip ? c.mlp_in : 0, skip ? nullptr : bias[l], perm_S);
      if (e != cudaSuccess) return e;
      // dY_{l-1} = (dY_l W_l[:, hidden]) * leaky'(a_{l-1})
      Gemm g{};
      g.a = dy; g.lda = ld_dy; g.m_rows = n;  // the zero pad columns of d heads meet the zero pad columns of Wt
      g.b = simt.Wt[l] + (size_t)(skip ? simt.in_pad : 0) * simt.Np[l]; g.ldb = simt.Np[l]; g.n_rows = W;
      g.k_len = ld_dy;
      g.act = a_prev; g.out = fp(t.dy[(L - 1 - l) & 1]); g.ld_out = W; g.slope = c.leaky_slope;
      train_gemm_kernel<false><<<dim3(cdiv(n, 128), W / BN, 1), NT, SMEM_BYTES, st>>>(g);
      e = cudaGetLastError();
      if (e != cudaSuccess) return e;
    }
  }
  return cudaSuccess;
}

}  // namespace hr
