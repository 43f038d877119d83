// Sample-prediction network on the Hopper tensor cores (HR_MLP_BF16X3_TC), wgmma.
//
// Math (reference: nlf/nets/mlp.py:159-172 behind nlf/embedding/ray.py:320-326): every fp32 operand x is split into
// bf16 hi = rn(x) and lo = rn(x - hi) and each Linear layer is
//     D = A_hi*B_hi + A_lo*B_hi + A_hi*B_lo          (three wgmma m64nWk16 per k-step, in this order, k-steps ascending,
//                                                      fp32 accumulation in registers);
// the dropped A_lo*B_lo term and the split residuals are O(2^-16) relative per product (DESIGN.md).
// Hidden width W = 128 or 256 (a template parameter), encoded input up to 64 features (one or two 32-wide input chunks).
//
// Layout (one persistent CTA per SM, one 128-ray tile at a time):
//   * warpgroups 0 and 1 each own 64 rays of the tile (wgmma M = 64) and everything about them: they encode their rays
//     into the input operand, issue the wgmmas of every layer, and run the epilogues.  A warpgroup's operand rows are
//     read by its own wgmmas only, so the two warpgroups never wait for each other, and one's epilogue runs under the
//     other's MMAs;
//   * every Linear layer is issued as passes of N = W output columns: a hidden layer is one pass held in one register
//     accumulator (128 registers at W = 256), the last layer is ceil(out / W) zero-padded passes;
//   * the activation operand A (hi and lo, 2 x 64 KB at W = 256, K-major no-swizzle) is rewritten in place by the
//     epilogue of the layer that reads it: the warpgroup's wgmmas of that layer have all retired by then
//     (wgmma.wait_group 0);
//   * warpgroup 2 streams the weight images (bf16 hi + lo, consumption order, hr_tc_pack.cu) through a 4-stage
//     cp.async.bulk ring of 16 KB stages (one k-step at W = 256) guarded by mbarriers; each consumer warpgroup releases a
//     stage once the wgmmas that read it have retired, so every stage is loaded once per tile for both.
// The last layer's columns go from the accumulators (+ bias) straight to the heads scratch in global memory, 4 consecutive
// columns per 16-byte store; the hidden epilogues write the activation operand with stmatrix.
//
// SAVE (the training forward, hr_mlp_train.cu): the same arithmetic, plus every fp32 value the epilogues split goes to global
// memory as well -- the encoded input (sv.enc) and each hidden layer's LeakyReLU output (sv.act) -- and the heads are stored
// in the reference's sample-major column order instead of channel-major.
#include <cuda.h>
#include <cuda_bf16.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "hr_encode.cuh"
#include "hr_handle.h"
#include "hr_tc_prims.cuh"

namespace hr {

namespace tc2 {
using namespace tc;

constexpr int NSTAGE = 4;            // weight ring depth
constexpr int STAGE_BYTES = 16384;   // one ring stage: k-step images of W x 16 k x (hi + lo) bf16, 1 (W = 256) or 2 (W = 128)
constexpr int KSTEP_BYTES = 4096;    // activation k-step image: 128 rays x 16 k bf16
constexpr int CONSUMERS = 2;         // warpgroups of 64 rays
constexpr int NTHREADS = (CONSUMERS + 1) * 128;  // + the producer warpgroup (one thread of it issues the copies)
// register split of the 64 K registers (setmaxnreg): the producer warpgroup gives up what the consumers need beside their
// 128 accumulator registers at W = 256
constexpr int PRODUCER_REGS = 40;
constexpr int CONSUMER_REGS = 232;
static_assert(128 * PRODUCER_REGS + CONSUMERS * 128 * CONSUMER_REGS <= 65536, "register file");

// shared memory map (bytes)
constexpr int A_BYTES = 16 * KSTEP_BYTES;                    // 64 KB: one half (hi or lo) of the activation operand
constexpr int OFF_AHI = 0;
constexpr int OFF_ALO = OFF_AHI + A_BYTES;
constexpr int X_BYTES = 4 * KSTEP_BYTES;                     // encoded input: up to 4 k-steps (64 k) hi, then as many lo
constexpr int OFF_X = OFF_ALO + A_BYTES;                     // 131072
constexpr int OFF_B = OFF_X + 2 * X_BYTES;                   // 163840
constexpr int OFF_BAR = OFF_B + NSTAGE * STAGE_BYTES;        // 229376
constexpr int SMEM_BYTES = OFF_BAR + 128;                    // 229504 (of 232448 available)
static_assert(SMEM_BYTES <= 232448, "shared memory budget");

// barrier slots (8 bytes each) inside OFF_BAR
constexpr int BAR_FULL = 0;                   // [NSTAGE]
constexpr int BAR_EMPTY = BAR_FULL + NSTAGE;  // [NSTAGE]
static_assert((BAR_EMPTY + NSTAGE) * 8 <= 128, "barrier block");

}  // namespace tc2

template <int W, bool SAVE>
__global__ void __launch_bounds__(tc2::NTHREADS, 1)
mlp_tc2_kernel(const __grid_constant__ hr_config cfg, const __grid_constant__ MlpTcPack pk, const float* __restrict__ rays,
               float* __restrict__ heads, long long n_rays, float* __restrict__ rays_copy, const TrainSave sv) {
  using namespace tc2;
  constexpr int NACC = W / 2;                        // accumulator registers of one W-column pass
  constexpr int NK = W / 16;                         // k-steps of the hidden activation operand
  constexpr int IMG_BYTES = W * 64;                  // weight image of one k-step: W x 16 k, hi then lo
  constexpr int KPS = STAGE_BYTES / IMG_BYTES;       // k-steps per ring stage
  static_assert(KPS * IMG_BYTES == STAGE_BYTES && NK * KSTEP_BYTES <= A_BYTES, "pass width");
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  auto bar = [&](int slot) -> uint32_t { return sbase + OFF_BAR + slot * 8; };

  // ---- one-time setup ----
  {
    // pull the weight stream into L2 once (every CTA walks the same weights per tile; after a cold start the first walk
    // would otherwise pay DRAM latency on every ring stage)
    const char* w = reinterpret_cast<const char*>(pk.wpack);
    const long long lines = pk.wpack_bytes >> 7;
    for (long long i = (long long)blockIdx.x * NTHREADS + tid; i < lines; i += (long long)gridDim.x * NTHREADS)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(w + i * 128));
  }
  for (int i = tid; i < (2 * X_BYTES) / 16; i += NTHREADS)  // encoded-input operand: columns >= mlp_in stay zero
    reinterpret_cast<uint4*>(smem + OFF_X)[i] = make_uint4(0u, 0u, 0u, 0u);
  if (tid == 0) {
    for (int s = 0; s < NSTAGE; ++s) { mbar_init(bar(BAR_FULL + s), 1); mbar_init(bar(BAR_EMPTY + s), CONSUMERS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const long long n_tiles = (n_rays + BM - 1) / BM;
  const int n_passes = pk.n_passes;
  // tiles blockIdx.x, blockIdx.x + gridDim.x, ... : every role of this CTA runs exactly this many iterations
  const long long n_iters = ((long long)blockIdx.x < n_tiles) ? (n_tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;

  if (warp >= CONSUMERS * 4) {
    // =========================== producer: weight images, in consumption order ===========================
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == CONSUMERS * 4 && lane == 0) {
      const int n_stages = (int)(pk.wpack_bytes / STAGE_BYTES);  // every pass is a whole number of stages
      uint32_t stage = 0, phase = 0;
      for (long long iter = 0; iter < n_iters; ++iter) {
        const uint8_t* src = reinterpret_cast<const uint8_t*>(pk.wpack);
        for (int i = 0; i < n_stages; ++i) {
          mbar_wait(bar(BAR_EMPTY + stage), phase ^ 1);
          mbar_expect_tx(bar(BAR_FULL + stage), STAGE_BYTES);
          bulk_g2s(sbase + OFF_B + stage * STAGE_BYTES, src, STAGE_BYTES, bar(BAR_FULL + stage));
          src += STAGE_BYTES;
          if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // =========================== consumer warpgroups: 64 rays each ===========================
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = warp >> 2;                 // 0 .. CONSUMERS-1
  const int wt = tid & 127;                 // thread within the warpgroup
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // tile rows of accumulator elements (i / 2) % 2 == 0; +8 for 1
  const int q2 = (lane & 3) * 2;            // first of the two columns of an accumulator pair
  const int in_chunks = pk.in_chunks;
  const int L = cfg.mlp_layers;
  const uint32_t x_lo_off = (uint32_t)(2 * in_chunks * KSTEP_BYTES);  // lo half follows the hi k-steps
  const uint32_t rows_off = (uint32_t)wg * 1024u;                     // this warpgroup's 8 row groups of a k-step image
  const uint32_t full0 = bar(BAR_FULL), empty0 = bar(BAR_EMPTY);
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(rays) | reinterpret_cast<uintptr_t>(rays_copy)) & 15) == 0;
  uint32_t stage = 0, phase = 0;
  int pend = -1;  // ring stage whose wgmmas were committed but not yet waited for

  float acc[NACC];

  auto stage_begin = [&]() {
    mbar_wait(full0 + stage * 8, phase);
    wgmma_fence();
    acc_fence(acc);
  };
  // the ring stage of each k-step group is released one stage later, once its wgmmas have retired
  auto stage_end = [&]() {
    wgmma_commit();
    acc_fence(acc);
    wgmma_wait<1>();
    if (pend >= 0 && wt == 0) mbar_arrive(empty0 + pend * 8);
    pend = (int)stage;
    if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
  };
  auto b_img = [&](int sub) -> uint32_t { return sbase + OFF_B + stage * STAGE_BYTES + (uint32_t)sub * IMG_BYTES; };
  // one pass: acc = A(chunks of P) * B(P)^T, 3 wgmmas per k-step
  auto run_pass = [&](const TcPass& P) {
    int ki = 0;  // k-steps issued in this pass; the input's count (2 per chunk) is even, so a stage never straddles
    if (P.first_chunk == 0) {  // encoded input: hi and lo from shared memory
      for (; ki < 2 * in_chunks; ki += KPS) {
        stage_begin();
#pragma unroll
        for (int sub = 0; sub < KPS; ++sub) {
          const uint32_t a_hi = sbase + OFF_X + (uint32_t)(ki + sub) * KSTEP_BYTES + rows_off, b = b_img(sub);
          const uint64_t ah = gmma_desc(a_hi, 2048, 128), al = gmma_desc(a_hi + x_lo_off, 2048, 128);
          const uint64_t bh = gmma_desc(b, W * 16, 128), bl = gmma_desc(b + W * 32, W * 16, 128);
          wgmma_ss(acc, ah, bh, (ki + sub) != 0 ? 1u : 0u);
          wgmma_ss(acc, al, bh, 1u);
          wgmma_ss(acc, ah, bl, 1u);
        }
        stage_end();
      }
    }
    if (P.first_chunk + P.n_chunks > in_chunks) {  // hidden activation
      const uint32_t scale0 = ki != 0 ? 1u : 0u;
#pragma unroll
      for (int kk = 0; kk < NK; ++kk) {
        if (kk % KPS == 0) stage_begin();
        const uint32_t a_hi = sbase + OFF_AHI + (uint32_t)kk * KSTEP_BYTES + rows_off, b = b_img(kk % KPS);
        const uint64_t ah = gmma_desc(a_hi, 2048, 128), al = gmma_desc(a_hi + (OFF_ALO - OFF_AHI), 2048, 128);
        const uint64_t bh = gmma_desc(b, W * 16, 128), bl = gmma_desc(b + W * 32, W * 16, 128);
        wgmma_ss(acc, ah, bh, kk != 0 ? 1u : scale0);
        wgmma_ss(acc, al, bh, 1u);
        wgmma_ss(acc, ah, bl, 1u);
        if (kk % KPS == KPS - 1) stage_end();
      }
    }
  };
  auto drain = [&]() {
    wgmma_wait<0>();
    acc_fence(acc);
    if (pend >= 0 && wt == 0) mbar_arrive(empty0 + pend * 8);
    pend = -1;
  };
  // hidden epilogue: A(l+1) = LeakyReLU(acc + bias), split into hi / lo.  The accumulator fragment of columns 8 j .. 8 j + 7
  // and rows 8 h .. 8 h + 7 of the warp is an 8x8 stmatrix fragment, and its destination rows are 16-byte core-matrix
  // rows of A, so one stmatrix.x4 writes a whole 16-wide k-step of the warp's 16 rows: matrix i = 2 (j % 2) + h, lane t
  // addresses row t % 8 of matrix t / 8.
  const int st_row = wg * 64 + (warp & 3) * 16 + 8 * ((lane >> 3) & 1) + (lane & 7);
  const uint32_t st_off = ks_slot(st_row, lane >> 4);
  auto store_hidden = [&](const float* bias, int layer, long long tile) {
#pragma unroll
    for (int m = 0; m < W / 16; ++m) {
      uint32_t hi[4], lo[4];
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const int j = 2 * m + jj, k = 8 * j + q2;
        const float2 b = __ldg(reinterpret_cast<const float2*>(bias + k));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float t0 = acc[4 * j + 2 * h] + b.x, t1 = acc[4 * j + 2 * h + 1] + b.y;
          t0 = fmaxf(t0, t0 * cfg.leaky_slope);  // LeakyReLU, slope in (0,1)
          t1 = fmaxf(t1, t1 * cfg.leaky_slope);
          split2(t0, t1, hi[2 * jj + h], lo[2 * jj + h]);
          if constexpr (SAVE) {
            const long long ray = tile * BM + row0 + 8 * h;
            if (ray < n_rays) *reinterpret_cast<float2*>(sv.act + layer * sv.act_stride + ray * W + k) = make_float2(t0, t1);
          }
        }
      }
      const uint32_t a = sbase + st_off + (uint32_t)m * KSTEP_BYTES;
      stmatrix_x4(a + OFF_AHI, hi);
      stmatrix_x4(a + OFF_ALO, lo);
    }
  };

  for (long long iter = 0; iter < n_iters; ++iter) {
    const long long tile = iter * gridDim.x + blockIdx.x;
    // ---- RayParam + WindowedPE of this warpgroup's 64 rays, two threads per ray, straight into the bf16 hi / lo slots ----
    {
      const int r = wg * 64 + (wt & 63), part = wt >> 6;
      const long long ray = tile * BM + r;
      auto put = [&](int k, float val) {
        if constexpr (SAVE) {
          if (ray < n_rays) sv.enc[ray * sv.ld_enc + k] = val;
        }
        const __nv_bfloat16 hi = __float2bfloat16_rn(val);
        const __nv_bfloat16 lo = __float2bfloat16_rn(val - __bfloat162float(hi));
        const uint32_t off = (uint32_t)(k >> 4) * KSTEP_BYTES + ks_slot(r, (k >> 3) & 1) + (uint32_t)(k & 7) * 2u;
        *reinterpret_cast<__nv_bfloat16*>(smem + OFF_X + off) = hi;
        *reinterpret_cast<__nv_bfloat16*>(smem + OFF_X + x_lo_off + off) = lo;
      };
      if (ray < n_rays) {
        // `rays` may be pinned host memory (zero-copy input of hr_render_host): each ray is read once per thread, with
        // vector loads, and `rays_copy` receives the device copy the render kernel reads.
        float rbuf[16];
        const float* src = rays + ray * cfg.c_in;
        if (cfg.c_in == 8 && vec_ok) {
          const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
          rbuf[0] = a.x; rbuf[1] = a.y; rbuf[2] = a.z; rbuf[3] = a.w; rbuf[4] = b.x; rbuf[5] = b.y; rbuf[6] = b.z; rbuf[7] = b.w;
          if (rays_copy != nullptr && part == 0) {
            float4* dst = reinterpret_cast<float4*>(rays_copy + ray * 8);
            dst[0] = a; dst[1] = b;
          }
        } else {
          for (int i = 0; i < cfg.c_in; ++i) rbuf[i] = src[i];
          if (rays_copy != nullptr && part == 0)
            for (int i = 0; i < cfg.c_in; ++i) rays_copy[ray * cfg.c_in + i] = rbuf[i];
        }
        encode_ray_features(cfg, rbuf, part, 2, put);
        if constexpr (SAVE) {
          if (part == 0)
            for (int k = cfg.mlp_in; k < sv.ld_enc; ++k) sv.enc[ray * sv.ld_enc + k] = 0.0f;  // the padding the dW GEMM reads
        }
      } else if (part == 0) {
        for (int k = 0; k < cfg.mlp_in; ++k) put(k, 0.0f);  // masked row: defined (never stored) values
      }
      fence_async_smem();
      wg_sync(1 + wg);
    }
    // ---- the hidden layers: one pass each (passes[l] is layer l) ----
    for (int l = 0; l < L - 1; ++l) {
      run_pass(pk.passes[l]);
      drain();
      wg_sync(1 + wg);  // every warp's wgmmas that read A(l) have retired before A(l+1) overwrites it
      store_hidden(pk.bias + pk.passes[l].bias_off, l, tile);
      fence_async_smem();
      wg_sync(1 + wg);
    }
    // ---- last layer: accumulators + bias -> heads scratch (rows past n_rays / columns past mlp_out are dropped) ----
    for (int p = L - 1; p < n_passes; ++p) {
      const TcPass& P = pk.passes[p];
      run_pass(P);
      drain();
      const float* bias = pk.bias + P.bias_off;
      if constexpr (SAVE) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long ray = tile * BM + row0 + 8 * h;
          if (ray >= n_rays) continue;
          float* row = heads + ray * cfg.mlp_out;
#pragma unroll
          for (int j = 0; j < W / 8; ++j) {
            const int c = 8 * j + q2;
            if (P.out_col0 + c < cfg.mlp_out) {  // mlp_out is a multiple of 4: the pair is in or out as a whole
              const float2 b = __ldg(reinterpret_cast<const float2*>(bias + c));
              // channel-major column c*S+s -> the reference's s*stride+c
              const int c0 = P.out_col0 + c, c1 = c0 + 1, S = cfg.n_samples;
              row[(c0 % S) * cfg.head_stride + c0 / S] = acc[4 * j + 2 * h] + b.x;
              row[(c1 % S) * cfg.head_stride + c1 / S] = acc[4 * j + 2 * h + 1] + b.y;
            }
          }
        }
      } else {
        // Lanes 2i and 2i + 1 hold 4 consecutive columns of the same row in column groups j and j + 1: they swap one pair
        // so that each stores 4 consecutive columns with one 16-byte store (the even lane in group j, the odd one in
        // group j + 1).  mlp_out is a multiple of 4, so the 4 columns are in or out as a whole.
        const bool odd = (lane & 1) != 0;
#pragma unroll
        for (int jp = 0; jp < W / 16; ++jp) {
          const int j = 2 * jp, c = 8 * j + q2;
          const float2 b0 = __ldg(reinterpret_cast<const float2*>(bias + c));
          const float2 b1 = __ldg(reinterpret_cast<const float2*>(bias + c + 8));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float2 v0 = make_float2(acc[4 * j + 2 * h] + b0.x, acc[4 * j + 2 * h + 1] + b0.y);
            const float2 v1 = make_float2(acc[4 * j + 4 + 2 * h] + b1.x, acc[4 * j + 4 + 2 * h + 1] + b1.y);
            const float2 send = odd ? v0 : v1;
            const float2 recv = make_float2(__shfl_xor_sync(0xffffffffu, send.x, 1), __shfl_xor_sync(0xffffffffu, send.y, 1));
            const int c4 = odd ? c + 6 : c;  // first of the lane's 4 columns
            const long long ray = tile * BM + row0 + 8 * h;
            if (ray < n_rays && P.out_col0 + c4 < cfg.mlp_out)
              *reinterpret_cast<float4*>(heads + ray * cfg.mlp_out + P.out_col0 + c4) =
                  odd ? make_float4(recv.x, recv.y, v1.x, v1.y) : make_float4(v0.x, v0.y, recv.x, recv.y);
          }
        }
      }
    }
  }
}

// Pass table + weight images (format: hr_tc_pack.cu).  Called by hr_upload with the handle's device current.
int pack_mlp_tc2(hr_handle* h, const hr_config& c, MlpTcPack& pk, size_t& alloc_bytes, int& alloc_bias,
                 const float* const* w_dev, const float* const* b_dev, cudaStream_t st) {
  const int W = c.mlp_width;
  if (W != 128 && W != 256) return hr_fail("tensor-core sample net: hidden width must be 128 or 256 (got %d)", W);
  if (c.mlp_in > 64) return hr_fail("tensor-core sample net: encoded input wider than 64 features (%d)", c.mlp_in);
  const int in_chunks = (c.mlp_in + 31) / 32;
  const int L = c.mlp_layers;
  // the layout is a pure function of the config: when a pack of the same layout exists only its contents are rewritten
  // (no cudaFree / cudaMalloc on a parameter refresh -- needed once per optimiser step by the training path)
  MlpTcPack np_{};
  np_.in_chunks = in_chunks;
  int np = 0, bias_off = 0;
  size_t bytes = 0;
  for (int l = 0; l < L; ++l) {
    const bool last = (l == L - 1);
    const int out = last ? c.mlp_out : W;
    const int n_parts = (out + W - 1) / W;  // one pass per hidden layer
    for (int part = 0; part < n_parts; ++part) {
      if (np >= HR_TC_MAX_PASSES) return hr_fail("tensor-core sample net: too many passes (%d output columns)", c.mlp_out);
      TcPass& P = np_.passes[np++];
      const bool reads_input = (l == 0 || l == c.mlp_skip);
      P.layer = l;
      P.n = W;  // a partial last pass is zero padded
      P.first_chunk = reads_input ? 0 : in_chunks;
      P.n_chunks = (l == 0) ? in_chunks : (W / 32 + (reads_input ? in_chunks : 0));
      P.bias_off = bias_off;
      P.is_final = last ? 1 : 0;
      P.out_col0 = part * W;
      P.wait_a = (part == 0) ? 1 : 0;
      bias_off += P.n;
      bytes += (size_t)P.n_chunks * 2 * P.n * 64;
    }
  }
  np_.n_passes = np;
  np_.bias_count = bias_off;
  np_.wpack_bytes = (long long)bytes;
  if (alloc_bytes != bytes || alloc_bias != bias_off || !pk.wpack) {
    if (pk.wpack) cudaFree(const_cast<void*>(pk.wpack));
    if (pk.bias) cudaFree(const_cast<float*>(pk.bias));
    pk.wpack = nullptr; pk.bias = nullptr;
    alloc_bytes = 0; alloc_bias = 0;
    void* wp = nullptr; float* bp = nullptr;
    cudaError_t e = cudaMalloc(&wp, bytes);
    if (e != cudaSuccess) return hr_fail("cudaMalloc(tc weights %zu): %s", bytes, cudaGetErrorString(e));
    e = cudaMalloc((void**)&bp, (size_t)bias_off * sizeof(float));
    if (e != cudaSuccess) { cudaFree(wp); return hr_fail("cudaMalloc(tc bias): %s", cudaGetErrorString(e)); }
    np_.wpack = wp; np_.bias = bp;
    alloc_bytes = bytes; alloc_bias = bias_off;
    // opt in to the 224 KB of dynamic shared memory once per (handle, device)
    e = (W == 256) ? cudaFuncSetAttribute(mlp_tc2_kernel<256, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc2::SMEM_BYTES)
                   : cudaFuncSetAttribute(mlp_tc2_kernel<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc2::SMEM_BYTES);
    if (e != cudaSuccess) return hr_fail("cudaFuncSetAttribute(mlp_tc2_kernel): %s", cudaGetErrorString(e));
  } else {
    np_.wpack = pk.wpack; np_.bias = pk.bias;
  }
  pk = np_;
  uint8_t* wp = (uint8_t*)const_cast<void*>(pk.wpack);
  float* bp = const_cast<float*>(pk.bias);
  size_t off = 0;
  for (int p = 0; p < np; ++p) {
    const TcPass& P = pk.passes[p];
    const int l = P.layer;
    const bool last = (l == L - 1), skip = (l == c.mlp_skip), first = (l == 0);
    const int in_src = first ? c.mlp_in : (skip ? c.mlp_in + W : W);
    launch_pack_tc_pass(w_dev[l], b_dev[l], wp + off, bp + P.bias_off, P.n, P.first_chunk, P.n_chunks, in_src, c.mlp_in,
                        skip ? 1 : 0, in_chunks, last ? c.mlp_out : W, last ? c.n_samples : 0, c.head_stride, P.out_col0, st);
    off += (size_t)P.n_chunks * 2 * P.n * 64;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return hr_fail("tc pack launch failed: %s", cudaGetErrorString(e));
  return 0;
}

void free_mlp_tc2(hr_handle* h) {
  if (h->tc.wpack) cudaFree(const_cast<void*>(h->tc.wpack));
  if (h->tc.bias) cudaFree(const_cast<float*>(h->tc.bias));
  h->tc.wpack = nullptr; h->tc.bias = nullptr;
  h->tc_alloc_bytes = 0; h->tc_alloc_bias = 0;
  if (h->tc_pre.wpack) cudaFree(const_cast<void*>(h->tc_pre.wpack));
  if (h->tc_pre.bias) cudaFree(const_cast<float*>(h->tc_pre.bias));
  h->tc_pre.wpack = nullptr; h->tc_pre.bias = nullptr;
  h->tc_pre_alloc_bytes = 0; h->tc_pre_alloc_bias = 0;
}

cudaError_t launch_mlp_tc2(const hr_config& cfg, const MlpTcPack& pk, const float* rays, float* heads, long long n, int num_sms,
                           cudaStream_t stream, float* rays_copy) {
  // the epilogue stores column pairs and drops a pair past mlp_out as a whole
  if ((cfg.mlp_out % 4) != 0 || ((uintptr_t)heads % 16) != 0) return cudaErrorInvalidValue;
  long long tiles = (n + tc::BM - 1) / tc::BM;
  int grid = (int)(tiles < num_sms ? tiles : num_sms);
  if (grid < 1) grid = 1;
  if (cfg.mlp_width == 256)
    mlp_tc2_kernel<256, false><<<grid, tc2::NTHREADS, tc2::SMEM_BYTES, stream>>>(cfg, pk, rays, heads, n, rays_copy, TrainSave{});
  else if (cfg.mlp_width == 128)
    mlp_tc2_kernel<128, false><<<grid, tc2::NTHREADS, tc2::SMEM_BYTES, stream>>>(cfg, pk, rays, heads, n, rays_copy, TrainSave{});
  else
    return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_mlp_tc2_train(const hr_config& cfg, const MlpTcPack& pk, const float* rays, float* heads, long long n,
                                 int num_sms, cudaStream_t stream, const TrainSave& sv) {
  if ((cfg.mlp_out % 4) != 0) return cudaErrorInvalidValue;
  long long tiles = (n + tc::BM - 1) / tc::BM;
  int grid = (int)(tiles < num_sms ? tiles : num_sms);
  if (grid < 1) grid = 1;
  auto kern = cfg.mlp_width == 256 ? mlp_tc2_kernel<256, true> : mlp_tc2_kernel<128, true>;
  if (cfg.mlp_width != 256 && cfg.mlp_width != 128) return cudaErrorInvalidValue;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, tc2::SMEM_BYTES);
  if (e != cudaSuccess) return e;
  kern<<<grid, tc2::NTHREADS, tc2::SMEM_BYTES, stream>>>(cfg, pk, rays, heads, n, nullptr, sv);
  return cudaGetLastError();
}

}  // namespace hr
