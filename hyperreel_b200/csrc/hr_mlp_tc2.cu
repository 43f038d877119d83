// Sample-prediction network on the Hopper tensor cores (HR_MLP_BF16X3_TC, and HR_MLP_FP16_TC: F16 below), wgmma.
//
// Math (reference: nlf/nets/mlp.py:159-172 behind nlf/embedding/ray.py:320-326): every fp32 operand x is split into
// bf16 hi = rn(x) and lo = rn(x - hi) and each Linear layer is
//     D = A_hi*B_hi + A_lo*B_hi + A_hi*B_lo          (three wgmma k16 products per k-step and output element, in this
//                                                      order, k-steps ascending, fp32 accumulation in registers);
// the dropped A_lo*B_lo term and the split residuals are O(2^-16) relative per product (DESIGN.md).
// Hidden width W = 128 or 256 (a template parameter), encoded input up to 64 features (one or two 32-wide input chunks).
//
// Layout (one persistent CTA per SM, one 128-ray tile at a time):
//   * every Linear layer is issued as passes of W output columns (a hidden layer is one pass, the last layer
//     ceil(out / W) zero-padded passes), and warpgroup g computes columns [g W/2, (g + 1) W/2) of every pass for all
//     128 rays: two m64n(W/2)k16 accumulators (rows 0-63 and 64-127, 128 registers at W = 256);
//   * each warpgroup has its own weight ring: warp g of the producer warpgroup streams that warpgroup's column half of
//     the weight images (bf16 hi + lo, consumption order, hr_tc_pack.cu) through 4 cp.async.bulk stages of 8 KB (one
//     k-step at W = 256) guarded by mbarriers, so every weight byte is loaded once per tile and the warpgroups are not
//     tied to each other's progress by the ring;
//   * the activation operand A (hi and lo, 2 x 64 KB at W = 256, K-major no-swizzle) is rewritten in place: warpgroup
//     g's epilogue writes the k-steps that hold its own column half.  Both warpgroups read all of A, so the two are
//     ordered by named barriers (pair_arrive / pair_wait): an epilogue overwrites its half only once the other
//     warpgroup's wgmmas that read the previous contents have retired (NB_RET), and a pass reads the other half only
//     once the other epilogue has written it (NB_WR).  Warpgroup 0 reads its own half first and announces its epilogue
//     only when it is half way through the next pass, so warpgroup 1 runs half a layer behind: each warpgroup's
//     epilogue runs while the other one issues wgmmas alone;
//   * the encoded input X (rows of both warpgroups, read by layer 0 and the skip layer) has the same two kinds of
//     signal (NB_XW, NB_XR); the next tile is encoded as soon as both warpgroups are past the last pass that reads X.
// The last layer's columns go from the accumulators (+ bias) straight to the heads scratch in global memory, 4 consecutive
// columns per 16-byte store (NARROW: 8- or 4-byte stores, for rows that are not 16-byte aligned); the hidden epilogues write
// the activation operand with stmatrix.
//
// F16 (HR_MLP_FP16_TC, inference only): what CUDA autocast computes for each F.linear -- the operands rounded to fp16, one
// wgmma product per k-step (.f32.f16.f16, fp32 accumulation), the fp16 bias added and the sum rounded once to fp16, LeakyReLU
// on that fp16 value (a negative one rounded again after x * slope).  One operand image (no lo half of A, X or the weights),
// so the shared-memory map and ring stages differ (tc2::Layout<true>); the last layer's fp16 values go to the heads as fp32.
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

constexpr int KSTEP_BYTES = 4096;    // activation k-step image: 128 rays x 16 k bf16 (or fp16)
constexpr int CONSUMERS = 2;         // warpgroups of W/2 output columns
constexpr int NTHREADS = (CONSUMERS + 1) * 128;  // + the producer warpgroup (lane 0 of its first two warps issues the copies)
// register split of the 64 K registers (setmaxnreg): the producer warpgroup gives up what the consumers need beside their
// 128 accumulator registers at W = 256
constexpr int PRODUCER_REGS = 40;
constexpr int CONSUMER_REGS = 232;
static_assert(128 * PRODUCER_REGS + CONSUMERS * 128 * CONSUMER_REGS <= 65536, "register file");

// Shared memory map (bytes) and weight ring.  bf16x3: the activation operand A and the encoded input X as hi then lo images,
// rings of 4 stages of 8 KB (k-step weight images of W/2 x 16 k x (hi + lo) bf16, 1 at W = 256 or 2 at W = 128 per stage).
// F16: A and X as one fp16 image each, rings of 8 stages of 4 KB (the same k-steps per stage, each image half the size).
template <bool F16>
struct Layout {
  static constexpr int PARTS = F16 ? 1 : 2;                   // operand images per k-step: hi (+ lo)
  static constexpr int NSTAGE = F16 ? 8 : 4;                  // depth of each warpgroup's weight ring
  static constexpr int STAGE_BYTES = F16 ? 4096 : 8192;       // one ring stage
  static constexpr int A_BYTES = 16 * KSTEP_BYTES;            // 64 KB: one image (hi or lo) of the activation operand
  static constexpr int OFF_AHI = 0;
  static constexpr int OFF_ALO = OFF_AHI + A_BYTES;           // bf16x3 only
  static constexpr int X_BYTES = 4 * KSTEP_BYTES;             // encoded input: up to 4 k-steps (64 k) hi, then as many lo
  static constexpr int OFF_X = PARTS * A_BYTES;               // 131072 (F16: 65536)
  static constexpr int OFF_B = OFF_X + PARTS * X_BYTES;       // 163840 (81920): ring of warpgroup 0, then of warpgroup 1
  static constexpr int OFF_BAR = OFF_B + CONSUMERS * NSTAGE * STAGE_BYTES;  // 229376 (147456)
  static constexpr int BAR_BYTES = 2 * CONSUMERS * NSTAGE * 8;              // 128 (256)
  static constexpr int SMEM_BYTES = OFF_BAR + BAR_BYTES;      // 229504 (147712) of 232448 available
  // barrier slots (8 bytes each) inside OFF_BAR
  static constexpr int BAR_FULL = 0;                               // [CONSUMERS][NSTAGE]
  static constexpr int BAR_EMPTY = BAR_FULL + CONSUMERS * NSTAGE;  // [CONSUMERS][NSTAGE]
  static_assert(SMEM_BYTES <= 232448, "shared memory budget");
};

// named barriers: 1 + g is warpgroup g's own (wg_sync); id + g below is a signal from warpgroup g to the other one
constexpr int NB_RET = 3;  // g's wgmmas that read the other warpgroup's half of A have retired: that half may be rewritten
constexpr int NB_WR = 5;   // g's half of A holds the next layer's input
constexpr int NB_XW = 7;   // g's rows of the encoded input are written
constexpr int NB_XR = 9;   // g's wgmmas that read the encoded input have retired: the next tile may be encoded

}  // namespace tc2

// NARROW: the heads rows of the render net (SAVE = false) are stored with 8- or 4-byte stores, each column guarded, for an
// mlp_out that is not a multiple of 4 or a heads pointer that is not 16-byte aligned (launch_mlp_tc2 picks it).
template <int W, bool SAVE, bool NARROW, bool F16 = false>
__global__ void __launch_bounds__(tc2::NTHREADS, 1)
mlp_tc2_kernel(const __grid_constant__ hr_config cfg, const __grid_constant__ MlpTcPack pk, const float* __restrict__ rays,
               float* __restrict__ heads, long long n_rays, float* __restrict__ rays_copy, const TrainSave sv) {
  using namespace tc2;
  static_assert(!(F16 && SAVE), "the training forward is bf16x3 only");
  using Lay = Layout<F16>;
  constexpr int NSTAGE = Lay::NSTAGE, STAGE_BYTES = Lay::STAGE_BYTES, OFF_AHI = Lay::OFF_AHI, OFF_ALO = Lay::OFF_ALO;
  constexpr int X_BYTES = Lay::X_BYTES, OFF_X = Lay::OFF_X, OFF_B = Lay::OFF_B, OFF_BAR = Lay::OFF_BAR;
  constexpr int BAR_FULL = Lay::BAR_FULL, BAR_EMPTY = Lay::BAR_EMPTY;
  constexpr int WH = W / 2;                          // output columns of one warpgroup
  constexpr int NACC = WH / 2;                       // registers of one m64nWH accumulator
  constexpr int NK = W / 16;                         // k-steps of the hidden activation operand
  constexpr int NKH = NK / 2;                        // k-steps holding one column half
  constexpr int IMG_BYTES = WH * 32 * Lay::PARTS;    // weight image of one k-step of a column half: WH x 16 k, hi (then lo)
  constexpr int KPS = STAGE_BYTES / IMG_BYTES;       // k-steps per ring stage
  static_assert(KPS * IMG_BYTES == STAGE_BYTES && NKH % KPS == 0 && NK * KSTEP_BYTES <= Lay::A_BYTES, "pass width");
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
  for (int i = tid; i < (Lay::PARTS * X_BYTES) / 16; i += NTHREADS)  // encoded-input operand: columns >= mlp_in stay zero
    reinterpret_cast<uint4*>(smem + OFF_X)[i] = make_uint4(0u, 0u, 0u, 0u);
  if (tid == 0) {
    for (int s = 0; s < CONSUMERS * NSTAGE; ++s) { mbar_init(bar(BAR_FULL + s), 1); mbar_init(bar(BAR_EMPTY + s), 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const long long n_tiles = (n_rays + BM - 1) / BM;
  const int n_passes = pk.n_passes;
  // tiles blockIdx.x, blockIdx.x + gridDim.x, ... : every role of this CTA runs exactly this many iterations
  const long long n_iters = ((long long)blockIdx.x < n_tiles) ? (n_tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;

  if (warp >= CONSUMERS * 4) {
    // ============ producer: warp g feeds warpgroup g's ring with its column half, in consumption order ============
    setmaxnreg_dec<PRODUCER_REGS>();
    const int g = warp - CONSUMERS * 4;
    if (g < CONSUMERS && lane == 0) {
      const long long half_bytes = pk.wpack_bytes / CONSUMERS;  // the pack holds all of half 0, then all of half 1
      const int n_stages = (int)(half_bytes / STAGE_BYTES);     // every pass is a whole number of stages
      const uint32_t full0 = bar(BAR_FULL + g * NSTAGE), empty0 = bar(BAR_EMPTY + g * NSTAGE);
      const uint32_t ring = sbase + OFF_B + (uint32_t)(g * NSTAGE * STAGE_BYTES);
      uint32_t stage = 0, phase = 0;
      for (long long iter = 0; iter < n_iters; ++iter) {
        const uint8_t* src = reinterpret_cast<const uint8_t*>(pk.wpack) + g * half_bytes;
        for (int i = 0; i < n_stages; ++i) {
          mbar_wait(empty0 + stage * 8, phase ^ 1);
          mbar_expect_tx(full0 + stage * 8, STAGE_BYTES);
          bulk_g2s(ring + stage * STAGE_BYTES, src, STAGE_BYTES, full0 + stage * 8);
          src += STAGE_BYTES;
          if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // =========================== consumer warpgroups: W/2 output columns each ===========================
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = warp >> 2;                 // 0 .. CONSUMERS-1
  const int wt = tid & 127;                 // thread within the warpgroup
  const int rowq = (warp & 3) * 16 + (lane >> 2);  // row (within an M half) of accumulator elements (i / 2) % 2 == 0; +8 for 1
  const int q2 = (lane & 3) * 2;            // first of the two columns of an accumulator pair
  const int col0 = wg * WH;                 // first output column of this warpgroup within a pass
  const int in_chunks = pk.in_chunks;
  const int L = cfg.mlp_layers;
  const uint32_t x_lo_off = (uint32_t)(2 * in_chunks * KSTEP_BYTES);  // lo half follows the hi k-steps
  const uint32_t full0 = bar(BAR_FULL + wg * NSTAGE), empty0 = bar(BAR_EMPTY + wg * NSTAGE);
  const uint32_t ring = sbase + OFF_B + (uint32_t)(wg * NSTAGE * STAGE_BYTES);
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(rays) | reinterpret_cast<uintptr_t>(rays_copy)) & 15) == 0;
  int x_last = 0;  // the last pass that reads the encoded input (layer 0's, or the skip layer's)
  for (int p = 0; p < n_passes; ++p)
    if (pk.passes[p].first_chunk == 0) x_last = p;
  uint32_t stage = 0, phase = 0;
  int pend = -1;  // ring stage whose wgmmas were committed but not yet waited for

  float acc[2][NACC];  // rows 0-63 and 64-127 of the tile

  auto stage_begin = [&]() {
    mbar_wait(full0 + stage * 8, phase);
    wgmma_fence();
    acc_fence(acc[0]);
    acc_fence(acc[1]);
  };
  // the ring stage of each k-step group is released one stage later, once its wgmmas have retired
  auto stage_end = [&]() {
    wgmma_commit();
    acc_fence(acc[0]);
    acc_fence(acc[1]);
    wgmma_wait<1>();
    if (pend >= 0 && wt == 0) mbar_arrive(empty0 + pend * 8);
    pend = (int)stage;
    if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
  };
  auto b_img = [&](int sub) -> uint32_t { return ring + stage * STAGE_BYTES + (uint32_t)sub * IMG_BYTES; };
  // one k-step: the three products for both M halves (a: hi k-step image of all 128 rows, its lo image a_lo bytes later);
  // F16: the one fp16 product
  auto kstep = [&](uint32_t a, uint32_t a_lo, uint32_t b, uint32_t scale) {
    if constexpr (F16) {
      const uint64_t bh = gmma_desc(b, WH * 16, 128);
      const uint64_t ah0 = gmma_desc(a, 2048, 128), ah1 = gmma_desc(a + 1024, 2048, 128);
      wgmma_ss<true>(acc[0], ah0, bh, scale);
      wgmma_ss<true>(acc[1], ah1, bh, scale);
    } else {
      const uint64_t bh = gmma_desc(b, WH * 16, 128), bl = gmma_desc(b + WH * 32, WH * 16, 128);
      const uint64_t ah0 = gmma_desc(a, 2048, 128), ah1 = gmma_desc(a + 1024, 2048, 128);
      const uint64_t al0 = gmma_desc(a + a_lo, 2048, 128), al1 = gmma_desc(a + a_lo + 1024, 2048, 128);
      wgmma_ss(acc[0], ah0, bh, scale);
      wgmma_ss(acc[1], ah1, bh, scale);
      wgmma_ss(acc[0], al0, bh, 1u);
      wgmma_ss(acc[1], al1, bh, 1u);
      wgmma_ss(acc[0], ah0, bl, 1u);
      wgmma_ss(acc[1], ah1, bl, 1u);
    }
  };
  // One pass: acc = A(chunks of P) * B(P)^T.  fresh: the first pass that reads the A an epilogue just wrote; x_ret /
  // ret: signal NB_XR / NB_RET as soon as the reads of X / of the other warpgroup's half of A have retired (warpgroup 1
  // reads that half first, so its signal comes mid-pass; warpgroup 0's comes after the pass, from the caller).
  auto run_pass = [&](const TcPass& P, bool fresh, bool x_ret, bool ret) {
    int ki = 0;  // k-steps issued in this pass; the input's count (2 per chunk) is even, so a stage never straddles
    if (P.first_chunk == 0) {  // encoded input: hi and lo from shared memory
      for (; ki < 2 * in_chunks; ki += KPS) {
        stage_begin();
#pragma unroll
        for (int sub = 0; sub < KPS; ++sub)
          kstep(sbase + OFF_X + (uint32_t)(ki + sub) * KSTEP_BYTES, x_lo_off, b_img(sub), (ki + sub) != 0 ? 1u : 0u);
        stage_end();
      }
    }
    if (P.first_chunk + P.n_chunks > in_chunks) {  // hidden activation
      const uint32_t scale0 = ki != 0 ? 1u : 0u;
#pragma unroll
      for (int kk = 0; kk < NK; ++kk) {
        if (kk % KPS == 0) {
          if (fresh && kk == (wg == 0 ? NKH : 0)) {  // first k-step of the other warpgroup's half
            if (wg == 0) pair_arrive(NB_WR + 0);     // warpgroup 0's half was written before this pass began
            pair_wait(NB_WR + (wg ^ 1));
          }
          stage_begin();
        }
        kstep(sbase + OFF_AHI + (uint32_t)kk * KSTEP_BYTES, OFF_ALO - OFF_AHI, b_img(kk % KPS), kk != 0 ? 1u : scale0);
        if (kk % KPS == KPS - 1) {
          stage_end();  // every stage before this one has retired
          if (x_ret && kk == KPS - 1) pair_arrive(NB_XR + wg);
          if (ret && wg == 1 && kk == NKH + KPS - 1) pair_arrive(NB_RET + 1);
        }
      }
    }
  };
  auto drain = [&]() {
    wgmma_wait<0>();
    acc_fence(acc[0]);
    acc_fence(acc[1]);
    if (pend >= 0 && wt == 0) mbar_arrive(empty0 + pend * 8);
    pend = -1;
  };
  // hidden epilogue: this warpgroup's columns of A(l+1) = LeakyReLU(acc + bias), split into hi / lo (F16: LeakyReLU of
  // rn16(acc + bias), rounded to fp16 again).  The accumulator
  // fragment of columns 8 j .. 8 j + 7 and rows 8 h .. 8 h + 7 of the warp is an 8x8 stmatrix fragment, and its
  // destination rows are 16-byte core-matrix rows of A, so one stmatrix.x4 writes a whole 16-wide k-step of the warp's 16
  // rows: matrix i = 2 (j % 2) + h, lane t addresses row t % 8 of matrix t / 8.
  const int st_row = (warp & 3) * 16 + 8 * ((lane >> 3) & 1) + (lane & 7);
  const uint32_t st_off = ks_slot(st_row, lane >> 4);  // rows 64-127: + 1024
  auto store_hidden = [&](const float* bias, int layer, long long tile) {
#pragma unroll
    for (int kk = 0; kk < NKH; ++kk) {
      float2 b[2];
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) b[jj] = __ldg(reinterpret_cast<const float2*>(bias + col0 + 8 * (2 * kk + jj) + q2));
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        uint32_t hi[4], lo[4];
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const int j = 2 * kk + jj, k = col0 + 8 * j + q2;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float t0 = acc[m][4 * j + 2 * h] + b[jj].x, t1 = acc[m][4 * j + 2 * h + 1] + b[jj].y;
            if constexpr (F16) {
              t0 = rn16(t0);
              t1 = rn16(t1);
            }
            t0 = fmaxf(t0, t0 * cfg.leaky_slope);  // LeakyReLU, slope in (0,1)
            t1 = fmaxf(t1, t1 * cfg.leaky_slope);
            if constexpr (F16)
              hi[2 * jj + h] = pack_half2(t0, t1);
            else
              split2(t0, t1, hi[2 * jj + h], lo[2 * jj + h]);
            if constexpr (SAVE) {
              const long long ray = tile * BM + 64 * m + rowq + 8 * h;
              if (ray < n_rays) *reinterpret_cast<float2*>(sv.act + layer * sv.act_stride + ray * W + k) = make_float2(t0, t1);
            }
          }
        }
        const uint32_t a = sbase + st_off + (uint32_t)m * 1024u + (uint32_t)(wg * NKH + kk) * KSTEP_BYTES;
        stmatrix_x4(a + OFF_AHI, hi);
        if constexpr (!F16) stmatrix_x4(a + OFF_ALO, lo);
      }
    }
  };
  // RayParam + WindowedPE of this warpgroup's 64 rays (tile rows 64 wg ..), two threads per ray, straight into the bf16
  // hi / lo slots of X (F16: its fp16 slots); after_x: X still holds the previous tile, wait until the other warpgroup's
  // reads of it retired
  auto encode = [&](long long tile, bool after_x) {
    if (after_x) pair_wait(NB_XR + (wg ^ 1));
    const int r = wg * 64 + (wt & 63), part = wt >> 6;
    const long long ray = tile * BM + r;
    auto put = [&](int k, float val) {
      if constexpr (SAVE) {
        if (ray < n_rays) sv.enc[ray * sv.ld_enc + k] = val;
      }
      if constexpr (F16) {
        const uint32_t off = (uint32_t)(k >> 4) * KSTEP_BYTES + ks_slot(r, (k >> 3) & 1) + (uint32_t)(k & 7) * 2u;
        *reinterpret_cast<__half*>(smem + OFF_X + off) = __float2half_rn(val);
      } else {
        const __nv_bfloat16 hi = __float2bfloat16_rn(val);
        const __nv_bfloat16 lo = __float2bfloat16_rn(val - __bfloat162float(hi));
        const uint32_t off = (uint32_t)(k >> 4) * KSTEP_BYTES + ks_slot(r, (k >> 3) & 1) + (uint32_t)(k & 7) * 2u;
        *reinterpret_cast<__nv_bfloat16*>(smem + OFF_X + off) = hi;
        *reinterpret_cast<__nv_bfloat16*>(smem + OFF_X + x_lo_off + off) = lo;
      }
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
    pair_arrive(NB_XW + wg);
  };

  for (long long iter = 0; iter < n_iters; ++iter) {
    const long long tile = iter * gridDim.x + blockIdx.x;
    const bool more = iter + 1 < n_iters;
    if (iter == 0) encode(tile, false);  // later tiles are encoded during the previous one (after its pass x_last)
    pair_wait(NB_XW + (wg ^ 1));         // the other warpgroup's rows of X
    for (int p = 0; p < n_passes; ++p) {
      const TcPass& P = pk.passes[p];
      const bool reads_a = P.first_chunk + P.n_chunks > in_chunks;
      const bool hidden = p < L - 1;  // passes[l] is hidden layer l
      // the other warpgroup's next epilogue (of this tile's next layer, or of the next tile's layer 0) waits for these
      // reads of its half of A
      const bool ret = reads_a && (hidden || (p == n_passes - 1 && more));
      const bool x_ret = p == x_last && more;
      run_pass(P, reads_a && P.wait_a != 0, x_ret, ret);
      drain();
      if (x_ret && !reads_a) pair_arrive(NB_XR + wg);
      if (ret && wg == 0) pair_arrive(NB_RET + 0);
      if (hidden) {
        wg_sync(1 + wg);  // every warp's wgmmas that read A(l) have retired before A(l+1) overwrites it
        if (p > 0 || iter > 0) pair_wait(NB_RET + (wg ^ 1));  // ... and the other warpgroup's reads of this half
        store_hidden(pk.bias + P.bias_off, p, tile);
        fence_async_smem();
        wg_sync(1 + wg);
        if (wg == 1) pair_arrive(NB_WR + 1);  // warpgroup 0 signals its half in the next pass (run_pass)
      } else {
        // ---- last layer: accumulators + bias -> heads scratch (rows past n_rays / columns past mlp_out are dropped) ----
        const float* bias = pk.bias + P.bias_off;
        auto out = [](float v) -> float {  // F16: the layer's fp16 result, stored as fp32
          if constexpr (F16) return rn16(v);
          return v;
        };
        if constexpr (SAVE) {
#pragma unroll
          for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const long long ray = tile * BM + 64 * m + rowq + 8 * h;
              if (ray >= n_rays) continue;
              float* row = heads + ray * cfg.mlp_out;
#pragma unroll
              for (int j = 0; j < WH / 8; ++j) {
                const int c = col0 + 8 * j + q2;
                if (P.out_col0 + c < cfg.mlp_out) {  // each column of the pair is guarded: mlp_out may be odd
                  const float2 b = __ldg(reinterpret_cast<const float2*>(bias + c));
                  // channel-major column c*S+s -> the reference's s*stride+c
                  const int c0 = P.out_col0 + c, c1 = c0 + 1, S = cfg.n_samples;
                  row[(c0 % S) * cfg.head_stride + c0 / S] = acc[m][4 * j + 2 * h] + b.x;
                  if (c1 < cfg.mlp_out) row[(c1 % S) * cfg.head_stride + c1 / S] = acc[m][4 * j + 2 * h + 1] + b.y;
                }
              }
            }
        } else if constexpr (NARROW) {
          // any mlp_out: a lane's column pair is one 8-byte store when every row starts 8-byte aligned, else two 4-byte
          // stores; a column past mlp_out is dropped on its own
          const bool pairs = (cfg.mlp_out % 2) == 0 && (reinterpret_cast<uintptr_t>(heads) & 7) == 0;
#pragma unroll
          for (int j = 0; j < WH / 8; ++j) {
            const int c = col0 + 8 * j + q2, c0 = P.out_col0 + c;
            const float2 b = __ldg(reinterpret_cast<const float2*>(bias + c));
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const long long ray = tile * BM + 64 * m + rowq + 8 * h;
                if (ray >= n_rays || c0 >= cfg.mlp_out) continue;
                float* dst = heads + ray * cfg.mlp_out + c0;
                const float v0 = out(acc[m][4 * j + 2 * h] + b.x), v1 = out(acc[m][4 * j + 2 * h + 1] + b.y);
                if (pairs) {
                  *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
                } else {
                  dst[0] = v0;
                  if (c0 + 1 < cfg.mlp_out) dst[1] = v1;
                }
              }
          }
        } else {
          // Lanes 2i and 2i + 1 hold 4 consecutive columns of the same row in column groups j and j + 1: they swap one pair
          // so that each stores 4 consecutive columns with one 16-byte store (the even lane in group j, the odd one in
          // group j + 1).  launch_mlp_tc2 runs this store only when mlp_out is a multiple of 4, so the 4 columns are in or
          // out as a whole.
          const bool odd = (lane & 1) != 0;
#pragma unroll
          for (int jp = 0; jp < WH / 16; ++jp) {
            const int j = 2 * jp, c = col0 + 8 * j + q2;
            const float2 b0 = __ldg(reinterpret_cast<const float2*>(bias + c));
            const float2 b1 = __ldg(reinterpret_cast<const float2*>(bias + c + 8));
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const float2 v0 = make_float2(out(acc[m][4 * j + 2 * h] + b0.x), out(acc[m][4 * j + 2 * h + 1] + b0.y));
                const float2 v1 = make_float2(out(acc[m][4 * j + 4 + 2 * h] + b1.x), out(acc[m][4 * j + 4 + 2 * h + 1] + b1.y));
                const float2 send = odd ? v0 : v1;
                const float2 recv = make_float2(__shfl_xor_sync(0xffffffffu, send.x, 1), __shfl_xor_sync(0xffffffffu, send.y, 1));
                const int c4 = odd ? c + 6 : c;  // first of the lane's 4 columns
                const long long ray = tile * BM + 64 * m + rowq + 8 * h;
                if (ray < n_rays && P.out_col0 + c4 < cfg.mlp_out)
                  *reinterpret_cast<float4*>(heads + ray * cfg.mlp_out + P.out_col0 + c4) =
                      odd ? make_float4(recv.x, recv.y, v1.x, v1.y) : make_float4(v0.x, v0.y, recv.x, recv.y);
              }
          }
        }
      }
      if (x_ret) encode(tile + gridDim.x, true);
    }
  }
}

// the inference kernel of a net: width 128 or 256 (anything else is 128: callers check), narrow heads stores, fp16 or bf16x3
using Tc2Kernel = void (*)(const hr_config, const MlpTcPack, const float*, float*, long long, float*, const TrainSave);
static Tc2Kernel tc2_kernel(int W, bool narrow, bool f16) {
  if (f16)
    return W == 256 ? (narrow ? mlp_tc2_kernel<256, false, true, true> : mlp_tc2_kernel<256, false, false, true>)
                    : (narrow ? mlp_tc2_kernel<128, false, true, true> : mlp_tc2_kernel<128, false, false, true>);
  return W == 256 ? (narrow ? mlp_tc2_kernel<256, false, true> : mlp_tc2_kernel<256, false, false>)
                  : (narrow ? mlp_tc2_kernel<128, false, true> : mlp_tc2_kernel<128, false, false>);
}
static int tc2_smem_bytes(bool f16) { return f16 ? tc2::Layout<true>::SMEM_BYTES : tc2::Layout<false>::SMEM_BYTES; }

// Pass table + weight images (format: hr_tc_pack.cu).  Called by hr_upload with the handle's device current.
int pack_mlp_tc2(SampleNet& net, const float* const* w_dev, const float* const* b_dev, cudaStream_t st) {
  const hr_config& c = net.cfg;
  MlpTcPack& pk = net.tc;
  size_t& alloc_bytes = net.tc_alloc_bytes;
  int& alloc_bias = net.tc_alloc_bias;
  const int W = c.mlp_width;
  const bool f16 = c.mlp_mode == HR_MLP_FP16_TC;
  const int img_bytes = f16 ? 32 : 64;  // bytes of one k-step image per output column: 16 k of fp16, or bf16 hi + lo
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
      bytes += (size_t)P.n_chunks * 2 * P.n * img_bytes;
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
    // opt in to the 224 KB (F16: 144 KB) of dynamic shared memory once per (handle, device)
    for (int narrow = 0; narrow < 2 && e == cudaSuccess; ++narrow)
      e = cudaFuncSetAttribute(tc2_kernel(W, narrow != 0, f16), cudaFuncAttributeMaxDynamicSharedMemorySize, tc2_smem_bytes(f16));
    if (e != cudaSuccess) return hr_fail("cudaFuncSetAttribute(mlp_tc2_kernel): %s", cudaGetErrorString(e));
  } else {
    np_.wpack = pk.wpack; np_.bias = pk.bias;
  }
  pk = np_;
  // two weight streams, one per consumer warpgroup: every pass's images of columns [0, W/2), then every pass's images of
  // columns [W/2, W), each a pass of W/2 columns in the format of hr_tc_pack.cu
  uint8_t* wp = (uint8_t*)const_cast<void*>(pk.wpack);
  float* bp = const_cast<float*>(pk.bias);
  const int WH = W / 2;
  for (int half = 0; half < 2; ++half) {
    size_t off = (size_t)half * (bytes / 2);
    for (int p = 0; p < np; ++p) {
      const TcPass& P = pk.passes[p];
      const int l = P.layer;
      const bool last = (l == L - 1), skip = (l == c.mlp_skip), first = (l == 0);
      const int in_src = first ? c.mlp_in : (skip ? c.mlp_in + W : W);
      launch_pack_tc_pass(w_dev[l], b_dev[l], wp + off, bp + P.bias_off + half * WH, WH, P.first_chunk, P.n_chunks, in_src,
                          c.mlp_in, skip ? 1 : 0, in_chunks, last ? c.mlp_out : W, last ? c.n_samples : 0, c.head_stride,
                          P.out_col0 + half * WH, f16 ? 1 : 0, st);
      off += (size_t)P.n_chunks * 2 * WH * img_bytes;
    }
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return hr_fail("tc pack launch failed: %s", cudaGetErrorString(e));
  return 0;
}

void free_mlp_tc2(SampleNet& net) {
  if (net.tc.wpack) cudaFree(const_cast<void*>(net.tc.wpack));
  if (net.tc.bias) cudaFree(const_cast<float*>(net.tc.bias));
  net.tc.wpack = nullptr; net.tc.bias = nullptr;
  net.tc_alloc_bytes = 0; net.tc_alloc_bias = 0;
}

cudaError_t launch_mlp_tc2(const hr_config& cfg, const MlpTcPack& pk, const float* rays, float* heads, long long n, int num_sms,
                           cudaStream_t stream, float* rays_copy) {
  long long tiles = (n + tc::BM - 1) / tc::BM;
  int grid = (int)(tiles < num_sms ? tiles : num_sms);
  if (grid < 1) grid = 1;
  // the 16-byte heads stores need every row to start 16-byte aligned; any other row takes the narrow stores
  const bool narrow = (cfg.mlp_out % 4) != 0 || ((uintptr_t)heads % 16) != 0;
  const bool f16 = cfg.mlp_mode == HR_MLP_FP16_TC;
  if (cfg.mlp_width != 256 && cfg.mlp_width != 128) return cudaErrorInvalidValue;
  tc2_kernel(cfg.mlp_width, narrow, f16)<<<grid, tc2::NTHREADS, tc2_smem_bytes(f16), stream>>>(cfg, pk, rays, heads, n, rays_copy,
                                                                                              TrainSave{});
  return cudaGetLastError();
}

cudaError_t launch_mlp_tc2_train(const hr_config& cfg, const MlpTcPack& pk, const float* rays, float* heads, long long n,
                                 int num_sms, cudaStream_t stream, const TrainSave& sv) {
  long long tiles = (n + tc::BM - 1) / tc::BM;
  int grid = (int)(tiles < num_sms ? tiles : num_sms);
  if (grid < 1) grid = 1;
  auto kern = cfg.mlp_width == 256 ? mlp_tc2_kernel<256, true, false> : mlp_tc2_kernel<128, true, false>;
  if (cfg.mlp_width != 256 && cfg.mlp_width != 128) return cudaErrorInvalidValue;
  constexpr int smem = tc2::Layout<false>::SMEM_BYTES;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  kern<<<grid, tc2::NTHREADS, smem, stream>>>(cfg, pk, rays, heads, n, nullptr, sv);
  return cudaGetLastError();
}

}  // namespace hr
