// Sample-net weight packs and launchers shared between hr_api.cu and the kernels.
#pragma once
#include <cuda_runtime.h>
#include "hyperreel_b200.h"

namespace hr {

// fp32 CUDA-core path: per layer a k-major matrix Wt[Kp][Np] (zero padded) and a bias[Np].
//   layer 0      : rows = encoded input, padded to in_pad
//   skip layer   : rows = [input (in_pad) ; hidden (W)]   (mlp.py:167-168: cat([input_x, x]))
//   other layers : rows = hidden (W)
//   last layer   : columns permuted to channel-major (column c*S+s  <-  reference row s*stride+c)
struct MlpSimtPack {
  const float* Wt[HR_MAX_LAYERS];
  const float* bias[HR_MAX_LAYERS];
  int Kp[HR_MAX_LAYERS];
  int Np[HR_MAX_LAYERS];
  int in_pad;
  int n_layers;
  int skip;
};

// wgmma path (HR_MLP_BF16X3_TC, HR_MLP_FP16_TC): see hr_mlp_tc2.cu.  A "pass" is one accumulator's worth of output columns
// (W = hidden width: a whole hidden layer, or W columns of the last layer); its weights are stored as n_chunks*2 k-step
// images.  At most HR_TC_MAX_PASSES passes (hyperreel_b200.h).
struct TcPass {
  int layer;        // Linear layer index
  int n;            // output columns of this pass (128; a partial last-layer pass is zero padded)
  int first_chunk;  // first A chunk consumed (0 = encoded input, in_chunks = first hidden chunk)
  int n_chunks;     // chunks of 32 k
  int bias_off;     // offset into the bias table
  int is_final;     // last layer: results go to HBM instead of the next A operand
  int out_col0;     // first output column (channel-major order) of a last-layer pass
  int wait_a;       // the issuer must wait for the A chunks (first pass of a layer)
};
struct MlpTcPack {
  const void* wpack;   // bf16 hi/lo (fp16: fp16) weight images, K-major no-swizzle layout, consumption order: columns [0, W/2) of
                       // every pass, then columns [W/2, W) (wpack_bytes / 2 each)
  const float* bias;   // [bias_count]
  long long wpack_bytes;
  int n_passes;
  int bias_count;
  int in_chunks;       // 32-wide k-chunks of the encoded input (1: mlp_in <= 32, 2: mlp_in <= 64)
  TcPass passes[HR_TC_MAX_PASSES];
};

size_t mlp_simt_smem_bytes(const MlpSimtPack& pk, int W);
cudaError_t launch_mlp_simt(const hr_config& cfg, const MlpSimtPack& pk, const float* rays, float* heads,
                            long long n, int num_sms, cudaStream_t stream);

// rays may point to pinned host memory (read once, by the encoding threads); rays_copy (optional) receives a device copy
cudaError_t launch_mlp_tc2(const hr_config& cfg, const MlpTcPack& pk, const float* rays, float* heads, long long n,
                           int num_sms, cudaStream_t stream, float* rays_copy = nullptr);

// Training net on the tensor cores (hr_mlp_train.cu).  The forward is mlp_tc2_kernel<W, SAVE = true, false>: it also writes the
// encoded input enc [n][ld_enc] (zero padded past mlp_in) and hidden layer l's LeakyReLU output at act + l * act_stride,
// [n][W], all fp32, and stores the heads in the reference's order.
struct TrainSave {
  float* enc;
  float* act;
  long long act_stride;  // floats between two layers' activations
  int ld_enc;
};
cudaError_t launch_mlp_tc2_train(const hr_config& cfg, const MlpTcPack& pk, const float* rays, float* heads, long long n,
                                 int num_sms, cudaStream_t stream, const TrainSave& sv);

// Workspace of one training step of the net over n rays (byte offsets, each 256-byte aligned): the forward's saved
// activations, the channel-major d heads [n][ld_dlast] (mlp_out rounded up to 4, zero pad columns: the GEMM loaders read
// float4 rows), two [n][W] buffers for the hidden layers' dY, the dW GEMM's split-K partials.
struct TrainNetLayout {
  size_t enc, act, act_stride, dlast, dy[2], part, dbpart, total;
  int ld_enc, ld_dlast;
};
TrainNetLayout train_net_layout(const hr_config& c, long long n, int num_sms);
// d_heads_cm [n][mlp_out] channel-major (inside the workspace at dlast) -> every layer's dW / db into weight[l] / bias[l]
// ([out, in] / [out] of the uploaded weights).  W_t: the fp32 CUDA-core pack (MlpSimtPack), read as the transposed weights.
cudaError_t train_net_backward(const hr_config& c, const MlpSimtPack& simt, long long n, float* const* weight,
                               float* const* bias, uint8_t* ws, int num_sms, cudaStream_t st);
}  // namespace hr

struct SampleNet;
namespace hr {
// packs the net `net.cfg` describes into net.tc; net.tc_alloc_bytes / tc_alloc_bias remember the allocation behind it
// (reused while unchanged)
int pack_mlp_tc2(SampleNet& net, const float* const* w_dev, const float* const* b_dev, cudaStream_t st);
void free_mlp_tc2(SampleNet& net);
}
