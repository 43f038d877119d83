/*
 * hyperreel_b200 -- C-ABI of the H100-native HyperReel per-ray rendering hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch types.  The reference has no
 * FFI (it is pure PyTorch); every entry point below names the reference interface it replaces
 * (file:line under the reference checkout).  The Python binding a maintainer would add is the ctypes
 * stub shown in INTEGRATION.md (hyperreel_b200/lib.py is that stub, complete).
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on error; hr_last_error() gives the message
 *     (the reference raises Python exceptions / asserts: nlf/nets/tensorf_dynamic.py:744-745;
 *     the Python shim turns a non-zero status into RuntimeError);
 *   - all work is enqueued on the caller's cudaStream_t (passed as void*): the reference runs on
 *     torch's current stream (nlf/__init__.py:486-502); no hidden synchronisation except in
 *     hr_render_host, which is synchronous by contract;
 *   - a handle is re-entrant per handle, no global state except the thread-local error string;
 *   - there is NO CPU fallback: if no sm_90 device is present hr_create fails.
 */
#ifndef HYPERREEL_B200_H
#define HYPERREEL_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HR_ABI_VERSION 26

#define HR_MAX_GROUPS 4   /* ray-parameterisation groups feeding the sample net (ray.py:235-263) */
#define HR_MAX_LAYERS 10  /* Linear layers of the sample net (mlp.py:127-154) */
#define HR_MAX_SAMPLES 256 /* z_channels S (per-ray sample primitives) */
#define HR_MAX_PEERS 8    /* destination buffers of hr_render_scatter (GPUs of one NVSwitch domain) */
/* Passes of an HR_MLP_BF16X3_TC or HR_MLP_FP16_TC sample net: (mlp_layers - 1) hidden layers + ceil(last layer's outputs / mlp_width).  The
 * table is a kernel parameter; 40 passes hold every shape at width 256 and, at width 128, depth 10 with S * head_stride up
 * to 3968 (S = 256 x 15 channels).  hr_create refuses a tensor-core net that needs more (the fp32 net has no such limit). */
#define HR_TC_MAX_PASSES 40

/* Activation y = f(x*inner_fac + shift) * outer_fac  (nlf/activations.py:53-69,121-137,163-178).
 * EaseValue (activations.py:462-496) wrapped around it: while its window is open (eased != 0) the result is blended with the
 * start value, y' = y * ease_mul + ease_add (each op rounded), where the host computes in double ease_mul = w and
 * ease_add = (1 - w) * start_value from the ease weight w at the current iteration (activations.py:473-489).  A closed window
 * is eased = 0: the plain activation, ease_mul / ease_add ignored (and zero).  Only the density heads act_sigma,
 * act_point_sigma and pre_act_sigma may be eased (the only open windows of the shipped model YAMLs); the kernels ignore
 * `eased` elsewhere, and hr_set_activations refuses it.  `ease_pad` keeps the struct a multiple of 8 bytes, so that every
 * hr_config member keeps the 8-byte alignment it had before the ease members existed (the render kernels load pairs of
 * configuration words with 64-bit uniform loads; a shifted alignment changes their register allocation). */
enum { HR_ACT_IDENTITY = 0, HR_ACT_SIGMOID = 1, HR_ACT_TANH = 2 };
typedef struct hr_act {
  int32_t kind;
  float inner_fac, shift, outer_fac;
  int32_t eased;
  float ease_mul, ease_add;
  int32_t ease_pad;  /* 0 */
} hr_act;

/* One `params:` group of RayPredictionEmbedding (nlf/embedding/ray.py:235-263,320-326):
 * rays[:, start:end] -> RayParam fn -> WindowedPE (all windows open). */
enum { HR_PARAM_IDENTITY = 0, HR_PARAM_TWO_PLANE = 1, HR_PARAM_PLUECKER = 2 };
typedef struct hr_encode_group {
  int32_t start, end;        /* channel slice of the ray                                    */
  int32_t fn;                /* HR_PARAM_* (nlf/param.py:20-24, 63-118, 223-256)             */
  int32_t n_freqs;           /* WindowedPE bands 2^1..2^n (nlf/pe.py:148,210-221)            */
  int32_t exclude_identity;  /* pe.py:160-168                                               */
  float freq_mult;           /* freq_multiplier (pe.py:147)                                 */
  float base_mult;           /* base_multiplier (pe.py:151)                                 */
  float near, far;           /* two_plane plane offsets (param.py:78-79)                    */
  float dir_mult, mom_mult;  /* pluecker multipliers (param.py:236-237)                     */
} hr_encode_group;

enum { HR_ISECT_Z_PLANE = 0, HR_ISECT_SPHERE = 1, HR_ISECT_CYLINDER = 2, HR_ISECT_SPHERE_NEW = 3,
       HR_ISECT_DISTANCE = 4,  /* z.py:16-97, primitive.py:366-438, :181-250, :440-546, :126-180 (euclidean_distance_unified) */
       HR_ISECT_VOXEL = 5,     /* voxel_grid: axis-aligned planes, sample s = plane s/3 of axis s%3 (voxel.py:19-112)        */
       HR_ISECT_PLANE = 6 };   /* deformable_voxel_grid: predicted plane normals + offsets (voxel.py:115-214)                */
enum { HR_CONTRACT_NONE = 0, HR_CONTRACT_MIPNERF = 1, HR_CONTRACT_AFFINE = 2 };  /* AFFINE: bbox / z_depth (contract.py:65-110) */
enum { HR_SHADE_SH = 0, HR_SHADE_RGB = 1 };
enum { HR_DENSE_RELU = 0, HR_DENSE_SOFTPLUS = 1, HR_DENSE_RELU_ABS = 2 };

/* Sample-net arithmetic.  FP32_SIMT: fp32 FMA on CUDA cores (bit-level closest to the reference's
 * cuBLAS SGEMM).  BF16X3_TC: wgmma tensor cores, every fp32 operand split into bf16 hi+lo and the
 * three leading cross products accumulated in fp32 registers (error ~2^-16 per product, see DESIGN.md).
 * FP16_TC: the reference's mixed precision (its interactive viewer runs the net under CUDA autocast): every Linear layer
 * with fp16 operands and bias, one wgmma product per k-step accumulated in fp32, each layer's result rounded to fp16 and
 * LeakyReLU applied to it in fp16; the last layer's fp16 outputs are stored as fp32 heads and everything after the net is
 * the fp32 pipeline.  Rendering only: the training net (hr_train_net_*) is bf16x3. */
enum { HR_MLP_FP32_SIMT = 0, HR_MLP_BF16X3_TC = 1,
       HR_MLP_ZERO = 2, /* `net: {type: zero}` (ZeroMLP, nlf/nets/mlp.py:14-33): every head is 0, no network runs */
       HR_MLP_FP16_TC = 3 };

/* The recognised pipeline signature (SURVEY.md section 8(a)); one struct describes what the
 * reference assembles from conf/experiment/model/<name>.yaml.  Anything the YAML asks for that this
 * struct cannot express is rejected by the host binding at construction (no fallback). */
typedef struct hr_config {
  int32_t abi_version;  /* = HR_ABI_VERSION */
  int32_t c_in;         /* ray channels: 6 static, 8 video (datasets/technicolor.py:360-396) */

  /* --- sample-prediction net input (a5,a6) --- */
  int32_t n_groups;
  hr_encode_group groups[HR_MAX_GROUPS];

  /* --- sample-prediction net (a7): nlf/nets/mlp.py:60-178 --- */
  int32_t mlp_in;      /* sum of PE output channels                                   */
  int32_t mlp_width;   /* hidden_channels W                                           */
  int32_t mlp_layers;  /* number of Linear layers = yaml depth (ray.py:283-285)        */
  int32_t mlp_skip;    /* index of the layer whose input is cat([in, h]) or -1         */
  int32_t mlp_out;     /* S * head_stride                                             */
  float leaky_slope;   /* 0.01 (activations.py:14-29)                                 */
  int32_t mlp_mode;    /* HR_MLP_*                                                    */

  /* --- per-sample heads (a8): ray.py:331-337; channel offsets inside one sample, -1 = absent --- */
  int32_t n_samples;    /* S                                                          */
  int32_t head_stride;  /* channels per sample (15 for the shipped targets)            */
  int32_t off_z, n_z;   /* z_vals: 1 channel (z_plane) or 4 (sphere: origin3 + radius) */
  int32_t off_flow, off_sigma, off_point_sigma, off_offset, off_cscale, off_cshift;
  hr_act act_z, act_flow, act_sigma, act_point_sigma, act_offset, act_cscale, act_cshift;

  /* --- intersection (a10-a13): nlf/intersect/base.py:142-259 --- */
  int32_t isect_type;             /* HR_ISECT_*                                        */
  hr_act isect_act;               /* `activation:` of the intersect block (base.py:119) */
  int32_t isect_use_sigma;        /* base.py:155-161                                   */
  int32_t isect_density_off;      /* head channel used as sigma there, -1 = zeros      */
  float z_scale;                  /* |samples[1]-samples[0]| (z.py:60-71)              */
  float isect_near, isect_far;    /* mask bounds (base.py:194-203)                     */
  int32_t isect_sort;             /* base.py:206-210                                   */
  float samples[HR_MAX_SAMPLES];  /* base primitives, host-computed linspace (z.py:50-57) */
  int32_t contract_type;          /* HR_CONTRACT_* (nlf/contract.py:113-192)           */
  int32_t contract_samples;       /* inverse-contract z before intersecting (base.py:132-133) */
  float contract_start_radius, contract_end_radius;      /* end may be +inf          */
  float contract_start_distance, contract_end_distance;
  float sphere_origin_initial[3]; /* primitive.py:388                                  */
  float sphere_origin_scale;      /* origin_scale_factor (primitive.py:387)            */

  /* --- keyframe snap + flow (a14): nlf/embedding/point.py:780-831, utils/flow_utils.py:10-35 --- */
  int32_t use_flow;
  int32_t num_keyframes, num_frames;  /* K, F                                          */
  hr_act flow_act;                    /* spatial_flow_activation (point.py:817)         */

  /* --- point offset (a15): point.py:371-396 --- */
  int32_t use_offset;
  int32_t offset_density_off;  /* head channel of `in_density_field`, -1 = zeros       */
  hr_act offset_act;

  /* --- TensoRF decode + composite (a17-a23) --- */
  int32_t dynamic;      /* 1: tensor_vm_split_time, 0: tensor_vm_split_no_sample         */
  float aabb[6];        /* min xyz, max xyz (tensorf_base.py:148)                        */
  float distance_scale; /* tensorf_base.py:212                                          */
  int32_t n_sigma[3];   /* n_lamb_sigma                                                 */
  int32_t n_app[3];     /* n_lamb_sh                                                    */
  int32_t app_dim;      /* data_dim_color: 27 (SH) or 3 (RGB)                           */
  int32_t shading;      /* HR_SHADE_*                                                   */
  int32_t white_bg, black_bg;
  float weight_thre;    /* rm_weight_mask_thre                                          */
  int32_t fea2dense;    /* HR_DENSE_*                                                   */
  float density_shift;
  int32_t use_color_scale_shift; /* 'color_scale' reaches the colour net (tensorf_dynamic.py:780-784) */
  int32_t clamp_output; /* eval(): clamp(0,1) (tensorf_dynamic.py:805-806)              */

  /* --- ABI 5 / 6 additions (SURVEY 8 f3) --- */
  /* HR_CONTRACT_AFFINE: c(p) = (p - min) / den per axis (BBoxContract :83-84: den = max - min; ZDepthContract :109-110:
   * min = 0, den = fac), distances are divided / multiplied by dist_fac (:77-81, :103-107).                             */
  float contract_affine_min[3], contract_affine_den[3];
  float contract_dist_fac;
  /* per-ray colour heads applied after compositing: rgb_map * (1 + scale[:,0]) + shift[:,0]
   * (scale_shift_color_one, utils/tensorf_utils.py:275-281; tensorf_dynamic.py:798-800); -1 = absent                 */
  int32_t off_cscale_global, off_cshift_global;
  hr_act act_cscale_global, act_cshift_global;
  /* HR_ISECT_SPHERE_NEW (8 z channels: origin 3, resize 3, offset 1, radius 1; primitive.py:489-546):
   * origin = z[0:3] * sphere_origin_scale, resize = z[3:6] * sphere_resize_scale + sphere_resize_initial           */
  float sphere_resize_scale;
  float sphere_resize_initial[3];

  /* --- ABI 10 additions --- */
  /* HR_ISECT_VOXEL / HR_ISECT_PLANE: `samples` holds one linspace per axis interleaved (sample s = plane s / isect_axes of
   * axis s % isect_axes); z_scale3 = spacing per axis (voxel.py:58-63; HR_ISECT_PLANE and the other primitives: z_scale x3) */
  int32_t isect_axes;       /* 3 (voxel_grid), number of start normals (deformable_voxel_grid), 1 otherwise              */
  float z_scale3[3];
  int32_t isect_outward;    /* voxel_grid outward_facing: z *= sign(d_axis) (voxel.py:80-83)                            */
  int32_t isect_max_axis;   /* voxel_grid max_axis: drop the planes of the non-dominant axes (voxel.py:100-110)          */
  float plane_normal[9];    /* deformable_voxel_grid start_normal rows (voxel.py:120-128)                                */
  float plane_normal_scale; /* normal_scale_factor (voxel.py:129)                                                        */
  /* ColorTransformEmbedding (point.py:558-612) + transform_color_one (utils/tensorf_utils.py:308-331): the composited pixel
   * becomes rgb + M rgb + shift with (M, shift) = row round(rays[:, -2]) of hr_params.color_embedding [n_color_views, 12];
   * 0 = off (no such embedding, or the dataset does not validate on every camera) */
  int32_t n_color_views;
  hr_act act_ctransform, act_ctshift;

  /* --- cascaded pipelines (PointPredictionEmbedding, nlf/embedding/point.py:39-219) ---
   * cascade == 1:  ray_prediction -> ray_intersect (pre_samples z-planes) -> point_prediction -> ray_intersect -> ...
   * The fields above then describe the SECOND stage: `groups` / `mlp_*` are the point net (evaluated once per first-stage
   * point on the 8-float row pt_src describes, emitting n_samples / pre_samples samples each, :142-206), the heads and the
   * intersection are those of the second ray_intersect.  The first stage -- a ray net or none, z-planes only -- is: */
  int32_t cascade;
  int32_t pre_samples;                      /* S0 = z_channels of the first stage (<= 32, divides n_samples)             */
  int32_t pre_n_groups;
  hr_encode_group pre_groups[HR_MAX_GROUPS];
  int32_t pre_mlp_in, pre_mlp_width, pre_mlp_layers, pre_mlp_skip;
  int32_t pre_mlp_mode;                     /* HR_MLP_ZERO or the same mode as mlp_mode                                  */
  int32_t pre_head_stride, pre_off_z, pre_off_sigma;  /* first-stage heads: z_vals (1 channel) and optionally sigma      */
  hr_act pre_act_z, pre_act_sigma, pre_isect_act;
  int32_t pre_use_sigma, pre_sort;
  float pre_z_scale, pre_near, pre_far;     /* like z_scale / isect_near / isect_far                                     */
  float pre_samples_tab[32];
  int32_t pt_src[8];                        /* HR_PT_*: what channel k of the point net's input row holds (:151-160)     */
} hr_config;

/* sources of the point net's inputs (`inputs:` of point_prediction; the named tensors are concatenated in YAML order) */
enum { HR_PT_NONE = -1, HR_PT_POINT_X = 0, HR_PT_POINT_Y = 1, HR_PT_POINT_Z = 2, HR_PT_VIEW_X = 3, HR_PT_VIEW_Y = 4,
       HR_PT_VIEW_Z = 5, HR_PT_ORIGIN_X = 6, HR_PT_ORIGIN_Y = 7, HR_PT_ORIGIN_Z = 8, HR_PT_TIME = 9 };

/* Parameters in the reference's own state_dict layout (SURVEY.md Appendix B), fp32, contiguous.
 * hr_upload re-lays them out on the device (channel-last tables, packed / split net weights) into
 * memory owned by the handle; the caller's buffers are not referenced after the call returns
 * (device sources: after the stream reaches that point). */
typedef struct hr_params {
  int32_t on_device;                     /* 1: pointers are device pointers, 0: host     */
  const float* mlp_weight[HR_MAX_LAYERS];/* layers.{l}[.0].weight  [out_l, in_l] row-major */
  const float* mlp_bias[HR_MAX_LAYERS];  /* layers.{l}[.0].bias    [out_l]               */
  /* density_plane[_space].{i} / app_plane[_space].{i}: [1, C_i, H_i, W_i]  (C_i may be 0 -> NULL) */
  const float* sigma_plane[3];
  const float* app_plane[3];
  int32_t plane_h[3], plane_w[3];
  /* second factor: dynamic  density_plane_time.{i} / app_plane_time.{i}  [1, C_i, K, L_i]
   *                static   density_line.{i}       / app_line.{i}        [1, C_i, L_i, 1]      */
  const float* sigma_second[3];
  const float* app_second[3];
  int32_t second_len[3];                 /* L_i                                          */
  const float* basis_mat;                /* basis_mat.weight [app_dim, sum(n_app)]       */
  const float* color_embedding;          /* embeddings.{i}.color_embedding [n_color_views, 12] (NULL when n_color_views == 0) */
  /* cascade: the first-stage ray net (embeddings.0.net); mlp_weight / mlp_bias above are then the point net's */
  const float* pre_mlp_weight[HR_MAX_LAYERS];
  const float* pre_mlp_bias[HR_MAX_LAYERS];
} hr_params;

typedef struct hr_handle hr_handle;

/* Version of this ABI (compare with HR_ABI_VERSION). */
int hr_abi_version(void);

/* Last error message of the calling thread ("" if none).  Replaces: Python exceptions. */
const char* hr_last_error(void);

/* Replaces: model_dict['lightfield'](cfg.model, system) + render_fn_dict['lightfield'](...)
 * construction (nlf/__init__.py:351-364, nlf/models/models.py:104-129, nlf/rendering.py:59-70).
 * `device` is the CUDA ordinal.  Fails if the device is not sm_90 or the signature is unsupported. */
int hr_create(const hr_config* cfg, int device, hr_handle** out);

/* Replaces: INRSystem.load_state_dict (nlf/__init__.py:433-479) for the render path: ingest a
 * state_dict (any grid size: sizes come from the tensors, Appendix B), pack for the kernels. */
int hr_upload(hr_handle* h, const hr_params* p, void* stream);

/* Bytes of scratch hr_render needs for n rays (per-ray sample-net outputs).  Bounded: hr_render walks a large batch in
 * sub-batches of 16 sample-net tile waves (16 x num_sms x 128 rays), so the scratch never exceeds ~0.6 GB. */
int64_t hr_workspace_bytes(const hr_handle* h, int64_t n_rays);
/* Scratch of hr_render_heads / hr_render_backward (two full [n, mlp_out] buffers). */
int64_t hr_train_workspace_bytes(const hr_handle* h, int64_t n_rays);
/* Tuning: rays per sub-batch of hr_render (0 = default: 16 tile waves; < 0 = never split, scratch grows with n). */
int hr_set_sub_batch(hr_handle* h, int64_t rays);

/* Replaces: RenderLightfield.forward -> LightfieldModel.forward (nlf/rendering.py:72-77,
 * nlf/models/models.py:135-138) for one chunk: rays [n, c_in] fp32 device -> rgb [n,3] fp32 device.
 * `workspace` is device scratch of at least hr_workspace_bytes(h, n) bytes (16B aligned). */
int hr_render(hr_handle* h, const float* rays, int64_t n_rays, float* rgb,
              void* workspace, int64_t workspace_bytes, void* stream);

/* Ray-sharded rendering (SURVEY.md section 8(e); the reference renders a frame on rank 0 only, nlf/__init__.py:810-811).
 * Like hr_render, but the finished pixels of rays [0, n_rays) are stored at rows [row0, row0 + n_rays) of EVERY buffer
 * dst[0..n_dst): the caller passes its own [N_total,3] gather buffer and the peer-mapped gather buffers of the other ranks
 * (CUDA IPC / symmetric memory over NVLink), so the render kernel's epilogue is the gather of the pixel tiles -- 12 bytes
 * per ray and peer cross the fabric, no collective kernel follows.  The caller orders the peers' reads (a barrier after
 * the kernel on `stream`). */
int hr_render_scatter(hr_handle* h, const float* rays, int64_t n_rays, float* const* dst, int32_t n_dst, int64_t row0,
                      void* workspace, int64_t workspace_bytes, void* stream);

/* Debug/bisect variant (SURVEY.md section 4 "stage-boundary tests").  Any output pointer may be
 * NULL.  mlp_out [n, mlp_out] is in the reference's order (sample-major, ray.py:333);
 * distances [n,S] sorted t (base.py:206-210,257); points [n,S,3] final sample points (after flow
 * and offset); sigma [n,S]; weights [n,S] compositing weights (tensorf_utils.py:242-253); rgb_samples [n,S,3] the shaded
 * colour of every sample (renderModule output scattered by app_mask, tensorf_dynamic.py:757-777) before the colour transform. */
int hr_render_stages(hr_handle* h, const float* rays, int64_t n_rays, float* rgb,
                     float* mlp_out, float* distances, float* points, float* sigma, float* weights, float* rgb_samples,
                     void* workspace, int64_t workspace_bytes, void* stream);

/* ---- extra outputs of the colour net (SURVEY.md section 8 row a24) ----
 * Replaces: the `fields` / `no_over_fields` / `pred_weights_fields` render_kwargs of TensorVMKeyframeTime.forward /
 * TensorVMNoSample.forward (nlf/nets/tensorf_dynamic.py:808-837, nlf/nets/tensorf_no_sample.py:254-278) and the per-sample
 * dict RayPointEmbedding.forward returns to render_fn.embed (nlf/embedding/embedding.py:100-117).  A field is a key of the
 * dict `x` that reaches the colour net after `extract_fields`; the render kernel's epilogue reduces it in the warp that owns
 * the ray, nothing per-sample is written unless HR_FIELD_NO_OVER asks for it. */
enum {
  HR_FIELD_POINTS = 0,      /* x['points']       3 channels (after flow and offset)                   */
  HR_FIELD_DISTANCES = 1,   /* x['distances']    1           (sorted, contracted)                      */
  HR_FIELD_BASE_TIMES = 2,  /* x['base_times']   1           keyframe time (flow_utils.py:18-31)       */
  HR_FIELD_TIME_OFFSET = 3, /* x['time_offset']  1           t - base_time                             */
  HR_FIELD_TIMES = 4,       /* x['times']        1           rays[:, -1] broadcast (point.py:864-867)  */
  HR_FIELD_VIEWDIRS = 5,    /* x['viewdirs']     3           rays[:, 3:6] broadcast                    */
  HR_FIELD_WEIGHTS = 6,     /* x['weights']      1           ones (base.py:183-191, no weight_fn)      */
  /* per-sample heads of the sample net after their activation (ray.py:333-337), reachable through render_kwargs['fields']
   * (ExtractFieldsEmbedding adds them, point.py:236-244) */
  HR_FIELD_COLOR_SCALE = 7,   /* x['color_scale']   3                                                    */
  HR_FIELD_COLOR_SHIFT = 8,   /* x['color_shift']   3                                                    */
  HR_FIELD_SPATIAL_FLOW = 9,  /* x['spatial_flow']  3   as AdvectPoints leaves it (point.py:815-817)           */
  HR_FIELD_SIGMA = 10,        /* x['sigma']         1                                                    */
  HR_FIELD_POINT_SIGMA = 11,  /* x['point_sigma']   1                                                    */
  HR_FIELD_POINT_OFFSET = 12, /* x['point_offset']  3   as PointOffset leaves it: act(.) * (1 - sigma) (point.py:383-389) */
  HR_FIELD_COLOR_SCALE_GLOBAL = 13, /* x['color_scale_global'] 3  (per-sample head; the colour net uses sample 0's, tensorf_utils.py:275-281) */
  HR_FIELD_COLOR_SHIFT_GLOBAL = 14, /* x['color_shift_global'] 3                                                                   */
  HR_N_FIELDS = 15
};
enum {
  HR_FIELD_OVER = 0,         /* out [n, dim]   = sum_s w_s * x_s            (tensorf_dynamic.py:832-836)            */
  HR_FIELD_NO_OVER = 1,      /* out [n, S*dim] = x                          (:824-825)                              */
  HR_FIELD_PRED_WEIGHTS = 2  /* out [n, dim]   = sum_s alpha2weights(x['weights'])_s * x_s   (:818-819, :826-830)   */
};
typedef struct hr_field_request {
  int32_t field;  /* HR_FIELD_*                       */
  int32_t mode;   /* HR_FIELD_OVER / NO_OVER / PRED_WEIGHTS */
  float* out;     /* device buffer, shape per mode    */
} hr_field_request;

/* hr_render plus extra outputs: rgb [n,3]; render_weights [n,S] (the 'render_weights' key, :822-823) when non-NULL; every
 * request in req[0..n_req).  A field the pipeline does not carry (e.g. base_times of a static model) is an error. */
int hr_render_fields(hr_handle* h, const float* rays, int64_t n_rays, float* rgb, float* render_weights,
                     const hr_field_request* req, int32_t n_req, void* workspace, int64_t workspace_bytes, void* stream);

/* Replaces: INRSystem.forward(coords) on HOST buffers, i.e. the `.cuda()` upload, render_chunked
 * (nlf/rendering.py:100-150) and the `.cpu()` read-back of validation_video
 * (nlf/__init__.py:828-855).  rays_host/rgb_host should be pinned; the call splits the batch in
 * `chunk` rays (0 = default), overlaps H2D / kernels / D2H on internal streams and returns when the
 * rgb is on the host. */
int hr_render_host(hr_handle* h, const float* rays_host, int64_t n_rays, float* rgb_host, int64_t chunk);

/* ---- the step before the path: camera -> rays on the device (SURVEY.md section 8(f) row f2) ----
 * Replaces: get_coords_from_camera / get_coords (datasets/base.py:485-518, datasets/technicolor.py:360-396), i.e.
 * get_ray_directions_K + get_rays (+ get_ndc_rays_fx_fy) of utils/ray_utils.py:98-164, executed on the CPU by the
 * reference and uploaded with .cuda() per frame (nlf/__init__.py:828-834).  Pixel p = y*width + x, row-major like
 * kornia.create_meshgrid(H, W, normalized_coordinates=False). */
typedef struct hr_camera {
  float c2w[12];            /* camera-to-world, row-major 3x4 (pose[:3,:4])                         */
  float fx, fy, cx, cy;     /* K[0,0], K[1,1], K[0,2], K[1,2]                                       */
  int32_t width, height;    /* W, H                                                                 */
  int32_t centered_pixels;  /* +0.5 pixel offset (ray_utils.py:103-104)                             */
  int32_t flipped;          /* sign of the y direction (ray_utils.py:108)                           */
  int32_t normalize;        /* get_rays(normalize=True) (ray_utils.py:127-128)                      */
  int32_t use_ndc;          /* get_ndc_rays_fx_fy (ray_utils.py:137-164) with H, W, fx, fy of this camera */
  float ndc_near;           /* dataset.near                                                         */
  float cam_idx, time;      /* channels 6 and 7 when c_in == 8 (technicolor.py:389-393)             */
  int32_t fisheye;          /* 0: pinhole; otherwise the two-coefficient fisheye below (ABI 17)     */
  float k1, k2;             /* radial_distortion[:2] of the camera in models.json, as float32       */
  int32_t two_plane;        /* 0: c2w / K camera above; otherwise the light-field view below (ABI 20) */
  float lf_s;               /* s of the view on the st plane (LightfieldDataset.get_coord), as float32 */
  float lf_t;               /* t of the view, as float32                                            */
  float lf_st_scale;        /* st_scale (vis_st_scale for the render split), as float32             */
  float lf_uv_scale;        /* uv_scale (vis_uv_scale for the render split), as float32             */
  float lf_near;            /* near plane z (lightfield.near, default -1), as float32               */
  float lf_far;             /* far plane z (lightfield.far, default 0), as float32                  */
  float lf_aspect;          /* the dataset's aspect, img_wh[0] / img_wh[1], as float32; nonzero     */
} hr_camera;
/* Fisheye cameras (ABI 17): the Immersive dataset's train and validation views (ImmersiveDataset.get_coords,
 * datasets/immersive.py:494-573).  When fisheye != 0 the pinhole direction's (x, y) -- centred pixels, y negated unless
 * flipped -- is undistorted as cv2.fisheye.undistortPoints(points, I, [k1, k2, 0, 0]) does (perspective_to_fisheye, :43-48),
 * the direction (u, v, -1) is normalised (F.normalize), then get_rays / NDC / cam_idx / time follow as for the pinhole.  A
 * point the solve does not bring back (no convergence in 10 Newton steps, or a flipped angle) becomes OpenCV's (-1e6, -1e6)
 * and its row is written like any other, as the reference does.  k1 = k2 = 0 is not the pinhole (the radius maps
 * r -> tan r), hence the flag.  k1 and k2 must be finite: hr_generate_rays and hr_render_frame_to8b_host refuse a fisheye
 * record otherwise and write nothing.  The render split's cameras (K * 0.75, no distortion) are pinholes.
 * Two-plane light-field views (ABI 20): the Stanford light-field dataset's views (get_lightfield_rays, utils/ray_utils.py:14-45,
 * as LightfieldDataset.get_coords drives it, datasets/lightfield.py:193-219).  When two_plane != 0, c2w, K, centered_pixels,
 * flipped, normalize, use_ndc, ndc_near and the fisheye fields are ignored, and pixel (x, y) of the width x height view is the
 * row, in fp32 with each operation rounded as torch's CPU kernels round it,
 *   S = s * st_scale, T = t * st_scale, u = linspace(-1, 1, width)[x] * uv_scale, v = (linspace(1, -1, height)[y] / aspect) * uv_scale,
 *   origin (S, T, near), direction F.normalize((u - S, v - T, far - near)),
 * with linspace evaluated as torch's CPU kernel does (fma(step, i, start) below the midpoint, fma(-step, steps - 1 - i, end)
 * from it; [start] for one step) and the norm as sqrt(fma(dz, dz, fma(dy, dy, dx * dx))), then cam_idx and time as for the
 * other models.  The reference subtracts far - near in double; the record's
 * far - near in fp32 must be that value rounded (hyperreel_b200.TwoPlaneCamera checks it).  hr_generate_rays,
 * hr_render_frame_to8b_host and hr_render_video_to8b refuse, and write nothing for, a record with both two_plane and fisheye
 * set, a non-finite lf_* field or lf_aspect == 0.  The training entry points read their records on the device and do not
 * inspect them: the same must hold there. */

/* rays_out [n_pixels, c_in] fp32 device, for pixels first_pixel .. first_pixel + n_pixels - 1; c_in is 6 or 8. */
int hr_generate_rays(const hr_camera* cam, int32_t c_in, int64_t first_pixel, int64_t n_pixels, float* rays_out,
                     void* stream);

/* Pixel formats of uint8 images (ABI 23).  HR_PIXEL_RGB8: [.., 3] RGB.  HR_PIXEL_RGBA8: [.., 4] RGBA, the frames of the
 * datasets whose get_rgb loads RGBA (datasets/donerf.py, catacaustics.py); where such an image is consumed as a colour, that
 * colour is their get_rgb's composite over white, rgb * a + (1 - a) of the u8 / 255 values (T.ToTensor()), each of the
 * multiply, subtract and add rounded on its own in fp32 (no FMA), as torch computes it on the CPU.  4-byte aligned. */
#define HR_PIXEL_RGB8 0
#define HR_PIXEL_RGBA8 1

/* ---- training batches from images on the device (SURVEY.md section 2 row 23) ----
 * Replaces: the training split of the reference's datasets in its default mode (datasets/base.py:111-143,202-227,254-289): the
 * host table all_inputs = cat([all_coords, all_rgb, all_weights]) of every training ray, re-permuted every epoch
 * (np.random.permutation) and handed out in consecutive slices that format_batch splits and the loop copies to the GPU.
 * Handle-free.  cameras: device array of n_views records, each of width `width` and height `height`; images: device uint8
 * [n_views, height, width, 3] for pixel_format HR_PIXEL_RGB8, [n_views, height, width, 4] (4-byte aligned) for HR_PIXEL_RGBA8
 * (ABI 23), when each row's rgb is its pixel's composite over white; rays, order, draws and ids do not depend on the format.
 * An unknown pixel_format, or RGBA images not 4-byte aligned, is refused.  Pixel p in [0, N), N = n_views*height*width, is
 * view p / (height*width), then row-major within the view like hr_generate_rays.  Row r of the batch is pixel
 *   order[r]                                        when order (device int64, batch_size entries) is given;
 *   element batch_index*batch_size + r of epoch's permutation of [0, N), keyed by (seed, epoch)   otherwise
 * (a Feistel network over the next power of two >= N with cycle-walking, so an epoch visits every pixel exactly once;
 * csrc/hr_train_batch.cu states it).  Without order, batch_index must lie in [0, ceil(N / batch_size)) and the last batch of an
 * epoch is short: *n_rows (host, may be NULL) receives the row count, batch_size or fewer.  Outputs (device, n_rows rows):
 *   coords [n, c_in] fp32, bit-identical to the row hr_generate_rays writes for that pixel of that view's camera; c_in 6 or 8;
 *   rgb [n, 3] fp32, u8 / 255 (T.ToTensor());  weight [n, 1] fp32, 1;  pixel_ids [n] int64 (may be NULL), the pixel of each row.
 * An order entry outside [0, N) gives a zero row of weight 0 and pixel id -1.  coords, order and pixel_ids 8-byte aligned, the
 * rest 4.  No float atomics, no host synchronisation: two calls with the same arguments write the same bits.
 * Each row takes its view's camera model (ABI 17: a fisheye record's rays as hr_generate_rays writes them; ABI 20: a two-plane
 * record's), so one batch may mix pinhole, fisheye and two-plane views; the records' fisheye coefficients must be finite and
 * their two-plane records well formed as hr_generate_rays requires (the device array is not inspected). */
int hr_sample_train_batch(const hr_camera* cameras, int32_t n_views, const uint8_t* images, int32_t pixel_format,
                          int32_t height, int32_t width, int32_t c_in, uint64_t seed, int64_t epoch, int64_t batch_index,
                          int64_t batch_size, const int64_t* order, float* coords, float* rgb, float* weight,
                          int64_t* pixel_ids, int64_t* n_rows, void* stream);

/* Training batches over a table of per-view pixel subsets, drawn with or without replacement.
 * Replaces: the training split of the video datasets (datasets/technicolor.py:211-269, datasets/neural_3d.py:168-185,217-269),
 * which keep per view only the pixels with (x + y + offset) % stride == 0, sampled as the shipped training configs do
 * (sample_with_replacement: RandomSampler(replacement=True, num_samples=num_iters * batch_size), nlf/__init__.py:222-237).
 * cameras, n_views, images, pixel_format, height, width, c_in: as hr_sample_train_batch.  The table is implicit:
 * view_start (device int64 [n_views + 1]) is the exclusive prefix of the per-view row counts and view_rule (device int32
 * [n_views, 2]) each view's (stride >= 1, offset); table row k is in view v with view_start[v] <= k < view_start[v + 1], at
 * rank k - view_start[v] of that view's kept pixels in row-major order (the reference's all_coords order).  Row r of the
 * batch is table row
 *   table_rows[r]                                       when table_rows (device int64, batch_size entries) is given;
 *   element batch_index*batch_size + r of epoch's permutation of [0, n_table)   when mode == HR_SAMPLE_PERMUTE
 *     (hr_sample_train_batch's permutation; batch_index in [0, ceil(n_table / batch_size)), the last batch short);
 *   an independent uniform draw from [0, n_table), keyed by (seed, epoch, batch_index*batch_size + r)
 *                                                       when mode == HR_SAMPLE_REPLACE (every batch full, batch_index >= 0).
 * n_table lies in [1, n_views*height*width] and is view_start[n_views] for a well-formed plan.  Outputs: coords, rgb, weight as
 * hr_sample_train_batch; pixel_ids [n] (may be NULL) view*H*W + y*W + x; table_ids [n] (may be NULL) the table row.  A row
 * the plan does not hold (a table_rows entry outside [0, n_table), a malformed plan) gives a zero row of weight 0 and ids -1,
 * and nothing outside the arrays is read or written.  coords, view_start and the int64 arrays 8-byte aligned, the rest 4.  No
 * float atomics, no host synchronisation: two calls with the same arguments write the same bits. */
#define HR_SAMPLE_PERMUTE 0
#define HR_SAMPLE_REPLACE 1
int hr_sample_train_rows(const hr_camera* cameras, int32_t n_views, const uint8_t* images, int32_t pixel_format,
                         int32_t height, int32_t width, int32_t c_in, const int64_t* view_start, const int32_t* view_rule,
                         int64_t n_table, int32_t mode, uint64_t seed, int64_t epoch, int64_t batch_index,
                         int64_t batch_size, const int64_t* table_rows, float* coords, float* rgb, float* weight,
                         int64_t* pixel_ids, int64_t* table_ids, int64_t* n_rows, void* stream);

/* The Immersive dataset's training table: per-view keep masks chosen by image content.
 * Replaces: ImmersiveDataset.prepare_train_data / subsample / importance_subsample (datasets/immersive.py:295-391).  Views are
 * video-major with each video's frames in order; an importance view v keeps the pixels with diff > thr and dz < -0.05 in
 * row-major order, diff = mean over channels of |rgb_v - rgb_{v-1}| (u8 / 255 in fp32, ((d0 + d1) + d2) / 3), thr = diff's value
 * of ascending rank (N - num_take) % N (N = height*width; duplicates counted), dz = channel 5 of hr_generate_rays's row for the
 * pixel.  cameras, n_views, height, width: as hr_sample_train_batch (height*width < 2^31); images HR_PIXEL_RGB8.  plan:
 * HOST int64 [n_views, 2], per view (num_take, prev): (-1, -1) for a whole view, else num_take in [0, N] and prev == v - 1
 * (the previous frame of the same video; v >= 1).  At most 65535 importance views per call; n_slots is their number.
 * Outputs (device): view_slot int32 [n_views], the view's slot (its rank among the importance views) or -1;
 *   masks uint32 [n_slots, B, 8], B = ceil(N / 256): bit (p & 31) of word p >> 5 of the slot's mask keeps pixel p;
 *   block_start uint32 [n_slots, B]: exclusive prefix of the kept counts of each 256-pixel block within the view;
 *   view_rows int64 [n_views]: the kept counts (N for whole views);  view_start int64 [n_views + 1]: their exclusive prefix.
 * masks and block_start may be NULL when n_slots == 0.  workspace: device, 256-byte aligned, at least
 * hr_importance_workspace_bytes(n_slots) bytes.  A malformed plan or argument returns non-zero and writes nothing.  A fixed
 * number of launches whatever n_views, integer atomics only: two builds write the same bits.  No host synchronisation beyond
 * the copy of the plan's slots from host memory. */
int64_t hr_importance_workspace_bytes(int32_t n_slots);
int hr_build_importance_table(const hr_camera* cameras, int32_t n_views, const uint8_t* images, int32_t height, int32_t width,
                              const int64_t* plan, void* workspace, int64_t workspace_bytes, int32_t* view_slot,
                              uint32_t* block_start, uint32_t* masks, int64_t* view_rows, int64_t* view_start, void* stream);

/* Training batches over a table of per-view keep masks (hr_build_importance_table's outputs): as hr_sample_train_rows, with
 * view_slot, block_start and masks in place of view_rule, and images HR_PIXEL_RGB8 (the Immersive dataset's frames are
 * RGB).  Table row k is in view v with view_start[v] <= k < view_start[v + 1], at rank k - view_start[v] of that view's kept
 * pixels in row-major order (every pixel for slot -1).  n_table is view_start[n_views] for a well-formed table; a row the
 * table does not hold gives a zero row of weight 0 and ids -1. */
int hr_sample_train_mask_rows(const hr_camera* cameras, int32_t n_views, const uint8_t* images, int32_t height, int32_t width,
                              int32_t c_in, const int64_t* view_start, const int32_t* view_slot, const uint32_t* block_start,
                              const uint32_t* masks, int64_t n_table, int32_t mode, uint64_t seed, int64_t epoch,
                              int64_t batch_index, int64_t batch_size, const int64_t* table_rows, float* coords, float* rgb,
                              float* weight, int64_t* pixel_ids, int64_t* table_ids, int64_t* n_rows, void* stream);

/* ---- the step after the path: 8-bit packing (SURVEY.md section 8(f) row f4) ----
 * Replaces: to8b(x) = (255 * clip(x, 0, 1)).astype(uint8) (utils/__init__.py:47) applied to the rendered frame before
 * it is written or displayed (nlf/__init__.py:857-891, utils/gui_utils.py:174-186).  Same as hr_render, but the fused
 * kernel's epilogue stores rgb8 [n,3] uint8 (3 B/ray instead of 12 B/ray leave the GPU). */
int hr_render_to8b(hr_handle* h, const float* rays, int64_t n_rays, uint8_t* rgb8, void* workspace,
                   int64_t workspace_bytes, void* stream);

/* Whole frame on HOST output: rays generated on the device from `cam`, rendered, packed to 8 bit, copied into the
 * (pinned) host buffer rgb8_host [width*height, 3]; synchronous.  Replaces one iteration of validation_video /
 * NeRFGUI.test_step (nlf/__init__.py:828-891, utils/gui_utils.py:139-212). */
int hr_render_frame_to8b_host(hr_handle* h, const hr_camera* cam, uint8_t* rgb8_host, int64_t chunk);

/* ---- videos on the device (ABI 19) ----
 * Replaces: the loop of validation_video over the render dataset's poses (nlf/__init__.py:809-891, run every render_every
 * epochs and by render_only, :998-1008): per frame, rays built on the CPU, uploaded, rendered, copied back, to8b.
 * cameras: HOST array of n_frames records, all of one width x height, each pinhole, fisheye (ABI 17) or two-plane (ABI 20); times: HOST fp32
 * [n_frames], frame f's time column (channel 7 when c_in == 8; the records' own `time` is not used).  video: DEVICE uint8
 * [n_frames, height, width, 3], frame f's pixels as hr_render_frame_to8b_host renders records[f] with time = times[f], bit for
 * bit.  workspace: device scratch of hr_video_workspace_bytes(h, n_frames, height, width) bytes (16B aligned): the records
 * and times, then scratch bounded whatever n_frames, two slots (one for a video of at most one sub-batch), each one sub-batch
 * of rays (hr_render's sub-batch, 16 sample-net tile waves) and its render scratch.  The video's rays are generated and
 * rendered sub-batch by sub-batch across frame boundaries, alternating between two streams of the handle that are forked
 * from and joined back to `stream` by events: the call is ordered on `stream` like any other work.  No host
 * synchronisation (the records and times are copied with cudaMemcpyAsync, so the host arrays may be reused when the call
 * returns).  Refused before anything is enqueued: n_frames < 1, frames of
 * different sizes, a size whose output bytes overflow int64, a non-finite record field, time or fisheye coefficient, a
 * malformed two-plane record (ABI 20). */
int64_t hr_video_workspace_bytes(const hr_handle* h, int32_t n_frames, int32_t height, int32_t width);
int hr_render_video_to8b(hr_handle* h, const hr_camera* cameras, const float* times, int32_t n_frames, uint8_t* video,
                         void* workspace, int64_t workspace_bytes, void* stream);

/* ---- held-out splits scored on the device (ABI 21) ----
 * Replaces: the reference's evaluation of a validation / test split (nlf/__init__.py:249-265, :895-982, :1015-1030): per
 * view, rays built on the CPU, the view rendered, copied to the host and scored with scikit-image.  cameras / times: HOST
 * arrays of n_views records (one width x height, >= 11 x 11, pinhole, fisheye and two-plane mixed freely) and fp32 times, as
 * hr_render_video_to8b takes them.  gt: DEVICE uint8, the views' ground truth: [n_views, height, width, 3] for pixel_format
 * HR_PIXEL_RGB8, [n_views, height, width, 4] (4-byte aligned) for HR_PIXEL_RGBA8 (ABI 23).  out: DEVICE fp64
 * [n_views][2] = (mse, ssim) of each view, bit for bit hr_image_metrics of the fp32 frame hr_render makes of the view's rays
 * (clamped output, the configured background, no to8b) against gt / 255 correctly rounded in fp32 (T.ToTensor()'s conversion; NumPy's, and torch's on the CPU),
 * or for RGBA against its fp32 composite over white (HR_PIXEL_RGBA8 above).
 * workspace: device scratch of hr_score_views_workspace_bytes(h, n_views, height, width) bytes (16B aligned, -1 for a size
 * hr_score_views refuses): the records and times (sizeof(hr_camera) + 4 = 148 bytes per view, copied once on `stream`),
 * then scratch bounded whatever n_views, a ring of whole fp32 frames (enough for two sub-batches and one frame more), two
 * metrics partial buffers and the video path's one or two slots.  The split is one ray sequence rendered in
 * hr_render_video_to8b's sub-batches on its two streams (forked from and joined back to `stream` by events), a sub-batch
 * also cut where it would wrap the ring; a sub-batch that completes frames scores them with one metrics launch on its own
 * stream, after an event of the other stream for a frame that straddles the two, and a ring frame is reused only after the
 * launch that scored it.  No host synchronisation, no float atomics:
 * two calls write the same bits.  Refused before anything is enqueued (out untouched): null or misaligned pointers
 * (out 8B, workspace 16B, RGBA gt 4B), an unknown pixel_format, n_views < 1, views of different sizes or smaller than
 * 11 x 11, a size whose bytes overflow int64, a non-finite record field, time or fisheye coefficient, a malformed two-plane
 * record, a workspace too small. */
int64_t hr_score_views_workspace_bytes(const hr_handle* h, int32_t n_views, int32_t height, int32_t width);
int hr_score_views(hr_handle* h, const hr_camera* cameras, const float* times, int32_t n_views, const uint8_t* gt,
                   int32_t pixel_format, double* out, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- embedding maps of a video or split (ABI 25) ----
 * Replaces: the embedding visualiser's second render pass per frame (EmbeddingVisualizer.validation, nlf/visualizers/
 * embedding.py:37-90, called by validation_video and validation_image, nlf/__init__.py:809-940) and its visualize_warp +
 * to8b (utils/visualization.py:24-52, utils/__init__.py:47).  One request per map: the field `field` reduced in mode `mode`
 * (HR_FIELD_OVER or HR_FIELD_PRED_WEIGHTS) as hr_render_fields reduces it, then, each step rounded on its own in fp32:
 * |x| when use_abs; (x - lo) / (hi - lo) when bounded, hi - lo rounded once; when normalize, (x - min) / (max - min) with
 * min and max per channel over the frame's pixels (NaN when the frame holds one); clamp to [0, 1] and (uint8)(255 * x),
 * truncated, a NaN giving 0.  out: DEVICE uint8 [n_frames, height, width, channels]; channels must be the field's (1 or 3). */
typedef struct hr_visual_request {
  int32_t field;      /* HR_FIELD_*                              */
  int32_t mode;       /* HR_FIELD_OVER / HR_FIELD_PRED_WEIGHTS    */
  int32_t channels;   /* 1 or 3, the field's channel count        */
  int32_t use_abs;    /* 0 / 1                                    */
  int32_t bounded;    /* 0 / 1: lo and hi apply                   */
  int32_t normalize;  /* 0 / 1: per-frame min / max               */
  float lo, hi;       /* finite, hi != lo, when bounded           */
  uint8_t* out;
} hr_visual_request;

/* cameras / times: HOST records and fp32 times as hr_render_video_to8b takes them.  video: DEVICE uint8 [n_frames, height,
 * width, 3] or NULL; when given, bit for bit what hr_render_video_to8b writes.  Every map comes from the same render pass as
 * the video.  A request without normalize is mapped to uint8 in the render kernel's epilogue (no fp32 field is written); a
 * request with normalize stages the field's fp32 values in a ring of whole frames (enough for two sub-batches and one frame
 * more), and each completed frame gets a min / max reduction (per-block partials, no atomics) and a map launch on the stream
 * of the sub-batch that completed it, a ring frame being rendered again only after its map launch.  The sub-batches, streams
 * and events are hr_score_views'; no host synchronisation; two calls write the same bits.  workspace: device scratch of
 * hr_render_visuals_workspace_bytes(h, req, n_req, n_frames, height, width) bytes (16B aligned, -1 for a call refused): the
 * records and times (148 bytes per frame), then scratch bounded whatever n_frames; without a request it is
 * hr_video_workspace_bytes', and the call is hr_render_video_to8b's.  Refused before anything is enqueued (outputs
 * untouched): null or misaligned pointers (workspace 16B), n_req < 0 or a null list with n_req > 0, nothing to write, an
 * unknown field or mode, a field requested twice or not carried by the pipeline, channels other than the field's 1 or 3, non-finite bounds or hi == lo, the checks of
 * hr_render_video_to8b on the records, times and size, a workspace too small. */
int64_t hr_render_visuals_workspace_bytes(const hr_handle* h, const hr_visual_request* req, int32_t n_req, int32_t n_frames,
                                          int32_t height, int32_t width);
int hr_render_visuals(hr_handle* h, const hr_camera* cameras, const float* times, int32_t n_frames, uint8_t* video,
                      const hr_visual_request* req, int32_t n_req, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- backward pass of the path (SURVEY.md section 8 row f1) ----
 * Replaces: what loss.backward() runs for the render path inside INRSystem.training_step (nlf/__init__.py:634-709): the
 * autograd graph of RayPointEmbedding + TensorVMKeyframeTime / TensorVMNoSample.  The sample net's Linear layers stay with
 * the caller (their forward / backward are plain GEMMs on activations the caller keeps); the library provides the three
 * pieces around them, all hand-written kernels:
 *   hr_encode_rays      rays -> encoded sample-net input (RayParam + PE, ray.py:320-326), kernel feature order
 *   hr_render_heads     sample-net output -> rgb, the forward of everything after the net (training or eval semantics)
 *   hr_render_backward  d rgb -> d (sample-net output); gradients of the VM tables and basis_mat accumulate in the handle
 *   hr_grad_zero / hr_grad_read   clear / export the accumulated parameter gradients in the reference's tensor layouts
 * Supported: z_plane / sphere / cylinder (origin_scale_factor == 0) / euclidean-distance / voxel-grid / deformable-plane
 * primitives, no / mipnerf / bbox / z_depth contraction, per-sample and per-ray colour heads, the per-camera colour transform
 * with at most 512 views (its gradient is summed per CTA in shared memory), at most 64 samples per ray; sphere_new, cascaded (point_prediction) pipelines and learned primitive origins are rejected
 * (hr_last_error). */
typedef struct hr_train_opts {
  int32_t clamp_output; /* 1: eval() forward, clamp(0,1) (tensorf_dynamic.py:805-806); 0: training forward            */
  int32_t white_bg;     /* rgb_map += 1 - acc_map: cfg.white_bg, or the training coin flip of :795-796 drawn by the caller */
} hr_train_opts;

typedef struct hr_grads {  /* device buffers in the reference's layouts (hr_params), overwritten by hr_grad_read; NULL = skip */
  float* sigma_plane[3];
  float* app_plane[3];
  float* sigma_second[3];
  float* app_second[3];
  float* basis_mat;
  float* color_embedding;  /* [n_color_views, 12]; ignored when n_color_views == 0 */
} hr_grads;

/* enc [n, mlp_in] fp32 device */
int hr_encode_rays(hr_handle* h, const float* rays, int64_t n_rays, float* enc, void* stream);
/* heads [n, mlp_out] in the reference's order (sample-major: column s*head_stride + c, ray.py:333); workspace of
 * hr_train_workspace_bytes(h, n) */
int hr_render_heads(hr_handle* h, const float* rays, const float* heads, int64_t n_rays, float* rgb, const hr_train_opts* opts,
                    void* workspace, int64_t workspace_bytes, void* stream);
/* d_rgb [n,3] -> d_heads [n, mlp_out] (reference order); workspace of hr_train_workspace_bytes(h, n) */
int hr_render_backward(hr_handle* h, const float* rays, const float* heads, int64_t n_rays, const float* d_rgb, float* d_heads,
                       const hr_train_opts* opts, void* workspace, int64_t workspace_bytes, void* stream);
int hr_grad_zero(hr_handle* h, void* stream);
int hr_grad_read(hr_handle* h, const hr_grads* out, void* stream);

/* ---- the sample net's training forward / backward on the tensor cores ----
 * Replaces: the sample net's Linear layers in the training graph (BaseMLP.forward, nlf/nets/mlp.py:159-172, and what
 * loss.backward() runs for them), as the alternative to keeping them with the caller (hr_encode_rays).  Every GEMM is
 * bf16x3 on wgmma (hi*hi + lo*hi + hi*lo, fp32 accumulation), like the HR_MLP_BF16X3_TC render net:
 *   hr_train_net_forward   rays -> heads [n, mlp_out] in the reference's order, bit-identical to the render net's heads;
 *                          the encoded input and every hidden activation are saved in the workspace
 *   hr_train_net_backward  d heads [n, mlp_out] (reference order) -> every layer's dW / db, written (not accumulated) into
 *                          the caller's buffers; the same workspace, untouched since the forward, is read.  The
 *                          gradients are bit-reproducible (split-K partials summed in a fixed order, no atomics).
 * The weights are those of the last hr_upload.  Needs a handle with mlp_mode HR_MLP_BF16X3_TC; cascaded pipelines and zero
 * nets are refused (hr_last_error).
 * Workspace (hr_train_net_workspace_bytes, 256-byte aligned): fp32 encoded input [n, mlp_in rounded up to 16], fp32
 * activations [mlp_layers - 1][n, mlp_width], d heads [n, mlp_out rounded up to 4], two [n, mlp_width] dY buffers and the split-K partials
 * (2 x SMs x 128 x 128 floats) -- 0.62 GB at 65,536 rays on the Technicolor
 * shape (6 layers of width 256, 9 input features, 480 outputs). */
int64_t hr_train_net_workspace_bytes(const hr_handle* h, int64_t n_rays);
int hr_train_net_forward(hr_handle* h, const float* rays, int64_t n_rays, float* heads, void* workspace, int64_t workspace_bytes,
                         void* stream);
typedef struct hr_net_grads {  /* device buffers in nn.Linear's layouts of the uploaded net (hr_params.mlp_weight / mlp_bias) */
  float* weight[HR_MAX_LAYERS]; /* [out, in] */
  float* bias[HR_MAX_LAYERS];   /* [out]     */
} hr_net_grads;
int hr_train_net_backward(hr_handle* h, const float* d_heads, int64_t n_rays, const hr_net_grads* out, void* workspace,
                          int64_t workspace_bytes, void* stream);

/* Replaces: EaseValue.set_iter (activations.py:495-496) reached through LightfieldModel.set_iter each training iteration.
 * Copies every hr_act member of `cfg` (act_*, isect_act, flow_act, offset_act, pre_act_*, pre_isect_act) into the handle;
 * every other member must equal the handle's configuration, else the call fails and the handle is unchanged.  No allocation,
 * no upload, no device synchronisation: launches enqueued after the call returns use the new activations (kernel parameters
 * are copied at launch), launches already enqueued keep the old ones.  The graph hr_render_host caches is dropped (its kernel
 * nodes hold the old configuration by value) and captured again by the next hr_render_host call. */
int hr_set_activations(hr_handle* h, const hr_config* cfg);

/* ---- held-out view scoring (handle-free) ----
 * Replaces: the host-side metrics of INRSystem.validation_image (nlf/__init__.py:976-980), i.e. metrics.psnr / metrics.ssim
 * (metrics.py:25-34) = scikit-image's peak_signal_noise_ratio(data_range=1) and structural_similarity(win_size=11,
 * multichannel, gaussian_weights, data_range=1) run on the CPU after a device-to-host copy of the frame.
 * pred, gt: [n_images, height, width, 3] fp32 device, channel-last.  out: device [n_images][2] fp64 = (mse, ssim) per image:
 *   mse  = mean over all height*width*3 values of (pred - gt)^2, difference and square in fp32, summed in fp64;
 *   ssim = per channel, the 11x11 Gaussian window (sigma 1.5, truncate 3.5, SciPy's normalised weights) moments filtered in
 *          fp64, sample covariance (121/120), C1 = 0.01^2, C2 = 0.03^2, mean of the SSIM map over [5, height-5) x
 *          [5, width-5), averaged over the 3 channels.
 * Deterministic: no float atomics, per-tile partials summed in a fixed order, so two calls give identical bits and an image's
 * result does not depend on the batch it is scored in.  height and width must be >= 11 (the window must fit), n_images in
 * [1, 65535]; out and workspace 8-byte aligned, the workspace (device) at least hr_image_metrics_workspace_bytes(n_images,
 * height, width) bytes (-1 for arguments hr_image_metrics refuses).  On error nothing is enqueued and `out` is untouched. */
int64_t hr_image_metrics_workspace_bytes(int32_t n_images, int32_t height, int32_t width);
int hr_image_metrics(const float* pred, const float* gt, int32_t n_images, int32_t height, int32_t width, double* out,
                     void* workspace, int64_t workspace_bytes, void* stream);

/* ---- frame resize to the training resolution (handle-free) ----
 * Replaces: the resize in the datasets' get_rgb, run on the host per image: Pillow's Image.resize (datasets/technicolor.py,
 * llff.py, spaces.py, stanford.py: LANCZOS to _img_wh, then BOX to img_wh) and cv2.resize (datasets/neural_3d.py,
 * immersive.py: the flag they pass sits in the dst slot, so both of their steps are OpenCV's default INTER_LINEAR).
 * src: DEVICE uint8 [n, H0, W0, C] contiguous, C = 3 for pixel_format HR_PIXEL_RGB8 and 4 for HR_PIXEL_RGBA8 (ABI 23).
 * dst: DEVICE uint8, frame f's row y at dst + (f * H + y) * dst_row_stride (dst_row_stride >= C * W bytes), so a slice of a
 * larger [N, H, W, C] tensor can be written in place.  method: one of HR_RESIZE_*; bit for bit the library's result on each
 * frame (Pillow 12's 8-bit convolution resampler with its filter; OpenCV 4's CV_8UC3 INTER_LINEAR, or INTER_AREA for
 * integer factors, with INTER_LINEAR sent to INTER_AREA at exactly 2x).  A frame of the same size is copied, as both
 * libraries do.  flags: HR_RESIZE_BGR reads src as BGR (channels 0 and 2 swapped), which is what OpenCV decodes; dst is
 * RGB.  For RGBA, HR_RESIZE_BGR reads BGRA and dst is RGBA, resized as the datasets that load RGBA resize it
 * (datasets/donerf.py, catacaustics.py): the Pillow methods resample the premultiplied RGBa image and convert back, as
 * Image.resize does for an RGBA image on every call (premultiply MULDIV255(c, a); unpremultiply c for a of 0 or 255, else
 * min(255, 255 * c / a)); cv2_area resamples the four channels independently, as OpenCV does.  workspace: device, 256-byte
 * aligned, at least hr_resize_workspace_bytes(n, H0, W0, H, W, method, pixel_format) bytes (-1 for sizes, a method or a
 * pixel_format hr_resize_frames refuses; 0 for the copy and the INTER_AREA paths): the coefficient tables, copied in with
 * the launch, and for the two Pillow passes the uint8 intermediate of the rows the vertical pass reads (premultiplied RGBa,
 * 4 bytes per pixel, for RGBA).  Kernels use integer multiply-adds only (INTER_AREA at factors other than 2 x 2 rounds
 * sum * (1.f / area) in fp32, as OpenCV does), no float atomics and no host synchronisation: two calls write the same bits.
 * Refused before anything is enqueued (dst untouched): null pointers, unknown method, flags or pixel_format, cv2_linear for
 * RGBA, sizes < 1, an enlargement in either direction, cv2_area at a non-integer factor, a Pillow reduction needing more
 * filter coefficients than Pillow allows (outSize > INT_MAX / (ksize * 8), where Pillow raises MemoryError), source,
 * destination or workspace bytes that overflow int64, a short dst_row_stride, a missing, misaligned or short workspace. */
#define HR_RESIZE_PIL_LANCZOS 0
#define HR_RESIZE_PIL_BICUBIC 1
#define HR_RESIZE_PIL_BOX 2
#define HR_RESIZE_CV2_LINEAR 3
#define HR_RESIZE_CV2_AREA 4
#define HR_RESIZE_BGR 1
int64_t hr_resize_workspace_bytes(int32_t n, int32_t H0, int32_t W0, int32_t H, int32_t W, int32_t method,
                                  int32_t pixel_format);
int hr_resize_frames(const uint8_t* src, int32_t n, int32_t H0, int32_t W0, uint8_t* dst, int32_t H, int32_t W,
                     int64_t dst_row_stride, int32_t method, int32_t flags, int32_t pixel_format, void* workspace,
                     int64_t workspace_bytes, void* stream);

/* Number of kernels hr_render launched since creation (bench.py's gpu_launches). */
int64_t hr_launch_count(const hr_handle* h);

/* Average device time (ms, CUDA events on the launching stream) of the dominant kernel -- the fused
 * gather+decode+composite kernel -- over launches since the last hr_timing_reset; needs
 * hr_timing_enable(h, 1).  Used by bench.py for roofline.achieved. */
int hr_timing_enable(hr_handle* h, int enable);
int hr_timing_reset(hr_handle* h);
int hr_timing_read(hr_handle* h, double* render_ms_avg, double* mlp_ms_avg, int64_t* launches);
/* same for the render-backward kernel of hr_render_backward */
int hr_timing_read_backward(hr_handle* h, double* backward_ms_avg, int64_t* launches);

/* Replaces: module destruction. */
int hr_destroy(hr_handle* h);

#ifdef __cplusplus
}
#endif
#endif /* HYPERREEL_B200_H */
