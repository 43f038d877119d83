// Training batches from images on the device: shuffled pixel rows with their rays generated per batch.
// Reference: the training split of datasets/base.py (prepare_train_data / update_all_data :111-143, shuffle :202-227,
// __getitem__ / format_batch :254-289).  The reference concatenates every training ray into a host table
// all_inputs = [coords | rgb | weight] (48 B per ray with c_in = 8), re-permutes the whole table every epoch and hands out
// consecutive slices.  Here the images stay on the device as uint8 and the table never exists: row r of batch b is element
// p = b*B + r of a keyed permutation of [0, N), N = n_views*H*W, and the kernel evaluates that pixel's ray (camera_ray,
// hr_rays.cuh, bit-identical to hr_generate_rays) and its colour (T.ToTensor(): u8 / 255 in fp32).
//
// Permutation: a Feistel network over [0, 2^k), 2^k the next power of two >= N, with cycle-walking (re-apply it until the
// value falls below N), so it is a bijection of [0, N) and each epoch visits every pixel exactly once.  The k bits split into
// a low half of k/2 bits and a high half of k - k/2 bits; the rounds alternately XOR the low half with F(high half) and the
// high half with F(low half), each round a bijection.  F(v) = mix64(v ^ round_key), mix64 the splitmix64 finaliser.  Keys:
// epoch_key = mix64(mix64(seed) + G*(epoch + 1)), round_key[i] = mix64(epoch_key + G*(i + 1)), G = 0x9E3779B97F4A7C15, all
// uint64 arithmetic modulo 2^64.  tests/train_order_oracle.py restates it in NumPy.
//
// RGBA images (HR_PIXEL_RGBA8, the DoNeRF and Catacaustics datasets): a row's colour is the composite their get_rgb returns,
// rgb * a + (1 - a) of the u8 / 255 values (rgba_over_white, hr_common.cuh, which the held-out scores share), from one
// aligned 4-byte load of the pixel.
//
// One thread per row: one 3-byte (or 4-byte) gather and one 48-byte row write (plus 8 B of pixel id when asked).  No float atomics, no
// host synchronisation; two calls with the same arguments write the same bits.  The camera records live on the device, so
// each row branches on its own record's fisheye and two_plane flags (camera_ray<true, true>) and one batch may mix pinhole,
// fisheye and two-plane views.
#include <algorithm>
#include <type_traits>
#include <vector>

#include "hr_handle.h"
#include "hr_rays.cuh"

namespace hr {
namespace {

constexpr int kRounds = 6;
constexpr uint64_t kGolden = 0x9E3779B97F4A7C15ull;

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

struct FeistelKey {
  uint64_t round[kRounds];
  uint64_t n;       // domain [0, n)
  int lo_bits;      // low half of the k bits; the high half has k - lo_bits
  uint64_t lo_mask, hi_mask;
};

FeistelKey feistel_key(uint64_t seed, int64_t epoch, uint64_t n) {
  FeistelKey k;
  int bits = 0;
  while (bits < 63 && (1ull << bits) < n) ++bits;
  k.n = n;
  k.lo_bits = bits / 2;
  k.lo_mask = (1ull << k.lo_bits) - 1;
  k.hi_mask = (1ull << (bits - k.lo_bits)) - 1;
  const uint64_t epoch_key = mix64(mix64(seed) + kGolden * ((uint64_t)epoch + 1));
  for (int i = 0; i < kRounds; ++i) k.round[i] = mix64(epoch_key + kGolden * (uint64_t)(i + 1));
  return k;
}

__device__ __forceinline__ uint64_t feistel_permute(uint64_t x, const FeistelKey& k) {
  do {
    uint64_t lo = x & k.lo_mask, hi = x >> k.lo_bits;
#pragma unroll
    for (int i = 0; i < kRounds; ++i) {
      if (i & 1) hi ^= mix64(lo ^ k.round[i]) & k.hi_mask;
      else lo ^= mix64(hi ^ k.round[i]) & k.lo_mask;
    }
    x = (hi << k.lo_bits) | lo;
  } while (x >= k.n);  // cycle-walking: terminates, the cycle through the start value returns below n
  return x;
}

// ---- the training tables: train_rows_kernel<Plan> maps table row k to its pixel through the plan's table_pixel ----
// table_pixel(plan, start, height, width, k, v, y, x) gives the pixel of table row k as (view, y, x); false for a row the plan
// does not hold (k outside [0, n_table), or a malformed plan), so a malformed plan reads and writes nothing out of bounds.
// start: the plan's prefix, staged in shared memory by the kernel when it fits.

// Every pixel of every view (hr_sample_train_batch): table row k is pixel k.  It has no view prefix, so the kernel stages
// nothing and searches nothing.  The kernel also tests kWhole where hr_sample_train_batch's arguments are fixed (permute
// mode, no table ids, the row's pixel id is k), so that instantiation does no per-row work that only the other plans need.
struct WholePlan {
  long long n_table;  // n_views*H*W
};
template <class Plan>
constexpr bool kWhole = std::is_same<Plan, WholePlan>::value;

__device__ __forceinline__ bool table_pixel(const WholePlan& plan, const int64_t*, int height, int width, long long k,
                                            int& v, int& y, int& x) {
  if (k < 0 || k >= plan.n_table) return false;
  const long long hw = (long long)height * width;
  v = (int)(k / hw);
  const long long q = k - v * hw;
  y = (int)(q / width);
  x = (int)(q - (long long)y * width);
  return true;
}

// The view of table row k, for the plans with a per-view row prefix: the last view v with start[v] <= k, and k's rank q
// within it; false for k outside [0, n_table) or a prefix that does not bracket k.
__device__ __forceinline__ bool find_view(const int64_t* start, int n_views, long long n_table, long long k, int& v,
                                          long long& q) {
  if (k < 0 || k >= n_table) return false;
  int lo = 0, hi = n_views;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (start[mid] <= k) lo = mid;
    else hi = mid;
  }
  v = lo;
  const long long s0 = start[v];
  if (k < s0 || k >= start[v + 1]) return false;
  q = k - s0;
  return true;
}

// ---- training table of per-view pixel subsets (hr_sample_train_rows) ----
// The reference's video datasets keep, per training view v, the pixels with (x + y + o_v) % s_v == 0 (datasets/technicolor.py
// :211-269, datasets/neural_3d.py:168-185,217-269; s_v = 1 keeps the whole view) and concatenate them view by view, each view's
// kept pixels in row-major order (coords[mask]).  Table row k is in view v = upper_bound(start, k) - 1 at rank q = k - start[v]
// of that view's list; start is the exclusive prefix of the per-view row counts.  Every s consecutive image rows hold exactly W
// kept pixels (for each x exactly one of them satisfies the rule), so rank q lies in rows [s*(q/W), s*(q/W) + s) and a walk of at
// most s rows finds it.  Row y's kept pixels are x0(y) + s*j, x0(y) = (s - (y + o) mod s) mod s, count(y) = x0 < W ? (W - 1 -
// x0)/s + 1 : 0.
//
// Sampling modes: HR_SAMPLE_PERMUTE, row r of batch b is table row feistel_permute(b*B + r) over [0, n_table) (the permutation
// above); HR_SAMPLE_REPLACE, row r of batch b is an independent uniform draw umulhi(h, n_table), h the splitmix64 output
// mix64(draw_key + G*(b*B + r + 1)), draw_key = mix64(mix64(seed ^ kDrawDomain) + G*(epoch + 1)).  The bias of that reduction
// is at most n_table / 2^64.  kDrawDomain keeps the draw keys apart from the Feistel keys of the same (seed, epoch).
constexpr uint64_t kDrawDomain = 0x5245504C41434531ull;  // "REPLACE1"

uint64_t draw_key(uint64_t seed, int64_t epoch) {
  return mix64(mix64(seed ^ kDrawDomain) + kGolden * ((uint64_t)epoch + 1));
}

struct TablePlan {
  const int64_t* start;  // [n_views + 1] exclusive prefix of per-view row counts
  const int32_t* rule;   // [n_views, 2] (stride, offset)
  int n_views;
  long long n_table;     // rows drawn or permuted: [0, n_table)
};

// Not held besides the rows find_view refuses: a stride < 1, or a rank past the view's last kept pixel.
__device__ __forceinline__ bool table_pixel(const TablePlan& plan, const int64_t* start, int height, int width, long long k,
                                            int& v, int& y, int& x) {
  long long q;
  if (!find_view(start, plan.n_views, plan.n_table, k, v, q)) return false;
  const int s = plan.rule[2 * v], o = plan.rule[2 * v + 1];
  if (s < 1) return false;
  long long block, rem;
  if (q <= 0x7fffffffLL) {  // 32-bit division for every view of fewer than 2^31 pixels
    block = (unsigned)q / (unsigned)width;
    rem = (unsigned)q - (unsigned)block * (unsigned)width;
  } else {
    block = q / width;
    rem = q - block * width;
  }
  if (block >= ((long long)height + s - 1) / s) return false;
  y = (int)(block * s);
  int m = (int)(((long long)y + o) % s);  // (y + o) mod s, advanced with y
  if (m < 0) m += s;
  for (int i = 0; i < s && y < height; ++i, ++y) {
    const int x0 = m == 0 ? 0 : s - m;
    const int cnt = x0 < width ? (width - 1 - x0) / s + 1 : 0;
    if (rem < cnt) {
      x = x0 + s * (int)rem;
      return true;
    }
    rem -= cnt;
    if (++m == s) m = 0;
  }
  return false;
}

// ---- training table of per-view keep masks (hr_sample_train_mask_rows) ----
// The Immersive dataset keeps per view a content-dependent set of pixels (importance_subsample), stored as a keep bitmask
// built by hr_build_importance_table below: bit (p & 31) of word p >> 5 of the view's mask is pixel p = y*W + x.  The mask's
// 256-pixel blocks (8 words each) carry the exclusive prefix of their kept counts within the view, so rank q of the view's
// kept pixels lies in the last block b with block_start[b] <= q (a binary search) and is the (q - block_start[b])-th set bit of
// that block's 8 words (a popc walk, then __fns).  A view with slot < 0 keeps every pixel (rank q is pixel q).
constexpr int kMaskBlock = 256;  // pixels per mask block: 8 words of 32 bits
constexpr int kMaskWords = kMaskBlock / 32;

struct MaskPlan {
  const int64_t* start;         // [n_views + 1] exclusive prefix of per-view row counts
  const int32_t* slot;          // [n_views] the view's mask slot, or -1 for a whole view
  const uint32_t* block_start;  // [n_slots, blocks] exclusive prefix of kept counts per block, within the view
  const uint32_t* masks;        // [n_slots, blocks, 8] keep bits
  int n_views;
  int blocks;                   // ceil(H*W / 256)
  long long n_table;            // rows drawn or permuted: [0, n_table)
};

// Not held besides the rows find_view refuses: a rank past the view's last kept pixel.
__device__ __forceinline__ bool table_pixel(const MaskPlan& plan, const int64_t* start, int height, int width, long long k,
                                            int& v, int& y, int& x) {
  long long q;
  if (!find_view(start, plan.n_views, plan.n_table, k, v, q)) return false;
  const long long hw = (long long)height * width;
  long long p = q;
  const int slot = plan.slot[v];
  if (slot >= 0) {
    if (q > 0xffffffffLL) return false;
    const uint32_t* bs = plan.block_start + (long long)slot * plan.blocks;
    int b = 0, bh = plan.blocks;  // the last block b with bs[b] <= q
    while (bh - b > 1) {
      const int mid = (b + bh) >> 1;
      if (bs[mid] <= (unsigned)q) b = mid;
      else bh = mid;
    }
    unsigned rem = (unsigned)q - bs[b];
    const uint32_t* w = plan.masks + ((long long)slot * plan.blocks + b) * kMaskWords;
    int i = 0;
    uint32_t word = w[0];
    for (unsigned c = __popc(word); rem >= c; c = __popc(word)) {
      if (++i == kMaskWords) return false;
      rem -= c;
      word = w[i];
    }
    p = (long long)b * kMaskBlock + 32 * i + (int)__fns(word, 0, (int)rem + 1);
  }
  if (p >= hw) return false;
  y = (int)(p / width);
  x = (int)(p - (long long)y * width);
  return true;
}

constexpr int kStagedViews = 4095;  // prefixes of up to this many views are staged in shared memory (32 KB)

// Plan: WholePlan (every pixel), TablePlan (a (stride, offset) rule per view) or MaskPlan (a keep mask per view).  kC: bytes
// per pixel, 3 (RGB) or 4 (RGBA, composited over white).
template <class Plan, int kC>
__global__ void __launch_bounds__(256)
train_rows_kernel(const hr_camera* __restrict__ cams, const uint8_t* __restrict__ images, int height, int width,
                  const __grid_constant__ Plan plan, const __grid_constant__ FeistelKey key, uint64_t dkey, int mode,
                  long long first, long long rows, const int64_t* __restrict__ table_rows, int c_in, float* __restrict__ coords,
                  float* __restrict__ rgb, float* __restrict__ weight, int64_t* __restrict__ pixel_ids,
                  int64_t* __restrict__ table_ids) {
  const int64_t* start = nullptr;
  if constexpr (!kWhole<Plan>) {
    extern __shared__ int64_t staged[];
    start = plan.start;
    if (plan.n_views <= kStagedViews) {  // the binary search's dependent loads then hit shared memory
      for (int i = threadIdx.x; i <= plan.n_views; i += blockDim.x) staged[i] = plan.start[i];
      __syncthreads();
      start = staged;
    }
  }
  const long long hw = (long long)height * width;
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x) {
    long long k;
    if (table_rows) k = (long long)table_rows[r];
    else if (kWhole<Plan> || mode == HR_SAMPLE_PERMUTE) k = (long long)feistel_permute((uint64_t)(first + r), key);
    else k = (long long)__umul64hi(mix64(dkey + kGolden * ((uint64_t)(first + r) + 1)), (uint64_t)plan.n_table);
    float row[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, w = 0.f;
    long long p = -1;
    int v, y, x;
    if (table_pixel(plan, start, height, width, k, v, y, x)) {
      p = kWhole<Plan> ? k : v * hw + (long long)y * width + x;
      const hr_camera& cam = cams[v];
      camera_ray<true, true>(cam, x, y, ndc_scale(cam), row);
      if constexpr (kC == 4) {
        const uint32_t q = *reinterpret_cast<const uint32_t*>(images + 4 * p);  // 4-byte aligned (checked by the host)
        c0 = rgba_over_white(q, 0);
        c1 = rgba_over_white(q, 1);
        c2 = rgba_over_white(q, 2);
      } else {
        const uint8_t* px = images + 3 * p;
        c0 = u8_unit(px[0]);
        c1 = u8_unit(px[1]);
        c2 = u8_unit(px[2]);
      }
      w = 1.0f;
    } else {
      k = -1;  // a row the plan does not hold: a zero row of weight 0 (the Python binding validates plans and rows)
    }
    float2* cr = reinterpret_cast<float2*>(coords + r * c_in);
    cr[0] = make_float2(row[0], row[1]);
    cr[1] = make_float2(row[2], row[3]);
    cr[2] = make_float2(row[4], row[5]);
    if (c_in == 8) cr[3] = make_float2(row[6], row[7]);
    rgb[3 * r + 0] = c0;
    rgb[3 * r + 1] = c1;
    rgb[3 * r + 2] = c2;
    weight[r] = w;
    if (pixel_ids) pixel_ids[r] = p;
    if (!kWhole<Plan> && table_ids) table_ids[r] = k;
  }
}

// ---- importance table build (hr_build_importance_table) ----
// ImmersiveDataset.importance_subsample (datasets/immersive.py:295-321) keeps, of a frame with N = H*W pixels, the pixels with
// diff > thr and dz < -0.05, diff = mean over the channels of |rgb - last_rgb| (both u8 / 255 in fp32, last_rgb the previous
// frame of the same video) and thr = the value of ascending rank (N - num_take) % N of diff (Python's sorted[-num_take]).
// diff is the key: the fp32 bits of a non-negative float order as uint32, so thr is an exact radix select over the keys, three
// histogram passes of 11, 11 and 10 bits with integer atomics (kSelectBits), each followed by a one-block select that narrows
// (prefix, rank) to the bin holding the rank.  The keys are recomputed from the uint8 frames in every pass: 6 bytes read per
// pixel instead of 4 B of stored key per pixel.  Then the mask pass packs the keep bits with ballot and counts them per block,
// a per-view scan turns the block counts into block_start, and a one-block scan gives every view's row count and the int64
// prefix over views.
constexpr int kSelectBins = 2048;
__host__ __device__ constexpr int select_shift(int pass) { return pass == 0 ? 21 : pass == 1 ? 10 : 0; }
__host__ __device__ constexpr int select_bits(int pass) { return pass == 2 ? 10 : 11; }

struct ImportanceSlot {
  int32_t view;  // the importance view; its previous frame is view - 1
  uint32_t rank; // ascending rank of the threshold, (N - num_take) % N
};

// mean(|rgb - last_rgb|, -1) with torch's operation order on CPU: ((d0 + d1) + d2) / 3, every step rounded, no contraction.
__device__ __forceinline__ uint32_t diff_key(const uint8_t* cur, const uint8_t* prev) {
  float d[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) d[c] = fabsf(__fsub_rn(u8_unit(cur[c]), u8_unit(prev[c])));
  return __float_as_uint(__fdiv_rn(__fadd_rn(__fadd_rn(d[0], d[1]), d[2]), 3.0f));
}

// Inclusive scan over a CTA of kThreads threads, one value per thread, through the shared array part[kThreads]; returns this
// thread's inclusive sum.  Ends with a barrier, so every thread may then read any element of part.
template <class T, int kThreads>
__device__ __forceinline__ T block_inclusive_scan(T* part, T value) {
  const int t = threadIdx.x;
  part[t] = value;
  __syncthreads();
  for (int off = 1; off < kThreads; off <<= 1) {
    const T add = t >= off ? part[t - off] : T(0);
    __syncthreads();
    part[t] += add;
    __syncthreads();
  }
  return part[t];
}

// grid (chunks, n_slots): histogram of pass kPass over the keys whose bits above this pass's equal the slot's prefix.
template <int kPass>
__global__ void __launch_bounds__(256)
importance_hist_kernel(const uint8_t* __restrict__ images, long long hw, const ImportanceSlot* __restrict__ slots,
                       const uint32_t* __restrict__ state, uint32_t* __restrict__ hist) {
  __shared__ uint32_t h[kSelectBins];
  for (int i = threadIdx.x; i < kSelectBins; i += blockDim.x) h[i] = 0;
  __syncthreads();
  const int s = blockIdx.y;
  const ImportanceSlot slot = slots[s];
  const uint8_t* cur = images + 3 * (long long)slot.view * hw;
  const uint8_t* prev = cur - 3 * hw;
  constexpr int shift = select_shift(kPass), above = shift + select_bits(kPass);
  const uint32_t prefix = kPass == 0 ? 0u : state[2 * s];
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < hw; p += (long long)gridDim.x * blockDim.x) {
    const uint32_t key = diff_key(cur + 3 * p, prev + 3 * p);
    if (kPass == 0 || (key >> (above & 31)) == (prefix >> (above & 31)))
      atomicAdd(&h[(key >> shift) & ((1u << select_bits(kPass)) - 1)], 1u);
  }
  __syncthreads();
  uint32_t* g = hist + (long long)s * kSelectBins;
  for (int i = threadIdx.x; i < kSelectBins; i += blockDim.x)
    if (h[i]) atomicAdd(&g[i], h[i]);
}

// grid n_slots, 256 threads: the bin of pass kPass that holds the slot's remaining rank; clears the histogram for the next
// pass.  state[2 s] is the threshold's bits found so far, state[2 s + 1] the rank left within them.
template <int kPass>
__global__ void __launch_bounds__(256)
importance_select_kernel(const ImportanceSlot* __restrict__ slots, uint32_t* __restrict__ state, uint32_t* __restrict__ hist) {
  constexpr int kPer = kSelectBins / 256;
  __shared__ uint32_t part[256];
  const int s = blockIdx.x, t = threadIdx.x;
  uint32_t* g = hist + (long long)s * kSelectBins;
  uint32_t c[kPer], sum = 0;
#pragma unroll
  for (int j = 0; j < kPer; ++j) {
    c[j] = g[t * kPer + j];
    sum += c[j];
  }
  const uint32_t incl = block_inclusive_scan<uint32_t, 256>(part, sum);
  const uint32_t prefix = kPass == 0 ? 0u : state[2 * s];
  const uint32_t rank = kPass == 0 ? slots[s].rank : state[2 * s + 1];
  uint32_t before = incl - sum;
  __syncthreads();  // every thread has read state before the owner of the rank overwrites it
  if (rank >= before && rank < incl) {
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      if (rank < before + c[j]) {
        state[2 * s] = prefix | ((uint32_t)(t * kPer + j) << select_shift(kPass));
        state[2 * s + 1] = rank - before;
        break;
      }
      before += c[j];
    }
  }
#pragma unroll
  for (int j = 0; j < kPer; ++j) g[t * kPer + j] = 0u;
}

// grid (chunks, n_slots), 256 threads: one thread per pixel of a 256-pixel mask block.  Writes the block's 8 keep words and
// its kept count (into block_start, scanned by importance_scan_kernel).
__global__ void __launch_bounds__(256)
importance_mask_kernel(const hr_camera* __restrict__ cams, const uint8_t* __restrict__ images, int height, int width,
                       int blocks, const ImportanceSlot* __restrict__ slots, const uint32_t* __restrict__ state,
                       uint32_t* __restrict__ masks, uint32_t* __restrict__ block_start) {
  __shared__ uint32_t counts[kMaskWords];
  const int s = blockIdx.y;
  const ImportanceSlot slot = slots[s];
  const long long hw = (long long)height * width;
  const uint8_t* cur = images + 3 * (long long)slot.view * hw;
  const uint8_t* prev = cur - 3 * hw;
  const uint32_t thr = state[2 * s];
  const hr_camera& cam = cams[slot.view];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int b = blockIdx.x; b < blocks; b += gridDim.x) {
    const long long p = (long long)b * kMaskBlock + threadIdx.x;
    bool keep = false;
    if (p < hw && diff_key(cur + 3 * p, prev + 3 * p) > thr) {
      const int y = (int)(p / width), x = (int)(p - (long long)y * width);
      float row[8];
      camera_ray<true, true>(cam, x, y, ndc_scale(cam), row);
      keep = row[5] < -0.05f;  // coords[..., 5] < -0.05 of an fp32 tensor compares in fp32
    }
    const uint32_t bits = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) {
      masks[((long long)s * blocks + b) * kMaskWords + warp] = bits;
      counts[warp] = __popc(bits);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t n = 0;
#pragma unroll
      for (int i = 0; i < kMaskWords; ++i) n += counts[i];
      block_start[(long long)s * blocks + b] = n;
    }
    __syncthreads();
  }
}

// grid n_slots, 256 threads: exclusive scan of the slot's block counts in place; the total is the view's row count.
__global__ void __launch_bounds__(256)
importance_scan_kernel(int blocks, const ImportanceSlot* __restrict__ slots, uint32_t* __restrict__ block_start,
                       int64_t* __restrict__ view_rows) {
  __shared__ uint32_t part[256];
  const int s = blockIdx.x, t = threadIdx.x;
  uint32_t* bs = block_start + (long long)s * blocks;
  const int per = (blocks + 255) / 256, b0 = min(blocks, t * per), b1 = min(blocks, b0 + per);
  uint32_t sum = 0;
  for (int b = b0; b < b1; ++b) sum += bs[b];
  const uint32_t incl = block_inclusive_scan<uint32_t, 256>(part, sum);
  uint32_t run = incl - sum;
  for (int b = b0; b < b1; ++b) {
    const uint32_t n = bs[b];
    bs[b] = run;
    run += n;
  }
  if (t == 255) view_rows[slots[s].view] = incl;
}

// one block of 1024 threads: whole views' row counts (H*W) and the exclusive int64 prefix over all views.
__global__ void __launch_bounds__(1024)
importance_views_kernel(int n_views, long long hw, const int32_t* __restrict__ view_slot, int64_t* __restrict__ view_rows,
                        int64_t* __restrict__ view_start) {
  __shared__ long long part[1024];
  const int t = threadIdx.x;
  const int per = (n_views + 1023) / 1024, v0 = min(n_views, t * per), v1 = min(n_views, v0 + per);
  long long sum = 0;
  for (int v = v0; v < v1; ++v) {
    if (view_slot[v] < 0) view_rows[v] = hw;
    sum += view_rows[v];
  }
  long long run = block_inclusive_scan<long long, 1024>(part, sum) - sum;
  if (t == 0) view_start[0] = 0;
  for (int v = v0; v < v1; ++v) {
    run += view_rows[v];
    view_start[v + 1] = run;
  }
}

}  // namespace
}  // namespace hr

namespace {

// The checks, batch range and launch shared by the three sampling entry points; `plan` carries the table, kC the bytes per
// pixel of `images` (3 or 4).
template <class Plan, int kC = 3>
int sample_rows(const char* fn, const Plan& plan, const hr_camera* cameras, int32_t n_views, const uint8_t* images,
                int32_t height, int32_t width, int32_t c_in, int32_t mode, uint64_t seed, int64_t epoch, int64_t batch_index,
                int64_t batch_size, const int64_t* table_rows, float* coords, float* rgb, float* weight, int64_t* pixel_ids,
                int64_t* table_ids, int64_t* n_rows, void* stream) {
  if (n_views < 1 || height < 1 || width < 1)
    return hr_fail("%s: bad image stack %d x %d x %d", fn, n_views, height, width);
  if (c_in != 6 && c_in != 8) return hr_fail("%s: c_in must be 6 or 8, got %d", fn, c_in);
  if (mode != HR_SAMPLE_PERMUTE && mode != HR_SAMPLE_REPLACE) return hr_fail("%s: unknown mode %d", fn, mode);
  if (batch_size < 1) return hr_fail("%s: batch_size must be >= 1, got %lld", fn, (long long)batch_size);
  uintptr_t view_start = 0;  // WholePlan has none
  if constexpr (!hr::kWhole<Plan>) view_start = (uintptr_t)plan.start;
  if (((uintptr_t)coords % 8) || ((uintptr_t)rgb % 4) || ((uintptr_t)weight % 4) || ((uintptr_t)pixel_ids % 8) ||
      ((uintptr_t)table_ids % 8) || ((uintptr_t)table_rows % 8) || (view_start % 8) || ((uintptr_t)cameras % 4))
    return hr_fail("%s: misaligned pointer (coords, view_start and the int64 row arrays need 8 bytes, the rest 4)", fn);
  if (kC == 4 && ((uintptr_t)images % 4)) return hr_fail("%s: misaligned pointer (RGBA images need 4 bytes)", fn);
  const uint64_t n = (uint64_t)n_views * (uint64_t)height * (uint64_t)width;
  if (n > (1ull << 62)) return hr_fail("%s: %llu pixels, at most 2^62", fn, (unsigned long long)n);
  const int64_t n_table = plan.n_table;
  if (n_table < 1 || (uint64_t)n_table > n)
    return hr_fail("%s: n_table %lld outside [1, %llu]", fn, (long long)n_table, (unsigned long long)n);
  long long first = 0, rows = batch_size;
  if (!table_rows) {
    if (batch_index < 0) return hr_fail("%s: batch_index %lld < 0", fn, (long long)batch_index);
    if (mode == HR_SAMPLE_PERMUTE) {
      const int64_t n_batches = (n_table - 1) / batch_size + 1;  // ceil(n_table / batch_size) without overflow
      if (batch_index >= n_batches)
        return hr_fail("%s: batch_index %lld outside [0, %lld)", fn, (long long)batch_index, (long long)n_batches);
      first = batch_index * batch_size;
      if (rows > n_table - first) rows = n_table - first;  // the epoch's short last batch
    } else {
      if (batch_index > (INT64_MAX - batch_size) / batch_size)
        return hr_fail("%s: batch_index %lld too large", fn, (long long)batch_index);
      first = batch_index * batch_size;
    }
  }
  const hr::FeistelKey key = hr::feistel_key(seed, epoch, (uint64_t)n_table);
  long long g = (rows + 255) / 256;
  if (g > 148 * 16) g = 148 * 16;
  const size_t smem =
      !hr::kWhole<Plan> && n_views <= hr::kStagedViews ? (size_t)(n_views + 1) * sizeof(int64_t) : 0;
  hr::train_rows_kernel<Plan, kC><<<(unsigned)g, 256, smem, (cudaStream_t)stream>>>(
      cameras, images, height, width, plan, key, hr::draw_key(seed, epoch), mode, first, rows, table_rows, c_in, coords, rgb,
      weight, pixel_ids, table_ids);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return hr_fail("%s: %s", fn, cudaGetErrorString(e));
  if (n_rows) *n_rows = rows;
  return 0;
}

// Workspace of hr_build_importance_table: the slots, the select state and one histogram per slot.
size_t importance_workspace(int64_t n_slots) {
  return align256((size_t)n_slots * sizeof(hr::ImportanceSlot)) + align256((size_t)n_slots * 2 * sizeof(uint32_t)) +
         (size_t)n_slots * hr::kSelectBins * sizeof(uint32_t);
}

}  // namespace

extern "C" int hr_sample_train_batch(const hr_camera* cameras, int32_t n_views, const uint8_t* images, int32_t pixel_format,
                                     int32_t height, int32_t width, int32_t c_in, uint64_t seed, int64_t epoch,
                                     int64_t batch_index, int64_t batch_size, const int64_t* order, float* coords, float* rgb,
                                     float* weight, int64_t* pixel_ids, int64_t* n_rows, void* stream) {
  const char* fn = "hr_sample_train_batch";
  if (!cameras || !images || !coords || !rgb || !weight) return hr_fail("%s: null argument", fn);
  if (((uintptr_t)coords % 8) || ((uintptr_t)rgb % 4) || ((uintptr_t)weight % 4) || ((uintptr_t)pixel_ids % 8) ||
      ((uintptr_t)order % 8) || ((uintptr_t)cameras % 4))
    return hr_fail("%s: misaligned pointer (coords and pixel_ids / order need 8 bytes, the rest 4)", fn);
  const int px = hr::pixel_bytes(pixel_format);
  if (!px) return hr_fail("%s: unknown pixel format %d", fn, pixel_format);
  // the table is every pixel (sample_rows refuses a bad image stack and more than 2^62 pixels before n_table is used)
  const hr::WholePlan plan{(long long)((uint64_t)n_views * (uint64_t)height * (uint64_t)width)};
  return px == 4 ? sample_rows<hr::WholePlan, 4>(fn, plan, cameras, n_views, images, height, width, c_in, HR_SAMPLE_PERMUTE,
                                                 seed, epoch, batch_index, batch_size, order, coords, rgb, weight,
                                                 pixel_ids, nullptr, n_rows, stream)
                 : sample_rows(fn, plan, cameras, n_views, images, height, width, c_in, HR_SAMPLE_PERMUTE, seed, epoch,
                               batch_index, batch_size, order, coords, rgb, weight, pixel_ids, nullptr, n_rows, stream);
}

extern "C" int hr_sample_train_rows(const hr_camera* cameras, int32_t n_views, const uint8_t* images, int32_t pixel_format,
                                    int32_t height, int32_t width, int32_t c_in, const int64_t* view_start,
                                    const int32_t* view_rule, int64_t n_table, int32_t mode, uint64_t seed, int64_t epoch,
                                    int64_t batch_index, int64_t batch_size, const int64_t* table_rows, float* coords,
                                    float* rgb, float* weight, int64_t* pixel_ids, int64_t* table_ids, int64_t* n_rows,
                                    void* stream) {
  const char* fn = "hr_sample_train_rows";
  if (!cameras || !images || !view_start || !view_rule || !coords || !rgb || !weight) return hr_fail("%s: null argument", fn);
  if ((uintptr_t)view_rule % 4) return hr_fail("%s: misaligned pointer (view_rule needs 4 bytes)", fn);
  const int px = hr::pixel_bytes(pixel_format);
  if (!px) return hr_fail("%s: unknown pixel format %d", fn, pixel_format);
  const hr::TablePlan plan{view_start, view_rule, n_views, n_table};
  return px == 4 ? sample_rows<hr::TablePlan, 4>(fn, plan, cameras, n_views, images, height, width, c_in, mode, seed,
                                                 epoch, batch_index, batch_size, table_rows, coords, rgb, weight,
                                                 pixel_ids, table_ids, n_rows, stream)
                 : sample_rows(fn, plan, cameras, n_views, images, height, width, c_in, mode, seed, epoch, batch_index,
                               batch_size, table_rows, coords, rgb, weight, pixel_ids, table_ids, n_rows, stream);
}

extern "C" int hr_sample_train_mask_rows(const hr_camera* cameras, int32_t n_views, const uint8_t* images, int32_t height,
                                         int32_t width, int32_t c_in, const int64_t* view_start, const int32_t* view_slot,
                                         const uint32_t* block_start, const uint32_t* masks, int64_t n_table, int32_t mode,
                                         uint64_t seed, int64_t epoch, int64_t batch_index, int64_t batch_size,
                                         const int64_t* table_rows, float* coords, float* rgb, float* weight,
                                         int64_t* pixel_ids, int64_t* table_ids, int64_t* n_rows, void* stream) {
  if (!cameras || !images || !view_start || !view_slot || !coords || !rgb || !weight)
    return hr_fail("hr_sample_train_mask_rows: null argument");
  if (((uintptr_t)view_slot % 4) || ((uintptr_t)block_start % 4) || ((uintptr_t)masks % 4))
    return hr_fail("hr_sample_train_mask_rows: misaligned pointer (view_slot, block_start and masks need 4 bytes)");
  if ((int64_t)height * width >= (1ll << 31))
    return hr_fail("hr_sample_train_mask_rows: %lld pixels per view, at most 2^31 - 1", (long long)height * width);
  const int blocks = (int)(((int64_t)height * width + hr::kMaskBlock - 1) / hr::kMaskBlock);
  const hr::MaskPlan plan{view_start, view_slot, block_start, masks, n_views, blocks, n_table};
  return sample_rows("hr_sample_train_mask_rows", plan, cameras, n_views, images, height, width, c_in, mode, seed, epoch,
                     batch_index, batch_size, table_rows, coords, rgb, weight, pixel_ids, table_ids, n_rows, stream);
}

extern "C" int64_t hr_importance_workspace_bytes(int32_t n_slots) {
  return n_slots < 0 ? -1 : (int64_t)importance_workspace(n_slots);
}

extern "C" int hr_build_importance_table(const hr_camera* cameras, int32_t n_views, const uint8_t* images, int32_t height,
                                         int32_t width, const int64_t* plan, void* workspace, int64_t workspace_bytes,
                                         int32_t* view_slot, uint32_t* block_start, uint32_t* masks, int64_t* view_rows,
                                         int64_t* view_start, void* stream) {
  const char* fn = "hr_build_importance_table";
  if (!cameras || !images || !plan || !view_slot || !view_rows || !view_start) return hr_fail("%s: null argument", fn);
  if (n_views < 1 || height < 1 || width < 1)
    return hr_fail("%s: bad image stack %d x %d x %d", fn, n_views, height, width);
  const int64_t hw = (int64_t)height * width;
  if (hw >= (1ll << 31)) return hr_fail("%s: %lld pixels per view, at most 2^31 - 1", fn, (long long)hw);
  std::vector<int32_t> slot(n_views, -1);
  std::vector<hr::ImportanceSlot> slots;
  for (int v = 0; v < n_views; ++v) {
    const int64_t take = plan[2 * v], prev = plan[2 * v + 1];
    if (take == -1 && prev == -1) continue;  // a whole view
    if (take < 0 || take > hw)
      return hr_fail("%s: view %d takes %lld pixels, outside [0, %lld]", fn, v, (long long)take, (long long)hw);
    if (prev != v - 1 || v == 0)
      return hr_fail("%s: view %d's previous frame is view %lld, it must be view %d of the same video", fn, v,
                     (long long)prev, v - 1);
    slot[v] = (int32_t)slots.size();
    slots.push_back({v, (uint32_t)((hw - take) % hw)});
  }
  const int64_t n_slots = (int64_t)slots.size();
  if (n_slots > 65535) return hr_fail("%s: %lld importance views, at most 65535 per call", fn, (long long)n_slots);
  if (n_slots > 0 && (!block_start || !masks || !workspace)) return hr_fail("%s: null argument", fn);
  if (((uintptr_t)cameras % 4) || ((uintptr_t)view_slot % 4) || ((uintptr_t)block_start % 4) || ((uintptr_t)masks % 4) ||
      ((uintptr_t)view_rows % 8) || ((uintptr_t)view_start % 8) || ((uintptr_t)workspace % 256))
    return hr_fail("%s: misaligned pointer (view_rows and view_start need 8 bytes, workspace 256, the rest 4)", fn);
  if (workspace_bytes < (int64_t)importance_workspace(n_slots))
    return hr_fail("%s: workspace of %lld bytes, %lld needed", fn, (long long)workspace_bytes,
                   (long long)importance_workspace(n_slots));
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemcpyAsync(view_slot, slot.data(), slot.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess && n_slots > 0) {
    char* ws = (char*)workspace;
    auto* dslots = (hr::ImportanceSlot*)ws;
    auto* state = (uint32_t*)(ws + align256((size_t)n_slots * sizeof(hr::ImportanceSlot)));
    auto* hist = (uint32_t*)((char*)state + align256((size_t)n_slots * 2 * sizeof(uint32_t)));
    const int blocks = (int)((hw + hr::kMaskBlock - 1) / hr::kMaskBlock);
    // about 16 blocks of 256 threads per SM over all slots, each block a slice of one view
    const unsigned chunks = (unsigned)std::max<int64_t>(1, std::min<int64_t>(blocks, (148 * 16 + n_slots - 1) / n_slots));
    const dim3 grid(chunks, (unsigned)n_slots);
    e = cudaMemcpyAsync(dslots, slots.data(), slots.size() * sizeof(hr::ImportanceSlot), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(hist, 0, (size_t)n_slots * hr::kSelectBins * sizeof(uint32_t), st);
    if (e == cudaSuccess) {
      hr::importance_hist_kernel<0><<<grid, 256, 0, st>>>(images, hw, dslots, state, hist);
      hr::importance_select_kernel<0><<<(unsigned)n_slots, 256, 0, st>>>(dslots, state, hist);
      hr::importance_hist_kernel<1><<<grid, 256, 0, st>>>(images, hw, dslots, state, hist);
      hr::importance_select_kernel<1><<<(unsigned)n_slots, 256, 0, st>>>(dslots, state, hist);
      hr::importance_hist_kernel<2><<<grid, 256, 0, st>>>(images, hw, dslots, state, hist);
      hr::importance_select_kernel<2><<<(unsigned)n_slots, 256, 0, st>>>(dslots, state, hist);
      hr::importance_mask_kernel<<<grid, 256, 0, st>>>(cameras, images, height, width, blocks, dslots, state, masks,
                                                        block_start);
      hr::importance_scan_kernel<<<(unsigned)n_slots, 256, 0, st>>>(blocks, dslots, block_start, view_rows);
      e = cudaGetLastError();
    }
  }
  if (e == cudaSuccess) {
    hr::importance_views_kernel<<<1, 1024, 0, st>>>(n_views, hw, view_slot, view_rows, view_start);
    e = cudaGetLastError();
  }
  if (e != cudaSuccess) return hr_fail("%s: %s", fn, cudaGetErrorString(e));
  return 0;
}
