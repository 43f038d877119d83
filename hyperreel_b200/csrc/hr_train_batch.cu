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
// One thread per row: one 3-byte gather and one 48-byte row write (plus 8 B of pixel id when asked).  No float atomics, no
// host synchronisation; two calls with the same arguments write the same bits.  The camera records live on the device, so
// each row branches on its own record's fisheye flag (camera_ray<true>) and one batch may mix fisheye and pinhole views.
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

__global__ void __launch_bounds__(256)
train_batch_kernel(const hr_camera* __restrict__ cams, const uint8_t* __restrict__ images, int height, int width,
                   const __grid_constant__ FeistelKey key, long long first, long long rows, const int64_t* __restrict__ order,
                   int c_in, float* __restrict__ coords, float* __restrict__ rgb, float* __restrict__ weight,
                   int64_t* __restrict__ pixel_ids) {
  const long long hw = (long long)height * width;
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x) {
    long long p = order ? (long long)order[r] : (long long)feistel_permute((uint64_t)(first + r), key);
    float row[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, w = 0.f;
    if (p >= 0 && p < (long long)key.n) {
      const int v = (int)(p / hw);
      const long long q = p - v * hw;
      const int y = (int)(q / width), x = (int)(q - (long long)y * width);
      const hr_camera& cam = cams[v];
      camera_ray<true>(cam, x, y, ndc_scale(cam), row);
      const uint8_t* px = images + 3 * p;
      c0 = __fdiv_rn((float)px[0], 255.0f);
      c1 = __fdiv_rn((float)px[1], 255.0f);
      c2 = __fdiv_rn((float)px[2], 255.0f);
      w = 1.0f;
    } else {
      p = -1;  // an explicit order entry outside [0, N): a zero row of weight 0 (the host binding refuses such orders)
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
  }
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

// The pixel of table row k as (view, y, x); false for a row the plan does not hold (k outside [0, n_table), a start prefix
// that does not bracket k, a stride < 1, or a rank past the view's last kept pixel), so a malformed plan reads and writes
// nothing out of bounds.
// start: the plan's prefix, staged in shared memory by the caller when it fits.
__device__ __forceinline__ bool table_pixel(const TablePlan& plan, const int64_t* start, int height, int width, long long k,
                                            int& v, int& y, int& x) {
  if (k < 0 || k >= plan.n_table) return false;
  int lo = 0, hi = plan.n_views;  // the largest v in [0, n_views) with start[v] <= k
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (start[mid] <= k) lo = mid;
    else hi = mid;
  }
  v = lo;
  const long long s0 = start[v];
  if (k < s0 || k >= start[v + 1]) return false;
  const int s = plan.rule[2 * v], o = plan.rule[2 * v + 1];
  if (s < 1) return false;
  const long long q = k - s0;
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

constexpr int kStagedViews = 4095;  // prefixes of up to this many views are staged in shared memory (32 KB)

__global__ void __launch_bounds__(256)
train_rows_kernel(const hr_camera* __restrict__ cams, const uint8_t* __restrict__ images, int height, int width,
                  const __grid_constant__ TablePlan plan, const __grid_constant__ FeistelKey key, uint64_t dkey, int mode,
                  long long first, long long rows, const int64_t* __restrict__ table_rows, int c_in, float* __restrict__ coords,
                  float* __restrict__ rgb, float* __restrict__ weight, int64_t* __restrict__ pixel_ids,
                  int64_t* __restrict__ table_ids) {
  extern __shared__ int64_t staged[];
  const int64_t* start = plan.start;
  if (plan.n_views <= kStagedViews) {  // the binary search's dependent loads then hit shared memory
    for (int i = threadIdx.x; i <= plan.n_views; i += blockDim.x) staged[i] = plan.start[i];
    __syncthreads();
    start = staged;
  }
  const long long hw = (long long)height * width;
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x) {
    long long k;
    if (table_rows) k = (long long)table_rows[r];
    else if (mode == HR_SAMPLE_PERMUTE) k = (long long)feistel_permute((uint64_t)(first + r), key);
    else k = (long long)__umul64hi(mix64(dkey + kGolden * ((uint64_t)(first + r) + 1)), (uint64_t)plan.n_table);
    float row[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, w = 0.f;
    long long p = -1;
    int v, y, x;
    if (table_pixel(plan, start, height, width, k, v, y, x)) {
      p = v * hw + (long long)y * width + x;
      const hr_camera& cam = cams[v];
      camera_ray<true>(cam, x, y, ndc_scale(cam), row);
      const uint8_t* px = images + 3 * p;
      c0 = __fdiv_rn((float)px[0], 255.0f);
      c1 = __fdiv_rn((float)px[1], 255.0f);
      c2 = __fdiv_rn((float)px[2], 255.0f);
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
    if (table_ids) table_ids[r] = k;
  }
}

}  // namespace
}  // namespace hr

extern "C" int hr_sample_train_batch(const hr_camera* cameras, int32_t n_views, const uint8_t* images, int32_t height,
                                     int32_t width, int32_t c_in, uint64_t seed, int64_t epoch, int64_t batch_index,
                                     int64_t batch_size, const int64_t* order, float* coords, float* rgb, float* weight,
                                     int64_t* pixel_ids, int64_t* n_rows, void* stream) {
  if (!cameras || !images || !coords || !rgb || !weight) return hr_fail("hr_sample_train_batch: null argument");
  if (n_views < 1 || height < 1 || width < 1)
    return hr_fail("hr_sample_train_batch: bad image stack %d x %d x %d", n_views, height, width);
  if (c_in != 6 && c_in != 8) return hr_fail("hr_sample_train_batch: c_in must be 6 or 8, got %d", c_in);
  if (batch_size < 1) return hr_fail("hr_sample_train_batch: batch_size must be >= 1, got %lld", (long long)batch_size);
  if (((uintptr_t)coords % 8) || ((uintptr_t)rgb % 4) || ((uintptr_t)weight % 4) || ((uintptr_t)pixel_ids % 8) ||
      ((uintptr_t)order % 8) || ((uintptr_t)cameras % 4))
    return hr_fail("hr_sample_train_batch: misaligned pointer (coords and pixel_ids / order need 8 bytes, the rest 4)");
  const uint64_t n = (uint64_t)n_views * (uint64_t)height * (uint64_t)width;
  if (n > (1ull << 62)) return hr_fail("hr_sample_train_batch: %llu pixels, at most 2^62", (unsigned long long)n);
  long long first = 0, rows = batch_size;
  if (!order) {
    const int64_t n_batches = (int64_t)((n + (uint64_t)batch_size - 1) / (uint64_t)batch_size);
    if (batch_index < 0 || batch_index >= n_batches)
      return hr_fail("hr_sample_train_batch: batch_index %lld outside [0, %lld)", (long long)batch_index,
                     (long long)n_batches);
    first = batch_index * batch_size;
    if ((uint64_t)(first + rows) > n) rows = (long long)(n - (uint64_t)first);  // the epoch's short last batch
  }
  const hr::FeistelKey key = hr::feistel_key(seed, epoch, n);
  long long g = (rows + 255) / 256;
  if (g > 148 * 16) g = 148 * 16;
  hr::train_batch_kernel<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>(cameras, images, height, width, key, first, rows, order,
                                                                       c_in, coords, rgb, weight, pixel_ids);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return hr_fail("hr_sample_train_batch: %s", cudaGetErrorString(e));
  if (n_rows) *n_rows = rows;
  return 0;
}

extern "C" int hr_sample_train_rows(const hr_camera* cameras, int32_t n_views, const uint8_t* images, int32_t height,
                                    int32_t width, int32_t c_in, const int64_t* view_start, const int32_t* view_rule,
                                    int64_t n_table, int32_t mode, uint64_t seed, int64_t epoch, int64_t batch_index,
                                    int64_t batch_size, const int64_t* table_rows, float* coords, float* rgb, float* weight,
                                    int64_t* pixel_ids, int64_t* table_ids, int64_t* n_rows, void* stream) {
  if (!cameras || !images || !view_start || !view_rule || !coords || !rgb || !weight)
    return hr_fail("hr_sample_train_rows: null argument");
  if (n_views < 1 || height < 1 || width < 1)
    return hr_fail("hr_sample_train_rows: bad image stack %d x %d x %d", n_views, height, width);
  if (c_in != 6 && c_in != 8) return hr_fail("hr_sample_train_rows: c_in must be 6 or 8, got %d", c_in);
  if (mode != HR_SAMPLE_PERMUTE && mode != HR_SAMPLE_REPLACE) return hr_fail("hr_sample_train_rows: unknown mode %d", mode);
  if (batch_size < 1) return hr_fail("hr_sample_train_rows: batch_size must be >= 1, got %lld", (long long)batch_size);
  if (((uintptr_t)coords % 8) || ((uintptr_t)rgb % 4) || ((uintptr_t)weight % 4) || ((uintptr_t)pixel_ids % 8) ||
      ((uintptr_t)table_ids % 8) || ((uintptr_t)table_rows % 8) || ((uintptr_t)view_start % 8) ||
      ((uintptr_t)view_rule % 4) || ((uintptr_t)cameras % 4))
    return hr_fail("hr_sample_train_rows: misaligned pointer (coords, view_start and the int64 row arrays need 8 bytes, "
                   "the rest 4)");
  const uint64_t n = (uint64_t)n_views * (uint64_t)height * (uint64_t)width;
  if (n > (1ull << 62)) return hr_fail("hr_sample_train_rows: %llu pixels, at most 2^62", (unsigned long long)n);
  if (n_table < 1 || (uint64_t)n_table > n)
    return hr_fail("hr_sample_train_rows: n_table %lld outside [1, %llu]", (long long)n_table, (unsigned long long)n);
  long long first = 0, rows = batch_size;
  if (!table_rows) {
    if (batch_index < 0) return hr_fail("hr_sample_train_rows: batch_index %lld < 0", (long long)batch_index);
    if (mode == HR_SAMPLE_PERMUTE) {
      const int64_t n_batches = (n_table + batch_size - 1) / batch_size;
      if (batch_index >= n_batches)
        return hr_fail("hr_sample_train_rows: batch_index %lld outside [0, %lld)", (long long)batch_index,
                       (long long)n_batches);
      first = batch_index * batch_size;
      if (first + rows > n_table) rows = n_table - first;  // the epoch's short last batch
    } else {
      if (batch_index > (INT64_MAX - batch_size) / batch_size)
        return hr_fail("hr_sample_train_rows: batch_index %lld too large", (long long)batch_index);
      first = batch_index * batch_size;
    }
  }
  const hr::TablePlan plan{view_start, view_rule, n_views, n_table};
  const hr::FeistelKey key = hr::feistel_key(seed, epoch, (uint64_t)n_table);
  long long g = (rows + 255) / 256;
  if (g > 148 * 16) g = 148 * 16;
  const size_t smem = n_views <= hr::kStagedViews ? (size_t)(n_views + 1) * sizeof(int64_t) : 0;
  hr::train_rows_kernel<<<(unsigned)g, 256, smem, (cudaStream_t)stream>>>(cameras, images, height, width, plan, key,
                                                                      hr::draw_key(seed, epoch), mode, first, rows, table_rows,
                                                                      c_in, coords, rgb, weight, pixel_ids, table_ids);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return hr_fail("hr_sample_train_rows: %s", cudaGetErrorString(e));
  if (n_rows) *n_rows = rows;
  return 0;
}
