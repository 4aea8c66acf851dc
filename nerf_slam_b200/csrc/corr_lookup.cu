// A3 — correlation-volume lookup (bilinear (2r+1)^2 window), fused over the 4 pyramid levels.
//
// Replaces corr_index_forward_kernel (reference src/correlation_kernels.cu:19-70) and the
// python loop CorrBlock.__call__ (networks/modules/corr.py:40-50).
//
// Reference semantics kept exactly (see SURVEY.md §9.2):
//   * out[n][i][j][y][x], i <-> x-offset, j <-> y-offset, flattened channel = i*(2r+1)+j
//   * level l samples at coords / 2^l, window offsets -r .. r+1 around floor(), OOB taps add 0
//   * arithmetic in the volume dtype: for fp16 every tap contribution is
//        acc = half(acc + half(s * half(w)))   accumulated in the reference's tap order
//     (c10::Half arithmetic goes through fp32 and rounds after every operator), which is
//     what __hmul_rn/__hadd_rn compute => the fp16 path is bit-exact w.r.t. the reference.
//
// Design: instead of 4 launches that zero-fill the output and then issue up to 256
// global read-modify-writes per thread, one launch covers all levels; each thread gathers its
// (2r+2)^2 taps into registers with independent loads (64 requests in flight per thread),
// combines them in registers and writes each output channel exactly once (coalesced along x).
// Algorithmic traffic per edge at 640x480: 4.38 MB (SURVEY.md §8d).
#include <atomic>
#include <cstdlib>
#include "common.cuh"

namespace nslam {

template <typename T> struct Arith;
template <> struct Arith<__half> {
  static __device__ __forceinline__ __half zero() { return __float2half_rn(0.f); }
  static __device__ __forceinline__ __half cvt(float w) { return __float2half_rn(w); }
  static __device__ __forceinline__ __half mac(__half acc, __half s, __half w) {
    return __hadd_rn(acc, __hmul_rn(s, w));
  }
};
template <> struct Arith<float> {
  static __device__ __forceinline__ float zero() { return 0.f; }
  static __device__ __forceinline__ float cvt(float w) { return w; }
  static __device__ __forceinline__ float mac(float acc, float s, float w) {
    return __fadd_rn(acc, __fmul_rn(s, w));
  }
};

struct LookupLevels {
  const void* vol[4];
  int h2[4];
  int w2[4];
};

// grid: (ceil(h1*w1 / 128), num_levels, n)   block: 128
template <typename T, int R>
__global__ void __launch_bounds__(128)
corr_lookup_kernel(LookupLevels lv, const float* __restrict__ coords, T* __restrict__ out,
                   int h1, int w1, int num_levels, int scale_coords,
                   const int* __restrict__ slots, int nhwc_stride, int coords_nhwc) {
  constexpr int RD = 2 * R + 1;
  constexpr int NT = RD + 1;  // taps per axis
  const int hw = h1 * w1;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int l = blockIdx.y;
  const int n = blockIdx.z;
  if (p >= hw) return;

  const int h2 = lv.h2[l], w2 = lv.w2[l];
  const int vn = slots ? slots[n] : n;  // arena slot of edge n (CorrPool) or dense index
  const T* __restrict__ vol =
      reinterpret_cast<const T*>(lv.vol[l]) + ((size_t)vn * hw + p) * (size_t)(h2 * w2);

  // coords either [n,2,h1,w1] (reference layout) or [n,h1,w1,2] (what reproject produces)
  float x0, y0;
  if (coords_nhwc) {
    const float2 c = reinterpret_cast<const float2*>(coords)[(size_t)n * hw + p];
    x0 = c.x; y0 = c.y;
  } else {
    x0 = coords[((size_t)n * 2 + 0) * hw + p];
    y0 = coords[((size_t)n * 2 + 1) * hw + p];
  }
  if (scale_coords) {
    // coords / 2**l of the python caller: exact power-of-two scaling
    const float s = 1.0f / (float)(1 << l);
    x0 *= s;
    y0 *= s;
  }
  const float fx0 = floorf(x0), fy0 = floorf(y0);
  const float dx = x0 - fx0, dy = y0 - fy0;
  const int xb = (int)fx0 - R, yb = (int)fy0 - R;

  // gather taps: tap[i][j] with i = x index, j = y index
  T tap[NT][NT];
#pragma unroll
  for (int j = 0; j < NT; j++) {
    const int y1 = yb + j;
    const bool yin = (y1 >= 0) && (y1 < h2);
    const T* row = vol + (size_t)(yin ? y1 : 0) * w2;
#pragma unroll
    for (int i = 0; i < NT; i++) {
      const int x1 = xb + i;
      const bool in = yin && (x1 >= 0) && (x1 < w2);
      tap[i][j] = in ? __ldg(row + x1) : Arith<T>::zero();
    }
  }

  const T w11 = Arith<T>::cvt(dx * dy);
  const T w10 = Arith<T>::cvt(dx * (1.0f - dy));
  const T w01 = Arith<T>::cvt((1.0f - dx) * dy);
  const T w00 = Arith<T>::cvt((1.0f - dx) * (1.0f - dy));

  // output: reference layout [n][L*RD*RD][h1][w1], or channels-last [n][h1][w1][nhwc_stride]
  // (operand layout of the wgmma convolution; channels >= L*RD*RD are zero-filled by level 0)
  const size_t ostride = nhwc_stride ? 1 : (size_t)hw;
  T* __restrict__ o = nhwc_stride
                          ? out + ((size_t)n * hw + p) * nhwc_stride + (size_t)l * (RD * RD)
                          : out + ((size_t)n * num_levels + l) * (size_t)(RD * RD) * hw + p;
  if (nhwc_stride && l == 0)
    for (int c = num_levels * RD * RD; c < nhwc_stride; c++)
      out[((size_t)n * hw + p) * nhwc_stride + c] = Arith<T>::zero();
#pragma unroll
  for (int i = 0; i < RD; i++) {
#pragma unroll
    for (int j = 0; j < RD; j++) {
      // Reference visiting order for output (i,j): taps (i,j), (i,j+1), (i+1,j), (i+1,j+1).
      // OOB taps are skipped there; adding half(0*w)=+0 here is the identity on the running sum
      // except for the sign of an all-zero result (-0 vs +0), which compares equal.
      T acc = Arith<T>::zero();
      acc = Arith<T>::mac(acc, tap[i][j], w00);
      acc = Arith<T>::mac(acc, tap[i][j + 1], w01);
      acc = Arith<T>::mac(acc, tap[i + 1][j], w10);
      acc = Arith<T>::mac(acc, tap[i + 1][j + 1], w11);
      o[(size_t)(i * RD + j) * ostride] = acc;
    }
  }
}

// Channels-last variant (operand layout of the tensor-core update operator): one CTA = 32 pixels x
// 4 levels (thread = (level, pixel)); the 32 x nhwc_stride output rows are assembled in shared
// memory and written as ONE contiguous, 16-byte-vectorised chunk (32 pixels x 400 B at stride 200).
// grid: (ceil(h1*w1/32), 1, n)   block: 32 * num_levels   dynamic smem: 32 * nhwc_stride * sizeof(T)
template <typename T, int R>
__global__ void __launch_bounds__(128)
corr_lookup_nhwc_kernel(LookupLevels lv, const float* __restrict__ coords, T* __restrict__ out,
                        int h1, int w1, int num_levels, const int* __restrict__ slots,
                        int nhwc_stride, int coords_nhwc) {
  constexpr int RD = 2 * R + 1;
  constexpr int NT = RD + 1;
  extern __shared__ unsigned char lk_smem[];
  T* tile = reinterpret_cast<T*>(lk_smem);           // [32][nhwc_stride]
  const int hw = h1 * w1;
  const int pp = threadIdx.x & 31, l = threadIdx.x >> 5;
  const int p0 = blockIdx.x * 32;
  const int p = p0 + pp;
  const int n = blockIdx.z;
  // zero the padding channels
  const int used = num_levels * RD * RD;
  for (int id = threadIdx.x; id < 32 * (nhwc_stride - used); id += blockDim.x)
    tile[(id / (nhwc_stride - used)) * nhwc_stride + used + id % (nhwc_stride - used)] = Arith<T>::zero();
  if (p < hw) {
    const int h2 = lv.h2[l], w2 = lv.w2[l];
    const int vn = slots ? slots[n] : n;
    const T* __restrict__ vol = reinterpret_cast<const T*>(lv.vol[l]) + ((size_t)vn * hw + p) * (size_t)(h2 * w2);
    float x0, y0;
    if (coords_nhwc) {
      const float2 c = reinterpret_cast<const float2*>(coords)[(size_t)n * hw + p];
      x0 = c.x; y0 = c.y;
    } else {
      x0 = coords[((size_t)n * 2 + 0) * hw + p];
      y0 = coords[((size_t)n * 2 + 1) * hw + p];
    }
    const float sc = 1.0f / (float)(1 << l);
    x0 *= sc; y0 *= sc;
    const float fx0 = floorf(x0), fy0 = floorf(y0);
    const float dx = x0 - fx0, dy = y0 - fy0;
    const int xb = (int)fx0 - R, yb = (int)fy0 - R;
    T tap[NT][NT];
#pragma unroll
    for (int j = 0; j < NT; j++) {
      const int y1 = yb + j;
      const bool yin = (y1 >= 0) && (y1 < h2);
      const T* row = vol + (size_t)(yin ? y1 : 0) * w2;
#pragma unroll
      for (int i = 0; i < NT; i++) {
        const int x1 = xb + i;
        tap[i][j] = (yin && x1 >= 0 && x1 < w2) ? __ldg(row + x1) : Arith<T>::zero();
      }
    }
    const T w11 = Arith<T>::cvt(dx * dy), w10 = Arith<T>::cvt(dx * (1.0f - dy));
    const T w01 = Arith<T>::cvt((1.0f - dx) * dy), w00 = Arith<T>::cvt((1.0f - dx) * (1.0f - dy));
    T* o = tile + pp * nhwc_stride + l * (RD * RD);
#pragma unroll
    for (int i = 0; i < RD; i++) {
#pragma unroll
      for (int j = 0; j < RD; j++) {
        T acc = Arith<T>::zero();
        acc = Arith<T>::mac(acc, tap[i][j], w00);
        acc = Arith<T>::mac(acc, tap[i][j + 1], w01);
        acc = Arith<T>::mac(acc, tap[i + 1][j], w10);
        acc = Arith<T>::mac(acc, tap[i + 1][j + 1], w11);
        o[i * RD + j] = acc;
      }
    }
  }
  __syncthreads();
  // contiguous chunk: pixels p0 .. p0+31 (clipped) x nhwc_stride channels
  const int npx = min(32, hw - p0);
  const size_t bytes = (size_t)npx * nhwc_stride * sizeof(T);
  unsigned char* dst = reinterpret_cast<unsigned char*>(out + ((size_t)n * hw + p0) * nhwc_stride);
  const unsigned char* src = reinterpret_cast<const unsigned char*>(tile);
  for (size_t b = (size_t)threadIdx.x * 16; b < bytes; b += (size_t)blockDim.x * 16)
    *reinterpret_cast<uint4*>(dst + b) = *reinterpret_cast<const uint4*>(src + b);
}

// (A 128-bit variant of the kernel above — aligned 16-byte chunk pairs + a select network on levels 0/1, the CTA's
// contiguous level-2/3 slices staged in shared memory — gave bit-identical output but was slower: the two-byte gathers
// already coalesce into the same 32-byte sectors, and the select network costs more issue slots than the gathers it
// replaces.  Removed.)

template <typename T>
static int launch_lookup(const LookupLevels& lv, const float* coords, void* out, int n, int h1,
                         int w1, int num_levels, int radius, int scale_coords,
                         const int* slots, int nhwc_stride, int coords_nhwc, cudaStream_t st) {
  if (n == 0) return 0;
  if (nhwc_stride > 0 && radius == 3 && scale_coords && (nhwc_stride * sizeof(T)) % 16 == 0 && num_levels <= 4) {
    dim3 g2((h1 * w1 + 31) / 32, 1, n);
    corr_lookup_nhwc_kernel<T, 3><<<g2, 32 * num_levels, 32 * nhwc_stride * sizeof(T), st>>>(
        lv, coords, (T*)out, h1, w1, num_levels, slots, nhwc_stride, coords_nhwc);
    NSLAM_CHECK_LAUNCH();
    return 0;
  }
  dim3 grid((h1 * w1 + 127) / 128, num_levels, n), block(128);
  switch (radius) {
    case 3:
      corr_lookup_kernel<T, 3><<<grid, block, 0, st>>>(lv, coords, (T*)out, h1, w1, num_levels,
                                                      scale_coords, slots, nhwc_stride, coords_nhwc);
      break;
    case 4:
      corr_lookup_kernel<T, 4><<<grid, block, 0, st>>>(lv, coords, (T*)out, h1, w1, num_levels,
                                                      scale_coords, slots, nhwc_stride, coords_nhwc);
      break;
    case 2:
      corr_lookup_kernel<T, 2><<<grid, block, 0, st>>>(lv, coords, (T*)out, h1, w1, num_levels,
                                                      scale_coords, slots, nhwc_stride, coords_nhwc);
      break;
    case 1:
      corr_lookup_kernel<T, 1><<<grid, block, 0, st>>>(lv, coords, (T*)out, h1, w1, num_levels,
                                                      scale_coords, slots, nhwc_stride, coords_nhwc);
      break;
    default:
      return (int)cudaErrorInvalidValue;
  }
  NSLAM_CHECK_LAUNCH();
  return 0;
}

}  // namespace nslam

extern "C" {

// dtype: 0 = fp16, 1 = fp32 (volume and output share it, like the reference)
int nslam_corr_index_forward(const void* volume, int dtype, const float* coords, void* out,
                             int n, int h1, int w1, int h2, int w2, int radius, void* stream) {
  nslam::LookupLevels lv{};
  lv.vol[0] = volume; lv.h2[0] = h2; lv.w2[0] = w2;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == 0)
    return nslam::launch_lookup<__half>(lv, coords, out, n, h1, w1, 1, radius, 0, nullptr, 0, 0, st);
  if (dtype == 1)
    return nslam::launch_lookup<float>(lv, coords, out, n, h1, w1, 1, radius, 0, nullptr, 0, 0, st);
  return (int)cudaErrorInvalidValue;
}

// Fused pyramid lookup: out[n][num_levels*(2r+1)^2][h1][w1]; level l is sampled at coords/2^l.
int nslam_corr_lookup_pyramid(const void* const* volumes, const int* h2s, const int* w2s,
                              int num_levels, int dtype, const float* coords, void* out, int n,
                              int h1, int w1, int radius, const int* slots, int nhwc_stride,
                              int coords_nhwc, void* stream) {
  if (num_levels < 1 || num_levels > 4) return (int)cudaErrorInvalidValue;
  nslam::LookupLevels lv{};
  for (int l = 0; l < num_levels; l++) {
    lv.vol[l] = volumes[l]; lv.h2[l] = h2s[l]; lv.w2[l] = w2s[l];
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == 0)
    return nslam::launch_lookup<__half>(lv, coords, out, n, h1, w1, num_levels, radius, 1, slots, nhwc_stride, coords_nhwc, st);
  if (dtype == 1)
    return nslam::launch_lookup<float>(lv, coords, out, n, h1, w1, num_levels, radius, 1, slots, nhwc_stride, coords_nhwc, st);
  return (int)cudaErrorInvalidValue;
}

}  // extern "C"
