// A17 — 8x convex upsampling with border-masked softmax over the 3x3 neighbourhood.
//
// Replaces cvx_upsample (reference utils/flow_viz.py:166-183), called on inverse depths and on
// depth covariances at slam/visual_frontends/visual_frontend.py:444-446.
//   data [K,ht,wd] fp32, mask [K,576,ht,wd] (fp16 under autocast, or fp32),  out [K,8ht,8wd] fp32
//   mask channel = n9*64 + sy*8 + sx, n9 = 3*(dy+1) + (dx+1); neighbours that fall outside the
//   image get -inf BEFORE the softmax (the reference writes -inf into the mask tensor in place;
//   we only mask functionally and never mutate the caller's tensor);
//   for an fp16 mask the softmax weights are rounded to fp16 like torch.softmax(half) does.
//
// Reference: F.unfold + a 7-D broadcast product.  Here one CTA handles one coarse row segment of
// 32 pixels: the 576x32 mask slab is read once, coalesced along x, into shared memory and the
// 8x256 output patch is written with coalesced rows.  Algorithmic bytes per depth map at 640x480:
// 576*4800*2 (mask fp16) + 4800*4 + 307200*4 = 6.8 MB.
#include "common.cuh"

namespace nslam {

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }

constexpr int UX = 32;        // coarse pixels per CTA
constexpr int UROW = 576 + 8; // smem row (one coarse pixel) for channels-last masks: +8 halfs keeps the
                              // 4 pixels a warp touches on distinct banks

// grid: (ceil(wd/UX), ht, K)  block: 256.  Up to two data planes share one softmax (inverse depth
// and its covariance are upsampled with the same mask, visual_frontend.py:444-446).
template <typename T, bool NHWC>
__global__ void __launch_bounds__(256)
cvx_upsample_kernel(const float* __restrict__ data, const float* __restrict__ data2, const T* __restrict__ mask,
                    float* __restrict__ out, float* __restrict__ out2, const long long* __restrict__ index,
                    int ht, int wd, float pw) {
  extern __shared__ unsigned char smraw[];
  T* ms = reinterpret_cast<T*>(smraw);  // NHWC: [UX][UROW]   NCHW: [576][UX]
  __shared__ float nb[2][3][UX + 2];
  const int k = blockIdx.z, y = blockIdx.y, x0 = blockIdx.x * UX;
  const int hw = ht * wd;
  const size_t kd = index ? (size_t)index[k] : (size_t)k;     // row of data / out this mask plane applies to
  if (NHWC) {
    // channels-last mask [K,ht,wd,576] (what the tensor-core update operator produces): 16-byte copies
    const T* mk = mask + ((size_t)k * hw + (size_t)y * wd + x0) * 576;
    constexpr int V = 16 / sizeof(T), NV = 576 / V;
    for (int id = threadIdx.x; id < NV * UX; id += 256) {
      const int xx = id / NV, c = (id % NV) * V;
      uint4 v = make_uint4(0, 0, 0, 0);
      if (x0 + xx < wd) v = *reinterpret_cast<const uint4*>(mk + (size_t)xx * 576 + c);
      *reinterpret_cast<uint4*>(ms + xx * UROW + c) = v;
    }
  } else {
    const T* mk = mask + (size_t)k * 576 * hw + (size_t)y * wd + x0;
    for (int id = threadIdx.x; id < 576 * UX; id += 256) {
      const int c = id / UX, xx = id % UX;
      ms[id] = (x0 + xx < wd) ? mk[(size_t)c * hw + xx] : T(0);
    }
  }
  for (int id = threadIdx.x; id < 2 * 3 * (UX + 2); id += 256) {
    const int pl = id / (3 * (UX + 2)), r = (id / (UX + 2)) % 3, xx = id % (UX + 2);
    const int yy = y + r - 1, xg = x0 + xx - 1;
    const float* src = pl ? data2 : data;
    nb[pl][r][xx] = (src && yy >= 0 && yy < ht && xg >= 0 && xg < wd) ? src[kd * hw + yy * wd + xg] : 0.f;
  }
  __syncthreads();
  // 8 x (8*UX) outputs; thread -> (sy, X)
  const int W8 = 8 * wd;
  for (int id = threadIdx.x; id < 8 * 8 * UX; id += 256) {
    const int sy = id / (8 * UX), X = id % (8 * UX);
    const int xx = X / 8, sx = X % 8;
    const int x = x0 + xx;
    if (x >= wd) continue;
    float m[9], mx = -INFINITY;
#pragma unroll
    for (int n = 0; n < 9; n++) {
      const int dy = n / 3 - 1, dx = n % 3 - 1;
      const bool inb = (y + dy >= 0) && (y + dy < ht) && (x + dx >= 0) && (x + dx < wd);
      const int c = n * 64 + sy * 8 + sx;
      m[n] = inb ? to_f<T>(NHWC ? ms[xx * UROW + c] : ms[c * UX + xx]) : -INFINITY;
      mx = fmaxf(mx, m[n]);
    }
    float e[9], sum = 0.f;
#pragma unroll
    for (int n = 0; n < 9; n++) { e[n] = expf(m[n] - mx); sum += e[n]; }
    float acc = 0.f, acc2 = 0.f;
#pragma unroll
    for (int n = 0; n < 9; n++) {
      float wgt = e[n] / sum;
      if (sizeof(T) == 2) wgt = __half2float(__float2half_rn(wgt));
      if (pw != 1.0f) wgt = powf(wgt, pw);
      acc += wgt * nb[0][n / 3][xx + n % 3];
      acc2 += wgt * nb[1][n / 3][xx + n % 3];
    }
    const size_t o = (kd * 8 * ht + (size_t)y * 8 + sy) * W8 + (size_t)x0 * 8 + X;
    out[o] = acc;
    if (out2) out2[o] = acc2;
  }
}

template <typename T, bool NHWC>
static int launch_upsample(const float* data, const float* data2, const void* mask, float* out, float* out2,
                           const long long* index, int K, int ht, int wd, float pw, cudaStream_t st) {
  dim3 grid((wd + UX - 1) / UX, ht, K);
  const size_t smem = (NHWC ? (size_t)UX * UROW : (size_t)576 * UX) * sizeof(T);
  if (cudaError_t e = ensure_dyn_smem<cvx_upsample_kernel<T, NHWC>>(smem)) return (int)e;
  cvx_upsample_kernel<T, NHWC><<<grid, 256, smem, st>>>(data, data2, (const T*)mask, out, out2, index, ht, wd, pw);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

}  // namespace nslam

/* data2/out2 may be NULL (single plane) */
extern "C" int nslam_cvx_upsample2(const float* data, const float* data2, const void* mask, int mask_dtype,
                                   float* out, float* out2, const long long* index, int K, int ht, int wd,
                                   float pw, int mask_nhwc, void* stream) {
  using namespace nslam;
  if (K == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (mask_dtype == 0)
    return mask_nhwc ? launch_upsample<__half, true>(data, data2, mask, out, out2, index, K, ht, wd, pw, st)
                     : launch_upsample<__half, false>(data, data2, mask, out, out2, index, K, ht, wd, pw, st);
  if (mask_dtype == 1)
    return mask_nhwc ? launch_upsample<float, true>(data, data2, mask, out, out2, index, K, ht, wd, pw, st)
                     : launch_upsample<float, false>(data, data2, mask, out, out2, index, K, ht, wd, pw, st);
  return (int)cudaErrorInvalidValue;
}

extern "C" int nslam_cvx_upsample(const float* data, const void* mask, int mask_dtype, float* out,
                                  int K, int ht, int wd, float pw, int mask_nhwc, void* stream) {
  return nslam_cvx_upsample2(data, nullptr, mask, mask_dtype, out, nullptr, nullptr, K, ht, wd, pw, mask_nhwc, stream);
}
