// Backward passes of the two correlation lookups (training only; the SLAM path runs without autograd).
//
// corr_index_backward  replaces corr_index_backward_kernel (reference src/correlation_kernels.cu:73-124,
//                      host :157-185).  Gradient of the bilinear (2r+1)^2 window lookup w.r.t. the volume.
// altcorr_backward     replaces altcorr_backward_kernel (reference src/altcorr_kernel.cu:152-286, host :321-356).
//                      Gradients of the on-the-fly correlation w.r.t. both feature maps (fp32).
//
// ---- corr_index_backward -------------------------------------------------------------------------------------
// volume_grad[n][y][x][y1][x1] = g(i = x1 - xb, j = y1 - yb) inside the (2r+2)^2 tap window of source pixel (y,x)
// (xb = floor(x0) - r, yb = floor(y0) - r), 0 everywhere else, with
//   g(i,j) = 0 (+) cg[i-1][j-1]*w11 (+) cg[i-1][j]*w10 (+) cg[i][j-1]*w01 (+) cg[i][j]*w00
// in that order, terms with an index outside [0, 2r] skipped, w11 = dx*dy, w10 = dx*(1-dy), w01 = (1-dx)*dy,
// w00 = (1-dx)*(1-dy) rounded to the volume dtype.  fp16: every multiply and add rounds to half (c10::Half
// arithmetic).  fp32: the reference's build contracts each step into one fused multiply-add, so this one does too.
// The reference finally stores `0 + g` into a zeroed tensor, which turns a -0 into +0; the same add is done here.
// Each source pixel owns its [h2,w2] slice, so no two threads write one element.  A CTA takes a run of consecutive
// source pixels, puts their window values into shared memory, then writes its contiguous slice range once with
// 16-byte stores, zeros included (the reference zero-fills the tensor and then read-modify-writes the windows).
//
// ---- altcorr_backward ----------------------------------------------------------------------------------------
// Per source pixel p (batch b, coordinate set n) and tap (iy, ix) at (yb+iy, xb+ix), channel = iy + (2r+1)*ix:
//   g = (cg[(iy-1)+rd(ix-1)]*dy*dx) + (cg[(iy-1)+rd*ix]*dy*(1-dx)) + (cg[iy+rd(ix-1)]*(1-dy)*dx) + (cg[iy+rd*ix]*(1-dy)*(1-dx))
//   fmap1_grad[p] += g * fmap2[tap],  fmap2_grad[tap] += g * fmap1[p]      (taps outside fmap2 contribute nothing)
// fmap1_grad is owned by p: one warp per source pixel gathers its taps in the order (n, iy, ix).
// fmap2_grad is a data-dependent scatter; the reference adds it with float atomics, in arrival order.  Here every
// sum has a fixed order, so the result is the same on every run:
//   1. key:    every (n, p) gets the bucket of its window origin (yb, xb) — a source contributes to target q iff
//              q lies in the (2r+2)^2 window at that origin — or no bucket when the window misses fmap2.  Its rank
//              among the sources of its 512-wide block with the same bucket comes from an ordered compare loop;
//              the block's count per bucket goes to a [bucket][block] table.
//   2. scan:   one ordered exclusive scan of that table per batch (integers: exact).
//   3. fill:   source s goes to record offset[bucket][block] + rank: each bucket's list is sorted by source index.
//   4. gather: one warp per target pixel q walks the buckets whose windows cover q, in bucket order; the buckets of
//              one origin row are consecutive, so that is 2r+2 contiguous record runs.  Every lane takes one record,
//              recomputes its weight g from corr_grad, and the warp adds g * fmap1[p] in record order.
// Scratch holds one record per window (not per tap), sized on the host from the shapes alone:
// 3 ints per (b, n, p) plus the bucket table, (H2+2r+1)(W2+2r+1) * ceil(N*H1*W1/512) + 1 ints per batch.
// coords_grad is left to the caller: the reference allocates it with zeros and never writes it.
#include <cstdint>
#include "common.cuh"

namespace nslam {

// ---------------------------------------------------------------------------------------------------- helpers
template <typename T> struct BwdArith;
template <> struct BwdArith<__half> {
  static __device__ __forceinline__ __half zero() { return __float2half_rn(0.f); }
  static __device__ __forceinline__ __half cvt(float w) { return __float2half_rn(w); }
  static __device__ __forceinline__ __half mac(__half acc, __half s, __half w) { return __hadd_rn(acc, __hmul_rn(s, w)); }
  static __device__ __forceinline__ __half add(__half a, __half b) { return __hadd_rn(a, b); }
};
template <> struct BwdArith<float> {
  static __device__ __forceinline__ float zero() { return 0.f; }
  static __device__ __forceinline__ float cvt(float w) { return w; }
  static __device__ __forceinline__ float mac(float acc, float s, float w) { return __fmaf_rn(s, w, acc); }
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
};

// floor(v) as an int that cannot wrap: coordinates beyond +-2^24 are moved to +-2^24, which is outside every
// window of any map this library handles; NaN goes to -2^24 (no tap)
__device__ __forceinline__ int floor_clamped(float v) {
  return (int)fminf(fmaxf(floorf(v), -16777216.f), 16777216.f);
}

// ---------------------------------------------------------------------------------------------------- corr_index
constexpr int CIB_THREADS = 256;
constexpr int CIB_MAXPIX = 32;

// grid: ceil(n*h1*w1 / pix)   block: CIB_THREADS
template <typename T, int R>
__global__ void __launch_bounds__(CIB_THREADS)
corr_index_backward_kernel(const float* __restrict__ coords, const T* __restrict__ corr_grad, T* __restrict__ vgrad,
                           int npix, int hw, int h2, int w2, int pix) {
  constexpr int RD = 2 * R + 1, NT = RD + 1, NTAP = NT * NT;
  constexpr int VE = 16 / sizeof(T);
  __shared__ T gtab[CIB_MAXPIX * NTAP];                     // [k][j][i]
  __shared__ int org[CIB_MAXPIX][2];                        // xb, yb
  const int P0 = blockIdx.x * pix;
  const int np = min(pix, npix - P0);

  for (int idx = threadIdx.x; idx < np * NTAP; idx += blockDim.x) {
    const int k = idx / NTAP, t = idx - k * NTAP;
    const int P = P0 + k, n = P / hw, p = P - n * hw;
    const float x0 = coords[((size_t)n * 2 + 0) * hw + p];
    const float y0 = coords[((size_t)n * 2 + 1) * hw + p];
    const float dx = x0 - floorf(x0), dy = y0 - floorf(y0);
    const T w11 = BwdArith<T>::cvt(dx * dy), w10 = BwdArith<T>::cvt(dx * (1.0f - dy));
    const T w01 = BwdArith<T>::cvt((1.0f - dx) * dy), w00 = BwdArith<T>::cvt((1.0f - dx) * (1.0f - dy));
    const int j = t / NT, i = t - j * NT;                     // i <-> x offset, j <-> y offset
    const T* cg = corr_grad + (size_t)n * RD * RD * hw + p;  // cg[(i*RD + j) * hw]
    T g = BwdArith<T>::zero();
    if (i > 0 && j > 0) g = BwdArith<T>::mac(g, cg[(size_t)((i - 1) * RD + j - 1) * hw], w11);
    if (i > 0 && j < RD) g = BwdArith<T>::mac(g, cg[(size_t)((i - 1) * RD + j) * hw], w10);
    if (i < RD && j > 0) g = BwdArith<T>::mac(g, cg[(size_t)(i * RD + j - 1) * hw], w01);
    if (i < RD && j < RD) g = BwdArith<T>::mac(g, cg[(size_t)(i * RD + j) * hw], w00);
    gtab[idx] = BwdArith<T>::add(BwdArith<T>::zero(), g);
    if (t == 0) {
      org[k][0] = floor_clamped(x0) - R;
      org[k][1] = floor_clamped(y0) - R;
    }
  }
  __syncthreads();

  const unsigned S = (unsigned)(h2 * w2);
  const size_t base = (size_t)P0 * S, end = base + (size_t)np * S;
  auto value = [&](unsigned k, int y, int x) -> T {
    const unsigned i = (unsigned)(x - org[k][0]), j = (unsigned)(y - org[k][1]);
    return (i <= (unsigned)RD && j <= (unsigned)RD) ? gtab[k * NTAP + j * NT + i] : BwdArith<T>::zero();
  };
  // unaligned head and tail element by element, the rest as 16-byte vectors
  const size_t v0 = (base + VE - 1) / VE, v1 = end / VE;
  if (v0 >= v1) {
    for (size_t e = base + threadIdx.x; e < end; e += blockDim.x) {
      const unsigned le = (unsigned)(e - base), k = le / S, rem = le - k * S;
      vgrad[e] = value(k, rem / w2, rem % w2);
    }
    return;
  }
  for (size_t e = base + threadIdx.x; e < v0 * VE; e += blockDim.x) {
    const unsigned le = (unsigned)(e - base), k = le / S, rem = le - k * S;
    vgrad[e] = value(k, rem / w2, rem % w2);
  }
  for (size_t e = v1 * VE + threadIdx.x; e < end; e += blockDim.x) {
    const unsigned le = (unsigned)(e - base), k = le / S, rem = le - k * S;
    vgrad[e] = value(k, rem / w2, rem % w2);
  }
  for (size_t v = v0 + threadIdx.x; v < v1; v += blockDim.x) {
    const unsigned le = (unsigned)(v * VE - base);
    unsigned k = le / S;
    const unsigned rem = le - k * S;
    int y = rem / w2, x = rem - y * w2;
    union { uint4 u; T e[VE]; } pk;
#pragma unroll
    for (int q = 0; q < VE; q++) {
      pk.e[q] = value(k, y, x);
      if (++x == w2) {
        x = 0;
        if (++y == h2) { y = 0; ++k; }
      }
    }
    *reinterpret_cast<uint4*>(vgrad + v * VE) = pk.u;
  }
}

template <typename T>
static int launch_corr_index_backward(const float* coords, const void* corr_grad, void* vgrad, int n, int h1, int w1,
                                      int h2, int w2, int radius, cudaStream_t st) {
  const long long npix = (long long)n * h1 * w1;
  if (npix == 0 || h2 <= 0 || w2 <= 0) return 0;
  if (npix > INT32_MAX || (long long)h2 * w2 * CIB_MAXPIX > INT32_MAX) return (int)cudaErrorInvalidValue;
  if (reinterpret_cast<uintptr_t>(vgrad) % 16 != 0) return (int)cudaErrorMisalignedAddress;
  const int S = h2 * w2, VE = 16 / sizeof(T);
  // about 4 vectors per thread per CTA, whole source pixels
  int pix = (CIB_THREADS * 4 * VE + S - 1) / S;
  pix = max(1, min(pix, CIB_MAXPIX));
  const dim3 grid((unsigned)((npix + pix - 1) / pix));
#define NSLAM_CIB(RR)                                                                                     \
  corr_index_backward_kernel<T, RR><<<grid, CIB_THREADS, 0, st>>>(coords, (const T*)corr_grad, (T*)vgrad, \
                                                                  (int)npix, h1 * w1, h2, w2, pix)
  switch (radius) {
    case 1: NSLAM_CIB(1); break;
    case 2: NSLAM_CIB(2); break;
    case 3: NSLAM_CIB(3); break;
    case 4: NSLAM_CIB(4); break;
    default: return (int)cudaErrorInvalidValue;
  }
#undef NSLAM_CIB
  NSLAM_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------- altcorr
constexpr int ACB_BLOCK = 512;   // sources per key block
constexpr int ACB_WARPS = 4;     // warps per CTA of the two gather kernels

struct AcbShape {
  int B, N, H1, W1, H2, W2, C;
  int hw, S, nblk, K, KW;         // S = N*hw sources per batch, K = buckets per batch, KW = bucket row width
  long long tab;                  // K*nblk + 1
};

static AcbShape acb_shape(int B, int N, int H1, int W1, int H2, int W2, int C, int radius) {
  AcbShape s;
  const int RD = 2 * radius + 1;
  s.B = B; s.N = N; s.H1 = H1; s.W1 = W1; s.H2 = H2; s.W2 = W2; s.C = C;
  s.hw = H1 * W1;
  s.S = N * s.hw;
  s.nblk = (s.S + ACB_BLOCK - 1) / ACB_BLOCK;
  s.KW = W2 + RD;
  s.K = (H2 + RD) * s.KW;
  s.tab = (long long)s.K * s.nblk + 1;
  return s;
}

// weight of tap (iy, ix) for a source whose window-relative fractions are dx, dy (src/altcorr_kernel.cu:237-252)
template <int R>
__device__ __forceinline__ float tap_weight(const float* __restrict__ cg, int hw, int iy, int ix, float dx, float dy) {
  constexpr int RD = 2 * R + 1;
  float g = 0.f;
  if (iy > 0 && ix > 0) g += cg[(size_t)((iy - 1) + RD * (ix - 1)) * hw] * dy * dx;
  if (iy > 0 && ix < RD) g += cg[(size_t)((iy - 1) + RD * ix) * hw] * dy * (1.f - dx);
  if (iy < RD && ix > 0) g += cg[(size_t)(iy + RD * (ix - 1)) * hw] * (1.f - dy) * dx;
  if (iy < RD && ix < RD) g += cg[(size_t)(iy + RD * ix) * hw] * (1.f - dy) * (1.f - dx);
  return g;
}

// 1. key + rank.  grid: (nblk, B)   block: ACB_BLOCK
template <int R>
__global__ void __launch_bounds__(ACB_BLOCK)
altcorr_bwd_key_kernel(const float* __restrict__ coords, AcbShape s, int* __restrict__ key, int* __restrict__ rank,
                       int* __restrict__ tab) {
  constexpr int RD = 2 * R + 1;
  __shared__ int sk[ACB_BLOCK];
  const int b = blockIdx.y, blk = blockIdx.x;
  const int src = blk * ACB_BLOCK + threadIdx.x;
  int k = -1;
  if (src < s.S) {
    const float* c = coords + ((size_t)b * s.S + src) * 2;
    const int xb = floor_clamped(c[0]) - R, yb = floor_clamped(c[1]) - R;
    if (yb >= -RD && yb < s.H2 && xb >= -RD && xb < s.W2) k = (yb + RD) * s.KW + (xb + RD);
  }
  sk[threadIdx.x] = k;
  __syncthreads();
  if (src >= s.S) return;
  int before = 0, total = 0;
  if (k >= 0) {
    for (int t = 0; t < ACB_BLOCK; t++) {
      const int m = sk[t] == k;
      total += m;
      before += m & (t < (int)threadIdx.x);
    }
  }
  key[(size_t)b * s.S + src] = k;
  rank[(size_t)b * s.S + src] = before;
  if (k >= 0 && before == 0) tab[(size_t)b * s.tab + (size_t)k * s.nblk + blk] = total;
}

// 2. exclusive scan of each batch's table, in place; the last entry gets the total.  grid: B   block: 1024
constexpr int SCAN_THREADS = 1024, SCAN_IPT = 8;
__global__ void __launch_bounds__(SCAN_THREADS) altcorr_bwd_scan_kernel(int* __restrict__ tab, long long len) {
  __shared__ int wsum[SCAN_THREADS / 32];
  __shared__ int carry_s;
  int* t = tab + (size_t)blockIdx.x * len;
  const long long n = len - 1;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (long long t0 = 0; t0 < n; t0 += (long long)SCAN_THREADS * SCAN_IPT) {
    const long long i0 = t0 + (long long)threadIdx.x * SCAN_IPT;
    int v[SCAN_IPT], sum = 0;
#pragma unroll
    for (int q = 0; q < SCAN_IPT; q++) {
      v[q] = (i0 + q < n) ? t[i0 + q] : 0;
      sum += v[q];
    }
    int inc = sum;                                        // inclusive scan over the block
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += u;
    }
    if (lane == 31) wsum[wid] = inc;
    __syncthreads();
    if (wid == 0) {
      int w = wsum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += u;
      }
      wsum[lane] = w;
    }
    __syncthreads();
    const int carry = carry_s;
    int run = carry + (wid > 0 ? wsum[wid - 1] : 0) + inc - sum;
#pragma unroll
    for (int q = 0; q < SCAN_IPT; q++) {
      if (i0 + q < n) t[i0 + q] = run;
      run += v[q];
    }
    __syncthreads();
    if (threadIdx.x == 0) carry_s = carry + wsum[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) t[n] = carry_s;
}

// 3. fill.  grid: (nblk, B)   block: ACB_BLOCK
__global__ void __launch_bounds__(ACB_BLOCK)
altcorr_bwd_fill_kernel(AcbShape s, const int* __restrict__ key, const int* __restrict__ rank,
                        const int* __restrict__ tab, int* __restrict__ rec) {
  const int b = blockIdx.y, blk = blockIdx.x;
  const int src = blk * ACB_BLOCK + threadIdx.x;
  if (src >= s.S) return;
  const int k = key[(size_t)b * s.S + src];
  if (k < 0) return;
  const int off = tab[(size_t)b * s.tab + (size_t)k * s.nblk + blk] + rank[(size_t)b * s.S + src];
  rec[(size_t)b * s.S + off] = src;
}

// channel chunk of 4 floats per lane; C % 4 == 0 and C <= 32 * 4 * CMAX
constexpr int ACB_CMAX = 4;

// 4. fmap2_grad: one warp per target pixel.  grid: (ceil(H2*W2 / ACB_WARPS), B)   block: 32*ACB_WARPS
template <int R>
__global__ void __launch_bounds__(32 * ACB_WARPS)
altcorr_bwd_fmap2_kernel(const float* __restrict__ fmap1, const float* __restrict__ coords,
                         const float* __restrict__ corr_grad, AcbShape s, const int* __restrict__ tab,
                         const int* __restrict__ rec, float* __restrict__ fmap2_grad) {
  constexpr int RD = 2 * R + 1, NT = RD + 1;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = blockIdx.x * ACB_WARPS + warp, b = blockIdx.y;
  if (q >= s.H2 * s.W2) return;  // warp-uniform
  const int h2 = q / s.W2, w2 = q - h2 * s.W2;
  const int* tb = tab + (size_t)b * s.tab;
  const int* rb = rec + (size_t)b * s.S;
  const float* f1b = fmap1 + (size_t)b * s.hw * s.C;
  float4 acc[ACB_CMAX];
#pragma unroll
  for (int u = 0; u < ACB_CMAX; u++) acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = 0; r < NT; r++) {
    const int yb = h2 - RD + r;                            // origin rows h2-RD .. h2, ascending
    const int k0 = (yb + RD) * s.KW + (w2 - RD + RD);      // origin columns w2-RD .. w2: buckets k0 .. k0+RD
    const int lo = tb[(size_t)k0 * s.nblk], hi = tb[(size_t)(k0 + NT) * s.nblk];
    for (int c0 = lo; c0 < hi; c0 += 32) {
      const int m = min(32, hi - c0);
      float g = 0.f;
      int p = 0;
      if (lane < m) {
        const int src = rb[c0 + lane];
        const int n = src / s.hw;
        p = src - n * s.hw;
        const float* c = coords + ((size_t)b * s.S + src) * 2;
        const float x0 = c[0], y0 = c[1];
        const float dx = x0 - floorf(x0), dy = y0 - floorf(y0);
        const int iy = h2 - (floor_clamped(y0) - R), ix = w2 - (floor_clamped(x0) - R);
        g = tap_weight<R>(corr_grad + (((size_t)b * s.N + n) * RD * RD) * s.hw + p, s.hw, iy, ix, dx, dy);
      }
      for (int j = 0; j < m; j++) {
        const float gj = __shfl_sync(0xffffffffu, g, j);
        const int pj = __shfl_sync(0xffffffffu, p, j);
        const float* f1 = f1b + (size_t)pj * s.C;
#pragma unroll
        for (int u = 0; u < ACB_CMAX; u++) {
          const int c = (u * 32 + lane) * 4;
          if (c < s.C) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(f1 + c));
            acc[u].x = fmaf(gj, v.x, acc[u].x); acc[u].y = fmaf(gj, v.y, acc[u].y);
            acc[u].z = fmaf(gj, v.z, acc[u].z); acc[u].w = fmaf(gj, v.w, acc[u].w);
          }
        }
      }
    }
  }
  float* o = fmap2_grad + ((size_t)b * s.H2 * s.W2 + q) * s.C;
#pragma unroll
  for (int u = 0; u < ACB_CMAX; u++) {
    const int c = (u * 32 + lane) * 4;
    if (c < s.C) *reinterpret_cast<float4*>(o + c) = acc[u];
  }
}

// 5. fmap1_grad: one warp per source pixel, taps in the order (n, iy, ix).
//    grid: (ceil(H1*W1 / ACB_WARPS), B)   block: 32*ACB_WARPS
template <int R>
__global__ void __launch_bounds__(32 * ACB_WARPS)
altcorr_bwd_fmap1_kernel(const float* __restrict__ fmap2, const float* __restrict__ coords,
                         const float* __restrict__ corr_grad, AcbShape s, float* __restrict__ fmap1_grad) {
  constexpr int RD = 2 * R + 1, NT = RD + 1, NTAP = NT * NT;
  constexpr int TPL = (NTAP + 31) / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p = blockIdx.x * ACB_WARPS + warp, b = blockIdx.y;
  if (p >= s.hw) return;  // warp-uniform
  const float* f2b = fmap2 + (size_t)b * s.H2 * s.W2 * s.C;
  float4 acc[ACB_CMAX];
#pragma unroll
  for (int u = 0; u < ACB_CMAX; u++) acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int n = 0; n < s.N; n++) {
    const float* c = coords + (((size_t)b * s.N + n) * s.hw + p) * 2;
    const float x0 = c[0], y0 = c[1];
    const float dx = x0 - floorf(x0), dy = y0 - floorf(y0);
    const int xb = floor_clamped(x0) - R, yb = floor_clamped(y0) - R;
    const float* cg = corr_grad + (((size_t)b * s.N + n) * RD * RD) * s.hw + p;
    float g[TPL];
#pragma unroll
    for (int u = 0; u < TPL; u++) {
      const int t = lane + 32 * u;
      g[u] = t < NTAP ? tap_weight<R>(cg, s.hw, t / NT, t % NT, dx, dy) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < TPL; u++) {
      for (int tl = 0; tl < 32; tl++) {
        const int t = 32 * u + tl;
        if (t >= NTAP) break;
        const int h2 = yb + t / NT, w2 = xb + t % NT;
        const float gt = __shfl_sync(0xffffffffu, g[u], tl);
        if (h2 < 0 || h2 >= s.H2 || w2 < 0 || w2 >= s.W2) continue;  // warp-uniform
        const float* f2 = f2b + ((size_t)h2 * s.W2 + w2) * s.C;
#pragma unroll
        for (int v = 0; v < ACB_CMAX; v++) {
          const int ch = (v * 32 + lane) * 4;
          if (ch < s.C) {
            const float4 f = __ldg(reinterpret_cast<const float4*>(f2 + ch));
            acc[v].x = fmaf(gt, f.x, acc[v].x); acc[v].y = fmaf(gt, f.y, acc[v].y);
            acc[v].z = fmaf(gt, f.z, acc[v].z); acc[v].w = fmaf(gt, f.w, acc[v].w);
          }
        }
      }
    }
  }
  float* o = fmap1_grad + ((size_t)b * s.hw + p) * s.C;
#pragma unroll
  for (int v = 0; v < ACB_CMAX; v++) {
    const int ch = (v * 32 + lane) * 4;
    if (ch < s.C) *reinterpret_cast<float4*>(o + ch) = acc[v];
  }
}

static bool acb_supported(int B, int N, int H1, int W1, int H2, int W2, int C, int radius) {
  if (radius < 1 || radius > 4 || C <= 0 || C % 4 != 0 || C > 128 * ACB_CMAX) return false;
  if (B < 0 || N < 0 || H1 < 0 || W1 < 0 || H2 <= 0 || W2 <= 0) return false;
  const long long S = (long long)N * H1 * W1, RD = 2 * radius + 1;
  const long long K = (long long)(H2 + RD) * (W2 + RD);
  return S < INT32_MAX && K * ((S + ACB_BLOCK - 1) / ACB_BLOCK) + 1 < INT32_MAX;
}

static size_t acb_scratch_bytes(const AcbShape& s) {
  return ((size_t)s.B * s.S * 3 + (size_t)s.B * s.tab) * sizeof(int);
}

template <int R>
static int launch_altcorr_backward(const float* fmap1, const float* fmap2, const float* coords, const float* corr_grad,
                                   float* fmap1_grad, float* fmap2_grad, void* scratch, const AcbShape& s,
                                   cudaStream_t st) {
  int* key = (int*)scratch;
  int* rank = key + (size_t)s.B * s.S;
  int* rec = rank + (size_t)s.B * s.S;
  int* tab = rec + (size_t)s.B * s.S;
  const dim3 g2((s.H2 * s.W2 + ACB_WARPS - 1) / ACB_WARPS, s.B);
  if (s.S > 0) {
    cudaError_t e = cudaMemsetAsync(tab, 0, (size_t)s.B * s.tab * sizeof(int), st);
    if (e != cudaSuccess) return (int)e;
    const dim3 gk(s.nblk, s.B);
    altcorr_bwd_key_kernel<R><<<gk, ACB_BLOCK, 0, st>>>(coords, s, key, rank, tab);
    altcorr_bwd_scan_kernel<<<s.B, SCAN_THREADS, 0, st>>>(tab, s.tab);
    altcorr_bwd_fill_kernel<<<gk, ACB_BLOCK, 0, st>>>(s, key, rank, tab, rec);
    NSLAM_CHECK_LAUNCH();
    const dim3 g1((s.hw + ACB_WARPS - 1) / ACB_WARPS, s.B);
    altcorr_bwd_fmap1_kernel<R><<<g1, 32 * ACB_WARPS, 0, st>>>(fmap2, coords, corr_grad, s, fmap1_grad);
    altcorr_bwd_fmap2_kernel<R><<<g2, 32 * ACB_WARPS, 0, st>>>(fmap1, coords, corr_grad, s, tab, rec, fmap2_grad);
  } else {
    // no source pixel: every target gradient is zero (and fmap1_grad is empty)
    cudaError_t e = cudaMemsetAsync(fmap2_grad, 0, (size_t)s.B * s.H2 * s.W2 * s.C * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
  }
  NSLAM_CHECK_LAUNCH();
  return 0;
}

}  // namespace nslam

extern "C" {

// dtype: 0 = fp16, 1 = fp32 (coords fp32; corr_grad and volume_grad in the volume dtype)
int nslam_corr_index_backward(const float* coords, const void* corr_grad, int dtype, void* volume_grad, int n, int h1,
                              int w1, int h2, int w2, int radius, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == 0)
    return nslam::launch_corr_index_backward<__half>(coords, corr_grad, volume_grad, n, h1, w1, h2, w2, radius, st);
  if (dtype == 1)
    return nslam::launch_corr_index_backward<float>(coords, corr_grad, volume_grad, n, h1, w1, h2, w2, radius, st);
  return (int)cudaErrorInvalidValue;
}

int nslam_altcorr_backward_scratch(int B, int N, int H1, int W1, int H2, int W2, int C, int radius,
                                   unsigned long long* bytes) {
  if (!nslam::acb_supported(B, N, H1, W1, H2, W2, C, radius)) return (int)cudaErrorInvalidValue;
  *bytes = nslam::acb_scratch_bytes(nslam::acb_shape(B, N, H1, W1, H2, W2, C, radius));
  return 0;
}

int nslam_altcorr_backward(const float* fmap1, const float* fmap2, const float* coords, const float* corr_grad,
                           float* fmap1_grad, float* fmap2_grad, void* scratch, unsigned long long scratch_bytes, int B,
                           int N, int H1, int W1, int H2, int W2, int C, int radius, void* stream) {
  if (!nslam::acb_supported(B, N, H1, W1, H2, W2, C, radius)) return (int)cudaErrorInvalidValue;
  const nslam::AcbShape s = nslam::acb_shape(B, N, H1, W1, H2, W2, C, radius);
  if (B == 0) return 0;
  if (scratch_bytes < nslam::acb_scratch_bytes(s)) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  switch (radius) {
    case 1: return nslam::launch_altcorr_backward<1>(fmap1, fmap2, coords, corr_grad, fmap1_grad, fmap2_grad, scratch, s, st);
    case 2: return nslam::launch_altcorr_backward<2>(fmap1, fmap2, coords, corr_grad, fmap1_grad, fmap2_grad, scratch, s, st);
    case 3: return nslam::launch_altcorr_backward<3>(fmap1, fmap2, coords, corr_grad, fmap1_grad, fmap2_grad, scratch, s, st);
    case 4: return nslam::launch_altcorr_backward<4>(fmap1, fmap2, coords, corr_grad, fmap1_grad, fmap2_grad, scratch, s, st);
  }
  return (int)cudaErrorInvalidValue;
}

}  // extern "C"
