// Path B — tiny-MLP forward on Hopper tensor cores (wgmma), fused with the hash-grid encoding (sm_90a).
//
// Same function as ngp::forward_kernel (csrc/ngp_train.cu): coords -> (rgb, sigma), but the five
// dense layers run as wgmma on a 128-sample tile:
//   thread = sample (128 threads / CTA = one warpgroup, persistent CTAs):
//     hash encode (128 independent fp16 gathers) -> row of the A tile in shared memory (fp16,
//     K-major, 128B-swizzled) -> the warpgroup issues 2 x (M64 x N{64,16} x K16) wgmmas against the
//     layer's pre-packed weight image -> fp32 accumulator fragments -> shared fp32 tile -> the thread's
//     own row -> ReLU / exp / SH / sigmoid in registers -> next layer's A row ... activations never leave the SM.
// Weights: fp16 copies of the fp32 master, packed by ngp_pack_mlp_kernel after every Adam step into
// wgmma-ready images B_l[n][k] = W_l[k][n] (K padded to 64).
// FLOPs per sample: 2 * 10 240; roofline: tensor pipe (north_star target for the tiny MLP), in
// practice bounded by the gather + epilogue.
#include "ngp_common.cuh"
#include "tc.cuh"
#include "../../include/nslam_ngp.h"

namespace ngp {

// packed weight images (bytes): W1 [64][128B], W2 [16][128B], W3 [64][128B], W4 [64][128B], W5 [16][128B]
constexpr int PW1 = 0, PW2 = 8192, PW3 = 10240, PW4 = 18432, PW5 = 26624, PW_TOTAL = 28672;

__global__ void pack_mlp_kernel(const float* __restrict__ mlp, unsigned char* __restrict__ packed) {
  // one thread per (layer, n, k) element of the padded [N][64] images
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  const int offs[5] = {PW1, PW2, PW3, PW4, PW5};
  const int Ns[5] = {64, 16, 64, 64, 16};
  const int Ks[5] = {32, 64, 32, 64, 64};
  const int woff[5] = {W1_OFF, W2_OFF, W3_OFF, W4_OFF, W5_OFF};
  int base = 0;
  for (int l = 0; l < 5; l++) {
    const int cnt = Ns[l] * 64;
    if (id < base + cnt) {
      const int e = id - base, n = e / 64, k = e % 64;
      const float v = (k < Ks[l]) ? mlp[woff[l] + k * Ns[l] + n] : 0.f;
      // row n, 16-byte chunk (k/8) stored at chunk position (k/8) ^ (n & 7)
      __half* dst = reinterpret_cast<__half*>(packed + offs[l] + n * 128 + (((k >> 3) ^ (n & 7)) << 4)) + (k & 7);
      *dst = __float2half_rn(v);
      return;
    }
    base += cnt;
  }
}

// fp32 accumulator tile [128][SCR_LD] (<= 64 columns + 8 of padding: conflict-free fragment stores)
constexpr int SCR_LD = 72;
constexpr int SCR_BYTES = 128 * SCR_LD * 4;

struct FwdSmem {
  static constexpr int W = 0;                 // PW_TOTAL (1024-aligned images)
  static constexpr int A = 28672;             // [128][128 B]
  static constexpr int SCR = A + 16384;       // accumulator tile
  static constexpr int BAR = SCR + SCR_BYTES;
  static constexpr int TOTAL = BAR + 64;
};

__device__ __forceinline__ void store_row_chunk(unsigned char* arow, int row, int chunk, const float* v8) {
  __half2 h2[4];
#pragma unroll
  for (int j = 0; j < 4; j++) h2[j] = __floats2half2_rn(v8[2 * j], v8[2 * j + 1]);
  *reinterpret_cast<uint4*>(arow + ((chunk ^ (row & 7)) << 4)) = *reinterpret_cast<const uint4*>(h2);
}

// one layer, issued by the whole CTA (one warpgroup): A tile (already written + fenced + synced, 128 rows) x packed
// weights -> fp32 tile scr[128][SCR_LD] columns [0, N), visible to every thread on return
template <int N>
__device__ __forceinline__ void mma_layer(uint32_t a_addr, uint32_t b_addr, int ksteps, float* scr, int tid) {
  float d[2][N / 2];
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int i = 0; i < N / 2; i++) d[h][i] = 0.f;
  const uint64_t bd = tc::desc_sw128(b_addr);
  tc::wgmma_fence();
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const uint64_t ad = tc::desc_sw128(a_addr + h * 8192);      // rows 64h .. 64h+63
    for (int k = 0; k < ksteps; k++) tc::wgmma_f16<N>(d[h], ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), k ? 1u : 0u);
  }
  tc::wgmma_commit();
  tc::wgmma_wait<0>();
#pragma unroll
  for (int h = 0; h < 2; h++) {
    tc::acc_fence(d[h]);
    tc::acc_to_smem<N>(scr, SCR_LD, 64 * h, 0, d[h], tid);
  }
  __syncthreads();
}

__global__ void __launch_bounds__(128)
forward_tc_kernel(const float* __restrict__ coords, const int* __restrict__ counters, int n_fixed,
                  const __half2* __restrict__ grid, LevelInfo lv, const unsigned char* __restrict__ packed,
                  float* __restrict__ rgbsigma, __half* __restrict__ enc_out) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sm = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* scr = reinterpret_cast<float*>(sm + FwdSmem::SCR);
  const int tid = threadIdx.x;
  const int n = n_fixed >= 0 ? n_fixed : counters[0];
  const int ntiles = (n + 127) / 128;

  for (int i = tid; i < PW_TOTAL / 16; i += 128)
    reinterpret_cast<uint4*>(sm + FwdSmem::W)[i] = reinterpret_cast<const uint4*>(packed)[i];
  tc::fence_proxy_async();
  __syncthreads();
  const uint32_t a_addr = tc::smem_u32(sm + FwdSmem::A);
  const uint32_t w_addr = tc::smem_u32(sm + FwdSmem::W);
  unsigned char* arow = sm + FwdSmem::A + tid * 128;

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int s = tile * 128 + tid;
    const bool act = s < n;
    float c7[7] = {0.5f, 0.5f, 0.5f, 0.f, 0.f, 0.f, 1.f};
    if (act) {
#pragma unroll
      for (int k = 0; k < 7; k++) c7[k] = coords[(size_t)s * 7 + k];
    }
    // ---- encode -> A row (cols 0..31), zero cols 32..63
    {
      float enc[ENC_DIM];
      hash_encode(c7, grid, lv, enc);
      const float z8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
      for (int c = 0; c < 4; c++) store_row_chunk(arow, tid, c, enc + 8 * c);
#pragma unroll
      for (int c = 4; c < 8; c++) store_row_chunk(arow, tid, c, z8);
      if (enc_out && act) {
        // keep the fp16 encoding for the backward pass (saves its 128 gathers per sample)
#pragma unroll
        for (int c = 0; c < 4; c++)
          reinterpret_cast<uint4*>(enc_out + (size_t)s * ENC_DIM)[c] = *reinterpret_cast<const uint4*>(arow + ((c ^ (tid & 7)) << 4));
      }
    }
    tc::fence_proxy_async();
    __syncthreads();
    // ---- layer 1: 32 -> 64, ReLU
    mma_layer<64>(a_addr, w_addr + PW1, 2, scr, tid);
    {
      uint32_t r[32];
      float v[8];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        tc::smem_row_ld<32>(scr, SCR_LD, tid, h * 32, r);
#pragma unroll
        for (int c = 0; c < 4; c++) {
#pragma unroll
          for (int j = 0; j < 8; j++) v[j] = fmaxf(__uint_as_float(r[c * 8 + j]), 0.f);
          store_row_chunk(arow, tid, h * 4 + c, v);
        }
      }
    }
    tc::fence_proxy_async();
    __syncthreads();
    // ---- layer 2: 64 -> 16 (density head)
    mma_layer<16>(a_addr, w_addr + PW2, 4, scr, tid);
    float sigma;
    {
      uint32_t r[32];
      tc::smem_row_ld<32>(scr, SCR_LD, tid, 0, r);     // 16 valid columns
      float o[16], sh[16];
#pragma unroll
      for (int j = 0; j < 16; j++) o[j] = __uint_as_float(r[j]);
      sigma = __expf(o[0]);
      sh4(c7 + 4, sh);
      const float z8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      store_row_chunk(arow, tid, 0, o); store_row_chunk(arow, tid, 1, o + 8);
      store_row_chunk(arow, tid, 2, sh); store_row_chunk(arow, tid, 3, sh + 8);
#pragma unroll
      for (int c = 4; c < 8; c++) store_row_chunk(arow, tid, c, z8);
    }
    tc::fence_proxy_async();
    __syncthreads();
    // ---- layers 3, 4: -> 64, ReLU
#pragma unroll 1
    for (int l = 0; l < 2; l++) {
      mma_layer<64>(a_addr, w_addr + (l == 0 ? PW3 : PW4), l == 0 ? 2 : 4, scr, tid);
      uint32_t r[32];
      float v[8];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        tc::smem_row_ld<32>(scr, SCR_LD, tid, h * 32, r);
#pragma unroll
        for (int c = 0; c < 4; c++) {
#pragma unroll
          for (int j = 0; j < 8; j++) v[j] = fmaxf(__uint_as_float(r[c * 8 + j]), 0.f);
          store_row_chunk(arow, tid, h * 4 + c, v);
        }
      }
      tc::fence_proxy_async();
      __syncthreads();
    }
    // ---- layer 5: 64 -> 3 (16), sigmoid
    mma_layer<16>(a_addr, w_addr + PW5, 4, scr, tid);
    {
      uint32_t r[32];
      tc::smem_row_ld<32>(scr, SCR_LD, tid, 0, r);
      if (act) {
        float4 out;
        out.x = 1.f / (1.f + __expf(-__uint_as_float(r[0])));
        out.y = 1.f / (1.f + __expf(-__uint_as_float(r[1])));
        out.z = 1.f / (1.f + __expf(-__uint_as_float(r[2])));
        out.w = sigma;
        reinterpret_cast<float4*>(rgbsigma)[s] = out;
      }
    }
    __syncthreads();      // accumulator tile + A tile reusable by the next tile
  }
}


// ============================================================================================
// Backward on tensor cores.  Per 128-sample tile (thread = sample):
//   forward recompute (layers 1-4) keeping every layer's INPUT tile in shared memory,
//   then for l = 5..1 two MMA groups per layer, issued together:
//     dW_l   += A_l^T (features x samples) . delta_l (samples x N_l)     [M = 64 features; fp32 fragments
//                                                                         accumulate in registers across tiles]
//     dIn_l   = delta_l (samples x N_l)    . W_l^T                       [-> ACC, masked by ReLU']
//   Operands are fp16 (deltas carry a loss scale), accumulation fp32.  The transposed operand
//   tiles (K = the 128 samples) are written by the owning threads with 2-byte swizzled stores.
//   At the end of the persistent loop each CTA flushes its dW accumulators with fp32 atomics.
// backward weight images B[k][n] = W[k][n], n padded to 64: WB5 [64][128B], WB4 [64][128B], WB3 [32][128B], WB2 [64][128B], WB1 [32][128B]
constexpr int PB5 = 0, PB4 = 8192, PB3 = 16384, PB2 = 20480, PB1 = 28672, PB_TOTAL = 32768;

__global__ void pack_mlp_bwd_kernel(const float* __restrict__ mlp, unsigned char* __restrict__ packed) {
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  const int offs[5] = {PB5, PB4, PB3, PB2, PB1};
  const int Ks[5] = {64, 64, 32, 64, 32};      // rows
  const int Ns[5] = {16, 64, 64, 16, 64};      // real columns
  const int woff[5] = {W5_OFF, W4_OFF, W3_OFF, W2_OFF, W1_OFF};
  int base = 0;
  for (int l = 0; l < 5; l++) {
    const int cnt = Ks[l] * 64;
    if (id < base + cnt) {
      const int e = id - base, k = e / 64, n = e % 64;
      const float v = (n < Ns[l]) ? mlp[woff[l] + k * Ns[l] + n] : 0.f;
      __half* dst = reinterpret_cast<__half*>(packed + offs[l] + k * 128 + (((n >> 3) ^ (k & 7)) << 4)) + (n & 7);
      *dst = __float2half_rn(v);
      return;
    }
    base += cnt;
  }
}

struct BwdSmem {
  static constexpr int W = 0;                      // forward images   28672
  static constexpr int WB = 28672;                 // backward images  32768
  static constexpr int ACT = WB + PB_TOTAL;        // 5 x 16384 : inputs of layers 1..5 (row-major, swizzled)
  static constexpr int AT = ACT + 5 * 16384;       // transposed activations: 2 sample halves x [64 features][128B]
  static constexpr int D = AT + 16384;             // delta, row-major [128][128B]
  static constexpr int DT = D + 16384;             // delta transposed: 2 halves x [64][128B]
  static constexpr int SCR = DT + 16384;           // fp32 accumulator tile [128][SCR_LD]
  static constexpr int BAR = SCR + SCR_BYTES;
  static constexpr int TOTAL = BAR + 64;
  static_assert(TOTAL + 1024 <= 227 * 1024, "shared memory plan");
};

// element (row f, sample s) of a K-major [rows][128 samples] operand split in two 64-sample halves
__device__ __forceinline__ void store_T(unsigned char* base, int half_bytes, int f, int s, float v) {
  __half* p = reinterpret_cast<__half*>(base + (s >> 6) * half_bytes + f * 128 + ((((s & 63) >> 3) ^ (f & 7)) << 4)) + (s & 7);
  *p = __float2half_rn(v);
}
// transpose this thread's row of a row-major swizzled tile (first nf features) into AT
__device__ __forceinline__ void transpose_row(const unsigned char* tile, unsigned char* at, int row, int nf) {
  const unsigned char* arow = tile + row * 128;
  for (int c = 0; c < nf / 8; c++) {
    const uint4 raw = *reinterpret_cast<const uint4*>(arow + ((c ^ (row & 7)) << 4));
    const __half* h = reinterpret_cast<const __half*>(&raw);
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const int f = c * 8 + j;
      __half* p = reinterpret_cast<__half*>(at + (row >> 6) * 8192 + f * 128 + ((((row & 63) >> 3) ^ (f & 7)) << 4)) + (row & 7);
      *p = h[j];
    }
  }
}
// write a delta vector (n values, fp32) as this thread's row of D (zero-padded to 64) and column of DT
template <int NV>
__device__ __forceinline__ void store_delta(unsigned char* dtile, unsigned char* dt, int row, const float* d) {
  unsigned char* drow = dtile + row * 128;
  const float z8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
  for (int c = 0; c < 8; c++) store_row_chunk(drow, row, c, (c * 8 < NV) ? d + c * 8 : z8);
#pragma unroll
  for (int n = 0; n < NV; n++) store_T(dt, 8192, n, row, d[n]);
}

// dW (fragments `dw`, M = 64 features x N) += AT-operand x DT-operand over the 128 samples; then
// scr = D x WB (N_out columns, `ks` K-steps).  Issued by the whole CTA (one warpgroup), one commit covers both.
template <int N, int NOUT>
__device__ __forceinline__ void mma_bwd_layer(uint32_t at_addr, uint32_t dt_addr, uint32_t d_addr, uint32_t wb_addr,
                                              float (&dw)[N / 2], int ks, float* scr, int tid) {
  float acc[2][NOUT / 2];
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int i = 0; i < NOUT / 2; i++) acc[h][i] = 0.f;
  tc::wgmma_fence();
  tc::acc_fence(dw);
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int k = 0; k < 4; k++)
      tc::wgmma_f16<N>(dw, tc::desc_sw128(at_addr + h * 8192 + k * 32), tc::desc_sw128(dt_addr + h * 8192 + k * 32), 1u);
  const uint64_t bd = tc::desc_sw128(wb_addr);
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const uint64_t ad = tc::desc_sw128(d_addr + h * 8192);
    for (int k = 0; k < ks; k++) tc::wgmma_f16<NOUT>(acc[h], ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), k ? 1u : 0u);
  }
  tc::wgmma_commit();
  tc::wgmma_wait<0>();
  tc::acc_fence(dw);
#pragma unroll
  for (int h = 0; h < 2; h++) {
    tc::acc_fence(acc[h]);
    tc::acc_to_smem<NOUT>(scr, SCR_LD, 64 * h, 0, acc[h], tid);
  }
  __syncthreads();
}

// weight-gradient flush: fragment element (feature k, column n) of dW [kmax][N] -> this CTA's slot of the partials
template <int N>
__device__ __forceinline__ void flush_dw(const float (&d)[N / 2], float* __restrict__ g, int kmax, float scale, int tid) {
  const int w = tid >> 5, l = tid & 31;
#pragma unroll
  for (int j = 0; j < N / 8; j++)
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const int k = 16 * w + (l >> 2) + 8 * i, n = 8 * j + 2 * (l & 3);
      if (k < kmax) *reinterpret_cast<float2*>(g + k * N + n) = make_float2(d[4 * j + 2 * i] * scale, d[4 * j + 2 * i + 1] * scale);
    }
}

__device__ __forceinline__ void ld_relu_store(const float* scr, unsigned char* arow, int row, uint32_t* mask) {
  uint32_t r[32];
  float v[8];
#pragma unroll
  for (int h = 0; h < 2; h++) {
    tc::smem_row_ld<32>(scr, SCR_LD, row, h * 32, r);
    uint32_t m = 0;
#pragma unroll
    for (int c = 0; c < 4; c++) {
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const float x = __uint_as_float(r[c * 8 + j]);
        m |= (x > 0.f ? 1u : 0u) << (c * 8 + j);
        v[j] = fmaxf(x, 0.f);
      }
      store_row_chunk(arow, row, h * 4 + c, v);
    }
    mask[h] = m;
  }
}

#define NGP_TC_SYNC()            \
  do {                           \
    tc::fence_proxy_async();     \
    __syncthreads();             \
  } while (0)

__global__ void __launch_bounds__(128, 1)
backward_tc_kernel(const float* __restrict__ coords, const int* __restrict__ counters,
                   const __half2* __restrict__ grid, LevelInfo lv, const unsigned char* __restrict__ packed_fwd,
                   const unsigned char* __restrict__ packed_bwd, const float* __restrict__ dout,
                   float* __restrict__ dw_part, float* __restrict__ grid_grad, float loss_scale,
                   const __half* __restrict__ enc_in, __half* __restrict__ denc_out) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sm = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* scr = reinterpret_cast<float*>(sm + BwdSmem::SCR);
  const int tid = threadIdx.x;
  const int n = counters[0];
  const int ntiles = (n + 127) / 128;
  for (int i = tid; i < PW_TOTAL / 16; i += 128) reinterpret_cast<uint4*>(sm + BwdSmem::W)[i] = reinterpret_cast<const uint4*>(packed_fwd)[i];
  for (int i = tid; i < PB_TOTAL / 16; i += 128) reinterpret_cast<uint4*>(sm + BwdSmem::WB)[i] = reinterpret_cast<const uint4*>(packed_bwd)[i];
  for (int i = tid; i < (16384 + 16384 + 16384) / 16; i += 128) reinterpret_cast<uint4*>(sm + BwdSmem::AT)[i] = make_uint4(0, 0, 0, 0);
  NGP_TC_SYNC();
  const uint32_t w_addr = tc::smem_u32(sm + BwdSmem::W), wb_addr = tc::smem_u32(sm + BwdSmem::WB);
  const uint32_t act_addr = tc::smem_u32(sm + BwdSmem::ACT);
  const uint32_t at_addr = tc::smem_u32(sm + BwdSmem::AT), d_addr = tc::smem_u32(sm + BwdSmem::D), dt_addr = tc::smem_u32(sm + BwdSmem::DT);
  unsigned char* act = sm + BwdSmem::ACT;
  unsigned char* AT = sm + BwdSmem::AT;
  unsigned char* Dt = sm + BwdSmem::D;
  unsigned char* DT = sm + BwdSmem::DT;
  bool first = true;
  const float inv_scale = 1.f / loss_scale;
  // weight-gradient accumulators (rows = input features 0..63)
  float dw1[32], dw2[8], dw3[32], dw4[32], dw5[8];
#pragma unroll
  for (int i = 0; i < 32; i++) { dw1[i] = 0.f; dw3[i] = 0.f; dw4[i] = 0.f; }
#pragma unroll
  for (int i = 0; i < 8; i++) { dw2[i] = 0.f; dw5[i] = 0.f; }

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int s = tile * 128 + tid;
    const bool actv = s < n;
    float c7[7] = {0.5f, 0.5f, 0.5f, 0.f, 0.f, 0.f, 1.f};
    float4 dg = make_float4(0.f, 0.f, 0.f, 0.f);
    if (actv) {
#pragma unroll
      for (int k = 0; k < 7; k++) c7[k] = coords[(size_t)s * 7 + k];
      dg = reinterpret_cast<const float4*>(dout)[s];
      dg.x *= loss_scale; dg.y *= loss_scale; dg.z *= loss_scale; dg.w *= loss_scale;
    }
    uint32_t m1[2], m3[2], m4[2];
    // ---------------- forward recompute, keeping the layer inputs
    {
      const float z8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      unsigned char* a0 = act + 0 * 16384 + tid * 128;
      if (enc_in) {
        // encoding saved by the forward pass: 64 contiguous bytes per sample
#pragma unroll
        for (int c = 0; c < 4; c++) {
          uint4 e4 = make_uint4(0, 0, 0, 0);
          if (actv) e4 = reinterpret_cast<const uint4*>(enc_in + (size_t)s * ENC_DIM)[c];
          *reinterpret_cast<uint4*>(a0 + ((c ^ (tid & 7)) << 4)) = e4;
        }
      } else {
        float enc[ENC_DIM];
        hash_encode(c7, grid, lv, enc);
#pragma unroll
        for (int c = 0; c < 4; c++) store_row_chunk(a0, tid, c, enc + 8 * c);
      }
#pragma unroll
      for (int c = 4; c < 8; c++) store_row_chunk(a0, tid, c, z8);
    }
    NGP_TC_SYNC();
    mma_layer<64>(act_addr + 0 * 16384, w_addr + PW1, 2, scr, tid);
    ld_relu_store(scr, act + 1 * 16384 + tid * 128, tid, m1);
    NGP_TC_SYNC();
    mma_layer<16>(act_addr + 1 * 16384, w_addr + PW2, 4, scr, tid);
    {
      uint32_t r[32];
      tc::smem_row_ld<32>(scr, SCR_LD, tid, 0, r);
      float o[16], sh[16];
#pragma unroll
      for (int j = 0; j < 16; j++) o[j] = __uint_as_float(r[j]);
      sh4(c7 + 4, sh);
      const float z8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      unsigned char* a2 = act + 2 * 16384 + tid * 128;
      store_row_chunk(a2, tid, 0, o); store_row_chunk(a2, tid, 1, o + 8);
      store_row_chunk(a2, tid, 2, sh); store_row_chunk(a2, tid, 3, sh + 8);
#pragma unroll
      for (int c = 4; c < 8; c++) store_row_chunk(a2, tid, c, z8);
    }
    NGP_TC_SYNC();
    mma_layer<64>(act_addr + 2 * 16384, w_addr + PW3, 2, scr, tid);
    ld_relu_store(scr, act + 3 * 16384 + tid * 128, tid, m3);
    NGP_TC_SYNC();
    mma_layer<64>(act_addr + 3 * 16384, w_addr + PW4, 4, scr, tid);
    ld_relu_store(scr, act + 4 * 16384 + tid * 128, tid, m4);
    // ---------------- layer 5 backward: delta5 = d(raw rgb)
    float d64[64];
    {
      float d16[16] = {dg.x, dg.y, dg.z, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
      store_delta<16>(Dt, DT, tid, d16);
    }
    __syncthreads();                                   // ACT4 rows complete before anyone transposes... (own row only) 
    transpose_row(act + 4 * 16384, AT, tid, 64);
    NGP_TC_SYNC();
    mma_bwd_layer<16, 64>(at_addr, dt_addr, d_addr, wb_addr + PB5, dw5, 1, scr, tid);
    {
      uint32_t r[32];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        tc::smem_row_ld<32>(scr, SCR_LD, tid, h * 32, r);
#pragma unroll
        for (int j = 0; j < 32; j++) d64[h * 32 + j] = ((m4[h] >> j) & 1u) ? __uint_as_float(r[j]) : 0.f;
      }
    }
    __syncthreads();
    // ---------------- layer 4
    store_delta<64>(Dt, DT, tid, d64);
    transpose_row(act + 3 * 16384, AT, tid, 64);
    NGP_TC_SYNC();
    mma_bwd_layer<64, 64>(at_addr, dt_addr, d_addr, wb_addr + PB4, dw4, 4, scr, tid);
    {
      uint32_t r[32];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        tc::smem_row_ld<32>(scr, SCR_LD, tid, h * 32, r);
#pragma unroll
        for (int j = 0; j < 32; j++) d64[h * 32 + j] = ((m3[h] >> j) & 1u) ? __uint_as_float(r[j]) : 0.f;
      }
    }
    __syncthreads();
    // ---------------- layer 3 (input = [o(16) | sh(16)])
    store_delta<64>(Dt, DT, tid, d64);
    transpose_row(act + 2 * 16384, AT, tid, 32);
    NGP_TC_SYNC();
    mma_bwd_layer<64, 32>(at_addr, dt_addr, d_addr, wb_addr + PB3, dw3, 4, scr, tid);
    float d16[16];
    {
      uint32_t r[32];
      tc::smem_row_ld<32>(scr, SCR_LD, tid, 0, r);
#pragma unroll
      for (int j = 0; j < 16; j++) d16[j] = __uint_as_float(r[j]);
      d16[0] += dg.w;                                   // sigma path: d/d o0
    }
    __syncthreads();
    // ---------------- layer 2
    store_delta<16>(Dt, DT, tid, d16);
    transpose_row(act + 1 * 16384, AT, tid, 64);
    NGP_TC_SYNC();
    mma_bwd_layer<16, 64>(at_addr, dt_addr, d_addr, wb_addr + PB2, dw2, 1, scr, tid);
    {
      uint32_t r[32];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        tc::smem_row_ld<32>(scr, SCR_LD, tid, h * 32, r);
#pragma unroll
        for (int j = 0; j < 32; j++) d64[h * 32 + j] = ((m1[h] >> j) & 1u) ? __uint_as_float(r[j]) : 0.f;
      }
    }
    __syncthreads();
    // ---------------- layer 1
    store_delta<64>(Dt, DT, tid, d64);
    transpose_row(act + 0 * 16384, AT, tid, 32);
    NGP_TC_SYNC();
    mma_bwd_layer<64, 32>(at_addr, dt_addr, d_addr, wb_addr + PB1, dw1, 4, scr, tid);
    {
      uint32_t r[32];
      tc::smem_row_ld<32>(scr, SCR_LD, tid, 0, r);             // d/d enc [32], still loss-scaled
      if (denc_out) {
        // hand the (loss-scaled, fp16) encoding gradient to the scatter kernel
        if (actv) {
#pragma unroll
          for (int c = 0; c < 4; c++) {
            __half2 h2[4];
#pragma unroll
            for (int j = 0; j < 4; j++) h2[j] = __floats2half2_rn(__uint_as_float(r[c * 8 + 2 * j]), __uint_as_float(r[c * 8 + 2 * j + 1]));
            reinterpret_cast<uint4*>(denc_out + (size_t)s * ENC_DIM)[c] = *reinterpret_cast<const uint4*>(h2);
          }
        }
      } else if (actv) {
#pragma unroll 2
        for (int l = 0; l < N_LEVELS; l++) {
          const float ga = __uint_as_float(r[2 * l]) * inv_scale, gb = __uint_as_float(r[2 * l + 1]) * inv_scale;
          if (ga == 0.f && gb == 0.f) continue;
          const float sc = lv.scale[l];
          const float px = fmaf(c7[0], sc, 0.5f), py = fmaf(c7[1], sc, 0.5f), pz = fmaf(c7[2], sc, 0.5f);
          const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
          const float wx = px - fx, wy = py - fy, wz = pz - fz;
          const int ix = (int)fx, iy = (int)fy, iz = (int)fz;
          float2* gg = reinterpret_cast<float2*>(grid_grad) + lv.offset[l];
#pragma unroll
          for (int c = 0; c < 8; c++) {
            const int dx = c & 1, dy = (c >> 1) & 1, dz = c >> 2;
            const float w = (dx ? wx : 1.f - wx) * (dy ? wy : 1.f - wy) * (dz ? wz : 1.f - wz);
            atomicAdd(gg + grid_index(ix + dx, iy + dy, iz + dz, lv.res[l], lv.size[l], lv.dense[l]), make_float2(w * ga, w * gb));
          }
        }
      }
    }
    __syncthreads();
    first = false;
  }
  // ---------------- flush the weight-gradient accumulators into this CTA's slot (zeros when it had no tile);
  // dw_reduce_kernel adds the slots in CTA order
  float* g = dw_part + (size_t)blockIdx.x * W_TOTAL;
  flush_dw<64>(dw1, g + W1_OFF, 32, inv_scale, tid);
  flush_dw<16>(dw2, g + W2_OFF, 64, inv_scale, tid);
  flush_dw<64>(dw3, g + W3_OFF, 32, inv_scale, tid);
  flush_dw<64>(dw4, g + W4_OFF, 64, inv_scale, tid);
  flush_dw<16>(dw5, g + W5_OFF, 64, inv_scale, tid);
}

// mlp_grad[i] += sum over CTAs c (in order) of dw_part[c][i]
__global__ void dw_reduce_kernel(const float* __restrict__ dw_part, int nparts, float* __restrict__ mlp_grad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= W_TOTAL) return;
  float s = 0.f;
  for (int c = 0; c < nparts; c++) s += dw_part[(size_t)c * W_TOTAL + i];
  mlp_grad[i] += s;
}


// hash-grid gradient scatter: one thread per (sample, level) -> 8 float2 atomics.  Split from the MLP
// backward so that the atomics run at full occupancy instead of behind 4 warps per SM.
// A warp holds 32 CONSECUTIVE samples of ONE level: consecutive samples of a ray fall into the same
// cell on the coarse levels (cell >> step), so equal table indices form runs across the lanes; each
// run is summed with a segmented shuffle scan and only its head lane issues the atomic (about 40 %
// fewer atomics overall, >90 % fewer on the contended coarse levels).
constexpr float GRID_FX = 1099511627776.f;          // 2^40: fixed-point scale of the hash-grid gradient accumulator

__global__ void __launch_bounds__(256)
grid_scatter_kernel(const float* __restrict__ coords, const int* __restrict__ counters, const __half* __restrict__ denc,
                    LevelInfo lv, long long* __restrict__ grid_acc, float inv_scale) {
  const int n = counters[0];
  const int lane = threadIdx.x & 31;
  const size_t nwork = ((size_t)(n + 31) / 32) * N_LEVELS;              // (32-sample group, level) per warp
  for (size_t wid = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5; wid < nwork;
       wid += ((size_t)gridDim.x * blockDim.x) >> 5) {
    const int l = (int)(wid % N_LEVELS);
    const size_t s = (wid / N_LEVELS) * 32 + lane;
    const bool actv = s < (size_t)n;
    float ga = 0.f, gb = 0.f, wx = 0.f, wy = 0.f, wz = 0.f;
    int ix = 0, iy = 0, iz = 0;
    if (actv) {
      const float2 gd = __half22float2(reinterpret_cast<const __half2*>(denc)[s * N_LEVELS + l]);
      ga = gd.x * inv_scale; gb = gd.y * inv_scale;
      const float sc = lv.scale[l];
      const float px = fmaf(coords[s * 7 + 0], sc, 0.5f), py = fmaf(coords[s * 7 + 1], sc, 0.5f), pz = fmaf(coords[s * 7 + 2], sc, 0.5f);
      const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
      wx = px - fx; wy = py - fy; wz = pz - fz;
      ix = (int)fx; iy = (int)fy; iz = (int)fz;
    }
    long long* gg = grid_acc + 2 * (size_t)lv.offset[l];
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const int dx = c & 1, dy = (c >> 1) & 1, dz = c >> 2;
      const float w = (dx ? wx : 1.f - wx) * (dy ? wy : 1.f - wy) * (dz ? wz : 1.f - wz);
      uint32_t idx = actv ? grid_index(ix + dx, iy + dy, iz + dz, lv.res[l], lv.size[l], lv.dense[l]) : 0xffffffffu;
      float va = w * ga, vb = w * gb;
      const uint32_t prev = __shfl_up_sync(0xffffffffu, idx, 1);
      const bool head = (lane == 0) || (prev != idx);
      // run key = lane of the run's head (equal indices that are NOT adjacent are separate runs)
      const uint32_t hm = __ballot_sync(0xffffffffu, head);
      const int run = 31 - __clz(hm & (0xffffffffu >> (31 - lane)));
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int nr = __shfl_down_sync(0xffffffffu, run, o);
        const float na = __shfl_down_sync(0xffffffffu, va, o), nb = __shfl_down_sync(0xffffffffu, vb, o);
        if (lane + o < 32 && nr == run) { va += na; vb += nb; }
      }
      if (head && actv && (va != 0.f || vb != 0.f)) { fx_add(gg + 2 * (size_t)idx, va, GRID_FX); fx_add(gg + 2 * (size_t)idx + 1, vb, GRID_FX); }
    }
  }
}

// occupancy-grid refresh on tensor cores: cell -> jittered point -> hash encode -> density MLP (layers 1-2)
// -> EMA-max into density[].  Same sampling rule as ngp::density_sample_kernel (csrc/ngp_train.cu).
__global__ void __launch_bounds__(128)
density_tc_kernel(const __half2* __restrict__ grid, LevelInfo lv, const unsigned char* __restrict__ packed,
                  float aabb_lo, float inv_extent, int cascades, int n_per_cascade, uint32_t seed, float decay,
                  float* __restrict__ density) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sm = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* scr = reinterpret_cast<float*>(sm + FwdSmem::SCR);
  const int tid = threadIdx.x;
  const int total = n_per_cascade * cascades;
  const int ntiles = (total + 127) / 128;
  for (int i = tid; i < PW3 / 16; i += 128)          // W1 and W2 images only
    reinterpret_cast<uint4*>(sm + FwdSmem::W)[i] = reinterpret_cast<const uint4*>(packed)[i];
  NGP_TC_SYNC();
  const uint32_t a_addr = tc::smem_u32(sm + FwdSmem::A), w_addr = tc::smem_u32(sm + FwdSmem::W);
  unsigned char* arow = sm + FwdSmem::A + tid * 128;
  const int NC = GRID * GRID * GRID;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int i = tile * 128 + tid;
    bool actv = i < total;
    size_t gi = 0;
    float s = 1.f, x01[3] = {0.5f, 0.5f, 0.5f};
    if (actv) {
      const int mip = i / n_per_cascade, j = i % n_per_cascade;
      const uint32_t cell = (n_per_cascade >= NC) ? (uint32_t)j : density_cell(seed, mip, j);
      gi = (size_t)mip * NC + cell;
      actv = density[gi] >= 0.f;                     // never visible from a training camera -> skip
      const int ix = cell % GRID, iy = (cell / GRID) % GRID, iz = cell / (GRID * GRID);
      s = scalbnf(1.f, mip);
      const float p[3] = {((ix + rnd01(seed, i, 11)) / GRID - 0.5f) * s + 0.5f,
                          ((iy + rnd01(seed, i, 12)) / GRID - 0.5f) * s + 0.5f,
                          ((iz + rnd01(seed, i, 13)) / GRID - 0.5f) * s + 0.5f};
#pragma unroll
      for (int k = 0; k < 3; k++) x01[k] = (p[k] - aabb_lo) * inv_extent;
    }
    {
      float enc[ENC_DIM];
      if (actv) {
        hash_encode(x01, grid, lv, enc);
      } else {
#pragma unroll
        for (int k = 0; k < ENC_DIM; k++) enc[k] = 0.f;
      }
      const float z8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
      for (int c = 0; c < 4; c++) store_row_chunk(arow, tid, c, enc + 8 * c);
#pragma unroll
      for (int c = 4; c < 8; c++) store_row_chunk(arow, tid, c, z8);
    }
    NGP_TC_SYNC();
    mma_layer<64>(a_addr, w_addr + PW1, 2, scr, tid);
    {
      uint32_t r[32];
      float v[8];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        tc::smem_row_ld<32>(scr, SCR_LD, tid, h * 32, r);
#pragma unroll
        for (int c = 0; c < 4; c++) {
#pragma unroll
          for (int j = 0; j < 8; j++) v[j] = fmaxf(__uint_as_float(r[c * 8 + j]), 0.f);
          store_row_chunk(arow, tid, h * 4 + c, v);
        }
      }
    }
    NGP_TC_SYNC();
    mma_layer<16>(a_addr, w_addr + PW2, 4, scr, tid);
    {
      uint32_t r[32];
      tc::smem_row_ld<32>(scr, SCR_LD, tid, 0, r);
      if (actv) {
        const float thick = __expf(__uint_as_float(r[0])) * MIN_STEP * s;   // optical thickness of one minimal step
        density[gi] = fmaxf(density[gi] * decay, thick);
      }
    }
    __syncthreads();
  }
}

}  // namespace ngp

extern "C" {

int nslam_ngp_pack_mlp(const float* mlp, void* packed, void* stream) {
  const int total = (64 + 16 + 64 + 64 + 16) * 64;
  ngp::pack_mlp_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(mlp, (unsigned char*)packed);
  const int totalb = (64 + 64 + 32 + 64 + 32) * 64;
  ngp::pack_mlp_bwd_kernel<<<(totalb + 255) / 256, 256, 0, (cudaStream_t)stream>>>(mlp, (unsigned char*)packed + ngp::PW_TOTAL);
  return (int)cudaGetLastError();
}

/* tensor-core variant of nslam_ngp_forward: coords [n,7] (n < 0: read counters[0]) -> rgbsigma [n,4] */
int nslam_ngp_forward_tc(const nslam_ngp_model* m, const void* packed, const float* coords, const int* counters,
                         int n, int max_samples, float* rgbsigma, void* enc_out, int num_sms, void* stream) {
  using namespace ngp;
  LevelInfo lv;
  for (int l = 0; l < N_LEVELS; l++) {
    lv.scale[l] = m->scale[l]; lv.res[l] = m->res[l]; lv.size[l] = m->size[l];
    lv.offset[l] = m->offset[l]; lv.dense[l] = m->dense[l];
  }
  const int smem = FwdSmem::TOTAL + 1024;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(forward_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  const int cap = n >= 0 ? n : max_samples;
  if (cap == 0) return 0;
  int grid = (cap + 127) / 128;
  if (grid > 4 * num_sms) grid = 4 * num_sms;
  forward_tc_kernel<<<grid, 128, smem, (cudaStream_t)stream>>>(coords, counters, n, (const __half2*)m->grid_half, lv,
                                                              (const unsigned char*)packed, rgbsigma, (__half*)enc_out);
  cudaError_t e = cudaGetLastError();
  return (int)e;
}

/* tensor-core backward: recompute + all gradients; reads the sample count from counters[0].
 * mlp_grad / grid_grad accumulate (fp32 atomics); `dout` as produced by the loss kernel. */
int nslam_ngp_backward_tc(const nslam_ngp_model* m, const void* packed,
                          const float* coords, const int* counters, const float* dout, float loss_scale,
                          const void* enc_in, void* denc_scratch, int max_samples, int num_sms, void* stream) {
  using namespace ngp;
  LevelInfo lv;
  for (int l = 0; l < N_LEVELS; l++) {
    lv.scale[l] = m->scale[l]; lv.res[l] = m->res[l]; lv.size[l] = m->size[l];
    lv.offset[l] = m->offset[l]; lv.dense[l] = m->dense[l];
  }
  const int smem = BwdSmem::TOTAL + 1024;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(backward_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* dw_part = (float*)ngp_scratch(NGP_SCRATCH_DW, (size_t)num_sms * W_TOTAL * sizeof(float));
  if (!dw_part) return (int)cudaErrorMemoryAllocation;
  backward_tc_kernel<<<num_sms, 128, smem, st>>>(coords, counters, (const __half2*)m->grid_half, lv,
                                                 (const unsigned char*)packed, (const unsigned char*)packed + PW_TOTAL,
                                                 dout, dw_part, m->grid_grad, loss_scale, (const __half*)enc_in,
                                                 (__half*)denc_scratch);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  dw_reduce_kernel<<<(W_TOTAL + 255) / 256, 256, 0, st>>>(dw_part, num_sms, m->mlp_grad);
  e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  if (denc_scratch) {
    // one thread per (sample, level); the sample count lives on the device -> grid-stride over the capacity.
    // Gradients go to a fixed-point accumulator (order-independent sums) and are added to grid_grad afterwards.
    const size_t n_vals = 2 * (size_t)m->n_grid;
    long long* acc = (long long*)ngp_scratch(NGP_SCRATCH_GRID, n_vals * sizeof(long long));
    if (!acc) return (int)cudaErrorMemoryAllocation;
    size_t want = (((size_t)max_samples + 31) / 32 * N_LEVELS * 32 + 255) / 256;
    const size_t cap = (size_t)num_sms * 32;
    grid_scatter_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, st>>>(coords, counters, (const __half*)denc_scratch, lv,
                                                                            acc, 1.f / loss_scale);
    fx_flush_kernel<<<(unsigned)(num_sms * 8), 256, 0, st>>>(acc, m->grid_grad, n_vals, 1.f / GRID_FX);
    e = cudaGetLastError();
  }
  return (int)e;
}

/* one training step with the network on tensor cores: sample -> forward_tc -> loss -> backward_tc
 * (same contract as nslam_ngp_train_step; `packed` from nslam_ngp_pack_mlp of the CURRENT weights) */
int nslam_ngp_train_step_tc(const nslam_ngp_model* m, const nslam_ngp_images* im, const nslam_ngp_batch* b,
                            const void* packed, int n_rays, unsigned seed, float lambda_depth, float bg_r,
                            float bg_g, float bg_b, float loss_scale, int num_sms, void* stream) {
  int r = nslam_ngp_sample_phase(m, im, b, n_rays, seed, stream);
  if (r) return r;
  r = nslam_ngp_forward_tc(m, packed, b->coords, b->counters, -1, b->max_samples, b->rgbsigma, b->enc, num_sms, stream);
  if (r) return r;
  r = nslam_ngp_loss_phase(b, n_rays, lambda_depth, bg_r, bg_g, bg_b, stream);
  if (r) return r;
  return nslam_ngp_backward_tc(m, packed, b->coords, b->counters, b->dout, loss_scale, b->enc, b->denc, b->max_samples,
                               num_sms, stream);
}

/* tests: loss + gradients on caller-provided rays/samples through the tensor-core kernels */
int nslam_ngp_loss_backward_tc(const nslam_ngp_model* m, const nslam_ngp_batch* b, const void* packed, int n_rays,
                               int n_samples, float lambda_depth, float bg_r, float bg_g, float bg_b,
                               float loss_scale, int num_sms, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  int h[4] = {n_samples, n_rays, n_rays, 0};
  cudaMemcpyAsync(b->counters, h, sizeof(h), cudaMemcpyHostToDevice, st);
  cudaMemsetAsync(b->loss, 0, sizeof(float), st);
  int r = nslam_ngp_forward_tc(m, packed, b->coords, b->counters, -1, b->max_samples, b->rgbsigma, b->enc, num_sms, stream);
  if (r) return r;
  r = nslam_ngp_loss_phase(b, n_rays, lambda_depth, bg_r, bg_g, bg_b, stream);
  if (r) return r;
  return nslam_ngp_backward_tc(m, packed, b->coords, b->counters, b->dout, loss_scale, b->enc, b->denc, b->max_samples,
                               num_sms, stream);
}

/* density MLP on tensor cores for the occupancy-grid refresh (phase of nslam_ngp_update_density_grid) */
int nslam_ngp_density_sample_tc(const nslam_ngp_model* m, const void* packed, int n_per_cascade, unsigned seed,
                                float decay, int num_sms, void* stream) {
  using namespace ngp;
  LevelInfo lv;
  for (int l = 0; l < N_LEVELS; l++) {
    lv.scale[l] = m->scale[l]; lv.res[l] = m->res[l]; lv.size[l] = m->size[l];
    lv.offset[l] = m->offset[l]; lv.dense[l] = m->dense[l];
  }
  const int smem = FwdSmem::TOTAL + 1024;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(density_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  const int total = n_per_cascade * m->cascades;
  if (total == 0) return 0;
  int grid = (total + 127) / 128;
  if (grid > 4 * num_sms) grid = 4 * num_sms;
  density_tc_kernel<<<grid, 128, smem, (cudaStream_t)stream>>>((const __half2*)m->grid_half, lv, (const unsigned char*)packed,
                                                              0.5f - 0.5f * m->aabb_scale, 1.f / m->aabb_scale, m->cascades,
                                                              n_per_cascade, seed, decay, m->density);
  return (int)cudaGetLastError();
}

}  // extern "C"
