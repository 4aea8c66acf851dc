// A5/A19 — the whole update operator (UpdateModule.forward + GraphAgg, reference
// networks/droid_net.py:59-75,118-150) as ONE host call: the 15 tensor-core convolutions, the fused glue
// kernels and the global-context GEMV are sequenced here on one stream with every intermediate in a
// caller-provided workspace.  The Python host then issues ~10 calls per update() instead of ~60
// (0.15 ms instead of ~1 ms of host time), which removes the need to re-capture a CUDA graph whenever
// the edge set changes.  Same kernels, same order and same arithmetic as conv.py::UpdateOperatorTC.__call__.
#include "common.cuh"
#include "../../include/nslam_nn.h"

namespace nslam {

// g3[e][o] = b[o] + sum_c w[o][c] * half(gsum[e][c] / HW)     (the reference's `glo` is an fp16 tensor)
__global__ void __launch_bounds__(128)
glo_context_kernel(const float* __restrict__ gsum, const float* __restrict__ w, const float* __restrict__ b,
                   float inv_hw, float* __restrict__ gzr, float* __restrict__ gq, int E) {
  __shared__ float g[128];
  const int e = blockIdx.x;
  g[threadIdx.x] = __half2float(__float2half_rn(gsum[(size_t)e * 128 + threadIdx.x] * inv_hw));
  __syncthreads();
  for (int o = threadIdx.x; o < 384; o += 128) {
    const float4* wr = reinterpret_cast<const float4*>(w + (size_t)o * 128);
    float acc = 0.f;
#pragma unroll 8
    for (int c = 0; c < 32; c++) {
      const float4 w4 = wr[c];
      acc = fmaf(w4.x, g[4 * c], acc); acc = fmaf(w4.y, g[4 * c + 1], acc);
      acc = fmaf(w4.z, g[4 * c + 2], acc); acc = fmaf(w4.w, g[4 * c + 3], acc);
    }
    acc += b[o];
    if (o < 256) gzr[(size_t)e * 256 + o] = acc; else gq[(size_t)e * 128 + (o - 256)] = acc;
  }
}

}  // namespace nslam

extern "C" int nslam_update_op_step(const nslam_update_ctx* c, void* stream) {
  using namespace nslam;
  cudaStream_t st = (cudaStream_t)stream;
  const int E = c->E, K = c->K, H = c->H, W = c->W, S = c->num_sms;
  if (E <= 0) return 0;
  int r;
  auto conv = [&](const void* const* srcs, const int* ch, int ns, int B, int k, int N, int wi, int mode, int act,
                  const float* gctx, const void* net, const void* zbuf, float* gsum, void* out0, int oc, void* out1) {
    // mode 3 (glo): its per-tile partials live behind gsum[E][128] in the same workspace slice
    return nslam_conv_igemm(srcs, ch, ns, B, H, W, k, k, k / 2, N, c->wp[wi], c->bias[wi], mode, act, gctx, net, zbuf, gsum,
                            out0, oc, out1, mode == 3 ? gsum + (size_t)B * 128 : nullptr, S, stream);
  };
  // correlation / motion encoders
  { const void* s[1] = {c->corr}; int ch[1] = {c->corr_channels};
    if ((r = conv(s, ch, 1, E, 1, 128, NSLAM_W_CE0, 0, 1, nullptr, nullptr, nullptr, nullptr, c->c1, 128, nullptr))) return r; }
  { const void* s[1] = {c->c1}; int ch[1] = {128};
    if ((r = conv(s, ch, 1, E, 3, 128, NSLAM_W_CE2, 0, 1, nullptr, nullptr, nullptr, nullptr, c->c2, 128, nullptr))) return r; }
  if ((r = nslam_motion_im2col(c->coords1, c->coords0, c->target, c->mcol, E, H, W, stream))) return r;
  { const void* s[1] = {c->mcol}; int ch[1] = {200};
    if ((r = conv(s, ch, 1, E, 1, 128, NSLAM_W_FE0, 0, 1, nullptr, nullptr, nullptr, nullptr, c->f1, 128, nullptr))) return r; }
  { const void* s[1] = {c->f1}; int ch[1] = {128};
    if ((r = conv(s, ch, 1, E, 3, 64, NSLAM_W_FE2, 0, 1, nullptr, nullptr, nullptr, nullptr, c->f2, 64, nullptr))) return r; }
  // global context
  { cudaError_t me = cudaMemsetAsync(c->gsum, 0, (size_t)E * 128 * sizeof(float), st); if (me != cudaSuccess) return (int)me; }
  { const void* s[1] = {c->net}; int ch[1] = {128};
    if ((r = conv(s, ch, 1, E, 1, 128, NSLAM_W_GLO, 3, 0, nullptr, c->net, nullptr, c->gsum, nullptr, 0, nullptr))) return r; }
  glo_context_kernel<<<E, 128, 0, st>>>(c->gsum, c->glo_w, c->glo_b, 1.0f / (float)(H * W), c->gzr, c->gq, E);
  NSLAM_CHECK_LAUNCH();
  // ConvGRU: z | r gates, then q + state update written IN PLACE into the hidden state (the q convolution reads
  // `net` only in its epilogue, pixel by pixel, and none of its A-operand sources is `net`)
  { const void* s[4] = {c->net, c->inp, c->c2, c->f2}; int ch[4] = {128, 128, 128, 64};
    if ((r = conv(s, ch, 4, E, 3, 256, NSLAM_W_ZR, 1, 0, c->gzr, c->net, nullptr, nullptr, c->z, 128, c->rnet))) return r; }
  { const void* s[4] = {c->rnet, c->inp, c->c2, c->f2}; int ch[4] = {128, 128, 128, 64};
    if ((r = conv(s, ch, 4, E, 3, 128, NSLAM_W_Q, 2, 0, c->gq, c->net, c->z, nullptr, c->net_out, 128, nullptr))) return r; }
  // heads
  { const void* s[1] = {c->net_out}; int ch[1] = {128};
    if ((r = conv(s, ch, 1, E, 3, 256, NSLAM_W_H0, 0, 1, nullptr, nullptr, nullptr, nullptr, c->h0, 256, nullptr))) return r; }
  { const void* s[1] = {c->h0}; int ch[1] = {256};
    if ((r = conv(s, ch, 1, E, 3, 16, NSLAM_W_H2, 0, 0, nullptr, nullptr, nullptr, nullptr, c->h2, 16, nullptr))) return r; }
  if ((r = nslam_flow_heads_post(c->h2, c->coords1, c->flow, c->conf, c->ba_target, c->ba_weight, E, H * W, stream))) return r;
  if (K <= 0) return 0;
  // GraphAgg
  { const void* s[1] = {c->net_out}; int ch[1] = {128};
    if ((r = conv(s, ch, 1, E, 3, 128, NSLAM_W_A1, 0, 1, nullptr, nullptr, nullptr, nullptr, c->a1, 128, nullptr))) return r; }
  if ((r = nslam_segment_mean(c->a1, c->seg_ptr, c->seg_edges, c->am, K, H * W, stream))) return r;
  { const void* s[1] = {c->am}; int ch[1] = {128};
    if ((r = conv(s, ch, 1, K, 3, 128, NSLAM_W_A2, 0, 1, nullptr, nullptr, nullptr, nullptr, c->a2, 128, nullptr))) return r; }
  { const void* s[1] = {c->a2}; int ch[1] = {128};
    if ((r = conv(s, ch, 1, K, 3, 16, NSLAM_W_ETA, 0, 0, nullptr, nullptr, nullptr, nullptr, c->e16, 16, nullptr))) return r; }
  { const void* s[1] = {c->a2}; int ch[1] = {128};
    __half* um = (__half*)c->upmask;
    if ((r = conv(s, ch, 1, K, 1, 256, NSLAM_W_UM0, 0, 0, nullptr, nullptr, nullptr, nullptr, um, 576, nullptr))) return r;
    if ((r = conv(s, ch, 1, K, 1, 256, NSLAM_W_UM1, 0, 0, nullptr, nullptr, nullptr, nullptr, um + 256, 576, nullptr))) return r;
    if ((r = conv(s, ch, 1, K, 1, 64, NSLAM_W_UM2, 0, 0, nullptr, nullptr, nullptr, nullptr, um + 512, 576, nullptr))) return r; }
  if (c->damping)
    if ((r = nslam_eta_damping(c->e16, c->ux, c->damping, K, c->kx_ba, c->ba_damp, c->Kba, H * W, c->ep, stream))) return r;
  return 0;
}
