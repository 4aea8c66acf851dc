/* C ABI of the tensor-core convolution used by the update operator (SURVEY.md §8 rows A5, A1).
 * Replaces the cuDNN convolutions + torch.cat + elementwise gating kernels behind
 * UpdateModule.forward (networks/droid_net.py:118-150), ConvGRU.forward
 * (networks/modules/gru.py:19-32) and GraphAgg.forward (networks/droid_net.py:59-75).
 * See nerf_slam_b200/csrc/conv_igemm.cu for the epilogue modes. */
#ifndef NSLAM_NN_H_
#define NSLAM_NN_H_
#ifdef __cplusplus
extern "C" {
#endif

/* srcs: HOST array of n_src (<=4) DEVICE pointers to NHWC fp16 tensors [B,H,W,src_channels[i]]
 * (src_channels: HOST ints, each a multiple of 8); wpacked: DEVICE, packed by
 * nerf_slam_b200/conv.py::pack_weights; bias/gctx/gsum fp32 DEVICE; out0/out1 NHWC fp16 DEVICE
 * (out0 may be a channel slice: pass the pointer to its first channel and the FULL channel count
 * of the underlying tensor as out0_channels).  N in {16,64,128,256}.
 * partials: DEVICE fp32 scratch of B * T * 4 * N floats (T = ceil(H/8) * ceil(W/16) tiles per image) for mode 3,
 * NULL otherwise: per-tile column sums, reduced in a fixed order into gsum (+=) so that gsum is the same on every run. */
int nslam_conv_igemm(const void* const* srcs, const int* src_channels, int n_src, int B, int H, int W,
                     int KH, int KW, int pad, int N, const void* wpacked, const float* bias, int mode,
                     int act, const float* gctx, const void* net, const void* zbuf, float* gsum,
                     void* out0, int out0_channels, void* out1, float* partials, int num_sms, void* stream);

/* extended form: mode 4 = encoder layer (BasicEncoder, networks/modules/extractor.py:118-198):
 *   stats [B][N][2] fp32 (zeroed by the caller) or NULL: per-image channel sum / sum of squares of the fp16
 *   outputs, consumed by nslam_inorm_apply; sub = 2: stride-2 convolution (out0 is [B,ceil(H/2),ceil(W/2),C]).
 *   With stats, partials = B * T * 4 * N * 2 floats of scratch (T as above, from the stride-1 H, W). */
int nslam_conv_igemm_ex(const void* const* srcs, const int* src_channels, int n_src, int B, int H, int W,
                        int KH, int KW, int pad, int N, const void* wpacked, const float* bias, int mode,
                        int act, const float* gctx, const void* net, const void* zbuf, float* gsum,
                        void* out0, int out0_channels, void* out1, float* stats, int sub, float* partials,
                        int num_sms, void* stream);
/* im2col of the encoders' 7x7 / stride-2 / 3-channel first layer: x [B,3,H,W] fp32 -> [B,H/2,W/2,152] fp16,
 * K index = (ky*7 + kx)*3 + c (147 real columns) -> the layer runs as a 1x1 GEMM (extractor.py:139). */
int nslam_im2col7_s2(const float* x, void* out, int B, int H, int W, void* stream);

/* ---- fused glue around the update operator (csrc/update_glue.cu); all DEVICE pointers -------------
 * motion_im2col: motion = clamp([coords1-coords0 | target-coords1], +-64) (visual_frontend.py:392-394)
 *   laid out as the 7x7 im2col [E,ht,wd,200] fp16 (tap-major, 4 channels per tap, cols 196..199 zero) so
 *   that flow_encoder.0 (droid_net.py:95) runs as a 1x1 GEMM; target may be NULL (motion filter: zeros).
 * flow_heads_post: h2 [E,ht,wd,16] fp16 (delta | weight logits, droid_net.py:138-139) ->
 *   flow = coords1 + delta, conf = sigmoid(.) as [E,ht,wd,2] fp32 and (optional) planar [E,2,ht,wd] copies
 *   straight into the BA input buffers (visual_frontend.py:404-405,431-436).
 * segment_mean: GraphAgg scatter_mean over edges with the same source keyframe (droid_net.py:67);
 *   seg_ptr [K+1], seg_edges [E] (CSR, host-built), a [E,hw,128] fp16 -> out [K,hw,128] fp16.
 * eta_damping: e16 [K,hw,16] fp16 -> damping[ux[k]] = 0.01 softplus(col 0) (droid_net.py:73);
 *   ba_damp[j] = 0.2 damping[kx_ba[j]] + ep (visual_frontend.py:423). */
int nslam_motion_im2col(const float* coords1, const float* coords0, const float* target, void* out,
                        int E, int ht, int wd, void* stream);
int nslam_flow_heads_post(const void* h2, const float* coords1, float* flow, float* conf, float* ba_target,
                          float* ba_weight, int E, int hw, void* stream);
int nslam_segment_mean(const void* a, const int* seg_ptr, const int* seg_edges, void* out, int K, int hw,
                       void* stream);
int nslam_eta_damping(const void* e16, const long long* ux, float* damping, int K, const long long* kx_ba,
                      float* ba_damp, int Kba, int hw, float ep, void* stream);

/* ---- the whole update operator in one host call (csrc/update_step.cu) -------------------------------------
 * UpdateModule.forward + GraphAgg (networks/droid_net.py:59-75,118-150) on a fixed edge set: every pointer is a
 * DEVICE pointer, the struct itself lives on the host.  Weight slots follow conv.py::UpdateOperatorTC (packed by
 * pack_weights).  net_out may alias net (in-place hidden-state update).  K == 0: skip GraphAgg. */
enum { NSLAM_W_CE0 = 0, NSLAM_W_CE2, NSLAM_W_FE0, NSLAM_W_FE2, NSLAM_W_GLO, NSLAM_W_ZR, NSLAM_W_Q, NSLAM_W_H0, NSLAM_W_H2,
       NSLAM_W_A1, NSLAM_W_A2, NSLAM_W_ETA, NSLAM_W_UM0, NSLAM_W_UM1, NSLAM_W_UM2, NSLAM_W_COUNT };
typedef struct nslam_update_ctx {
  int E, K, H, W, num_sms, corr_channels, Kba;
  float ep;
  /* inputs */
  const void* net; const void* inp; const void* corr;          /* [E,H,W,128] x2, [E,H,W,corr_channels] fp16 */
  const float* coords1; const float* coords0; const float* target;   /* [E,H,W,2], [H,W,2], [E,H,W,2] or NULL */
  const int* seg_ptr; const int* seg_edges;                     /* GraphAgg CSR: [K+1], [E] */
  /* outputs */
  void* net_out;                                                /* [E,H,W,128] fp16 */
  float* flow; float* conf; float* ba_target; float* ba_weight; /* [E,H,W,2] x2, planar [E,2,H,W] x2 (or NULL) */
  void* upmask;                                                 /* [K,H,W,576] fp16 */
  const long long* ux; float* damping; const long long* kx_ba; float* ba_damp;   /* eta -> damping (or damping NULL) */
  /* weights */
  const void* wp[NSLAM_W_COUNT]; const float* bias[NSLAM_W_COUNT];
  const float* glo_w; const float* glo_b;                        /* [384,128], [384] fp32 */
  /* workspace (fp16 unless noted) */
  /* gsum: [E][128] followed by the glo convolution's partials [E][T][4][128] (T = ceil(H/8) * ceil(W/16)) */
  void* c1; void* c2; void* mcol; void* f1; void* f2; float* gsum; float* gzr; float* gq;
  void* z; void* rnet; void* h0; void* h2; void* a1; void* am; void* a2; void* e16;
} nslam_update_ctx;
int nslam_update_op_step(const nslam_update_ctx* ctx, void* stream);

/* ---- instance norm of the feature encoder (csrc/inorm.cu), NHWC fp16 ----------------------------------
 * Replaces F.instance_norm + ReLU (+ residual add + ReLU) of BasicEncoder/ResidualBlock with
 * norm_fn='instance' (networks/modules/extractor.py:6-60,118-198): biased variance, eps 1e-5, fp32
 * statistics, fp16 rounding after the normalisation and after the residual add like the library path.
 * stats [B,C,2] = per-(image, channel) sum and sum of squares. */
int nslam_inorm_stats(const void* x, float* stats, int B, int HW, int C, int zero_first, void* stream);
int nslam_inorm_apply(const void* x, const float* stats, const void* res, const float* res_stats, void* out,
                      int B, int HW, int C, float eps, int relu, void* stream);

#ifdef __cplusplus
}
#endif
#endif
