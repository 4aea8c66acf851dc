/* C ABI of Path B — hash-grid NeRF training / rendering (SURVEY.md §8 rows B1-B4).
 *
 * Replaces the `pyngp` module of the reference's instant-ngp fork as driven by
 * fusion/nerf_fusion.py: Testbed.frame() (:299) = nslam_ngp_train_step + nslam_ngp_adam
 * (+ nslam_ngp_update_density_grid every 16 steps), Testbed.render() (:416,424) =
 * nslam_ngp_render_tile, nerf.training.update_training_images() (:285-289) = nslam_ngp_ingest_image
 * into pre-allocated device slots.  The fork's sources are absent from /root/reference
 * (empty submodule) — semantics follow the published instant-ngp algorithm; see oracle/ngp.py.
 *
 * All pointers are DEVICE pointers (the structs themselves live on the host); every call
 * launches on `stream` and never synchronises.  Returns 0 or a cudaError_t value.
 */
#ifndef NSLAM_NGP_H_
#define NSLAM_NGP_H_

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nslam_ngp_model {
  void* grid_half;        /* __half2 [n_grid]   fp16 compute copy of the hash table            */
  float* grid_master;     /* [n_grid*2]         fp32 master                                    */
  float* grid_grad;       /* [n_grid*2]                                                        */
  float* grid_m; float* grid_v;   /* Adam moments                                              */
  float* mlp;             /* [10240] fp32: W1[32][64] W2[64][16] W3[32][64] W4[64][64] W5[64][16] */
  float* mlp_grad; float* mlp_m; float* mlp_v;
  float* density;         /* [cascades*128^3] optical thickness, -1 = never visible            */
  unsigned char* bits;    /* [cascades*128^3/8] occupancy bitfield                             */
  float* stats;           /* [2] scratch                                                       */
  float aabb_scale; int cascades; float cone; float near_distance;
  float scale[16]; int res[16]; unsigned size[16]; unsigned offset[16]; int dense[16];
  unsigned n_grid;
} nslam_ngp_model;

typedef struct nslam_ngp_images {
  const void* rgba;       /* __half [N,H,W,4] linear premultiplied                             */
  const float* depth;     /* [N,H,W] metric z-depth, <= 0 = none                               */
  const float* depth_cov; /* [N,H,W]                                                           */
  const void* cams;       /* [N] {float c2w[12]; float fx,fy,cx,cy; int w,h;}                  */
  const int* active;      /* [n_active] slots used for training                                */
  int n_active, H, W;
} nslam_ngp_images;

typedef struct nslam_ngp_batch {
  float* rays;       /* [max_rays,16]   */
  float* coords;     /* [max_samples,7] */
  float* tdist;      /* [max_samples]   */
  float* rgbsigma;   /* [max_samples,4] */
  float* dout;       /* [max_samples,4] */
  int* counters;     /* [4]: samples, rays kept */
  float* loss;       /* [1] */
  int max_rays, max_samples;
  void* enc;         /* __half [max_samples,32]  hash encodings kept by the tensor-core forward (or NULL) */
  void* denc;        /* __half [max_samples,32]  loss-scaled encoding gradients for the scatter kernel (or NULL) */
} nslam_ngp_batch;

int nslam_ngp_train_step(const nslam_ngp_model* m, const nslam_ngp_images* im, const nslam_ngp_batch* b,
                         int n_rays, unsigned seed, float lambda_depth, float bg_r, float bg_g,
                         float bg_b, int num_sms, void* stream);
int nslam_ngp_adam(const nslam_ngp_model* m, int step, float lr, float beta1, float beta2, float eps,
                   float l2_mlp, void* stream);
int nslam_ngp_forward(const nslam_ngp_model* m, const float* coords, int n, float* rgbsigma, void* stream);
int nslam_ngp_loss_backward(const nslam_ngp_model* m, const nslam_ngp_batch* b, int n_rays, int n_samples,
                            float lambda_depth, float bg_r, float bg_g, float bg_b, int num_sms, void* stream);
/* packed != NULL: the density MLP of the refresh runs on tensor cores (nslam_ngp_density_sample_tc) */
int nslam_ngp_update_density_grid(const nslam_ngp_model* m, const nslam_ngp_images* im, int n_per_cascade,
                                  unsigned seed, float decay, float min_thickness, const void* packed, int num_sms,
                                  void* stream);
int nslam_ngp_density_sample_tc(const nslam_ngp_model* m, const void* packed, int n_per_cascade, unsigned seed,
                                float decay, int num_sms, void* stream);
/* packed (see nslam_ngp_pack_mlp) != NULL: network on tensor cores; NULL: fp32 CUDA-core forward */
int nslam_ngp_render_tile(const nslam_ngp_model* m, const nslam_ngp_batch* b, const float* cam18_host,
                          int x0, int y0, int tw, int th, int max_per_ray, float bg_r, float bg_g,
                          float bg_b, float* out_rgbd, const void* packed, int num_sms, void* stream);
int nslam_ngp_ingest_image(const unsigned char* rgb_chw, const float* idepth_up, const float* depth_cov_up,
                           int H, int W, void* rgba_slot, float* depth_slot, float* cov_slot, void* stream);
/* process_slam + send_data (fusion/nerf_fusion.py:140-289) for a whole packet in one launch, device to device: images,
 * depths (1 / idepth), covariances into slots ids[k]; camera records from the packet's cam_T_world poses [n,7] (t, q_xyzw;
 * world_T_cam 3x4 = inverse, nerf scale 1 / offset 0) or untouched when cam_T_world is NULL.  ids: DEVICE int64 [n].
 * cams_base [N] / cam_state [3,N,6] (offsets | Adam m | v) / cam_steps [N], all or none: pose-refinement state, the slots
 * written get the new base camera and a reset refinement (see nslam_ngp_cam_adam_apply). */
int nslam_ngp_ingest_batch(const unsigned char* rgb_chw, const float* idepth_up, const float* depth_cov_up,
                           const long long* ids, int n, int H, int W, void* rgba, float* depth, float* depth_cov,
                           const float* cam_T_world, float fx, float fy, float cx, float cy, void* cams, void* cams_base,
                           float* cam_state, int* cam_steps, int n_slots, void* stream);

/* Camera-pose refinement (`nerf.training.optimize_extrinsics`, fusion/nerf_fusion.py:99; csrc/ngp_extrinsics.cu):
 * gradient of the batch just back-propagated w.r.t. each camera's translation and rotation vector, accumulated into
 * cam_grad [n_images,6]; then Adam on the offsets [n_images,6] and the effective cameras the sampler reads. */
int nslam_ngp_cam_grad(const void* grid_half, const float* scale16, const int* res16, const unsigned* size16,
                       const unsigned* offset16, const int* dense16, float aabb_scale, const float* rays, int max_rays,
                       const float* coords, const float* tdist, const void* denc, float loss_scale, float* cam_grad,
                       int n_images, void* stream);
int nslam_ngp_cam_adam_apply(const void* base_cams, void* eff_cams, float* offsets, float* cam_grad, float* m, float* v,
                             int* steps, int n, float lr, float beta1, float beta2, float eps, float l2, void* stream);

/* tensor-core (wgmma) variants of the network forward / backward, fused with the hash encoding
 * (csrc/ngp_tc.cu).  `packed` = 61 440-byte buffer of fp16 wgmma-ready weight images (forward images
 * B[n][k] at 0, backward images B[k][n] at 28 672) produced by nslam_ngp_pack_mlp from the fp32 MLP blob
 * (re-run after every optimiser step).  n < 0: sample count read from counters[0].  The backward
 * carries its deltas in fp16 multiplied by `loss_scale` (instant-ngp's mixed-precision recipe) and
 * accumulates weight gradients in registers across all tiles of a CTA. */
int nslam_ngp_pack_mlp(const float* mlp, void* packed, void* stream);
int nslam_ngp_forward_tc(const nslam_ngp_model* m, const void* packed, const float* coords, const int* counters,
                         int n, int max_samples, float* rgbsigma, void* enc_out, int num_sms, void* stream);
/* enc_in (from forward_tc's enc_out) or NULL = re-gather; denc_scratch or NULL = scatter inside the kernel.
 * With denc_scratch the hash-grid scatter runs as its own full-occupancy kernel (one thread per
 * sample x level) after the MLP backward. */
int nslam_ngp_backward_tc(const nslam_ngp_model* m, const void* packed, const float* coords, const int* counters,
                          const float* dout, float loss_scale, const void* enc_in, void* denc_scratch,
                          int max_samples, int num_sms, void* stream);
int nslam_ngp_train_step_tc(const nslam_ngp_model* m, const nslam_ngp_images* im, const nslam_ngp_batch* b,
                            const void* packed, int n_rays, unsigned seed, float lambda_depth, float bg_r,
                            float bg_g, float bg_b, float loss_scale, int num_sms, void* stream);
int nslam_ngp_loss_backward_tc(const nslam_ngp_model* m, const nslam_ngp_batch* b, const void* packed, int n_rays,
                               int n_samples, float lambda_depth, float bg_r, float bg_g, float bg_b,
                               float loss_scale, int num_sms, void* stream);
/* the non-network phases of a step (shared by both variants) */
int nslam_ngp_sample_phase(const nslam_ngp_model* m, const nslam_ngp_images* im, const nslam_ngp_batch* b,
                           int n_rays, unsigned seed, void* stream);
int nslam_ngp_loss_phase(const nslam_ngp_batch* b, int n_rays, float lambda_depth, float bg_r, float bg_g,
                         float bg_b, void* stream);

#ifdef __cplusplus
}
#endif
#endif
