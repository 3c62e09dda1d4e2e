/* lion_b200 -- C ABI of the H100-native (sm_90a) LION sampling hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b).  Every entry point takes plain device pointers,
 * sizes and a cudaStream_t (as void*), returns 0 on success or a negative code (never exits
 * the process -- the reference's kernels exit(-1) on a launch error,
 * third_party/pvcnn/functional/src/cuda_utils.cuh:28-37), allocates nothing on the stream
 * path and is CUDA-graph capturable after one warm-up call.  lion_last_error() describes the
 * last failure of the calling thread.  "reference" paths below are relative to the
 * reference repository.
 */
#ifndef LION_B200_H
#define LION_B200_H
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct LionCtx LionCtx;       /* device + scratch arena                         */
typedef struct LionModel LionModel;   /* packed weights of one network / one block      */

int lion_version(void);
const char* lion_last_error(void);
int lion_ctx_create(int device, LionCtx** out);
int lion_ctx_destroy(LionCtx* ctx);
/* kernels launched by the last network-level call on this context (bench.py: gpu_launches) */
int lion_ctx_last_launches(LionCtx* ctx);
/* Scratch-arena generation: bumped whenever a call had to re-allocate the per-device arena or zero grid.  A CUDA graph
 * captured on this context has the arena addresses baked in; it must not be replayed once the generation changed
 * (lion_b200._lib.capture_graph checks this and raises). */
unsigned lion_ctx_generation(LionCtx* ctx);
/* Diagnostic (contexts created with LION_TIMELINE=1 in the environment only): the network-level forward drops
 * %globaltimer stamps into both of its streams at block boundaries; this returns the stamps of the last forward
 * (or of the last replay of a graph captured from it): t_ns[i] and a 24-byte name per entry.  Returns the count,
 * < 0 on error.  Synchronises the device.  Used by tools/timeline_step.py (the image has no nsys). */
int lion_ctx_timeline(LionCtx* ctx, unsigned long long* t_ns, char* names, int max_entries);
size_t lion_ctx_arena_bytes(LionCtx* ctx);
/* device scratch the context currently owns (arena + persistent zero grid).  Entry points size it with a dry
 * pass and grow it on demand -- outside stream capture: run one eager call per shape before capturing. */
size_t lion_workspace_bytes(LionCtx* ctx);

/* ---------------------------------------------------------------------------------------
 * The seven operators of third_party/pvcnn/functional (reference layouts: features [B,C,N]
 * channel-major fp32, coords [B,3,N], flat voxel index x*r*r + y*r + z).  Outputs are
 * caller-allocated (the reference's C++ wrappers allocate them with torch::zeros).
 * ------------------------------------------------------------------------------------- */
/* replaces avg_voxelize_forward, src/bindings.cpp:33 -> voxelization/vox.cpp:17-43.
 * out [B,C,r^3] fp32, ind [B,N] int32, cnt [B,r^3] int32 (all written). */
int lion_avg_voxelize(const float* features, const int* coords, float* out, int* ind, int* cnt,
                      int B, int C, int N, int r, void* stream);
/* replaces trilinear_devoxelize_forward, src/bindings.cpp:29 -> interpolate/trilinear_devox.cpp:18-55.
 * grid [B,C,r^3], coords [B,3,N] fp32 in voxel units; out [B,C,N]; inds/wgts [B,8,N] written
 * only when is_training (may be NULL otherwise). */
int lion_trilinear_devoxelize(const float* grid, const float* coords, float* out, int* inds, float* wgts,
                              int B, int C, int N, int r, int is_training, void* stream);
/* replaces furthest_point_sampling, src/bindings.cpp:15 -> sampling/sampling.cpp:43-58. idx [B,M] int32. */
int lion_furthest_point_sampling(const float* coords, int* idx, int B, int N, int M, void* stream);
/* replaces gather_features_forward, src/bindings.cpp:11 -> sampling/sampling.cpp:6-24. out [B,C,M]. */
int lion_gather(const float* features, const int* idx, float* out, int B, int C, int N, int M, void* stream);
/* replaces ball_query, src/bindings.cpp:17 -> ball_query/ball_query.cpp:6-27. out [B,M,K] int32, K<=32. */
int lion_ball_query(const float* centers, const float* points, int* out, int B, int N, int M, float radius, int K,
                    void* stream);
/* replaces grouping_forward, src/bindings.cpp:18 -> grouping/grouping.cpp:6-24. out [B,C,M,U]. */
int lion_grouping(const float* features, const int* idx, float* out, int B, int C, int N, int M, int U, void* stream);
/* replaces three_nearest_neighbors_interpolate_forward, src/bindings.cpp:22 ->
 * interpolate/neighbor_interpolate.cpp:10-41. out [B,C,N], idx/wgt [B,3,N] (all written). */
int lion_three_nn_interpolate(const float* points, const float* centers, const float* centers_features, float* out,
                              int* idx, float* wgt, int B, int C, int N, int M, void* stream);
/* the coordinate half of Voxelization.forward (models/pvcnn2_ada.py:173-188):
 * norm_coords [B,3,N] fp32 in [0,r-1], vox [B,3,N] int32 = round-half-even. */
int lion_voxel_coords(const float* coords, float* norm_coords, int* vox, int B, int N, int r, int normalize, float eps,
                      void* stream);

/* ---- backward passes of the five differentiable operators (training path, SURVEY.md 8f rank 4).  Reference:
 * src/bindings.cpp:12-13 gather_features_backward, :19-20 grouping_backward, :24-25
 * three_nearest_neighbors_interpolate_backward, :29-30 trilinear_devoxelize_backward, :33-34 avg_voxelize_backward
 * (kernels vox.cu:86-110, trilinear_devox.cu:119-162, grouping.cu:58-77, neighbor_interpolate.cu:145-170,
 * sampling.cu:52-66).  Same layouts as the forward entry points; grad_x is fully written (zeroed inside where the
 * gradient is a scatter-add). ---- */
int lion_avg_voxelize_backward(const float* grad_y /*[B,C,r^3]*/, const int* ind /*[B,N]*/, const int* cnt /*[B,r^3]*/,
                               float* grad_x /*[B,C,N]*/, int B, int C, int N, int r, void* stream);
int lion_trilinear_devoxelize_backward(const float* grad_y /*[B,C,N]*/, const int* inds /*[B,8,N]*/, const float* wgts /*[B,8,N]*/,
                                       float* grad_x /*[B,C,r^3]*/, int B, int C, int N, int r, void* stream);
int lion_grouping_backward(const float* grad_y /*[B,C,M,U]*/, const int* idx /*[B,M,U]*/, float* grad_x /*[B,C,N]*/, int B, int C,
                           int N, int M, int U, void* stream);
int lion_three_nn_interpolate_backward(const float* grad_y /*[B,C,N]*/, const int* idx /*[B,3,N]*/, const float* wgt /*[B,3,N]*/,
                                       float* grad_x /*[B,C,M]*/, int B, int C, int N, int M, void* stream);
int lion_gather_backward(const float* grad_y /*[B,C,M]*/, const int* idx /*[B,M]*/, float* grad_x /*[B,C,N]*/, int B, int C, int N,
                         int M, void* stream);

/* ---------------------------------------------------------------------------------------
 * Networks and blocks.  A model is created from an int descriptor (architecture) and the
 * module's parameters as device pointers in the reference's state_dict order; the pointers
 * must stay valid (weights are re-packed into kernel layouts at creation).
 * kinds: */
enum { LION_KIND_UNET = 1, LION_KIND_PVCONV = 2, LION_KIND_SA = 3, LION_KIND_FP = 4, LION_KIND_ATTN = 5,
       LION_KIND_SHARED_MLP = 6, LION_KIND_GLOBAL_PRIOR = 7, LION_KIND_ADAGN = 8, LION_KIND_CONV3D = 9,
       LION_KIND_STYLE_ENC = 10 };
int lion_model_create(LionCtx* ctx, int kind, const int* desc, int ndesc, const float* const* params, int nparams,
                      LionModel** out);
int lion_model_destroy(LionModel* m);
/* re-pack after the parameter tensors changed in place (load_state_dict) */
int lion_model_refresh(LionModel* m);

/* PVCNN2Unet.forward (models/latent_points_ada.py:117-173) as called by PVCNN2Prior.forward
 * (models/latent_points_ada_localprior.py:72-83) and LatentPointDecPVC.forward
 * (models/latent_points_ada.py:255-272): x [B,N,D] point-major (= the reference's
 * x.view(B,N,D) before its permute), t [B] or NULL, style [B,S], clip [B,clip_dim] or NULL,
 * out [B,N,num_classes] point-major. */
int lion_unet_forward(LionModel* m, const float* x, const float* t, const float* style, const float* clip, float* out,
                      int B, int N, void* stream);
/* Hoist of the step-invariant part of PVCNN2Unet.forward out of the sampling loop: the CLIP mixing
 * (models/latent_points_ada.py:132-137) and the 61 AdaGN style Linears (models/adagn.py:59-61) are evaluated once for
 * style [B,S] (+ clip [B,clip_dim] or NULL) into a buffer owned by the model; lion_unet_forward calls with style == NULL
 * (same B) then skip them.  Values are identical to recomputing them every step. */
int lion_unet_cache_style(LionModel* m, const float* style, const float* clip, int B, void* stream);
/* PointNetPlusEncoder.forward (models/shapelatent_modules.py:35-52), the VAE's global style encoder on the non-Ada
 * PVCNN blocks of models/pvcnn2.py (PVConv :170-247, PointNetSAModule :288-351, SharedMLP :117-138; plain
 * GroupNorm(8)): x [B,N,3] point-major -> out [B, 2*zdim] = [mu_1d | sigma_1d (log sigma)].  Model kind
 * LION_KIND_STYLE_ENC, descriptor [input_dim, zdim, use_att, n_sa, {has_conv, oc, nblk, res, m, radius_bits, k,
 * n_mlp, mlp...}*], parameters in state_dict order (layers.*, mlp.weight, mlp.bias). */
int lion_style_encoder_forward(LionModel* m, const float* x, float* out, int B, int N, void* stream);
/* PVConv.forward (models/pvcnn2_ada.py:235-280): features [B,Cin,N], coords [B,3,N] -> out [B,Cout,N] */
int lion_pvconv_fwd(LionModel* m, const float* features, const float* coords, const float* style, float* out,
                    int B, int N, void* stream);
/* PointNetSAModule.forward (models/pvcnn2_ada.py:354-382): -> out_features [B,Cout,M], out_coords [B,3,M] */
int lion_sa_module_fwd(LionModel* m, const float* features, const float* coords, const float* style,
                       float* out_features, float* out_coords, int B, int N, void* stream);
/* PointNetFPModule.forward (models/pvcnn2_ada.py:393-411): points_features may be NULL -> out [B,Cout,N] */
int lion_fp_module_fwd(LionModel* m, const float* points_coords, const float* centers_coords,
                       const float* centers_features, const float* points_features, const float* style, float* out,
                       int B, int N, int M, void* stream);
/* LinearAttention.forward (models/pvcnn2_ada.py:54-71): x [B,C,N] -> out [B,C,N] */
int lion_linear_attention_fwd(LionModel* m, const float* x, float* out, int B, int N, void* stream);
/* SharedMLP.forward (models/pvcnn2_ada.py:140-164): x [B,C,R] -> out [B,Cout,R] */
int lion_shared_mlp_fwd(LionModel* m, const float* x, const float* style, float* out, int B, int R, void* stream);
/* AdaGN.forward (models/adagn.py:45-65), stand-alone: x [B,C,R] (R = product of the trailing dims) -> out [B,C,R] */
int lion_adagn_fwd(LionModel* m, const float* x, const float* style, float* out, int B, int R, void* stream);
/* SE3d.forward (models/pvcnn2_ada.py:40-41): x [B,C,V] * sigmoid(W2 relu(W1 mean_V x)); w1 [C/8,C], w2 [C,C/8] */
int lion_se3d_fwd(LionCtx* ctx, const float* w1, const float* w2, const float* x, float* out, int B, int C, int V, void* stream);
/* Swish.forward (models/pvcnn2_ada.py:74-83): x * sigmoid(x), elementwise over n floats */
int lion_swish_fwd(const float* x, float* out, size_t n, void* stream);
/* nn.Conv3d(Cin, Cout, 3, stride 1, padding 1) of a PVConv (models/pvcnn2_ada.py:211-222), stand-alone, with
 * the fused GroupNorm statistics of the following AdaGN (models/adagn.py:36).  Model kind LION_KIND_CONV3D,
 * descriptor [Cin, Cout, r], parameters [weight [Cout,Cin,3,3,3], bias [Cout]].  x [B,Cin,r,r,r] ->
 * out [B,Cout,r,r,r]; gn_sum / gn_sqsum (both or neither; [B,Cout] doubles) receive per (shape, channel) the
 * sum and the sum of squares of the outputs over the r^3 voxels.  TF32 operands, fp32 accumulation, like the
 * reference's cuDNN path under torch's default flags. */
int lion_conv3d_gn_fwd(LionModel* m, const float* x, float* out, double* gn_sum, double* gn_sqsum, int B, void* stream);
/* Prior.forward with SE cells (models/score_sde/resnet.py:195-218): x [B,D], t [B], clip [B,clip_dim] or NULL */
int lion_global_prior_forward(LionModel* m, const float* x, const float* t, const float* clip, float* out, int B,
                              void* stream);
/* the same call under the name SURVEY.md 8(b) lists (one denoising-step evaluation of the global prior) */
int lion_global_prior_step(LionModel* m, const float* x, const float* t, const float* clip, float* out, int B,
                           void* stream);

/* ---------------------------------------------------------------------------------------
 * One ancestral DDPM step (utils/diffusion_pvd.py:283-296 + :475-486), elementwise over n.
 * The step index t (the reference's loop variable, T-1 .. 0) is read from *step_ptr on the
 * device and selects row t of `tables` ([T][4] fp32), so a captured graph can be replayed:
 *   t > 0 : row = {1/sqrt(alpha_t), beta_t, sqrt(1-abar_t), exp(0.5*log beta_t)}
 *           x_out = row0 * (x - (row1*eps)/row2) + (row3*noise)*temp
 *   t = 0 : row = {1/sqrt(abar_0), sqrt(1-abar_0), 1, 0}
 *           x_out = row0 * (x - row1*eps)                       (noise unused)
 * evaluated in the reference's operation order without FMA contraction.  x_out may alias x.
 * hist (optional, [T][n]): the result is also stored at slot T-1-t (the reference keeps every
 * intermediate in output_list['pred_x']).
 * ------------------------------------------------------------------------------------- */
int lion_ddpm_update(const float* x, const float* eps, const float* noise, float* x_out, const float* tables,
                     const int* step_ptr, float temp, size_t n, float* hist, int T, void* stream);
/* set / decrement the device-side step counter and write the model's timestep (t+1, 1..T) into t_out[B] */
int lion_ddpm_set_step(int* step_ptr, float* t_out, int B, int t_index, void* stream);
int lion_ddpm_next_step(int* step_ptr, float* t_out, int B, void* stream);
/* dst[n] = block[t][n] with t = *step_ptr on the device: the noise of the current step out of a device-resident
 * [T][n] block (the `given_noise` of run_denoising_diffusion, utils/diffusion_pvd.py:283-285, uploaded ahead of the
 * loop), so that the copy is part of the captured step.  n % 4 == 0, 16-byte aligned pointers. */
int lion_ddpm_fetch_noise(float* dst, const float* block, const int* step_ptr, size_t n, void* stream);

/* ---------------------------------------------------------------------------------------
 * One DDIM step (utils/diffusion_pvd.py:389-473, update at :450 and :464-465), elementwise:
 *   x_out = x*a + (c*eps + sigma*noise[i])        row i of `tables` ([S][4] fp32) = {a, c, sigma, t_i + 1}
 * with a = sqrt(abar_next/abar_t), c = sqrt(1-abar_next-sigma^2) - sqrt(1-abar_t)*a and sigma
 * built on the host with the reference's own fp32 scalar expressions; i = *step_ptr (0..S-1,
 * ascending) is read on the device so the captured step graph can be replayed.  `noise` is the
 * whole [S][n] block of per-step draws (the reference draws them on the CPU generator, one per
 * step including the last, where sigma = 0) or NULL (treated as zeros); hist (optional, [S][n])
 * receives every intermediate (output_list).  x_out may alias x.
 * ------------------------------------------------------------------------------------- */
int lion_ddim_update(const float* x, const float* eps, const float* noise, float* x_out, const float* tables,
                     const int* step_ptr, size_t n, float* hist, void* stream);
/* set / increment the device-side step index and write the model's timestep tables[i][3] into t_out[B] */
int lion_ddim_set_step(int* step_ptr, float* t_out, const float* tables, int B, int S, int index, void* stream);
int lion_ddim_next_step(int* step_ptr, float* t_out, const float* tables, int B, int S, void* stream);

/* ---------------------------------------------------------------------------------------
 * One step of the diffusers-style DDPM scheduler used by LION.sample (models/lion.py:24-26,:55,:70;
 * the scheduler itself is the un-vendored dependency diffusers==0.11.1 -- its published
 * DDPMScheduler.step is restated, PARITY UNPINNED, see DESIGN.md section 2):
 *   x0 = (x - r0*eps)/r1;  prev = r2*x0 + r3*x;  x_out = prev + r4*noise (t > 0), prev (t = 0)
 * row t of `tables` ([T][8] fp32) = {sqrt(1-abar_t), sqrt(abar_t), c0, c1, sqrt(var_t), 0,0,0};
 * t = *step_ptr on the device (use lion_ddpm_set_step / lion_ddpm_next_step).  x_out may alias x.
 * ------------------------------------------------------------------------------------- */
int lion_scheduler_step(const float* x, const float* eps, const float* noise, float* x_out, const float* tables,
                        const int* step_ptr, size_t n, void* stream);

/* ---------------------------------------------------------------------------------------
 * Generation metrics that follow sampling (SURVEY.md 8f rank 2): Chamfer nearest neighbours.
 *
 * lion_chamfer_forward replaces chamfer_3D.forward (third_party/ChamferDistancePytorch/chamfer3D/
 * chamfer_cuda.cpp:17-19 -> chamfer3D.cu:12-143): xyz1 [B,N,3], xyz2 [B,M,3] point-major ->
 * dist1 [B,N] (squared distance to the nearest point of xyz2), idx1 [B,N] (its index; lowest index on
 * exact ties), dist2 [B,M], idx2 [B,M] the other way round.  idx1 / idx2 may be NULL.  Distances are
 * bit-identical to the reference kernel (same FMA contraction), indices exact.
 *
 * lion_chamfer_pairwise computes the whole CD matrix of utils/evaluation_metrics_fast.py:272-340
 * (_pairwise_EMD_CD_, metric 'CD'): samples [Ns,N,3], refs [Nr,M,3] -> out [Ns,Nr],
 * out[i][j] = mean_n dist(samples_i -> refs_j) + mean_m dist(refs_j -> samples_i), one CTA per pair,
 * deterministic.  N, M <= 2048.  (The means are summed in a fixed order that differs from torch's
 * reduction order: equal to the reference within fp32 rounding of a 2048-term sum.)
 * ------------------------------------------------------------------------------------- */
int lion_chamfer_forward(const float* xyz1, const float* xyz2, float* dist1, float* dist2, int* idx1, int* idx2,
                         int B, int N, int M, void* stream);
int lion_chamfer_pairwise(const float* samples, const float* refs, float* out, int n_sample, int n_ref, int N, int M,
                          void* stream);

/* Backward of lion_chamfer_forward (replaces chamfer_3D.backward, chamfer3D.cu:155-195): given the forward's
 * idx1 / idx2 and the incoming graddist1 [B,N], graddist2 [B,M], writes (does not accumulate into)
 *   gradxyz1[i] = g_i (xyz1_i - xyz2_idx1[i])  + sum over j with idx2[j] == i, ascending, of -(g'_j (xyz2_j - xyz1_i))
 *   gradxyz2[j] = sum over i with idx1[i] == j, ascending, of -(g_i (xyz1_i - xyz2_j))  + g'_j (xyz2_j - xyz1_idx2[j])
 * with g = 2 graddist1, g' = 2 graddist2, every product and sum rounded separately.  No atomics: the result is
 * bit-reproducible, and an element with at most one scattered term equals the reference's bit for bit (the
 * reference's fp32 atomicAdd order, and so its result, varies from run to run).  At most 65535 pairs per call. */
int lion_chamfer_backward(const float* xyz1, const float* xyz2, const int* idx1, const int* idx2,
                          const float* graddist1, const float* graddist2, float* gradxyz1, float* gradxyz2,
                          int B, int N, int M, void* stream);

/* Approximate earth mover's distance (third_party/PyTorchEMD/cuda/emd_kernel.cu:23-170 approxmatch +
 * :196-246 matchcost, as driven by emd_nograd.py:9-45): xyz1 [B,N,3], xyz2 [B,M,3] -> cost [B]
 * = sum_{k,l} |xyz1_k - xyz2_l|^2 * match[l][k] (NOT yet divided by N; the Python wrapper does that).
 * One fused kernel, a CTA per pair, the match matrix is never materialised.  N, M <= 2048.
 * lion_emd_pairwise: samples [Ns,N,3] x refs [Nr,M,3] -> out [Ns,Nr] (the 'EMD' matrix of
 * utils/evaluation_metrics_fast.py:272-340) without expanding the sample clouds. */
int lion_emd_approx(const float* xyz1, const float* xyz2, float* cost, int B, int N, int M, void* stream);
int lion_emd_pairwise(const float* samples, const float* refs, float* out, int n_sample, int n_ref, int N, int M,
                      void* stream);

/* Differentiable approximate EMD (emd.py:6-24 EarthMoverDistanceFunction; emd_kernel.cu:280-396 matchcostgrad1/2).
 * lion_emd_approx_saved computes the same cost as lion_emd_approx, bit for bit, and also writes the capacity ratios of
 * every annealing level t = 0..9 (level -4^(7-t), the last 0): ratios [B][10][N+M], ratioL_t in [b][t][0..N),
 * ratioR_t in [b][t][N..N+M) -- 40 (N+M) bytes per pair instead of the reference's 4 N M byte match matrix.
 * lion_emd_backward rebuilds match[l][k] = sum_t exp(level_t |xyz1_k - xyz2_l|^2) ratioL_t[k] ratioR_t[l] from them on
 * the fly (never in memory) and writes
 *   grad1[k] = grad_cost[b] * sum_l 2 match[l][k] (xyz1_k - xyz2_l),   grad2[l] = grad_cost[b] * sum_k 2 match[l][k] (xyz2_l - xyz1_k)
 * treating match as a constant, as the reference does.  Sums run in a fixed order: bit-reproducible.  N, M <= 2048. */
int lion_emd_approx_saved(const float* xyz1, const float* xyz2, float* cost, float* ratios,
                          int B, int N, int M, void* stream);
int lion_emd_backward(const float* xyz1, const float* xyz2, const float* ratios, const float* grad_cost,
                      float* grad1, float* grad2, int B, int N, int M, void* stream);

/* measurement hook (bench.py roofline leg): average device time of `iters` launches of the
 * convolution kernel alone (CUDA events on `stream`), on synthetic data: ntaps = 27 -> 3x3x3
 * over [B, cin, r^3] (r_or_rows = r), ntaps = 1 -> 1x1 over r_or_rows rows.  flops_out = the
 * algorithmic FLOPs of one launch (2*B*rows*ntaps*cin*cout, halo work not counted). */
int lion_bench_conv(LionCtx* ctx, int ntaps, int cin, int cout, int r_or_rows, int B, int iters, int warmup,
                    float* ms_out, double* flops_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif
