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
/* voxel blocks per work item of the last 128-channel 3x3x3 convolution on this context: 2, or 4 when there are enough
 * groups to give every SM work (0 when the last convolution ran on 128-row tiles) */
int lion_ctx_last_conv_group(LionCtx* ctx);
/* taps per weight stage of the last tensor-core convolution on this context: 9 when each 3x3x3 weight slab (one channel
 * chunk and x-plane) was streamed whole, 3 when it was streamed in three 3-tap parts, 1 for a 1x1 convolution */
int lion_ctx_last_conv_stage_taps(LionCtx* ctx);
/* For tests: on != 0 makes every later 3x3x3 convolution on this context stream whole weight slabs (the outputs are
 * bitwise the same either way; only the shared-memory rings differ); 0 restores the automatic choice.  Returns 0. */
int lion_ctx_set_conv_whole_slabs(LionCtx* ctx, int on);
/* For tests: on != 0 makes the sparse first convolution of every later PVConv on this context store its whole raw
 * output and the activation pass after it read every interior position, as before the activity mask existed (the
 * outputs are bitwise the same either way); 0 restores the default, which stores and reads only voxels with an occupied
 * neighbour.  Returns 0. */
int lion_ctx_set_sparse_conv1_dense(LionCtx* ctx, int on);
/* For tests: how the second convolution of every later PVConv whose first convolution ran sparse treats its 64-row
 * blocks whose every input is the inactive-voxel value or a halo zero.  0 (default): their copies and MMAs are skipped
 * and their outputs and GroupNorm sums come from the 27 border-class values; 1: every block is computed; 2: as 0, with
 * the output grid filled with NaNs first (rows that are not stored then stay NaN).  The outputs are bitwise the same in
 * all three.  Returns 0, or an error for another mode. */
int lion_ctx_set_conv2_class_mode(LionCtx* ctx, int mode);
/* The blocks that the last such convolution on this context found class-valued (*flagged) out of those it examined
 * (*total: shapes x two per 128-row tile).  Synchronises the device.  Returns 0. */
int lion_ctx_last_conv2_class_blocks(LionCtx* ctx, long long* flagged, long long* total);
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
/* Forward flags, chosen per call (a captured graph replays the mode it was captured in):
 * LION_FWD_CONV_FP16 -- the autocast(float16) route: the second 3x3x3 convolution of every PVConv takes FP16 operands
 * (activations and weights rounded to nearest even) and accumulates in fp32; its input grid is stored in FP16.
 * Everything else, and every output, stays fp32.  The model's first FP16 call packs the FP16 weights (outside stream
 * capture). */
#define LION_FWD_CONV_FP16 1
int lion_unet_forward_flags(LionModel* m, const float* x, const float* t, const float* style, const float* clip, float* out,
                            int B, int N, int flags, void* stream);
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
/* flags LION_FWD_CONV_FP16: FP16 operands (x and the weights rounded to nearest even), fp32 accumulation, for the shapes
 * the FP16 kernel serves (Cin = Cout in {32, 64, 128}); any other shape runs exactly as with flags = 0. */
int lion_conv3d_gn_fwd_flags(LionModel* m, const float* x, float* out, double* gn_sum, double* gn_sqsum, int B, int flags,
                             void* stream);
/* Stage probes for tests: the product code of one stage, with results a module's output hides.
 * lion_pvconv_conv1_probe: a PVConv model's first convolution (voxelisation, scatter, convolution): out [B,Cout,r,r,r]
 * raw output, gn_sum / gn_sqsum [B,Cout] its fused GroupNorm sums.  path: 0 = the path lion_pvconv_fwd chooses,
 * 1 = dense tensor-core convolution, 2 = sparse; a forced path that cannot serve the layer is an error.  *path_taken
 * (may be NULL) = 1 (dense) or 2 (sparse). */
int lion_pvconv_conv1_probe(LionModel* m, const float* features, const float* coords, int path, float* out,
                            double* gn_sum, double* gn_sqsum, int* path_taken, int B, int N, void* stream);
/* lion_pvconv_conv1_mask_probe: the sparse first convolution's voxel ids and activity mask.  vgrid [B,r+2,r+2,r+2]
 * int32 = compact id of the occupied voxel at each (haloed) position, -1 where empty; mask [B,ceil(r^3/32)] uint32, bit j
 * of word w set when interior voxel 32 w + j (x-major, z fastest) has an occupied voxel among its 27 neighbours.  An
 * error where the sparse path cannot serve the layer. */
int lion_pvconv_conv1_mask_probe(LionModel* m, const float* features, const float* coords, int* vgrid, unsigned* mask, int B,
                                 int N, void* stream);
/* lion_sa_mlp_probe: an SA model's MLP.  path: 0 = the path lion_sa_module_fwd chooses, 1 = unfused kernels, 2 = fused.
 * Per layer l with C_l channels, at offset B * (C_0 + ... + C_{l-1}): gn_sum / gn_sqsum [B,C_l] (doubles) and the folded
 * AdaGN scale / shift [B,C_l]; pool_mm [B][C_last/4][M][2][4] the minimum (index 0) and maximum (1) of the last layer's
 * pre-activation over each centre's 32 neighbours; centers [B,3,M]; *path_taken (may be NULL) = 1 or 2. */
int lion_sa_mlp_probe(LionModel* m, const float* features, const float* coords, const float* style, int path,
                      float* centers, double* gn_sum, double* gn_sqsum, float* scale, float* shift, float* pool_mm,
                      int* path_taken, int B, int N, void* stream);
/* lion_pvconv_probe: a whole PVConv as lion_pvconv_fwd runs it (C = cout).  raw1 / raw2 [B,C,r,r,r] the raw outputs of
 * the two 3x3x3 convolutions; act1 [B,C,r+2,r+2,r+2] the AdaGN-1 + Swish grid the second convolution reads, halo
 * included; rawp [B,C,N] the point branch's raw 1x1 output; sums [4][B][C] (doubles) the second convolution's GroupNorm
 * sum and sum of squares, then the point branch's; affine [6][B][C] the folded scale and shift of AdaGN-1, of the point
 * branch's AdaGN and of AdaGN-2 with the SE gate multiplied in; fused [B,C,N] devoxelised + point branch (the attention's
 * input; without attention the module output); out [B,C,N] the module output; *conv2_kernel (may be NULL) = the second
 * convolution's kernel: 0 SIMT, 1 tensor-core row tiles, 2 or 4 interior-block groups of that many blocks.  The grids of
 * raw1, act1 and raw2 are NaN-filled before their producers run. */
int lion_pvconv_probe(LionModel* m, const float* features, const float* coords, const float* style, float* raw1, float* act1,
                      float* raw2, float* rawp, double* sums, float* affine, float* fused, float* out, int* conv2_kernel,
                      int B, int N, void* stream);
/* the same with forward flags; under LION_FWD_CONV_FP16 act1 is the FP16 grid, widened to fp32 in the same layout */
int lion_pvconv_probe_flags(LionModel* m, const float* features, const float* coords, const float* style, float* raw1,
                            float* act1, float* raw2, float* rawp, double* sums, float* affine, float* fused, float* out,
                            int* conv2_kernel, int B, int N, int flags, void* stream);
/* lion_attention_probe: a linear attention as lion_linear_attention_fwd runs it.  qkv [B, 3*heads*32, N] (q, k, v of
 * every head), o [B, heads*32, N] the output before the projection, out [B,C,N]. */
int lion_attention_probe(LionModel* m, const float* x, float* qkv, float* o, float* out, int B, int N, void* stream);
/* lion_fp_probe: an FP module as lion_fp_module_fwd runs it.  nn_idx / nn_wgt [B,3,N] the 3 nearest centres of every
 * point and their weights; cat [B, cc + roundup(cp,4), N] the MLP input [interpolated | skip], padding channels
 * included (NaN-filled before its producers run).  Per MLP layer l with C_l channels: raw / act [B,C_l,N] at offset
 * B*N*(C_0 + ... + C_{l-1}) the raw 1x1 output and the activated output (the last layer's is the module output);
 * gn_sum / gn_sqsum [B,C_l] (doubles) and the folded AdaGN scale / shift [B,C_l] at offset B*(C_0 + ... + C_{l-1}). */
int lion_fp_probe(LionModel* m, const float* points_coords, const float* centers_coords, const float* centers_features,
                  const float* points_features, const float* style, int* nn_idx, float* nn_wgt, float* cat, float* raw,
                  float* act, double* gn_sum, double* gn_sqsum, float* scale, float* shift, int B, int N, int M, void* stream);
/* lion_unet_probe: a U-Net forward as lion_unet_forward runs it (style == NULL: the lion_unet_cache_style vectors),
 * with its glue copied into caller buffers as it is computed.  taps holds 4 + 6*n_fp + 5 device pointers, each may be
 * NULL; PF = packed [B][ceil(C/4)][R][4]:
 *   sinu, h, temb [B,E] (the sinusoid, after Linear + LeakyReLU, the time embedding); aff [B, style_total];
 *   per FP stage: cf PF [C_in + E, M] (centre features after the time-embedding concat), nn_idx (int) and nn_wgt
 *   [B][N][3], skip PF [roundup(cp,4), N], cat PF [cc + roundup(cp,4), N] (NaN-filled before its producers run),
 *   out PF [C, N] (the stage's output after its PVConvs);
 *   head: feat PF [C, N], cls_raw PF [128, N], cls_sums [2][B][128] (doubles), cls_aff [2][B][128] (scale, shift),
 *   hc PF [128, N].
 * style_table [n_style][2] (host, may be NULL): (offset, width) of every AdaGN style Linear's output in aff, in build
 * order; n_style must be the network's number of them. */
int lion_unet_probe(LionModel* m, const float* x, const float* t, const float* style, const float* clip, float* out,
                    void* const* taps, int ntaps, int* style_table, int n_style, int B, int N, void* stream);
/* Prior.forward with SE cells (models/score_sde/resnet.py:195-218): x [B,D], t [B], clip [B,clip_dim] or NULL */
int lion_global_prior_forward(LionModel* m, const float* x, const float* t, const float* clip, float* out, int B,
                              void* stream);
/* lion_global_prior_probe: a global-prior forward as lion_global_prior_forward runs it, with every Linear's output
 * copied into caller buffers.  taps holds 5 + 4*ncell device pointers [B, width] fp32, each may be NULL:
 *   pe [emb] (the positional embedding), t0 [4*emb] (first temb Linear), temb [nf] (second temb Linear),
 *   cmap [nf] (clip_feat_mapping; CLIP networks only, NULL otherwise), h0 [nf] (input layer);
 *   per cell: a [nf] (conv1 + ReLU), bb [nf] (conv2 + ReLU), s [nf/8] (SE fc0 + ReLU), h [nf] (sigmoid(fc2) * bb + h). */
int lion_global_prior_probe(LionModel* m, const float* x, const float* t, const float* clip, float* out,
                            void* const* taps, int ntaps, int B, void* stream);
/* the same call under the name SURVEY.md 8(b) lists (one denoising-step evaluation of the global prior) */
int lion_global_prior_step(LionModel* m, const float* x, const float* t, const float* clip, float* out, int B,
                           void* stream);
/* Training the global prior.  lion_global_prior_saved_floats: the size in floats of the buffer the training forward
 * fills for the backward (0 for a bad model or B).  Its layout, [B][width] fp32 tensors back to back: x [D], pe [emb],
 * t0 [4*emb], temb [nf], cmap [nf] (CLIP networks only), h0 [nf], then per cell a [nf] (conv1 + ReLU, times the dropout
 * mask), bb [nf], s [nf/8], gate [nf] (sigmoid(fc2)), h [nf] (the cell output). */
size_t lion_global_prior_saved_floats(LionModel* m, int B);
/* lion_global_prior_forward with the dropout of ResBlockSEDrop applied and the saved buffer filled.  drop_mask
 * [ncell][B][nf] fp32: the scaled mask (0 or 1/(1-p)) multiplied into each cell's conv1 + ReLU output, or NULL for no
 * dropout, in which case out has the bits lion_global_prior_forward gives. */
int lion_global_prior_forward_train(LionModel* m, const float* x, const float* t, const float* clip,
                                    const float* drop_mask, float* saved, float* out, int B, void* stream);
/* The backward of the training forward that filled `saved` (same model, clip, drop_mask and B; the parameters unchanged
 * since): from gout [B][D] = dL/d out, writes gx [B][D] = dL/d x and gparams[i] = dL/d params[i] for every parameter
 * in the order lion_model_create took them (nparams of them; each is overwritten, not accumulated).  No gradient
 * reaches t or clip.  Deterministic: no atomics, every sum in a fixed order. */
int lion_global_prior_backward(LionModel* m, const float* saved, const float* clip, const float* drop_mask,
                               const float* gout, float* gx, float* const* gparams, int nparams, int B, void* stream);
/* lion_global_prior_backward with the gradients between the Linears copied into caller buffers.  taps holds
 * 4 + 5*ncell device pointers [B, width] fp32, each may be NULL: gtemb [nf] (dL/d temb, summed over the cells),
 * gt0 [4*emb] (dL/d t0), gcmap [nf] (dL/d clip_feat_mapping output; CLIP networks only), gh0 [nf] (dL/d h0);
 * per cell: gh [nf] (dL/d cell output), gz [nf] (dL/d fc2 before the sigmoid), gs [nf/8] (dL/d fc0 before its ReLU),
 * gbb [nf] (dL/d conv2 before its ReLU), gz1 [nf] (dL/d conv1 before its ReLU).  taps = NULL: no copies. */
int lion_global_prior_backward_probe(LionModel* m, const float* saved, const float* clip, const float* drop_mask,
                                     const float* gout, float* gx, float* const* gparams, int nparams,
                                     void* const* taps, int ntaps, int B, void* stream);

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
 * Device-resident adaptive RK45 for the probability-flow ODE of the VPSDE (utils/diffusion_continuous.py:90-176
 * compute_ode_nll and :178-249 sample_model_ode, both through scipy's RK45 as solve_ivp(..., t_eval=...) drives it:
 * scipy/integrate/_ivp/rk.py RungeKutta._step_impl, rk_step, the RK45 tableaux and RkDenseOutput; common.py
 * select_initial_step and norm).  The integration variable s runs from t0 to t_bound (either direction); the model
 * sees t = s, or t = -s with the right-hand side negated when `negate` is set (torchdiffeq's treatment of a
 * decreasing time span).  All integrator state is on the device:
 *   st  one LionOdeState (below), written by these calls only;
 *   y, y_new [n] float64; K [7][n] float64 (the stages, K[6] = f at the step's end); partials [2][256] float64;
 *   x [n] fp32 the model input of the current evaluation, t_model [B] fp32 its time (every row the same).
 * One evaluation = lion_ode_stage (x, t_model) -> the caller's model forward (eps [n] fp32) -> lion_ode_rhs.
 * Driver: lion_ode_init; evaluation of stage 0; lion_ode_norms/control(LION_ODE_INIT_H0); evaluation of stage
 * LION_ODE_STAGE_PROBE; lion_ode_norms/control(LION_ODE_INIT_H1); then per step attempt: lion_ode_control(BEGIN),
 * evaluations of stages 1..6, lion_ode_norms/control(END), lion_ode_commit -- until st->status != RUNNING; then
 * lion_ode_dense_end.  Every call after lion_ode_init reads the status on the device and does nothing once the
 * integration stopped, so a captured step attempt can be replayed without host-side parameters.
 * Sums run in a fixed order without FMA contraction and the norms reduce fixed-size partials in a fixed order:
 * results are bit-reproducible.  Requires n > 0 and B > 0.
 * ------------------------------------------------------------------------------------- */
enum { LION_ODE_RUNNING = 0, LION_ODE_DONE = 1, LION_ODE_TOO_SMALL = 2 };
enum { LION_ODE_INIT_H0 = 0, LION_ODE_INIT_H1 = 1, LION_ODE_END = 2, LION_ODE_BEGIN = 3 };
#define LION_ODE_STAGE_PROBE 7     /* the second evaluation of select_initial_step: y0 + h0 * direction * f0 */
typedef struct LionOdeState {
  double t, t_bound, direction, rtol, atol;
  double h_abs;                    /* scipy's self.h_abs, the loop-local h_abs during a step attempt */
  double h, t_new, min_step;       /* the current attempt */
  double h0, d1, err_norm;         /* select_initial_step; the last attempt's error norm */
  int status, nfe, n_accepted, n_rejected;
  int step_rejected, new_step, accepted, negate;
} LionOdeState;
size_t lion_ode_state_bytes(void);
/* st <- start at t0 (y = y0 widened, rtol / atol as given, nfe = 0; status DONE when t0 == t_bound) */
int lion_ode_init(LionOdeState* st, const float* y0, double* y, size_t n, double t0, double t_bound, double rtol,
                  double atol, int negate, void* stream);
/* x <- the model input of `stage` rounded to fp32, t_model[0..B) <- float32(+-(t + c_stage h)); stage 6 also writes
 * y_new.  stage 0: y at t; 1..5: y + (sum_j a_sj K_j) h; 6: y + h sum_j b_j K_j at t + h; LION_ODE_STAGE_PROBE. */
int lion_ode_stage(LionOdeState* st, const double* y, double* y_new, const double* K, size_t n, int stage, float* x,
                   float* t_model, int B, void* stream);
/* K[stage] <- (+-) (f(t) x + ((0.5 g2(t)) eps) / sqrt(var(t))) in fp32, widened; t = t_model[0]; the probe writes
 * K[1].  beta_start, beta_end, sigma2_0: the VPSDE's (utils/diffusion_continuous.py:571-621); nfe += 1. */
int lion_ode_rhs(LionOdeState* st, const float* x, const float* eps, double* K, size_t n, int stage, double beta_start,
                 double beta_end, double sigma2_0, const float* t_model, void* stream);
/* fixed-order partial sums of squares for the norm that lion_ode_control(`what`) consumes */
int lion_ode_norms(const LionOdeState* st, const double* y, const double* y_new, const double* K, size_t n, int what,
                   double* partials, void* stream);
/* the step-size controller, one thread: what = INIT_H0 / INIT_H1 (select_initial_step), BEGIN (min_step, clamp to
 * t_bound, too-small check), END (accept / reject, SAFETY 0.9, factors 0.2 .. 10, exponent -1/5) */
int lion_ode_control(LionOdeState* st, const double* partials, size_t n, int what, void* stream);
/* after END: on an accepted step that did not finish, y <- y_new and K[0] <- K[6] (FSAL) */
int lion_ode_commit(const LionOdeState* st, double* y, const double* y_new, double* K, size_t n, void* stream);
/* out [n] fp32 <- the last step's dense-output polynomial at its end point (RkDenseOutput at x = 1), which is what
 * solve_ivp returns for t_eval = t_bound; y holds the step's start (lion_ode_commit leaves it on the last step) */
int lion_ode_dense_end(const LionOdeState* st, const double* y, const double* K, size_t n, float* out, void* stream);

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

/* Occupancy grid of the JSD score (utils/evaluation_metrics_fast.py:604-647, entropy_of_occupancy_grid).
 * clouds [S,N,3] point-major, cells [K,3] (the cell centres, any order) -> for every cell c
 *   point_counts[c] = number of points, over all clouds, whose nearest cell is c   (the reference's grid_counters)
 *   cloud_counts[c] = number of clouds with at least one point whose nearest cell is c   (grid_bernoulli_rvars)
 * Both outputs are overwritten (zeroed on `stream` first).  The nearest cell minimises the exact float64 squared
 * distance (dx*dx + dy*dy) + dz*dz of the float32 inputs, every operation rounded separately (no contraction); on an
 * exact tie the lowest cell index wins.  Integer atomics only: the counts are deterministic.  Brute force over the
 * cells (no pruning), so points anywhere -- also far outside the cell table -- get their exact nearest cell.
 * Requires S, N, K > 0, S * N <= INT_MAX and K <= 1,572,864 cells (the per-cloud bitmap lives in shared memory). */
int lion_occupancy_grid(const float* clouds, const float* cells, int S, int N, int K, int* point_counts,
                        int* cloud_counts, void* stream);

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
