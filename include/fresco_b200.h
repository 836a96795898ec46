/* fresco_b200 -- C ABI of the H100-native (sm_90a) FRESCO hot path (libfresco_b200.so).
 *
 * The reference (williamyang1991/FRESCO) has no FFI on this path: its boundary is a Python
 * monkey-patch surface over diffusers (SURVEY.md 8b).  The host side of this repo
 * (fresco_b200/*.py) mirrors that surface and binds these entry points with ctypes; each
 * entry point cites the reference lines whose work it replaces (paths relative to the
 * reference root).
 *
 * Conventions
 *  - every pointer is a DEVICE pointer owned by the caller (torch allocator); nothing is
 *    allocated, freed or synchronised inside; `stream` is a cudaStream_t.
 *  - return value: 0 = ok, negative = FRESCO_ERR_*; fresco_last_error() gives the text
 *    (thread-local).  Functions never throw and never touch the host-side oracle.
 *  - "half" tensors are IEEE fp16; layouts are stated per function, innermost dimension last.
 */
#ifndef FRESCO_B200_H_
#define FRESCO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FRESCO_ABI_VERSION 1

#define FRESCO_OK 0
#define FRESCO_ERR_ARG (-1)          /* null pointer / inconsistent shape            */
#define FRESCO_ERR_UNSUPPORTED (-2)  /* shape outside what the kernels are built for */
#define FRESCO_ERR_CUDA (-3)         /* CUDA runtime / launch error                  */
#define FRESCO_ERR_TENSORMAP (-4)    /* cuTensorMapEncodeTiled failed                */

int fresco_abi_version(void);
const char* fresco_last_error(void);
/* number of kernels launched by this library in this process (for bench.py's gpu_launches) */
long long fresco_launch_count(void);
/* name of the last kernel this library launched on the calling thread, with its template arguments where the launch
 * site picks an instantiation (e.g. "warp_loss_group_kernel<18,1>"); "" before the first launch (thread-local string) */
const char* fresco_last_kernel(void);
/* tuning option by the name of its environment variable (FRESCO_ATTN_WIDE, FRESCO_ATTN_POLY, FRESCO_ATTN_ROWSUM,
 * FRESCO_TEMPORAL_V, FRESCO_GRAM_V); the environment is read once, this overrides it;
 * value < 0 restores the built-in default. */
int fresco_set_option(const char* name, int value);
/* name of the kernel fresco_attn_fwd launches for a head dim under the current options (thread-local string) */
const char* fresco_attn_variant(int head_dim);

/* ---- A2: cross-frame K/V selection --------------------------------------------------------
 * replaces src/diffusion_hacked.py:234-247 (`key[:, attn_mask]` + `repeat(...)`).
 * k, v      half [chunks, rows_per_chunk, channels]   (rows_per_chunk = frames * tokens)
 * idx       int32 [n_sel] row indices into one chunk (row-major over (frame, token))
 * k_out/v_out half [chunks, n_sel, channels]; shared by every query frame (no N x broadcast) */
int fresco_kv_compact(const void* k, const void* v, const int32_t* idx, void* k_out, void* v_out, int chunks,
                      int rows_per_chunk, int n_sel, int channels, void* stream);
/* same selection, K and V rows side by side: kv_out half [chunks, out_rows, 2*channels], rows [0, n_sel) written
 * (the send buffer of the frame-sharded K/V exchange, SURVEY 8e exchange 1; out_rows >= n_sel is the padded count) */
int fresco_kv_compact_packed(const void* k, const void* v, const int32_t* idx, void* kv_out, int chunks,
                             int rows_per_chunk, int n_sel, int out_rows, int channels, void* stream);
/* row gather / scatter by index (16-byte granularity), the data movement around the collectives of the frame-sharded
 * path: gather  dst[r, dst_offset : dst_offset+row_bytes] = src[idx[r], :]  (dst rows dst_stride_bytes apart);
 *       scatter dst[idx[r], :] = src[r, :]. */
int fresco_rows_gather(const void* src, const int32_t* idx, void* dst, long long n_rows, int row_bytes,
                       int dst_stride_bytes, int dst_offset_bytes, void* stream);
int fresco_rows_scatter(const void* src, const int32_t* idx, void* dst, long long n_rows, int row_bytes, void* stream);

/* ---- A3 / A4: dense attention forward (wgmma + TMA) ---------------------------------------
 * replaces F.scaled_dot_product_attention at src/diffusion_hacked.py:281-285 (spatial-guided:
 * q = to_q(ref), k = to_k(ref), v = current query, softmax_scale = 0.2/sqrt(d), diag_bias =
 * intraattn_bias) and :303-305 (cross-frame: shared compacted K/V, q_per_kv = frames).
 * q, out  half [batch_q, q_len, heads*head_dim];  k, v half [batch_q/q_per_kv, kv_len, heads*head_dim]
 * out = softmax(q k^T * softmax_scale + diag_bias * I) v, per head. head_dim in {40,64,80,128}. */
int fresco_attn_fwd(const void* q, const void* k, const void* v, void* out, int batch_q, int q_len, int kv_len,
                    int heads, int head_dim, int q_per_kv, float softmax_scale, float diag_bias, void* stream);
/* same with explicit K/V strides in elements (rows kv_row_stride apart, batches kv_batch_stride apart): K and V may
 * live side by side in one [batch, kv_len, 2*heads*head_dim] buffer (v = k + heads*head_dim), as the frame-sharded
 * exchange delivers them. */
int fresco_attn_fwd_kv_strided(const void* q, const void* k, const void* v, void* out, int batch_q, int q_len,
                               int kv_len, int heads, int head_dim, int q_per_kv, long long kv_row_stride,
                               long long kv_batch_stride, float softmax_scale, float diag_bias, void* stream);

/* ---- A5: temporal-guided (FLATTEN) attention, fused gather -> N x N softmax -> scatter -----
 * replaces src/diffusion_hacked.py:320-367.
 * q_raw, k_raw, v_src, out  half [chunks*frames, tokens, heads*head_dim]  (v_src = output of A4)
 * fwd_map int64 [frames, tokens] (trajectory p sits at token fwd_map[f][p] of frame f; a permutation)
 * traj_mask uint8 [tokens, frames, frames] (traj_mask[p][f][g] = 1: frame f of trajectory p attends to frame g).
 *   Every row traj_mask[p][f][.] must keep at least one key; the reference's masks always keep the diagonal, and
 *   the kernels rely on a finite row maximum (a fully masked row is undefined input).
 * out[b,f,fwd_map[f][p]] = sum_g softmax_g(q[f,pos]·k[g,pos] * scale, masked) v[g,pos]
 * frames > 16 run only with dense inputs (in_row_stride == heads*head_dim): the strided entry point returns
 * FRESCO_ERR_UNSUPPORTED there.                                                                 */
int fresco_temporal_attn_fwd(const void* q_raw, const void* k_raw, const void* v_src, void* out,
                             const int64_t* fwd_map, const uint8_t* traj_mask, int chunks, int frames, int tokens,
                             int heads, int head_dim, float scale, void* stream);
/* same with the q/k/v token rows in_row_stride elements apart (>= heads*head_dim; e.g. q | k | v interleaved in one
 * 3C-wide row, as the trajectory-sharded exchange delivers them); out stays dense. */
int fresco_temporal_attn_fwd_strided(const void* q_raw, const void* k_raw, const void* v_src, void* out,
                                     const int64_t* fwd_map, const uint8_t* traj_mask, int chunks, int frames,
                                     int tokens, int heads, int head_dim, int in_row_stride, float scale, void* stream);

/* ---- W3: bilinear flow warp (zero padding per tap, pixel coordinates) ----------------------
 * replaces gmflow/geometry.py:65-72 (flow_warp) + :41-62 (grid_sample, align_corners=True).
 * src, dst float [batch, channels, h, w]; flow float [flow_batch, 2, h, w] (x, y); sample b uses
 * flow (b % flow_batch).                                                                        */
int fresco_flow_warp(const float* src, const float* flow, float* dst, int batch, int channels, int h, int w,
                     int flow_batch, void* stream);

/* ---- W1: warp_tensor frame chain ----------------------------------------------------------
 * replaces the loop at src/flow_utils.py:41-51.  One CTA per (chunk, channel) keeps the running
 * frame plane in shared memory; the N-1 sequential blends need no grid-wide sync.
 * sample/out  [chunks*frames, channels, h, w], half (is_half=1) or float; may alias.
 * bwd_flow    float [frames, 2, h, w] (resized);  fwd_flow_last float [2, h, w] (frame N-1)
 * blend       float [frames, h, w]: entries 0..N-2 = (1-bwd_occ[i])*sal[i+1]*warp_sal[i];
 *             entry N-1 = closing mask (1-fwd_occ[N-1])*sal[N-1]*warp_sal_last                   */
int fresco_warp_fuse_chain(const void* sample, void* out, int is_half, const float* bwd_flow,
                           const float* fwd_flow_last, const float* blend, int chunks, int frames, int channels,
                           int h, int w, void* stream);

/* ---- O2: temporal-consistency loss, forward + backward -------------------------------------
 * replaces src/diffusion_hacked.py:461-466 and its autograd backward.
 * cs, grad float [chunks, frames, channels, h, w]; fwd_flow/bwd_flow float [frames,2,h,w];
 * fwd_keep/bwd_keep float [frames,h,w] (= 1 - occlusion), each value 0 or 1 (what every caller passes: max_pool of
 * binary occlusions); the quad and group kernels store sgn(r) * keep in fp16, exact only for such masks.  The adjoint
 * of the bilinear warp is applied as a gather through a per-frame ELL matrix built once per batch from
 * fresco_warp_taps + a sort by destination:
 * *_ell uint32 [frames, h*w, 8], entry = (round(weight*65535) << 16) | source pixel (0 = empty slot).  A row's used
 * slots come first and a slot whose weight field is 0 ends the row (the quad kernel stops a warp's walk there), so a
 * tap whose weight rounds to a 0 field (< 2^-17) is left out of the ELL and the overflow list alike;
 * overflow int32 [2 (bwd,fwd), frames, n_overflow, 3] = (destination | -1, source, float bits of weight) for
 * destinations with more than 8 taps.  h*w <= 65535.  grad is overwritten (accumulate=0) or added to;
 * *loss_acc (device float, may be null) gets the loss value added.
 * fresco_warp_taps: the 4 bilinear taps of every source pixel: dest int32 [frames, h*w, 4] (-1 = no tap),
 * weight float [frames, h*w, 4].                                                                 */
int fresco_warp_taps(const float* flow, int32_t* dest, float* weight, int frames, int h, int w, void* stream);
int fresco_warp_loss_fwd_bwd(const float* cs, const float* fwd_flow, const float* bwd_flow, const float* fwd_keep,
                             const float* bwd_keep, const void* bwd_ell, const void* fwd_ell, const int32_t* overflow,
                             int n_overflow, float* grad, float* loss_acc, int accumulate, int chunks, int frames,
                             int channels, int h, int w, void* stream);
/* Open-chain form for a frame-sharded batch (SURVEY 8e, exchange 3; the reference's ring is
 * src/diffusion_hacked.py:444,461-466): this rank holds `frames` consecutive frames of a ring of `total_frames`; pair
 * f = (frame f, frame f+1) uses flow / keep / ELL entry f of the arrays passed (the caller passes its slice); the "next"
 * frame of the last pair is halo_cs float [chunks, channels, h, w] (the following rank's first frame) and what that
 * frame receives from the pair is written to halo_grad (same shape, overwritten), to be added to the following rank's
 * grad of its first frame.  The loss mean runs over total_frames.  halo_cs = halo_grad = NULL and total_frames = frames
 * is fresco_warp_loss_fwd_bwd.  frames >= 1.  Results are bit-identical to the closed ring (every gradient element is
 * the same sum of the same two rounded products).                                                              */
int fresco_warp_loss_fwd_bwd_halo(const float* cs, const float* fwd_flow, const float* bwd_flow, const float* fwd_keep,
                                  const float* bwd_keep, const void* bwd_ell, const void* fwd_ell,
                                  const int32_t* overflow, int n_overflow, float* grad, float* loss_acc, int accumulate,
                                  int chunks, int frames, int channels, int h, int w, const float* halo_cs,
                                  float* halo_grad, int total_frames, void* stream);

/* ---- O3: spatial-consistency (normalised Gram, L1) loss, forward + backward -----------------
 * replaces src/diffusion_hacked.py:469-476 and its backward.
 * step 1  fresco_gram_normalize: cs float [batch, channels, tokens] -> xhat half [batch, tokens, channels]
 *         (row-normalised, token-major) and norms float [batch, tokens].
 * step 2  fresco_gram_sign (wgmma): G = xhat xhat^T per batch; T = sign(G - A) + sign(G - A^T)
 *         written as half [batch, tokens, tokens]; loss += weight/(batch*tokens^2) * sum|G - A|.
 *         target float [batch, tokens, tokens] is the reference's correlation_matrix entry.
 * step 3  fresco_gram_grad (wgmma): ghat = T xhat * weight/(batch*tokens^2), projected through the
 *         normalisation Jacobian and added to grad float [batch, channels, tokens].
 * Every step takes any tokens >= 1 (channels a multiple of 8); T stays a contiguous half [batch, tokens, tokens].  */
int fresco_gram_normalize(const float* cs, void* xhat, float* norms, int batch, int channels, int tokens,
                          void* stream);
int fresco_gram_sign(const void* xhat, const float* target, void* tsign, float* loss_acc, int batch, int tokens,
                     int channels, float weight, void* stream);
int fresco_gram_grad(const void* tsign, const void* xhat, const float* norms, float* grad, int batch, int tokens,
                     int channels, float weight, void* workspace, size_t workspace_bytes, void* stream);
size_t fresco_gram_grad_workspace_bytes(int batch, int tokens, int channels);
/* step 2 with the Gram target RECOMPUTED in the kernel from the row-normalised reference features
 * yhat half [batch, tokens, channels] (what src/diffusion_hacked.py:889-893 feeds its bmm): D = xhat xhat^T - yhat yhat^T in
 * one K = 2*channels contraction, tsign = 2 sign(D), loss += weight/(batch*tokens^2) * sum |D|.  The fp32
 * [batch, tokens, tokens] target (1.07 GB per Adam iteration at layer 3) is never read or stored.
 * fresco_gram_tx: the tensor-core product of step 3 alone, ghat float [batch, tokens, channels] = alpha * tsign xhat. */
int fresco_gram_sign_ref(const void* xhat, const void* yhat, void* tsign, float* loss_acc, int batch, int tokens,
                         int channels, float weight, void* stream);
int fresco_gram_tx(const void* tsign, const void* xhat, float* ghat, int batch, int tokens, int channels, float alpha,
                   void* stream);
/* the three steps above with the loss scale given directly: `scale` multiplies every |D| of the loss and the T xhat
 * product of the gradient, and is rounded to fp32 once.  The `weight` forms pass (double)weight/(batch*tokens^2).  A
 * frame-sharded caller passes the scale of the whole batch, intra_weight/(chunks*total_frames*tokens^2), computed in
 * double: rounding a rank's share of the weight to fp32 first would give a scale that differs from the unsharded one. */
int fresco_gram_sign_scaled(const void* xhat, const float* target, void* tsign, float* loss_acc, int batch, int tokens,
                            int channels, double scale, void* stream);
int fresco_gram_sign_ref_scaled(const void* xhat, const void* yhat, void* tsign, float* loss_acc, int batch, int tokens,
                                int channels, double scale, void* stream);
int fresco_gram_grad_scaled(const void* tsign, const void* xhat, const float* norms, float* grad, int batch, int tokens,
                            int channels, double scale, void* workspace, size_t workspace_bytes, void* stream);

/* ---- O4 / O5: Adam update and AdaIN ---------------------------------------------------------
 * fresco_adam_step replaces torch.optim.Adam.step at src/diffusion_hacked.py:433,485
 * (betas 0.9/0.999, eps 1e-8, bias correction; `step` is 1-based).
 * fresco_adain replaces src/utils.py:70-78 incl. the eps quirk (style eps = 1, content eps = 1e-5,
 * unbiased variance).  content float [planes, hw]; style/out half or float [planes, hw].          */
int fresco_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n, int step,
                     double lr, double beta1, double beta2, double eps, void* stream);
int fresco_adain(const float* content, const void* style, void* out, int is_half, int planes, int hw, void* stream);

/* ---- W2: binary dilation of occlusion masks (background smoothing at image resolution) -------
 * replaces Dilate, src/utils.py:81-93 (replicate padding + conv2d with ones(k x k) + clamp to [0,1]).
 * in, out float [planes, h, w]; kernel odd.                                                     */
int fresco_dilate(const float* in, float* out, int planes, int h, int w, int kernel, void* stream);

/* ---- S1: classifier-free guidance + DDPM step arithmetic -----------------------------------
 * replaces the elementwise parts of src/pipe_FRESCO.py: guidance (:212-215) fused with the predicted x0 (:22-35), and
 * the posterior mean + noise (:49-73); two entry points because the background-smoothing VAE round trip may replace
 * x0 between them (:44-47).  Tensors half (is_half=1) or float, n elements; noise_text may be null (no guidance).
 * x0 = (sample - sqrt(1-alpha_prod_t) * (u + g (t - u))) / sqrt(alpha_prod_t)
 * prev = c_x0 * x0 + c_xt * sample + sigma * noise[repeat_noise ? i % per_frame : i]                 */
int fresco_cfg_pred_x0(const void* noise_uncond, const void* noise_text, const void* sample, void* x0, int is_half,
                       long long n, float guidance_scale, float alpha_prod_t, void* stream);
int fresco_ddpm_prev(const void* x0, const void* sample, const void* noise, void* prev, int is_half, long long n,
                     long long per_frame, int repeat_noise, float c_x0, float c_xt, float sigma, void* stream);

/* ---- G1: GMFlow global correlation + softmax + expected coordinates -------------------------
 * replaces gmflow/matching.py:7-36.  feature0/1 float [batch, channels, h, w];
 * flow float [batch*(bidir?2:1), 2, h, w], order [fwd(batch), bwd(batch)].  The L x L volume is
 * never materialised.  workspace: fresco_gmflow_corr_workspace_bytes().                           */
int gmflow_global_corr_softmax(const float* feature0, const float* feature1, float* flow, int batch, int channels,
                               int h, int w, int bidir, void* workspace, size_t workspace_bytes, void* stream);
size_t fresco_gmflow_corr_workspace_bytes(int batch, int channels, int h, int w);
/* GMFlow's flow-propagation attention, replaces FeatureFlowAttention.forward, gmflow/transformer.py:353-374 (the global
 * path): out = softmax(q k^T * softmax_scale) values.  q, k half [batch, tokens, channels] (token-major projections);
 * values float [batch, tokens, 2] (the flow field, channel-last); out float [batch, 2, tokens].  The [batch, tokens, tokens]
 * probability volume (1 GB at 512 x 512) is never materialised. */
int gmflow_flow_attention(const void* q, const void* k, const float* values, float* out, int batch, int tokens,
                          int channels, float softmax_scale, void* stream);

/* ---- M1: pixel correspondence between two frames (integer, bit-exact) -----------------------
 * replaces get_single_mapping_ind, src/flow_utils.py:57-102 (incl. the sequential loop :84-101).
 * bwd_flow float [2,H,W] (x,y), bwd_occ float [H,W], imgs float [2,3,H,W] = [frame1, frame2];
 * scale = integer downsample factor (1 or even).  Outputs over L = (H/scale)*(W/scale) pixels:
 * mapping int64 [L], unlinked uint8 [L].  workspace: fresco_mapping_workspace_bytes(L).          */
int fresco_mapping_single(const float* bwd_flow, const float* bwd_occ, const float* imgs, int height, int width,
                          int scale, int64_t* mapping, uint8_t* unlinked, void* workspace, size_t workspace_bytes,
                          void* stream);
size_t fresco_mapping_workspace_bytes(int tokens);

/* ---- B1: propagation-stage frame blending ---------------------------------------------------
 * replaces video_blend.py:172-255 with blender/histogram_blend.py:19-50 and blender/poisson_fusion.py:54-93.
 * Images are uint8 [frames, h, w, 3] (BGR or cv2 8-bit Lab), masks uint8 [frames, h, w] in {0, 1}.
 * lut_gather: out[p] = lut[(in[p][0] << 16 | in[p][1] << 8 | in[p][2])], lut uint8 [2^24, 3] (cv2's conversion of
 *   every triple, built by the caller).
 * mask_chain: frame k = 0 .. interval-2 of one sequence: error mask of dist1/dist2 float [interval-1, h, w] with
 *   weight1 = k / (interval-1), OR'd with frame k-1's mask warped (nearest, torch CPU grid_sample bit for bit) by
 *   flows float [interval-1, 2, h, w] (flow 0 unused; may be null when interval == 2).
 * histogram: blend() in Lab; lab_min_error may be null, then the min-error image is a where mask is 0, b where 1;
 *   weights double [frames, 2] are blend()'s weight1, weight2 per frame.
 * poisson: the exact least-squares solution of poisson_fusion's system per Lab channel (Chebyshev iteration in fp64,
 *   fresco_blend_cheby_iterations(h, w, weight) steps), clip [0, 255], truncated; `solution` double
 *   [frames, 3, h, w] (may be null) receives the unclipped solution.
 * workspace: fresco_blend_workspace_bytes(frames, h, w) (histogram and poisson).                              */
int fresco_blend_lut_gather(const uint8_t* in, const uint8_t* lut, uint8_t* out, long long pixels, void* stream);
int fresco_blend_mask_chain(const float* dist1, const float* dist2, const float* flows, uint8_t* masks, int interval,
                            int h, int w, void* stream);
int fresco_blend_histogram(const uint8_t* lab_a, const uint8_t* lab_b, const uint8_t* lab_min_error,
                           const uint8_t* masks, const double* weights, uint8_t* lab_out, int frames, int h, int w,
                           void* workspace, size_t workspace_bytes, void* stream);
int fresco_blend_poisson(const uint8_t* lab_target, const uint8_t* lab_a, const uint8_t* lab_b, const uint8_t* masks,
                         double weight0, double weight1, double weight2, uint8_t* lab_out, double* solution,
                         int frames, int h, int w, void* workspace, size_t workspace_bytes, void* stream);
int fresco_blend_cheby_iterations(int h, int w, double weight);
size_t fresco_blend_workspace_bytes(int frames, int h, int w);

#ifdef __cplusplus
}
#endif
#endif /* FRESCO_B200_H_ */
