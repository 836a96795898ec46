"""Drop-in for the reference's ``src/pipe_FRESCO.py``: one DDPM step with background smoothing (``step``, :14-77) and
the per-batch denoising loop (``inference``, :81-234), SURVEY 8a row S1 / 8(f)-3, 8(f)-4.

Same names, arguments and behaviour.  What changes underneath:
* the elementwise arithmetic of a step -- classifier-free guidance, predicted x0, posterior mean + noise -- runs in two
  fused kernels of libfresco_b200.so instead of ~15 torch ops (fresco_cfg_pred_x0 / fresco_ddpm_prev);
* background smoothing calls this package's warp_tensor (image-resolution chain, dilation kernel);
* ``inference(..., shard=(world, rank, group))`` (not in the reference) runs ONE keyframe batch frame-sharded over the
  GPUs of a box: every rank holds frames frame_range(N, G, rank) = [rank*N//G, (rank+1)*N//G); the initial noise and the per-step noise are drawn
  for ALL N frames from identically seeded generators on every rank and sliced, so the sample paths are those of the
  unsharded run (``repeat_noise`` needs frame 0's noise everywhere, :67-68, :150-151); ``record_latents`` (frames 0
  and N-1, :175-179) is assembled with one tiny all-gather per step; restoring frames 0-1 in propagation mode touches
  rank 0 (and rank 1 when a rank holds a single frame); the background-smoothing steps decode, warp and re-encode only
  this rank's frames (``warp_tensor(shard=...)`` gathers the decoded frames for the image-resolution chain).
The VAE, ControlNet, scheduler tables and the UNet body stay what the caller passes in (diffusers objects or the bench
harness).
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import ops
from .dist import ShardLayout, batch_layout, shard_layout
from .flow_utils import warp_tensor


def _step_coefficients(scheduler, timestep):
    """alpha / beta products of a DDPM step, computed exactly as src/pipe_FRESCO.py:22-31,51-58 does (0-dim tensors of
    the scheduler's own dtype), returned as python floats"""
    prev_timestep = scheduler.previous_timestep(timestep)
    alpha_prod_t = scheduler.alphas_cumprod[timestep]
    alpha_prod_t_prev = scheduler.alphas_cumprod[prev_timestep] if prev_timestep >= 0 else scheduler.one
    beta_prod_t = 1 - alpha_prod_t
    beta_prod_t_prev = 1 - alpha_prod_t_prev
    current_alpha_t = alpha_prod_t / alpha_prod_t_prev
    current_beta_t = 1 - current_alpha_t
    c_x0 = (alpha_prod_t_prev ** 0.5 * current_beta_t) / beta_prod_t
    c_xt = current_alpha_t ** 0.5 * beta_prod_t_prev / beta_prod_t
    variance = torch.clamp(torch.as_tensor(beta_prod_t_prev / beta_prod_t * current_beta_t), min=1e-20)
    return float(alpha_prod_t), float(c_x0), float(c_xt), float(variance ** 0.5)


def step(pipe, model_output, timestep, sample, generator, repeat_noise=False, visualize_pipeline=False, flows=None,
         occs=None, saliency=None, guidance_scale: Optional[float] = None, noise: Optional[torch.Tensor] = None,
         shard=None):
    """DDPM step with background smoothing (src/pipe_FRESCO.py:14-77).

    ``model_output`` is the guided noise prediction [N, ...] as in the reference; if ``guidance_scale`` is given it is
    the raw UNet output [2N, ...] (uncond | text) and the guidance (:212-215) is fused into the first kernel.
    ``noise`` (optional) replaces the ``torch.randn`` draw of :61-62 (the frame-sharded loop passes its slice).
    ``shard=(world, rank[, group])``: ``sample`` holds this rank's frames of a frame-sharded batch (``flows`` / ``occs``
    / ``saliency`` the whole batch's); background smoothing decodes and re-encodes those frames only and warps them
    along the whole chain.  ``shard`` may be a ``dist.ShardLayout``; in its half and unequal-halves layouts
    ``model_output`` is this rank's CFG half of the raw UNet output [n, ...]: the other half's rows of the same frames
    come from the peers (one batched send / receive), so every rank runs the guidance on a contiguous [uncond; text]
    block, and the smoothing round trip runs on the ranks of half 0, which send its rows to their peers.  On an idle
    rank of a ``dist.Box`` it returns ``(sample, sample)`` at once.  A ``dist.Box`` itself takes the frame count from
    ``flows``; without them, pass its layout (``dist.shard_layout(N, box)``), as ``inference`` does."""
    layout = batch_layout(shard, flows, sample, 1, "step(shard=Box(...)) without flows does not know the batch's frame "
                                                   "count: pass dist.shard_layout(n_frames, box)")
    if layout.idle:
        return (sample, sample)
    alpha_prod_t, c_x0, c_xt, sigma = _step_coefficients(pipe.scheduler, timestep)
    sample = sample.contiguous()
    do_cfg = guidance_scale is not None
    model_output = layout.guided(model_output, do_cfg)
    pred_original_sample = ops.cfg_pred_x0(model_output.contiguous(), sample, guidance_scale if do_cfg else 0.0,
                                           alpha_prod_t, do_cfg=do_cfg)
    if saliency is not None and flows is not None and occs is not None:                        # :44-47
        def smooth():
            image = pipe.vae.decode(pred_original_sample / pipe.vae.config.scaling_factor).sample
            image = warp_tensor(image, flows, occs, saliency, unet_chunk_size=1, shard=layout)
            return (pipe.vae.config.scaling_factor * pipe.vae.encode(image).latent_dist.sample()).contiguous()
        pred_original_sample = layout.share(smooth, (pred_original_sample.shape, pred_original_sample.dtype,
                                                     pred_original_sample.device))
    if noise is None:
        noise = torch.randn(sample.shape, generator=generator, device=sample.device, dtype=sample.dtype)
    pred_prev_sample = ops.ddpm_prev(pred_original_sample, sample, noise.contiguous(), c_x0, c_xt, sigma,
                                     repeat_noise=repeat_noise)
    return (pred_prev_sample, pred_original_sample)


def _gather_first_last(latents_local, layout: ShardLayout):
    """[x_0, x_{N-1}] of the batch (src/pipe_FRESCO.py:177,179), whose frames may be spread over the exchange group"""
    if layout.world == 1:
        return latents_local[[0, len(latents_local) - 1]].detach().clone()
    import torch.distributed as dist
    mine = torch.stack([latents_local[0], latents_local[-1]])                  # my first / last frame
    allp = torch.empty((layout.world,) + tuple(mine.shape), dtype=mine.dtype, device=mine.device)
    dist.all_gather_into_tensor(allp.view(-1, *mine.shape[1:]), mine, group=layout.group)
    return torch.stack([allp[0, 0], allp[layout.world - 1, 1]]).clone()


@torch.no_grad()
def inference(pipe, controlnet, frescoProc, imgs, prompt_embeds, edges, timesteps, cond_scale=[0.7] * 20,
              num_inference_steps=20, num_warmup_steps=6, do_classifier_free_guidance=True, seed=0, guidance_scale=7.5,
              use_controlnet=True, record_latents=[], propagation_mode=False, visualize_pipeline=False, flows=None,
              occs=None, saliency=None, repeat_noise=False, num_intraattn_steps=1, step_interattn_end=350,
              bg_smoothing_steps=[16, 17], shard=None):
    """Video-to-video translation of one keyframe batch with FRESCO (src/pipe_FRESCO.py:81-234).

    ``imgs`` / ``edges`` / ``prompt_embeds`` / ``flows`` / ``occs`` / ``saliency`` hold ALL N frames (every rank gets the
    same arguments); with ``shard=(world, rank[, group])`` this rank denoises frames [rank*N//G, (rank+1)*N//G) and
    returns their latents, the background-smoothing steps included.  With ``shard=dist.Box(...)`` every frame count
    runs (``dist.shard_layout``); an idle rank returns empty latents [0, 4, h, w] at once and leaves ``record_latents``
    as it is."""
    device = pipe._execution_device
    noise_scheduler = pipe.scheduler
    B, C, H, W = imgs.shape
    layout = shard_layout(B, shard)
    if layout.idle:
        f = getattr(pipe, "vae_scale_factor", 8)
        return torch.empty(0, pipe.unet.config.in_channels, H // f, W // f, dtype=prompt_embeds.dtype, device=device)
    generator = torch.Generator(device=device).manual_seed(seed)
    lo, hi = layout.lo, layout.hi
    cfg_chunks = 2 if do_classifier_free_guidance else 1
    chunks = layout.chunks(cfg_chunks)                                          # the halves need both CFG halves
    if hasattr(frescoProc, "set_batch_frames"):
        frescoProc.set_batch_frames(B)
    latents = pipe.prepare_latents(B, pipe.unet.config.in_channels, H, W, prompt_embeds.dtype, device, generator,
                                   latents=None)                                # all N frames: same Philox stream everywhere
    if repeat_noise:
        latents = latents[0:1].repeat(B, 1, 1, 1).detach()
    if num_warmup_steps < 0:
        latents_init = latents.detach()[lo:hi]
        num_warmup_steps = 0
    else:
        def encode():
            return pipe.vae.config.scaling_factor * pipe.vae.encode(imgs[lo:hi].to(pipe.unet.dtype)).latent_dist.sample()
        # partners must hold the same latents: the posterior sample is drawn once, on the half-0 rank
        latent_x0 = layout.share(encode, (latents[lo:hi].shape, getattr(pipe.vae, "dtype", pipe.unet.dtype),
                                          latents.device))
        latents_init = noise_scheduler.add_noise(latent_x0, latents[lo:hi], timesteps[num_warmup_steps]).detach()
    n_local = hi - lo
    pe = layout.rows(prompt_embeds, cfg_chunks)                                 # (b f) layout: the frames held
    latents = latents_init
    for i, t in enumerate(timesteps[num_warmup_steps:]):
        if i >= num_intraattn_steps:
            frescoProc.controller.disable_intraattn()
        if t < step_interattn_end:
            frescoProc.controller.disable_interattn()
        if propagation_mode:                                                     # :175-177
            if lo < 2:                                                           # this rank holds frame 0 or 1
                rec = record_latents[i].detach().clone()
                for f in range(2):
                    if lo <= f < hi:
                        latents[f - lo] = rec[f]
            first_last = _gather_first_last(latents, layout)
            if i < len(record_latents):
                record_latents[i] = first_last
            else:                                                                # idle in the first batch of a Box
                record_latents.append(first_last)
        else:
            record_latents += [_gather_first_last(latents, layout)]
        # one CFG half per rank in the half layout: its latents, prompt and edge rows only
        latent_model_input = torch.cat([latents] * chunks) if chunks > 1 else latents
        if use_controlnet:
            e = layout.rows(edges, cfg_chunks)
            down_block_res_samples, mid_block_res_sample = controlnet(
                latent_model_input, t, encoder_hidden_states=pe, controlnet_cond=e,
                conditioning_scale=cond_scale[i + num_warmup_steps], guess_mode=False, return_dict=False)
        else:
            down_block_res_samples, mid_block_res_sample = None, None
        noise_pred = pipe.unet(latent_model_input, t, encoder_hidden_states=pe, cross_attention_kwargs=None,
                               down_block_additional_residuals=down_block_res_samples,
                               mid_block_additional_residual=mid_block_res_sample, return_dict=False)[0]
        # per-step noise for ALL frames from the shared generator, then this rank's slice (frame 0's under repeat_noise)
        full_noise = torch.randn((B,) + tuple(latents.shape[1:]), generator=generator, device=latents.device,
                                 dtype=latents.dtype)
        noise = full_noise[0:1].expand(n_local, *latents.shape[1:]).contiguous() if repeat_noise else full_noise[lo:hi]
        smooth = (i + num_warmup_steps) in bg_smoothing_steps
        latents = step(pipe, noise_pred, t, latents, generator, visualize_pipeline=visualize_pipeline,
                       flows=flows if smooth else None, occs=occs if smooth else None, saliency=saliency if smooth else None,
                       guidance_scale=guidance_scale if do_classifier_free_guidance else None, noise=noise,
                       shard=layout)[0]
    return latents
