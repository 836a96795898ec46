"""Drop-in for the reference's ``src/flow_utils.py`` + the geometry helpers it
uses, backed by the sm_90a kernels (no PyTorch fallback for the hot ops).

Public names and argument meaning follow the reference:
``warp_tensor`` (src/flow_utils.py:18-53), ``get_single_mapping_ind`` (:56-102),
``get_mapping_ind`` (:105-138), ``flow_warp`` / ``forward_backward_consistency_check``
(gmflow/geometry.py:65-96).  Small per-batch preparation (resizing flows, pooling
occlusion masks) stays in torch; the per-step work runs in libfresco_b200.so.
"""
from __future__ import annotations

from typing import List, Sequence

import torch
import torch.nn.functional as F

from . import ops


# --------------------------------------------------------------------------- geometry
def flow_warp(feature: torch.Tensor, flow: torch.Tensor) -> torch.Tensor:
    """Bilinear warp at pixel coordinates (x+flow_x, y+flow_y), zeros outside.
    gmflow/geometry.py:65-72.  fp32 kernel; other dtypes are converted."""
    out = ops.flow_warp(feature.float().contiguous(), flow.float().contiguous())
    return out.to(feature.dtype)


def forward_backward_consistency_check(fwd_flow, bwd_flow, alpha=0.01, beta=0.5):
    """gmflow/geometry.py:75-96."""
    mag = torch.norm(fwd_flow, dim=1) + torch.norm(bwd_flow, dim=1)
    warped_bwd = flow_warp(bwd_flow, fwd_flow)
    warped_fwd = flow_warp(fwd_flow, bwd_flow)
    thr = alpha * mag + beta
    fwd_occ = (torch.norm(fwd_flow + warped_bwd, dim=1) > thr).float()
    bwd_occ = (torch.norm(bwd_flow + warped_fwd, dim=1) > thr).float()
    return fwd_occ, bwd_occ


def _dilate(x: torch.Tensor, k: int) -> torch.Tensor:
    """k x k binary dilation with replicate padding (src/utils.py:81-93)."""
    return ops.dilate(x.float().contiguous(), k)


_PREP_CACHE: "dict" = {}
_PREP_CACHE_MAX = 16


def _tensor_key(t: torch.Tensor):
    return (id(t), t._version)


def clear_prep_cache() -> None:
    """Drop every cached per-batch preparation (called when a new keyframe batch is installed)."""
    _PREP_CACHE.clear()


def _cache_get(tag, tensors, make):
    """Per-batch preparation (resized flows, pooled masks, blend weights, warp adjoints) depends only on the flow /
    occlusion / saliency tensors, which are constant over the denoise steps of a batch: the reference recomputes it at
    every call (flow_utils.py:24-39).  An entry is keyed on the IDENTITY (and in-place version counter) of those
    tensors and keeps a reference to them, so a hit is validated with ``is`` -- an address the allocator hands out
    again for the next batch's flows can never alias a live entry."""
    key = (tag,) + tuple(_tensor_key(t) for t in tensors)
    hit = _PREP_CACHE.get(key)
    if hit is not None and len(hit[0]) == len(tensors) and all(a is b for a, b in zip(hit[0], tensors)):
        return hit[1]
    if len(_PREP_CACHE) >= _PREP_CACHE_MAX:
        _PREP_CACHE.pop(next(iter(_PREP_CACHE)))            # oldest entry (insertion order)
    value = make()
    _PREP_CACHE[key] = (tuple(tensors), value)
    return value


def resize_flows_occs(flows: Sequence[torch.Tensor], occs: Sequence[torch.Tensor], size_h: int):
    """Flows / occlusions at the resolution of a feature map.
    src/flow_utils.py:24-33 == src/diffusion_hacked.py:437-442."""
    return _cache_get(("resize", size_h), (flows[0], flows[1], occs[0], occs[1]),
                      lambda: _resize_flows_occs(flows, occs, size_h))


def _resize_flows_occs(flows, occs, size_h):
    scale = size_h * 1.0 / flows[0].shape[2]
    kernel = int(1 / scale)
    bwd_flow = F.interpolate(flows[1] * scale, scale_factor=scale, mode="bilinear")
    fwd_flow = F.interpolate(flows[0] * scale, scale_factor=scale, mode="bilinear")
    bwd_occ = F.max_pool2d(occs[1].unsqueeze(1), kernel_size=kernel)
    fwd_occ = F.max_pool2d(occs[0].unsqueeze(1), kernel_size=kernel)
    return scale, fwd_flow.float().contiguous(), bwd_flow.float().contiguous(), fwd_occ.float(), bwd_occ.float()


def adjoint_csr(flows, occs, size_h: int):
    """ELL matrices of the warp adjoints (backward of flow_warp) at a feature resolution, cached per batch."""
    def make():
        _, fwd_flow, bwd_flow, _, _ = resize_flows_occs(flows, occs, size_h)
        return ops.warp_adjoint_pair(bwd_flow, fwd_flow)
    return _cache_get(("adjoint", size_h), (flows[0], flows[1], occs[0], occs[1]), make)


# --------------------------------------------------------------------------- warp_tensor
def chain_operands(flows, occs, saliency, n: int, h: int, w: int):
    """The operands of warp_tensor's frame chain at an h x w feature map (src/flow_utils.py:24-51), cached per batch:
    bwd_flow [n, 2, h, w], fwd_flow_last [2, h, w] and the blend weights [n, 1, h, w], all fp32."""
    def prepare():
        scale, fwd_flow, bwd_flow, fwd_occ, bwd_occ = resize_flows_occs(flows, occs, h)
        if scale == 1:
            bwd_occ = _dilate(bwd_occ, 13)
            fwd_occ = _dilate(fwd_occ, 13)
        scale2 = h * 1.0 / saliency.shape[2]
        sal = F.interpolate(saliency.float(), scale_factor=scale2, mode="bilinear").contiguous()
        warp_sal = ops.flow_warp(sal, bwd_flow)                                    # :38
        warp_sal_last = ops.flow_warp(sal[0:1].contiguous(), fwd_flow[n - 1:n].contiguous())   # :39
        blend = torch.empty(n, 1, h, w, dtype=torch.float32, device=bwd_flow.device)
        blend[:n - 1] = (1 - bwd_occ[:n - 1]) * sal[1:n] * warp_sal[:n - 1]       # :45
        blend[n - 1:] = (1 - fwd_occ[n - 1:n]) * sal[n - 1:n] * warp_sal_last      # :50
        return bwd_flow, fwd_flow[n - 1].contiguous(), blend.contiguous()

    return _cache_get(("warp_tensor", n, h, w), (flows[0], flows[1], occs[0], occs[1], saliency), prepare)


@torch.no_grad()
def warp_tensor(sample, flows, occs, saliency, unet_chunk_size, shard=None):
    """Warp + fuse along the frame chain (src/flow_utils.py:18-53).

    Unlike the reference (which aliases and mutates fp32 inputs, :36) this never
    modifies ``sample``; the result has the dtype of ``sample``.

    ``shard=(world, rank[, group])`` (not in the reference): ``sample`` holds this rank's frames of a frame-sharded
    batch (flows / occs / saliency describe ALL N frames).  With fewer frames than ranks (``dist.shard_layout``'s half
    and unequal-halves layouts) ``sample`` holds one CFG half of this rank's frames, [n_local, ...] whatever
    ``unet_chunk_size`` says, and everything below runs within the ranks of that half (``shard`` may also be the
    ``ShardLayout`` itself); an idle rank of a ``dist.Box`` gets ``sample`` back.  The
    chain is sequential over frames but independent per (chunk, channel) plane, so the batch is re-sharded by CHANNEL
    for the chain: one all-to-all turns
    [frames/G, all channels] into [all frames, channels/G], every rank runs the chain kernel on its channel slice, a
    second all-to-all brings the frames back (SURVEY 8e, "sequential pieces").  When the channels do not split over the
    ranks (a decoded image has 3: background smoothing, src/pipe_FRESCO.py:46) every rank all-gathers the frames instead,
    runs the chain on the whole batch and keeps its own frames."""
    from .dist import shard_layout
    layout = shard_layout(flows[0].shape[0], shard)
    if layout.idle:
        return sample                                           # an idle rank of a dist.Box holds no frame
    # a rank holding one CFG half (or, in background smoothing, the decoded frames on the ranks of half 0) holds one
    # chunk, and the exchanges run within the ranks of its half
    chunks = min(unet_chunk_size, layout.halves[1] - layout.halves[0])
    world, n = layout.world, layout.n_frames
    h, w = sample.shape[2], sample.shape[3]

    bwd_flow, fwd_flow_last, blend = chain_operands(flows, occs, saliency, n, h, w)

    def chain(planes, chunks):
        return ops.warp_fuse_chain(planes, bwd_flow, fwd_flow_last, blend, chunks)

    def chain_input(t):
        # the shared-memory chain kernel takes fp16 or fp32 planes up to 100 KB; image-resolution planes (background
        # smoothing, src/pipe_FRESCO.py:46, fp16 VAE output) run the per-step kernel, which works on fp32 like the
        # reference's own `.to(torch.float32)` copy (flow_utils.py:36)
        if t.dtype not in (torch.float16, torch.float32) or 2 * h * w * 4 > 200 * 1024:
            return t.float()
        return t

    lo, hi = layout.lo, layout.hi
    n_local, C = hi - lo, sample.shape[1]
    if sample.shape[0] != chunks * n_local:
        raise ValueError(f"warp_tensor: rank {layout.rank} of {world} owns frames [{lo}, {hi}) of {n}, "
                         f"so sample needs {chunks * n_local} planes, got {sample.shape[0]}")
    if world == 1:
        return chain(chain_input(sample.contiguous()), chunks).to(sample.dtype)
    import torch.distributed as dist
    from .dist import block_sizes
    if C % world != 0:
        # gather path: the frames travel in the dtype of ``sample`` (fp16 VAE output: 1.5 MB per 512^2 frame), the chain
        # runs on exactly the batch the unsharded call sees
        full = layout.gather_frames(sample, chunks)                                   # [chunk, frame, C, h, w]
        fused = chain(chain_input(full), chunks).view(chunks, n, C, h, w)
        return fused[:, lo:hi].reshape(chunks * n_local, C, h, w).to(sample.dtype)
    x = chain_input(sample.contiguous())
    cg = C // world
    frames = block_sizes(n, world)                              # split sizes of the all-to-alls, in frames
    send = x.view(chunks, n_local, world, cg, h * w).permute(2, 1, 0, 3, 4).contiguous()      # [dest, frame, chunk, cg, hw]
    send = send.view(world * n_local, chunks * cg * h * w)
    recv = torch.empty(n, chunks * cg * h * w, dtype=x.dtype, device=x.device)
    dist.all_to_all_single(recv, send, frames, [n_local] * world, group=layout.group)   # [source rank = frame block, frame, ...]
    planes = recv.view(n, chunks * cg, h, w)                    # all N frames x my channel slice of both chunks
    fused = chain(planes, 1)
    back = torch.empty_like(send)
    dist.all_to_all_single(back, fused.view(n, -1), [n_local] * world, frames, group=layout.group)   # [source = channel block, ...]
    out = back.view(world, n_local, chunks, cg, h * w).permute(2, 1, 0, 3, 4).reshape(chunks * n_local, C, h, w)
    return out.contiguous().to(sample.dtype)


# --------------------------------------------------------------------------- pixel mapping
@torch.no_grad()
def get_single_mapping_ind(bwd_flow, bwd_occ, imgs, scale=1.0):
    """Pixel correspondence between two frames (src/flow_utils.py:56-102).
    The sequential conflict loop (:84-97) is replaced by a parallel lexicographic
    arg-min kernel; results are bit-identical to the reference's CPU output."""
    mapping, unlinked = ops.mapping_single(bwd_flow.float().contiguous(), bwd_occ.float().contiguous(),
                                           imgs.float().contiguous(), int(scale))
    return mapping, unlinked


@torch.no_grad()
def get_mapping_ind(bwd_flows, bwd_occs, imgs, scale=1.0):
    """Chain pairwise correspondences over the N frames of a batch
    (src/flow_utils.py:105-138): returns fwd_mappings [N,1,L], bwd_mappings
    [N,1,L] (int64) and the trajectory mask [L,1,N,N] (bool)."""
    n = imgs.shape[0]
    H, W = int(imgs.shape[2] // scale), int(imgs.shape[3] // scale)
    L = H * W
    dev = imgs.device
    mask = torch.ones(L, n, n, dtype=torch.bool, device=dev)
    ar = torch.arange(L, device=dev)
    fwd: List[torch.Tensor] = [ar]
    bwd: List[torch.Tensor] = [ar]
    for i in range(n - 1):
        cut = torch.ones(n, n, dtype=torch.bool, device=dev)
        cut[:i + 1, i + 1:] = False
        cut[i + 1:, :i + 1] = False
        mp, unl = get_single_mapping_ind(bwd_flows[i:i + 1], bwd_occs[i:i + 1], imgs[i:i + 2], scale)
        sel = unl[fwd[-1]]
        mask[sel] = mask[sel] & cut
        nxt = mp[fwd[-1]]
        fwd.append(nxt)
        inv = torch.empty_like(nxt)
        inv[nxt] = ar                       # argsort of a permutation == its inverse
        bwd.append(inv)
    return torch.stack(fwd, 0).unsqueeze(1), torch.stack(bwd, 0).unsqueeze(1), mask.unsqueeze(1)
