"""Tensor-level wrappers over the C ABI: allocate outputs with torch, pass raw
device pointers + the current CUDA stream.  No arithmetic happens here."""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import _lib as L

# Optional device-side timing of individual launches (bench.py sets this to a list; each entry is
# (tag, work, start_event, end_event) recorded on the launching stream).
PROFILE = None


def _prof_begin():
    if PROFILE is None:
        return None
    ev = torch.cuda.Event(enable_timing=True)
    ev.record(torch.cuda.current_stream())
    return ev


def _prof_end(ev, tag, work, bound="tensor"):
    """``work`` = algorithmic flops (bound "tensor") or bytes (bound "hbm") of the launch(es) between the two events,
    per SURVEY.md 8(d)."""
    if ev is not None:
        end = torch.cuda.Event(enable_timing=True)
        end.record(torch.cuda.current_stream())
        PROFILE.append((tag, work, ev, end, bound))


def kv_compact(k: torch.Tensor, v: torch.Tensor, idx: torch.Tensor, chunks: int):
    """k, v [chunks*frames, tokens, C] fp16; idx int32 [n_sel] over (frame, token) -> [chunks, n_sel, C]."""
    B, tokens, C = k.shape
    rows = (B // chunks) * tokens
    n_sel = idx.numel()
    k_out = torch.empty(chunks, n_sel, C, dtype=k.dtype, device=k.device)
    v_out = torch.empty_like(k_out)
    ev = _prof_begin()
    L.check(L.lib().fresco_kv_compact(L.ptr(k), L.ptr(v), L.ptr(idx), L.ptr(k_out), L.ptr(v_out), chunks, rows,
                                      n_sel, C, L.stream()), "fresco_kv_compact")
    _prof_end(ev, "kv_compact_C%d_n%d" % (C, n_sel), 8.0 * chunks * n_sel * C, "hbm")     # K and V rows: read + write
    return k_out, v_out


def kv_compact_packed(k: torch.Tensor, v: torch.Tensor, idx: torch.Tensor, kv_out: torch.Tensor, chunks: int):
    """Selected K and V rows side by side into rows [0, n_sel) of kv_out [chunks, out_rows, 2C] (exchange send buffer)."""
    B, tokens, C = k.shape
    rows = (B // chunks) * tokens
    ev = _prof_begin()
    L.check(L.lib().fresco_kv_compact_packed(L.ptr(k), L.ptr(v), L.ptr(idx), L.ptr(kv_out), chunks, rows, idx.numel(),
                                             kv_out.shape[1], C, L.stream()), "fresco_kv_compact_packed")
    _prof_end(ev, "kv_compact_C%d_n%d" % (C, idx.numel()), 8.0 * chunks * idx.numel() * C, "hbm")
    return kv_out


def rows_gather(src: torch.Tensor, idx: torch.Tensor, dst: torch.Tensor, dst_col: int = 0):
    """dst[r, dst_col : dst_col + W] = src[idx[r], :] for 2-D row views (src [*, W], dst [n, >= dst_col + W])."""
    W = src.shape[-1]
    es = src.element_size()
    L.check(L.lib().fresco_rows_gather(L.ptr(src), L.ptr(idx), L.ptr(dst), idx.numel(), W * es, dst.shape[-1] * es,
                                       dst_col * es, L.stream()), "fresco_rows_gather")
    return dst


def rows_scatter(src: torch.Tensor, idx: torch.Tensor, dst: torch.Tensor):
    """dst[idx[r], :] = src[r, :]."""
    W = src.shape[-1]
    L.check(L.lib().fresco_rows_scatter(L.ptr(src), L.ptr(idx), L.ptr(dst), idx.numel(), W * src.element_size(),
                                        L.stream()), "fresco_rows_scatter")
    return dst


def attn_fwd_kv_packed(q: torch.Tensor, kv: torch.Tensor, heads: int, q_per_kv: int, softmax_scale: float,
                       out: Optional[torch.Tensor] = None):
    """q [Bq, Lq, C]; kv [Bq/q_per_kv, Lk, 2C] with K in columns [0, C) and V in [C, 2C) of every row."""
    Bq, Lq, C = q.shape
    d = C // heads
    Lk = kv.shape[1]
    if q.dtype != torch.float16 or kv.dtype != torch.float16 or kv.shape[2] != 2 * C:
        raise L.FrescoError("attn_fwd_kv_packed: fp16 q [B,L,C] and kv [B/q_per_kv, Lk, 2C] expected")
    if out is None:
        out = torch.empty_like(q)
    ev = _prof_begin()
    kp = L.ptr(kv)
    L.check(L.lib().fresco_attn_fwd_kv_strided(L.ptr(q), kp, kp + C * 2, L.ptr(out), Bq, Lq, Lk, heads, d, q_per_kv,
                                               2 * C, Lk * 2 * C, float(softmax_scale), 0.0, L.stream()),
            "fresco_attn_fwd_kv_strided")
    _prof_end(ev, "attn_d%d_L%d_Lk%d" % (d, Lq, Lk), 4.0 * Bq * Lq * Lk * C)
    return out


def _check_temporal_operands(what, tensors, width, fwd_map, traj_mask, chunks, heads):
    """Refuse, before any launch, operands the kernels would reinterpret: the C ABI takes raw pointers, so an fp32 q, an
    int32 map or a mask of the wrong shape would otherwise be read as fp16 / int64 / [tokens, N, N] bytes."""
    if any(t.dtype != torch.float16 or t.dim() != 3 for t in tensors):
        raise L.FrescoError(f"{what}: q, k, v must be fp16 [chunks*frames, tokens, C]")
    B, tokens, C = tensors[0].shape
    if any(t.shape != tensors[0].shape for t in tensors) or C % width:
        raise L.FrescoError(f"{what}: q, k, v shapes differ")
    C //= width
    if chunks <= 0 or B % chunks:
        raise L.FrescoError(f"{what}: {B} rows do not split into {chunks} chunks")
    if heads <= 0 or C % heads:
        raise L.FrescoError(f"{what}: C = {C} is not a multiple of heads = {heads}")
    frames = B // chunks
    if fwd_map.dtype != torch.int64 or tuple(fwd_map.shape) != (frames, tokens):
        raise L.FrescoError(f"{what}: fwd_map must be int64 [{frames}, {tokens}], got {fwd_map.dtype} "
                            f"{list(fwd_map.shape)}")
    if traj_mask.dtype not in (torch.uint8, torch.bool) or tuple(traj_mask.shape) != (tokens, frames, frames):
        raise L.FrescoError(f"{what}: traj_mask must be uint8 or bool [{tokens}, {frames}, {frames}], got "
                            f"{traj_mask.dtype} {list(traj_mask.shape)}")
    return frames, tokens, C


def temporal_attn_fwd_packed(qkv: torch.Tensor, fwd_map, traj_mask, chunks: int, heads: int, scale: float):
    """qkv [chunks*frames, tokens, 3C] with q | k | v side by side in every row -> out [chunks*frames, tokens, C]."""
    frames, tokens, C = _check_temporal_operands("temporal_attn_fwd_packed", (qkv,), 3, fwd_map, traj_mask, chunks,
                                                 heads)
    B = qkv.shape[0]
    C3 = 3 * C
    out = torch.empty(B, tokens, C, dtype=qkv.dtype, device=qkv.device)
    base = L.ptr(qkv)
    ev = _prof_begin()
    L.check(L.lib().fresco_temporal_attn_fwd_strided(base, base + 2 * C, base + 4 * C, L.ptr(out), L.ptr(fwd_map),
                                                     L.ptr(traj_mask), chunks, frames, tokens, heads, C // heads, C3,
                                                     float(scale), L.stream()), "fresco_temporal_attn_fwd_strided")
    _prof_end(ev, "temporal_d%d_L%d_N%d" % (C // heads, tokens, frames), 8.0 * B * tokens * C, "hbm")
    return out


def attn_fwd(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, q_per_kv: int = 1,
             softmax_scale: Optional[float] = None, diag_bias: float = 0.0, out: Optional[torch.Tensor] = None):
    """q [Bq, Lq, C], k/v [Bq/q_per_kv, Lk, C] fp16 token-major -> [Bq, Lq, C]."""
    Bq, Lq, C = q.shape
    d = C // heads
    if q.dtype != torch.float16 or k.dtype != torch.float16 or v.dtype != torch.float16:
        raise L.FrescoError("fresco attention kernels are fp16 (the reference's GPU dtype)")
    if softmax_scale is None:
        softmax_scale = 1.0 / math.sqrt(d)
    if out is None:
        out = torch.empty_like(q)
    ev = _prof_begin()
    L.check(L.lib().fresco_attn_fwd(L.ptr(q), L.ptr(k), L.ptr(v), L.ptr(out), Bq, Lq, k.shape[1], heads, d,
                                    q_per_kv, float(softmax_scale), float(diag_bias), L.stream()),
            "fresco_attn_fwd")
    _prof_end(ev, "attn_d%d_L%d_Lk%d" % (d, Lq, k.shape[1]), 4.0 * Bq * Lq * k.shape[1] * C)
    return out


def temporal_attn_fwd(q_raw, k_raw, v_src, fwd_map, traj_mask, chunks: int, heads: int, scale: float):
    """q_raw, k_raw, v_src [chunks*frames, tokens, C] fp16; fwd_map int64 [frames, tokens]; traj_mask uint8 / bool
    [tokens, frames, frames] -> out like v_src (include/fresco_b200.h, A5)."""
    frames, tokens, C = _check_temporal_operands("temporal_attn_fwd", (q_raw, k_raw, v_src), 1, fwd_map, traj_mask,
                                                 chunks, heads)
    B = q_raw.shape[0]
    out = torch.empty_like(v_src)
    ev = _prof_begin()
    L.check(L.lib().fresco_temporal_attn_fwd(L.ptr(q_raw), L.ptr(k_raw), L.ptr(v_src), L.ptr(out), L.ptr(fwd_map),
                                             L.ptr(traj_mask), chunks, frames, tokens, heads, C // heads,
                                             float(scale), L.stream()), "fresco_temporal_attn_fwd")
    # algorithmic bytes (SURVEY 8d): 3 reads + 1 write of [B, L, C] fp16 (+ indices and mask, < 1 %)
    _prof_end(ev, "temporal_d%d_L%d_N%d" % (C // heads, tokens, frames), 8.0 * B * tokens * C, "hbm")
    return out


def flow_warp(src: torch.Tensor, flow: torch.Tensor) -> torch.Tensor:
    """fp32 [B,C,h,w] warped by flow [Bf,2,h,w] (sample b uses flow b % Bf)."""
    B, C, h, w = src.shape
    dst = torch.empty_like(src)
    L.check(L.lib().fresco_flow_warp(L.ptr(src), L.ptr(flow), L.ptr(dst), B, C, h, w, flow.shape[0], L.stream()),
            "fresco_flow_warp")
    return dst


def warp_fuse_chain(sample, bwd_flow, fwd_flow_last, blend, chunks: int, out=None):
    B, C, h, w = sample.shape
    if out is None:
        out = torch.empty_like(sample)
    is_half = 1 if sample.dtype == torch.float16 else 0
    if not is_half and sample.dtype != torch.float32:
        raise L.FrescoError("warp_fuse_chain: fp16 or fp32 only")
    ev = _prof_begin()
    L.check(L.lib().fresco_warp_fuse_chain(L.ptr(sample), L.ptr(out), is_half, L.ptr(bwd_flow), L.ptr(fwd_flow_last),
                                           L.ptr(blend), chunks, B // chunks, C, h, w, L.stream()),
            "fresco_warp_fuse_chain")
    # every frame read once and written once (SURVEY 8d counts 3 fp32 passes for the reference's unfused chain)
    _prof_end(ev, "warp_chain_C%d_%dx%d" % (C, h, w), 2.0 * sample.numel() * sample.element_size(), "hbm")
    return out


ELL_SLOTS = 8

_WORKSPACES: dict = {}


def _workspace(key, nbytes: int, device) -> torch.Tensor:
    """Scratch buffers of the kernels that need one, kept per (use, device) and grown on demand (a fresh torch.empty per
    call costs an allocator round trip 80 times per optimised step)."""
    ws = _WORKSPACES.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        _WORKSPACES[key] = ws
    return ws


def warp_adjoint_ell(flow: torch.Tensor):
    """Per-batch operands of the temporal-consistency loss for the warp by ``flow`` [F,2,h,w]: the bilinear taps of
    every source pixel (fresco_warp_taps) packed into the ADJOINT of that warp by :func:`_pack_adjoint`."""
    Fr, _, h, w = flow.shape
    dest = torch.empty(Fr, h * w, 4, dtype=torch.int32, device=flow.device)
    wgt = torch.empty(Fr, h * w, 4, dtype=torch.float32, device=flow.device)
    L.check(L.lib().fresco_warp_taps(L.ptr(flow), L.ptr(dest), L.ptr(wgt), Fr, h, w, L.stream()), "fresco_warp_taps")
    return _pack_adjoint(dest, wgt, h, w)


def _pack_adjoint(dest: torch.Tensor, wgt: torch.Tensor, h: int, w: int):
    """Taps dest int [F, hw, 4] (-1 = none) / wgt fp32 [F, hw, 4] of the warp -> its ADJOINT in ELL form, row =
    destination pixel, up to 8 entries (round(w*65535) << 16) | source in uint32 (``ell_packed`` [F, hw, 8]);
    destinations with more than 8 taps spill to ``ovf`` int32 [F, n_ovf, 3] = (destination | -1, source, float bits
    of the weight).  Pure torch (runs on any device).

    Invariant the loss kernels rely on: a row's used slots come first and a slot whose weight field is 0 ends the row
    (warp_loss_quad_kernel stops a warp's walk at the first slot that is 0 in all of its lanes).  A tap whose weight
    rounds to a 0 field (w < 2^-17) is therefore dropped, from the ELL and from the overflow list alike: it would
    contribute nothing through the ELL anyway, and it sorts by source, so it can come before the row's main tap.
    (The loss kernels also take keep masks in {0, 1}: their fp16 sgn(r) * keep planes are exact only for those.)"""
    Fr = dest.shape[0]
    dest = dest.reshape(Fr, -1)
    wgt = wgt.reshape(Fr, -1)
    return _pack_ell(torch.where((wgt * 65535.0).round() > 0, dest, torch.full_like(dest, -1)), wgt, h, w)


def _pack_ell(dest: torch.Tensor, wgt: torch.Tensor, h: int, w: int):
    """The packing of :func:`_pack_adjoint` for every tap with dest >= 0, whatever its weight (dest, wgt [F, 4 hw])."""
    Fr = dest.shape[0]
    hw = h * w
    dev = dest.device
    dest = dest.long()
    src = torch.arange(hw, device=dev).repeat_interleave(4)[None].expand(Fr, -1)
    key = torch.where(dest >= 0, dest, torch.full_like(dest, hw))            # tap-less entries sort to the end
    order = torch.argsort(key, dim=1, stable=True)
    key_s = torch.gather(key, 1, order).contiguous()
    src_s = torch.gather(src, 1, order)
    w_s = torch.gather(wgt, 1, order)
    bounds = torch.arange(hw + 1, device=dev)[None].expand(Fr, -1).contiguous()
    row_ptr = torch.searchsorted(key_s, bounds)                               # [F, hw+1]
    valid = key_s < hw
    rank = torch.arange(4 * hw, device=dev)[None] - torch.gather(row_ptr, 1, key_s.clamp(max=hw - 1))
    in_ell = valid & (rank < ELL_SLOTS)
    slot = (key_s.clamp(max=hw - 1) * ELL_SLOTS + rank.clamp(0, ELL_SLOTS - 1))
    slot = torch.where(in_ell, slot, torch.zeros_like(slot))                  # slot 0 of row 0 gets +0 for the rest
    ell_src = torch.zeros(Fr, hw * ELL_SLOTS, dtype=torch.int64, device=dev)
    ell_src.scatter_add_(1, slot, torch.where(in_ell, src_s, torch.zeros_like(src_s)))
    ell_w = torch.zeros(Fr, hw * ELL_SLOTS, dtype=torch.float32, device=dev)
    ell_w.scatter_add_(1, slot, torch.where(in_ell, w_s, torch.zeros_like(w_s)))
    packed = ((ell_w * 65535.0).round().long() << 16) | ell_src
    # uint32 payload stored in an int32 tensor (two's complement wrap)
    packed = torch.where(packed >= 2 ** 31, packed - 2 ** 32, packed).to(torch.int32).reshape(Fr, hw, ELL_SLOTS).contiguous()
    over = valid & (rank >= ELL_SLOTS)
    n_ovf = int(over.sum(1).max().item())
    ovf = torch.full((Fr, max(n_ovf, 1), 3), -1, dtype=torch.int32, device=dev)
    if n_ovf > 0:
        for f in range(Fr):
            sel = torch.nonzero(over[f]).reshape(-1)
            ovf[f, :sel.numel(), 0] = key_s[f, sel].to(torch.int32)
            ovf[f, :sel.numel(), 1] = src_s[f, sel].to(torch.int32)
            ovf[f, :sel.numel(), 2] = w_s[f, sel].contiguous().view(torch.int32)
    return {"ell_packed": packed, "ovf": ovf, "n_ovf": n_ovf}


class WarpAdjoint:
    """Per-batch operands of fresco_warp_loss_* for one (backward flow, forward flow) pair (see warp_adjoint_ell)."""

    def __init__(self, bwd: dict, fwd: dict):
        self.bwd, self.fwd = bwd, fwd
        self.n_ovf = max(bwd["n_ovf"], fwd["n_ovf"])
        Fr = bwd["ovf"].shape[0]
        ovf = torch.full((2, Fr, max(self.n_ovf, 1), 3), -1, dtype=torch.int32, device=bwd["ovf"].device)
        ovf[0, :, :bwd["ovf"].shape[1]] = bwd["ovf"]
        ovf[1, :, :fwd["ovf"].shape[1]] = fwd["ovf"]
        self.ovf = ovf.contiguous()


def warp_adjoint_pair(bwd_flow, fwd_flow) -> WarpAdjoint:
    return WarpAdjoint(warp_adjoint_ell(bwd_flow), warp_adjoint_ell(fwd_flow))


class WarpAdjointSlice:
    """Frames [lo, hi) of a :class:`WarpAdjoint` (a frame-sharded batch keeps only its own pairs)."""

    def __init__(self, full: WarpAdjoint, lo: int, hi: int):
        self.bwd = {"ell_packed": full.bwd["ell_packed"][lo:hi].contiguous()}
        self.fwd = {"ell_packed": full.fwd["ell_packed"][lo:hi].contiguous()}
        self.n_ovf = full.n_ovf
        self.ovf = full.ovf[:, lo:hi].contiguous()


def warp_loss_fwd_bwd(cs, fwd_flow, bwd_flow, fwd_keep, bwd_keep, grad, loss_acc=None, accumulate=False,
                      adjoint=None, halo_cs=None, halo_grad=None, total_frames=None):
    """``adjoint`` = :class:`WarpAdjoint` from :func:`warp_adjoint_pair` (cached per batch by the caller).
    ``halo_cs`` / ``halo_grad`` [chunks, C, h, w] fp32 + ``total_frames``: the open-chain form of a frame-sharded batch
    (fresco_warp_loss_fwd_bwd_halo): ``cs`` holds this rank's frames, the per-pair operands its slice."""
    chunks, frames, C, h, w = cs.shape
    if adjoint is None:
        adjoint = warp_adjoint_pair(bwd_flow, fwd_flow)
    a = adjoint
    if (halo_cs is None) != (halo_grad is None):
        raise L.FrescoError("warp_loss_fwd_bwd: halo_cs and halo_grad go together")
    if halo_cs is not None and (tuple(halo_cs.shape) != (chunks, C, h, w) or tuple(halo_grad.shape) != (chunks, C, h, w)
                                or not halo_cs.is_contiguous() or not halo_grad.is_contiguous()):
        raise L.FrescoError("warp_loss_fwd_bwd: halo planes must be contiguous [chunks, C, h, w]")
    if fwd_flow.shape[0] != frames or a.bwd["ell_packed"].shape[0] != frames:
        raise L.FrescoError("warp_loss_fwd_bwd: per-pair operands must have one entry per local frame")
    lp = L.ptr(loss_acc) if loss_acc is not None else None
    ev = _prof_begin()
    L.check(L.lib().fresco_warp_loss_fwd_bwd_halo(
        L.ptr(cs), L.ptr(fwd_flow), L.ptr(bwd_flow), L.ptr(fwd_keep), L.ptr(bwd_keep), L.ptr(a.bwd["ell_packed"]),
        L.ptr(a.fwd["ell_packed"]), L.ptr(a.ovf), int(a.n_ovf), L.ptr(grad), lp, 1 if accumulate else 0, chunks, frames, C, h,
        w, L.ptr(halo_cs) if halo_cs is not None else None, L.ptr(halo_grad) if halo_grad is not None else None,
        int(total_frames) if total_frames is not None else frames, L.stream()), "fresco_warp_loss_fwd_bwd_halo")
    # SURVEY 8d, O2: read c1, c2 + write g1, g2 = 4 fp32 passes (the fused kernels move 2 + 1/N of them)
    _prof_end(ev, "warp_loss_C%d_%dx%d" % (C, h, w), 16.0 * cs.numel(), "hbm")
    return grad


def gram_normalize(cs_bcl: torch.Tensor):
    """cs [B, C, L] fp32 -> xhat [B, L, C] fp16, norms [B, L] fp32."""
    B, C, Lt = cs_bcl.shape
    xhat = torch.empty(B, Lt, C, dtype=torch.float16, device=cs_bcl.device)
    norms = torch.empty(B, Lt, dtype=torch.float32, device=cs_bcl.device)
    ev = _prof_begin()
    L.check(L.lib().fresco_gram_normalize(L.ptr(cs_bcl), L.ptr(xhat), L.ptr(norms), B, C, Lt, L.stream()),
            "fresco_gram_normalize")
    _prof_end(ev, "gram_normalize_C%d_L%d" % (C, Lt), 6.0 * B * C * Lt, "hbm")          # fp32 in, fp16 out
    return xhat, norms


def _gram_scale(weight: float, B: int, Lt: int) -> float:
    """loss scale of the Gram-L1 term, weight / (B * L^2), in double: the launcher rounds it to fp32 once, so a rank's
    share of the weight (intra_weight * n / total) gives the same fp32 scale as the unsharded call"""
    return float(weight) / (B * Lt * Lt)


def gram_sign(xhat, target, weight: float, loss_acc=None):
    B, Lt, C = xhat.shape
    tsign = torch.empty(B, Lt, Lt, dtype=torch.float16, device=xhat.device)
    ev = _prof_begin()
    L.check(L.lib().fresco_gram_sign_scaled(L.ptr(xhat), L.ptr(target), L.ptr(tsign),
                                            L.ptr(loss_acc) if loss_acc is not None else None, B, Lt, C,
                                            _gram_scale(weight, B, Lt), L.stream()), "fresco_gram_sign_scaled")
    _prof_end(ev, "gram_sign_C%d_L%d" % (C, Lt), 2.0 * B * Lt * Lt * C, "tensor")       # SURVEY 8d: forward Gram
    return tsign


def gram_sign_ref(xhat, yhat, weight: float, loss_acc=None):
    """T = 2 sign(xhat xhat^T - yhat yhat^T) with the target recomputed in the kernel from the normalised reference
    features yhat [B, L, C] fp16 (no [B, L, L] fp32 target)."""
    B, Lt, C = xhat.shape
    tsign = torch.empty(B, Lt, Lt, dtype=torch.float16, device=xhat.device)
    ev = _prof_begin()
    L.check(L.lib().fresco_gram_sign_ref_scaled(L.ptr(xhat), L.ptr(yhat), L.ptr(tsign),
                                                L.ptr(loss_acc) if loss_acc is not None else None, B, Lt, C,
                                                _gram_scale(weight, B, Lt), L.stream()), "fresco_gram_sign_ref_scaled")
    _prof_end(ev, "gram_sign_C%d_L%d" % (C, Lt), 2.0 * B * Lt * Lt * C, "tensor")       # SURVEY 8d: forward Gram
    return tsign


def gram_grad(tsign, xhat, norms, grad_bcl, weight: float):
    B, Lt, C = xhat.shape
    nbytes = int(L.lib().fresco_gram_grad_workspace_bytes(B, Lt, C))
    ws = _workspace(("gram_grad", xhat.device), max(nbytes, 16), xhat.device)
    ev = _prof_begin()
    L.check(L.lib().fresco_gram_grad_scaled(L.ptr(tsign), L.ptr(xhat), L.ptr(norms), L.ptr(grad_bcl), B, Lt, C,
                                            _gram_scale(weight, B, Lt), L.ptr(ws), nbytes, L.stream()),
            "fresco_gram_grad_scaled")
    _prof_end(ev, "gram_grad_C%d_L%d" % (C, Lt), 4.0 * B * Lt * Lt * C, "tensor")       # SURVEY 8d: the two backward products
    return grad_bcl


def adam_step(param, grad, exp_avg, exp_avg_sq, step: int, lr=0.2, beta1=0.9, beta2=0.999, eps=1e-8):
    ev = _prof_begin()
    L.check(L.lib().fresco_adam_step(L.ptr(param), L.ptr(grad), L.ptr(exp_avg), L.ptr(exp_avg_sq), param.numel(),
                                     int(step), lr, beta1, beta2, eps, L.stream()), "fresco_adam_step")
    _prof_end(ev, "adam_n%d" % param.numel(), 28.0 * param.numel(), "hbm")               # read p, g, m, v; write p, m, v


def adain(content_f32: torch.Tensor, style: torch.Tensor) -> torch.Tensor:
    n, c, h, w = style.shape
    out = torch.empty_like(style)
    is_half = 1 if style.dtype == torch.float16 else 0
    if not is_half and style.dtype != torch.float32:
        raise L.FrescoError("adain: fp16 or fp32 style only")
    ev = _prof_begin()
    L.check(L.lib().fresco_adain(L.ptr(content_f32), L.ptr(style), L.ptr(out), is_half, n * c, h * w, L.stream()),
            "fresco_adain")
    _prof_end(ev, "adain_C%d_%dx%d" % (c, h, w), style.numel() * (4.0 + 2 * style.element_size()), "hbm")
    return out


def gmflow_global_corr_softmax(f0: torch.Tensor, f1: torch.Tensor, bidir: bool):
    b, c, h, w = f0.shape
    flow = torch.empty(b * (2 if bidir else 1), 2, h, w, dtype=torch.float32, device=f0.device)
    nbytes = int(L.lib().fresco_gmflow_corr_workspace_bytes(b, c, h, w))
    ws = _workspace(("gmflow", f0.device), max(nbytes, 16), f0.device)
    ev = _prof_begin()
    L.check(L.lib().gmflow_global_corr_softmax(L.ptr(f0), L.ptr(f1), L.ptr(flow), b, c, h, w, 1 if bidir else 0,
                                               L.ptr(ws), nbytes, L.stream()), "gmflow_global_corr_softmax")
    Lt = h * w
    _prof_end(ev, "gmflow_corr_C%d_L%d" % (c, Lt), 2.0 * b * Lt * Lt * c + 2.0 * (2 * b) * Lt * Lt * 2, "tensor")   # SURVEY 8d, G1
    return flow


def gmflow_flow_attention(q: torch.Tensor, k: torch.Tensor, values: torch.Tensor, softmax_scale: float):
    """q, k fp16 [B, L, C]; values fp32 [B, L, 2] -> fp32 [B, 2, L] = softmax(q k^T * scale) values."""
    B, Lt, C = q.shape
    out = torch.empty(B, 2, Lt, dtype=torch.float32, device=q.device)
    ev = _prof_begin()
    L.check(L.lib().gmflow_flow_attention(L.ptr(q), L.ptr(k), L.ptr(values), L.ptr(out), B, Lt, C, float(softmax_scale),
                                          L.stream()), "gmflow_flow_attention")
    _prof_end(ev, "gmflow_flow_attn_C%d_L%d" % (C, Lt), 2.0 * B * Lt * Lt * C + 2.0 * B * Lt * Lt * 2, "tensor")
    return out


def dilate(x: torch.Tensor, k: int) -> torch.Tensor:
    """fp32 [..., h, w] masks -> k x k dilation with replicate padding (src/utils.py:81-93)."""
    h, w = x.shape[-2], x.shape[-1]
    out = torch.empty_like(x)
    L.check(L.lib().fresco_dilate(L.ptr(x), L.ptr(out), x.numel() // (h * w), h, w, int(k), L.stream()), "fresco_dilate")
    return out


def cfg_pred_x0(noise_pred_2n: torch.Tensor, sample: torch.Tensor, guidance_scale: float, alpha_prod_t: float,
                do_cfg: bool = True) -> torch.Tensor:
    """noise_pred [2N, ...] (uncond | text chunks, or [N, ...] when do_cfg is False), sample [N, ...] -> predicted x0."""
    n = sample.numel()
    x0 = torch.empty_like(sample)
    is_half = 1 if sample.dtype == torch.float16 else 0
    base = L.ptr(noise_pred_2n)
    text = base + n * sample.element_size() if do_cfg else None
    L.check(L.lib().fresco_cfg_pred_x0(base, text, L.ptr(sample), L.ptr(x0), is_half, n, float(guidance_scale),
                                       float(alpha_prod_t), L.stream()), "fresco_cfg_pred_x0")
    return x0


def ddpm_prev(x0, sample, noise, c_x0: float, c_xt: float, sigma: float, repeat_noise: bool = False):
    prev = torch.empty_like(sample)
    is_half = 1 if sample.dtype == torch.float16 else 0
    per_frame = sample[0].numel()
    L.check(L.lib().fresco_ddpm_prev(L.ptr(x0), L.ptr(sample), L.ptr(noise), L.ptr(prev), is_half, sample.numel(),
                                     per_frame, 1 if repeat_noise else 0, float(c_x0), float(c_xt), float(sigma),
                                     L.stream()), "fresco_ddpm_prev")
    return prev


def mapping_single(bwd_flow: torch.Tensor, bwd_occ: torch.Tensor, imgs: torch.Tensor, scale: int):
    """bwd_flow [1,2,H,W], bwd_occ [1,H,W], imgs [2,3,H,W] fp32 -> mapping int64 [L], unlinked bool [L]."""
    H, W = imgs.shape[2], imgs.shape[3]
    Lt = (H // scale) * (W // scale)
    mapping = torch.empty(Lt, dtype=torch.int64, device=imgs.device)
    unlinked = torch.empty(Lt, dtype=torch.uint8, device=imgs.device)
    nbytes = int(L.lib().fresco_mapping_workspace_bytes(Lt))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=imgs.device)
    L.check(L.lib().fresco_mapping_single(L.ptr(bwd_flow), L.ptr(bwd_occ), L.ptr(imgs), H, W, int(scale),
                                          L.ptr(mapping), L.ptr(unlinked), L.ptr(ws), nbytes, L.stream()),
            "fresco_mapping_single")
    return mapping, unlinked.bool()


# ---- B1: propagation-stage frame blending (include/fresco_b200.h) ----

def _check_blend(what, **named):
    """Refuse, before any launch, operands the blend kernels would reinterpret: each entry is name -> (tensor, dtype,
    shape), with None in the shape for a free dimension."""
    for name, (t, dtype, shape) in named.items():
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise L.FrescoError(f"{what}: {name} must be a CUDA tensor")
        if t.dtype != dtype:
            raise L.FrescoError(f"{what}: {name} must be {dtype}, got {t.dtype}")
        if t.dim() != len(shape) or any(s is not None and s != d for s, d in zip(shape, t.shape)):
            raise L.FrescoError(f"{what}: {name} must have shape {list(shape)}, got {list(t.shape)}")
        if not t.is_contiguous():
            raise L.FrescoError(f"{what}: {name} must be contiguous")


def blend_lut_gather(img: torch.Tensor, lut: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """uint8 [..., 3] colour triples -> lut[triple] (lut uint8 [2^24, 3], cv2's conversion of every triple)."""
    if img.dim() < 1:
        raise L.FrescoError("blend_lut_gather: img must be uint8 [..., 3]")
    _check_blend("blend_lut_gather", img=(img, torch.uint8, (None,) * (img.dim() - 1) + (3,)),
                 lut=(lut, torch.uint8, (1 << 24, 3)))
    if out is None:
        out = torch.empty_like(img)
    _check_blend("blend_lut_gather", out=(out, torch.uint8, tuple(img.shape)))
    n = img.numel() // 3
    if n:
        ev = _prof_begin()
        L.check(L.lib().fresco_blend_lut_gather(L.ptr(img), L.ptr(lut), L.ptr(out), n, L.stream()),
                "fresco_blend_lut_gather")
        _prof_end(ev, "blend_lut_gather", 9.0 * n, "hbm")      # 3 bytes in, 3 gathered, 3 out per pixel
    return out


def blend_mask_chain(dist1: torch.Tensor, dist2: torch.Tensor, flows: torch.Tensor,
                     out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Error masks of one sequence, each OR'd with the previous one warped by its backward flow.  dist1, dist2 fp32
    [interval-1, h, w]; flows fp32 [interval-1, 2, h, w] (flow 0 unused) -> uint8 [interval-1, h, w] in {0, 1}."""
    if dist1.dim() != 3:
        raise L.FrescoError("blend_mask_chain: dist1 must be fp32 [interval-1, h, w]")
    F_, h, w = dist1.shape
    _check_blend("blend_mask_chain", dist1=(dist1, torch.float32, (F_, h, w)), dist2=(dist2, torch.float32, (F_, h, w)),
                 flows=(flows, torch.float32, (F_, 2, h, w)))
    if out is None:
        out = torch.empty(F_, h, w, dtype=torch.uint8, device=dist1.device)
    _check_blend("blend_mask_chain", out=(out, torch.uint8, (F_, h, w)))
    ev = _prof_begin()
    L.check(L.lib().fresco_blend_mask_chain(L.ptr(dist1), L.ptr(dist2), L.ptr(flows), L.ptr(out), F_ + 1, h, w,
                                            L.stream()), "fresco_blend_mask_chain")
    _prof_end(ev, "blend_mask_chain_%dx%d" % (h, w), 17.0 * F_ * h * w, "hbm")    # 2 dists, flow, mask in, mask out
    return out


def _blend_workspace(frames: int, h: int, w: int, device) -> torch.Tensor:
    nbytes = int(L.lib().fresco_blend_workspace_bytes(frames, h, w))
    return _workspace(("blend", device), nbytes, device)


def blend_histogram(lab_a: torch.Tensor, lab_b: torch.Tensor, weights: torch.Tensor,
                    lab_min_error: Optional[torch.Tensor] = None, masks: Optional[torch.Tensor] = None,
                    out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """blender/histogram_blend.blend in Lab, before its Lab -> BGR: lab_a, lab_b uint8 [F, h, w, 3]; weights fp64
    [F, 2] (blend's weight1, weight2); the min-error image either given (uint8 [F, h, w, 3]) or selected from a (mask 0)
    and b (mask 1) by masks uint8 [F, h, w]."""
    if lab_a.dim() != 4:
        raise L.FrescoError("blend_histogram: lab_a must be uint8 [frames, h, w, 3]")
    F_, h, w, _ = lab_a.shape
    img = (F_, h, w, 3)
    args = dict(lab_a=(lab_a, torch.uint8, img), lab_b=(lab_b, torch.uint8, img),
                weights=(weights, torch.float64, (F_, 2)))
    if (lab_min_error is None) == (masks is None):
        raise L.FrescoError("blend_histogram: pass exactly one of lab_min_error and masks")
    if lab_min_error is not None:
        args["lab_min_error"] = (lab_min_error, torch.uint8, img)
    else:
        args["masks"] = (masks, torch.uint8, (F_, h, w))
    _check_blend("blend_histogram", **args)
    if out is None:
        out = torch.empty_like(lab_a)
    _check_blend("blend_histogram", out=(out, torch.uint8, img))
    ws = _blend_workspace(F_, h, w, lab_a.device)
    ev = _prof_begin()
    L.check(L.lib().fresco_blend_histogram(
        L.ptr(lab_a), L.ptr(lab_b), L.ptr(lab_min_error) if lab_min_error is not None else None,
        L.ptr(masks) if masks is not None else None, L.ptr(weights), L.ptr(out), F_, h, w, L.ptr(ws), ws.numel(),
        L.stream()), "fresco_blend_histogram")
    _prof_end(ev, "blend_histogram_%dx%d" % (h, w), 34.0 * F_ * h * w, "hbm")    # 4 passes over a, b, mask + the output
    return out


def blend_cheby_iterations(h: int, w: int, weight: float) -> int:
    """Chebyshev steps fresco_blend_poisson runs for one channel (oracle/blend_bound.py derives the count)."""
    return int(L.lib().fresco_blend_cheby_iterations(int(h), int(w), float(weight)))


def blend_poisson(lab_target: torch.Tensor, lab_a: torch.Tensor, lab_b: torch.Tensor, masks: torch.Tensor,
                  grad_weight=(2.5, 0.5, 0.5), out: Optional[torch.Tensor] = None,
                  solution: Optional[torch.Tensor] = None) -> torch.Tensor:
    """blender/poisson_fusion.poisson_fusion in Lab, before its Lab -> BGR: the exact least-squares solution per
    channel, clipped to [0, 255] and truncated.  Images uint8 [F, h, w, 3], masks uint8 [F, h, w]; ``solution`` fp64
    [F, 3, h, w], if given, receives the unclipped solution."""
    if lab_target.dim() != 4:
        raise L.FrescoError("blend_poisson: lab_target must be uint8 [frames, h, w, 3]")
    F_, h, w, _ = lab_target.shape
    img = (F_, h, w, 3)
    _check_blend("blend_poisson", lab_target=(lab_target, torch.uint8, img), lab_a=(lab_a, torch.uint8, img),
                 lab_b=(lab_b, torch.uint8, img), masks=(masks, torch.uint8, (F_, h, w)))
    gw = [float(x) for x in grad_weight]
    if len(gw) != 3:
        raise L.FrescoError("blend_poisson: grad_weight must have one weight per channel")
    if out is None:
        out = torch.empty_like(lab_target)
    _check_blend("blend_poisson", out=(out, torch.uint8, img))
    if solution is not None:
        _check_blend("blend_poisson", solution=(solution, torch.float64, (F_, 3, h, w)))
    ws = _blend_workspace(F_, h, w, lab_target.device)
    ev = _prof_begin()
    L.check(L.lib().fresco_blend_poisson(L.ptr(lab_target), L.ptr(lab_a), L.ptr(lab_b), L.ptr(masks), gw[0], gw[1],
                                         gw[2], L.ptr(out), L.ptr(solution) if solution is not None else None, F_, h,
                                         w, L.ptr(ws), ws.numel(), L.stream()), "fresco_blend_poisson")
    if ev is not None:
        # every Chebyshev step reads the iterate (5-point, cached), the previous iterate and b, and writes one plane
        iters = sum(blend_cheby_iterations(h, w, x) for x in gw)
        _prof_end(ev, "blend_poisson_%dx%d" % (h, w), 32.0 * F_ * h * w * iters, "hbm")
    return out
