"""Drop-ins for the attention functions of GMFlow's transformer (``gmflow/transformer.py``), SURVEY 8(f)-1:

* ``single_head_full_attention(q, k, v)``                       (:8-17)
* ``single_head_split_window_attention(q, k, v, num_splits, with_shift, h, w, attn_mask)``   (:46-105) -- the 12 Swin
  attentions of the feature transformer (6 blocks x self / cross; 2 x 2 windows of 32 x 32 tokens at 512 x 512, C = 128)
* ``feature_flow_attention(module, feature0, flow)``            (:353-374) -- flow propagation, V = the 2-channel flow

All three run on the wgmma attention kernel of libfresco_b200.so (head_dim = C, one head, fp16 operands / fp32
softmax; SURVEY 9 measured fp16 operands adequate for GMFlow's LayerNorm-scale features).  The shifted-window variant
does not add the reference's -100 mask to a dense score matrix: a masked pair contributes exp(-100) ~ 4e-44 of its row,
i.e. nothing in fp32, so each window is split into the (up to four) regions inside which tokens may attend each other,
the tokens of every region are gathered into a contiguous block (fresco_rows_gather), blocks of equal size share one
launch, and the result rows are scattered back.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch

from . import ops
from ._lib import FrescoError

_PLANS: Dict[tuple, List[Tuple[int, torch.Tensor]]] = {}


def _window_blocks(h: int, w: int, num_splits: int, with_shift: bool, device) -> List[Tuple[int, torch.Tensor]]:
    """[(tokens per block, int64 [n_blocks, tokens] original token indices)]: the blocks inside which attention is
    allowed -- whole windows without shift; with shift the windows of the rolled grid cut along the wrap-around seams
    (generate_shift_window_attn_mask, gmflow/transformer.py:20-43)."""
    key = (h, w, num_splits, bool(with_shift), str(device))
    if key in _PLANS:
        return _PLANS[key]
    wh, ww = h // num_splits, w // num_splits
    sh, sw = (wh // 2, ww // 2) if with_shift else (0, 0)
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")           # coordinates of the ROLLED grid
    orig = ((ys + sh) % h) * w + ((xs + sw) % w)                                         # token that sits there after the roll
    win = (ys // wh) * num_splits + (xs // ww)
    if with_shift:
        rc = (ys >= h - wh).long() + (ys >= h - sh).long()
        cc = (xs >= w - ww).long() + (xs >= w - sw).long()
        region = rc * 3 + cc
    else:
        region = torch.zeros_like(win)
    block = (win * 9 + region).reshape(-1)
    order = torch.argsort(block, stable=True)                                           # row-major inside a block
    ids, counts = torch.unique_consecutive(block[order], return_counts=True)
    plans: Dict[int, List[torch.Tensor]] = {}
    start = 0
    for cnt in counts.tolist():
        plans.setdefault(cnt, []).append(orig.reshape(-1)[order[start:start + cnt]])
        start += cnt
    out = [(cnt, torch.stack(v).to(device)) for cnt, v in sorted(plans.items(), reverse=True)]
    _PLANS[key] = out
    return out


def _attend(q16, k16, v16, scale):
    return ops.attn_fwd(q16, k16, v16, heads=1, q_per_kv=1, softmax_scale=scale)


def _check(q, k, v):
    if not (q.dim() == k.dim() == v.dim() == 3):
        raise FrescoError("GMFlow attention: q, k, v must be [B, L, C]")
    c = q.shape[2]
    if c not in (64, 128):
        raise FrescoError("GMFlow attention: feature width %d is not built (64 / 128)" % c)
    return c


@torch.no_grad()
def single_head_full_attention(q, k, v):
    c = _check(q, k, v)
    out = _attend(q.half().contiguous(), k.half().contiguous(), v.half().contiguous(), 1.0 / math.sqrt(c))
    return out.to(q.dtype)


@torch.no_grad()
def single_head_split_window_attention(q, k, v, num_splits=1, with_shift=False, h=None, w=None, attn_mask=None):
    c = _check(q, k, v)
    assert h is not None and w is not None and q.shape[1] == h * w
    b, L, _ = q.shape
    scale = 1.0 / math.sqrt(c)
    q16, k16, v16 = (t.half().contiguous().view(b * L, c) for t in (q, k, v))
    out16 = torch.empty(b * L, c, dtype=torch.float16, device=q.device)
    boff = (torch.arange(b, device=q.device) * L)[:, None, None]
    for cnt, idx in _window_blocks(h, w, num_splits, with_shift, q.device):
        rows = (idx[None] + boff).reshape(-1).to(torch.int32)                          # [b * n_blocks * cnt]
        n = rows.numel()
        gq, gk, gv = (torch.empty(n, c, dtype=torch.float16, device=q.device) for _ in range(3))
        ops.rows_gather(q16, rows, gq)
        ops.rows_gather(k16, rows, gk)
        ops.rows_gather(v16, rows, gv)
        o = _attend(gq.view(-1, cnt, c), gk.view(-1, cnt, c), gv.view(-1, cnt, c), scale)
        ops.rows_scatter(o.view(n, c), rows, out16)
    return out16.view(b, L, c).to(q.dtype)


@torch.no_grad()
def feature_flow_attention(module, feature0, flow, local_window_attn=False, local_window_radius=1, **kwargs):
    """FeatureFlowAttention.forward (gmflow/transformer.py:343-374) with ``module`` the reference layer (its q_proj /
    k_proj weights).  The local-window variant (:376-413, not used by FRESCO's call: prop_radius_list=[-1]) is left
    to the reference implementation."""
    if local_window_attn:
        return module.forward_local_window_attn(feature0, flow, local_window_radius=local_window_radius)
    b, c, h, w = feature0.shape
    query = module.q_proj(feature0.view(b, c, h * w).permute(0, 2, 1))
    key = module.k_proj(query)                                       # (sic: the reference projects the projected query)
    values = flow.view(b, flow.size(1), h * w).permute(0, 2, 1).float().contiguous()
    if values.shape[2] != 2:
        raise FrescoError("flow attention: V must have 2 channels")
    out = ops.gmflow_flow_attention(query.half().contiguous(), key.half().contiguous(), values, 1.0 / math.sqrt(c))
    return out.view(b, 2, h, w).to(flow.dtype)
