"""TEST / BENCH INFRASTRUCTURE ONLY -- the reference's math in PyTorch eager ON THE GPU.

bench.py's ``gpu_eager_baseline`` leg: what the reference itself executes on a CUDA device (SURVEY 8d: "time the
reference on the same GPU in PyTorch eager -- that, not the CPU number, is the >= 10x bar"), restated with the same
torch calls the reference makes (F.scaled_dot_product_attention, boolean-mask indexing + repeat, torch.gather,
F.grid_sample, fp32 bmm, autograd + torch.optim.Adam), fp16 activations for attention as shipped
(run_fresco.py:75-76), fp32 inside optimize_feature (diffusion_hacked.py:430).  Never imported by the product path.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from . import fresco_oracle as O


@torch.no_grad()
def fresco_layer(x, wq, wk, wv, wo, bo, heads, attn_mask, ref_hidden, fwd_map, bwd_map, inter_mask, chunks=2,
                 use_intra=True, use_inter=True, intra_scale=0.2, inter_scale=0.2, intra_bias=0.0):
    """One FRESCO self-attention layer as FRESCOAttnProcessor2_0.__call__ runs it (diffusion_hacked.py:169-387).
    x, ref_hidden [2N, L, C]; attn_mask bool [N, L]; fwd_map / bwd_map int64 [N, 1, L]; inter_mask bool [L, 1, N, N]."""
    B, L, C = x.shape
    N = B // chunks
    d = C // heads
    q = x @ wq.t()                                                              # :201-215
    k = x @ wk.t()
    v = x @ wv.t()
    q_raw, k_raw = q.clone(), k.clone()                                         # :218-219
    # cross-frame K/V: boolean-mask indexing on [b, f, L, C], then the N x broadcast is MATERIALISED (:234-247)
    k = k.view(chunks, N, L, C)[:, attn_mask]
    v = v.view(chunks, N, L, C)[:, attn_mask]
    k = k[:, None].repeat(1, N, 1, 1).reshape(B, -1, C)
    v = v[:, None].repeat(1, N, 1, 1).reshape(B, -1, C)

    def split(t):
        return t.view(t.shape[0], -1, heads, d).transpose(1, 2)

    qh = split(q)
    if use_intra:                                                               # :257-288, dense [L, L] mask tensor
        q_ = split(ref_hidden @ wq.t())
        k_ = split(ref_hidden @ wk.t()) * intra_scale
        dense = torch.eye(L, dtype=x.dtype, device=x.device) * intra_bias
        qh = F.scaled_dot_product_attention(q_, k_, qh, attn_mask=dense)
    a = F.scaled_dot_product_attention(qh, split(k), split(v))                  # :303-305
    if use_inter:                                                               # :309-367
        pos = fwd_map[:, 0]
        gi = pos[None, :, :, None].expand(chunks, N, L, C)
        a_tok = a.transpose(1, 2).reshape(chunks, N, L, C)
        qt = torch.gather(q_raw.view(chunks, N, L, C), 2, gi)
        kt = torch.gather(k_raw.view(chunks, N, L, C), 2, gi) * inter_scale
        vt = torch.gather(a_tok, 2, gi)

        def traj(t):                                                            # -> [(b L), heads, N, d]
            return t.view(chunks, N, L, heads, d).permute(0, 2, 3, 1, 4).reshape(chunks * L, heads, N, d)

        m = inter_mask.repeat(chunks, 1, 1, 1)                                  # [2L, 1, N, N]
        o = F.scaled_dot_product_attention(traj(qt), traj(kt), traj(vt), attn_mask=m)
        o = o.view(chunks, L, heads, N, d).permute(0, 3, 1, 2, 4).reshape(chunks, N, L, C)
        bi = bwd_map[:, 0][None, :, :, None].expand(chunks, N, L, C)
        a = torch.gather(o, 2, bi).reshape(B, L, heads, d).transpose(1, 2)
    return a.transpose(1, 2).reshape(B, L, C) @ wo.t() + bo                     # :371-377


def optimize_feature(sample, flows, occs, target, intra_weight=1e2, iters=20, chunks=2):
    """diffusion_hacked.py:416-488 as written there: cs = Parameter, torch.optim.Adam(lr=0.2), closure with the
    temporal L1 loss through F.grid_sample and the normalised-Gram L1 loss through fp32 bmm, autograd backward."""
    n = sample.shape[0] // chunks
    _, C, h, w = sample.shape
    latent = sample.to(torch.float32).reshape(chunks, n, C, h, w)
    cs = torch.nn.Parameter(latent.detach().clone())
    opt = torch.optim.Adam([cs], lr=0.2)
    scale = h * 1.0 / flows[0].shape[2]
    ff, bf, fo, bo = O._resize_flow_occ(flows, occs, scale)
    ff, bf = ff.repeat(chunks, 1, 1, 1), bf.repeat(chunks, 1, 1, 1)
    mf, mb = 1 - fo.repeat(chunks, 1, 1, 1), 1 - bo.repeat(chunks, 1, 1, 1)
    resh = list(range(1, n)) + [0]

    def closure():
        opt.zero_grad()
        c1 = cs.reshape(chunks * n, C, h, w)
        c2 = cs[:, resh].reshape(chunks * n, C, h, w)
        loss = ((c2 - O.flow_warp(c1, bf)).abs() * mb + (c1 - O.flow_warp(c2, ff)).abs() * mf).mean() * 2
        X = cs.reshape(chunks * n, C, h * w).transpose(1, 2)
        X = X / ((X ** 2).sum(dim=2, keepdim=True) ** 0.5)
        loss = loss + F.l1_loss(torch.bmm(X, X.transpose(-1, -2)), target) * intra_weight
        loss.backward()
        return loss

    for _ in range(iters):
        opt.step(closure)
    with torch.no_grad():
        return O.adain(cs.data.to(sample.dtype).reshape(chunks * n, C, h, w), sample)


@torch.no_grad()
def warp_tensor(sample, flows, occs, saliency, chunks):
    """src/flow_utils.py:18-53: 2N sequential grid_sample launches of one frame each."""
    return O.warp_tensor(sample, flows, occs, saliency, chunks)
