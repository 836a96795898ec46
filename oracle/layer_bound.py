"""fp64 staged reference of one FRESCO self-attention layer (``FRESCOAttnProcessor2_0._fresco_self_attention`` and
``ShardedFRESCOAttention.__call__``), an elementwise bound composed from the bounds of the kernels it chains, and layer
input families built to break the glue between them.

CHECKER ONLY (see ``oracle/__init__``).  Written from the reference's description of the layer (src/diffusion_hacked.py
:225-367), not from the product's host code: it works on the layer's operands q, k, v and, under spatial guidance,
q_ref, k_ref = the projections of the stored reference features, [chunks*N, L, H*d] in (chunk, frame) order, in any
dtype (the kernels' operands are fp16; the golden fixtures' fp32 projections are evaluated in fp64 as they are).

The stages
----------
1. spatial-guided (``use_intra``): y1 = softmax(fp32(s_intra / sqrt(d)) q_ref k_ref^T + fp32(bias) [i == j]) q per frame;
   y1 replaces the query.
2. cross-frame (``use_cf``): the mask with ``shape[1] == L`` (the last such in the list) selects rows of the (frame,
   token) row-major plane of k and v per chunk; without one, every frame attends frame 0 of its chunk.  y2 =
   softmax(fp32(1 / sqrt(d)) q2 k_sel^T) v_sel for every frame of the chunk (``q_per_kv = N``).  Without ``use_cf``
   each frame attends its own k, v.
3. temporal-guided (``use_inter``): along every trajectory p of the mapping with ``shape[2] == L`` (token fwd[f, p] of
   frame f), y3 = softmax_g(fp32(s_inter / sqrt(d)) q_f k_g, masked by mask[p, f, g]) y2_g with q, k the RAW projections,
   scattered back to token fwd[f, p] (``temporal_bound.gather`` / ``scatter``).
4. ``to_out[0]`` (optional): y = a W_o^T + b_o.

Every stage can be evaluated on a subset of the query rows (``sample``): a sample of trajectories under temporal
guidance (all frames' rows of each), of tokens otherwise.  The fp64 work is blocked so that no intermediate exceeds
``BUDGET`` bytes; a full [16, 8, 4096, 15587] logit tensor would take 65 GB.

The composed bound
------------------
Each stage's kernel is held to its own bound (``attention_bound`` with the variant's poly / rowsum, ``temporal_bound``
with kernel "rows" for N <= 16 and "round1" beyond), evaluated on the operands that kernel actually received (the fp16
output of the stage before; ``received``), plus a term for the error it inherits:

* Stage 1 inherits nothing (its operands are the projections).  E1 = its own bound.
* Stage 2 inherits the query error |q2^ - y1| <= E1.  For row i, every logit moves by at most
  Delta_i = fp32(scale) max_j sum_c E1_ic |k_jc|, so every weight moves by a factor in [e^-2Delta, e^2Delta]
  (numerator e^delta_j, denominator a convex combination of e^delta), and with sum_j (w'_ij - w_ij) = 0

      |y2(q2^) - y2(y1)|_ic = |sum_j (w'_ij - w_ij)(v_jc - y_ic)| <= (e^(2 Delta_i) - 1) sum_j w_ij |v_jc - y_ic|

  with w and y those of the reference.  Exact, not first order.  E2 = own bound at q2^ + this term.
* Stage 3 inherits the V error |V^ - y2| <= E2 (q and k are the raw projections, exact).  The weights are convex, so
  |y3(V^) - y3(y2)| <= sum_g w_g E2_g along the trajectory -- the temporal reference with V = E2.
  E3 = own bound at V^ + this term.
* ``to_out[0]`` in fp32 with TF32 off, on a = the fp16 attention result cast to fp32:
  |W_o| E3 + F (C + 1) u (|W_o| |a| + |b_o|), C products and the bias add each rounding once (u = 2^-24).

F = 2 (``SAFETY``) as in the other modules; nothing else is widened.  Without stage 1, stage 2 receives the raw q and
inherits nothing; without stage 3 the layer's attention result is stage 2's.

Exact answers
-------------
The ``exact`` family makes every stage one-hot (the hot key >= 45 nats above every other, which therefore flush to
zero in fp16 P) and every trajectory self-only, so the layer output is a copy of rows of V.  V's channels 0, 1, 2 of
every head encode (chunk, frame, token) and the head as exact fp16 integers, so a misrouted row names itself.
"""
from __future__ import annotations

import math
from typing import Dict, List, NamedTuple, Optional

import numpy as np
import torch
import torch.nn.functional as F

from . import attention_bound as AB
from . import temporal_bound as TB

U = 2.0 ** -24
SAFETY = 2.0
BUDGET = 2 * 1024 ** 3             # bytes of fp64 intermediates per block
MUTANTS = {                        # glue mutant -> (family, mode flags) that separate it from the layer
    "spatial-scale-without-0.2": ("realistic", 3),
    "temporal-q-from-q-main": ("temporal-dominant", 6),
    "temporal-k-without-scale": ("realistic", 5),
    "scatter-through-bwd-map": ("exact", 7),
    "chunk1-reads-chunk0-kv": ("exact", 7),
    "own-frame-kv": ("exact", 7),
    "mask-of-other-resolution": ("mask-multi", 7),
    "heads-split-d-h": ("realistic", 7),
    "transposed-trajectory-mask": ("temporal-huge", 7),
    "diag-bias-dropped": ("diag-bias", 7),
}


def _f32(x: float) -> float:
    return float(np.float32(x))


class Operands(NamedTuple):
    q: torch.Tensor                  # [chunks*N, L, C]
    k: torch.Tensor
    v: torch.Tensor
    q_ref: Optional[torch.Tensor]    # projections of the stored reference features (spatial guidance) or None
    k_ref: Optional[torch.Tensor]
    heads: int
    chunks: int


class Control(NamedTuple):
    """What ``AttentionControl`` holds for one keyframe batch."""
    use_cf: bool
    use_intra: bool
    use_inter: bool
    masks: Optional[List[torch.Tensor]] = None          # bool [N, L_s] per resolution
    fwd_maps: Optional[List[torch.Tensor]] = None       # int64 [N, 1, L_s]
    bwd_maps: Optional[List[torch.Tensor]] = None
    inter_masks: Optional[List[torch.Tensor]] = None    # bool [L_s, 1, N, N]
    intra_scale: float = 0.2
    intra_bias: float = 0.0
    inter_scale: float = 0.2

    def modes(self, flags: int) -> "Control":
        """bit 0 cross-frame, bit 1 spatial-guided, bit 2 temporal-guided (the golden fixtures' ``out_{flags}``)"""
        return self._replace(use_cf=bool(flags & 1), use_intra=bool(flags & 2), use_inter=bool(flags & 4))


# ============================================================================================== host-side selections
def kv_rows(ctl: Control, N: int, L: int, mutant=None) -> Optional[torch.Tensor]:
    """(frame, token) row-major indices of the K/V rows the mask for L tokens selects; None: no mask, frame 0."""
    if not ctl.masks:
        return None
    hits = [i for i, m in enumerate(ctl.masks) if m.shape[1] == L]
    if not hits:
        return None
    i = hits[-1]
    if mutant == "mask-of-other-resolution":
        i = (i + 1) % len(ctl.masks)
        return torch.nonzero(ctl.masks[i].reshape(-1).cpu()).reshape(-1) % (N * L)
    return torch.nonzero(ctl.masks[i].reshape(-1).cpu()).reshape(-1)


def trajectories(ctl: Control, L: int):
    """(fwd [N, L], bwd [N, L], mask bool [L, N, N]) of the mapping for L tokens, or None."""
    found = None
    for i, f in enumerate(ctl.fwd_maps or []):
        if f.shape[2] == L:
            found = (f[:, 0].cpu().long(), ctl.bwd_maps[i][:, 0].cpu().long(), ctl.inter_masks[i][:, 0].cpu().bool())
    return found


def sample_rows(ctl: Control, B: int, N: int, L: int, sample=None) -> torch.Tensor:
    """int64 [B, R]: the token of each evaluated row of every batch element.  Under temporal guidance ``sample`` lists
    trajectories (row i of frame f is token fwd[f, sample[i]]), otherwise tokens; None: all of them."""
    P = torch.arange(L) if sample is None else torch.as_tensor(sample).long().cpu()
    if ctl.use_inter:
        tr = trajectories(ctl, L)
        if tr is None:
            raise ValueError(f"temporal-guided attention enabled but no mapping matches {L} tokens")
        fr = torch.arange(B) % N
        return tr[0][fr][:, P]
    return P[None].expand(B, -1).contiguous()


def _take(t, rows):
    """t [B, L, C] at rows [B, R] -> [B, R, C]"""
    return torch.gather(t, 1, rows.to(t.device)[..., None].expand(-1, -1, t.shape[-1]))


def to_tokens(t: torch.Tensor, rows: torch.Tensor, L: int) -> torch.Tensor:
    """[B, R, C] in the sample layout -> [B, L, C] (NaN where no row was evaluated)"""
    out = torch.full((t.shape[0], L, t.shape[2]), float("nan"), dtype=t.dtype, device=t.device)
    out.scatter_(1, rows.to(t.device)[..., None].expand(-1, -1, t.shape[-1]), t)
    return out


def _heads_perm(C, heads):
    """channel h*d + j of the [H, d] split <- channel j*H + h of the [d, H] one"""
    d = C // heads
    return (torch.arange(d)[None, :] * heads + torch.arange(heads)[:, None]).reshape(-1)


# ============================================================================================== per-stage math
def _block(heads, Lk, d=1):
    return max(1, int(BUDGET // (8 * 6 * heads * max(Lk, 1) * d)))


def _attn_rows(q, k, v, rows, kv_of, heads, scale, bias, poly, rowsum):
    """(ref, tol) fp64 [B, R, C] of attention for the query rows ``rows`` [B, R] of q [B, L, C] against k / v batch
    kv_of[b]; the diagonal bias follows the absolute row index.  rows None: q holds the rows already [B, R, C]."""
    if rows is None:
        rows = torch.arange(q.shape[1])[None].expand(q.shape[0], -1)
    B, R = rows.shape
    C = q.shape[-1]
    ref = torch.empty(B, R, C, dtype=torch.float64, device=q.device)
    tol = torch.empty_like(ref)
    blk = _block(heads, k.shape[1])
    for b in range(B):
        kb, vb = k[kv_of[b]:kv_of[b] + 1], v[kv_of[b]:kv_of[b] + 1]
        for s in range(0, R, blk):
            r = rows[b, s:s + blk].to(q.device)
            o, t = AB.ref_and_bound(q[b:b + 1].index_select(1, r), kb, vb, heads, 1, scale, bias, poly, rowsum, rows=r)
            ref[b, s:s + blk], tol[b, s:s + blk] = o[0], t[0]
    return ref, tol


def logit_propagation(q2, E1, k, v, kv_of, heads, scale):
    """(e^(2 Delta_i) - 1) sum_j w_ij |v_jc - y_ic| with Delta_i = fp32(scale) max_j sum_c E1_ic |k_jc| (module
    docstring), fp64 [B, R, C]; q2 / E1 [B, R, C] are the reference query rows and their bound."""
    B, R, C = q2.shape
    d = C // heads
    out = torch.empty(B, R, C, dtype=torch.float64, device=q2.device)
    blk = _block(heads, k.shape[1], 2)
    sc = _f32(scale)
    for b in range(B):
        kh, vh = AB._heads(k[kv_of[b]:kv_of[b] + 1], heads)[0], AB._heads(v[kv_of[b]:kv_of[b] + 1], heads)[0]
        for s in range(0, R, blk):
            qh = AB._heads(q2[b:b + 1, s:s + blk], heads)[0]                   # [H, r, d]
            eh = AB._heads(E1[b:b + 1, s:s + blk], heads)[0]
            w = torch.softmax((qh @ kh.transpose(-1, -2)) * sc, -1)            # [H, r, Lk]
            y = w @ vh
            delta = sc * (eh @ kh.abs().transpose(-1, -2)).amax(-1, keepdim=True)
            spread = torch.empty_like(y)                                        # sum_j w_ij |v_jc - y_ic|
            for c in range(d):
                spread[..., c] = (w * (vh[:, None, :, c] - y[..., c:c + 1]).abs()).sum(-1)
            out[b, s:s + blk] = (torch.expm1(2 * delta) * spread).transpose(0, 1).reshape(-1, C)
    return out


class Layer(NamedTuple):
    rows: torch.Tensor                 # int64 [B, R]: token of every evaluated row (all of them: the token order)
    ref: Dict[str, torch.Tensor]       # stage -> fp64 [B, R, C]
    tol: Dict[str, torch.Tensor]       # stage -> the composed bound of that stage's kernel output
    own: Dict[str, torch.Tensor]       # stage -> the kernel's own bound on the operands it received


def temporal_kernel(N: int) -> str:
    return "rows" if N <= 16 else "round1"


def evaluate(ops: Operands, ctl: Control, sample=None, received=None, mutant=None, poly=0, rowsum=False,
             device=None) -> Layer:
    """The staged fp64 reference and composed bound of the layer's attention result (stages "spatial", "cross",
    "temporal" as enabled).  ``received``: the fp16 operands the kernels got, at the full [B, L, C] --
    "cross_q" (stage 2's query) and "temporal_v" (stage 3's V); absent, the fp16 rounding of the reference is used.
    ``mutant``: one of ``MUTANTS``, a deliberately wrong layer."""
    if mutant is not None and mutant not in MUTANTS:
        raise ValueError(mutant)
    dev = device if device is not None else ops.q.device
    q, k, v = (t.to(dev) for t in (ops.q, ops.k, ops.v))
    q_ref, k_ref = (None if t is None else t.to(dev) for t in (ops.q_ref, ops.k_ref))
    received = {n: t.to(dev) for n, t in (received or {}).items()}
    heads, chunks = ops.heads, ops.chunks
    B, L, C = q.shape
    N, d = B // chunks, C // heads
    inv = 1.0 / math.sqrt(d)
    perm = None
    if mutant == "heads-split-d-h":
        perm = _heads_perm(C, heads).to(dev)
        q, k, v = q[..., perm], k[..., perm], v[..., perm]
        q_ref, k_ref = (None if t is None else t[..., perm] for t in (q_ref, k_ref))
    rows = sample_rows(ctl, B, N, L, sample)
    R = rows.shape[1]
    refs, tols, own = {}, {}, {}
    ident = list(range(B))

    # ---- stage 1: spatial-guided attention, the result replaces the query
    q2, E1 = _take(q, rows).double(), None
    if ctl.use_intra:
        scale = (1.0 if mutant == "spatial-scale-without-0.2" else ctl.intra_scale) * inv
        bias = 0.0 if mutant == "diag-bias-dropped" else float(ctl.intra_bias)
        q2, E1 = _attn_rows(q_ref, k_ref, q, rows, ident, heads, scale, bias, poly, rowsum)
        refs["spatial"], tols["spatial"], own["spatial"] = q2, E1, E1

    # ---- stage 2: cross-frame attention on the selected K/V (or each frame's own)
    if ctl.use_cf:
        idx = kv_rows(ctl, N, L, mutant)
        if idx is None:
            k_att, v_att = k.view(chunks, N, L, C)[:, 0], v.view(chunks, N, L, C)[:, 0]
        else:
            idx = idx.to(dev)
            k_att, v_att = k.reshape(chunks, N * L, C)[:, idx], v.reshape(chunks, N * L, C)[:, idx]
        kv_of = [b // N for b in range(B)]
        if mutant == "chunk1-reads-chunk0-kv":
            kv_of = [0] * B
        if mutant == "own-frame-kv":
            k_att, v_att, kv_of = k, v, ident
    else:
        k_att, v_att, kv_of = k, v, ident
    q2_got = _take(received["cross_q"], rows) if "cross_q" in received else (q2.half() if E1 is not None else q2)
    y2, _ = _attn_rows(q2, k_att, v_att, None, kv_of, heads, inv, 0.0, poly, rowsum)
    _, E2 = _attn_rows(q2_got, k_att, v_att, None, kv_of, heads, inv, 0.0, poly, rowsum)
    own["cross"] = E2
    if E1 is not None:
        E2 = E2 + logit_propagation(q2, E1, k_att, v_att, kv_of, heads, inv)
    refs["cross"], tols["cross"] = y2, E2

    # ---- stage 3: temporal-guided attention along the trajectories, V = stage 2
    if ctl.use_inter:
        fwd, bwd, tmask = trajectories(ctl, L)
        P = torch.arange(L) if sample is None else torch.as_tensor(sample).long().cpu()
        msk = tmask[P]
        if mutant == "transposed-trajectory-mask":
            msk = msk.transpose(1, 2)
        qt = refs["spatial"] if mutant == "temporal-q-from-q-main" and ctl.use_intra else _take(q, rows)
        kt = _take(k, rows)
        scale = (1.0 if mutant == "temporal-k-without-scale" else ctl.inter_scale) * inv
        idm = torch.arange(R)[None].expand(N, R)
        kern = temporal_kernel(N)
        v3_got = _take(received["temporal_v"], rows) if "temporal_v" in received else y2.half()
        y3, _ = TB.ref_and_bound(qt, kt, y2, idm, msk, chunks, heads, scale, kern)
        _, E3 = TB.ref_and_bound(qt, kt, v3_got, idm, msk, chunks, heads, scale, kern)
        own["temporal"] = E3
        E3 = E3 + TB.ref_and_bound(qt, kt, E2, idm, msk, chunks, heads, scale, kern)[0]
        if mutant == "scatter-through-bwd-map":
            if sample is not None:
                raise ValueError("the bwd-map scatter mutant needs every trajectory")
            # row p of frame f lands on token bwd[f, p] instead of fwd[f, p]; read back at the evaluated tokens
            fr = torch.arange(B) % N
            tok = torch.empty_like(y3)
            tok.scatter_(1, bwd[fr].to(dev)[..., None].expand(-1, -1, C), y3)
            y3 = _take(tok, rows)
        refs["temporal"], tols["temporal"] = y3, E3
    if perm is not None:
        inv_perm = torch.empty_like(perm)
        inv_perm[perm] = torch.arange(C, device=dev)
        for dct in (refs, tols, own):
            for n in dct:
                dct[n] = dct[n][..., inv_perm]
    if sample is None and ctl.use_inter:                    # every row evaluated: back to the token layout
        for dct in (refs, tols, own):
            for n in dct:
                dct[n] = to_tokens(dct[n], rows, L)
        rows = torch.arange(L)[None].expand(B, L)
    return Layer(rows, refs, tols, own)


def attention_result(layer: Layer):
    """(ref, tol) of the layer's attention result (the last enabled stage)"""
    last = "temporal" if "temporal" in layer.ref else "cross"
    return layer.ref[last], layer.tol[last]


def out_stage(a_ref, a_tol, W, b, a_got=None):
    """(ref, tol) of to_out[0] = a W^T + b run in fp32 (TF32 off) on the fp32 cast of the fp16 attention result."""
    W64 = W.double().to(a_ref.device)
    b64 = b.double().to(a_ref.device) if b is not None else torch.zeros(W.shape[0], dtype=torch.float64,
                                                                         device=a_ref.device)
    a = a_ref if a_got is None else a_got.double().to(a_ref.device)
    C = W.shape[1]
    ref = a_ref @ W64.T + b64
    tol = a_tol @ W64.abs().T + SAFETY * (C + 1) * U * (a.abs() @ W64.abs().T + b64.abs())
    return ref, tol


def ratio(out, ref, tol):
    r = (out.double().to(ref.device) - ref).abs() / tol
    return torch.nan_to_num(r, nan=float("inf"))


# ============================================================================================== layer families
FAMILIES = ("exact", "amplify", "temporal-dominant", "temporal-huge", "realistic", "diag-bias",
            "mask-frame0", "mask-all", "mask-none", "mask-multi")


class Case(NamedTuple):
    family: str
    ops: Operands                     # fp16 projections (for "realistic": of x and ref_hidden through ``weights``)
    ctl: Control                      # every mode on; select with ``ctl.modes(flags)``
    x: Optional[torch.Tensor] = None          # fp32 hidden states and reference features ("realistic")
    ref_hidden: Optional[torch.Tensor] = None
    weights: Optional[tuple] = None           # (Wq, Wk, Wv) fp32 [C, C]


def _layernorm(t, gain=1.0):
    return gain * (t - t.mean(-1, keepdim=True)) / t.std(-1, keepdim=True, unbiased=False)


def _random_mask(N, L, g, p=0.3):
    m = torch.rand(N, L, generator=g) < p
    m[0] = True
    return m


def _maps(fwd, tmask):
    return [fwd[:, None]], [torch.argsort(fwd, 1)[:, None]], [tmask[:, None]]


def project(x, weights, dtype=torch.float32):
    return tuple((x.to(dtype) @ w.to(dtype).T).half() for w in weights)


def _codes(n, d, R):
    """n <= 2d exactly orthogonal or opposite code vectors of norm R: R e_(a mod d), sign by a // d"""
    a = torch.arange(n)
    c = torch.zeros(n, d)
    c[a, a % d] = torch.where(a // d == 0, float(R), -float(R))
    return c


def _exact(N, L, heads, d, chunks, g, use_cf=True):
    """every stage one-hot (>= 45 nats), self-only trajectories; V encodes (chunk, frame, token) and the head"""
    R = 8.0
    s1, s2 = _f32(0.2 / math.sqrt(d)), _f32(1.0 / math.sqrt(d))
    val1, val2 = math.ceil(46.0 / (s1 * R)), math.ceil(46.0 / (s2 * R))
    mask = _random_mask(N, L, g)
    nbf = max(1, min(16, (2 * d) // N))                               # beacons per frame, unique codes per chunk
    for f in range(1, N):                                             # enough selected tokens for the beacons
        if mask[f].sum() < nbf:
            mask[f, torch.randperm(L, generator=g)[:nbf]] = True
    beacon_tok = torch.stack([torch.nonzero(mask[f]).reshape(-1)[torch.randperm(int(mask[f].sum()), generator=g)[:nbf]]
                              if mask[f].sum() >= nbf else torch.randperm(L, generator=g)[:nbf] for f in range(N)])
    nbf = beacon_tok.shape[1]
    codes = _codes(N * nbf, d, R)
    k = torch.zeros(chunks, N, L, heads, d)
    for f in range(N):
        k[:, f, beacon_tok[f]] = codes[f * nbf:(f + 1) * nbf][None, :, None, :]
    # the beacons each frame sees: all of the chunk's (cross-frame) or its own (self-attention)
    if use_cf:
        visible = [list(range(N * nbf))] * N
    else:
        visible = [list(range(f * nbf, (f + 1) * nbf)) for f in range(N)]
    q = torch.zeros(chunks, N, L, heads, d)
    for f in range(N):
        vis = torch.tensor(visible[f])
        pick = vis[torch.randint(0, len(vis), (chunks, L, heads), generator=g)]
        q[:, f] = codes[pick] / R * val2
    nb1 = min(2 * d, 16, L)
    k_ref = torch.zeros(chunks, N, L, heads, d)
    c1 = _codes(nb1, d, R)
    for f in range(N):
        k_ref[:, f, torch.randperm(L, generator=g)[:nb1]] = c1[None, :, None, :]
    q_ref = c1[torch.randint(0, nb1, (chunks, N, L, heads), generator=g)] / R * val1
    v = torch.randn(chunks, N, L, heads, d, generator=g)
    n = (torch.arange(N)[:, None] * L + torch.arange(L)[None]).float()
    v[..., 0] = (n % 1024)[None, :, :, None]
    v[..., 1] = (torch.arange(chunks)[:, None, None] * 64 + torch.div(n, 1024, rounding_mode="floor")[None])[..., None]
    v[..., 2] = torch.arange(heads).float()
    tok = lambda t: t.reshape(chunks * N, L, heads * d).half()
    fwd = TB._perms(N, L, g)
    f_, b_, i_ = _maps(fwd, torch.eye(N, dtype=torch.bool).expand(L, N, N).clone())
    ops = Operands(tok(q), tok(k), tok(v), tok(q_ref), tok(k_ref), heads, chunks)
    return ops, Control(True, True, True, [mask], f_, b_, i_)


def _generic(N, L, heads, d, chunks, g):
    C = heads * d
    t = lambda: _layernorm(torch.randn(chunks * N, L, C, generator=g)).half()
    return t(), t(), t(), t(), t()


def _realistic(N, Hs, Ws, heads, d, chunks, g, seed):
    from . import fresco_oracle as O
    C, L = heads * d, Hs * Ws
    base = torch.randn(1, L, C, generator=g)
    x = _layernorm(base + 0.7 * torch.randn(chunks * N, L, C, generator=g))
    ref_hidden = _layernorm(x + 0.5 * torch.randn(chunks * N, L, C, generator=g))
    weights = tuple(torch.randn(C, C, generator=g) / math.sqrt(C) for _ in range(3))
    flows, occs = O.synth_flows(N, 8 * Hs, 8 * Ws, seed=seed, mag=12.0)
    if N > 1:
        masks = O.cross_frame_masks(occs[1])
    else:                                                             # one frame: it keeps every token at each scale
        masks = [torch.ones(1, int(8 * Hs // s) * int(8 * Ws // s), dtype=torch.bool) for s in (8.0, 16.0, 32.0)]
    imgs = F.interpolate(torch.rand(N, 3, 8, 8, generator=g) * 2 - 1, size=(8 * Hs, 8 * Ws), mode="bilinear")
    fm, bm, im = [], [], []
    for s in (8.0, 16.0):
        if Hs * 8 / s >= 1 and Ws * 8 / s >= 1:
            a, b, c = O.mapping_ind(flows[1], occs[1], imgs, scale=s)
            fm.append(a), bm.append(b), im.append(c)
    q, k, v = project(x, weights)
    q_ref, k_ref = project(ref_hidden, weights[:2])
    return Case("realistic", Operands(q, k, v, q_ref, k_ref, heads, chunks),
                Control(True, True, True, masks, fm, bm, im), x, ref_hidden, weights)


def make_case(family, N, L, heads, d, chunks=2, seed=0, grid=None, use_cf=True) -> Case:
    """One layer case on CPU tensors.  ``grid`` = (H, W) of the L tokens (the realistic family's flows); ``use_cf``
    matters to the exact family only (which beacons a frame can see)."""
    g = torch.Generator().manual_seed(seed * 7919 + N * 131 + L * 7 + d)
    if family == "realistic":
        Hs, Ws = grid if grid is not None else (L, 1)
        assert Hs * Ws == L
        return _realistic(N, Hs, Ws, heads, d, chunks, g, seed)
    B, C = chunks * N, heads * d
    fwd = TB._perms(N, L, g)
    if family == "exact":
        ops, ctl = _exact(N, L, heads, d, chunks, g, use_cf)
        return Case(family, ops, ctl)
    if family == "amplify":
        R = 8.0
        s1 = _f32(0.2 / math.sqrt(d))
        val1 = math.ceil(46.0 / (s1 * R))
        na = min(d, 16, L // 2)
        c1 = _codes(na, d, R)
        k_ref = torch.zeros(chunks, N, L, heads, d)
        for f in range(N):
            pos = torch.randperm(L, generator=g)[:2 * na]
            k_ref[:, f, pos[:na]] = c1[None, :, None, :]
            k_ref[:, f, pos[na:]] = (c1 * (1 + 2.0 ** -10))[None, :, None, :]      # a near tie: 0.045 nat apart
        q_ref = c1[torch.randint(0, na, (chunks, N, L, heads), generator=g)] / R * val1
        q = 30.0 * torch.randn(B, L, C, generator=g)
        k = 4.0 * torch.randn(B, L, C, generator=g)
        v = torch.randn(B, L, C, generator=g)
        tok = lambda t: t.reshape(B, L, C).half()
        f_, b_, i_ = _maps(fwd, TB.reference_mask(N, L, g))
        return Case(family, Operands(tok(q), tok(k), tok(v), tok(q_ref), tok(k_ref), heads, chunks),
                    Control(True, True, True, [_random_mask(N, L, g)], f_, b_, i_))
    if family in ("temporal-dominant", "temporal-huge"):
        tc = TB.make_case(family.split("-")[1], N, L, heads, d, chunks, seed)
        _, _, v, q_ref, k_ref = _generic(N, L, heads, d, chunks, g)
        f_, b_, i_ = _maps(tc.fwd_map, tc.mask)
        # interattn_scale_factor 1: the temporal logits are the family's own (built at scale 1 / sqrt(d))
        return Case(family, Operands(tc.q, tc.k, v, q_ref, k_ref, heads, chunks),
                    Control(True, True, True, [_random_mask(N, L, g)], f_, b_, i_, inter_scale=1.0))
    q, k, v, q_ref, k_ref = _generic(N, L, heads, d, chunks, g)
    ops = Operands(q, k, v, q_ref, k_ref, heads, chunks)
    f_, b_, i_ = _maps(fwd, TB.reference_mask(N, L, g))
    if family == "diag-bias":
        return Case(family, ops, Control(True, True, True, [_random_mask(N, L, g)], f_, b_, i_,
                                         intra_scale=0.35, intra_bias=2.5, inter_scale=0.3))
    if family == "mask-frame0":
        m = torch.zeros(N, L, dtype=torch.bool)
        m[0] = True
        return Case(family, ops, Control(True, True, True, [m], f_, b_, i_))
    if family == "mask-all":
        return Case(family, ops, Control(True, True, True, [torch.ones(N, L, dtype=torch.bool)], f_, b_, i_))
    if family == "mask-none":
        return Case(family, ops, Control(True, True, True, [_random_mask(N, 2 * L, g)], f_, b_, i_))
    if family == "mask-multi":
        # masks at three resolutions, the matching one in the middle; mappings at two, the matching one first
        masks = [_random_mask(N, 4 * L, g), _random_mask(N, L, g, 0.5), _random_mask(N, max(1, L // 4), g)]
        lo = max(1, L // 4)
        f2, b2, i2 = _maps(TB._perms(N, lo, g), TB.reference_mask(N, lo, g))
        return Case(family, ops, Control(True, True, True, masks, f_ + f2, b_ + b2, i_ + i2))
    raise ValueError(family)


# ---------------------------------------------------------------------------------------------- family properties
def family_property(case: Case, flags: int = 7, sample=None, device=None) -> None:
    """Assert the property that makes the family sensitive; a change to a generator that made it harmless fails here.
    ``sample``: as ``evaluate`` takes it, for the families whose property needs the layer's reference."""
    ops, ctl = case.ops, case.ctl.modes(flags)
    B, L, C = ops.q.shape
    N, heads = B // ops.chunks, ops.heads
    d = C // heads
    fam = case.family
    if fam == "exact":
        lay = evaluate(ops, ctl, sample, device=device)
        a = attention_result(lay)[0].half().cpu()
        R = a.shape[1]
        v = ops.v.cpu().reshape(ops.chunks, N * L, heads, d)
        code = a.reshape(B, R, heads, d).float()
        n = (code[..., 1] % 64) * 1024 + code[..., 0]
        ch = torch.div(code[..., 1], 64, rounding_mode="floor")
        assert (code[..., 2] == torch.arange(heads).float()).all(), f"{fam}: a row does not carry its head"
        src = v[ch.long(), n.long(), torch.arange(heads)[None, None]]                    # [B, L, H, d]
        assert torch.equal(src.reshape(B, R, C), a), f"{fam}: the layer's answer is not a copy of V rows"
    elif fam == "amplify":
        if ctl.use_intra:
            lay = evaluate(ops, ctl, sample, device=device)
            eh = AB._heads(lay.tol["spatial"][:1], heads)                 # frame 0's keys: selected at every mask
            delta = _f32(1 / math.sqrt(d)) * (eh @ AB._heads(ops.k[:1].to(eh.device), heads).abs().transpose(-1, -2)).amax(-1)
            assert delta.max().item() >= 2.0, f"{fam}: the spatial stage's error moves a logit by {delta.max():.2f} nat"
    elif fam.startswith("temporal-"):
        tr = trajectories(ctl, L)
        tc = TB.Case(fam.split("-")[1], ops.q, ops.k, ops.v, tr[0], tr[2], ops.chunks, heads,
                     ctl.inter_scale / math.sqrt(d))
        TB.family_property(tc)
    elif fam == "realistic":
        idx = kv_rows(ctl, N, L)
        assert idx is not None and (N == 1 or L < idx.numel() < N * L), \
            f"{fam}: {None if idx is None else idx.numel()} rows selected"
        tr = trajectories(ctl, L)
        assert tr is not None and (N == 1 or (~tr[2]).any()), f"{fam}: no trajectory is cut"
    elif fam == "diag-bias":
        r = torch.arange(min(L, 256))
        x, _, _ = AB._logits(ops.q_ref[:1, :len(r)], ops.k_ref[:1], heads, 1, ctl.intra_scale / math.sqrt(d),
                             ctl.intra_bias, rows=r)
        wd = torch.softmax(x, -1).diagonal(dim1=-2, dim2=-1)
        assert (wd * L).median() >= 2.0, f"{fam}: the diagonal key is not favoured"
    elif fam == "mask-frame0":
        assert kv_rows(ctl, N, L).numel() == L, fam
    elif fam == "mask-all":
        assert kv_rows(ctl, N, L).numel() == N * L, fam
    elif fam == "mask-none":
        assert kv_rows(ctl, N, L) is None and ctl.masks, fam
    elif fam == "mask-multi":
        sizes = [m.shape[1] for m in ctl.masks]
        assert sizes.count(L) == 1 and len(sizes) == 3 and sizes.index(L) not in (0, len(sizes) - 1), sizes
        assert len(ctl.fwd_maps) == 2 and ctl.fwd_maps[0].shape[2] == L, fam
    else:
        raise ValueError(fam)
