"""fp64 references of GMFlow's global correlation softmax and flow attention (``tile_gemm_kernel<EPI_GMFLOW>``,
gemm_wgmma.cu), an elementwise bound on the kernel's error, and input families built to break its online softmax.

CHECKER ONLY (see ``oracle/__init__``).  Everything is evaluated in fp64 from the operands exactly as the kernel reads
them: ``gmflow_global_corr_softmax`` rounds the fp32 features to fp16 with round-to-nearest (to_token_major_f16_kernel),
``gmflow_flow_attention`` reads fp16 q / k, fp32 V and an fp32 softmax scale.

The kernel
----------
One CTA row of 128 queries walks every 128-key tile.  Per tile: S = A B^T in fp32 on the tensor cores; each thread
holds two rows and, per row, 32 of the tile's columns (acc_col: 8 k + 2 (lane & 3) + {0, 1}); the row max over the
valid columns (gn < N) is reduced over the quad, m_new = max(m_run, fp32(max S * c)) with c = fp32(scale log2 e),
alpha = ex2(m_run - m_new) rescales the lane's running l, x and y sums, then for each valid column
p = ex2.approx.ftz(fma(S, c, -m_new)), l += p, x = fma(p, v_x, x), y = fma(p, v_y, y) in column order.  After the last
tile two xor shuffles add the quad's four partial sums, and the output is x * (1.f / l) (IEEE division: the build
passes --use_fast_math=false) minus the query's own coordinate in coordinate mode.  P never leaves fp32.

V is either the key's pixel coordinate (gn % w, gn / w) -- coordinate mode, the global correlation -- or an explicit
[B, L, 2] fp32 field -- the flow attention.

The bound
---------
For one row i and output channel, with raw scores s_ij = a_i . b_j, logits x_ij = scale s_ij (nats), exact weights
w_ij = exp(x_ij - m_i) / l_i, E_i = sum_j w_ij v_j, u = 2^-24, n = 2 ceil(L / 8) (the most columns one lane sums) and
n_t = ceil(L / 128):

    A_i = sum_j w_ij |v_j|        D_i = sum_j w_ij |v_j - E_i|        ref_i = E_i - q_i   (q_i = 0 with explicit V)

    tol = F * ( expm1(2 (eps_i + sigma_i)) D_i + (2 n + 2 n_t + 6) u A_i + u |ref_i|
                + 2^-126 (sum_j |v_j| + L |E_i|) / l_i )

Each term, in the order the kernel does the work:

* ``sigma_i`` -- fp32 S.  Products of fp16 operands are exact in fp32; accumulating C of them errs by at most
  C u sum_k |a_ik b_jk|, so every logit of row i by at most sigma_i = scale C u max_j sum_k |a_ik b_jk| (nats).
* ``eps_i`` -- the exponential.  The argument fma(S, c, -m_new) carries the rounding of c (u relative for the
  correlation, whose c is rounded once from a double; 2u for the flow attention, fp32(scale) * fp32(log2 e)) applied
  to s - m with |s - m| <= 2 X_i (X_i = max_j |x_ij| log2 e), 4 u X_i; the FFMA's own rounding, u |arg| <= 2 u X_i; and
  the rounding of m_new = fp32(max S * c), u X_i.  7 u X_i in log2 units is a relative error of ln 2 * 7 u X_i =
  7 u max_j |x_ij| on p.  On top comes ex2.approx.ftz.f32 itself, within 2 ulp (2^-22):
  eps_i = 2^-22 + 7 u max_j |x_ij|.  alpha needs no term: it is quad-uniform (m_run is reduced over the quad) and
  scales l, x and y alike, so its error cancels in the ratio.
* ``expm1(2 rho) D`` -- what a perturbation of the weights does to the result.  If every p_j is off by a factor
  e^(delta_j) with |delta_j| <= rho, the normalised weights w'_j / w_j lie in [e^-2rho, e^2rho], and
  E' - E = sum_j (w'_j - w_j)(v_j - E), so |E' - E| <= expm1(2 rho) sum_j w_j |v_j - E| = expm1(2 rho) D.  In
  coordinate mode E is an absolute coordinate up to w - 1 and a term in A would scale with it; D scales with the
  spread of the matches, which is what the softmax actually mixes.  (To first order expm1(2 rho) = 2 rho.)
* ``(2 n + 2 n_t + 6) u A`` -- the sums.  Each lane adds at most n terms in sequence (l += p; the FMAs of x and y round
  once each), rescales its sums by alpha once per tile (n_t roundings) and the quad shuffles add twice: the numerator
  errs by (n + n_t + 2) u sum_j p_j |v_j|, l by (n + n_t + 2) u l (all p >= 0), which moves E by
  (n + n_t + 2) u (A + |E|) <= 2 (n + n_t + 2) u A.  1.f / l and the multiply add u |E| <= u A each.
* ``u |ref|`` -- the subtraction of the query coordinate (exact, and so zero, with explicit V).  nvcc contracts
  x * inv - q_x into one FFMA in some builds, so the multiply may not be rounded on its own; the bound keeps u A.
* ``2^-126 (...) / l`` -- ex2.approx.ftz flushes p below 2^-126 (and every alpha below it) to zero; a flushed key
  leaves at most 2^-126 |v_j| out of the numerator and 2^-126 out of l.

The terms are first order (except expm1).  F = 2 is the one safety factor: it covers the products of first-order errors
and the accumulation order inside the tensor core, which is not documented.  Nothing else is widened.

Operand rounding
----------------
``operand_rounding_term`` bounds the distance between the fp16-operand reference above and the reference on the fp32
features (``oracle.fresco_oracle.global_correlation_softmax`` evaluated in fp64): fp16 round-to-nearest errs by at
most e(t) = 2^-11 |t| + 2^-25 per element (2^-25: the subnormal range), so every logit moves by at most
tau_i = scale max_j sum_k (e(a_ik) |b^_jk| + |a_ik| e(b_jk)), and by the weight argument above the result by
expm1(2 tau_i) D_i (D from the fp32 weights).  That term is exact, not first order, and carries no safety factor.
"""
from __future__ import annotations

import math
from typing import NamedTuple

import torch

U = 2.0 ** -24
SAFETY = 2.0
EPS_EX2 = 2.0 ** -22          # ex2.approx.ftz.f32
LOG2E = 1.4426950408889634
TILE = 128


def _f32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


def to_tokens(f: torch.Tensor) -> torch.Tensor:
    """[B, C, h, w] -> [B, L, C], as to_token_major_f16_kernel lays it out (fp32, not rounded)."""
    B, C, h, w = f.shape
    return f.reshape(B, C, h * w).transpose(1, 2)


def f16(t: torch.Tensor) -> torch.Tensor:
    """Round to fp16 with round-to-nearest (__float2half_rn), as fp64."""
    return t.float().half().double()


def coords(h: int, w: int, device) -> torch.Tensor:
    """[L, 2] fp64 (x, y) of every token: the kernel's V in coordinate mode and the subtracted query coordinate."""
    n = torch.arange(h * w, device=device, dtype=torch.float64)
    return torch.stack([n % w, torch.div(n, w, rounding_mode="floor")], -1)


def _row(a, b, V, q, scale):
    """One row set: a [L, C] queries, b [Lk, C] keys (fp64, already as the kernel reads them), V [Lk, 2], q [L, 2] or 0.
    Returns (ref [2, L], tol [2, L])."""
    L, C = a.shape
    Lk = b.shape[0]
    x = (a @ b.T) * scale
    m = x.amax(-1, keepdim=True)
    e = torch.exp(x - m)
    l = e.sum(-1, keepdim=True)
    wgt = e / l
    del e
    E = wgt @ V                                                        # [L, 2]
    A = wgt @ V.abs()
    D = torch.stack([(wgt * (V[None, :, c] - E[:, c:c + 1]).abs()).sum(-1) for c in range(2)], -1)
    Xmax = x.abs().amax(-1, keepdim=True)
    del x, wgt
    sigma = scale * C * U * (a.abs() @ b.abs().T).amax(-1, keepdim=True)
    eps = EPS_EX2 + 7 * U * Xmax
    n = 2 * math.ceil(Lk / 8)
    nt = math.ceil(Lk / TILE)
    ref = E - q
    flush = 2.0 ** -126 * (V.abs().sum(0, keepdim=True) + Lk * E.abs()) / l
    tol = SAFETY * (torch.expm1(2 * (eps + sigma)) * D + (2 * n + 2 * nt + 6) * U * A + U * ref.abs() + flush)
    return ref.T, tol.T


def corr_ref_and_bound(f0: torch.Tensor, f1: torch.Tensor, bidir: bool):
    """gmflow_global_corr_softmax: (flow, tol), fp64 [B * (2 if bidir else 1), 2, h, w], order [fwd(B), bwd(B)]."""
    B, C, h, w = f0.shape
    scale = 1.0 / math.sqrt(C)
    g = coords(h, w, f0.device)
    t0, t1 = f16(to_tokens(f0)), f16(to_tokens(f1))
    pairs = [(t0, t1)] + ([(t1, t0)] if bidir else [])
    refs, tols = [], []
    for qa, kb in pairs:                                               # backward: softmax over the transposed volume
        for b in range(B):
            r, t = _row(qa[b], kb[b], g, g, scale)
            refs.append(r)
            tols.append(t)
    shape = (len(refs), 2, h, w)
    return torch.stack(refs).reshape(shape), torch.stack(tols).reshape(shape)


def flow_attn_ref_and_bound(q: torch.Tensor, k: torch.Tensor, vals: torch.Tensor, scale: float):
    """gmflow_flow_attention: q, k fp16 [B, L, C], vals fp32 [B, L, 2] -> (out, tol) fp64 [B, 2, L]."""
    scale = _f32(scale)
    refs, tols = [], []
    for b in range(q.shape[0]):
        r, t = _row(q[b].double(), k[b].double(), vals[b].double(), 0.0, scale)
        refs.append(r)
        tols.append(t)
    return torch.stack(refs), torch.stack(tols)


def _e16(t):
    return 2.0 ** -11 * t.abs() + 2.0 ** -25


def operand_rounding_term(f0: torch.Tensor, f1: torch.Tensor, bidir: bool):
    """(fp32-feature reference in fp64, |fp16-operand reference - it| bound), both [B(*2), 2, h, w] (docstring)."""
    B, C, h, w = f0.shape
    scale = 1.0 / math.sqrt(C)
    g = coords(h, w, f0.device)
    t0, t1 = to_tokens(f0).double(), to_tokens(f1).double()
    pairs = [(t0, t1)] + ([(t1, t0)] if bidir else [])
    refs, terms = [], []
    for qa, kb in pairs:
        for b in range(B):
            a, bb = qa[b], kb[b]
            x = (a @ bb.T) * scale
            wgt = torch.softmax(x, -1)
            del x
            E = wgt @ g
            D = torch.stack([(wgt * (g[None, :, c] - E[:, c:c + 1]).abs()).sum(-1) for c in range(2)], -1)
            del wgt
            tau = scale * (_e16(a) @ f16(bb).abs().T + a.abs() @ _e16(bb).T).amax(-1, keepdim=True)
            refs.append((E - g).T)
            terms.append((torch.expm1(2 * tau) * D).T)
    shape = (len(refs), 2, h, w)
    return torch.stack(refs).reshape(shape), torch.stack(terms).reshape(shape)


# ============================================================================================== exactly known answers
def tie_sums(a: torch.Tensor, b: torch.Tensor, V: torch.Tensor, gap_log2: float = 150.0):
    """For a row set whose best keys tie exactly and every other key is at least ``gap_log2`` below them (log2 units),
    the kernel's sums are exact: every tied p = ex2(0) = 1 (the tied score times c must be exact in fp32, see
    ``family``), every other p and every alpha across tiles flushes to 0.  Returns (l [L], s [L, 2]) -- the count of
    tied keys and the sum of their V -- or raises if the rows do not have that structure.  a, b fp64 [L, C]."""
    C = a.shape[1]
    s = a @ b.T
    top = s.amax(-1, keepdim=True)
    tied = s == top
    gap = ((top - s.masked_fill(tied, float("-inf")).amax(-1, keepdim=True)) * LOG2E / math.sqrt(C))
    if b.shape[0] > 1 and not (tied.all(-1, keepdim=True) | (gap >= gap_log2)).all():
        raise AssertionError(f"rows without an exact answer: smallest gap {gap.min().item():.1f} < {gap_log2} log2")
    return tied.double().sum(-1), tied.double() @ V


def exact_out(l: torch.Tensor, s: torch.Tensor, q) -> torch.Tensor:
    """The kernel's last roundings on exact sums: fp32(1 / l), then s * inv - q either as one fma or as a rounded
    multiply and a subtraction.  nvcc may contract the two, and does so for one output channel and not the other
    depending on the build, so both are valid answers.  Returns [2 (fused, separate), 2, L] fp32.  (s * inv is exact
    in fp64, and so is the difference at these sizes.)"""
    l32, s32 = l.float(), s.float()
    assert torch.equal(l32.double(), l) and torch.equal(s32.double(), s), "sums not exact in fp32"
    inv = torch.ones_like(l32) / l32
    fused = s32.double() * inv.double()[:, None]
    separate = (s32 * inv[:, None]).double()
    if not isinstance(q, float):
        fused, separate = fused - q, separate - q
    return torch.stack([fused.float().T, separate.float().T])


def corr_exact(f0: torch.Tensor, f1: torch.Tensor, bidir: bool) -> torch.Tensor:
    """The bit-exact flow of an exact family (``tie_sums``): fp32 [2 (fused, separate), B(*2), 2, h, w]."""
    B, C, h, w = f0.shape
    g = coords(h, w, f0.device)
    t0, t1 = f16(to_tokens(f0)), f16(to_tokens(f1))
    outs = []
    for qa, kb in [(t0, t1)] + ([(t1, t0)] if bidir else []):
        for b in range(B):
            outs.append(exact_out(*tie_sums(qa[b], kb[b], g), g))
    return torch.stack(outs, 1).reshape(2, len(outs), 2, h, w)


def flow_attn_exact(q: torch.Tensor, k: torch.Tensor, vals: torch.Tensor) -> torch.Tensor:
    """fp32 [2 (fused, separate), B, 2, L]; the two agree (q = 0)."""
    return torch.stack([exact_out(*tie_sums(q[b].double(), k[b].double(), vals[b].double()), 0.0)
                        for b in range(q.shape[0])], 1)


def matches_exact(out: torch.Tensor, want: torch.Tensor) -> torch.Tensor:
    """Elementwise: ``out`` equals one of the two valid roundings of ``corr_exact`` / ``flow_attn_exact`` bit for bit."""
    bits = out.reshape(want.shape[1:]).contiguous().view(torch.int32)
    return (bits == want[0].view(torch.int32)) | (bits == want[1].view(torch.int32))


# ============================================================================================== input families
class Family(NamedTuple):
    name: str
    f0: torch.Tensor            # [B, C, h, w] fp32, fp16-representable
    f1: torch.Tensor
    exact: bool                 # corr_exact / flow_attn_exact give the answer bit for bit


EXACT = ("uniform", "translated", "bimodal")
FAMILIES = ("uniform", "translated", "bimodal", "late", "early", "negative-floor", "peaky1", "peaky2", "peaky3")


def _gen(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def _grid(t, B, C, h, w):
    """[B, L, C] -> [B, C, h, w]."""
    return t.transpose(1, 2).reshape(B, C, h, w).contiguous()


def sign_code(C: int):
    """(g, h0): token patterns +-g on channels 1..C-1 and +-h0 on channel 0 with (C - 1) g^2 + h0^2 a power of two
    (so the self score times c is exact in fp32 and a match gives p = ex2(0) = 1), and one sign flip on a g channel
    2 g^2 >= 150 / c below the match (so every other p flushes to 0)."""
    c = LOG2E / math.sqrt(C)
    g = 1.0
    while 2 * g * g * c < 150.0:
        g *= 2
    for k in range(64):
        r = 2 ** k - (C - 1)
        if r >= 1 and math.isqrt(r) ** 2 == r:
            return g, g * math.isqrt(r)
    raise ValueError(C)


def _patterns(n, C, g, device):
    """n distinct sign patterns [n, C] scaled by sign_code."""
    gs, h0 = sign_code(C)
    for s in range(100):
        sg = torch.randint(0, 2, (n, C), generator=_gen(g + 1000 * s, device), device=device).float() * 2 - 1
        if torch.unique(sg, dim=0).shape[0] == n:
            sc = torch.full((C,), gs, device=device)
            sc[0] = h0
            return sg * sc
    raise RuntimeError("no distinct patterns")


def _layernorm(t):
    return (t - t.mean(-1, keepdim=True)) / t.std(-1, keepdim=True, unbiased=False)


def family(name: str, B: int, C: int, h: int, w: int, seed: int = 0, device="cpu", shift=(3, -5)) -> Family:
    """One input family on an h x w grid (module docstring of tests/test_gpu_gmflow.py lists what each one pins)."""
    L = h * w
    dy, dx = shift
    roll = lambda t: torch.roll(t.reshape(B, h, w, C), (dy, dx), (1, 2)).reshape(B, L, C)
    if name == "uniform":
        t = torch.zeros(B, L, C, device=device)
        t[..., 0] = 0.5                                                # s = 0.25 for every pair: p = ex2(0) = 1
        return Family(name, _grid(t, B, C, h, w), _grid(t, B, C, h, w), True)
    if name == "translated":
        t0 = torch.stack([_patterns(L, C, seed + b, device) for b in range(B)])
        return Family(name, _grid(t0, B, C, h, w), _grid(roll(t0), B, C, h, w), True)
    if name == "bimodal":
        # every pattern on two tokens, (y, x) of the top half and (y + h/2, x + 5) of the bottom half: two equal best
        # matches at least h/2 rows - 1 apart, so in different key tiles, the ragged last tile included
        assert h % 2 == 0
        t0 = torch.empty(B, h, w, C, device=device)
        for b in range(B):
            top = _patterns(L // 2, C, seed + b, device).reshape(h // 2, w, C)
            t0[b, :h // 2] = top
            t0[b, h // 2:] = torch.roll(top, 5, 1)
        t0 = t0.reshape(B, L, C)
        return Family(name, _grid(t0, B, C, h, w), _grid(roll(t0), B, C, h, w), True)
    gen = _gen(seed, device)
    base = lambda: _layernorm(torch.randn(B, L, C, generator=gen, device=device))
    if name in ("late", "early"):
        # channel 0: 96 r on the target tile's tokens, 16 r elsewhere (r = (C / 128)^(1/4)); with channels 1.. at
        # LayerNorm scale / 4, every query scores the target tile >= 100 nats above every other key, both directions
        t0, t1 = 0.25 * base(), 0.25 * roll(base())
        n_tiles = (L + TILE - 1) // TILE
        tgt = torch.zeros(L, dtype=torch.bool, device=device)
        if name == "late":
            tgt[(n_tiles - 1) * TILE:] = True
        else:
            tgt[:TILE] = True
        r = (C / 128) ** 0.25
        for t in (t0, t1):
            t[..., 0] = torch.where(tgt, 96.0 * r, 16.0 * r)
        return Family(name, _grid(t0, B, C, h, w).half().float(), _grid(t1, B, C, h, w).half().float(), False)
    if name == "negative-floor":
        # every logit in about [-125, -100] nats: a zero-filled column (logit 0) would take the row, and with it in
        # the max every p flushes to 0
        t0, t1 = 0.25 * base(), 0.25 * roll(base())
        sc = math.sqrt(C) / 32.0
        t0[..., 0] = 32.0
        t1[..., 0] = -sc * (100.0 + 25.0 * torch.rand(B, L, generator=gen, device=device))
        return Family(name, _grid(t0, B, C, h, w).half().float(), _grid(t1, B, C, h, w).half().float(), False)
    if name.startswith("peaky"):
        gain = float(name[5:])
        f0 = base()
        f1 = _layernorm(roll(f0) + 0.5 * base())
        return Family(name, _grid(gain * f0, B, C, h, w).half().float(), _grid(gain * f1, B, C, h, w).half().float(),
                      False)
    raise ValueError(name)


def family_property(fam: Family) -> None:
    """Assert on the fp64 logits (first batch, forward) the property that makes the family sensitive."""
    B, C, h, w = fam.f0.shape
    L = h * w
    a, b = f16(to_tokens(fam.f0))[0], f16(to_tokens(fam.f1))[0]
    x = (a @ b.T) / math.sqrt(C)
    name = fam.name
    if fam.exact:
        l, _ = tie_sums(a, b, coords(h, w, a.device))
        want = {"uniform": L, "translated": 1, "bimodal": 2}[name]
        assert (l == want).all(), f"{name}: tied keys per row {l.unique().tolist()}, want {want}"
        if name == "bimodal":
            s = a @ b.T
            cols = (s == s.amax(-1, keepdim=True)).nonzero()[:, 1].view(L, 2)
            assert (cols[:, 0] // TILE != cols[:, 1] // TILE).all(), f"{name}: two matches in one key tile"
            assert (cols >= (L - 1) // TILE * TILE).any(), f"{name}: no match in the last key tile"
    elif name in ("late", "early"):
        n_tiles = (L + TILE - 1) // TILE
        sl = slice((n_tiles - 1) * TILE, L) if name == "late" else slice(0, TILE)
        inside = x[:, sl].amax(-1)
        rest = x.clone()
        rest[:, sl] = float("-inf")
        gap = (inside - rest.amax(-1)).min().item()
        assert n_tiles >= 2 and gap >= 100, f"{name}: target tile only {gap:.1f} nats above the rest"
    elif name == "negative-floor":
        assert x.amax().item() <= -90 and x.amin().item() >= -140, (x.amin().item(), x.amax().item())
    elif name.startswith("peaky"):
        top = x.amax(-1).median().item()
        assert 3 <= top <= 300, f"{name}: median row max {top:.1f} nats"
    else:
        raise ValueError(name)
