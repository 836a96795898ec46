"""fp64 reference of the temporal-consistency loss (O2: ``warp_loss_quad_kernel``, ``warp_loss_group_kernel``,
``warp_loss_kernel`` in hbm_kernels.cu, the adjoint ELL of ``ops._pack_adjoint``), an elementwise bound on the
kernels' error, and input families built to break them.

CHECKER ONLY (see ``oracle/__init__``).  The operands are the kernels' own: ``cs`` fp32 [chunks, frames, C, h, w],
flows fp32 [frames, 2, h, w], keep masks fp32 in {0, 1} [frames, h, w] and k = fp32(2 / (chunks total_frames C h w)).
Pair f = (frame f, frame f+1 | frame 0 (closed ring) | the halo plane (open chain)):

    r1 = c2 - W_bf c1     r2 = c1 - W_ff c2     loss = k sum(|r1| m_b + |r2| m_f)
    d/dc1 = s2 - W_bf^T s1    d/dc2 = s1 - W_ff^T s2    s1 = sgn(r1) m_b, s2 = sgn(r2) m_f

with bilinear taps from x + flow evaluated in fp64, and W^T applied as the exact transpose of the fp64 warp
(``index_add`` in fp64; never the kernels' ELL, so a packing mistake cannot hide).  A frame's gradient is
k (ga + cb): ga from the pair it starts, cb ("carry") from the pair it ends; frame 0 of the ring gets the carry of pair
N - 1, in the open chain that carry is ``halo_grad``.

The bound
---------
All three kernels compute the same terms in different orders: the quad and group kernels keep sgn m in fp16 (exact for
m in {0, 1}) and form fl(fl(ga k) + fl(cb k)); the one-CTA kernel folds k into s in fp32 (fl(sgn m k) = +-k exactly,
again because m is 0 or 1) and sums the scaled terms.  One bound covers the three; every term is evaluated elementwise.
u = 2^-24, F = 2.

* Residual band eps_r, per residual.  fp32 rounds x + flow; the kernels' coordinate differs from the fp64 one by
  d = |X32 - X64| + |Y32 - Y64| (evaluated exactly here; at most 2^-24 (|X| + |Y|)).  The bilinear surface is continuous
  and, inside a cell, has slope at most 2 max|c| over the cell's corners in each direction, so the sample moves by at
  most 2 L d, L = max|c| over the corners of the fp64 and the fp32 cell -- also when floor crosses an integer or a tap
  crosses the border (a tap's weight is a continuous hat function that vanishes there).  Then the weight products
  (1 - ax)(1 - ay) round three times (3u relative), the sum of four products and the subtraction at most five times in
  any association nvcc picks (5u): eps_r = F (2 L d + 8 u (|c_own| + sum_t w_t |c_t|)).  |r64| > eps_r means the
  kernel's residual has the reference's sign; inside the band the sign may differ (or be 0).
* Gradient element, for each of ga and cb:
  - in-band signs: 2 m for the element's own in-band residual, 2 w m for every tap whose source residual is in band;
  - adjoint weights: per (source, destination) pair max(|w_q - w64|, |w32 - w64|), summed with the source's mask.
    w_q is the ELL weight, fl(round(w32 65535) * fl(1/65535)), 0 for a tap the packing drops (field 0); w32 is what an
    overflow entry carries.  This is the quantisation (<= 2^-17 + 2^-23 per tap) and the coordinate rounding of the
    weights, evaluated per tap rather than by their upper bounds: a truncating packing (floor for round) stays inside
    2^-16 per tap and is only visible this way.  Pairs that exist in one of the fp32 and fp64 stencils only count with
    their whole weight;
  - fp32 sums: the running sum starts from s (exact), takes the overflow run (run-length roundings plus one add) and
    8 FMAs (0-weight slots add exactly 0); the one-CTA kernel adds two more (s - gather, then the previous frame's
    term): (10 + n_taps) u T, T = m_own + sum_t w m_src, n_taps the fp32 taps that reach the element;
  - the final two products and one add, the wrap-around add of frame 0 and the second add under accumulate=1:
    4 u k (T_a + T_b) + 2 u |prefill|.
  tol = F (k (A_a + A_b) + 4 u k (T_a + T_b) + 2 u |prefill|); the halo plane gets the cb part alone.
* Loss: k sum eps_r m for the residuals, plus the fp32 sum: each thread adds at most
  2 frames (16 + ceil(hw / 128)) terms in sequence (one-CTA: 2 per pixel every 256; group: 2 KT P <= 2 (4 + hw / 128);
  quad: 8 residuals of 4 P NQ = 16 pixel-channels per frame), two levels of warp_sum (10), the product with k and the
  atomicAdd of every CTA (<= chunks C of them): (n_seq + 12 + chunks C) u k sum (|r| + eps_r) m, times F.

F = 2 is the one safety factor (second-order terms and FMA contraction choices); nothing else is widened.
"""
from __future__ import annotations

import math

import torch

from . import fresco_oracle as O

U = 2.0 ** -24
SAFETY = 2.0
INV65535 = torch.tensor(1.0 / 65535.0, dtype=torch.float32).item()       # the kernels' fp32 1.0f / 65535.0f

FAMILIES = ("subthreshold", "integer", "dyadic", "edges", "overflow", "near-tie", "masks", "smooth")
SUBTHRESHOLD = ((0.0, 2e-6), (2e-6, 0.0), (2e-6, 2e-6))


def loss_scale(chunks: int, total_frames: int, C: int, h: int, w: int) -> float:
    """k as the launcher computes it: fp32(2 / numel), numel in double."""
    return torch.tensor(2.0 / (float(chunks) * total_frames * C * h * w), dtype=torch.float32).item()


# ------------------------------------------------------------------------------------------------ taps
def _grid(h, w, device, dtype):
    i = torch.arange(h * w, device=device)
    return (i % w).to(dtype), torch.div(i, w, rounding_mode="floor").to(dtype)


def _stencil(X, Y, h, w, dtype):
    """Bilinear taps at (X, Y) [hw]: idx [hw, 4] (clamped), weight [hw, 4] (0 outside), valid [hw, 4], order
    (x0, y0), (x1, y0), (x0, y1), (x1, y1) as make_taps; the weight products are evaluated in ``dtype``."""
    xf, yf = torch.floor(X), torch.floor(Y)
    ax, ay = X - xf, Y - yf
    x0, y0 = xf.long(), yf.long()
    x1, y1 = x0 + 1, y0 + 1
    one = torch.ones((), dtype=dtype, device=X.device)
    vx0, vx1 = (x0 >= 0) & (x0 <= w - 1), (x1 >= 0) & (x1 <= w - 1)
    vy0, vy1 = (y0 >= 0) & (y0 <= h - 1), (y1 >= 0) & (y1 <= h - 1)
    cx0, cx1, cy0, cy1 = x0.clamp(0, w - 1), x1.clamp(0, w - 1), y0.clamp(0, h - 1), y1.clamp(0, h - 1)
    idx = torch.stack([cy0 * w + cx0, cy0 * w + cx1, cy1 * w + cx0, cy1 * w + cx1], -1)
    valid = torch.stack([vx0 & vy0, vx1 & vy0, vx0 & vy1, vx1 & vy1], -1)
    wt = torch.stack([(one - ax) * (one - ay), ax * (one - ay), (one - ax) * ay, ax * ay], -1)
    wt = torch.where(valid, wt, torch.zeros_like(wt))
    return idx, wt, valid, x0, y0


def taps64(flow2: torch.Tensor):
    """fp64 taps of one frame's flow [2, h, w] (x + flow in fp64)."""
    _, h, w = flow2.shape
    xs, ys = _grid(h, w, flow2.device, torch.float64)
    X, Y = xs + flow2[0].reshape(-1).double(), ys + flow2[1].reshape(-1).double()
    idx, wt, valid, x0, y0 = _stencil(X, Y, h, w, torch.float64)
    return {"idx": idx, "w": wt, "valid": valid, "X": X, "Y": Y, "x0": x0, "y0": y0}


def taps32(flow2: torch.Tensor):
    """make_taps in fp32, as warp_taps_kernel and the loss kernels evaluate it (x + flow rounded to fp32)."""
    _, h, w = flow2.shape
    xs, ys = _grid(h, w, flow2.device, torch.float32)
    X, Y = xs + flow2[0].reshape(-1).float(), ys + flow2[1].reshape(-1).float()
    idx, wt, valid, x0, y0 = _stencil(X, Y, h, w, torch.float32)
    return {"idx": idx, "w": wt, "valid": valid, "X": X, "Y": Y, "x0": x0, "y0": y0}


def ell_weight(w32: torch.Tensor) -> torch.Tensor:
    """The weight the ELL gather multiplies by: the packed field round(w 65535) decoded in fp32 (0: tap dropped)."""
    n = (w32.float() * 65535.0).round()
    return n * torch.tensor(INV65535, dtype=torch.float32)


def _warp(c, T):
    """c [P, hw] (fp64) sampled through taps T -> [P, hw]."""
    out = torch.zeros_like(c)
    for t in range(4):
        out += T["w"][:, t].to(c.dtype) * c[:, T["idx"][:, t]]
    return out


def _adjoint(s, idx, wt):
    """Exact transpose of the warp with taps (idx, wt) applied to s [P, hw]: scatter-add in s's dtype."""
    out = torch.zeros_like(s)
    out.index_add_(1, idx.reshape(-1), (s[:, :, None] * wt.to(s.dtype)[None]).reshape(s.shape[0], -1))
    return out


def _discrepancy(T64, T32, hw, h, w):
    """Per source pixel and position of the 4 x 4 window at (x0_64 - 1, y0_64 - 1): max(|w_q - w64|, |w32 - w64|)
    (the fp32 cell is at most one pixel off), with the destination pixel (-1 outside the plane).  -> (E [hw, 16],
    dst [hw, 16])."""
    dev = T64["w"].device
    bx, by = T64["x0"] - 1, T64["y0"] - 1
    w64 = torch.zeros(hw, 16, dtype=torch.float64, device=dev)
    w32 = torch.zeros_like(w64)
    wq = torch.zeros_like(w64)
    offs = ((0, 0), (1, 0), (0, 1), (1, 1))
    for t, (ox, oy) in enumerate(offs):
        p64 = (T64["y0"] + oy - by) * 4 + (T64["x0"] + ox - bx)
        w64.scatter_add_(1, p64[:, None], T64["w"][:, t:t + 1])
        p32 = ((T32["y0"] + oy - by) * 4 + (T32["x0"] + ox - bx)).clamp(0, 15)
        w32.scatter_add_(1, p32[:, None], T32["w"][:, t:t + 1].double())
        wq.scatter_add_(1, p32[:, None], ell_weight(T32["w"][:, t:t + 1]).double())
    E = torch.maximum((wq - w64).abs(), (w32 - w64).abs())
    k = torch.arange(16, device=dev)
    px, py = bx[:, None] + k % 4, by[:, None] + k // 4
    inside = (px >= 0) & (px < w) & (py >= 0) & (py < h)
    dst = torch.where(inside, py * w + px, torch.full_like(px, -1))
    return E, dst


def _scatter16(v, E, dst, hw):
    """sum over sources p of E[p, j] v[:, p] into dst[p, j] -> [P, hw]."""
    out = torch.zeros(v.shape[0], hw, dtype=torch.float64, device=v.device)
    ok = dst >= 0
    val = v[:, :, None] * E[None]
    out.index_add_(1, dst[ok], val[:, ok])
    return out


# ------------------------------------------------------------------------------------------------ reference + bound
def reference_and_bound(cs, ff, bf, kf, kb, halo_cs=None, total_frames=None, prefill=None):
    """cs fp32 [chunks, frames, C, h, w]; ff / bf [frames, 2, h, w]; kf / kb [frames, h, w] in {0, 1}; halo_cs
    [chunks, C, h, w] for the open chain (total_frames: the ring's length, for k); prefill: grad before an
    accumulate=1 call.  Returns a dict: loss, grad (fp64 [chunks, frames, C, h, w]), halo (or None), their tolerances
    loss_tol / grad_tol / halo_tol, the unscaled parts ga / cb / halo_cb (for exact families), k and in_band (the
    share of residuals inside their band)."""
    chunks, N, C, h, w = cs.shape
    hw, Pl = h * w, chunks * C
    dev = cs.device
    total = N if total_frames is None else total_frames
    k = loss_scale(chunks, total, C, h, w)
    planes = cs.permute(1, 0, 2, 3, 4).reshape(N, Pl, hw).double()
    nxt_halo = halo_cs.reshape(Pl, hw).double() if halo_cs is not None else None
    ga = torch.zeros(N, Pl, hw, dtype=torch.float64, device=dev)
    cb = torch.zeros_like(ga)
    Aa, Ab, Ta, Tb = (torch.zeros_like(ga) for _ in range(4))
    halo_cb = halo_A = halo_T = None
    loss = loss_err = loss_abs = 0.0
    n_band = n_res = 0
    for f in range(N):
        c1 = planes[f]
        c2 = nxt_halo if (f + 1 == N and halo_cs is not None) else planes[(f + 1) % N]
        mb, mf = kb[f].reshape(1, hw).double(), kf[f].reshape(1, hw).double()
        sides = []
        for flow, own, src, m_own in ((bf[f], c2, c1, mb), (ff[f], c1, c2, mf)):   # r1 = c2 - W_bf c1; r2 = c1 - W_ff c2
            T64, T32 = taps64(flow), taps32(flow)
            r = own - _warp(src, T64)
            d = ((T32["X"].double() - T64["X"]).abs() + (T32["Y"].double() - T64["Y"]).abs())[None]
            Lc = torch.cat([T["valid"].double()[None] * src.abs()[:, T["idx"]] for T in (T64, T32)], -1).amax(-1)
            sabs = _warp(src.abs(), T64)
            eps = SAFETY * (2 * Lc * d + 8 * U * (own.abs() + sabs))
            band = r.abs() <= eps
            n_band += int(band.sum())
            n_res += band.numel()
            loss += (r.abs() * m_own).sum().item()
            loss_err += (eps * m_own).sum().item()
            loss_abs += ((r.abs() + eps) * m_own).sum().item()
            s = torch.sign(r) * m_own
            E, dst = _discrepancy(T64, T32, hw, h, w)
            n_taps = torch.zeros(hw, dtype=torch.float64, device=dev)
            n_taps.index_add_(0, T32["idx"].reshape(-1), (T32["w"] != 0).double().reshape(-1))
            m = m_own.expand(Pl, hw)
            disc = _scatter16(m, E, dst, hw)
            sides.append({"s": s, "adj": _adjoint(s, T64["idx"], T64["w"]), "own": 2 * m * band, "m": m,
                          "taps": _adjoint(2 * m * band, T64["idx"], T64["w"]) + disc,
                          "mag": _adjoint(m, T64["idx"], T64["w"]) + disc, "n": n_taps[None]})
        one, two = sides                    # one: r1 / bwd warp / s1;  two: r2 / fwd warp / s2
        # d/dc1 = s2 - W_bf^T s1 (frame f): own residual r2, the bwd warp's taps from the sources' r1; d/dc2 mirrored
        ga[f] = two["s"] - one["adj"]
        Ta[f] = two["m"] + one["mag"]
        Aa[f] = two["own"] + one["taps"] + (10 + one["n"]) * U * Ta[f]
        gb = one["s"] - two["adj"]
        Tg = one["m"] + two["mag"]
        Ag = one["own"] + two["taps"] + (10 + two["n"]) * U * Tg
        if f + 1 == N and halo_cs is not None:
            halo_cb, halo_A, halo_T = gb, Ag, Tg
        else:
            fn = (f + 1) % N
            cb[fn], Ab[fn], Tb[fn] = gb, Ag, Tg
    pre = torch.zeros_like(ga) if prefill is None else prefill.permute(1, 0, 2, 3, 4).reshape(N, Pl, hw).double()
    grad = pre + k * (ga + cb)
    grad_tol = SAFETY * (k * (Aa + Ab) + 4 * U * k * (Ta + Tb) + 2 * U * pre.abs())

    def back(t):                                                           # [N, chunks C, hw] -> [chunks, N, C, h, w]
        return t.reshape(N, chunks, C, h, w).permute(1, 0, 2, 3, 4)

    out = {"k": k, "loss": k * loss, "grad": back(grad), "grad_tol": back(grad_tol), "ga": back(ga), "cb": back(cb),
           "halo": None, "halo_tol": None, "halo_cb": None, "in_band": n_band / n_res}
    n_seq = 2 * N * (16 + math.ceil(hw / 128))
    out["loss_tol"] = SAFETY * (k * loss_err + (n_seq + 12 + Pl) * U * k * loss_abs)
    if halo_cb is not None:
        out["halo"] = (k * halo_cb).reshape(chunks, C, h, w)
        out["halo_tol"] = (SAFETY * (k * halo_A + 2 * U * k * halo_T)).reshape(chunks, C, h, w)
        out["halo_cb"] = halo_cb.reshape(chunks, C, h, w)
    return out


def exact_grad(ref, accumulate=False, prefill=None, ring=True):
    """The gradient the quad and group kernels produce when ga and cb are exact in fp32 (the integer family):
    fl(fl(ga k) + fl(cb k)), frame 0 of the ring as fl(fl(ga k) + fl(cb k)) after the prefill when accumulating.
    Returns (grad fp32, halo fp32 or None)."""
    k = torch.tensor(ref["k"], dtype=torch.float32, device=ref["ga"].device)
    ga, cb = ref["ga"].float(), ref["cb"].float()
    assert torch.equal(ga.double(), ref["ga"]) and torch.equal(cb.double(), ref["cb"]), "parts not exact in fp32"
    v = ga * k + cb * k
    if accumulate:
        v = prefill + v
        if ring:                        # frame 0: prefill + fl(ga k) first, the wrap-around carry added last
            v[:, 0] = (prefill[:, 0] + ga[:, 0] * k) + cb[:, 0] * k
    halo = None if ref["halo_cb"] is None else ref["halo_cb"].float() * k
    return v, halo


# ------------------------------------------------------------------------------------------------ input families
def _binary(g, shape, p, device):
    return (torch.rand(shape, generator=g) < p).float().to(device)


def _smooth_flows(frames, h, w, seed, mag=12.0):
    """O.synth_flows at 8x the plane, resized as the decoder layers see them: (ff, bf, keep_f, keep_b)."""
    flows, occs = O.synth_flows(frames, 8 * h, 8 * w, seed=seed, mag=mag)
    ff, bf, fo, bo = O._resize_flow_occ(flows, occs, 1 / 8)
    return ff, bf, (1 - fo).reshape(frames, h, w), (1 - bo).reshape(frames, h, w)


def family(name, chunks, frames, C, h, w, seed=0, halo=False, device="cpu"):
    """Operands of one call: cs [chunks, frames, C, h, w] (+ halo_cs [chunks, C, h, w] when ``halo``), ff / bf
    [frames, 2, h, w], kf / kb [frames, h, w] in {0, 1}.  Each family asserts the property it is built to have."""
    g = torch.Generator().manual_seed(seed * 7919 + sum(map(ord, name)))
    nf = frames + (1 if halo else 0)
    hw = h * w
    cs = torch.randn(chunks, nf, C, h, w, generator=g)
    kf, kb = _binary(g, (frames, h, w), 0.8, "cpu"), _binary(g, (frames, h, w), 0.8, "cpu")
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    if name == "subthreshold":
        # every weight is 1 - 2e-6 or 2e-6 (or their products): the 2e-6 taps have an ELL field of 0, and the source that
        # sends one to a destination comes before that destination's own pixel in source order
        def const(v):
            return torch.stack([torch.full((h, w), v[0]), torch.full((h, w), v[1])])
        bf = torch.stack([const(SUBTHRESHOLD[f % 3]) for f in range(frames)])
        ff = torch.stack([const(SUBTHRESHOLD[(f + 1) % 3]) for f in range(frames)])
        early = 0
        for fl in list(bf) + list(ff):
            T = taps32(fl)
            tiny = (T["w"] > 0) & ((T["w"] * 65535.0).round() == 0)
            src = torch.arange(hw)[:, None].expand(hw, 4)
            first_tiny = torch.full((hw,), hw).scatter_reduce(0, T["idx"][tiny], src[tiny], "amin")
            main = torch.full((hw,), -1).scatter_reduce(0, T["idx"][T["w"] > 0.5], src[T["w"] > 0.5], "amax")
            early += int(((first_tiny < main) & (main >= 0)).sum())
        assert early >= 0.25 * hw * 2 * frames, f"only {early} rows start with a zero-field tap"
    elif name == "integer":
        # integer flows, cs on a 2^-8 grid, and c2 = W_bf c1 exactly on about half the pixels: every weight is 0 or 1,
        # every residual exact (and many exactly 0), ga and cb exact in fp32
        ff = torch.randint(-3, 4, (frames, 2, h, w), generator=g).float()
        bf = torch.randint(-3, 4, (frames, 2, h, w), generator=g).float()
        cs = (cs * 256).round() / 256
        for f in range(nf - 1):
            T = taps64(bf[f])
            warped = _warp(cs[:, f].reshape(-1, hw).double(), T).float().reshape(chunks, C, h, w)
            sel = torch.rand(h, w, generator=g) < 0.5
            cs[:, f + 1] = torch.where(sel, warped, cs[:, f + 1])
        for fl in list(bf) + list(ff):
            assert ((taps64(fl)["w"] == 0) | (taps64(fl)["w"] == 1)).all()
        assert torch.equal((cs * 256).round(), cs * 256)
    elif name == "dyadic":
        # multiples of 2^-10 px: x + flow and every weight are exact in fp32; only the ELL fields and the sums round
        ff = (torch.randn(frames, 2, h, w, generator=g) * 3 * 1024).round() / 1024
        bf = (torch.randn(frames, 2, h, w, generator=g) * 3 * 1024).round() / 1024
        for fl in list(bf) + list(ff):
            assert torch.equal(taps32(fl)["w"].double(), taps64(fl)["w"])
    elif name == "edges":
        # flows past all four borders (fractional, so the border taps are partial), and every 5th row sampling nothing
        # (r = c2 there)
        def out(f):
            gain = 0.6 + 0.1 * (f % 3)
            fx = (xs - (w - 1) / 2) * gain + torch.rand(h, w, generator=g) - 0.5
            fy = (ys - (h - 1) / 2) * gain + torch.rand(h, w, generator=g) - 0.5
            fy[2::5] = -(h + 3.0)
            fx[:, 0], fx[:, -1], fy[0], fy[-1] = -0.5, 0.5, -0.5, 0.5       # half a pixel past each border
            return torch.stack([fx, fy])
        bf = torch.stack([out(f) for f in range(frames)])
        ff = torch.stack([out(f + 1) for f in range(frames)])
        for fl in list(bf) + list(ff):
            T = taps64(fl)
            none = (T["w"] == 0).all(-1)
            assert none.float().mean() >= 0.1, "too few pixels sample nothing"
            X, Y = T["X"], T["Y"]
            for side in ((X > -1) & (X < 0), (X > w - 1) & (X < w), (Y > -1) & (Y < 0), (Y > h - 1) & (Y < h)):
                assert side.any(), "a border without partial taps"
    elif name == "overflow":
        # contraction towards the centre: ~4 hw / (0.15 h + 1)(0.15 w + 1) taps per destination there, overflow lists
        # longer than the CTA has threads (so runs have heads on different threads) and runs longer than 8
        contract = torch.stack([((w - 1) / 2 - xs) * 0.85 + 0.3, ((h - 1) / 2 - ys) * 0.85 - 0.2])
        bf = torch.randn(frames, 2, h, w, generator=g) * 1.5
        ff = torch.randn(frames, 2, h, w, generator=g) * 1.5
        bf[0::2] = contract
        ff[1::2] = contract
        if frames == 1:
            ff[0] = contract
        worst, longest = 0, 0
        for fl in list(bf) + list(ff):
            T = taps32(fl)
            cnt = torch.zeros(hw).index_add_(0, T["idx"].reshape(-1), (T["w"] > 0).float().reshape(-1))
            worst = max(worst, int((cnt - 8).clamp(min=0).sum()))
            longest = max(longest, int(cnt.max()) - 8)
        assert worst > max(512, min(1024, hw)) and longest > 8, (worst, longest)      # 512 / 1024: the CTA sizes
    elif name == "near-tie":
        # c2 = W_bf c1 + tiny noise (in fp32): most r1 fall inside their band, where the sign is the kernel's choice
        ff, bf, _, _ = _smooth_flows(frames, h, w, seed)
        for f in range(nf - 1):
            c1 = cs[:, f].reshape(-1, hw).double()
            warped = _warp(c1, taps64(bf[f]))
            cs[:, f + 1] = (warped + 2e-7 * torch.randn(warped.shape, generator=g, dtype=torch.float64)).float().reshape(
                chunks, C, h, w)
    elif name == "masks":
        # keep masks all 0, all 1 and a checkerboard, every pattern in both roles
        ff, bf, _, _ = _smooth_flows(frames, h, w, seed)
        pats = [torch.zeros(h, w), torch.ones(h, w), ((xs + ys) % 2 == 0).float()]
        kf = torch.stack([pats[f % 3] for f in range(frames)])
        kb = torch.stack([pats[(f + 1) % 3] for f in range(frames)])
        if frames == 1:
            kf, kb = pats[2][None], pats[0][None]
    elif name == "smooth":
        ff, bf, kf, kb = _smooth_flows(frames, h, w, seed)
        kf, kb = kf.contiguous(), kb.contiguous()
    else:
        raise ValueError(name)
    assert ((kf == 0) | (kf == 1)).all() and ((kb == 0) | (kb == 1)).all()
    dev = torch.device(device)
    out = {"cs": cs[:, :frames].contiguous().to(dev), "ff": ff.float().contiguous().to(dev),
           "bf": bf.float().contiguous().to(dev), "kf": kf.float().contiguous().to(dev),
           "kb": kb.float().contiguous().to(dev), "halo_cs": None}
    if halo:
        out["halo_cs"] = cs[:, frames].contiguous().to(dev)
    return out


def ratio(out: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor) -> torch.Tensor:
    """|out - ref| / tol elementwise (0 where out == ref, also where tol is 0; NaN in out counts as infinitely wrong)."""
    err = (out.double() - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / tol)
    return torch.nan_to_num(r, nan=float("inf"))
