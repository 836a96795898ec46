"""The spatial-consistency (Gram-L1) kernels -- gram_normalize_kernel, gram2_kernel<G2_SIGN|G2_GRAD>,
tile_gemm_kernel<EPI_GRAM_SIGN,0>, tile_gemm_kernel<EPI_STORE,1> and gram_project_kernel -- restated in torch fp32 on
the CPU, in each kernel's order of work.

The tensor-core contractions run under three accumulator models (``MODELS``): sequential round-to-nearest fp32 adds,
exact k16 step sums rounded once, and k16 steps aligned to their largest product exponent (an fp16-subnormal operand
counting as 2^-14) and truncated (the model
``oracle.gram_bound.acc_coef`` is derived for).  The sign-mode loss runs in the kernels' order: every consumer thread's
chain over the accumulator pairs of each tile its persistent CTA walks (a grid of ``GRID`` CTAs, so chains span several
tiles), the warp butterfly, the fp32 scale and the atomics in CTA order.  The projection runs with and without the fma.

It checks the error model of ``oracle.gram_bound`` without a GPU: every model stays inside the bound on every family,
the exact families come out bit for bit and the worst err/tol is reported (so the bound is seen not to be vacuous);
each of ``MUTANTS`` -- a one-line mistake a change to the kernels could make -- leaves the bound or the exact answer on
the family named with it.
"""
import math

import pytest
import torch

from oracle import gram_bound as GB

MODELS = ("sequential", "block-exact", "block-trunc")
GRID = 5
B = 2
SHAPES = [(7, 16), (129, 24), (257, 64), (383, 24)]     # (L, C): 1, 2, 3 (odd) and 3 128-row tiles; partial K atoms
MUTANTS = {
    # name: (what it does, the family that must catch it, (L, C))
    "diag-x2": ("diagonal-block loss counted x2", "onehot", (129, 24)),
    "no-mirror": ("off-diagonal tile not mirrored to [J, I]", "realistic", (257, 64)),
    "sign0-is-2": ("T = 2 at D == 0", "onehot", (129, 24)),
    "drop-ref-tail": ("last partial K atom of the reference half dropped", "near-tie", (129, 24)),
    "drop-odd-pair": ("last column pair dropped at an odd count of 128-row tiles", "realistic", (257, 64)),
    "dense-2sgn": ("EPI_GRAM_SIGN writes 2 sgn(d1)", "asymmetric", (129, 24)),
    "proj-no-norm": ("projection not divided by the norm", "dominant", (129, 24)),
    "proj-plus": ("g + dot x^ instead of g - dot x^", "realistic", (129, 24)),
    "norm-drop-partial": ("one of the 8 norm partials dropped", "realistic", (129, 24)),
    "alpha-twice": ("alpha applied twice", "realistic", (129, 24)),
    "fp16-acc": ("D accumulated in fp16", "near-tie", (257, 64)),
}
WORST = {}          # (family, stage) -> worst err/tol over models and shapes


def _note(fam, stage, r):
    WORST[(fam, stage)] = max(WORST.get((fam, stage), 0.0), r)


# ------------------------------------------------------------------------------------------------ emulation
def _trunc24(t):
    """t (fp64) truncated toward zero to 24 significant bits."""
    _, e = torch.frexp(t)
    q = torch.ldexp(torch.ones_like(t), (e - 24).to(torch.int32))
    return torch.where(t == 0, t, torch.trunc(t / q) * q)


def contract(A, Bm, model, fp16_acc=False):
    """sum_k A[:, k] Bm[:, k] -> fp32 [M, N] with K (a multiple of 16) in order; A, Bm hold fp16 values (or T)."""
    A, Bm = A.double(), Bm.double()
    M, K = A.shape
    acc = torch.zeros(M, Bm.shape[0], dtype=torch.float16 if fp16_acc else torch.float32)
    for k0 in range(0, K, GB.KSTEP):
        p = A[:, k0:k0 + GB.KSTEP].T[:, :, None] * Bm[:, k0:k0 + GB.KSTEP].T[:, None, :]     # [16, M, N] exact
        if fp16_acc:
            for k in range(p.shape[0]):
                acc = (acc.float() + p[k].float()).half()
        elif model == "sequential":
            for k in range(p.shape[0]):
                acc = acc + p[k].float()
        elif model == "block-exact":
            acc = (acc.double() + p.sum(0)).float()
        else:                                          # align to the largest exponent, truncate, add, truncate
            terms = torch.cat([acc.double()[None], p])        # an fp16 subnormal aligns as 2^-14 (oracle docstring)
            pe = GB.mag(A[:, k0:k0 + GB.KSTEP]).T[:, :, None] * GB.mag(Bm[:, k0:k0 + GB.KSTEP]).T[:, None, :]
            m = torch.maximum(acc.double().abs(), pe.amax(0))
            _, e = torch.frexp(m)
            q = torch.ldexp(torch.ones_like(m), (e - 24).to(torch.int32))
            q = torch.where(m == 0, torch.ones_like(m), q)
            acc = _trunc24((torch.trunc(terms / q) * q).sum(0)).float()
    return acc.float()


def _pad_k(x, mult=64):
    """[R, K] -> [R, roundup(K, mult)] with zeros (the TMA zero fill of a partial atom)."""
    K = x.shape[1]
    return torch.cat([x, torch.zeros(x.shape[0], (-K) % mult, dtype=x.dtype)], 1)


def emulate_normalize(cs, mutant=None):
    Bn, C, L = cs.shape
    part = []
    for w in range(8):
        s = torch.zeros(Bn, L)
        for c in range(w, C, 8):
            v = cs[:, c, :].double()
            s = (v * v + s.double()).float()
        part.append(s)
    s = torch.zeros(Bn, L)
    for i in range(8):
        if mutant == "norm-drop-partial" and i == 7:
            continue
        s = s + part[i]
    nrm = torch.sqrt(s)
    inv = 1.0 / nrm
    xh = (cs * inv[:, None, :]).half().transpose(1, 2).contiguous()
    return xh, nrm


def _tile_threads(cols_per_thread):
    """rows [256, n] and columns [256, n] of every consumer thread's accumulator entries in a 128-row tile (acc_row,
    acc_col of common.cuh), for n = 64 (N = 128) or 128 (N = 256) registers."""
    t = torch.arange(256)
    wg, w, lane = t // 128, (t // 32) % 4, t % 32
    i = torch.arange(cols_per_thread)
    rows = (wg * 64 + 16 * w + lane // 4)[:, None] + 8 * ((i >> 1) & 1)[None]
    cols = 8 * (i >> 2)[None] + 2 * (lane & 3)[:, None] + (i & 1)[None]
    return rows, cols


def _reduce_loss(chains, scale):
    """chains [G, 256] fp32 -> warp butterfly (lane 0's order), fp32 scale, atomics in CTA order."""
    v = chains.view(-1, 8, 32)
    idx = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, :, idx ^ o]
    part = (v[:, :, 0] * torch.tensor(GB.f32(scale), dtype=torch.float32)).flatten()
    acc = torch.zeros((), dtype=torch.float32)
    for p in part:
        acc = acc + p
    return acc.item()


def _tsign(D, mutant):
    t = 2 * torch.sign(D)
    if mutant == "sign0-is-2":
        t = torch.where(D == 0, torch.full_like(t, 2.0), t)
    return t


def emulate_sign_ref(Dk, scale, mutant=None):
    """gram2_kernel<G2_SIGN>: Dk [B, L, L] fp32 (the accumulators) -> T fp16 (NaN where never written), loss."""
    Bn, L, _ = Dk.shape
    Tn = (L + 127) // 128
    P = Tn // 2 if mutant == "drop-odd-pair" else (Tn + 1) // 2
    tiles = [(b, I, Jp) for b in range(Bn) for I in range(Tn) for Jp in range(I >> 1, P)]
    G = min(GRID, max(len(tiles), 1))
    Dp = torch.zeros(Bn, Tn * 128, max(P, 1) * 256 + 128)
    Dp[:, :L, :L] = Dk
    rows, cols = _tile_threads(128)
    rows, cols = rows[:, 0::2], cols[:, 0::2]                        # pairs (j, j + 1)
    chains = torch.zeros(G, 256)
    covered = torch.zeros(Bn, L, L, dtype=torch.bool)
    for r in range(-(-len(tiles) // G)):
        for c in range(G):
            k = c + r * G
            if k >= len(tiles):
                continue
            b, I, Jp = tiles[k]
            gm, j = I * 128 + rows, Jp * 256 + cols
            J = j >> 7
            valid = (J >= I) & (gm < L) & (j < L)
            w = torch.where((J == I) & (mutant != "diag-x2"), 1.0, 2.0).float()
            d0, d1 = Dp[b, gm, j], Dp[b, gm, j + 1]
            for p in range(64):
                term = (d0[:, p].abs() + d1[:, p].abs()) * w[:, p]
                chains[c] = torch.where(valid[:, p], chains[c] + term, chains[c])
            gv, jv = gm[valid], j[valid]
            covered[b, gv, jv] = True
            pair = jv + 1 < L
            covered[b, gv[pair], jv[pair] + 1] = True
    T = torch.full((Bn, L, L), float("nan"), dtype=torch.float16)
    t = _tsign(Dk, mutant).half()
    T[covered] = t[covered]
    blk = torch.arange(L) >> 7
    if mutant != "no-mirror":
        mirror = covered & (blk[None, None, :] > blk[None, :, None])
        Tt = T.transpose(1, 2)
        Tt[mirror] = t[mirror]
    return T, _reduce_loss(chains, scale)


def emulate_dense(Gk, A, scale, mutant=None):
    """tile_gemm_kernel<EPI_GRAM_SIGN,0>: Gk [B, L, L] fp32, A [B, L, L] fp32 -> T fp16, loss."""
    Bn, L, _ = Gk.shape
    d1 = Gk - A
    d2 = Gk - A.transpose(1, 2)
    tv = torch.sign(d1) + torch.sign(d2) if mutant != "dense-2sgn" else 2 * torch.sign(d1)
    Tn = (L + 127) // 128
    pad = Tn * 128
    d1p, d2p = torch.zeros(Bn, pad, pad), torch.zeros(Bn, pad, pad)
    d1p[:, :L, :L], d2p[:, :L, :L] = d1, d2
    rows, cols = _tile_threads(64)
    ctas = [(b, I, J) for b in range(Bn) for I in range(Tn) for J in range(I, Tn)]
    chains = torch.zeros(len(ctas), 256)
    for c, (b, I, J) in enumerate(ctas):
        gm, gn = I * 128 + rows, J * 128 + cols
        valid = (gm < L) & (gn < L)
        a1, a2 = d1p[b, gm, gn].abs(), d2p[b, gm, gn].abs()
        for p in range(64):
            term = a1[:, p] + (0.0 if I == J else a2[:, p])
            chains[c] = torch.where(valid[:, p], chains[c] + term, chains[c])
    blk = torch.arange(L) >> 7
    upper = (blk[None, :, None] <= blk[None, None, :]).expand(Bn, L, L)
    T = torch.full((Bn, L, L), float("nan"), dtype=torch.float16)
    T[upper] = tv.half()[upper]
    mirror = (blk[None, :, None] < blk[None, None, :]).expand(Bn, L, L)
    Tt = T.transpose(1, 2)
    Tt[mirror] = tv.half()[mirror]
    return T, _reduce_loss(chains, scale)


def emulate_tx(T, X, scale, model, mutant=None):
    """alpha T X^ for one batch: T [L, L] fp16, X^ [L, C] fp16 -> fp32 [L, C]."""
    acc = contract(_pad_k(T.double()), _pad_k(X.double().T), model)
    alpha = torch.tensor(GB.f32(scale), dtype=torch.float32)
    g = acc * alpha
    return g * alpha if mutant == "alpha-twice" else g


def emulate_project(g, X, nrm, grad0, fma, mutant=None):
    """gram_project_kernel, one batch: g [L, C] fp32, X^ fp16, norms [L], grad0 [C, L] -> grad [C, L] fp32."""
    L, C = g.shape
    Cp = -(-C // 32) * 32
    gp = torch.zeros(L, Cp)
    xp = torch.zeros(L, Cp)
    gp[:, :C], xp[:, :C] = g, X.float()
    acc = torch.zeros(L, 32)
    for c0 in range(0, Cp, 32):
        acc = (gp[:, c0:c0 + 32].double() * xp[:, c0:c0 + 32].double() + acc.double()).float()
    idx = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, idx ^ o]
    dot = acc[:, :1]
    x = X.float()
    if mutant == "proj-plus":
        num = g + dot * x
    elif fma:
        num = (g.double() - dot.double() * x.double()).float()
    else:
        num = g - dot * x
    v = num if mutant == "proj-no-norm" else num / nrm[:, None]
    return grad0 + v.T


# ------------------------------------------------------------------------------------------------ one family, one model
def run(fam, L, C, model, mutant=None, seed=0):
    """Every stage of one family under one model -> {stage: worst err/tol} (inf: an exact answer or T wrong)."""
    f = GB.family(fam, B, L, C, seed)
    exact = fam in GB.EXACT
    out = {}
    if "cs" in f:
        xh, nrm = emulate_normalize(f["cs"], mutant)
        yh, _ = emulate_normalize(f["cs_ref"], mutant)
        n64, tol_n, x64, tol_x = GB.normalize_ref_and_bound(f["cs"])
        out["norms"] = GB.ratio(nrm, n64, tol_n).max().item()
        out["xhat"] = GB.ratio(xh, x64, tol_x).max().item()
        if exact and not (torch.equal(nrm.double(), n64) and torch.equal(xh.double(), x64)):
            out["xhat"] = math.inf
    else:
        xh, yh, nrm = f["xhat"], f["yhat"], f["norms"]
        x64 = tol_x = None
    scale = f["scale"] or 100.0 / (B * L * L)
    grad0 = torch.zeros(B, C, L) if exact else torch.randn(B, C, L, generator=torch.Generator().manual_seed(seed))
    if fam not in GB.DENSE_ONLY:
        Dk = torch.stack([contract(torch.cat([_pad_k(xh[b]), _pad_k(yh[b])], 1),
                                   torch.cat([_pad_k(xh[b]), -_ref_half(yh[b], C, mutant)], 1), model,
                                   fp16_acc=mutant == "fp16-acc") for b in range(B)])
        T, loss = emulate_sign_ref(Dk, scale, mutant)
        abs_sum = beta_sum = 0.0
        out["T"] = out["ref-formula"] = out["g^"] = out["grad"] = 0.0
        for b in range(B):
            D, beta = GB.sign_ref_band(xh[b], yh[b])
            n, r = GB.sign_ref_check(T[b], D, beta, exact)
            out["T"] = max(out["T"], math.inf if n and exact else r)
            abs_sum += D.abs().sum().item()
            beta_sum += beta.sum().item()
            if x64 is not None:
                D_ref, rho = GB.reference_formula_band(x64[b], tol_x[b], xh[b], yh[b], GB.fp16_target(yh[b]))
                n, _ = GB.sign_ref_check(T[b], D_ref, beta + rho)
                out["ref-formula"] = max(out["ref-formula"], math.inf if n else 0.0)
            g = emulate_tx(T[b], xh[b], scale, model, mutant)
            g64, tol_g = GB.gtx_ref_and_bound(T[b], xh[b], scale)
            out["g^"] = max(out["g^"], GB.ratio(g, g64, tol_g).max().item())
            if exact and not torch.equal(g, GB.gtx_exact(T[b], xh[b], scale)):
                out["g^"] = math.inf
            want, tol = GB.project_ref_and_bound(g64, tol_g, xh[b], nrm[b], grad0[b])
            for fma in (False, True):
                gr = emulate_project(g, xh[b], nrm[b], grad0[b], fma, mutant)
                out["grad"] = max(out["grad"], GB.ratio(gr.T, want, tol).max().item())
                if exact and not torch.equal(gr.T, want.float()):
                    out["grad"] = math.inf
        tol = GB.sign_ref_loss_bound(abs_sum, beta_sum, scale, B, L, GRID, exact)
        out["loss"] = abs(loss - scale * abs_sum) / tol
    A = f["target"] if "target" in f else torch.stack([GB.fp16_target(yh[b]) for b in range(B)])
    Gk = torch.stack([contract(_pad_k(xh[b]), _pad_k(xh[b]), model) for b in range(B)])
    Td, loss_d = emulate_dense(Gk, A, scale, mutant)
    abs_sum = beta_sum = 0.0
    bad = 0
    for b in range(B):
        d1, d2, beta = GB.dense_band(xh[b], A[b])
        bad += GB.dense_check(Td[b], d1, d2, beta, exact)
        abs_sum += d1.abs().sum().item()
        beta_sum += beta.sum().item()
    out["T dense"] = math.inf if bad else 0.0
    out["loss dense"] = abs(loss_d - scale * abs_sum) / GB.dense_loss_bound(abs_sum, beta_sum, scale, B, L, exact)
    return out


def _ref_half(Y, C, mutant):
    """The reference half's B operand; the mutant drops its last K atom when that atom is partial."""
    Yp = _pad_k(Y)
    if mutant == "drop-ref-tail" and C % 64:
        Yp = Yp.clone()
        Yp[:, (Yp.shape[1] // 64 - 1) * 64:] = 0
    return Yp


# ------------------------------------------------------------------------------------------------ the tests
@pytest.mark.parametrize("L,C", SHAPES)
@pytest.mark.parametrize("fam", GB.FAMILIES)
def test_emulation_within_bound(fam, L, C):
    for model in MODELS:
        out = run(fam, L, C, model)
        for stage, r in out.items():
            _note(fam, stage, r)
            assert r <= 1.0, f"{fam} L={L} C={C} {model} {stage}: err/tol {r:.3g}"


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_mutant_is_caught(name):
    what, fam, (L, C) = MUTANTS[name]
    out = run(fam, L, C, "sequential", mutant=name)
    worst = max(out.values())
    assert worst > 1.0, f"mutant {name} ({what}) stays inside the bound on {fam}: {out}"


def test_near_tie_family_is_near_the_band():
    """The near-tie family puts at least NEAR_TIE_SHARE of the off-diagonal entries just outside the band."""
    for L, C in SHAPES:
        f = GB.family("near-tie", B, L, C)
        for b in range(B):
            D, beta = GB.sign_ref_band(f["xhat"][b], f["yhat"][b])
            off = ~torch.eye(L, dtype=torch.bool)
            near = (D.abs() > beta) & (D.abs() <= 8 * beta) & off
            if L > 1:
                assert near.sum().item() >= GB.NEAR_TIE_SHARE * L * (L - 1), (L, C, near.sum().item())


def test_coherent_family_is_one_signed():
    """Features all positive and T mostly +2: the accumulator errors of T X^ all push the same way."""
    f = GB.family("coherent", B, 257, 64)
    xh, _ = emulate_normalize(f["cs"])
    yh, _ = emulate_normalize(f["cs_ref"])
    assert (xh > 0).all()
    D, _ = GB.sign_ref_band(xh[0], yh[0])
    assert (D > 0).double().mean().item() > 0.9


def test_report_worst_ratios():
    """Prints the largest err/tol per family and stage (-s to see it)."""
    if not WORST:
        pytest.skip("no emulation ran")
    print("\nworst err/tol per family and stage (CPU emulation, every model)")
    for (fam, stage), r in sorted(WORST.items()):
        print(f"  {fam:12s} {stage:12s} {r:.3g}")
