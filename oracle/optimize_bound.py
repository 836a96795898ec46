"""Staged fp64 reference of one ``optimize_feature`` iteration (O1-O5: ``diffusion_hacked.optimize_feature``,
src/diffusion_hacked.py:416-488), a bound composed from its kernels' bounds, and input families built to break the
glue between the kernels.

CHECKER ONLY (see ``oracle/__init__``).  Nothing here restates a kernel: every stage calls the module that already
bounds it (``warp_loss_bound``, ``gram_bound``, ``step_bound``).  What this module adds is the composition, and the
test's own restatement of the glue: the resize of flows and occlusions (:437-442), the keep masks, the first matching
``correlation_matrix`` entry, the chunk-major [chunks n, C, h w] view, the weight ``intra_weight n / total``, the step.

One iteration t, evaluated on the state the GPU holds at its start (cs_t, m_t, v_t)
-------------------------------------------------------------------------------------
cs is fp32 [chunks, n, C, h, w]; B = chunks n samples of L = h w tokens.

T  temporal.  ``warp_loss_bound.reference_and_bound(cs_t, ff, bf, kf, kb)``: the fp64 gradient g_T, the loss l_T and
   their own tolerances E_T (elementwise) and e_T.
S  spatial, on cs_t viewed [B, C, L].  The kernel's X^ and norms within ``gram_bound.normalize_ref_and_bound``; its
   T equal to 2 sgn(D_64) outside the band (``sign_ref_band`` / ``sign_ref_check`` for a GramTarget, ``dense_band`` /
   ``dense_check`` for a dense target); then ``composed_ref_and_bound(cs_b, T_kernel, scale, X^, norms, grad0)`` with
   scale = weight / (B L^2) in double (``ops._gram_scale``) and grad0 the buffer the temporal kernel actually wrote
   (on the spatial-only branch it must be exactly 0).  That gives grad0 + g_S and E_S on the received grad0.
   The gradient Adam should see is g_64 = g_T + g_S, and the kernel's g is within
       E_g = E_S + E_T
   of it: |g - (grad0 + g_S)| <= E_S and |grad0 - g_T| <= E_T.  The temporal error passes through grad0 + v unchanged;
   the rounding of that add is already in E_S (``project_ref_and_bound``'s last term).
A  Adam.  Own term: ``adam_reference_and_bound(p_t, g_received, m_t, v_t, t)`` gives p', m', v' on the gradient the
   kernel received, E_own.  Propagation: the kernel's gradient lies in I = [g_64 - E_g, g_64 + E_g], so the fp64 update
   on it differs from the update on g_64 by at most
       P = max over g in I of |u(g) - u(g_64)|,   u(g) = (lr / bc1) m'(g) / (sqrt(v'(g)) / sqrt(bc2) + eps),
   m'(g) = A + c1 g, v'(g) = V + c2 g^2, A = (1 - c1) m, V = b2 v (the launcher's fp32 constants, exactly as
   ``adam_reference_and_bound`` evaluates them).  u is continuous on I, so the extremes of u - u(g_64) lie at the
   endpoints, at g = 0 (where sqrt(v') has a kink when V = 0) or at a stationary point.  With r = 1 / sqrt(bc2) and
   s = sqrt(V + c2 g^2), s' = c2 g / s and
       u' = 0  <=>  c1 (r s + eps) s = (A + c1 g) r c2 g  <=>  c1 r V + c1 eps s = r c2 A g          (s^2 = V + c2 g^2)
   Squaring c1 eps s = r (c2 A g - c1 V) gives the quadratic
       (r^2 c2^2 A^2 - c1^2 eps^2 c2) g^2 - 2 r^2 c1 c2 A V g + c1^2 V (r^2 V - eps^2) = 0,
   whose real roots in I with c2 A g - c1 V >= 0 (the unsquared equation's right side is c1 eps s >= 0) are the
   stationary points.  A spurious candidate in I could only lower the maximum's estimate to a value u actually takes,
   never raise it, so the term is exact.  p' is held to E_own + P, m' to E_own + c1 E_g, v' to
   E_own + c2 ((|g_64| + E_g)^2 - g_64^2).
   At step 1 (m = v = 0) u(g) = lr g / (|g| + eps): an element whose interval I contains 0 gets a term of about 2 lr.
   That is honest -- step 1 moves every element by +-lr whatever the size of its gradient (DESIGN §4) -- and the tests
   report the share of such elements.
Loss.  The trace's value is l_T (the temporal kernels' atomics on a zeroed accumulator) plus the Gram kernel's sum.
   ``sign_ref_loss_bound`` / ``dense_loss_bound`` charge each of the Gram kernel's n_a atomicAdds u of the running sum,
   S + scale sum beta.  Here the accumulator already holds the kernel's l_T, within e_T of l_T, so each atomic rounds at
   most u (l_T + e_T + S + scale sum beta): the composed loss tolerance is
       e = e_T + e_S + F n_a u (|l_T| + e_T),
   n_a = 8 x (CTAs of ``sign_ref_schedule``) for the recomputed target, 8 B tiles (tiles + 1) / 2 for the dense one.
AdaIN, after the last iteration: ``adain_reference_and_bound(cs_T, sample)`` on the cs the last Adam wrote (the
   content rounded to fp16 first for an fp16 sample, the reference's ``cs.to(sample.dtype)``); ``ratio16`` for fp16.

``optimize_feature64`` runs the same stages without teacher forcing, in fp64 with T = 2 sgn(D) of the fp64 features:
the CPU tests pin it against the reference's own outputs (tests/golden/optimize*.npz).
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional

import torch
import torch.nn.functional as F

from . import fresco_oracle as O
from . import gram_bound as GB
from . import step_bound as SB
from . import warp_loss_bound as WB

U = 2.0 ** -24
SAFETY = 2.0
LR = 0.2
H100_SMS = 132                      # the Gram sign kernel's persistent grid on an H100 SXM

FAMILIES = ("realistic", "integer", "tie", "eps", "balance-temporal", "balance-spatial", "masks-all", "masks-none",
            "overflow", "dense")
BRANCHES = ("full", "no-target", "temporal-off", "no-flows", "no-match", "none")


# ------------------------------------------------------------------------------------------------ the glue, restated
class Prep(NamedTuple):
    ff: torch.Tensor                # fp32 [n, 2, h, w]
    bf: torch.Tensor
    kf: torch.Tensor                # fp32 [n, h, w] in {0, 1}
    kb: torch.Tensor


def restate_prep(flows, occs, h: int) -> Prep:
    """src/diffusion_hacked.py:437-442: flows scaled and bilinearly resized to the feature map, occlusions max-pooled by
    int(1 / scale); keep = 1 - occ."""
    scale = h * 1.0 / flows[0].shape[2]
    kernel = int(1 / scale)
    bf = F.interpolate(flows[1] * scale, scale_factor=scale, mode="bilinear")
    ff = F.interpolate(flows[0] * scale, scale_factor=scale, mode="bilinear")
    bo = F.max_pool2d(occs[1].unsqueeze(1), kernel_size=kernel)
    fo = F.max_pool2d(occs[0].unsqueeze(1), kernel_size=kernel)
    n, _, hh, w = ff.shape
    return Prep(ff.float().contiguous(), bf.float().contiguous(), (1 - fo).reshape(n, hh, w).float().contiguous(),
                (1 - bo).reshape(n, hh, w).float().contiguous())


def first_match(correlation_matrix, L: int):
    """The entry optimize_feature uses (:446-450): the first whose shape[1] is the token count."""
    for t in correlation_matrix:
        if t.shape[1] == L:
            return t
    return None


class Glue(NamedTuple):
    """What one call's iterations depend on besides the state: the test's restatement of the call's glue."""
    chunks: int
    n: int
    C: int
    h: int
    w: int
    prep: Optional[Prep]            # None: no temporal term
    target: object                  # None: no spatial term; else a dense [B, L, L] tensor or the GramTarget's yhat
    dense: bool
    weight: float                   # intra_weight n / total

    @property
    def scale(self) -> float:
        B, L = self.chunks * self.n, self.h * self.w
        return float(self.weight) / (B * L * L)


def glue(sample, flows, occs, correlation_matrix, intra_weight, chunks, optimize_temporal=True) -> Glue:
    """The glue of an unsharded call, restated (None: the call returns ``sample`` without a launch)."""
    _, C, h, w = sample.shape
    n = sample.shape[0] // chunks
    have_t = flows is not None and occs is not None and optimize_temporal
    if not have_t and (intra_weight == 0 or len(correlation_matrix) == 0):
        return None
    prep = restate_prep(flows, occs, h) if have_t else None
    t = first_match(correlation_matrix, h * w) if intra_weight > 0 else None
    dense = t is not None and not hasattr(t, "yhat")
    target = None if t is None else (t.to(torch.float32) if dense else t.yhat)
    total = n                                   # unsharded: this call holds the whole batch
    return Glue(chunks, n, C, h, w, prep, target, dense, intra_weight * (float(n) / float(total)))


# ------------------------------------------------------------------------------------------------ stages
def ratio(out, ref, tol):
    """|out - ref| / tol elementwise (0 where equal; NaN counts as infinitely wrong)."""
    return WB.ratio(out, ref, tol)


def temporal_stage(cs, prep: Prep):
    """-> warp_loss_bound's dict (grad, grad_tol, loss, loss_tol, ...) for cs [chunks, n, C, h, w]."""
    return WB.reference_and_bound(cs, prep.ff, prep.bf, prep.kf, prep.kb)


def n_atomics(g: Glue, grid: int) -> int:
    B, L = g.chunks * g.n, g.h * g.w
    if g.dense:
        tiles = (L + 127) // 128
        return 8 * B * tiles * (tiles + 1) // 2
    return 8 * GB.sign_ref_schedule(B, L, grid)[1]


def spatial_stage(g: Glue, cs, xhat, norms, tsign, grad0, grid: int, ratios=None):
    """The kernel's X^, norms and T checked against the band; -> dict want = grad0 + g_S [B, C, L] (fp64), tol (E_S on
    the received grad0), v = want - grad0, loss / loss_tol (the Gram kernel's own), wrong (signs outside the band)."""
    B, L = g.chunks * g.n, g.h * g.w
    cs_b = cs.reshape(B, g.C, L)
    GB.check_normalize(cs_b, xhat, norms, ratios=ratios)
    want = torch.empty(B, g.C, L, dtype=torch.float64, device=cs.device)
    tol = torch.empty_like(want)
    abs_sum = beta_sum = 0.0
    wrong = 0
    g0 = grad0.reshape(B, g.C, L)
    for b in range(B):
        if g.dense:
            d1, d2, beta = GB.dense_band(xhat[b], g.target[b])
            wrong += GB.dense_check(tsign[b], d1, d2, beta)
            abs_sum += d1.abs().sum().item()
            del d1, d2
        else:
            D, beta = GB.sign_ref_band(xhat[b], g.target[b])
            wrong += GB.sign_ref_check(tsign[b], D, beta)[0]
            abs_sum += D.abs().sum().item()
            del D
        beta_sum += beta.sum().item()
        del beta
        wb, tb = GB.composed_ref_and_bound(cs_b[b], tsign[b], g.scale, xhat[b], norms[b], g0[b])
        want[b], tol[b] = wb.T, tb.T
    if g.dense:
        loss_tol = GB.dense_loss_bound(abs_sum, beta_sum, g.scale, B, L)
    else:
        loss_tol = GB.sign_ref_loss_bound(abs_sum, beta_sum, g.scale, B, L, grid)
    return {"want": want, "tol": tol, "v": want - g0.double(), "loss": g.scale * abs_sum, "loss_tol": loss_tol,
            "wrong": wrong}


def adam_update(g, m, v, k):
    """u(g) of the module docstring in fp64 (k: ``step_bound.adam_constants``)."""
    m1 = m + (g - m) * k["c1"]
    v1 = v * k["b2"] + g * g * k["c2"]
    return k["step_size"] * m1 / (v1.sqrt() / k["sqrt_bc2"] + k["eps"])


def adam_candidates(g64, E_g, m, v, k):
    """The points of I = [g64 - E_g, g64 + E_g] where |u(g) - u(g64)| can be largest: both ends, 0 and the stationary
    points (module docstring) -> [..., 5] (NaN where a candidate does not exist)."""
    g64, E_g, m, v = (t.double() for t in (g64, E_g, m, v))
    c1, c2, e = k["c1"], k["c2"], k["eps"]
    r = 1.0 / k["sqrt_bc2"]
    A = m - m * c1
    V = v * k["b2"]
    lo, hi = g64 - E_g, g64 + E_g
    a = r * r * c2 * c2 * A * A - c1 * c1 * e * e * c2
    b = -2 * r * r * c1 * c2 * A * V
    c = c1 * c1 * V * (r * r * V - e * e)
    disc = b * b - 4 * a * c
    sq = disc.clamp_min(0).sqrt()
    q = -0.5 * (b + torch.where(b >= 0, sq, -sq))
    nan = torch.full_like(g64, float("nan"))
    lin = a == 0
    r1 = torch.where(lin, torch.where(b != 0, -c / b, nan), q / a)
    r2 = torch.where(lin | (q == 0), nan, c / q)
    roots = []
    for x in (r1, r2):
        ok = (disc >= 0) & torch.isfinite(x) & (x >= lo) & (x <= hi)
        rhs = c2 * A * x - c1 * V
        ok &= rhs >= -1e-9 * (c2 * (A * x).abs() + c1 * V)
        roots.append(torch.where(ok, x, nan))
    zero = torch.where((lo <= 0) & (hi >= 0), torch.zeros_like(g64), nan)
    return torch.stack([lo, hi, zero] + roots, -1)


def adam_propagation(g64, E_g, m, v, step, lr=LR):
    """P = max over g in [g64 - E_g, g64 + E_g] of |u(g) - u(g64)| -> (P, the candidate attaining it)."""
    k = SB.adam_constants(step, lr)
    g64, E_g, m, v = (t.double() for t in (g64, E_g, m, v))
    cand = adam_candidates(g64, E_g, m, v, k)
    u0 = adam_update(g64, m, v, k)
    du = (adam_update(cand, m[..., None], v[..., None], k) - u0[..., None]).abs()
    du = torch.nan_to_num(du, nan=-1.0)
    P, i = du.max(-1)
    return P.clamp_min(0.0), torch.gather(cand, -1, i[..., None])[..., 0]


def adam_stage(p, g_recv, m, v, step, g64, E_g, lr=LR):
    """-> {"p"|"m"|"v": (ref on g64, composed tol, ref on g_recv, own tol)} and the share of elements whose gradient
    interval contains 0 (step 1: the saturated ones)."""
    own = SB.adam_reference_and_bound(p, g_recv, m, v, step, lr)
    at64 = SB.adam_reference_and_bound(p, g64, m, v, step, lr)
    P, _ = adam_propagation(g64, E_g, m, v, step, lr)
    k = SB.adam_constants(step, lr)
    g64d, E = g64.double(), E_g.double()
    prop = {"p": P, "m": k["c1"] * E, "v": k["c2"] * ((g64d.abs() + E) ** 2 - g64d ** 2)}
    out = {key: (at64[key][0], own[key][1] + prop[key], own[key][0], own[key][1]) for key in ("p", "m", "v")}
    out["saturated"] = ((g64d - E <= 0) & (g64d + E >= 0)).double().mean().item()
    return out


def loss_stage(g: Glue, tem, spa, grid: int):
    """-> (reference, tolerance) of the trace's value after both terms."""
    lT, eT = (tem["loss"], tem["loss_tol"]) if tem is not None else (0.0, 0.0)
    if spa is None:
        return lT, eT
    corr = SAFETY * n_atomics(g, grid) * U * (abs(lT) + eT)
    return lT + spa["loss"], eT + spa["loss_tol"] + corr


def adain_stage(content, sample):
    """content fp32 [B, C, h, w] (the cs the last Adam wrote), sample [B, C, h, w] -> (ref, tol) shaped like sample."""
    B, C, h, w = sample.shape
    ref, tol = SB.adain_reference_and_bound(content.reshape(B * C, h * w), sample.reshape(B * C, h * w))
    return ref.reshape(sample.shape), tol.reshape(sample.shape)


def adain_ratio(out, ref, tol):
    return (SB.ratio16 if out.dtype == torch.float16 else SB.ratio)(out, ref, tol)


# ------------------------------------------------------------------------------------------------ one iteration, checked
class StageFailure(AssertionError):
    pass


def check_iteration(g: Glue, rec, t: int, grid: int, worst=None, family="", integer=False):
    """Everything one iteration recorded, against the staged reference on its own starting state.

    ``rec``: cs, m, v (before Adam; cs also what the loss kernels read), grad_T (the buffer after the temporal kernel,
    None without that term), xhat, norms, tsign (None without the spatial term), grad0 (the buffer the projection
    kernel received), grad (what Adam received), step, lr, p1, m1, v1 (after Adam), loss (the trace's value or None).
    A failure names the iteration, the stage and whether the stage's own bound alone also fails.  ``worst``: dict
    (family, stage) -> worst composed err/tol.  Returns the share of elements whose gradient interval contains 0."""
    def record(stage, r):
        if worst is not None:
            key = (family, stage)
            worst[key] = max(worst.get(key, 0.0), r)

    def fail(stage, r, own):
        raise StageFailure(f"iteration {t}, stage {stage}: worst err/tol {r:.3g} against the composed bound; its own bound "
                           f"alone {'also fails' if own > 1 else 'holds'} ({own:.3g})")

    assert rec["step"] == t, f"iteration {t}: Adam was given step {rec['step']}"
    assert rec["lr"] == LR, f"iteration {t}: Adam lr {rec['lr']}"
    cs = rec["cs"]
    B, L = g.chunks * g.n, g.h * g.w
    tem = spa = None
    g64 = torch.zeros(cs.shape, dtype=torch.float64, device=cs.device)
    E_g = torch.zeros_like(g64)
    if g.prep is not None:
        tem = temporal_stage(cs, g.prep)
        r = ratio(rec["grad_T"], tem["grad"], tem["grad_tol"]).max().item()
        record("temporal", r)
        if r > 1:
            fail("temporal", r, r)
        if integer:
            want, _ = WB.exact_grad(tem)
            if not torch.equal(rec["grad_T"], want.to(rec["grad_T"].device)):
                raise StageFailure(f"iteration {t}, stage temporal: integer family not bit-exact")
        g64, E_g = tem["grad"], tem["grad_tol"]
    if g.target is not None:
        grad0 = rec["grad0"]
        if g.prep is None and not bool((grad0 == 0).all()):
            raise StageFailure(f"iteration {t}, stage spatial: the gradient buffer is not zero on the spatial-only branch")
        if g.prep is not None and not torch.equal(grad0, rec["grad_T"]):
            raise StageFailure(f"iteration {t}, stage spatial: the projection did not add onto the temporal gradient")
        try:
            spa = spatial_stage(g, cs, rec["xhat"], rec["norms"], rec["tsign"], grad0, grid)
        except AssertionError as e:
            raise StageFailure(f"iteration {t}, stage spatial: {e}") from None
        if spa["wrong"]:
            raise StageFailure(f"iteration {t}, stage spatial: {spa['wrong']} signs outside the band")
        got = rec["grad"].reshape(B, g.C, L)
        own = ratio(got, spa["want"], spa["tol"]).max().item()
        g64 = g64 + spa["v"].reshape(cs.shape)
        E_g = E_g + spa["tol"].reshape(cs.shape)
        r = ratio(rec["grad"], g64, E_g).max().item()
        record("spatial", r)
        if r > 1:
            fail("spatial", r, own)
    elif g.prep is not None and not torch.equal(rec["grad"], rec["grad_T"]):
        raise StageFailure(f"iteration {t}, stage adam: Adam did not receive the temporal gradient")
    ada = adam_stage(rec["cs"], rec["grad"], rec["m"], rec["v"], t, g64, E_g)
    for key in ("p", "m", "v"):
        ref, tol, ref_own, tol_own = ada[key]
        got = rec[key + "1"]
        r = ratio(got, ref, tol).max().item()
        record("adam", r)
        if r > 1:
            fail(f"adam ({key})", r, ratio(got, ref_own, tol_own).max().item())
    if rec.get("loss") is not None:
        ref, tol = loss_stage(g, tem, spa, grid)
        r = abs(rec["loss"] - ref) / tol if tol > 0 else float(rec["loss"] != ref) * math.inf
        record("loss", r)
        if r > 1:
            fail("loss", r, r)
    return ada["saturated"]


# ------------------------------------------------------------------------------------------------ fp64 iterations
def kernel_like(g: Glue, cs):
    """The Gram kernels' operands for cs as an exact normalisation rounded once gives them: X^ = fp16(x_64), norms fp32,
    T = 2 sgn(D) of those (dense: sgn(G - A) + sgn(G - A^T))."""
    B, L = g.chunks * g.n, g.h * g.w
    n64, _, x64, _ = GB.normalize_ref_and_bound(cs.reshape(B, g.C, L).float())
    xhat, norms = x64.half(), n64.float()
    T = torch.empty(B, L, L, dtype=torch.float16, device=cs.device)
    loss = 0.0
    for b in range(B):
        Tb, s = sign64(xhat[b], g.target[b], g.dense)
        T[b] = Tb.half()
        loss += s
    return xhat, norms, T, g.scale * loss


def sign64(X, target_b, dense: bool):
    """One sample: T and sum |D| of features X [L, C] in fp64 -- dense: sgn(G - A) + sgn(G - A^T) and sum |G - A|
    (the reference's l1 over its stored target); recomputed: 2 sgn(X X^T - Y^ Y^T) and its sum."""
    X = X.double()
    G = X @ X.T
    if dense:
        A = target_b.double()
        D = G - A
        return torch.sign(D) + torch.sign(G - A.T), D.abs().sum().item()
    Y = target_b.double()
    D = G - Y @ Y.T
    return 2 * torch.sign(D), D.abs().sum().item()


def project64(T, X, nrm, scale: float):
    """One sample: the gradient of the Gram-L1 term through the normalisation, [L, C] fp64:
    (scale T X - (scale T X . X) X) / ||cs||."""
    X = X.double()
    gx = scale * (T.double() @ X)
    return (gx - (gx * X).sum(1, keepdim=True) * X) / nrm.double()[:, None]


def spatial64(g: Glue, cs):
    """The exact Gram-L1 term of cs: (loss, gradient [chunks, n, C, h, w] fp64) from the exactly normalised features."""
    B, L = g.chunks * g.n, g.h * g.w
    n64, _, x64, _ = GB.normalize_ref_and_bound(cs.reshape(B, g.C, L))
    loss = 0.0
    grad = torch.empty(B, g.C, L, dtype=torch.float64, device=cs.device)
    for b in range(B):
        T, s = sign64(x64[b], g.target[b], g.dense)
        loss += s
        grad[b] = project64(T, x64[b], n64[b], g.scale).T
    return g.scale * loss, grad.reshape(cs.shape)


MUTANTS = {
    # glue mutant -> (family, branch, iteration, stage that catches it)
    "adam-step+1": ("realistic", "full", 1, "adam"),
    "grad-not-zeroed": ("realistic", "temporal-off", 2, "spatial"),
    "weight-unsharded-half": ("realistic", "full", 1, "spatial"),
    "frame-major-view": ("realistic", "full", 1, "spatial"),
    "keep-occ": ("realistic", "full", 1, "temporal"),
    "flows-swapped": ("realistic", "full", 1, "temporal"),
    "last-match": ("dense", "full", 1, "spatial"),
    "adain-style-cs": ("realistic", "full", 1, "adain"),
    "adain-no-cast": ("eps", "full", 1, "adain"),
    "temporal-doubled": ("eps", "full", 1, "temporal"),
    "loss-without-spatial": ("realistic", "full", 1, "loss"),
}


def _mutated_glue(g: Glue, mutant, correlation_matrix=None):
    if mutant == "weight-unsharded-half":
        return g._replace(weight=g.weight / 2)
    if mutant == "keep-occ" and g.prep is not None:
        return g._replace(prep=g.prep._replace(kf=1 - g.prep.kf, kb=1 - g.prep.kb))
    if mutant == "flows-swapped" and g.prep is not None:
        return g._replace(prep=g.prep._replace(ff=g.prep.bf, bf=g.prep.ff))
    if mutant == "last-match":
        last = [t for t in correlation_matrix if t.shape[1] == g.h * g.w][-1]
        return g._replace(target=last.to(torch.float32) if g.dense else last.yhat)
    return g


def iteration64(g: Glue, state, t: int, mutant=None, correlation_matrix=None, gram_operands=None):
    """One iteration in fp64 from ``state`` (cs, m, v, grad = the buffer's previous content) -> dict grad_T, grad, loss,
    p, m, v (fp64).  ``gram_operands``: "exact" (fp64 features, for ``optimize_feature64``) or "kernel" (``kernel_like``,
    so T matches the operands the bound is evaluated on).  ``mutant``: one of ``MUTANTS``."""
    cs, m, v = state["cs"], state["m"], state["v"]
    mg = _mutated_glue(g, mutant, correlation_matrix)
    out = {"grad_T": None}
    loss = 0.0
    grad = torch.zeros(cs.shape, dtype=torch.float64, device=cs.device)
    if mg.prep is not None:
        tem = temporal_stage(cs, mg.prep)
        grad = tem["grad"] * (2 if mutant == "temporal-doubled" else 1)
        loss += tem["loss"]
        out["grad_T"] = grad
    elif mutant == "grad-not-zeroed" and state.get("grad") is not None:
        grad = state["grad"].double()
    if mg.target is not None:
        view = cs
        if mutant == "frame-major-view":
            view = cs.transpose(0, 1).contiguous()
        if gram_operands == "kernel":
            xhat, norms, T, lS = kernel_like(mg, view)
            B, L = g.chunks * g.n, g.h * g.w
            n64, _, x64, _ = GB.normalize_ref_and_bound(view.reshape(B, g.C, L))
            vS = torch.stack([project64(T[b], x64[b], n64[b], mg.scale).T for b in range(B)]).reshape(view.shape)
        else:
            lS, vS = spatial64(mg, view)
        if mutant == "frame-major-view":
            vS = vS.transpose(0, 1)
        grad = grad + vS
        if mutant != "loss-without-spatial":
            loss += lS
    out["grad"], out["loss"] = grad, loss
    step = t + 1 if mutant == "adam-step+1" else t
    a = SB.adam_reference_and_bound(cs, grad, m, v, step)
    out["p"], out["m"], out["v"] = a["p"][0], a["m"][0], a["v"][0]
    return out


def adain64(content, sample, mutant=None):
    """AdaIN of the final features in fp64 (``adain_stage``'s reference); mutants: the optimised features as the style,
    or the content not cast to the sample's dtype first."""
    if mutant == "adain-style-cs":
        return adain_stage(content, content.to(sample.dtype))[0]
    if mutant == "adain-no-cast" and sample.dtype != torch.float32:
        B, C, h, w = sample.shape
        ref, _ = SB.adain_reference_and_bound(content.reshape(B * C, h * w), sample.reshape(B * C, h * w).float())
        return ref.reshape(sample.shape)
    return adain_stage(content, sample)[0]


def composed_bounds(g: Glue, state, t: int, grid: int = H100_SMS):
    """The composed bound of iteration t from ``state``, evaluated on the operands the kernels would receive there
    (``kernel_like``; the temporal buffer as fp32): {"temporal": E_T, "spatial": E_g, "adam": p's tolerance,
    "loss": the loss tolerance} -- the yardstick a mutant's distance from the iteration is measured in."""
    cs = state["cs"].float()
    out = {}
    tem = spa = None
    E_g = torch.zeros(cs.shape, dtype=torch.float64, device=cs.device)
    g64 = torch.zeros_like(E_g)
    grad0 = torch.zeros_like(cs)
    if g.prep is not None:
        tem = temporal_stage(cs, g.prep)
        out["temporal"] = tem["grad_tol"]
        g64, E_g, grad0 = tem["grad"], tem["grad_tol"], tem["grad"].float()
    if g.target is not None:
        xhat, norms, T, _ = kernel_like(g, cs)
        spa = spatial_stage(g, cs, xhat, norms, T, grad0, grid)
        g64 = g64 + spa["v"].reshape(cs.shape)
        E_g = E_g + spa["tol"].reshape(cs.shape)
    out["spatial"] = E_g
    out["adam"] = adam_stage(cs, g64.float(), state["m"].float(), state["v"].float(), t, g64, E_g)["p"][1]
    out["loss"] = loss_stage(g, tem, spa, grid)[1]
    return out


def optimize_feature64(sample, flows, occs, correlation_matrix=(), intra_weight=1e2, iters=20, unet_chunk_size=2,
                       optimize_temporal=True):
    """optimize_feature from the stages, not teacher-forced, in fp64 -> (out in sample's dtype, losses, states).
    ``states[t - 1]``: the state iteration t starts from (cs, m, v, grad = the buffer's previous content)."""
    g = glue(sample, flows, occs, correlation_matrix, intra_weight, unet_chunk_size, optimize_temporal)
    if g is None:
        return sample, [], []
    cs = sample.to(torch.float32).reshape(g.chunks, g.n, g.C, g.h, g.w).double()
    state = {"cs": cs, "m": torch.zeros_like(cs), "v": torch.zeros_like(cs), "grad": None}
    losses, states = [], []
    for it in range(1, iters + 1):
        states.append(state)
        o = iteration64(g, state, it, gram_operands="exact")
        losses.append(o["loss"])
        state = {"cs": o["p"], "m": o["m"], "v": o["v"], "grad": o["grad"]}
    out = adain_stage(state["cs"].reshape(sample.shape), sample)[0]
    return out.to(sample.dtype), losses, states + [state]


# ------------------------------------------------------------------------------------------------ input families
class Case(NamedTuple):
    family: str
    sample: torch.Tensor            # [chunks n, C, h, w], fp32 or fp16
    flows: Optional[list]           # [fwd, bwd] fp32 [n, 2, H, W]
    occs: Optional[list]            # [fwd, bwd] fp32 [n, H, W]
    targets: list                   # ("gram", yhat [B, L', C] fp16) or ("dense", [B, L', L'] fp32) entries, in order
    intra_weight: float
    optimize_temporal: bool
    chunks: int


def _yhat(feat):
    """gram_targets' normalised features (src/diffusion_hacked.py:889-893) of [B, C, h, w] -> [B, L, C] fp16."""
    v = feat.double().reshape(feat.shape[0], feat.shape[1], -1).transpose(1, 2)
    return (v / v.norm(dim=2, keepdim=True)).half().contiguous()


def correlation_list(case: Case, gram_target_cls, device=None):
    """The case's correlation_matrix with GramTarget entries built by ``gram_target_cls``."""
    out = []
    for kind, t in case.targets:
        t = t.to(device) if device is not None else t
        out.append(gram_target_cls(t) if kind == "gram" else t)
    return out


def _contract(n, h, w):
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    c = torch.stack([((w - 1) / 2 - xs) * 0.75 + 0.3, ((h - 1) / 2 - ys) * 0.75 - 0.2])
    return c[None].repeat(n, 1, 1, 1)


def make_case(family, chunks=2, N=3, C=16, h=8, w=8, dtype=torch.float32, seed=0, res=None, branch="full") -> Case:
    """One call's operands.  ``res``: (H, W) of the flows (default 8h x 8w); ``branch`` switches the terms as
    ``BRANCHES`` names them.  realistic is ``_layer_case`` of tests/test_gpu_parity_r2.py: synth_flows, features with a
    shared per-channel base, the target the Gram of perturbed features."""
    g = torch.Generator().manual_seed(seed * 7919 + sum(map(ord, family)) + 31 * h + C)
    H, W = res if res is not None else (8 * h, 8 * w)
    B = chunks * N
    intra = 1e2
    base = torch.randn(chunks, 1, C, h, w, generator=g)
    cs = base + 0.5 * torch.randn(chunks, N, C, h, w, generator=g)
    flows = occs = None
    if family in ("integer", "overflow", "tie"):
        H, W = h, w                                 # flows at the feature resolution: the resize is the identity
    if family == "integer":
        # integer flows, every bilinear weight 0 or 1 (WB's integer family): the temporal gradient k (ga + cb) is exact
        fwd = torch.randint(-3, 4, (N, 2, h, w), generator=g).float()
        bwd = torch.randint(-3, 4, (N, 2, h, w), generator=g).float()
        occ = [(torch.rand(N, h, w, generator=g) < 0.2).float() for _ in range(2)]
        flows, occs = [fwd, bwd], occ
        cs = (cs * 256).round() / 256
    elif family == "tie":
        # identical frames, zero flow: every temporal residual is exactly 0
        cs = cs[:, :1].expand(chunks, N, C, h, w).contiguous()
        flows = [torch.zeros(N, 2, h, w), torch.zeros(N, 2, h, w)]
        occs = [(torch.rand(N, h, w, generator=g) < 0.2).float() for _ in range(2)]
    elif family == "overflow":
        # contracting flows (test_temporal_loss_adjoint_overflow_path): ELL rows of more than 8 taps
        fwd = torch.randn(N, 2, h, w, generator=g) * 1.5
        bwd = torch.randn(N, 2, h, w, generator=g) * 1.5
        bwd[0::2] = _contract(len(range(0, N, 2)), h, w)
        fwd[1::2] = _contract(len(range(1, N, 2)), h, w)
        flows = [fwd, bwd]
        occs = [(torch.rand(N, h, w, generator=g) > 0.8).float() for _ in range(2)]
    else:
        flows, occs = O.synth_flows(N, H, W, seed=seed + 17 * h, mag=12.0)
        if family == "masks-all":
            occs = [torch.ones_like(o) for o in occs]
        elif family == "masks-none":
            occs = [torch.zeros_like(o) for o in occs]
    if family == "eps":
        # planes at 8 +- 0.05, gradients of order eps: the temporal k = 2 / numel of a large plane count, the Gram term
        # weighted 1e-6
        cs = 8.0 + 0.05 * torch.randn(chunks, N, C, h, w, generator=g)
        intra = 1e-6
    elif family == "balance-temporal":
        intra = 1e-2
    elif family == "balance-spatial":
        intra = 1e4
    feats = cs.reshape(B, C, h, w)
    if family == "tie":
        targets = [("gram", _yhat(feats.to(dtype)))]          # the Gram of the sample itself: D = 0 on exact operands
    else:
        ref = feats + 0.7 * torch.randn(feats.shape, generator=g)
        targets = [("gram", _yhat(ref))]
    if family == "dense":
        # the reference's own fp32 [B, L, L]: a non-matching entry, then two matching ones (the first must be used)
        other = torch.randn(B, C, max(h // 2, 1), w, generator=g)
        y0 = _yhat(other).double()
        y1 = _yhat(ref).double()
        y2 = _yhat(feats + 0.7 * torch.randn(feats.shape, generator=g)).double()
        targets = [("dense", (y @ y.transpose(1, 2)).float()) for y in (y0, y1, y2)]
    if family == "integer":
        targets = []
    sample = feats.to(dtype).contiguous()
    optimize_temporal = True
    if branch == "no-target":
        targets = []
    elif branch == "temporal-off":
        optimize_temporal = False
    elif branch == "no-flows":
        flows = occs = None
    elif branch == "no-match":
        targets = [(k, t[:, : t.shape[1] // 2] if k == "gram" else t[:, :t.shape[1] // 2, :t.shape[1] // 2])
                   for k, t in targets]
    elif branch == "none":
        flows = occs = None
        targets = []
    return Case(family, sample, flows, occs, targets, intra, optimize_temporal, chunks)


def family_property(case: Case, g: Glue) -> None:
    """What the family is built to do, asserted on its operands (at iteration 1)."""
    fam = case.family
    cs = case.sample.float().reshape(g.chunks, g.n, g.C, g.h, g.w)
    if fam == "integer":
        assert g.target is None and g.prep is not None
        for fl in list(g.prep.ff) + list(g.prep.bf):
            w_ = WB.taps64(fl)["w"]
            assert ((w_ == 0) | (w_ == 1)).all(), "a weight other than 0 or 1"
        WB.exact_grad(temporal_stage(cs, g.prep))              # asserts ga and cb exact in fp32
    elif fam == "tie":
        tem = temporal_stage(cs, g.prep)
        assert bool((tem["grad"] == 0).all()) and tem["loss"] == 0.0, "a nonzero temporal residual"
        xhat = kernel_like(g, cs)[0]
        for b in range(g.chunks * g.n):
            D, beta = GB.sign_ref_band(xhat[b], g.target[b])
            assert bool((D.abs() <= beta).all()), "D outside the band"
    elif fam == "eps":
        tem = temporal_stage(cs, g.prep)
        _, vS = spatial64(g, cs)
        gg = (tem["grad"] + vS).abs()
        share = ((gg > 0) & (gg < 1e3 * 1e-8)).double().mean().item()
        assert share > 0.5, f"only {share:.2f} of the gradients within 1e3 eps"
        assert case.sample.dtype == torch.float16
    elif fam in ("balance-temporal", "balance-spatial"):
        tem = temporal_stage(cs, g.prep)
        _, vS = spatial64(g, cs)
        rT, rS = tem["grad"].abs().mean().item(), vS.abs().mean().item()
        assert (rT > 10 * rS) if fam == "balance-temporal" else (rS > 10 * rT), (fam, rT, rS)
    elif fam in ("masks-all", "masks-none"):
        want = 0.0 if fam == "masks-all" else 1.0
        assert bool((g.prep.kf == want).all()) and bool((g.prep.kb == want).all())
    elif fam == "overflow":
        over = 0
        for fl in list(g.prep.ff) + list(g.prep.bf):
            T = WB.taps32(fl)
            keep = (T["w"] * 65535.0).round() > 0
            cnt = torch.zeros(g.h * g.w).index_add_(0, T["idx"][keep], torch.ones(int(keep.sum())))
            over += int((cnt > 8).sum())
        assert over > 0, "no ELL row overflows"
    elif fam == "dense":
        L = g.h * g.w
        shapes = [t.shape[1] for _, t in case.targets]
        assert shapes[0] != L and shapes[1] == shapes[2] == L
        assert not torch.equal(case.targets[1][1], case.targets[2][1])
        assert torch.equal(g.target.cpu(), case.targets[1][1].float())
    elif fam == "realistic":
        tem = temporal_stage(cs, g.prep)
        assert tem["in_band"] < 0.05 and 0 < g.prep.kf.mean().item() < 1


# ------------------------------------------------------------------------------------------------ a spy on ``ops``
SPIED = ("warp_adjoint_pair", "warp_loss_fwd_bwd", "gram_normalize", "gram_sign_ref", "gram_sign", "gram_grad",
         "adam_step", "adain")


class OpsSpy:
    """Wraps the ``ops`` entry points optimize_feature reaches (install with a pytest ``monkeypatch``).  Per call it
    records the launch ``last_kernel`` names, checks the operands against the test's restated glue ``g`` (bit for bit)
    and, inside the Adam wrapper, checks the whole iteration with ``check_iteration`` and drops its clones (one state
    at layer 3 is 168 MB).  ``check_at``: the iterations to check (None: all); ``after_adam``: called with (t, cs, grad,
    m, v) after every Adam step."""

    def __init__(self, ops, last_kernel, g: Glue, sample, grid, family="", worst=None, check_at=None, integer=False,
                 after_adam=None):
        self.ops, self.last_kernel, self.g, self.sample, self.grid = ops, last_kernel, g, sample, grid
        self.family, self.worst, self.check_at, self.integer, self.after_adam = family, worst, check_at, integer, after_adam
        self.launches, self.t, self.rec, self.losses, self.saturated, self.adain_ratio = [], 1, {}, [], [], None
        self.real = {name: getattr(ops, name) for name in SPIED}

    def install(self, monkeypatch):
        for name in SPIED:
            monkeypatch.setattr(self.ops, name, getattr(self, name))

    def _checking(self):
        return self.check_at is None or self.t in self.check_at

    def _launched(self, what):
        self.launches.append((self.t, what, self.last_kernel()))

    def warp_adjoint_pair(self, bwd_flow, fwd_flow):
        assert torch.equal(bwd_flow, self.g.prep.bf) and torch.equal(fwd_flow, self.g.prep.ff), "adjoint of other flows"
        out = self.real["warp_adjoint_pair"](bwd_flow, fwd_flow)
        self._launched("warp_adjoint_pair")
        return out

    def warp_loss_fwd_bwd(self, cs, fwd_flow, bwd_flow, fwd_keep, bwd_keep, grad, loss_acc=None, **kw):
        g = self.g
        assert g.prep is not None, "temporal term on a call without one"
        for got, want, what in ((fwd_flow, g.prep.ff, "fwd flow"), (bwd_flow, g.prep.bf, "bwd flow"),
                                (fwd_keep, g.prep.kf, "fwd keep"), (bwd_keep, g.prep.kb, "bwd keep")):
            assert torch.equal(got, want), f"iteration {self.t}: the temporal kernel's {what} differs from the restatement"
        if self.t == 1:
            assert torch.equal(cs, self.sample.float().reshape(cs.shape)), "cs_1 is not sample.float()"
        if self._checking():
            self.rec["cs"] = cs.clone()
        out = self.real["warp_loss_fwd_bwd"](cs, fwd_flow, bwd_flow, fwd_keep, bwd_keep, grad, loss_acc, **kw)
        self._launched("warp_loss_fwd_bwd")
        self.loss_acc = loss_acc
        if self._checking():
            self.rec["grad_T"] = grad.clone()
        return out

    def gram_normalize(self, cs_bcl):
        g = self.g
        B, L = g.chunks * g.n, g.h * g.w
        assert tuple(cs_bcl.shape) == (B, g.C, L) and cs_bcl.is_contiguous(), "spatial view"
        out = self.real["gram_normalize"](cs_bcl)
        self._launched("gram_normalize")
        if self._checking():
            self.rec.setdefault("cs", cs_bcl.reshape(g.chunks, g.n, g.C, g.h, g.w).clone())
            self.rec["xhat"], self.rec["norms"] = out
        return out

    def _sign(self, name, xhat, target, weight, loss_acc=None):
        g = self.g
        assert weight == g.weight, f"iteration {self.t}: Gram weight {weight}, want {g.weight}"
        assert (name == "gram_sign") == g.dense and torch.equal(target, g.target), "another correlation_matrix entry"
        out = self.real[name](xhat, target, weight, loss_acc)
        self._launched(name)
        self.loss_acc = loss_acc
        if self._checking():
            self.rec["tsign"] = out
        return out

    def gram_sign_ref(self, xhat, yhat, weight, loss_acc=None):
        return self._sign("gram_sign_ref", xhat, yhat, weight, loss_acc)

    def gram_sign(self, xhat, target, weight, loss_acc=None):
        return self._sign("gram_sign", xhat, target, weight, loss_acc)

    def gram_grad(self, tsign, xhat, norms, grad_bcl, weight):
        if self._checking():
            self.rec["grad0"] = grad_bcl.clone().reshape(self.rec["cs"].shape)
        out = self.real["gram_grad"](tsign, xhat, norms, grad_bcl, weight)
        self._launched("gram_grad")
        return out

    def adam_step(self, param, grad, exp_avg, exp_avg_sq, step, lr=0.2, **kw):
        t = self.t
        if t == 1:
            assert not exp_avg.any() and not exp_avg_sq.any(), "m_1, v_1 not zero"
        rec = self.rec
        if self._checking():
            rec.setdefault("cs", param.clone())
            assert torch.equal(rec["cs"], param), "cs moved between the loss kernels and Adam"
            rec.update(m=exp_avg.clone(), v=exp_avg_sq.clone(), step=step, lr=lr)
        self.real["adam_step"](param, grad, exp_avg, exp_avg_sq, step, lr, **kw)
        self._launched("adam_step")
        loss = getattr(self, "loss_acc", None)
        self.losses.append(None if loss is None else float(loss.item()))
        if self._checking():
            rec.update(grad=grad, p1=param, m1=exp_avg, v1=exp_avg_sq, loss=self.losses[-1])
            self.saturated.append((t, check_iteration(self.g, rec, t, self.grid, self.worst, self.family, self.integer)))
        if self.after_adam is not None:
            self.after_adam(t, param, grad, exp_avg, exp_avg_sq)
        self.rec, self.t = {}, t + 1

    def adain(self, content, style):
        assert style is self.sample or torch.equal(style, self.sample), "AdaIN's style is not sample"
        out = self.real["adain"](content, style)
        self._launched("adain")
        assert out.dtype == self.sample.dtype, "AdaIN's output is not in sample's dtype"
        ref, tol = adain_stage(content, self.sample)
        r = adain_ratio(out, ref, tol).max().item()
        if self.worst is not None:
            self.worst[(self.family, "adain")] = max(self.worst.get((self.family, "adain"), 0.0), r)
        if r > 1:
            raise StageFailure(f"stage adain: worst err/tol {r:.3g}")
        self.adain_ratio = r
        return out

    def expected_launches(self, iters, warp_name, gram_names):
        """(iteration, entry point, launch name) in order, the per-batch adjoint left out: per iteration the loss
        kernels and Adam, then AdaIN."""
        g = self.g
        want, per = [], []
        if g.prep is not None:
            per.append(("warp_loss_fwd_bwd", warp_name))
        if g.target is not None:
            per += [("gram_normalize", "gram_normalize_kernel"),
                    ("gram_sign", gram_names["sign"]) if g.dense else ("gram_sign_ref", gram_names["sign_ref"]),
                    ("gram_grad", gram_names["grad"])]
        per.append(("adam_step", "adam_kernel"))
        for t in range(1, iters + 1):
            want += [(t, a, b) for a, b in per]
        half = self.sample.dtype == torch.float16
        want.append((iters + 1, "adain", "adain_kernel<half>" if half else "adain_kernel<float>"))
        return want
