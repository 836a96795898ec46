"""The staged fp64 reference of one optimize_feature iteration (oracle/optimize_bound.py) and the host glue around the
kernels, on the CPU.

* Run without teacher forcing, the staged reference reproduces the reference's own outputs (tests/golden/optimize.npz:
  full1, full5, temporal3, spatial3 and AdaIN; optimize_ragged*.npz) at the tolerances ``test_oracle_golden.py`` holds
  ``oracle.optimize_feature`` to.
* ``optimize_feature`` with fp64 stand-ins at the ``ops`` boundary (``_OptKernels``, ``resize_flows_occs`` and the
  per-batch caches run for real) equals the staged reference at every iteration, every family and every branch, to the
  fp32 storage of its buffers; with neither term it returns ``sample`` itself without a call.
* Adam's propagation term holds for densely sampled gradients in its interval, and a candidate attains it.
* Every glue mutant misses the iteration by more than twice the composed bound, on a named family, in a named stage.
"""
import numpy as np
import pytest
import torch

from oracle import fresco_oracle as O
from oracle import gram_bound as GB
from oracle import optimize_bound as OB
from oracle import step_bound as SB
from oracle import warp_loss_bound as WB

# family -> make_case shape (chunks, N, C, h, w, dtype)
SHAPES = {f: (2, 3, 16, 8, 8, torch.float32) for f in OB.FAMILIES}
SHAPES["eps"] = (2, 2, 1024, 16, 16, torch.float16)
SHAPES["overflow"] = (2, 3, 8, 32, 32, torch.float32)
SHAPES["realistic"] = (2, 3, 16, 8, 8, torch.float16)


def T(a):
    return torch.from_numpy(np.asarray(a))


def case(family, branch="full", shape=None, seed=0):
    chunks, N, C, h, w, dtype = shape or SHAPES[family]
    return OB.make_case(family, chunks, N, C, h, w, dtype, seed=seed, branch=branch)


def glue_of(c):
    from fresco_b200 import diffusion_hacked as dh
    corr = OB.correlation_list(c, dh.GramTarget)
    return OB.glue(c.sample, c.flows, c.occs, corr, c.intra_weight, c.chunks, c.optimize_temporal), corr


# ------------------------------------------------------------------------------------------------ pinned to the reference
def test_staged_reference_reproduces_golden_outputs(golden):
    g = golden("optimize")
    flows, occs = [T(g["fwd"]), T(g["bwd"])], [T(g["fwd_occ"]), T(g["bwd_occ"])]
    sample, target = T(g["sample"]), T(g["target"])
    cases = {"full1": dict(iters=1), "full5": dict(iters=5), "temporal3": dict(iters=3, correlation_matrix=[]),
             "spatial3": dict(iters=3, optimize_temporal=False)}
    for tag, kw in cases.items():
        kwargs = dict(correlation_matrix=[target], intra_weight=1e2)
        kwargs.update(kw)
        out, losses, _ = OB.optimize_feature64(sample, flows, occs, **kwargs)
        assert np.allclose(np.array(losses), g[f"{tag}_losses"], rtol=2e-4), (tag, losses)
        ref = T(g[f"{tag}_out"])
        if kw["iters"] == 1:
            assert (out - ref).abs().max() < 1e-4, tag
        else:
            assert (out - ref).abs().mean() / ref.abs().mean() < 5e-2, tag
    ada, _ = OB.adain_stage(T(g["adain_content"]), sample)
    assert (ada - T(g["adain_out"]).double()).abs().max() < 1e-5


def test_staged_reference_reproduces_ragged_golden(golden):
    g = golden("optimize_ragged")
    sample, target = T(g["sample"]), T(g["target"])
    flows, occs = [T(g["fwd"]), T(g["bwd"])], [T(g["fwd_occ"]), T(g["bwd_occ"])]
    for tag, kw in {"full1": dict(iters=1), "full4": dict(iters=4),
                    "spatial4": dict(iters=4, optimize_temporal=False)}.items():
        out, losses, states = OB.optimize_feature64(sample, flows, occs, correlation_matrix=[target], intra_weight=1e2,
                                                    **kw)
        assert np.allclose(np.array(losses), g[f"{tag}_losses"], rtol=2e-4), (tag, losses)
        ref = T(g[f"{tag}_out"])
        assert out.dtype == torch.float16
        diff = (out.float() - ref.float()).abs()
        if kw["iters"] == 1:
            # the reference's AdaIN runs in fp16 arithmetic on the fp16 cast of cs: evaluated so on the staged cs, the
            # output is within one fp16 ulp at its own scale (a last-bit difference of cs may flip one content ulp)
            ada = O.adain(states[-1]["cs"].float().reshape(sample.shape).to(sample.dtype), sample).float()
            d = (ada - ref.float()).abs().max().item()
            assert d <= 2.0 ** -10 * ref.float().abs().max().item(), (tag, d)
        else:
            assert diff.mean() / ref.float().abs().mean() < 5e-2, tag


# ------------------------------------------------------------------------------------------------ the product's host glue
class Fp64Ops:
    """fp64 stand-ins for the ``ops`` entry points optimize_feature reaches, recording one dict per iteration."""

    def __init__(self):
        self.recs, self.calls, self.adain_args = [], [], None

    def _rec(self):
        if not self.recs or "p1" in self.recs[-1]:
            self.recs.append({})
        return self.recs[-1]

    def warp_adjoint_pair(self, bwd_flow, fwd_flow):
        self.calls.append("warp_adjoint_pair")
        return ("adjoint", bwd_flow, fwd_flow)

    def warp_loss_fwd_bwd(self, cs, fwd_flow, bwd_flow, fwd_keep, bwd_keep, grad, loss_acc=None, accumulate=False,
                          adjoint=None, halo_cs=None, halo_grad=None, total_frames=None):
        self.calls.append("warp_loss_fwd_bwd")
        assert torch.equal(adjoint[1], bwd_flow) and torch.equal(adjoint[2], fwd_flow) and not accumulate and halo_cs is None
        rec = self._rec()
        rec["cs"] = cs.clone()
        rec["prep"] = OB.Prep(fwd_flow, bwd_flow, fwd_keep, bwd_keep)
        r = WB.reference_and_bound(cs, fwd_flow, bwd_flow, fwd_keep, bwd_keep)
        grad.copy_(r["grad"])
        if loss_acc is not None:
            loss_acc += r["loss"]
        rec["grad_T"] = grad.clone()
        return grad

    def gram_normalize(self, cs_bcl):
        self.calls.append("gram_normalize")
        rec = self._rec()
        rec.setdefault("cs", None)
        rec["view"] = cs_bcl.clone()
        n64, _, x64, _ = GB.normalize_ref_and_bound(cs_bcl)
        return x64, n64

    def _sign(self, xhat, target, weight, loss_acc, dense):
        B, L, _ = xhat.shape
        scale = float(weight) / (B * L * L)
        self._rec()["weight"] = weight
        self._rec()["target"] = target
        Ts, tot = [], 0.0
        for b in range(B):
            t, s = OB.sign64(xhat[b], target[b], dense)
            Ts.append(t)
            tot += s
        if loss_acc is not None:
            loss_acc += scale * tot
        return torch.stack(Ts)

    def gram_sign_ref(self, xhat, yhat, weight, loss_acc=None):
        self.calls.append("gram_sign_ref")
        return self._sign(xhat, yhat, weight, loss_acc, False)

    def gram_sign(self, xhat, target, weight, loss_acc=None):
        self.calls.append("gram_sign")
        return self._sign(xhat, target, weight, loss_acc, True)

    def gram_grad(self, tsign, xhat, norms, grad_bcl, weight):
        self.calls.append("gram_grad")
        B, L, _ = xhat.shape
        self._rec()["grad0"] = grad_bcl.clone()
        grad_bcl += torch.stack([OB.project64(tsign[b], xhat[b], norms[b], float(weight) / (B * L * L)).T
                                 for b in range(B)])
        return grad_bcl

    def adam_step(self, param, grad, exp_avg, exp_avg_sq, step, lr=0.2, beta1=0.9, beta2=0.999, eps=1e-8):
        self.calls.append("adam_step")
        rec = self._rec()
        if rec.get("cs") is None:
            rec["cs"] = param.clone()
        assert torch.equal(rec["cs"], param)
        rec.update(grad=grad.clone(), m=exp_avg.clone(), v=exp_avg_sq.clone(), step=step, lr=lr)
        a = SB.adam_reference_and_bound(param, grad, exp_avg, exp_avg_sq, step, lr, beta1, beta2, eps)
        param.copy_(a["p"][0])
        exp_avg.copy_(a["m"][0])
        exp_avg_sq.copy_(a["v"][0])
        rec.update(p1=param.clone(), m1=exp_avg.clone(), v1=exp_avg_sq.clone())

    def adain(self, content, style):
        self.calls.append("adain")
        self.adain_args = (content.clone(), style)
        return OB.adain_stage(content, style)[0].to(style.dtype)


NAMES = ("warp_adjoint_pair", "warp_loss_fwd_bwd", "gram_normalize", "gram_sign_ref", "gram_sign", "gram_grad",
         "adam_step", "adain")


def run_with_standins(monkeypatch, c, corr, iters, trace=True):
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import flow_utils, ops
    be = Fp64Ops()
    for name in NAMES:
        monkeypatch.setattr(ops, name, getattr(be, name))
    flow_utils.clear_prep_cache()
    tr = dh.OptimizeTrace() if trace else None
    out = dh.optimize_feature(c.sample, c.flows, c.occs, corr, c.intra_weight, iters, c.chunks, c.optimize_temporal,
                              trace=tr)
    flow_utils.clear_prep_cache()
    return out, be, tr


def staged_fp32(g, rec, t):
    """The staged reference of iteration t on the recorded starting state, each stage's result stored to fp32 as the
    glue's buffers store it: grad after the temporal term, grad after the spatial term, p / m / v after Adam."""
    cs, B, L = rec["cs"], g.chunks * g.n, g.h * g.w
    out = {"grad_T": None, "loss": 0.0}
    grad = torch.zeros_like(cs)
    if g.prep is not None:
        r = OB.temporal_stage(cs, g.prep)
        grad = r["grad"].float()
        out["grad_T"], out["loss"] = grad, r["loss"]
    if g.target is not None:
        n64, _, x64, _ = GB.normalize_ref_and_bound(cs.reshape(B, g.C, L))
        v = torch.empty(B, g.C, L, dtype=torch.float64)
        for b in range(B):
            Tb, s = OB.sign64(x64[b], g.target[b], g.dense)
            v[b] = OB.project64(Tb, x64[b], n64[b], g.scale).T
            out["loss"] += g.scale * s
        grad = (grad.double() + v.reshape(cs.shape)).float()
    out["grad"] = grad
    a = SB.adam_reference_and_bound(cs, grad, rec["m"], rec["v"], t)
    out["p1"], out["m1"], out["v1"] = (a[k][0].float() for k in ("p", "m", "v"))
    return out


GLUE = [(f, "full") for f in OB.FAMILIES] + [("realistic", b) for b in OB.BRANCHES[1:]] + [("dense", "temporal-off")]


@pytest.mark.parametrize("family,branch", GLUE, ids=[f"{f}-{b}" for f, b in GLUE])
def test_host_glue_equals_staged_reference(monkeypatch, family, branch):
    iters = 3
    c = case(family, branch)
    g, corr = glue_of(c)
    out, be, tr = run_with_standins(monkeypatch, c, corr, iters)
    if g is None:
        assert out is c.sample and be.calls == [], be.calls
        return
    B, L = g.chunks * g.n, g.h * g.w
    assert len(be.recs) == iters
    want_calls = (["warp_adjoint_pair"] if g.prep is not None else [])
    per_it = (["warp_loss_fwd_bwd"] if g.prep is not None else [])
    if g.target is not None:
        per_it += ["gram_normalize", "gram_sign" if g.dense else "gram_sign_ref", "gram_grad"]
    assert be.calls == want_calls + (per_it + ["adam_step"]) * iters + ["adain"], be.calls
    for t, rec in enumerate(be.recs, 1):
        if t == 1:
            assert torch.equal(rec["cs"], c.sample.float().reshape(rec["cs"].shape))
            assert not rec["m"].any() and not rec["v"].any()
        assert rec["step"] == t and rec["lr"] == 0.2
        if g.prep is not None:
            for a, b in zip(rec["prep"], g.prep):
                assert torch.equal(a, b), "temporal operands differ from the restated resize"
        if g.target is not None:
            assert rec["view"].shape == (B, g.C, L) and torch.equal(rec["view"], rec["cs"].reshape(B, g.C, L))
            assert rec["weight"] == g.weight
            assert torch.equal(rec["target"], g.target)
            if g.prep is None:
                assert not rec["grad0"].any(), "spatial-only branch: the buffer is not zero"
        want = staged_fp32(g, rec, t)
        for key in ("grad_T", "grad", "p1", "m1", "v1"):
            if want[key] is None:
                continue
            assert torch.equal(rec[key], want[key]), (family, branch, t, key)
        assert abs(tr.losses[t - 1] - want["loss"]) <= 2.0 ** -23 * abs(want["loss"]), (t, tr.losses, want["loss"])
    content, style = be.adain_args
    assert torch.equal(content, be.recs[-1]["p1"].reshape(c.sample.shape)) and style is c.sample
    assert out.dtype == c.sample.dtype


# ------------------------------------------------------------------------------------------------ the composed bound
@pytest.mark.parametrize("step", [1, 2, 10])
def test_adam_propagation_term_holds_under_adversarial_gradients(step):
    """|u(g) - u(g64)| <= the term for 4001 gradients spread over [g64 - E_g, g64 + E_g] plus the candidates, on
    elements whose gradients are of order eps, at a stationary point, straddling 0 and large; some candidate attains
    the term."""
    gen = torch.Generator().manual_seed(step)
    n = 512
    scales = torch.tensor([1e-9, 1e-8, 1e-7, 1e-4, 1e-2])[torch.randint(0, 5, (n,), generator=gen)].double()
    g64 = torch.randn(n, generator=gen, dtype=torch.float64) * scales
    E = scales * torch.rand(n, generator=gen, dtype=torch.float64) * 2
    m = torch.randn(n, generator=gen, dtype=torch.float64) * scales * (step > 1)
    v = torch.rand(n, generator=gen, dtype=torch.float64) * scales ** 2 * (step > 1)
    k = SB.adam_constants(step)
    if step > 1:                                    # put the interval over a stationary point for a quarter of them
        A, V = m * (1 - k["c1"]), v * k["b2"]
        stat = k["c1"] * V / (k["c2"] * A)          # the eps-free stationary point
        sel = torch.arange(n) % 4 == 0
        g64 = torch.where(sel, stat * 0.9, g64)
        E = torch.where(sel, stat.abs() * 0.3, E)
    P, arg = OB.adam_propagation(g64, E, m, v, step)
    u0 = OB.adam_update(g64, m, v, k)
    cand = OB.adam_candidates(g64, E, m, v, k)
    grid = g64[:, None] + E[:, None] * torch.linspace(-1, 1, 4001, dtype=torch.float64)[None]
    pts = torch.cat([grid, torch.nan_to_num(cand, nan=0.0)], 1)
    inside = (pts >= (g64 - E)[:, None]) & (pts <= (g64 + E)[:, None])
    du = (OB.adam_update(pts, m[:, None], v[:, None], k) - u0[:, None]).abs()
    du = torch.where(inside, du, torch.zeros_like(du))
    slack = 1e-12 * (u0.abs() + 1e-30)
    assert bool((du.max(1).values <= P + slack).all()), (du.max(1).values / P).max().item()
    attained = (OB.adam_update(arg, m, v, k) - u0).abs()
    assert torch.equal(attained, P)
    if step > 1:
        hit = cand[sel][:, 3:].isfinite().any(1).double().mean().item()
        assert hit > 0.2, f"only {hit:.2f} of the elements placed over a stationary point have one in their interval"


@pytest.mark.parametrize("family", OB.FAMILIES)
def test_family_properties(family):
    c = case(family)
    g, _ = glue_of(c)
    OB.family_property(c, g)


def _separation(mutant):
    family, branch, t, stage = OB.MUTANTS[mutant]
    c = case(family, branch)
    g, corr = glue_of(c)
    _, _, states = OB.optimize_feature64(c.sample, c.flows, c.occs, corr, c.intra_weight, t - 1, c.chunks,
                                         c.optimize_temporal)
    state = states[-1] if states else {"cs": c.sample.float().reshape(g.chunks, g.n, g.C, g.h, g.w).double(),
                                       "m": None, "v": None, "grad": None}
    if state["m"] is None:
        state["m"], state["v"] = torch.zeros_like(state["cs"]), torch.zeros_like(state["cs"])
    bounds = OB.composed_bounds(g, state, t)
    ref = OB.iteration64(g, state, t, gram_operands="kernel")
    if stage == "adain":
        content = ref["p"].float().reshape(c.sample.shape)
        want, tol = OB.adain_stage(content, c.sample)
        mut = OB.adain64(content, c.sample, mutant).to(c.sample.dtype)
        return OB.adain_ratio(mut, want, tol).max().item(), family, stage
    mut = OB.iteration64(g, state, t, mutant, corr, gram_operands="kernel")
    key = {"temporal": "grad_T", "spatial": "grad", "adam": "p", "loss": "loss"}[stage]
    if stage == "loss":
        return abs(mut["loss"] - ref["loss"]) / bounds["loss"], family, stage
    return OB.ratio(mut[key], ref[key], bounds[stage]).max().item(), family, stage


@pytest.mark.parametrize("mutant", list(OB.MUTANTS))
def test_mutant_separation(mutant):
    """Each glue mutant moves the named stage's output on its family by more than twice the composed bound: an
    optimize_feature within the bound cannot also be within it of the mutant."""
    sep, family, stage = _separation(mutant)
    print(f"\n{mutant}: {sep:.3g} x the composed bound in stage {stage} on {family}")
    assert sep > 2.0, f"{mutant} on {family}: at most {sep:.3g} x the bound in stage {stage}"


def test_doubled_temporal_gradient_is_adam_blind_except_near_eps():
    """The temporal gradient doubled with the loss left right: Adam divides the gradient by its own RMS, so where
    |g| >> eps the first step's update moves by less than the bound (the integer family at a 64-element batch, k = 1/32);
    only the gradient stage check sees it there.  Where |g| is of order eps (the eps family) the update itself misses by
    more than twice the bound."""
    for family, shape, blind in (("integer", (1, 2, 2, 4, 4, torch.float32), True), ("eps", None, False)):
        c = case(family, shape=shape)
        g, corr = glue_of(c)
        cs = c.sample.float().reshape(g.chunks, g.n, g.C, g.h, g.w).double()
        state = {"cs": cs, "m": torch.zeros_like(cs), "v": torch.zeros_like(cs), "grad": None}
        bounds = OB.composed_bounds(g, state, 1)
        ref = OB.iteration64(g, state, 1, gram_operands="kernel")
        mut = OB.iteration64(g, state, 1, "temporal-doubled", corr, gram_operands="kernel")
        stage_sep = OB.ratio(mut["grad_T"], ref["grad_T"], bounds["temporal"]).max().item()
        adam_sep = OB.ratio(mut["p"], ref["p"], bounds["adam"]).max().item()
        print(f"\ntemporal-doubled on {family}: gradient stage {stage_sep:.3g}, Adam {adam_sep:.3g}, "
              f"loss {abs(mut['loss'] - ref['loss']):.3g}")
        assert stage_sep > 2.0 and mut["loss"] == ref["loss"]
        assert (adam_sep < 1.0) if blind else (adam_sep > 2.0), (family, adam_sep)
