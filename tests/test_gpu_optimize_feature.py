"""optimize_feature on the GPU, one Adam iteration at a time, held to the bound composed from its kernels' bounds
(oracle/optimize_bound.py).

A spy on ``ops`` (``OpsSpy``) records every launch's operands, result and ``fresco_last_kernel`` name.  Per call:

* the launches, in order, per iteration and for the final AdaIN;
* the first stage's operands bit-equal the test's own restatement of src/diffusion_hacked.py:437-442
  (``F.interpolate(flows scale)``, ``1 - max_pool2d(occ, int(1 / scale))``), cs_1 = sample.float() in
  [chunks, n, C, h, w], m_1 = v_1 = 0, Adam's step = t and lr 0.2, the Gram weight intra_weight n / total and the first
  matching correlation_matrix entry;
* every stage within its own bound and the iteration within the composed bound, checked inside the Adam spy on the
  state the GPU held at the iteration's start (a failure names the iteration, the stage and whether the own bound
  alone also fails); each ``trace.losses[t]`` within the loss bound; the output within AdaIN's bound on the cs the last
  Adam wrote; the integer family's temporal gradient bit-exact.

Bit-exact invariances: ``trace=`` on and off give the same output; an fp16 sample and its fp32 upcast give the same cs
after every Adam step.  ``test_report_worst_ratios`` prints the worst err/tol per family and stage and the share of
step-1 elements whose gradient interval contains 0 (their update is +-lr either way).
"""
import collections

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import gram_bound as GB  # noqa: E402  (checker only)
from oracle import optimize_bound as OB  # noqa: E402  (checker only)

WORST = {}
SATURATED = collections.defaultdict(float)
SEEN = set()

# (id, family, chunks, N, C, h, w, dtype, flow resolution, iters, iterations checked (None: all))
F16, F32 = torch.float16, torch.float32
SHAPES = [
    ("512-8x8-N8", "realistic", 2, 8, 1280, 8, 8, F16, (512, 512), 20, None),
    ("512-16x16-N8", "realistic", 2, 8, 1280, 16, 16, F16, (512, 512), 20, None),
    ("512-32x32-N8", "realistic", 2, 8, 1280, 32, 32, F16, (512, 512), 2, None),
    ("512-64x64-N8", "realistic", 2, 8, 640, 64, 64, F16, (512, 512), 20, {1, 2, 3, 10, 20}),
    ("768-48x48-N4", "realistic", 2, 4, 1280, 48, 48, F16, (768, 768), 2, None),
    ("768-96x96-N2", "realistic", 2, 2, 640, 96, 96, F16, (768, 768), 1, None),
    ("320x448-5x7-N4", "realistic", 2, 4, 1280, 5, 7, F16, (320, 448), 2, None),
    ("320x448-10x14-N4", "realistic", 2, 4, 1280, 10, 14, F16, (320, 448), 2, None),
    ("N2-fp32", "realistic", 2, 2, 1280, 16, 16, F32, (128, 128), 2, None),
    ("N3", "realistic", 2, 3, 1280, 16, 16, F16, (128, 128), 2, None),
    ("N16", "realistic", 2, 16, 1280, 8, 8, F32, (64, 64), 2, None),
    ("chunks1", "realistic", 1, 4, 1280, 16, 16, F16, (128, 128), 2, None),
]
FAMILY_SHAPES = {
    "integer": (2, 3, 64, 16, 16, F32), "tie": (2, 3, 64, 16, 16, F16), "eps": (2, 2, 1024, 16, 16, F16),
    "balance-temporal": (2, 3, 320, 16, 16, F16), "balance-spatial": (2, 3, 320, 16, 16, F16),
    "masks-all": (2, 3, 64, 16, 16, F32), "masks-none": (2, 3, 64, 16, 16, F32), "overflow": (2, 3, 8, 32, 32, F32),
    "dense": (2, 3, 320, 32, 32, F32),
}
for fam, (ch, N_, C_, h_, w_, dt) in FAMILY_SHAPES.items():
    SHAPES.append((fam, fam, ch, N_, C_, h_, w_, dt, None, 2, None))


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib, diffusion_hacked, flow_utils, ops
    _lib.lib()      # fails loudly if the extension is missing
    torch.backends.cuda.matmul.allow_tf32 = False

    class NS:
        pass
    ns = NS()
    ns.lib, ns.ops, ns.dh, ns.fu = _lib, ops, diffusion_hacked, flow_utils
    ns.grid = torch.cuda.get_device_properties(0).multi_processor_count
    return ns


def cuda_case(fb, family, chunks, N, C, h, w, dtype, res, branch="full", seed=0):
    c = OB.make_case(family, chunks, N, C, h, w, dtype, seed=seed, res=res, branch=branch)
    dev = torch.device("cuda")
    c = c._replace(sample=c.sample.to(dev),
                   flows=None if c.flows is None else [f.to(dev) for f in c.flows],
                   occs=None if c.occs is None else [o.to(dev) for o in c.occs])
    corr = OB.correlation_list(c, fb.dh.GramTarget, dev)
    g = OB.glue(c.sample, c.flows, c.occs, corr, c.intra_weight, c.chunks, c.optimize_temporal)
    return c, corr, g


def run_checked(fb, monkeypatch, c, corr, g, iters, check_at=None, key="", trace=True, after_adam=None):
    """optimize_feature under the spy; asserts the launches and the trace.  -> (out, spy)."""
    spy = OB.OpsSpy(fb.ops, fb.lib.last_kernel, g, c.sample, fb.grid, key, WORST, check_at,
                    integer=c.family == "integer", after_adam=after_adam)
    with monkeypatch.context() as mp:
        spy.install(mp)
        fb.fu.clear_prep_cache()
        tr = fb.dh.OptimizeTrace() if trace else None
        out = fb.dh.optimize_feature(c.sample, c.flows, c.occs, corr, c.intra_weight, iters, c.chunks,
                                     c.optimize_temporal, trace=tr)
        torch.cuda.synchronize()
    fb.fu.clear_prep_cache()
    got = [x for x in spy.launches if x[1] != "warp_adjoint_pair"]
    want = spy.expected_launches(iters, None, GB.names(g.h * g.w))
    assert [(t, a) for t, a, _ in got] == [(t, a) for t, a, _ in want], got
    for (t, a, name), (_, _, wname) in zip(got, want):
        if a == "warp_loss_fwd_bwd":
            assert name.startswith("warp_loss_"), (t, name)
        else:
            assert name == wname, (t, a, name, wname)
        SEEN.add(name)
    if trace:
        assert tr.losses == spy.losses, (tr.losses, spy.losses)
    for t, share in spy.saturated:
        if t == 1:
            SATURATED[key] = max(SATURATED[key], share)
    return out, spy


@pytest.mark.parametrize("sid,family,chunks,N,C,h,w,dtype,res,iters,check_at", SHAPES, ids=[s[0] for s in SHAPES])
def test_optimize_feature_within_composed_bound(fb, monkeypatch, sid, family, chunks, N, C, h, w, dtype, res, iters,
                                                check_at):
    c, corr, g = cuda_case(fb, family, chunks, N, C, h, w, dtype, res, seed=h + N)
    if family != "realistic":
        OB.family_property(c._replace(sample=c.sample.cpu(), targets=c.targets), g._replace(
            prep=None if g.prep is None else OB.Prep(*(t.cpu() for t in g.prep)),
            target=None if g.target is None else g.target.cpu()))
    out, spy = run_checked(fb, monkeypatch, c, corr, g, iters, check_at, key=family)
    assert out.shape == c.sample.shape and out.dtype == c.sample.dtype and torch.isfinite(out).all()


@pytest.mark.parametrize("branch", [b for b in OB.BRANCHES if b != "full"])
def test_optimize_feature_branches(fb, monkeypatch, branch):
    c, corr, g = cuda_case(fb, "realistic", 2, 3, 1280, 16, 16, F16, (128, 128), branch=branch, seed=5)
    if g is None:
        before = fb.lib.launch_count()
        out = fb.dh.optimize_feature(c.sample, c.flows, c.occs, corr, c.intra_weight, 2, c.chunks, c.optimize_temporal)
        assert out is c.sample and fb.lib.launch_count() == before
        return
    run_checked(fb, monkeypatch, c, corr, g, 2, key="realistic")


def test_tie_family_keeps_zero_gradient_elements(fb, monkeypatch):
    """identical frames and zero flow, the temporal term alone: every residual is exactly 0, so is every gradient
    element Adam receives, and p, m and v come back bit for bit at step 1 (from m = v = 0)."""
    c, corr, g = cuda_case(fb, "tie", 2, 3, 64, 16, 16, F32, None, branch="no-target", seed=1)
    kept = {}

    def after(t, p, grad, m, v):
        kept[t] = (p.clone(), grad.clone(), m.clone(), v.clone())
    run_checked(fb, monkeypatch, c, corr, g, 1, key="tie", after_adam=after)
    p, grad, m, v = kept[1]
    assert not grad.any(), "a nonzero temporal gradient on identical frames"
    assert torch.equal(p, c.sample.float().reshape(p.shape)) and not m.any() and not v.any()


def test_trace_on_and_off_give_the_same_output(fb, monkeypatch):
    c, corr, g = cuda_case(fb, "realistic", 2, 4, 1280, 16, 16, F16, (128, 128), seed=9)
    a = fb.dh.optimize_feature(c.sample, c.flows, c.occs, corr, c.intra_weight, 5, c.chunks, trace=fb.dh.OptimizeTrace())
    b = fb.dh.optimize_feature(c.sample, c.flows, c.occs, corr, c.intra_weight, 5, c.chunks)
    assert torch.equal(a, b)


def test_fp16_sample_and_its_fp32_upcast_give_the_same_cs(fb, monkeypatch):
    c, corr, g = cuda_case(fb, "realistic", 2, 4, 1280, 16, 16, F16, (128, 128), seed=11)
    seen = {}
    for dt in (F16, F32):
        cs = seen.setdefault(dt, {})
        cc = c._replace(sample=c.sample.to(dt))
        run_checked(fb, monkeypatch, cc, corr, g, 4, check_at=set(), key="realistic",
                    after_adam=lambda t, p, *rest, cs=cs: cs.__setitem__(t, p.clone()))
    for t in range(1, 5):
        assert torch.equal(seen[F16][t], seen[F32][t]), t


def test_report_worst_ratios():
    """Prints the worst err/tol per family and stage, and per family the share of step-1 elements whose gradient
    interval contains 0 (run with -s)."""
    for (fam, stage), r in sorted(WORST.items()):
        print(f"{fam:18s} {stage:9s} worst err/tol {r:.3g}")
    for fam, s in sorted(SATURATED.items()):
        print(f"{fam:18s} step-1 elements with 0 in the gradient interval: {s:.4f}")
    print("launches seen:", sorted(SEEN))
    if WORST:
        assert max(WORST.values()) <= 1.0
        assert {"gram2_kernel<G2_SIGN>", "gram2_kernel<G2_SIGN,ragged>", "tile_gemm_kernel<EPI_GRAM_SIGN,0>",
                "adain_kernel<half>", "adain_kernel<float>"} <= SEEN, SEEN
        assert len({n for n in SEEN if n.startswith("warp_loss_")}) >= 2, SEEN
