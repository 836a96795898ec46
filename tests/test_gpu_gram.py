"""The spatial-consistency (Gram-L1) loss through the C ABI, every family of ``oracle.gram_bound`` on every entry point:
``fresco_gram_normalize``, ``fresco_gram_sign_ref[_scaled]``, ``fresco_gram_sign[_scaled]``, ``fresco_gram_tx`` and
``fresco_gram_grad[_scaled]`` under FRESCO_GRAM_V = 2 and 1.

Every call asserts its launch name, every output is NaN-prefilled between NaN guard rows, and every fp64 reference is
computed on the GPU from the kernels' own operands, one batch at a time.  The onehot, dyadic and asymmetric families
are bit-exact; the others are held elementwise to the derived bound.  Shapes: the four decoder layers at 512^2 and at
768^2 (B = 16 for the two largest), L in {1, 7, 31, 32, 33, 127, 128, 129, 255, 256, 257, 383, 384, 385} (the 32-token
CTAs of the normalisation and the projection, the 128-row tiles, odd counts of 128-row tiles where the 256-column
pairs straddle the edge) and C in {8, 24, 320} (a partial K atom, a partial 256-column pair of G2_GRAD).  The
sign with the recomputed target is also checked against the reference's own formula (fp32 cs, fp16 target) outside
beta + rho.  ``spatial_loss_grad`` is checked end to end from fp32 cs; one B = 16 call gives the bits of 16 calls at
B = 1; T is symmetric outside the diagonal blocks.  ``test_report_worst_ratios`` prints the worst err/tol per family
and output (-s).
"""
import pytest
import torch

from oracle import gram_bound as GB

pytestmark = pytest.mark.gpu
RATIOS = {}         # (family, output) -> worst err/tol
SEEN = set()
# every name fresco_last_kernel() reports for a Gram call; fresco_gram_grad under FRESCO_GRAM_V=1 launches
# tile_gemm_kernel<EPI_STORE,1[,ragged]> before gram_project_kernel, which test_gpu_gram_ragged.py reads from the profiler
ALL_NAMES = {"gram_normalize_kernel", "gram2_kernel<G2_SIGN>", "gram2_kernel<G2_SIGN,ragged>", "gram2_kernel<G2_GRAD>",
             "gram2_kernel<G2_GRAD,ragged>", "tile_gemm_kernel<EPI_GRAM_SIGN,0>", "gram_project_kernel"}
WEIGHT = 100.0

DECODER = [(16, 1280, 64), (16, 1280, 256), (16, 1280, 1024), (16, 640, 4096),        # 512^2: (B, C, L)
           (4, 1280, 144), (4, 1280, 576), (16, 1280, 2304), (16, 640, 9216)]         # 768^2
EDGE_L = [(2, 64, L) for L in (1, 7, 31, 32, 33, 127, 128, 129, 255, 256, 257, 383, 384, 385)]
EDGE_C = [(2, C, 257) for C in (8, 24, 320)]
SMALL_DECODER = [(4, 1280, 256), (2, 640, 4096)]


def _cases():
    out = []
    for fam in GB.FAMILIES:
        if fam == "realistic":
            shapes = DECODER + EDGE_L + EDGE_C
        elif fam == "coherent":
            shapes = DECODER
        elif fam == "asymmetric":
            shapes = EDGE_L + EDGE_C + SMALL_DECODER[:1]
        else:
            shapes = EDGE_L + EDGE_C + SMALL_DECODER
        out += [pytest.param(fam, *s, id=f"{fam}-{s[0]}x{s[1]}x{s[2]}") for s in shapes]
    return out


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib, diffusion_hacked, ops
    _lib.lib()      # fails loudly if the extension is missing
    torch.backends.cuda.matmul.allow_tf32 = False

    class NS:
        pass
    ns = NS()
    ns.lib, ns.c, ns.ops, ns.dh = _lib, _lib.lib(), ops, diffusion_hacked
    ns.grid = torch.cuda.get_device_properties(0).multi_processor_count
    return ns


def _normalize(fb, cs, exact, ratios):
    B, C, L = cs.shape
    bx, xhat = GB.guarded(B, L, C, torch.float16)
    bn, norms = GB.guarded(1, B, L, torch.float32)
    GB.launched(fb, "fresco_gram_normalize", fb.c.fresco_gram_normalize(cs.data_ptr(), xhat.data_ptr(),
                                                                        norms.data_ptr(), B, C, L, fb.lib.stream()),
                "gram_normalize_kernel", SEEN)
    torch.cuda.synchronize()
    GB.guards_intact(bx, "xhat")
    GB.guards_intact(bn, "norms")
    norms = norms[0]
    ref = GB.check_normalize(cs, xhat, norms, exact, ratios)
    return xhat, norms, ref


def _operands(fb, fam, B, C, L, ratios, dense=True):
    f = GB.family(fam, B, L, C, seed=L + C)
    exact = fam in GB.EXACT
    ref = None
    if "cs" in f:
        cs, cs_ref = f["cs"].cuda(), f["cs_ref"].cuda()
        xhat, norms, ref = _normalize(fb, cs, exact, ratios)
        yhat, _, _ = _normalize(fb, cs_ref, exact, None)
    else:
        cs = None
        xhat, yhat, norms = f["xhat"].cuda(), f["yhat"].cuda(), f["norms"].cuda()
    target = None
    if "target" in f:
        target = f["target"].cuda()
    elif dense:
        target = torch.empty(B, L, L, device="cuda")
        for b in range(B):
            target[b] = GB.fp16_target(yhat[b])
    scale = f["scale"] or WEIGHT / (B * L * L)
    weight = WEIGHT if f["scale"] is None else scale * B * L * L
    grad0 = torch.zeros(B, C, L, device="cuda") if exact else torch.randn(
        B, C, L, device="cuda", generator=torch.Generator(device="cuda").manual_seed(L))
    return cs, xhat, yhat, norms, target, grad0, scale, weight, ref


@pytest.mark.parametrize("fam,B,C,L", _cases())
def test_family(fb, fam, B, C, L):
    ratios = {}
    big = B * L * L > 16 * 4096 * 4096                 # the dense target of the 768^2 layer 3 alone is 5.4 GB
    cs, xhat, yhat, norms, target, grad0, scale, weight, ref = _operands(fb, fam, B, C, L, ratios, dense=not big)
    exact = fam in GB.EXACT
    dense_only = fam in GB.DENSE_ONLY
    run = GB.Run(fb, xhat, yhat, norms, target, grad0, weight, scale, SEEN, sign=not dense_only)
    run.hygiene()
    if not dense_only and weight == WEIGHT:
        assert torch.equal(run.tsign1, run.tsign), "T: the weight form differs from the scaled form"
        for v in (2, 1):
            assert torch.equal(run.grads[(v, "weight")], run.grads[(v, "scaled")]), f"grad V={v}: weight form differs"
    GB.check_run(run, xhat, yhat, norms, target, grad0, scale, fb.grid, exact, ratios,
                 ref_formula=ref)
    for k, r in ratios.items():
        RATIOS[(fam, k)] = max(RATIOS.get((fam, k), 0.0), r)


@pytest.mark.parametrize("B,C,L", [(16, 1280, 256), (16, 640, 257)])
def test_batch_invariance_and_mirror(fb, B, C, L):
    """One B = 16 call gives the bits of 16 calls at B = 1 (T, g^ and both gradients); T is symmetric outside the
    diagonal 128-blocks (the [J, I] mirror of each tile)."""
    f = GB.family("realistic", B, L, C, seed=5)
    cs, cs_ref = f["cs"].cuda(), f["cs_ref"].cuda()
    xhat, norms = fb.ops.gram_normalize(cs)
    yhat, _ = fb.ops.gram_normalize(cs_ref)
    grad0 = torch.randn(B, C, L, device="cuda")
    scale = WEIGHT / (B * L * L)
    full = GB.Run(fb, xhat, yhat, norms, None, grad0, WEIGHT, scale, SEEN)
    for b in range(B):
        one = GB.Run(fb, xhat[b:b + 1].contiguous(), yhat[b:b + 1].contiguous(), norms[b:b + 1].contiguous(), None,
                     grad0[b:b + 1].contiguous(), WEIGHT / B, scale, SEEN)      # a rank's share: the same scale
        assert torch.equal(one.tsign[0], full.tsign[b]), f"T batch {b}"
        assert torch.equal(one.ghat[0], full.ghat[b]), f"g^ batch {b}"
        for key in one.grads:
            assert torch.equal(one.grads[key][0], full.grads[key][b]), f"grad {key} batch {b}"
    blk = torch.arange(L, device="cuda") >> 7
    off = blk[:, None] != blk[None, :]
    for b in range(B):
        t = full.tsign[b]
        assert torch.equal(t[off], t.T[off]), f"T batch {b} not symmetric outside the diagonal blocks"


@pytest.mark.parametrize("fam,B,C,L", [("realistic", 16, 1280, 256), ("coherent", 4, 640, 1024),
                                       ("dominant", 2, 320, 385), ("realistic", 2, 640, 4096)])
def test_spatial_loss_grad_composed(fb, fam, B, C, L):
    """diffusion_hacked.spatial_loss_grad from fp32 cs against the gradient of the reference's formula given the
    kernel's T: the projection bound plus the normalisation's error carried through it."""
    f = GB.family(fam, B, L, C, seed=11)
    cs, cs_ref = f["cs"].cuda(), f["cs_ref"].cuda()
    yhat, _ = fb.ops.gram_normalize(cs_ref)
    target = fb.dh.GramTarget(yhat)
    xhat, norms = fb.ops.gram_normalize(cs)
    tsign = fb.ops.gram_sign_ref(xhat, yhat, WEIGHT)
    grad = torch.zeros(B, C, L, device="cuda")
    loss = torch.zeros(1, device="cuda")
    fb.dh.spatial_loss_grad(cs, target, WEIGHT, grad, loss)
    torch.cuda.synchronize()
    scale = WEIGHT / (B * L * L)
    for b in range(B):
        want, tol = GB.composed_ref_and_bound(cs[b], tsign[b], scale, xhat[b], norms[b], torch.zeros(C, L,
                                                                                                     device="cuda"))
        r = GB.ratio(grad[b].T, want, tol).max().item()
        RATIOS[(fam, "composed")] = max(RATIOS.get((fam, "composed"), 0.0), r)
        assert r <= 1, f"spatial_loss_grad batch {b}: worst err/tol {r:.3g}"


def test_every_launch_name_seen():
    if not SEEN:
        pytest.skip("no Gram case ran")
    assert SEEN == ALL_NAMES, sorted(ALL_NAMES - SEEN)


def test_report_worst_ratios():
    """Prints the largest err/tol seen per family and output (-s to see it)."""
    if not RATIOS:
        pytest.skip("no Gram case ran")
    print("\nworst err/tol per family and output")
    for (fam, k), r in sorted(RATIOS.items()):
        print(f"  {fam:12s} {k:12s} {r:.3g}")
