"""The blending oracle (oracle/blend_oracle.py) against the reference's own outputs (tests/golden/blend*.npz, made by
make_blend_golden.py), and the Poisson solver's derived bound (oracle/blend_bound.py) against a CPU emulation of
the iteration, with mutants that must break it.

Masks, min-error images and histogram blends are compared bit for bit (the histogram may differ only where numpy's
pre-round value lies within 1e-9 of a .5, which the test counts).  The reference solves the Poisson system with lsqr;
the oracle's exact solution must give the same uint8 Lab image except where lsqr's iterate and the exact solution
truncate to different integers -- those pixels are counted and the largest |lsqr - exact| is printed (-s)."""
import numpy as np
import pytest
import scipy.sparse
import scipy.sparse.linalg

from oracle import blend_bound as BB
from oracle import blend_oracle as BO

REPORT = {}


@pytest.fixture(scope="module")
def gb(golden):
    return golden("blend")


def cases(gb):
    return [str(c) for c in gb["cases"]]


def case(gb, tag):
    return {k[len(tag) + 1:]: v for k, v in gb.items() if k.startswith(tag + "_")}


def test_masks_and_min_error_bit_exact(gb):
    for tag in cases(gb):
        c = case(gb, tag)
        masks = BO.mask_chain(c["dist1"], c["dist2"], c["flows"], int(c["interval"]))
        assert np.array_equal(masks, c["masks"]), tag
        for k in range(masks.shape[0]):
            assert np.array_equal(BO.min_error(c["oa"][k], c["ob"][k], masks[k]), c["min_error"][k]), (tag, k)


def test_mask_families_are_exercised(gb):
    """all 0, all 1 and mixed (checkerboard, blocks) masks on the last frame (frame 0 has weight1 = 0: always 0)."""
    seen = set()
    for tag in cases(gb):
        m = case(gb, tag)["masks"]
        seen.add("zero" if m[-1].max() == 0 else "one" if m[-1].min() == 1 else "mixed")
    assert seen == {"zero", "one", "mixed"}


def test_histogram_blend_bit_exact_but_counted_ties(gb):
    ties = 0
    for tag in cases(gb):
        c = case(gb, tag)
        for k, (w1, w2) in enumerate(BO.seq_weights(int(c["interval"]))):
            la, lb = BO.to_lab(c["oa"][k]), BO.to_lab(c["ob"][k])
            lab, pre = BO.histogram_blend_lab(la, lb, BO.to_lab(c["min_error"][k]), 1 - w1, 1 - w2)
            got = BO.to_bgr(lab)
            near = (np.abs(np.abs(pre - np.floor(pre)) - 0.5) < 1e-9).any(-1)
            bad = (got != c["hist"][k]).any(-1)
            assert not (bad & ~near).any(), (tag, k)
            ties += int(bad.sum())
    REPORT["histogram .5 ties"] = ties


def test_poisson_exact_matches_lsqr_up_to_truncation(gb):
    differ, worst = 0, 0.0
    for tag in cases(gb):
        c = case(gb, tag)
        for k in range(c["masks"].shape[0]):
            tgt, la, lb = BO.to_lab(c["hist"][k]), BO.to_lab(c["oa"][k]), BO.to_lab(c["ob"][k])
            u = BO.poisson_exact(tgt, la, lb, c["masks"][k])
            lab = BO.finalize(u)
            lsqr = c["lsqr"][k].astype(np.float64)     # stored in fp32: 1e-4 covers its rounding
            worst = max(worst, float(np.abs(lsqr - u).max()))
            trunc_differs = BO.finalize(np.minimum(lsqr, u) - 1e-4) != BO.finalize(np.maximum(lsqr, u) + 1e-4)
            mismatch = lab != c["lab"][k]
            assert not (mismatch & ~trunc_differs).any(), (tag, k)
            differ += int(mismatch.sum())
            final = BO.to_bgr(lab)
            bad = (final != c["final"][k]).any(-1)
            assert not (bad & ~mismatch.any(-1)).any(), (tag, k)
    REPORT["lsqr vs exact: Lab values truncating differently"] = differ
    REPORT["lsqr vs exact: largest |difference|"] = worst


def test_clips_are_exercised(gb):
    """the goldens push gradients past +-100 and the solution past [0, 255]"""
    grad, lo, hi = 0, 0, 0
    for tag in cases(gb):
        c = case(gb, tag)
        for k in range(c["masks"].shape[0]):
            la, lb = BO.to_lab(c["oa"][k]).astype(float), BO.to_lab(c["ob"][k]).astype(float)
            grad += int((np.abs(np.diff(la, axis=0)) > 100).sum() + (np.abs(np.diff(lb, axis=1)) > 100).sum())
            u = BO.poisson_exact(BO.to_lab(c["hist"][k]), BO.to_lab(c["oa"][k]), BO.to_lab(c["ob"][k]), c["masks"][k])
            lo += int((u < 0).sum())
            hi += int((u > 255).sum())
    assert grad > 0 and lo + hi > 0, (grad, lo, hi)


def test_dct_solution_is_the_sparse_least_squares_solution():
    rng = np.random.default_rng(3)
    h, w = 9, 13
    la, lb, tgt = (rng.integers(0, 256, (h, w, 3)).astype(np.uint8) for _ in range(3))
    mask = (rng.random((h, w)) > 0.5).astype(np.uint8)
    u = BO.poisson_exact(tgt, la, lb, mask)
    As = BO.construct_A(h, w)
    gx, gy = BO.gradients(la, lb, mask)
    for c, g in enumerate(BO.GRAD_WEIGHT):
        b = np.concatenate([gx[:, :, c].ravel() * g, gy[:, :, c].ravel() * g, tgt[:, :, c].ravel().astype(float)])
        A = As[c]
        ref = scipy.sparse.linalg.spsolve((A.T @ A).tocsc(), A.T @ b).reshape(h, w)
        assert np.abs(ref - u[c]).max() < 1e-9


def test_process_seq_golden_matches_oracle(gb):
    beg, end = int(gb["seq_beg"]), int(gb["seq_end"])
    n = end - beg - 1
    oas = gb["seq_fwd"][1:n + 1]
    obs = np.stack([gb["seq_bwd"][end - beg - 1 - k] for k in range(n)])
    d1 = gb["seq_err_fwd"][1:n + 1]
    d2 = gb["seq_err_bwd"][1:n + 1]          # the reference reads these before it reorders obs
    got = BO.blend_sequence(oas, obs, d1, d2, gb["seq_flows"], end - beg)
    out = gb["seq_out"]
    assert np.array_equal(out[0], gb["seq_key"])
    for k in range(n):
        u = got["solution"][k]
        near = (np.abs(u - np.round(u)) < 1e-2).any(0) | (u < 1e-2).any(0) | (u > 255 - 1e-2).any(0)
        bad = (got["final"][k] != out[k + 1]).any(-1)
        assert not (bad & ~near).any(), k


# ---- the solver bound ----

def _planes(gb):
    for tag in cases(gb):
        c = case(gb, tag)
        k = c["masks"].shape[0] - 1
        tgt, la, lb = BO.to_lab(c["hist"][k]), BO.to_lab(c["oa"][k]), BO.to_lab(c["ob"][k])
        yield tag, tgt, la, lb, c["masks"][k]


def _emulate(tgt, la, lb, mask, c, weight, lam_max=None, apply=BB.apply_m, clip=True, swap=False):
    if swap:
        mask = 1 - mask
    gx, gy = BO.gradients(la, lb, mask) if clip else _unclipped(la, lb, mask)
    rhs = BO.normal_rhs(tgt, gx, gy, weight, c)
    h, w = mask.shape
    return BB.cheby_emulate(rhs, tgt[:, :, c].astype(np.float64), weight, BB.cheby_iterations(h, w, weight),
                            lam_max=lam_max, apply=apply)


def _unclipped(la, lb, mask):
    old = BO.GRAD_CLIP
    BO.GRAD_CLIP = np.inf
    try:
        return BO.gradients(la, lb, mask)
    finally:
        BO.GRAD_CLIP = old


def test_iteration_counts_follow_from_the_bound():
    assert BB.cheby_iterations(512, 896, 2.5) == 76 and BB.cheby_iterations(512, 896, 0.5) == 15
    for h, w, g in [(512, 896, 2.5), (64, 64, 0.5), (1, 896, 2.5), (37, 1, 0.5)]:
        k = BB.cheby_iterations(h, w, g)
        assert BB.truncation_bound(h, w, g, k) <= BB.TRUNC < BB.truncation_bound(h, w, g, k - 1)
    assert BB.cheby_iterations(1, 1, 2.5) == 0


@pytest.mark.parametrize("weight_c", [(2.5, 0), (0.5, 1), (0.5, 2)])
def test_emulated_iteration_within_bound(gb, weight_c):
    weight, c = weight_c
    worst = 0.0
    for tag, tgt, la, lb, mask in _planes(gb):
        exact = BO.poisson_exact(tgt, la, lb, mask)[c]
        err = np.abs(_emulate(tgt, la, lb, mask, c, weight) - exact).max()
        assert err <= BB.TOL, (tag, err)
        worst = max(worst, err / BB.TOL)
    REPORT[f"emulated Chebyshev err/tol, w={weight}"] = worst


def _dirichlet(y, weight):      # a missing boundary row: the stencil sees 0 outside the image
    lap = 4 * y.copy()
    lap[1:] -= y[:-1]
    lap[:-1] -= y[1:]
    lap[:, 1:] -= y[:, :-1]
    lap[:, :-1] -= y[:, 1:]
    return y + weight * weight * lap


MUTANTS = {
    "spectral bound 1 + 4 w^2": dict(lam_max=1 + 4 * 2.5 ** 2),
    "missing boundary row": dict(apply=_dirichlet),
    "gradients not clipped": dict(clip=False),
    "masks swapped": dict(swap=True),
}


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_mutants_break_the_bound(gb, name):
    broken = False
    for tag, tgt, la, lb, mask in _planes(gb):
        exact = BO.poisson_exact(tgt, la, lb, mask)[0]
        broken |= np.abs(_emulate(tgt, la, lb, mask, 0, 2.5, **MUTANTS[name]) - exact).max() > BB.TOL
    assert broken, name


def test_mutant_round_instead_of_truncate(gb):
    differs = False
    for tag, tgt, la, lb, mask in _planes(gb):
        u = BO.poisson_exact(tgt, la, lb, mask)
        rounded = np.clip(np.round(np.moveaxis(u, 0, -1)), 0, 255).astype(np.uint8)
        differs |= not np.array_equal(rounded, BO.finalize(u))
    assert differs


def test_report():
    for k, v in REPORT.items():
        print(f"{k}: {v}")


def test_every_blend_launch_name_is_checked():
    """Every kernel name csrc/blend/*.cu launches is either asserted as the last launch of a call by
    tests/test_gpu_blend.py or runs before such a launch, whose output depends on it; a new kernel fails here until it
    is placed.  (Needs no GPU.)"""
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    d = os.path.join(root, "fresco_b200", "csrc", "blend")
    names = set()
    for f in os.listdir(d):
        if f.endswith(".cu"):
            names.update(re.findall(r"check_launch\(\"(\w+_kernel(?:<\w+>)?)\"\)", open(os.path.join(d, f)).read()))
    gpu_tests = open(os.path.join(root, "tests", "test_gpu_blend.py")).read()
    asserted = set(re.findall(r"last_kernel\(\) == \"(\w+)\"", gpu_tests))
    not_last = {"blend_hist_stats_kernel<0>", "blend_hist_stats_kernel<1>", "blend_hist_stats_kernel<2>",
                "blend_hist_stats_kernel<3>", "blend_hist_moments_kernel<0>", "blend_hist_moments_kernel<1>",
                "blend_hist_moments_kernel<2>", "blend_hist_moments_kernel<3>",      # before blend_hist_apply_kernel
                "blend_poisson_rhs_kernel", "blend_cheby_kernel"}                    # before the Poisson finalize
    assert not asserted & not_last
    assert names == asserted | not_last, (sorted(names - asserted - not_last), sorted(asserted | not_last - names))
