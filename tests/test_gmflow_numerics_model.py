"""The EPI_GMFLOW epilogue of tile_gemm_kernel (gemm_wgmma.cu), restated in torch fp32 on the CPU.

``emulate`` runs the kernel's online softmax the way the kernel schedules it: 128-key tiles; the four lanes of a quad
each owning the columns acc_col gives them (8 k + 2 lane + {0, 1}) and summing l, x and y in that order; the row max
over the valid columns only, reduced over the quad; alpha = ex2(m_old - m_new) on all three sums; p = ex2.approx.ftz of
one FFMA; two xor shuffles; 1.f / l and the multiply-subtract; the coordinate decode (gn % w, gn / w) and the subtraction of the
query's own coordinate; the backward launch writing at flow_batch_offset = B.  It checks the error model of
``oracle.gmflow_bound`` without a GPU: the emulator stays inside the bound on every input family and matches the
exactly known answers of the exact families bit for bit, and each of ``MUTANTS`` -- a one-line mistake a change to the
epilogue could make -- leaves the bound or an exact answer on at least one family.
"""
import math

import pytest
import torch

from oracle import gmflow_bound as GB

MUTANTS = {
    "xy-swap": "coordinate decode swapped: (gn / w, gn % w)",
    "max-guard": "gn < N dropped in the row max: the zero-filled columns of the ragged tile enter it with S = 0",
    "sum-guard": "gn < N dropped in the sums: the zero-filled columns enter l, x and y",
    "alpha-xy": "alpha applied to l but not to the x and y sums",
    "bwd-offset0": "the backward launch writes at flow_batch_offset = 0",
}

# grid -> the families run there (C = 32; 24 x 40 is 7.5 key tiles, 16 x 24 three tiles)
GRIDS = [(24, 40), (16, 24)]
C = 32
B = 2


def _ex2(x):
    """ex2.approx.ftz.f32: results below 2^-126 flush to zero."""
    p = torch.exp2(x)
    return torch.where(p < 2.0 ** -126, torch.zeros((), dtype=torch.float32), p)


def _fma(a, b, c):
    """fp32 fma: the product of two fp32 values is exact in fp64, one rounding to fp32 after the add."""
    return (a.double() * b.double() + c.double()).float()


def _direction(a, b, h, w, mutant):
    """One launch's rows: a, b fp16 token-major [L, C] (queries, keys) -> fp32 [2, L]."""
    L, Cc = a.shape
    n_tiles = (L + GB.TILE - 1) // GB.TILE
    S = torch.zeros(L, n_tiles * GB.TILE, dtype=torch.float32)     # TMA zero-fills the keys past N
    S[:, :L] = (a.double() @ b.double().T).float()
    c = torch.tensor(GB.LOG2E / math.sqrt(Cc), dtype=torch.float32)
    m_run = torch.full((L, 1), float("-inf"))
    l = torch.zeros(L, 4)
    sx = torch.zeros(L, 4)
    sy = torch.zeros(L, 4)
    lane = torch.arange(4)
    for t in range(n_tiles):
        n0 = t * GB.TILE
        St = S[:, n0:n0 + GB.TILE]
        valid = (n0 + torch.arange(GB.TILE)) < L
        mx = St.amax(1, keepdim=True) if mutant == "max-guard" else St[:, valid].amax(1, keepdim=True)
        m_new = torch.maximum(m_run, mx * c)
        alpha = _ex2(m_run - m_new)
        m_run = m_new
        l = l * alpha
        if mutant != "alpha-xy":
            sx = sx * alpha
            sy = sy * alpha
        for k in range(16):
            for e in range(2):
                col = 8 * k + 2 * lane + e                              # [4]: this step's column of each lane
                gn = n0 + col
                ok = (gn < L) | (mutant == "sum-guard")
                pe = _ex2(_fma(St[:, col], c, -m_run))
                vx, vy = (gn % w).float(), torch.div(gn, w, rounding_mode="floor").float()
                if mutant == "xy-swap":
                    vx, vy = vy, vx
                l = torch.where(ok, l + pe, l)
                sx = torch.where(ok, _fma(pe, vx, sx), sx)
                sy = torch.where(ok, _fma(pe, vy, sy), sy)
    quad = lambda s: (s[:, 0] + s[:, 1]) + (s[:, 2] + s[:, 3])        # xor 1, then xor 2
    inv = torch.ones(L) / quad(l)
    gm = torch.arange(L)
    # s * inv - q as one FFMA (nvcc may also round the multiply first; the exact families accept either)
    return torch.stack([_fma(quad(sx), inv, -(gm % w).float()),
                        _fma(quad(sy), inv, -torch.div(gm, w, rounding_mode="floor").float())])


def emulate(f0, f1, bidir, mutant=None):
    """gmflow_global_corr_softmax on the CPU: fp32 [B(*2), 2, h, w], NaN where the launches write nothing."""
    Bb, Cc, h, w = f0.shape
    t0, t1 = GB.to_tokens(f0).half(), GB.to_tokens(f1).half()
    out = torch.full((Bb * (2 if bidir else 1), 2, h * w), float("nan"))
    for b in range(Bb):
        out[b] = _direction(t0[b], t1[b], h, w, mutant)
    if bidir:
        off = 0 if mutant == "bwd-offset0" else Bb
        for b in range(Bb):
            out[off + b] = _direction(t1[b], t0[b], h, w, mutant)
    return out.reshape(-1, 2, h, w)


def _verdict(fam, got):
    """(worst err / tol, exact answer matched or None)."""
    ref, tol = GB.corr_ref_and_bound(fam.f0, fam.f1, True)
    ratio = ((got.double() - ref).abs() / tol).nan_to_num(nan=float("inf")).max().item()
    exact = None
    if fam.exact:
        exact = bool(GB.matches_exact(got, GB.corr_exact(fam.f0, fam.f1, True)).all())
    return ratio, exact


_CACHE = {}


def _families(h, w):
    key = (h, w)
    if key not in _CACHE:
        _CACHE[key] = [GB.family(n, B, C, h, w, seed=7) for n in GB.FAMILIES]
    return _CACHE[key]


@pytest.mark.parametrize("grid", GRIDS, ids=lambda g: "%dx%d" % g)
def test_families_have_their_property(grid):
    for fam in _families(*grid):
        GB.family_property(fam)


@pytest.mark.parametrize("grid", GRIDS, ids=lambda g: "%dx%d" % g)
def test_emulated_kernel_within_bound_and_exact(grid):
    """The error model: the kernel's arithmetic, restated, stays inside gmflow_bound on every family and gives the
    exact families' answers bit for bit."""
    for fam in _families(*grid):
        ratio, exact = _verdict(fam, emulate(fam.f0, fam.f1, True))
        assert ratio <= 1.0, f"{fam.name}: emulated err / bound {ratio:.3g}"
        assert exact in (None, True), f"{fam.name}: not bit-exact"


# mutant -> a family that must catch it (on the 24 x 40 grid: ragged last tile)
MUTANT_CASES = {
    "xy-swap": "translated",
    "max-guard": "negative-floor",
    "sum-guard": "negative-floor",
    "alpha-xy": "late",
    "bwd-offset0": "translated",
}


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_emulated_mutants_are_caught(mutant):
    caught = []
    for fam in _families(*GRIDS[0]):
        ratio, exact = _verdict(fam, emulate(fam.f0, fam.f1, True, mutant))
        if ratio > 1.0 or exact is False:
            caught.append(fam.name)
    assert MUTANT_CASES[mutant] in caught, f"{mutant} ({MUTANTS[mutant]}) is caught only by {caught}"


def test_bound_is_not_vacuous():
    """The bound is orders of magnitude below the old 0.1 px tolerance on the realistic families."""
    for fam in _families(*GRIDS[0]):
        if fam.name.startswith("peaky"):
            _, tol = GB.corr_ref_and_bound(fam.f0, fam.f1, True)
            assert tol.max().item() < 1e-2, (fam.name, tol.max().item())
