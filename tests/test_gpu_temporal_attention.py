"""Temporal-guided attention (A5) through the C ABI, on both kernels, against ``oracle.temporal_bound``.

``fresco_temporal_attn_fwd[_strided]`` runs one of two kernels, and every case asserts the launch name:

* temporal_attn_rows_kernel<D, NMAX> for D = 40 / 64 / 80 and NMAX = 8 / 16: N swept over each NMAX's range at each
  head dim, 1 / 3 / 8 heads, heads * N = 256, one trajectory per CTA with more than 48 KB of shared memory, 1 / 2 / 3
  chunks, token counts that leave a ragged last CTA and a single token, the bench shapes on every trajectory, and every
  input family of the bound;
* the strided entry point: the packed call ShardedTrajectoryExchange.run makes (q | k | v in one 3C row, identity
  map, chunks = 1, the mask expanded over the chunks), a row stride wider than 3C with NaN in every gap column, and
  NaN guard rows before and after ``out`` that must stay NaN;
* temporal_attn_kernel (round 1): N = 17 / 31 / 32 / 33 / 48 (past 32 a lane owns two softmax rows), head dims
  8 / 16 / 24 / 128, heads * N > 256, FRESCO_TEMPORAL_V=1 at N <= 16, and the largest N whose shared memory fits.

Outputs are prefilled with NaN, so a row the kernel never writes fails.  Every output element must lie within the
bound; the exact families (self-only, dominant, uniform) must match their known answer bit for bit.  A handful of
invariances must hold bit for bit, since each row's arithmetic does not depend on how the launcher groups rows into
CTAs: dense == packed, one chunks = 2 call == two chunks = 1 calls, the packed call on a trajectory block
``dist.frame_range(L, G, s)`` == those rows of the full call (the kernel-level statement of the sharded exchange's
bit-identity), a consistent relabelling of tokens and trajectories permutes the output, and head h == a one-head
strided call at column offset h * d.  ``ops.temporal_attn_fwd[_packed]`` refuse operands the kernels would
reinterpret before any launch.

``test_report_worst_ratios`` prints the largest err / tol per kernel and family (-s to see it).
"""
import pytest
import torch

from fresco_b200.dist import frame_range
from oracle import temporal_bound as TB

pytestmark = pytest.mark.gpu

ROWS_D = (40, 64, 80)
ERR_UNSUPPORTED = -2
RATIOS = {}     # (kernel, family) -> worst err / tol


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib, ops
    _lib.lib()      # fails loudly if the extension is missing

    class NS:
        pass
    ns = NS()
    ns.lib, ns.ops, ns.c = _lib, ops, _lib.lib()
    return ns


def P(t):
    return t.data_ptr()


def rows_name(d, N):
    return f"temporal_attn_rows_kernel<{d},{8 if N <= 8 else 16}>"


def _gpu(case):
    mv = lambda t: t.cuda() if t is not None else None
    return case._replace(q=mv(case.q), k=mv(case.k), v=mv(case.v), fwd_map=mv(case.fwd_map), mask=mv(case.mask),
                         exact=mv(case.exact))


def make(fam, N, L, heads, d, chunks=2, seed=0):
    case = TB.make_case(fam, N, L, heads, d, chunks, seed)
    TB.family_property(case)
    return _gpu(case)


def _nan(*shape):
    return torch.full(shape, float("nan"), dtype=torch.float16, device="cuda")


def _u8(mask):
    return mask.to(torch.uint8).contiguous()


def call(fb, case, want, ptrs=None, stride=None, out=None):
    """fresco_temporal_attn_fwd_strided on ``case`` (dense unless ptrs / stride are given); asserts the launch name
    ``want`` and returns the output."""
    B, L, C = case.q.shape
    N = case.fwd_map.shape[0]
    d = C // case.heads
    if out is None:
        out = _nan(B, L, C)
    ptrs = ptrs or (P(case.q), P(case.k), P(case.v))
    rc = fb.c.fresco_temporal_attn_fwd_strided(*ptrs, P(out), P(case.fwd_map), P(_u8(case.mask)), case.chunks, N, L,
                                               case.heads, d, stride or C, case.scale, fb.lib.stream())
    fb.lib.check(rc, "fresco_temporal_attn_fwd_strided")
    assert fb.lib.last_kernel() == want, f"launched {fb.lib.last_kernel()}, expected {want}"
    return out


def check(case, out, kernel, what):
    """Every element within the bound (worst place reported); the exact families bit for bit."""
    ref, tol = TB.ref_and_bound(case.q, case.k, case.v, case.fwd_map, case.mask, case.chunks, case.heads, case.scale,
                                kernel)
    r = TB.ratio(out, ref, tol)
    worst = r.max().item()
    key = (kernel, case.family)
    RATIOS[key] = max(RATIOS.get(key, 0.0), worst)
    if not worst <= 1:
        row, tok, ch = (int(i) for i in torch.unravel_index(r.argmax(), r.shape))
        pytest.fail(f"{what} [{case.family}]: err/tol {worst:.3g} at row {row} token {tok} channel {ch}: out "
                    f"{out[row, tok, ch].item()!r} ref {ref[row, tok, ch].item():.6g} tol {tol[row, tok, ch].item():.3g}; "
                    f"{(r > 1).sum().item()} of {r.numel()} elements outside")
    if case.exact is not None:
        diff = (out != case.exact).sum().item()
        assert diff == 0, f"{what} [{case.family}]: {diff} elements differ from the exact answer"


# ------------------------------------------------------------------------------------------------ layouts
def traj_rows(t, case, lo, hi):
    """[chunks*N, L, C] -> [N, chunks*(hi - lo), C] fp16, row (f, b*Lg + t) = t[b*N + f, fwd_map[f, lo + t]]: the
    layout the trajectory exchange delivers to the rank owning trajectories [lo, hi)."""
    g = TB.gather(t, case.fwd_map, case.chunks, case.heads)[:, lo:hi]
    c, Lg, H, N, d = g.shape
    return g.permute(3, 0, 1, 2, 4).reshape(N, c * Lg, H * d).half()


def packed(case, lo=0, hi=None, stride=None, offsets=None):
    """(buffer, case) of the packed strided call on trajectories [lo, hi): q | k | v at ``offsets`` in rows ``stride``
    elements wide (every other column NaN), identity map, chunks = 1, the mask expanded over the chunks."""
    B, L, C = case.q.shape
    N = case.fwd_map.shape[0]
    hi = L if hi is None else hi
    stride = stride or 3 * C
    offsets = offsets or (0, C, 2 * C)
    Lt = case.chunks * (hi - lo)
    buf = _nan(N, Lt, stride)
    for o, t in zip(offsets, (case.q, case.k, case.v)):
        buf[..., o:o + C] = traj_rows(t, case, lo, hi)
    q, k, v = TB.unpack(buf, C, offsets)
    fwd = torch.arange(Lt, device="cuda")[None].expand(N, -1).contiguous()
    mask = case.mask[lo:hi][None].expand(case.chunks, -1, -1, -1).reshape(Lt, N, N).contiguous()
    exact = traj_rows(case.exact, case, lo, hi) if case.exact is not None else None
    return buf, case._replace(q=q, k=k, v=v, fwd_map=fwd, mask=mask, chunks=1, exact=exact)


def packed_ptrs(buf, offsets):
    return tuple(P(buf) + 2 * o for o in offsets)


# ================================================================================================ row kernel
def _row_sweep(d, nmax):
    """(N, heads, tokens, chunks, family) for one instantiation: every N of the NMAX range, heads 1 / 3 / 8 (where
    heads * N <= 256), token counts leaving a ragged last CTA, chunks rotating over 1 / 2 / 3, every family."""
    out = []
    for N in range(1 if nmax == 8 else 9, nmax + 1):
        fams = TB.families_for(N)
        for i, fam in enumerate(fams):
            heads = (1, 3, 8)[(i + N) % 3]
            tpb = 256 // (N * heads)                    # trajectories per CTA, as launch_temporal_rows picks them
            while tpb > 1 and tpb * (4 * N * heads * d + 4 * N) > 48 * 1024:
                tpb -= 1
            tokens = 3 * tpb + 1 + (i % 3)              # the last CTA holds 1 - 3 trajectories of tpb
            out.append((N, heads, tokens, 1 + (i + N) % 3, fam))
    return out


@pytest.mark.parametrize("d,nmax", [(d, n) for d in ROWS_D for n in (8, 16)])
def test_rows_families(fb, d, nmax):
    for N, heads, tokens, chunks, fam in _row_sweep(d, nmax):
        case = make(fam, N, tokens, heads, d, chunks, seed=N)
        out = call(fb, case, rows_name(d, N))
        check(case, out, "rows", f"rows d={d} N={N} heads={heads} tokens={tokens} chunks={chunks}")


@pytest.mark.parametrize("d", ROWS_D)
def test_rows_edges(fb, d):
    """A single token; heads * N = 256 (N = 16, 16 heads: one trajectory per CTA, over 48 KB of shared memory at
    d = 64 and 80); N = 1 with many heads."""
    for N, heads, tokens, chunks, fam in [(5, 3, 1, 2, "asymmetric"), (16, 1, 1, 1, "staircase-rising"),
                                          (16, 16, 5, 2, "reference"), (16, 16, 3, 1, "masked-max"),
                                          (8, 32, 7, 2, "asymmetric"), (1, 32, 9, 3, "huge")]:
        case = make(fam, N, tokens, heads, d, chunks, seed=heads)
        out = call(fb, case, rows_name(d, N))
        check(case, out, "rows", f"rows d={d} N={N} heads={heads} tokens={tokens} chunks={chunks}")


@pytest.mark.parametrize("N,L,d", [(8, 4096, 40), (8, 1024, 80), (16, 4096, 40), (16, 1024, 80)])
def test_rows_bench_shapes(fb, N, L, d):
    """The shapes bench.py runs (8 heads, two CFG chunks), every trajectory."""
    case = make("reference", N, L, 8, d, 2, seed=L)
    out = call(fb, case, rows_name(d, N))
    check(case, out, "rows", f"bench N={N} L={L} d={d}")


# ================================================================================================ strided entry point
@pytest.mark.parametrize("d,N", [(40, 16), (80, 16), (64, 5), (40, 3)])
def test_packed_call(fb, d, N):
    """The call ShardedTrajectoryExchange.run makes, on every family."""
    for fam in TB.families_for(N):
        case = make(fam, N, 37, 8 if N > 8 else 4, d, 2, seed=d)
        buf, pc = packed(case)
        C = case.q.shape[-1]
        out = call(fb, pc, rows_name(d, N), ptrs=packed_ptrs(buf, (0, C, 2 * C)), stride=3 * C)
        check(pc, out, "rows", f"packed d={d} N={N}")


@pytest.mark.parametrize("d", ROWS_D)
def test_strided_gaps_and_guard_rows(fb, d):
    """q, k, v at offsets 8, C + 16, 2C + 24 of rows 3C + 32 wide, every other column NaN: no NaN may reach the
    output.  ``out`` is an interior slice of a buffer whose rows before and after hold NaN and must keep it."""
    N, heads, tokens = 12, 4, 41
    case = make("reference", N, tokens, heads, d, 2, seed=5)
    C = heads * d
    offsets, stride = (8, C + 16, 2 * C + 24), 3 * C + 32
    buf, pc = packed(case, stride=stride, offsets=offsets)
    guard = 3
    full = _nan(N * pc.q.shape[1] + 2 * guard, C)
    out = full[guard:guard + N * pc.q.shape[1]].view(N, pc.q.shape[1], C)
    call(fb, pc, rows_name(d, N), ptrs=packed_ptrs(buf, offsets), stride=stride, out=out)
    assert torch.isnan(full[:guard]).all() and torch.isnan(full[-guard:]).all(), "a guard row was written"
    check(pc, out, "rows", f"strided gaps d={d}")


def test_strided_more_than_16_frames_unsupported(fb):
    """A trajectory-sharded batch of more than 16 frames cannot run today: the round-1 kernel has no strided form."""
    case = make("reference", 17, 20, 2, 40, 1)
    buf, pc = packed(case)
    C = case.q.shape[-1]
    before = (fb.lib.launch_count(), fb.lib.last_kernel())
    out = _nan(*pc.q.shape)
    rc = fb.c.fresco_temporal_attn_fwd_strided(*packed_ptrs(buf, (0, C, 2 * C)), P(out), P(pc.fwd_map), P(_u8(pc.mask)),
                                               1, 17, pc.q.shape[1], 2, 40, 3 * C, pc.scale, fb.lib.stream())
    assert rc == ERR_UNSUPPORTED and "strided inputs need frames <= 16" in fb.lib.last_error(), (rc, fb.lib.last_error())
    assert (fb.lib.launch_count(), fb.lib.last_kernel()) == before


# ================================================================================================ round-1 kernel
def _smem_round1(N, heads, d):
    return ((3 * N * d * 2 + N * N * 4 + 15) & ~15) * heads


@pytest.mark.parametrize("N,heads,d,tokens,opts", [
    (17, 8, 40, 40, None), (31, 4, 80, 20, None), (32, 2, 64, 20, None), (33, 3, 40, 20, None),
    (48, 2, 40, 12, None), (4, 4, 8, 40, None), (8, 2, 16, 40, None), (13, 3, 24, 30, None), (5, 2, 128, 30, None),
    (16, 20, 40, 10, None), (8, 8, 40, 40, {"FRESCO_TEMPORAL_V": 1}), (16, 4, 80, 20, {"FRESCO_TEMPORAL_V": 1}),
    (2, 1, 64, 20, {"FRESCO_TEMPORAL_V": 1}),
])
def test_round1_families(fb, N, heads, d, tokens, opts):
    for name, v in (opts or {}).items():
        fb.lib.set_option(name, v)
    try:
        for i, fam in enumerate(TB.families_for(N)):
            case = make(fam, N, tokens, heads, d, 1 + i % 3, seed=N + d)
            out = call(fb, case, "temporal_attn_kernel")
            check(case, out, "round1", f"round-1 N={N} heads={heads} d={d} opts={opts}")
    finally:
        for name in opts or {}:
            fb.lib.set_option(name, -1)


def test_round1_shared_memory_limit(fb):
    """The largest N whose shared memory fits 200 KB runs; the next N returns FRESCO_ERR_UNSUPPORTED and launches
    nothing."""
    heads, d = 8, 64
    n_max = max(n for n in range(17, 65) if _smem_round1(n, heads, d) <= 200 * 1024)
    assert n_max < 64
    case = make("reference", n_max, 6, heads, d, 1)
    out = call(fb, case, "temporal_attn_kernel")
    check(case, out, "round1", f"round-1 N={n_max} (largest that fits)")
    big = make("reference", n_max + 1, 6, heads, d, 1)
    before = (fb.lib.launch_count(), fb.lib.last_kernel())
    out = _nan(*big.q.shape)
    rc = fb.c.fresco_temporal_attn_fwd(P(big.q), P(big.k), P(big.v), P(out), P(big.fwd_map), P(_u8(big.mask)), 1,
                                       n_max + 1, 6, heads, d, big.scale, fb.lib.stream())
    assert rc == ERR_UNSUPPORTED, (rc, fb.lib.last_error())
    assert (fb.lib.launch_count(), fb.lib.last_kernel()) == before


# ================================================================================================ bit-exact invariances
def _gathered(out, case):
    return TB.gather(out, case.fwd_map, case.chunks, case.heads)


def _packed_gathered(res, chunks, heads):
    """packed output [N, chunks*Lg, C] -> [chunks, Lg, H, N, d]."""
    N, R, C = res.shape
    return res.double().reshape(N, chunks, R // chunks, heads, C // heads).permute(1, 2, 3, 0, 4)


@pytest.mark.parametrize("N,d", [(8, 40), (13, 80)])
def test_invariances(fb, N, d):
    heads, L, chunks = 4, 203, 2
    name = rows_name(d, N)
    case = make("reference", N, L, heads, d, chunks, seed=11)
    C = heads * d
    full = call(fb, case, name)
    fg = _gathered(full, case)
    # dense == packed, and the packed call on each trajectory block of G ranks == those rows of the full call
    for G in (1, 2, 3, 5):
        for s in range(G):
            lo, hi = frame_range(L, G, s)
            buf, pc = packed(case, lo, hi)
            res = call(fb, pc, name, ptrs=packed_ptrs(buf, (0, C, 2 * C)), stride=3 * C)
            assert torch.equal(_packed_gathered(res, chunks, heads), fg[:, lo:hi]), f"G={G} block {s} differs"
    # one chunks = 2 call == two chunks = 1 calls
    for b in range(chunks):
        sl = slice(b * N, (b + 1) * N)
        one = case._replace(q=case.q[sl].contiguous(), k=case.k[sl].contiguous(), v=case.v[sl].contiguous(), chunks=1)
        assert torch.equal(call(fb, one, name), full[sl]), f"chunk {b} alone differs"
    # relabel the tokens of every frame (pi_f) and the trajectories (sigma) consistently
    g = torch.Generator(device="cuda").manual_seed(3)
    pi = torch.stack([torch.randperm(L, device="cuda", generator=g) for _ in range(N)])        # token t -> pi[f, t]
    sigma = torch.randperm(L, device="cuda", generator=g)                                      # trajectory p -> sigma[p]
    fwd2 = torch.empty_like(case.fwd_map)
    fwd2[:, sigma] = torch.gather(pi, 1, case.fwd_map)
    mask2 = torch.empty_like(case.mask)
    mask2[sigma] = case.mask

    def relabel(t):
        t2 = torch.empty_like(t).view(chunks, N, L, C)
        for f in range(N):
            t2[:, f, pi[f]] = t.view(chunks, N, L, C)[:, f]
        return t2.view_as(t)
    moved = case._replace(q=relabel(case.q), k=relabel(case.k), v=relabel(case.v), fwd_map=fwd2, mask=mask2)
    assert torch.equal(call(fb, moved, name), relabel(full)), "relabelled tokens do not permute the output"
    # head h == a one-head strided call at column offset h * d
    for h in range(heads):
        out1 = _nan(chunks * N, L, d)
        rc = fb.c.fresco_temporal_attn_fwd_strided(P(case.q) + 2 * h * d, P(case.k) + 2 * h * d, P(case.v) + 2 * h * d,
                                                   P(out1), P(case.fwd_map), P(_u8(case.mask)), chunks, N, L, 1, d, C,
                                                   case.scale, fb.lib.stream())
        fb.lib.check(rc, "one-head strided call")
        assert fb.lib.last_kernel() == name
        assert torch.equal(out1, full[..., h * d:(h + 1) * d]), f"head {h} differs from the one-head call"


# ================================================================================================ operand validation
def test_operand_validation(fb):
    """ops.temporal_attn_fwd[_packed] refuse what the kernels would reinterpret, before any launch."""
    N, L, heads, d, chunks = 4, 16, 2, 40, 2
    case = make("reference", N, L, heads, d, chunks)
    q, k, v, fwd, mask = case.q, case.k, case.v, case.fwd_map, _u8(case.mask)
    qkv = torch.cat([q, k, v], -1).contiguous()
    bad_dense = {
        "fp32 q": (q.float(), k, v, fwd, mask, chunks, heads),
        "fp32 v": (q, k, v.float(), fwd, mask, chunks, heads),
        "int32 fwd_map": (q, k, v, fwd.int(), mask, chunks, heads),
        "fwd_map [N, L + 1]": (q, k, v, torch.zeros(N, L + 1, dtype=torch.int64, device="cuda"), mask, chunks, heads),
        "mask [N, L]": (q, k, v, fwd, mask[:, 0, :].t().contiguous(), chunks, heads),
        "float mask": (q, k, v, fwd, mask.float(), chunks, heads),
        "rows not divisible by chunks": (q, k, v, fwd, mask, 3, heads),
        "C not divisible by heads": (q, k, v, fwd, mask, chunks, 3),
    }
    bad_packed = {
        "fp32 qkv": (qkv.float(), fwd, mask, chunks, heads),
        "int32 fwd_map": (qkv, fwd.int(), mask, chunks, heads),
        "mask [L, N, N + 1]": (qkv, fwd, torch.ones(L, N, N + 1, dtype=torch.uint8, device="cuda"), chunks, heads),
        "rows not divisible by chunks": (qkv, fwd, mask, 3, heads),
        "C not divisible by heads": (qkv, fwd, mask, chunks, 3),
    }
    before = (fb.lib.launch_count(), fb.lib.last_kernel())
    for what, args in bad_dense.items():
        with pytest.raises(fb.lib.FrescoError):
            fb.ops.temporal_attn_fwd(*args, case.scale)
        assert (fb.lib.launch_count(), fb.lib.last_kernel()) == before, f"temporal_attn_fwd launched on {what}"
    for what, args in bad_packed.items():
        with pytest.raises(fb.lib.FrescoError):
            fb.ops.temporal_attn_fwd_packed(*args, case.scale)
        assert (fb.lib.launch_count(), fb.lib.last_kernel()) == before, f"temporal_attn_fwd_packed launched on {what}"
    # the valid calls still run, with bool masks too
    out = fb.ops.temporal_attn_fwd(q, k, v, fwd, case.mask, chunks, heads, case.scale)
    check(case, out, "rows", "ops.temporal_attn_fwd")
    res = fb.ops.temporal_attn_fwd_packed(qkv, fwd, mask, chunks, heads, case.scale)
    assert torch.equal(res, out)


def test_report_worst_ratios():
    if not RATIOS:
        pytest.skip("no temporal attention case ran")
    for (kernel, fam), r in sorted(RATIOS.items()):
        print(f"temporal worst err/tol {kernel:7s} {fam:18s} {r:.3g}")
