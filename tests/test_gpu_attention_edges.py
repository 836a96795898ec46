"""fresco_attn_kernel on inputs built to break its online softmax, on every instantiation the options select.

Each case fills the output with NaN, runs the C ABI, asserts the instantiation ``fresco_last_kernel()`` reports, and
checks every element against the fp64 reference with the elementwise bound of ``oracle.attention_bound``
(|out - ref| <= tol).  Inputs are built in fp32 and rounded to fp16; ``family_property`` asserts on the fp64 logits the
property that makes each family sensitive:

* staircase (rising, falling, sawtooth): the row max keeps moving, so alpha < 1 on every turn and a stale or misplaced
  rescale of O or l shows; V channel 0 is the key's 64-key block, so that output channel is the mean block index.
* one-hot: one key per row >= 30 nats above the rest, at the first tile, the last full tile, the ragged last key and
  both sides of 16-key k-steps; V encodes the key index, so a dropped, doubled or misplaced P V shows as a wrong key.
* negative floor: every logit <= -20 nats and V ~ 1, so a zero-filled key past kv_len (logit 0, V = 0) takes the row.
* flat: Lk = 15587 (the dominant launch) with all logits equal to within a fraction of a nat: l and O over 122 tiles.
* diagonal: diag_bias +8 / -8 / 1.5 at softmax_scale 0.2 / sqrt(d), Lq = Lk = 64 n +- 1 and Lq != Lk, across CTA tiles
  of 128 and 192 rows and key tiles of 64 and 128.
* peaky: logits spread over ~100 nats; most of P is subnormal or zero in fp16.

The one-hot and negative-floor families sweep kv_len at q_len = 129 (n_tiles = 1 up to two wraps of a 4-stage ring)
and q_len at kv_len = 4 KN + 1 (warpgroups whose rows are all past q_len).  Guard buffers check that no operand is
read and no output written past its end, and five bit-exact invariances pin what the kernel's structure guarantees.
``test_report_worst_ratios`` prints the largest err / tol per family and variant.
"""
import collections
import math

import pytest
import torch

from oracle import attention_bound as AB

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib
    _lib.lib()      # fails loudly if the extension is missing
    torch.backends.cuda.matmul.allow_tf32 = False

    class NS:
        pass
    ns = NS()
    ns.lib, ns.c = _lib, _lib.lib()
    return ns


Variant = collections.namedtuple("Variant", "d wide poly rowsum")
VARIANTS = [Variant(d, wide, poly, rowsum)
            for d in (40, 64, 80, 128)
            for wide in ((0, 1, 2) if d <= 64 else (0, 1))
            for poly in (0, 4, 8)
            for rowsum in ((0, 1) if wide == 0 else (0,))]
assert len(VARIANTS) == 42


def _vid(v):
    return "d%d-wide%d-poly%d-rowsum%d" % v


def _kn(v):
    return 64 if v.wide == 0 else 128


def _tile_m(v):
    return 192 if v.wide == 2 else 128


def _name(v):
    return "fresco_attn_kernel<%d,keys%d,wg%d,poly%d%s>" % (v.d, _kn(v), 3 if v.wide == 2 else 2, v.poly,
                                                           ",rowsum" if v.rowsum else "")


@pytest.fixture(params=VARIANTS, ids=_vid)
def v(fb, request):
    var = request.param
    opts = {"FRESCO_ATTN_WIDE": var.wide, "FRESCO_ATTN_POLY": var.poly, "FRESCO_ATTN_ROWSUM": var.rowsum}
    for name, val in opts.items():
        fb.lib.set_option(name, val)
    yield var
    for name in opts:
        fb.lib.set_option(name, -1)


RATIOS = {}     # (family, variant id) -> worst err / tol


def _launch(fb, v, q, k, vv, out, heads, qpk, scale, bias, kv_stride=None):
    """fresco_attn_fwd, or fresco_attn_fwd_kv_strided with kv_stride = (row, batch) in elements."""
    Bq, Lq, C = q.shape
    Lk = k.shape[1]
    if kv_stride is None:
        rc = fb.c.fresco_attn_fwd(q.data_ptr(), k.data_ptr(), vv.data_ptr(), out.data_ptr(), Bq, Lq, Lk, heads,
                                  C // heads, qpk, scale, bias, fb.lib.stream())
    else:
        rc = fb.c.fresco_attn_fwd_kv_strided(q.data_ptr(), k.data_ptr(), vv.data_ptr(), out.data_ptr(), Bq, Lq, Lk,
                                             heads, C // heads, qpk, kv_stride[0], kv_stride[1], scale, bias,
                                             fb.lib.stream())
    fb.lib.check(rc, "fresco_attn_fwd")
    assert fb.lib.last_kernel() == _name(v), f"launched {fb.lib.last_kernel()}, want {_name(v)}"


def _run(fb, v, q, k, vv, heads, qpk=1, scale=None, bias=0.0):
    out = torch.full(q.shape, float("nan"), dtype=torch.float16, device="cuda")
    scale = 1.0 / math.sqrt(q.shape[2] // heads) if scale is None else scale
    _launch(fb, v, q, k, vv, out, heads, qpk, scale, bias)
    return out


def _check(v, family, what, out, q, k, vv, heads, qpk, scale, bias):
    """|out - ref| <= tol on every element; the failure names the worst element, its CTA row tile and key read."""
    ref, tol = AB.ref_and_bound(q, k, vv, heads, qpk, scale, bias, v.poly, bool(v.rowsum))
    ratio = ((out.double() - ref).abs() / tol).nan_to_num(nan=float("inf"))
    worst = ratio.max().item()
    key = (family, _vid(v))
    RATIOS[key] = max(RATIOS.get(key, 0.0), worst)
    if worst <= 1.0:
        return
    b, row, ch = (int(i) for i in torch.unravel_index(ratio.argmax(), ratio.shape))
    d = q.shape[2] // heads
    n_bad = (ratio > 1).sum().item()
    rows_bad = sorted({int(r) // _tile_m(v) for r in (ratio > 1).any(-1).nonzero()[:, 1].tolist()})
    raise AssertionError(
        f"{family} {what}: {n_bad} elements over the bound; worst err/tol {worst:.3g} at batch {b} row {row} "
        f"(row tile {row // _tile_m(v)} of {_tile_m(v)} rows) head {ch // d} channel {ch % d}: "
        f"out {out[b, row, ch].item():.6g} ref {ref[b, row, ch].item():.6g} tol {tol[b, row, ch].item():.3g}; "
        f"channel 0 of that row {out[b, row, ch - ch % d].item():.6g} (ref {ref[b, row, ch - ch % d].item():.6g}); "
        f"failing row tiles {rows_bad}")


def _case(fb, v, case, what=""):
    AB.family_property(case, _kn(v))
    out = _run(fb, v, case.q, case.k, case.v, case.heads, case.q_per_kv, case.scale, case.diag_bias)
    _check(v, case.family, what, out, case.q, case.k, case.v, case.heads, case.q_per_kv, case.scale, case.diag_bias)


# ================================================================================================ input families
def test_staircase(fb, v):
    for i, kind in enumerate(("rising", "falling", "sawtooth")):
        _case(fb, v, AB.staircase(v.d, 193, 9 * 128 + 37, kind, kn=_kn(v), heads=2, seed=10 + i, device="cuda"))


def _kv_sweep(kn):
    return sorted({1, 2, 16, 17} | {n * kn + e for n in range(1, 10) for e in (-1, 0, 1)})


Q_SWEEP = (1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 257)


def test_one_hot_and_negative_floor_kv_len_sweep(fb, v):
    kn = _kn(v)
    for kv_len in _kv_sweep(kn):
        _case(fb, v, AB.one_hot(v.d, 129, kv_len, kn=kn, heads=2, seed=kv_len, device="cuda"), f"kv_len {kv_len}")
        _case(fb, v, AB.negative_floor(v.d, 129, kv_len, heads=2, seed=kv_len, device="cuda"), f"kv_len {kv_len}")


def test_one_hot_and_negative_floor_q_len_sweep(fb, v):
    kn = _kn(v)
    for q_len in Q_SWEEP:
        _case(fb, v, AB.one_hot(v.d, q_len, 4 * kn + 1, kn=kn, heads=2, seed=q_len, device="cuda"), f"q_len {q_len}")
        _case(fb, v, AB.negative_floor(v.d, q_len, 4 * kn + 1, heads=2, seed=q_len, device="cuda"), f"q_len {q_len}")


def test_flat_dominant_key_count(fb, v):
    _case(fb, v, AB.flat(v.d, 200, 15587, seed=3, device="cuda"), "Lk 15587")


DIAG_L = (63, 65, 127, 129, 191, 193, 255, 257, 383, 385, 575, 577, 767, 769, 959, 961)


def test_diagonal_bias(fb, v):
    for bias in (8.0, -8.0, 1.5):
        for L in DIAG_L:
            _case(fb, v, AB.diagonal(v.d, L, L, bias, seed=L, device="cuda"), f"Lq = Lk = {L}")
        for Lq in (193, 385):
            for Lk in (Lq // 2 + 3, 2 * Lq - 5):
                _case(fb, v, AB.diagonal(v.d, Lq, Lk, bias, seed=Lq + Lk, device="cuda"), f"Lq {Lq} Lk {Lk}")


def test_peaky(fb, v):
    _case(fb, v, AB.peaky(v.d, 193, 1000, heads=2, seed=5, device="cuda"))


# ================================================================================================ guard buffers
GUARD = 4096


def _inside(t):
    """t copied into the middle of a flat NaN allocation; returns (allocation, view of t)."""
    buf = torch.full((GUARD + t.numel() + GUARD,), float("nan"), dtype=t.dtype, device="cuda")
    buf[GUARD:GUARD + t.numel()] = t.flatten()
    return buf, buf[GUARD:GUARD + t.numel()].view(t.shape)


def test_guard_buffers(fb, v):
    """No operand row past the tensor end is read (it would bring NaN in), and no byte of the output allocation outside
    the output is written -- for fresco_attn_fwd and for fresco_attn_fwd_kv_strided with a padded batch stride."""
    kn, heads = _kn(v), 2
    a = AB.diagonal(v.d, 193, 2 * kn + 17, 1.5, heads=heads, seed=21, device="cuda")
    b = AB.diagonal(v.d, 193, 2 * kn + 17, 1.5, heads=heads, seed=22, device="cuda")
    q = torch.cat([a.q, b.q])                                         # two query frames per K/V batch
    C, Lk = q.shape[2], a.k.shape[1]
    # dense K and V
    _, qg = _inside(q)
    _, kg = _inside(a.k)
    _, vg = _inside(a.v)
    obuf, og = _inside(torch.full_like(q, float("nan")))
    before = obuf.view(torch.int16).clone()
    _launch(fb, v, qg, kg, vg, og, heads, 2, a.scale, a.diag_bias)
    outside = torch.ones(obuf.numel(), dtype=torch.bool, device="cuda")
    outside[GUARD:GUARD + q.numel()] = False
    assert torch.equal(obuf.view(torch.int16)[outside], before[outside]), "fresco_attn_fwd wrote outside the output"
    _check(v, "guard", "dense", og.clone(), q, a.k, a.v, heads, 2, a.scale, a.diag_bias)
    # K | V packed [1, Lk + pad, 2C], the pad rows NaN
    pad = 29
    kv = torch.full((1, Lk + pad, 2 * C), float("nan"), dtype=torch.float16, device="cuda")
    kv[:, :Lk, :C], kv[:, :Lk, C:] = a.k, a.v
    _, kvg = _inside(kv)
    obuf, og = _inside(torch.full_like(q, float("nan")))
    before = obuf.view(torch.int16).clone()
    _launch(fb, v, qg, kvg[:, :Lk, :C], kvg[:, :Lk, C:], og, heads, 2, a.scale, a.diag_bias,
            kv_stride=(2 * C, (Lk + pad) * 2 * C))
    assert torch.equal(obuf.view(torch.int16)[outside], before[outside]), "kv_strided wrote outside the output"
    _check(v, "guard", "kv_strided", og.clone(), q, a.k, a.v, heads, 2, a.scale, a.diag_bias)


# ================================================================================================ bit-exact invariances
def _bits(t):
    return t.view(torch.int16)


def test_bit_exact_invariances(fb, v):
    """(a) permuting query rows, within and across CTAs, permutes the output rows; (b) q_per_kv = 4 equals K/V
    replicated four times; (c) K | V packed through kv_strided equals dense K and V; (d) three heads equal three
    single-head calls; (e) a repeated call gives the same bits after another launch.  POLY variants give the
    polynomial to pairs of the second row each thread holds (row % 16 >= 8), so their permutation keeps every row in
    its half of its 16-row group."""
    d, heads, qpk, Lq, Lk = v.d, 3, 4, 385, 700
    g = torch.Generator(device="cuda").manual_seed(31 + d)
    C = heads * d
    q = (2.0 * torch.randn(qpk, Lq, C, device="cuda", generator=g)).half()
    k = torch.randn(1, Lk, C, device="cuda", generator=g).half()
    vv = torch.randn(1, Lk, C, device="cuda", generator=g).half()
    base = _run(fb, v, q, k, vv, heads, qpk)
    _check(v, "invariance", "base", base, q, k, vv, heads, qpk, 1.0 / math.sqrt(d), 0.0)
    # (a)
    pg = torch.Generator().manual_seed(7)
    if v.poly:
        rows = torch.arange(Lq)
        perm = torch.empty(Lq, dtype=torch.long)
        for half in (False, True):
            idx = rows[((rows % 16) >= 8) == half]
            perm[idx] = idx[torch.randperm(idx.numel(), generator=pg)]
    else:
        perm = torch.randperm(Lq, generator=pg)
    perm = perm.cuda()
    assert torch.equal(_bits(_run(fb, v, q[:, perm].contiguous(), k, vv, heads, qpk)), _bits(base[:, perm])), "(a)"
    # (b)
    got = _run(fb, v, q, k.repeat(qpk, 1, 1), vv.repeat(qpk, 1, 1), heads, 1)
    assert torch.equal(_bits(got), _bits(base)), "(b) q_per_kv against replicated K/V"
    # (c)
    kv = torch.cat([k, vv], -1).contiguous()
    out = torch.full_like(q, float("nan"))
    _launch(fb, v, q, kv[..., :C], kv[..., C:], out, heads, qpk, 1.0 / math.sqrt(d), 0.0, kv_stride=(2 * C, Lk * 2 * C))
    assert torch.equal(_bits(out), _bits(base)), "(c) kv_strided packed against dense"
    # (d)
    for h in range(heads):
        sl = slice(h * d, (h + 1) * d)
        got = _run(fb, v, q[..., sl].contiguous(), k[..., sl].contiguous(), vv[..., sl].contiguous(), 1, qpk)
        assert torch.equal(_bits(got), _bits(base[..., sl])), f"(d) head {h} alone"
    # (e)
    assert torch.equal(_bits(_run(fb, v, q, k, vv, heads, qpk)), _bits(base)), "(e) repeated call"


def test_report_worst_ratios():
    """Prints the largest err / tol seen per family (over variants) and per family and variant (-s to see it)."""
    if not RATIOS:
        pytest.skip("no attention case ran")
    fams = sorted({f for f, _ in RATIOS})
    print("\nworst err/tol per family: max over variants (variant), min over variants")
    for f in fams:
        items = {vid: r for (ff, vid), r in RATIOS.items() if ff == f}
        top = max(items, key=items.get)
        print(f"  {f:20s} {items[top]:.3f} ({top})  min {min(items.values()):.3f}")
    print("per family and variant:")
    for vid in sorted({vid for _, vid in RATIOS}):
        print("  " + vid + " " + " ".join(f"{f}={RATIOS[(f, vid)]:.3f}" for f in fams if (f, vid) in RATIOS))
