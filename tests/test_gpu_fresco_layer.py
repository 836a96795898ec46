"""One FRESCO self-attention layer end to end on the GPU, held to the bound composed from its kernels' bounds
(oracle/layer_bound.py).

Every layer family runs at every shape through ``FRESCOAttnProcessor2_0`` and through ``ShardedFRESCOAttention`` at
world 1, under the eight on/off combinations of cross-frame / spatial-guided / temporal-guided attention (the families
include the frame-0 fallback, a frame-0-only and an all-selecting mask and masks at several resolutions).  The
processor runs fp32 and fp16 modules on 3-D and 4-D hidden states, all four pairs over the eight modes (the sharded
layer takes the fp16 projections themselves).  A spy on ``ops`` (a spying backend for the sharded layer) records every
launch's operands, result and ``fresco_last_kernel`` name; a forward-pre-hook on ``to_out[0]`` records the attention
result.  Per call:

* the launches, in order, are the ones the modes select;
* the operands of the first stage bit-equal the test's own ``attn.to_q/k/v(x).half()``;
* each stage's result is within its composed bound (stage 1 its own, stage 2 its own on the query it received plus
  the propagated query error, stage 3 its own on the V it received plus the propagated V error), the first stage
  outside names itself;
* the attention result is within the composed bound, and for fp32 modules the processor's output within it plus the
  to_out term;
* the exact family's result is bit for bit the copy of V rows the reference names.

From ``LARGE`` tokens the fp64 reference is evaluated on all frames' rows of ``SAMPLE`` sampled trajectories (tokens
without temporal guidance).  A sequence of keyframe batches through the same layer objects checks that the cached
K/V indices, trajectories and exchange plans follow each batch.  The worst err/tol per family and stage is printed by
``test_report_worst_ratios``.
"""
import collections
import math
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import layer_bound as LB  # noqa: E402  (checker only)

# (name, N, (H, W) of the tokens, heads, head_dim, chunks)
SHAPES = [
    ("up3-64x64-N8", 8, (64, 64), 8, 40, 2),
    ("up2-32x32-N8", 8, (32, 32), 8, 80, 2),
    ("768-96x96-N2", 2, (96, 96), 8, 40, 2),
    ("768-48x48-N4", 4, (48, 48), 8, 80, 2),
    ("envelope-40x56-N4", 4, (40, 56), 8, 40, 2),
    ("envelope-20x28-N4", 4, (20, 28), 8, 80, 2),
    ("7x9-N3", 3, (7, 9), 2, 40, 2),
    ("N1-16x16", 1, (16, 16), 8, 40, 2),
    ("N16-16x16", 16, (16, 16), 8, 40, 2),
    ("N17-12x12", 17, (12, 12), 8, 40, 2),
    ("chunks1-16x16-N4", 4, (16, 16), 8, 40, 1),
]
LARGE = 1024                        # from this many tokens: the reference on a sample of the trajectories
SAMPLE = 256
WORST = collections.defaultdict(float)


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib, diffusion_hacked, dist, ops
    _lib.lib()
    torch.backends.cuda.matmul.allow_tf32 = False

    class NS:
        pass
    ns = NS()
    ns.ops, ns.dh, ns.dist, ns.lib = ops, diffusion_hacked, dist, _lib
    return ns


class Planted(torch.nn.Module):
    """A projection that returns the family's planted operand for each input it is given."""

    def __init__(self, table):
        super().__init__()
        self.table = table

    def forward(self, x):
        for inp, out in self.table:
            if inp.shape == x.shape and torch.equal(inp, x):
                return out.to(x.dtype)
        raise KeyError("input not planted")


class Attn(torch.nn.Module):
    def __init__(self, case, x, rh, dtype, seed):
        super().__init__()
        ops = case.ops
        C = ops.q.shape[-1]
        self.heads = ops.heads
        self.spatial_norm = self.group_norm = None
        self.norm_cross = self.residual_connection = False
        self.rescale_output_factor = 1.0
        if case.weights is not None:
            self.to_q, self.to_k, self.to_v = (torch.nn.Linear(C, C, bias=False) for _ in range(3))
            with torch.no_grad():
                for lin, w in zip((self.to_q, self.to_k, self.to_v), case.weights):
                    lin.weight.copy_(w)
        else:
            dev = x.device
            self.to_q = Planted([(x, ops.q.to(dev)), (rh, ops.q_ref.to(dev))])
            self.to_k = Planted([(x, ops.k.to(dev)), (rh, ops.k_ref.to(dev))])
            self.to_v = Planted([(x, ops.v.to(dev))])
        g = torch.Generator().manual_seed(seed)
        self.to_out = torch.nn.ModuleList([torch.nn.Linear(C, C), torch.nn.Dropout(0.0)])
        with torch.no_grad():
            self.to_out[0].weight.copy_(torch.randn(C, C, generator=g) / math.sqrt(C))
            self.to_out[0].bias.copy_(0.1 * torch.randn(C, generator=g))
        self.to(x.device, dtype)


def _controller(fb, ctl, ref_hidden, c=None):
    c = c if c is not None else fb.dh.AttentionControl()
    c.intraattn_scale_factor, c.intraattn_bias, c.interattn_scale_factor = ctl.intra_scale, ctl.intra_bias, ctl.inter_scale
    dev = ref_hidden.device
    if ctl.use_intra:
        c.stored_attn["decoder_attn"] = [ref_hidden]
        c.enable_intraattn()
    else:
        c.disable_intraattn()
    if ctl.use_inter:
        c.enable_interattn({"fwd_mappings": [t.to(dev) for t in ctl.fwd_maps],
                            "bwd_mappings": [t.to(dev) for t in ctl.bwd_maps],
                            "interattn_masks": [t.to(dev) for t in ctl.inter_masks]})
    else:
        c.disable_interattn()
    if ctl.use_cf:
        c.enable_cfattn([m.to(dev) for m in ctl.masks])
    else:
        c.disable_cfattn()
    return c


class Spy:
    """Records (entry point, args, result, launch name) of every call it wraps."""

    def __init__(self, fb):
        self.fb, self.calls = fb, []

    def wrap(self, name, fn):
        def call(*a, **kw):
            out = fn(*a, **kw)
            res = tuple(t.clone() for t in out) if isinstance(out, tuple) else out.clone()
            self.calls.append((name, a, kw, res, self.fb.lib.last_kernel()))
            return out
        return call


def _spying_backend(fb, spy):
    base = fb.dist._OpsBackend()

    class SpyBackend:
        pass
    be = SpyBackend()
    for name in ("kv_compact_packed", "rows_gather", "rows_scatter", "attn_fwd", "attn_fwd_kv_packed",
                 "temporal_attn_fwd", "temporal_attn_fwd_packed"):
        setattr(be, name, spy.wrap(name, getattr(base, name)))
    return be


def _variant(fb, d):
    name = fb.lib.lib().fresco_attn_variant(d).decode()
    poly = int(re.search(r"poly(\d+)", name).group(1))
    return name.replace(" (wgmma)", ""), poly, ",rowsum" in name


def _expected_launches(fb, ctl, N, L, d, sharded):
    attn, _, _ = _variant(fb, d)
    has_mask = LB.kv_rows(ctl, N, L) is not None
    names = []
    if sharded:
        names += [attn] if ctl.use_intra else []
        names += ["kv_compact_packed_kernel"] if ctl.use_cf and has_mask else []
        names += [attn]
    else:
        names += ["kv_compact_kernel"] if ctl.use_cf and has_mask else []
        names += [attn] * (2 if ctl.use_intra else 1)
    if ctl.use_inter:
        names += [f"temporal_attn_rows_kernel<{d},{8 if N <= 8 else 16}>" if N <= 16 else "temporal_attn_kernel"]
    return names


def _sample(case, ctl, L, seed):
    if L < LARGE:
        return None
    g = torch.Generator().manual_seed(seed)
    return torch.randperm(L, generator=g)[:SAMPLE].sort().values


def _record(key, r):
    WORST[key] = max(WORST[key], r)


def run_layer(fb, monkeypatch, case, flags, path, dtype, four_d, sample_seed=0, state=None):
    """One call of the layer on ``case`` under ``flags``; asserts everything the module docstring lists.  ``state``:
    (processor or sharded layer, controller) to run the same objects again (a second keyframe batch)."""
    ops, ctl = case.ops, case.ctl.modes(flags)
    B, L, C = ops.q.shape
    heads, chunks = ops.heads, ops.chunks
    N, d = B // chunks, C // heads
    Hs, Ws = case.grid
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(1000 + flags)
    if case.x is not None:
        x = case.x.to(dev, dtype)
        rh = case.ref_hidden.to(dev, dtype)
    else:
        x = torch.randn(B, L, C, generator=g, device=dev).to(dtype)
        rh = torch.randn(B, L, C, generator=g, device=dev).to(dtype)
    attn = Attn(case, x, rh, dtype, seed=flags)
    with torch.no_grad():
        want = {"q": attn.to_q(x).half(), "k": attn.to_k(x).half(), "v": attn.to_v(x).half(),
                "q_ref": attn.to_q(rh).half(), "k_ref": attn.to_k(rh).half()}
    spy = Spy(fb)
    got = {}
    if path == "processor":
        for name in ("kv_compact", "attn_fwd", "temporal_attn_fwd"):
            monkeypatch.setattr(fb.ops, name, spy.wrap(name, getattr(fb.ops, name)))
        if state is None:
            ctrl = _controller(fb, ctl, rh)
            layer = fb.dh.FRESCOAttnProcessor2_0(chunks, ctrl)
        else:
            layer, ctrl = state
            _controller(fb, ctl, rh, ctrl)
        attn.to_out[0].register_forward_pre_hook(lambda m, a: got.setdefault("a", a[0].clone()))
        hidden = x.transpose(1, 2).reshape(B, C, Hs, Ws) if four_d else x
        with torch.no_grad():
            y = layer(attn, hidden)
        monkeypatch.undo()
        if four_d:
            y = y.reshape(B, C, L).transpose(1, 2)
        a = got["a"]
    else:
        if state is None:
            ctrl = _controller(fb, ctl, rh)
            layer = fb.dist.ShardedFRESCOAttention(ctrl, 1, 0, chunks, backend=_spying_backend(fb, spy))
        else:
            layer, ctrl = state
            _controller(fb, ctl, rh, ctrl)
            layer.backend = _spying_backend(fb, spy)
        with torch.no_grad():
            a = layer(want["q"], want["k"], want["v"], heads, ref_q=want["q_ref"], ref_k=want["k_ref"])
        y = None
    torch.cuda.synchronize()
    what = f"{case.family} flags={flags} {path} {dtype} {'4-D' if four_d else '3-D'} N={N} L={L} d={d}"

    # launches, in order
    names = [c[4] for c in spy.calls if c[0] not in ("rows_gather", "rows_scatter")]
    assert names == _expected_launches(fb, ctl, N, L, d, path != "processor"), (what, names)

    # first-stage operands: the projections, bit for bit
    attn_calls = [c for c in spy.calls if c[0] in ("attn_fwd", "attn_fwd_kv_packed")]
    if ctl.use_intra:
        sq, sk, sv = attn_calls[0][1][:3]
        assert torch.equal(sq, want["q_ref"]) and torch.equal(sk, want["k_ref"]) and torch.equal(sv, want["q"]), what
    cross = attn_calls[-1]
    if not ctl.use_intra:
        assert torch.equal(cross[1][0], want["q"]), what
    if not ctl.use_cf:
        assert torch.equal(cross[1][1], want["k"]) and torch.equal(cross[1][2], want["v"]), what
    for c in spy.calls:
        if c[0] in ("kv_compact", "kv_compact_packed"):
            assert torch.equal(c[1][0], want["k"]) and torch.equal(c[1][1], want["v"]), what
    temporal = [c for c in spy.calls if c[0] == "temporal_attn_fwd"]
    if temporal:
        assert torch.equal(temporal[0][1][0], want["q"]) and torch.equal(temporal[0][1][1], want["k"]), what

    # the composed bound, stage by stage
    _, poly, rowsum = _variant(fb, d)
    ops_gpu = LB.Operands(want["q"], want["k"], want["v"], want["q_ref"], want["k_ref"], heads, chunks)
    received = {"cross_q": cross[1][0]}
    outs = {"cross": cross[3]}
    if ctl.use_intra:
        outs["spatial"] = attn_calls[0][3]
    if temporal:
        received["temporal_v"] = temporal[0][1][2]
        outs["temporal"] = temporal[0][3]
    sample = _sample(case, ctl, L, sample_seed)
    lay = LB.evaluate(ops_gpu, ctl, sample, received, poly=poly, rowsum=rowsum, device=dev)
    rows = lay.rows.to(dev)
    take = lambda t: torch.gather(t, 1, rows[..., None].expand(-1, -1, C))
    for stage in ("spatial", "cross", "temporal"):
        if stage not in lay.ref:
            continue
        r = LB.ratio(take(outs[stage]), lay.ref[stage], lay.tol[stage])
        _record((case.family, stage), r.max().item())
        if (r > 1).any():
            own = LB.ratio(take(outs[stage]), lay.ref[stage], lay.own[stage]) if stage != "spatial" else r
            pytest.fail(f"{what}: stage {stage} outside its composed bound (err/tol {r.max().item():.3g}; "
                        f"against its own kernel bound alone {own.max().item():.3g})")
    ref, tol = LB.attention_result(lay)
    r = LB.ratio(take(a), ref, tol)
    _record((case.family, "attention"), r.max().item())
    assert not (r > 1).any(), f"{what}: attention result err/tol {r.max().item():.3g}"
    if case.family == "exact":
        assert torch.equal(take(a.half()), ref.half()), f"{what}: not the V rows the reference names"
    if y is not None and dtype == torch.float32:
        yr, yt = LB.out_stage(ref, tol, attn.to_out[0].weight, attn.to_out[0].bias, take(a))
        r = LB.ratio(take(y), yr, yt)
        _record((case.family, "out"), r.max().item())
        assert not (r > 1).any(), f"{what}: processor output err/tol {r.max().item():.3g}"
    return layer, ctrl


class _Gridded:
    """a layer_bound.Case with the (H, W) of its tokens"""

    def __init__(self, case, grid):
        self.__dict__.update(case._asdict())
        self.grid = grid


CASES = [(s[0], f) for s in SHAPES for f in LB.FAMILIES]


def processor_module(flags):
    """(dtype, 4-D hidden states) of the processor's module under ``flags``: every pair twice over the eight modes,
    each pair with and without cross-frame and temporal-guided attention"""
    dtype = torch.float32 if bin(flags).count("1") % 2 == 0 else torch.float16
    return dtype, (flags >> 1) % 2 == 1


@pytest.mark.parametrize("shape,family", CASES, ids=[f"{s}-{f}" for s, f in CASES])
def test_layer_within_composed_bound(fb, monkeypatch, shape, family):
    _, N, grid, heads, d, chunks = next(s for s in SHAPES if s[0] == shape)
    L = grid[0] * grid[1]
    cases = {}
    for flags in range(8):
        cf = bool(flags & 1) if family == "exact" else True           # the exact family's beacons depend on it
        if cf not in cases:
            cases[cf] = _Gridded(LB.make_case(family, N, L, heads, d, chunks, seed=1, grid=grid, use_cf=cf), grid)
            LB.family_property(cases[cf], 7 if cf else 6, _sample(cases[cf], None, L, 0), device="cuda")
        dtype, four_d = processor_module(flags)
        run_layer(fb, monkeypatch, cases[cf], flags, "processor", dtype, four_d)
        run_layer(fb, monkeypatch, cases[cf], flags, "sharded", torch.float16, False)


# keyframe batches of one token count, one after another through the same layer: each changes the masks and mappings
BATCHES = [("realistic", 3), ("temporal-dominant", 4), ("exact", 5), ("temporal-dominant", 6)]


def test_keyframe_batches_rebuild_the_caches(fb, monkeypatch):
    """The same processor / sharded layer and controller on the batches of ``BATCHES``: the cached K/V indices,
    trajectories and exchange plans must follow each batch.  First it is shown that a layer keeping the previous
    batch's K/V indices or trajectories would miss every batch's reference by more than twice the composed bound."""
    N, grid, heads, d = 4, (16, 16), 8, 40
    L = grid[0] * grid[1]
    cases = [_Gridded(LB.make_case(f, N, L, heads, d, 2, seed=s, grid=grid), grid) for f, s in BATCHES]
    for before, case in zip(cases, cases[1:]):
        ctl = case.ctl.modes(7)
        ref, tol = LB.attention_result(LB.evaluate(case.ops, ctl, device="cuda"))
        for kind, old in (("kv-indices", ctl._replace(masks=before.ctl.masks)),
                          ("trajectories", ctl._replace(fwd_maps=before.ctl.fwd_maps, bwd_maps=before.ctl.bwd_maps,
                                                        inter_masks=before.ctl.inter_masks))):
            mut, _ = LB.attention_result(LB.evaluate(case.ops, old, device="cuda"))
            sep = ((mut - ref).abs() / tol).max().item()
            assert sep > 2.0, f"stale {kind} into {case.family}: only {sep:.3g} x the bound"
    for path in ("processor", "sharded"):
        state = None
        for case in cases:
            state = run_layer(fb, monkeypatch, case, 7, path, torch.float32 if path == "processor" else torch.float16,
                              False, state=state)


def test_report_worst_ratios():
    """Print the worst err/tol per family and stage (all <= 1 when the tests above pass)."""
    if not WORST:
        pytest.skip("no layer ran")
    for (fam, stage), r in sorted(WORST.items()):
        print(f"layer {fam:18s} {stage:9s} worst err/tol {r:.3g}")
