"""The staged fp64 reference of one FRESCO self-attention layer (oracle/layer_bound.py) and the host glue around the
kernels, on the CPU.

* The staged reference, on the golden fixtures' fp32 projections evaluated in fp64, reproduces the reference's own
  outputs (sets A and B, every mode combination the fixtures hold, and cross-frame attention without a mask at the
  layer's resolution), and equals ``oracle.fresco_attention`` run in fp64 at chunks 1 and 2, N = 1, ragged L and the
  frame-0 fallback.  This pins it to the reference as ``fresco_oracle`` is pinned.
* ``FRESCOAttnProcessor2_0`` (``ops`` replaced by fp64 stand-ins) and ``ShardedFRESCOAttention`` at world 1 (an fp64
  backend) equal the staged reference to fp64 rounding at every family and mode.
* The logit-propagation term of the composed bound holds under adversarial perturbations of the query.
* Every named glue mutant differs from the layer by more than twice the composed bound on its family: no layer within
  the bound could pass for both.
"""
import math

import numpy as np
import pytest
import torch

from oracle import attention_bound as AB
from oracle import fresco_oracle as O
from oracle import layer_bound as LB
from oracle import temporal_bound as TB

N, L, HEADS, D, GRID = 4, 64, 2, 40, (8, 8)


def _case(family, flags=7, N=N, L=L, heads=HEADS, d=D, chunks=2, seed=0, grid=GRID):
    return LB.make_case(family, N, L, heads, d, chunks, seed, grid=grid if family == "realistic" else None,
                        use_cf=bool(flags & 1))


# ------------------------------------------------------------------------------------------------ pinned to the reference
def _fixture_control(g, flags, masks=None):
    T = lambda k: torch.from_numpy(np.asarray(g[k]))
    masks = [T(f"attn_mask{i}") for i in range(3)] if masks is None else masks
    return LB.Control(False, False, False, masks, [T("fwd_map")], [T("bwd_map")], [T("inter_mask")]).modes(flags)


@pytest.mark.parametrize("fixture", ["attention", "set_b"])
def test_staged_reference_reproduces_golden_outputs(golden, fixture):
    g = golden(fixture)
    T = lambda k: torch.from_numpy(np.asarray(g[k])).double()
    heads, chunks = int(g["heads"]), 2
    x, rh = T("x"), T("ref_hidden")
    wq, wk, wv, wo, bo = (T(k) for k in ("wq", "wk", "wv", "wo", "bo"))
    ops = LB.Operands(x @ wq.T, x @ wk.T, x @ wv.T, rh @ wq.T, rh @ wk.T, heads, chunks)
    runs = [(f"out_{f}", _fixture_control(g, f)) for f in range(8) if f"out_{f}" in g]
    if "out_cf_nomask" in g:
        runs.append(("out_cf_nomask", _fixture_control(g, 1, [torch.from_numpy(np.asarray(g["attn_mask1"]))])))
    assert len(runs) >= 4
    for key, ctl in runs:
        lay = LB.evaluate(ops, ctl)
        a, _ = LB.attention_result(lay)
        y, _ = LB.out_stage(a, torch.zeros_like(a), wo, bo)
        want = T(key)
        err = (y - want).abs().max().item()
        assert err <= 2e-6 * want.abs().max().item(), (fixture, key, err)


@pytest.mark.parametrize("N_,L_,chunks,masked", [(4, 64, 2, True), (3, 50, 1, True), (1, 64, 2, True), (4, 40, 2, False),
                                                (5, 37, 2, True)])
def test_staged_reference_equals_fresco_oracle(N_, L_, chunks, masked):
    """chunks 1 and 2, N = 1, ragged L, the frame-0 fallback (no mask at this resolution), all eight modes"""
    g = torch.Generator().manual_seed(N_ * 100 + L_)
    C, heads = 80, 2
    B = chunks * N_
    x, rh = torch.randn(B, L_, C, generator=g, dtype=torch.float64), torch.randn(B, L_, C, generator=g, dtype=torch.float64)
    w = [torch.randn(C, C, generator=g, dtype=torch.float64) / math.sqrt(C) for _ in range(4)]
    bo = torch.randn(C, generator=g, dtype=torch.float64)
    mask = torch.rand(N_, L_, generator=g) < 0.4
    mask[0] = True
    masks = [mask if masked else torch.ones(N_, 2 * L_, dtype=torch.bool), torch.ones(N_, 7, dtype=torch.bool)]
    fwd = TB._perms(N_, L_, g)
    tm = TB.reference_mask(N_, L_, g)
    ctl = LB.Control(False, False, False, masks, [fwd[:, None]], [torch.argsort(fwd, 1)[:, None]], [tm[:, None]],
                     intra_bias=0.75)
    ops = LB.Operands(x @ w[0].T, x @ w[1].T, x @ w[2].T, rh @ w[0].T, rh @ w[1].T, heads, chunks)
    for flags in range(8):
        c = ctl.modes(flags)
        want = O.fresco_attention(x, *w, bo, heads, chunks=chunks, use_cfattn=c.use_cf, attn_masks=masks,
                                  use_intraattn=c.use_intra, ref_hidden=rh, intraattn_bias=0.75,
                                  use_interattn=c.use_inter, fwd_mappings=c.fwd_maps, bwd_mappings=c.bwd_maps,
                                  interattn_masks=c.inter_masks)
        a, _ = LB.attention_result(LB.evaluate(ops, c))
        y, _ = LB.out_stage(a, torch.zeros_like(a), w[3], bo)
        # the staged reference rounds the scales to fp32 as the kernels' C ABI does; the oracle keeps them in fp64
        assert (y - want).abs().max().item() <= 1e-6 * want.abs().max().item(), flags


# ------------------------------------------------------------------------------------------------ the product's host glue
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


class PlantedAttn(torch.nn.Module):
    def __init__(self, case, x, rh, dtype):
        super().__init__()
        ops = case.ops
        self.heads = ops.heads
        self.spatial_norm = self.group_norm = None
        self.norm_cross = self.residual_connection = False
        self.rescale_output_factor = 1.0
        self.to_q = Planted([(x, ops.q), (rh, ops.q_ref)])
        self.to_k = Planted([(x, ops.k), (rh, ops.k_ref)])
        self.to_v = Planted([(x, ops.v)])
        C = ops.q.shape[-1]
        self.to_out = torch.nn.ModuleList([torch.nn.Linear(C, C).to(dtype), torch.nn.Dropout(0.0)])


def controller(dh, case, flags, ref_hidden):
    ctl = case.ctl.modes(flags)
    c = dh.AttentionControl()
    c.intraattn_scale_factor, c.intraattn_bias, c.interattn_scale_factor = ctl.intra_scale, ctl.intra_bias, ctl.inter_scale
    if ctl.use_intra:
        c.stored_attn["decoder_attn"] = [ref_hidden]
        c.enable_intraattn()
    if ctl.use_inter:
        c.enable_interattn({"fwd_mappings": ctl.fwd_maps, "bwd_mappings": ctl.bwd_maps, "interattn_masks": ctl.inter_masks})
    if ctl.use_cf:
        c.enable_cfattn(ctl.masks)
    return c


class Fp64Backend:
    """fp64 stand-ins with the semantics of the kernels the layer launches"""

    def kv_compact(self, k, v, idx, chunks):
        B, L_, C = k.shape
        i = idx.long()
        return k.reshape(chunks, -1, C)[:, i].contiguous(), v.reshape(chunks, -1, C)[:, i].contiguous()

    def kv_compact_packed(self, k, v, idx, kv_out, chunks):
        ks, vs = self.kv_compact(k, v, idx, chunks)
        C = k.shape[-1]
        kv_out[:, :ks.shape[1], :C], kv_out[:, :ks.shape[1], C:] = ks, vs
        return kv_out

    def attn_fwd(self, q, k, v, heads, q_per_kv=1, softmax_scale=None, diag_bias=0.0):
        return AB.attention_ref(q, k, v, heads, q_per_kv, softmax_scale, diag_bias)

    def attn_fwd_kv_packed(self, q, kv, heads, q_per_kv, softmax_scale):
        C = q.shape[-1]
        return self.attn_fwd(q, kv[..., :C], kv[..., C:], heads, q_per_kv, softmax_scale)

    def temporal_attn_fwd(self, q, k, v, fwd_map, traj_mask, chunks, heads, scale):
        return TB.ref_and_bound(q, k, v, fwd_map, traj_mask, chunks, heads, scale)[0]


GLUE = [(f, fl) for f in LB.FAMILIES for fl in range(8)]


@pytest.mark.parametrize("path", ["processor", "sharded-world1"])
@pytest.mark.parametrize("family,flags", GLUE, ids=[f"{f}-{fl}" for f, fl in GLUE])
def test_host_glue_equals_staged_reference(monkeypatch, family, flags, path):
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import ops
    from fresco_b200.dist import ShardedFRESCOAttention
    case = _case(family, flags, N=3 if family == "realistic" else N)
    ops_ = case.ops
    B, L_, C = ops_.q.shape
    g = torch.Generator().manual_seed(flags)
    x = torch.randn(B, L_, C, generator=g, dtype=torch.float64)
    rh = torch.randn(B, L_, C, generator=g, dtype=torch.float64)
    be = Fp64Backend()
    lay = LB.evaluate(ops_, case.ctl.modes(flags))
    want = LB.attention_result(lay)[0]
    if path == "processor":
        for name in ("kv_compact", "attn_fwd", "temporal_attn_fwd"):
            monkeypatch.setattr(ops, name, getattr(be, name))
        attn = PlantedAttn(case, x, rh, torch.float64)
        got = {}
        attn.to_out[0].register_forward_pre_hook(lambda m, a: got.setdefault("a", a[0]))
        proc = dh.FRESCOAttnProcessor2_0(ops_.chunks, controller(dh, case, flags, rh))
        with torch.no_grad():
            proc(attn, x.clone())
        a = got["a"]
    else:
        sharded = ShardedFRESCOAttention(controller(dh, case, flags, rh), 1, 0, ops_.chunks, backend=be)
        a = sharded(ops_.q, ops_.k, ops_.v, ops_.heads, ref_q=ops_.q_ref, ref_k=ops_.k_ref)
    assert a.dtype == torch.float64
    err = (a - want).abs().max().item()
    assert err <= 1e-12 * max(1.0, want.abs().max().item()), (family, flags, path, err)


# ------------------------------------------------------------------------------------------------ the composed bound
@pytest.mark.parametrize("family", ["amplify", "realistic", "diag-bias"])
def test_logit_propagation_term_holds_under_adversarial_perturbations(family):
    """|y2(q2 + delta) - y2(q2)| <= (e^(2 Delta) - 1) sum_j w |v - y| for |delta| <= E1, the signs of delta chosen
    along the keys that hold the row (the largest weights), against them, all +, all -, and at random."""
    case = _case(family, flags=2)
    ops, ctl = case.ops, case.ctl.modes(2)                      # spatial-guided on, each frame attends its own K/V
    lay = LB.evaluate(ops, ctl)
    q2, E1 = lay.ref["spatial"], lay.tol["spatial"]
    B, L_, C = q2.shape
    d, heads = C // ops.heads, ops.heads
    inv = 1.0 / math.sqrt(d)
    y = lay.ref["cross"]
    term = LB.logit_propagation(q2, E1, ops.k, ops.v, list(range(B)), heads, inv)
    x, _, kh = AB._logits(q2, ops.k, heads, 1, inv, 0.0)
    top = x.topk(2, -1).indices                                  # [B, H, L, 2]
    signs = []
    for t in range(2):
        kt = torch.gather(kh, 2, top[..., t:t + 1].expand(-1, -1, -1, d).reshape(B, heads, -1, d)).sign()
        kt = kt.transpose(1, 2).reshape(B, L_, C)
        signs += [kt, -kt]
    g = torch.Generator().manual_seed(3)
    signs += [torch.ones_like(q2), -torch.ones_like(q2)] + [torch.randint(0, 2, q2.shape, generator=g).double() * 2 - 1
                                                         for _ in range(4)]
    worst = 0.0
    for s in signs:
        moved = AB.attention_ref(q2 + s * E1, ops.k, ops.v, heads, 1, inv)
        # 1e-12 |y|: the two fp64 evaluations' own rounding, which the term does not cover where it is ~0
        worst = max(worst, ((moved - y).abs() / (term + 1e-12 * y.abs().amax())).max().item())
    assert worst <= 1.0 + 1e-9, worst


@pytest.mark.parametrize("family", LB.FAMILIES)
def test_family_properties(family):
    for flags in (1, 3, 7, 6, 0):
        LB.family_property(_case(family, flags), flags)


@pytest.mark.parametrize("mutant", list(LB.MUTANTS))
def test_mutant_separation(mutant):
    """Each glue mutant moves some element of the layer's attention result on its family by more than twice the
    composed bound: a layer within the bound cannot also be within it of the mutant."""
    family, flags = LB.MUTANTS[mutant]
    case = _case(family, flags)
    ctl = case.ctl.modes(flags)
    ref, tol = LB.attention_result(LB.evaluate(case.ops, ctl))
    mut, _ = LB.attention_result(LB.evaluate(case.ops, ctl, mutant=mutant))
    sep = ((mut - ref).abs() / tol).max().item()
    assert sep > 2.0, f"{mutant} on {family}: at most {sep:.3g} x the bound from the layer"


# ------------------------------------------------------------------------------------------------ keyframe batch after batch
BATCHES = [("realistic", 3), ("temporal-dominant", 4), ("exact", 5), ("temporal-dominant", 6)]


def stale(ctl, before, kind):
    """``ctl`` with the masks ("kv-indices") or the mappings ("trajectories") of the batch before: what a layer whose
    cache survived the new batch computes"""
    if kind == "kv-indices":
        return ctl._replace(masks=before.masks)
    return ctl._replace(fwd_maps=before.fwd_maps, bwd_maps=before.bwd_maps, inter_masks=before.inter_masks)


@pytest.mark.parametrize("kind", ["kv-indices", "trajectories"])
def test_stale_cache_mutant_separation(kind):
    """Between every two consecutive batches of ``BATCHES`` (equal token counts, so a cache keyed by the token count
    would be hit), a layer that kept the previous batch's K/V indices or trajectories differs from the new batch's
    layer by more than twice the composed bound."""
    cases = [_case(f, seed=s) for f, s in BATCHES]
    for before, case in zip(cases, cases[1:]):
        ctl = case.ctl.modes(7)
        ref, tol = LB.attention_result(LB.evaluate(case.ops, ctl))
        mut, _ = LB.attention_result(LB.evaluate(case.ops, stale(ctl, before.ctl, kind)))
        sep = ((mut - ref).abs() / tol).max().item()
        assert sep > 2.0, f"stale {kind} from {before.family} into {case.family}: {sep:.3g} x the bound"


@pytest.mark.parametrize("path", ["processor", "sharded-world1"])
def test_host_glue_follows_each_keyframe_batch(monkeypatch, path):
    """One processor / sharded layer and one controller over the batches of ``BATCHES`` (new masks and mappings each
    time, as enable_cfattn / enable_interattn receive them): every batch equals its own staged reference."""
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import ops
    from fresco_b200.dist import ShardedFRESCOAttention
    be = Fp64Backend()
    for name in ("kv_compact", "attn_fwd", "temporal_attn_fwd"):
        monkeypatch.setattr(ops, name, getattr(be, name))
    ctrl = dh.AttentionControl()
    layer = dh.FRESCOAttnProcessor2_0(2, ctrl) if path == "processor" else ShardedFRESCOAttention(ctrl, 1, 0, 2, backend=be)
    for i, (family, seed) in enumerate(BATCHES):
        case = _case(family, seed=seed)
        ctl = case.ctl.modes(7)
        g = torch.Generator().manual_seed(i)
        x, rh = (torch.randn(case.ops.q.shape, generator=g, dtype=torch.float64) for _ in range(2))
        ctrl.intraattn_scale_factor, ctrl.intraattn_bias, ctrl.interattn_scale_factor = \
            ctl.intra_scale, ctl.intra_bias, ctl.inter_scale
        ctrl.stored_attn["decoder_attn"] = [rh]
        ctrl.enable_controller(interattn_paras={"fwd_mappings": ctl.fwd_maps, "bwd_mappings": ctl.bwd_maps,
                                                "interattn_masks": ctl.inter_masks}, attn_mask=ctl.masks)
        if path == "processor":
            attn, got = PlantedAttn(case, x, rh, torch.float64), {}
            attn.to_out[0].register_forward_pre_hook(lambda m, a: got.setdefault("a", a[0]))
            with torch.no_grad():
                layer(attn, x.clone())
            a = got["a"]
        else:
            o = case.ops
            a = layer(o.q, o.k, o.v, o.heads, ref_q=o.q_ref, ref_k=o.k_ref)
        want = LB.attention_result(LB.evaluate(case.ops, ctl))[0]
        assert (a - want).abs().max().item() <= 1e-12 * max(1.0, want.abs().max().item()), (path, family, seed)
