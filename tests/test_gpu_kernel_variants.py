"""Every kernel instantiation the launchers can select, at the shapes that select it, against fp64 references.

The launchers in hbm_kernels.cu, gemm_wgmma.cu, gram_wgmma.cu and attn_wgmma.cu pick a template instantiation from
the frame count, the head dim, the plane size measured against shared memory, the channel divisibility, the SM count,
whether the input rows are strided, and the tuning options.  The file is one table, ``ROWS``: an entry point, a shape,
the options, and the kernels the call must launch, in order, as ``fresco_last_kernel()`` names them.  Each row

* fills every output with NaN (or a NaN bit pattern) first, so a row or tile the kernel never writes is caught,
* runs the entry point through the C ABI and asserts the instantiation it launched -- a change to a selection rule
  fails here instead of quietly moving a row to another kernel,
* compares the output with a plain fp64 reference of the same operation, evaluated on the operands the kernel consumes
  (fp16-rounded where the kernel reads fp16).  The temporal-consistency loss rows are held elementwise to
  ``oracle.warp_loss_bound`` (``tests/test_gpu_warp_loss.py`` runs its input families on every loss kernel), the
  temporal attention rows to ``oracle.temporal_bound`` (``tests/test_gpu_temporal_attention.py``), the warp-chain rows
  to ``oracle.warp_chain_bound`` (``tests/test_gpu_warp_chain.py``).

Instantiations no row reaches are listed with the reason in ``NOT_LAST`` (launched, but another kernel of the same
call is what the record shows) or ``COVERED_ELSEWHERE`` (one instantiation per dtype, no selection; the named test
checks it).  ``test_launch_name_universe`` derives the instantiation lists from the launcher sources and checks that
every name is in exactly one of those places.
"""
import collections
import functools
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

from oracle import attention_bound as AB
from oracle import fresco_oracle as O
from oracle import gmflow_bound as GB
from oracle import gram_bound as GRB
from oracle import temporal_bound as TB
from oracle import warp_chain_bound as CB
from oracle import warp_loss_bound as WB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "fresco_b200", "csrc")


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib, ops
    _lib.lib()      # fails loudly if the extension is missing
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

    class NS:
        pass
    ns = NS()
    ns.lib, ns.ops, ns.c = _lib, ops, _lib.lib()
    return ns


def P(t):
    return t.data_ptr()


class Launches:
    """Checks each launch of a row against the table as it happens."""

    def __init__(self, fb, row):
        self.fb, self.row, self.i = fb, row, 0

    def __call__(self, what, rc=0):
        self.fb.lib.check(rc, what)
        name = self.fb.lib.last_kernel()
        assert self.i < len(self.row.kernels), f"{what}: unexpected launch of {name}"
        want = self.row.kernels[self.i]
        self.i += 1
        assert name == want, f"{what} launched {name}; the table expects {want}"
        SEEN.add(name)


Row = collections.namedtuple("Row", "id kernels run opts")
ROWS = []
SEEN = set()
RAN = set()


def row(id_, kernels, fn, opts=None, **kw):
    ROWS.append(Row(id_, tuple(kernels), functools.partial(fn, **kw), dict(opts or {})))


def _nan(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _check_close(out, ref, bound, what):
    """max |out - ref| <= bound over every element; NaN left in ``out`` (never written) fails."""
    out = out.double()
    unwritten = (~torch.isfinite(out)).sum().item()
    assert unwritten == 0, f"{what}: {unwritten} outputs not written (NaN) or not finite"
    err = (out - ref).abs().max().item()
    assert err <= bound, f"{what}: max error {err:.3g} > {bound:.3g}"


def _worst_tile(ratio, rows=128, cols=256):
    """Where err / tol is largest, by rows x cols output tile (ratio [R, C]; NaN counts as infinitely wrong)."""
    ratio = torch.nan_to_num(ratio.double(), nan=float("inf"))
    R, C = ratio.shape
    t = F.pad(ratio, (0, (-C) % cols, 0, (-R) % rows)).view((R + rows - 1) // rows, rows, (C + cols - 1) // cols, cols)
    t = t.amax((1, 3))
    i, j = divmod(int(t.argmax().item()), t.shape[1])
    return (f"worst {rows}x{cols} tile rows [{i * rows}, {(i + 1) * rows}) cols [{j * cols}, {(j + 1) * cols}): "
            f"max err/tol {t[i, j].item():.3g}; {(t > 1).sum().item()} of {t.numel()} tiles fail")


# ================================================================================================ temporal attention
def _trajectories(N, L, seed):
    """Random per-frame permutations and masks with the reference's structure (cuts between frames <= i and > i,
    flow_utils.py:126-133), plus 5 % of trajectories where a frame may only attend to itself."""
    g = torch.Generator().manual_seed(seed)
    fwd = torch.stack([torch.arange(L)] + [torch.randperm(L, generator=g) for _ in range(N - 1)])
    mask = torch.ones(L, N, N, dtype=torch.bool)
    for i in range(N - 1):
        cut = torch.ones(N, N, dtype=torch.bool)
        cut[:i + 1, i + 1:] = False
        cut[i + 1:, :i + 1] = False
        sel = torch.rand(L, generator=g) < 0.15
        mask[sel] = mask[sel] & cut
    mask[torch.rand(L, generator=g) < 0.05] = torch.eye(N, dtype=torch.bool)
    return fwd, mask


def _temporal(fb, launch, N, L, heads, d, packed=False, chunks=2, seed=0, kernel="rows"):
    """packed=False: fresco_temporal_attn_fwd on dense [chunks*N, L, C] tensors.  packed=True: the call
    ShardedTrajectoryExchange.run makes -- qkv [N, chunks*L, 3C] with q | k | v in every row, identity map, chunks=1,
    mask [chunks*L, N, N] (L = this rank's trajectories).  Every element within oracle.temporal_bound for ``kernel``
    (rows: temporal_attn_rows_kernel, round1: temporal_attn_kernel); tests/test_gpu_temporal_attention.py runs the
    bound's input families on both kernels."""
    C, scale = heads * d, 1.0 / math.sqrt(d)
    g = torch.Generator(device="cuda").manual_seed(seed)
    fwd, mask = _trajectories(N, L, seed)
    if packed:
        tokens = chunks * L
        qkv = torch.randn(N, tokens, 3 * C, device="cuda", generator=g)
        qkv[..., C:2 * C] *= 2.0
        qkv = qkv.half()
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
        pq, pk, pv = P(qkv), P(qkv) + 2 * C, P(qkv) + 4 * C
        fwd = torch.arange(tokens)[None].expand(N, -1).contiguous()
        mask = mask[None].expand(chunks, -1, -1, -1).reshape(tokens, N, N)
        kchunks, stride = 1, 3 * C
    else:
        tokens = L
        q = torch.randn(chunks * N, L, C, device="cuda", generator=g).half()
        k = (torch.randn(chunks * N, L, C, device="cuda", generator=g) * 2.0).half()
        v = torch.randn(chunks * N, L, C, device="cuda", generator=g).half()
        pq, pk, pv = P(q), P(k), P(v)
        kchunks, stride = chunks, C
    fwd_d, mask_d = fwd.cuda().contiguous(), mask.to(torch.uint8).cuda().contiguous()
    out = _nan((kchunks * N, tokens, C), torch.float16)
    launch("fresco_temporal_attn_fwd_strided",
           fb.c.fresco_temporal_attn_fwd_strided(pq, pk, pv, P(out), P(fwd_d), P(mask_d), kchunks, N, tokens, heads, d,
                                                 stride, scale, fb.lib.stream()))
    ref, tol = TB.ref_and_bound(q, k, v, fwd_d, mask_d, kchunks, heads, scale, kernel)
    ratio = TB.ratio(out, ref, tol)
    assert not (ratio > 1).any(), "temporal attention: " + _worst_tile(ratio.reshape(-1, C))


for _N, _d, _L in [(9, 40, 4096), (12, 40, 4096), (16, 40, 4096), (9, 80, 1024), (12, 80, 1024), (16, 80, 1024)]:
    # N = 16, 8 heads: 128 rows per trajectory, so at most 2 trajectories per CTA.  Each takes 2 * N * 2C bytes of
    # shared memory (+ 4 N): 20 KB at d = 40, so 2 per CTA; 40 KB at d = 80, where 2 would exceed the 48 KB the
    # launcher keeps a CTA under, so 1
    row(f"temporal-N{_N}-d{_d}", [f"temporal_attn_rows_kernel<{_d},16>"], _temporal, N=_N, L=_L, heads=8, d=_d)
row("temporal-N8-d40", ["temporal_attn_rows_kernel<40,8>"], _temporal, N=8, L=4096, heads=8, d=40)
row("temporal-N4-d80", ["temporal_attn_rows_kernel<80,8>"], _temporal, N=4, L=1024, heads=8, d=80)
row("temporal-N5-d64", ["temporal_attn_rows_kernel<64,8>"], _temporal, N=5, L=500, heads=4, d=64)
row("temporal-N13-d64", ["temporal_attn_rows_kernel<64,16>"], _temporal, N=13, L=500, heads=4, d=64)
row("temporal-packed-N16-d40", ["temporal_attn_rows_kernel<40,16>"], _temporal, N=16, L=4096 // 2, heads=8, d=40,
    packed=True)
row("temporal-packed-N16-d80", ["temporal_attn_rows_kernel<80,16>"], _temporal, N=16, L=1024 // 2, heads=8, d=80,
    packed=True)
row("temporal-packed-N5-d64", ["temporal_attn_rows_kernel<64,8>"], _temporal, N=5, L=300, heads=4, d=64, packed=True)
row("temporal-round1-N17-d40", ["temporal_attn_kernel"], _temporal, N=17, L=1024, heads=8, d=40, kernel="round1")
row("temporal-round1-N24-d80", ["temporal_attn_kernel"], _temporal, N=24, L=512, heads=8, d=80, kernel="round1")
row("temporal-round1-N4-d128", ["temporal_attn_kernel"], _temporal, N=4, L=300, heads=2, d=128, kernel="round1")
row("temporal-V1-N8-d40", ["temporal_attn_kernel"], _temporal, opts={"FRESCO_TEMPORAL_V": 1}, N=8, L=4096, heads=8,
    d=40, kernel="round1")


# ================================================================================================ cross-frame attention
def attn_name(d, wide, poly, rowsum):
    keys = 64 if wide == 0 else 128
    wg = 3 if wide == 2 and d <= 64 else 2
    return "fresco_attn_kernel<%d,keys%d,wg%d,poly%d%s>" % (d, keys, wg, poly, ",rowsum" if wide == 0 and rowsum else "")


def _attn(fb, launch, d, qpk, Lq, Lk, heads=8, chunks=2, pad=0, gain=4.0, seed=0, poly=0, rowsum=0):
    """fresco_attn_fwd_kv_strided as attn_fwd_kv_packed calls it: K | V side by side in one [chunks, Lk, 2C] buffer,
    q_per_kv query frames per K/V batch.  pad > 0: batches (Lk + pad) rows apart, the pad rows NaN (a padded exchange
    buffer); they must not reach the output.  Checked elementwise against oracle.attention_bound."""
    C, scale = heads * d, 1.0 / math.sqrt(d)
    g = torch.Generator(device="cuda").manual_seed(seed + d + qpk)
    q = (torch.randn(chunks * qpk, Lq, C, device="cuda", generator=g) * gain).half()
    kv = torch.randn(chunks, Lk + pad, 2 * C, device="cuda", generator=g).half()
    kv[:, Lk:] = float("nan")
    out = _nan(q.shape, torch.float16)
    launch("fresco_attn_fwd_kv_strided",
           fb.c.fresco_attn_fwd_kv_strided(P(q), P(kv), P(kv) + 2 * C, P(out), chunks * qpk, Lq, Lk, heads, d, qpk, 2 * C,
                                           (Lk + pad) * 2 * C, scale, 0.0, fb.lib.stream()))
    assert fb.c.fresco_attn_variant(d).decode() == fb.lib.last_kernel() + " (wgmma)"
    ref, tol = AB.ref_and_bound(q, kv[:, :Lk, :C], kv[:, :Lk, C:], heads, qpk, scale, 0.0, poly, bool(rowsum))
    ratio = (out.double() - ref).abs() / tol
    assert not (ratio > 1).any() and torch.isfinite(out).all(), "attention: " + _worst_tile(ratio.flatten(0, 1))


for _d in (40, 80):
    for _qpk in (2, 4, 8, 16):          # frame-sharded G = 8 / 4 / 2 (N_local query frames per K/V batch), unsharded N = 16
        for _wide in (1, 0):
            row(f"attn-kv-packed-d{_d}-qpk{_qpk}-wide{_wide}", [attn_name(_d, _wide, 0, 0)], _attn,
                opts={"FRESCO_ATTN_WIDE": _wide}, d=_d, qpk=_qpk, Lq=1000, Lk=150 * _qpk + 37)
    for _wide in (1, 0):
        row(f"attn-kv-padded-d{_d}-wide{_wide}", [attn_name(_d, _wide, 0, 0)], _attn, opts={"FRESCO_ATTN_WIDE": _wide},
            d=_d, qpk=4, Lq=700, Lk=613, pad=91)
# every variant the options select, at every head dim (three consumer warpgroups stop at head dim 64)
for _d in (40, 64, 80, 128):
    for _wide in ((0, 1, 2) if _d <= 64 else (0, 1)):
        for _poly in (0, 4, 8):
            for _rowsum in ((0, 1) if _wide == 0 else (0,)):
                row(f"attn-variant-d{_d}-wide{_wide}-poly{_poly}-rowsum{_rowsum}", [attn_name(_d, _wide, _poly, _rowsum)],
                    _attn, opts={"FRESCO_ATTN_WIDE": _wide, "FRESCO_ATTN_POLY": _poly, "FRESCO_ATTN_ROWSUM": _rowsum},
                    d=_d, qpk=2, Lq=300, Lk=1000, heads=2, poly=_poly, rowsum=_rowsum)


# ================================================================================================ data movement
def _bits(t):
    return t.view(torch.int16)


def _kv_compact_packed(fb, launch, chunks=2, N=4, tokens=500, C=320, extra=13):
    g = torch.Generator(device="cuda").manual_seed(1)
    k = torch.randn(chunks * N, tokens, C, device="cuda", generator=g).half()
    v = torch.randn(chunks * N, tokens, C, device="cuda", generator=g).half()
    idx = torch.nonzero(torch.rand(N * tokens, device="cuda", generator=g) < 0.4).reshape(-1).to(torch.int32)
    n_sel = idx.numel()
    kv = _nan((chunks, n_sel + extra, 2 * C), torch.float16)
    launch("fresco_kv_compact_packed", fb.c.fresco_kv_compact_packed(P(k), P(v), P(idx), P(kv), chunks, N * tokens, n_sel,
                                                                     n_sel + extra, C, fb.lib.stream()))
    li = idx.long()
    assert torch.equal(_bits(kv[:, :n_sel, :C]), _bits(k.reshape(chunks, N * tokens, C)[:, li]))
    assert torch.equal(_bits(kv[:, :n_sel, C:]), _bits(v.reshape(chunks, N * tokens, C)[:, li]))
    assert torch.equal(_bits(kv[:, n_sel:]), _bits(_nan((chunks, extra, 2 * C), torch.float16))), "rows past n_sel written"


def _rows_gather(fb, launch, col, R=3000, n=2500, C=320):
    g = torch.Generator(device="cuda").manual_seed(2 + col)
    src = torch.randn(R, C, device="cuda", generator=g).half()
    idx = torch.randint(0, R, (n,), device="cuda", generator=g, dtype=torch.int32)
    dst = _nan((n, 3 * C), torch.float16)
    launch("fresco_rows_gather", fb.c.fresco_rows_gather(P(src), P(idx), P(dst), n, C * 2, 3 * C * 2, col * C * 2,
                                                         fb.lib.stream()))
    want = _nan((n, 3 * C), torch.float16)
    want[:, col * C:(col + 1) * C] = src[idx.long()]
    assert torch.equal(_bits(dst), _bits(want))


def _rows_scatter(fb, launch, R=3000, n=2500, C=320):
    g = torch.Generator(device="cuda").manual_seed(3)
    src = torch.randn(n, C, device="cuda", generator=g).half()
    idx = torch.randperm(R, device="cuda", generator=g)[:n].to(torch.int32)
    dst = _nan((R, C), torch.float16)
    launch("fresco_rows_scatter", fb.c.fresco_rows_scatter(P(src), P(idx), P(dst), n, C * 2, fb.lib.stream()))
    want = _nan((R, C), torch.float16)
    want[idx.long()] = src
    assert torch.equal(_bits(dst), _bits(want))


row("kv-compact-packed-padded", ["kv_compact_packed_kernel"], _kv_compact_packed)
for _col in (0, 1, 2):
    row(f"rows-gather-col{_col}C", ["rows_gather_kernel"], _rows_gather, col=_col)
row("rows-scatter", ["rows_scatter_kernel"], _rows_scatter)


# ================================================================================================ temporal-consistency loss
def _loss_case(N, C, h, res, seed, chunks=2):
    flows, occs = O.synth_flows(N, res, res, seed=seed, mag=12.0)
    ff, bf, fo, bo = O._resize_flow_occ(flows, occs, h / res)
    assert ff.shape[-1] == h
    g = torch.Generator(device="cuda").manual_seed(seed + 50)
    base = torch.randn(chunks, 1, C, h, h, device="cuda", generator=g)
    cs = (base + 0.5 * torch.randn(chunks, N, C, h, h, device="cuda", generator=g)).contiguous()   # correlated frames
    return cs, ff.cuda().contiguous(), bf.cuda().contiguous(), (1 - fo).cuda(), (1 - bo).cuda()


def _warp_loss(fb, launch, N, C, h, res, seed=0):
    """fresco_warp_loss_fwd_bwd_halo (closed ring) on smooth flows: the loss and every gradient element within
    oracle.warp_loss_bound of the fp64 reference."""
    cs, ff, bf, kf, kb = _loss_case(N, C, h, res, seed=seed + h + C)
    kf, kb = kf.reshape(N, h, h).contiguous(), kb.reshape(N, h, h).contiguous()
    adj = fb.ops.warp_adjoint_pair(bf, ff)
    grad = torch.full_like(cs, float("nan"))
    loss = torch.zeros(1, device="cuda")
    fb.ops.warp_loss_fwd_bwd(cs, ff, bf, kf, kb, grad, loss, adjoint=adj)
    launch("fresco_warp_loss_fwd_bwd_halo")
    ref = WB.reference_and_bound(cs, ff, bf, kf, kb)
    assert ref["in_band"] < 0.01, ref["in_band"]
    assert abs(loss.item() - ref["loss"]) <= ref["loss_tol"], (loss.item(), ref["loss"], ref["loss_tol"])
    ratio = WB.ratio(grad, ref["grad"], ref["grad_tol"])
    assert not (ratio > 1).any(), "temporal loss: " + _worst_tile(ratio.reshape(-1, h * h))


# the quad kernel: 4 NQ channel planes per CTA (channels % (4 NQ) == 0, NQ > 1 only with a grid of >= one CTA per SM)
row("loss-quad-16x1280x32x32", ["warp_loss_quad_kernel<1,4>"], _warp_loss, N=8, C=1280, h=32, res=512)
row("loss-quad-16x1280x12x12", ["warp_loss_quad_kernel<1,4>"], _warp_loss, N=8, C=1280, h=12, res=768)
row("loss-quad-16x1280x24x24", ["warp_loss_quad_kernel<1,4>"], _warp_loss, N=8, C=1280, h=24, res=768)
row("loss-quad-16x640x32x32", ["warp_loss_quad_kernel<2,2>"], _warp_loss, N=8, C=640, h=32, res=512)
row("loss-quad-16x640x40x40", ["warp_loss_quad_kernel<2,2>"], _warp_loss, N=8, C=640, h=40, res=320)
row("loss-quad-16x640x64x64", ["warp_loss_quad_kernel<4,1>"], _warp_loss, N=8, C=640, h=64, res=512)
row("loss-quad-16x1280x48x48", ["warp_loss_quad_kernel<4,1>"], _warp_loss, N=8, C=1280, h=48, res=768)
# the channel-grouped kernel: P = ceil(hw / 512) pixels x KT planes per thread; KT > 1 only with >= 296 CTAs.
# Channel counts that are not multiples of 4 keep the quad kernel out.
for _h, _P in ((16, 1), (32, 2), (36, 3), (40, 4)):
    for _C, _KT in ((1190 if _h == 16 else 650, 4), (650 if _h == 16 else 450, 2), (6, 1)):
        row(f"loss-group-P{_P}-KT{_KT}-6x{_C}x{_h}x{_h}", [f"warp_loss_group_kernel<{_P},{_KT}>"], _warp_loss, N=3, C=_C,
            h=_h, res=8 * _h)
for _h, _P in ((48, 5), (64, 8)):
    for _C, _KT in ((450, 2), (6, 1)):
        row(f"loss-group-P{_P}-KT{_KT}-6x{_C}x{_h}x{_h}", [f"warp_loss_group_kernel<{_P},{_KT}>"], _warp_loss, N=3, C=_C,
            h=_h, res=8 * _h)
row("loss-group-16x640x96x96", ["warp_loss_group_kernel<18,1>"], _warp_loss, N=8, C=640, h=96, res=768)
# one CTA per plane: plane sizes no group instantiation takes (P = 7, P = 20)
row("loss-one-cta-6x6x56x56", ["warp_loss_kernel"], _warp_loss, N=3, C=6, h=56, res=448)
row("loss-one-cta-6x4x100x100", ["warp_loss_kernel"], _warp_loss, N=3, C=4, h=100, res=800)


# ================================================================================================ warp chain
def _chain(fb, launch, chunks, N, C, h, w, dtype, seed=0):
    """fresco_warp_fuse_chain on smooth non-dyadic flows (x + flow rounds in fp32, so the coordinate path real flows
    take is exercised), fractional blend weights and values of 1e-3 and 1e3 in one plane: every element within oracle.warp_chain_bound of the fp64 chain;
    tests/test_gpu_warp_chain.py runs the bound's input families on every chain kernel."""
    d = CB.family("magnitudes", chunks, N, C, h, w, dtype=dtype, seed=seed + C + h, device="cuda")      # 1e-3 and 1e3
    sample = d["sample"]
    out = torch.full_like(sample, float("nan"))
    fb.ops.warp_fuse_chain(sample, d["bwd"], d["fwd_last"], d["blend"], chunks, out=out)
    launch("fresco_warp_fuse_chain")
    ref, tol = CB.chain_reference_and_bound(sample, d["bwd"], d["fwd_last"], d["blend"], chunks)
    ratio = CB.ratio(out, ref, tol)
    assert not (ratio > 1).any(), "warp chain: " + _worst_tile(ratio.reshape(-1, h * w))


def _chain_rejects_fp16_image_planes(fb, launch):
    """Planes over 100 KB run the per-step kernel, which is fp32 only: fp16 is refused, not silently converted."""
    x = torch.zeros(2 * 3, 3, 176, 176, device="cuda", dtype=torch.float16)
    flow = torch.zeros(3, 2, 176, 176, device="cuda")
    with pytest.raises(fb.lib.FrescoError, match="need float"):
        fb.ops.warp_fuse_chain(x, flow, flow[0].contiguous(), torch.zeros(3, 176, 176, device="cuda"), 2)


for _dt, _tn in ((torch.float32, "float"), (torch.float16, "half")):
    for _h in (32, 16, 8):          # decoder features [16,1280,{8,16,32}^2]
        row(f"chain-quad-{_tn}-16x1280x{_h}x{_h}", [f"warp_chain_quad_kernel<{_tn},1,4>"], _chain, chunks=2, N=8, C=1280,
            h=_h, w=_h, dtype=_dt)
    row(f"chain-quad-{_tn}-16x640x32x32", [f"warp_chain_quad_kernel<{_tn},2,2>"], _chain, chunks=2, N=8, C=640, h=32,
        w=32, dtype=_dt)
    row(f"chain-quad-{_tn}-16x640x64x64", [f"warp_chain_quad_kernel<{_tn},4,1>"], _chain, chunks=2, N=8, C=640, h=64,
        w=64, dtype=_dt)
    # decoder shapes whose quad configuration, P * NQ = 4 float4 per thread, would need more than 1024 threads: (2,4)
    # at 40x40, (4,2) at 48x48.  No quad kernel takes them; the channel-grouped kernel does.
    row(f"chain-group8-{_tn}-16x1280x40x40", [f"warp_chain_group_kernel<{_tn},8>"], _chain, chunks=2, N=8, C=1280,
        h=40, w=40, dtype=_dt)
    row(f"chain-group3-{_tn}-16x1280x48x48", [f"warp_chain_group_kernel<{_tn},3>"], _chain, chunks=2, N=8, C=1280,
        h=48, w=48, dtype=_dt)
    row(f"chain-group8-{_tn}-6x1190x16x16", [f"warp_chain_group_kernel<{_tn},8>"], _chain, chunks=2, N=3, C=1190, h=16,
        w=16, dtype=_dt)
    row(f"chain-group3-{_tn}-6x450x32x32", [f"warp_chain_group_kernel<{_tn},3>"], _chain, chunks=2, N=3, C=450, h=32,
        w=32, dtype=_dt)
    row(f"chain-group1-{_tn}-6x6x32x24", [f"warp_chain_group_kernel<{_tn},1>"], _chain, chunks=2, N=3, C=6, h=32, w=24,
        dtype=_dt)
row("chain-per-step-float-6x3x176x192", ["warp_blend_step_kernel"], _chain, chunks=2, N=3, C=3, h=176, w=192,
    dtype=torch.float32)
row("chain-per-step-half-rejected", [], _chain_rejects_fp16_image_planes)


# ================================================================================================ GMFlow flow attention
def _gmflow_flow_attention(fb, launch, B=16, L=4096, C=128, seed=0):
    """GMFlow's flow propagation at 512 x 512: 64 x 64 tokens, V a flow field of tens of pixels; elementwise within
    oracle.gmflow_bound."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = (torch.randn(B, L, C, device="cuda", generator=g) * 2.0).half()
    k = torch.randn(B, L, C, device="cuda", generator=g).half()
    vals = torch.randn(B, L, 2, device="cuda", generator=g) * 20.0
    out = _nan((B, 2, L), torch.float32)
    scale = 1.0 / math.sqrt(C)
    launch("gmflow_flow_attention", fb.c.gmflow_flow_attention(P(q), P(k), P(vals), P(out), B, L, C, scale, fb.lib.stream()))
    ref, tol = GB.flow_attn_ref_and_bound(q, k, vals, scale)
    ratio = (out.double() - ref).abs() / tol
    assert not (ratio > 1).any() and torch.isfinite(out).all(), "flow attention: " + _worst_tile(ratio.flatten(0, 1))


row("gmflow-flow-attention-16x4096x128", ["tile_gemm_kernel<EPI_GMFLOW,0>"], _gmflow_flow_attention)


# ================================================================================================ Gram loss
def _gram(fb, launch, B, C, h, w, dense=False, weight=100.0, seed=0):
    """The spatial-consistency loss at a layer shape, operand-exact and elementwise within ``oracle.gram_bound``
    (``tests/test_gpu_gram.py`` runs its input families): every fp64 reference is computed from the kernels' own fp16
    xhat / yhat / tsign, one batch at a time on the GPU."""
    L = h * w
    g = torch.Generator(device="cuda").manual_seed(seed + C + L)
    base = torch.randn(B, C, 1, device="cuda", generator=g)
    cs = (base + torch.randn(B, C, L, device="cuda", generator=g)).contiguous()
    cs_ref = (base + torch.randn(B, C, L, device="cuda", generator=g)).contiguous()     # same statistics: D changes sign
    st = fb.lib.stream()
    # ---- row normalisation: xhat = fp16(x / |x|) token-major, norms fp32
    normed = []
    for src in (cs, cs_ref):
        xhat, norms = _nan((B, L, C), torch.float16), _nan((B, L), torch.float32)
        launch("fresco_gram_normalize", fb.c.fresco_gram_normalize(P(src), P(xhat), P(norms), B, C, L, st))
        GRB.check_normalize(src, xhat, norms)
        normed.append((xhat, norms))
    (xhat, norms), (yhat, _) = normed
    scale = weight / (B * L * L)

    class Out:
        pass
    run = Out()
    run.t1_buf, run.td_buf = True, None
    # ---- sign matrix with the recomputed target: D = X X^T - Y Y^T in one K = 2C contraction
    run.tsign = _nan((B, L, L), torch.float16)
    run.loss = torch.zeros(1, device="cuda")
    launch("fresco_gram_sign_ref", fb.c.fresco_gram_sign_ref(P(xhat), P(yhat), P(run.tsign), P(run.loss), B, L, C,
                                                             weight, st))
    # ---- ghat = alpha T X (tensor-core product of the backward), from the kernel's own T
    run.ghat = _nan((B, L, C), torch.float32)
    launch("fresco_gram_tx", fb.c.fresco_gram_tx(P(run.tsign), P(xhat), P(run.ghat), B, L, C, scale, st))
    # ---- grad += projection of ghat through the normalisation Jacobian, under both products fresco_gram_grad can use
    grad0 = torch.zeros(B, C, L, device="cuda")
    nbytes = int(fb.c.fresco_gram_grad_workspace_bytes(B, L, C))
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    run.grads = {}
    for v in (2, 1):
        fb.lib.set_option("FRESCO_GRAM_V", v)
        gr = grad0.clone()
        launch(f"fresco_gram_grad (FRESCO_GRAM_V={v})",
               fb.c.fresco_gram_grad(P(run.tsign), P(xhat), P(norms), P(gr), B, L, C, weight, P(ws), nbytes, st))
        run.grads[v] = gr
    fb.lib.set_option("FRESCO_GRAM_V", -1)
    A = None
    if dense:
        # the dense-target entry point (a caller holding the reference's fp32 correlation matrix): T = sign(G - A) +
        # sign(G - A^T), loss over |G - A|
        A = torch.empty(B, L, L, device="cuda")
        for b in range(B):
            A[b] = (xhat[b].double() @ xhat[b].double().T + 0.05 * torch.randn(L, L, device="cuda", generator=g,
                                                                               dtype=torch.float64)).float()
        run.td_buf, run.tsign_d = True, _nan((B, L, L), torch.float16)
        run.loss_d = torch.zeros(1, device="cuda")
        launch("fresco_gram_sign", fb.c.fresco_gram_sign(P(xhat), P(A), P(run.tsign_d), P(run.loss_d), B, L, C, weight,
                                                         st))
    torch.cuda.synchronize()
    GRB.check_run(run, xhat, yhat, norms, A, grad0, scale, torch.cuda.get_device_properties(0).multi_processor_count)


_GRAM_KERNELS = ["gram_normalize_kernel", "gram_normalize_kernel", "gram2_kernel<G2_SIGN>", "gram2_kernel<G2_GRAD>",
                 "gram_project_kernel", "gram_project_kernel"]
row("gram-16x640x64x64", _GRAM_KERNELS, _gram, opts={"FRESCO_GRAM_V": -1}, B=16, C=640, h=64, w=64)
row("gram-16x1280x32x32", _GRAM_KERNELS + ["tile_gemm_kernel<EPI_GRAM_SIGN,0>"], _gram, opts={"FRESCO_GRAM_V": -1}, B=16, C=1280, h=32, w=32,
    dense=True)
row("gram-16x640x96x96", _GRAM_KERNELS, _gram, opts={"FRESCO_GRAM_V": -1}, B=16, C=640, h=96, w=96)
row("gram-4x16x24x24", _GRAM_KERNELS + ["tile_gemm_kernel<EPI_GRAM_SIGN,0>"], _gram, opts={"FRESCO_GRAM_V": -1}, B=4, C=16, h=24, w=24, dense=True)


# ================================================================================================ what no row reaches
NOT_LAST = {
    "tile_gemm_kernel<EPI_STORE,1>": "fresco_gram_grad under FRESCO_GRAM_V=1 launches it before gram_project_kernel; the "
                                     "gram rows check the gradient it feeds elementwise under that option",
}
COVERED_ELSEWHERE = {
    "kv_compact_kernel": "test_gpu_kernels.py::test_kv_compact_bit_exact",
    "flow_warp_kernel": "test_gpu_warp_chain.py::test_flow_warp (within oracle.warp_chain_bound; also "
                        "test_gpu_kernels.py::test_flow_warp_and_consistency)",
    "warp_taps_kernel": "test_gpu_warp_loss.py::test_warp_taps_bit_exact (and it builds the adjoint of every "
                        "temporal-loss row here)",
    "adam_kernel": "test_gpu_step_kernels.py::test_adam_family (within oracle.step_bound; also test_adam_layer3_size)",
    "adain_kernel<half>": "test_gpu_step_kernels.py::test_adain_family (within oracle.step_bound; also "
                          "test_adain_decoder_layers)",
    "adain_kernel<float>": "test_gpu_step_kernels.py::test_adain_family (within oracle.step_bound; also "
                           "test_adain_decoder_layers)",
    "cfg_pred_x0_kernel<half>": "test_gpu_step_kernels.py::test_cfg_and_ddpm_family (within oracle.step_bound)",
    "cfg_pred_x0_kernel<float>": "test_gpu_step_kernels.py::test_cfg_and_ddpm_family (within oracle.step_bound)",
    "ddpm_prev_kernel<half>": "test_gpu_step_kernels.py::test_cfg_and_ddpm_family (within oracle.step_bound)",
    "ddpm_prev_kernel<float>": "test_gpu_step_kernels.py::test_cfg_and_ddpm_family (within oracle.step_bound)",
    "dilate_kernel": "test_gpu_step_kernels.py::test_dilate_family (within oracle.step_bound; binary and dyadic "
                     "bit-exact)",
    "to_token_major_f16_kernel": "test_gpu_gmflow.py::test_corr_families (the first two launches of every call; the "
                                 "fp16 rounding it does is what gmflow_bound evaluates)",
    "mapping_single_kernel": "test_mapping_conflicts.py::test_kernel_equals_the_oracle (bit-exact; also "
                             "test_gpu_kernels.py::test_mapping_bit_exact_golden)",
}


def _table_names():
    return {k for r in ROWS for k in r.kernels}


def _source_names():
    """Launch names the launchers can produce, from the instantiation lists in the sources."""
    src = {f: open(os.path.join(CSRC, f)).read() for f in os.listdir(CSRC) if f.endswith(".cu")}
    hbm, attn = src["hbm_kernels.cu"], src["attn_wgmma.cu"]
    names = set()
    for p, q in re.findall(r"\bLQ\((\d+), (\d+)\)", hbm):
        names.add(f"warp_loss_quad_kernel<{p},{q}>")
    for p, k in re.findall(r"\bLOSS_CASE\((\d+), (\d+)\)", hbm):
        names.add(f"warp_loss_group_kernel<{p},{k}>")
    for tn in ("float", "half"):
        for p, q in re.findall(r"\bCQ\((\d+), (\d+)\)", hbm):
            names.add(f"warp_chain_quad_kernel<{tn},{p},{q}>")
        for k in re.findall(r"launch_chain_group<T, (\d+)>", hbm):
            names.add(f"warp_chain_group_kernel<{tn},{k}>")
    nmax = re.findall(r"launch_temporal_rows<DD, (\d+)>", hbm)
    for d in re.findall(r"\bROWS\((\d+)\);", hbm):
        names.update(f"temporal_attn_rows_kernel<{d},{n}>" for n in nmax)
    for d in map(int, re.findall(r"\bATTN_CASE\((\d+)\);", attn)):
        for wide in ((0, 1, 2) if d <= 64 else (0, 1)):
            for poly in (0, 4, 8):
                for rowsum in ((0, 1) if wide == 0 else (0,)):
                    names.add(attn_name(d, wide, poly, rowsum))
    for epi, bmn in re.findall(r"launch_gemm<(EPI_\w+), (true|false)>", src["gemm_wgmma.cu"]):
        names.add(f"tile_gemm_kernel<{epi},{int(bmn == 'true')}>")
    names.update(re.findall(r"\"(gram2_kernel<G2_\w+>)\"", src["gram_wgmma.cu"]))
    # plain launch names: check_launch("name") / check_launch(c ? "name<half>" : "name<float>")
    for text in src.values():
        for call in re.findall(r"check_launch\(([^;]*)\);", text):
            names.update(re.findall(r"\"(\w+_kernel(?:<\w+>)?)\"", call))
    return names


def test_launch_name_universe():
    """Every launch name the sources can produce is a table row, not the last launch of its call, or checked by a
    named test elsewhere -- exactly one of those; a new kernel or instantiation fails here until it is placed.
    (Needs no GPU.)"""
    table = _table_names()
    buckets = [table, set(NOT_LAST), set(COVERED_ELSEWHERE)]
    for i in range(len(buckets)):
        for j in range(i + 1, len(buckets)):
            assert not buckets[i] & buckets[j], buckets[i] & buckets[j]
    known = set().union(*buckets)
    universe = _source_names()
    assert len(universe) > 80, len(universe)
    assert universe == known, {"not placed": sorted(universe - known), "not launchable": sorted(known - universe)}


@pytest.mark.gpu
@pytest.mark.parametrize("r", ROWS, ids=lambda r: r.id)
def test_kernel_variant(fb, r):
    for name, v in r.opts.items():
        fb.lib.set_option(name, v)
    try:
        launch = Launches(fb, r)
        r.run(fb, launch)
        assert launch.i == len(r.kernels), f"launched {launch.i} of the {len(r.kernels)} kernels the table expects"
    finally:
        for name in r.opts:
            fb.lib.set_option(name, -1)
        torch.cuda.empty_cache()
    RAN.add(r.id)


@pytest.mark.gpu
def test_every_reachable_name_was_launched(fb):
    """The names the rows saw are exactly the table's reachable set (runs after the rows, with all of them)."""
    if len(RAN) != len(ROWS):
        pytest.skip("only meaningful after every row has run and passed")
    assert SEEN == _table_names(), {"expected, not seen": sorted(_table_names() - SEEN), "seen": sorted(SEEN - _table_names())}
