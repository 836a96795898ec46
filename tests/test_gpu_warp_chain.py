"""warp_tensor's frame chain (W1) and the bilinear flow warp (W3) through the C ABI, against oracle.warp_chain_bound.

``fresco_warp_fuse_chain`` runs one of thirteen kernels, picked from the plane size, the channel divisibility and the SM
count; every case asserts the launch name:

* warp_chain_quad_kernel<float|half, P, NQ> for (1,4), (2,2) and (4,1);
* warp_chain_group_kernel<float|half, K> for K = 8, 3 (both with a partial last CTA: planes % K != 0) and 1;
* warp_blend_step_kernel, one launch per chain step, for planes over 100 KB (fp32 only).

Every input family of the bound runs on every kernel, at the shapes the ``chain-*`` rows of test_gpu_kernel_variants.py
use, with chunks 1 and 2 and 2, 3, 8 and 16 frames.  Outputs are prefilled with NaN between two NaN guard planes; every
element must lie within the bound, the exact families must match bit for bit, and the guard planes must stay NaN.
Bit-exact invariances: in place (``out`` is ``sample``) equals out of place on every kernel; relabelling channels
relabels the output; one chunks = 2 call equals two chunks = 1 calls; the same planes through different instantiations
(the channel-resharded warp_tensor of a 1280-channel call at G = 2 takes <2,2> where the unsharded call takes <1,4>, and
slices select <4,1>, group 8, 3 and 1) give the same bits.  ``flow_warp_kernel`` is held to its bound at 1, 2, 3 and 320
channels with flow_batch < batch, the consistency check's masks to the fp64 masks outside the band the warp bound
implies, and ``warp_tensor`` end to end on the host-prepared operands at the decoder and envelope grids and at fp16
image resolution.

``test_report_worst_ratios`` prints the largest err / tol per kernel and family (-s to see it).
"""
import numpy as np
import pytest
import torch

from oracle import fresco_oracle as O
from oracle import warp_chain_bound as CB

pytestmark = pytest.mark.gpu

# kernel -> the (chunks, C, h, w) that select it on a 132-SM H100 ({t}: float or half)
SHAPES = {
    "warp_chain_quad_kernel<{t},1,4>": [(2, 1280, 32, 32), (1, 2560, 16, 16), (2, 1280, 8, 8)],
    "warp_chain_quad_kernel<{t},2,2>": [(2, 640, 32, 32), (1, 1280, 32, 32)],
    "warp_chain_quad_kernel<{t},4,1>": [(2, 640, 64, 64), (1, 1280, 64, 64)],
    "warp_chain_group_kernel<{t},8>": [(2, 1190, 16, 16), (2, 1280, 40, 40)],      # 2380 % 8 = 4
    "warp_chain_group_kernel<{t},3>": [(2, 1280, 48, 48), (2, 450, 32, 32)],       # 2560 % 3 = 1
    "warp_chain_group_kernel<{t},1>": [(2, 6, 32, 24), (1, 6, 32, 24)],
    "warp_blend_step_kernel": [(2, 3, 176, 192), (1, 3, 176, 192)],
}
FRAMES = (2, 3, 8, 16)
RATIOS = {}     # (kernel, family) -> worst err / tol


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib, flow_utils, ops
    _lib.lib()      # fails loudly if the extension is missing
    assert torch.cuda.get_device_properties(0).multi_processor_count == 132, "the shapes select kernels on 132 SMs"

    class NS:
        pass
    ns = NS()
    ns.lib, ns.ops, ns.c, ns.fu = _lib, ops, _lib.lib(), flow_utils
    return ns


def P(t):
    return t.data_ptr()


def _kernels():
    out = []
    for k in SHAPES:
        for t in (("float", "half") if "{t}" in k else ("float",)):
            out.append((k.format(t=t), k, torch.float16 if t == "half" else torch.float32))
    return out


KERNELS = _kernels()


def _guarded(shape, dtype):
    """(buffer with one NaN guard plane before and after, the output view between them)."""
    buf = torch.full((shape[0] + 2,) + tuple(shape[1:]), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[1:-1]


def _chain(fb, d, chunks, out=None, kernel=None):
    """fresco_warp_fuse_chain on the family's operands through the C ABI -> out (NaN-prefilled between guard planes
    unless given)."""
    s = d["sample"]
    buf = None
    if out is None:
        buf, out = _guarded(s.shape, s.dtype)
    B, C, h, w = s.shape
    rc = fb.c.fresco_warp_fuse_chain(P(s), P(out), int(s.dtype == torch.float16), P(d["bwd"]), P(d["fwd_last"]),
                                     P(d["blend"]), chunks, B // chunks, C, h, w, fb.lib.stream())
    fb.lib.check(rc, "fresco_warp_fuse_chain")
    if kernel is not None:
        assert fb.lib.last_kernel() == kernel, f"launched {fb.lib.last_kernel()}, expected {kernel}"
    if buf is not None:
        assert torch.isnan(buf[0]).all() and torch.isnan(buf[-1]).all(), "a guard plane was written"
    return out


def _prepare(fb):
    def prep(flows, occs, sal, n, h, w):
        return fb.fu.chain_operands(flows, occs, sal, n, h, w)
    return prep


def _check(out, ref, tol, fam, dtype, what):
    assert torch.isfinite(out).all(), f"{what}: {(~torch.isfinite(out)).sum().item()} outputs not written or not finite"
    r = CB.ratio(out, ref, tol)
    worst = r.max().item()
    if worst > 1:
        bad = torch.nonzero(r > 1)
        i = tuple(bad[0].tolist())
        raise AssertionError(f"{what}: {bad.shape[0]} elements outside the bound, worst err/tol {worst:.3g}; first at "
                             f"{i}: out {out[i].item()!r} ref {ref[i].item()!r} tol {tol[i].item():.3g}")
    if fam in CB.EXACT:
        want = CB.exact_output(ref, dtype)
        assert torch.equal(out, want), f"{what}: {(out != want).sum().item()} elements not bit-exact"
    return worst


def _cases():
    out = []
    for name, key, dtype in KERNELS:
        for i, fam in enumerate(CB.FAMILIES):
            shape = SHAPES[key][i % len(SHAPES[key])]
            N = FRAMES[(i + len(name)) % 4]
            out.append(pytest.param(name, fam, shape, N, dtype, id=f"{name}-{fam}-c{shape[0]}x{shape[1]}x{shape[2]}x"
                                    f"{shape[3]}-n{N}"))
    return out


@pytest.mark.parametrize("kname,fam,shape,N,dtype", _cases())
def test_chain_family(fb, kname, fam, shape, N, dtype):
    chunks, C, h, w = shape
    d = CB.family(fam, chunks, N, C, h, w, dtype=dtype, seed=len(kname), device="cuda", prepare=_prepare(fb))
    out = _chain(fb, d, chunks, kernel=kname)
    ref, tol = CB.chain_reference_and_bound(d["sample"], d["bwd"], d["fwd_last"], d["blend"], chunks)
    RATIOS[(kname, fam)] = max(RATIOS.get((kname, fam), 0.0), _check(out, ref, tol, fam, dtype, f"{kname} {fam}"))


@pytest.mark.parametrize("kname,key,dtype", KERNELS, ids=[k[0] for k in KERNELS])
def test_chain_invariances(fb, kname, key, dtype):
    """In place equals out of place; relabelling channels relabels the output; a chunks = 2 call equals its chunks
    = 1 calls -- bit for bit.  (The chunks = 1 calls may select another instantiation.)"""
    chunks, C, h, w = SHAPES[key][0]
    N = 3
    d = CB.family("near-integer", chunks, N, C, h, w, dtype=dtype, seed=7, device="cuda")
    base = _chain(fb, d, chunks, kernel=kname)
    inplace = d["sample"].clone()
    _chain(fb, dict(d, sample=inplace), chunks, out=inplace, kernel=kname)
    assert torch.equal(inplace, base), f"in place: {(inplace != base).sum().item()} elements differ"
    perm = torch.randperm(C, generator=torch.Generator().manual_seed(3)).cuda()
    relabelled = _chain(fb, dict(d, sample=d["sample"][:, perm].contiguous()), chunks, kernel=kname)
    assert torch.equal(relabelled, base[:, perm]), "channel relabelling changes the bits"
    if chunks == 2:
        for j in range(2):
            part = _chain(fb, dict(d, sample=d["sample"][j * N:(j + 1) * N].contiguous()), 1)
            assert torch.equal(part, base[j * N:(j + 1) * N]), f"chunk {j} alone differs ({fb.lib.last_kernel()})"


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["float", "half"])
def test_same_planes_through_every_instantiation(fb, dtype):
    """One 1280-channel call at 32 x 32 (chunks 2: <1,4>) against calls on slices of its planes that select the other
    instantiations, bit for bit.  The first slice is the channel-resharded warp_tensor at G = 2 (config 4): all frames,
    channels [0, 640) of both chunks as one chunk of 1280 planes, which takes <2,2>."""
    t = "half" if dtype == torch.float16 else "float"
    chunks, C, h, w, N = 2, 1280, 32, 32, 8
    d = CB.family("realistic", chunks, N, C, h, w, dtype=dtype, seed=11, device="cuda", prepare=_prepare(fb))
    full = _chain(fb, d, chunks, kernel=f"warp_chain_quad_kernel<{t},1,4>")
    s5, f5 = d["sample"].view(chunks, N, C, h, w), full.view(chunks, N, C, h, w)

    def planes(x, c0, c1):                      # [frames, chunk-major planes of channels [c0, c1) of every chunk]
        return x[:, :, c0:c1].transpose(0, 1).reshape(N, chunks * (c1 - c0), h, w).contiguous()

    for c0, c1, kname in ((0, 640, f"warp_chain_quad_kernel<{t},2,2>"), (640, 1152, f"warp_chain_quad_kernel<{t},4,1>"),
                          (0, 1185, f"warp_chain_group_kernel<{t},8>"), (3, 598, f"warp_chain_group_kernel<{t},3>"),
                          (1277, 1280, f"warp_chain_group_kernel<{t},1>")):
        out = _chain(fb, dict(d, sample=planes(s5, c0, c1)), 1, kernel=kname)
        assert torch.equal(out, planes(f5, c0, c1)), f"{kname}: {(out != planes(f5, c0, c1)).sum().item()} differ"


def test_frames_one_refused_before_any_launch(fb):
    """frames = 1 is refused with FrescoError, through ops and the C ABI, and nothing is launched or written."""
    x = torch.randn(2, 8, 16, 16, device="cuda")
    flow = torch.zeros(1, 2, 16, 16, device="cuda")
    blend = torch.zeros(1, 16, 16, device="cuda")
    fb.ops.flow_warp(x, flow)
    torch.cuda.synchronize()
    assert fb.lib.last_kernel() == "flow_warp_kernel"
    out = torch.full_like(x, float("nan"))
    with pytest.raises(fb.lib.FrescoError, match="frames >= 2"):
        fb.ops.warp_fuse_chain(x, flow, flow[0].contiguous(), blend, 2, out=out)
    rc = fb.c.fresco_warp_fuse_chain(P(x), P(out), 0, P(flow), P(flow), P(blend), 2, 1, 8, 16, 16, fb.lib.stream())
    assert rc != 0 and b"frames >= 2" in fb.c.fresco_last_error()
    torch.cuda.synchronize()
    assert fb.lib.last_kernel() == "flow_warp_kernel" and torch.isnan(out).all()


# ------------------------------------------------------------------------------------------------ flow warp
@pytest.mark.parametrize("B,Bf,C,h,w", [(4, 2, 1, 37, 53), (3, 1, 2, 24, 40), (6, 4, 3, 64, 96), (2, 1, 320, 32, 32),
                                        (5, 5, 3, 1, 29), (2, 1, 2, 17, 1)])
@pytest.mark.parametrize("fam", ["edges", "realistic", "near-integer"])
def test_flow_warp(fb, fam, B, Bf, C, h, w):
    if fam != "edges" and min(h, w) == 1:
        pytest.skip("one-pixel axis: the edge family covers it")
    d = CB.family(fam, 1, max(Bf, 2), 1, h, w, seed=B + C, device="cuda", prepare=_prepare(fb))
    flow = torch.cat([d["bwd"], d["fwd_last"][None]])[:Bf].contiguous()
    g = torch.Generator(device="cuda").manual_seed(C)
    src = torch.randn(B, C, h, w, device="cuda", generator=g) * torch.logspace(-3, 3, C, device="cuda")[None, :, None, None]
    buf, dst = _guarded(src.shape, torch.float32)
    fb.lib.check(fb.c.fresco_flow_warp(P(src), P(flow), P(dst), B, C, h, w, Bf, fb.lib.stream()), "fresco_flow_warp")
    assert fb.lib.last_kernel() == "flow_warp_kernel"
    assert torch.isnan(buf[0]).all() and torch.isnan(buf[-1]).all(), "a guard plane was written"
    ref, tol = CB.flow_warp_reference_and_bound(src, flow)
    RATIOS[("flow_warp_kernel", fam)] = max(RATIOS.get(("flow_warp_kernel", fam), 0.0),
                                           _check(dst, ref, tol, fam, torch.float32, f"flow_warp {fam}"))


@pytest.mark.parametrize("N,H,W,mag", [(3, 64, 96, 10.0), (4, 128, 128, 12.0), (2, 96, 64, 30.0)])
def test_consistency_masks_outside_the_band(fb, N, H, W, mag):
    """forward_backward_consistency_check equals the fp64 masks at every pixel whose |norm - thr| lies outside the band
    the warp bound and the fp32 norms imply; at most 1e-3 of the pixels fall inside it."""
    flows, _ = O.synth_flows(N, H, W, seed=H + W, mag=mag)
    fwd, bwd = flows[0].cuda().contiguous(), flows[1].cuda().contiguous()
    fo, bo = fb.fu.forward_backward_consistency_check(fwd, bwd)
    ref = CB.consistency_reference(fwd, bwd)
    for name, got in (("fwd", fo), ("bwd", bo)):
        want, band = ref[name + "_occ"], ref[name + "_band"]
        bad = (got.bool() != want) & ~band
        assert not bad.any(), f"{name}_occ: {bad.sum().item()} pixels outside the band differ"
        assert band.float().mean().item() < 1e-3, f"{name}: {band.sum().item()} pixels inside the band"
        assert 0.01 < want.float().mean().item() < 0.99, "the masks should have both values"


# ------------------------------------------------------------------------------------------------ end to end
def _resize_dims(h, w, resolution):
    k = float(resolution) / min(h, w)
    return int(np.round(h * k / 64.0)) * 64, int(np.round(w * k / 64.0)) * 64


ENVELOPE = sorted({_resize_dims(h, w, s) for s in range(256, 512, 64)
                   for h, w in [(512, 512), (480, 640), (640, 480), (1080, 1920), (1920, 1080)]})
# (image H, W, decoder grid divisor, channels, dtype)
E2E = ([(512, 512, s, c, dt) for s, c in ((64, 1280), (32, 1280), (16, 1280), (8, 640))
        for dt in (torch.float32, torch.float16)]
       + [(H, W, s, 16, torch.float16 if (H + s) % 3 else torch.float32) for H, W in ENVELOPE for s in (8, 16, 32, 64)]
       + [(256, 320, 1, 3, torch.float16), (512, 512, 1, 3, torch.float16), (256, 256, 1, 3, torch.float32)])


@pytest.mark.parametrize("H,W,s,C,dtype", E2E, ids=lambda v: str(v).replace("torch.", ""))
def test_warp_tensor_end_to_end(fb, H, W, s, C, dtype):
    """warp_tensor (chunks 2, or 1 at image resolution) within the bound of the chain on the operands its own
    preparation made; image planes run the fp32 per-step kernel and round to fp16 once."""
    N, chunks = 3, (1 if s == 1 else 2)
    h, w = H // s, W // s
    flows, occs = O.synth_flows(N, H, W, seed=H * W + s, mag=12.0)
    sal = torch.rand(N, 1, H // 2, W // 2, generator=torch.Generator().manual_seed(s))
    fl, oc, sl = [f.cuda() for f in flows], [o.cuda() for o in occs], sal.cuda()
    g = torch.Generator(device="cuda").manual_seed(h * w)
    sample = torch.randn(chunks * N, C, h, w, device="cuda", generator=g).to(dtype)
    out = fb.fu.warp_tensor(sample, fl, oc, sl, chunks)
    assert out.dtype == dtype and out.shape == sample.shape
    bwd, fwd_last, blend = fb.fu.chain_operands(fl, oc, sl, N, h, w)
    chain_in = sample if 2 * h * w * 4 <= 200 * 1024 else sample.float()
    ref, tol = CB.chain_reference_and_bound(chain_in, bwd, fwd_last, blend, chunks, out_dtype=dtype)
    _check(out, ref, tol, "realistic", dtype, f"warp_tensor {H}x{W}/{s}")


def test_report_worst_ratios():
    """Prints the largest err / tol seen per kernel and family (-s to see it)."""
    if not RATIOS:
        pytest.skip("no warp-chain case ran")
    print("\nworst err/tol per kernel and family")
    for (kn, fam), r in sorted(RATIOS.items()):
        print(f"  {kn:36s} {fam:13s} {r:.3g}")
    for fam in CB.FAMILIES:
        rs = [r for k, r in RATIOS.items() if k[1] == fam]
        if rs:
            print(f"  max {fam:13s} {max(rs):.3g}")
