"""fp64 reference of warp_tensor's frame chain (W1: ``warp_chain_quad_kernel<T,P,NQ>``, ``warp_chain_group_kernel<T,K>``,
``warp_blend_step_kernel`` in hbm_kernels.cu) and of the bilinear flow warp (W3: ``flow_warp_kernel``), an elementwise
bound on the kernels' error, and input families built to break them.

CHECKER ONLY (see ``oracle/__init__``).  The operands are the kernels' own: ``sample`` fp16 or fp32
[chunks N, C, h, w] (chunk-major, as ``fresco_warp_fuse_chain`` reads it), ``bwd_flow`` fp32 [N, 2, h, w] (entry N - 1
unused), ``fwd_flow_last`` fp32 [2, h, w] and ``blend`` fp32 [N, h, w] (or [N, 1, h, w]).  Every (chunk, channel) plane
runs the chain of src/flow_utils.py:41-51 on its own:

    z_0 = s_0;   z_{i+1} = s_{i+1} (1 - m_i) + W_bwd[i](z_i) m_i   (i = 0 .. N-2)
    out_f = z_f (f < N-1);   out_{N-1} = z_{N-1} (1 - m_{N-1}) + W_fwd_last(s_0) m_{N-1}

with W the zero-padded bilinear warp at (x + flow_x, y + flow_y), its taps evaluated in fp64 (``warp_loss_bound.taps64``).
The flow warp is one W: out_b = W_{flow[b mod Bf]}(src_b).

The bound
---------
Every chain kernel does the same per-element work (``make_taps``, ``sample_taps`` / ``sample_taps4``, ``chain_blend``)
and carries z in fp32 between frames (shared memory or the fp32 planes of the per-step kernel); only the stores round to
the output type.  u = 2^-24, F = 2.  For one blend new = own (1 - m) + W(src) m, with ``own`` and ``src`` the kernel's
fp32 values:

* coordinate: the kernel rounds x + flow to fp32; it differs from the fp64 coordinate by d = |X32 - X64| + |Y32 - Y64|
  (evaluated exactly).  The zero-padded bilinear surface is continuous and, inside a cell, has slope at most 2 max|z|
  over the cell's corners in each direction, so the sample moves by at most 2 L d, L = max|src| over the valid corners
  of the fp64 and of the fp32 cell -- also when floor crosses an integer or a tap crosses the border (a tap's weight is
  a hat function that vanishes there).  This is the argument of ``warp_loss_bound``.
* weight products: ax = X - floor(X) is exact except for X in (-1, 0), where it rounds by at most u ax and the (1 - ax)
  column is the invalid x0 = -1; so each factor rounds once and the product once: 3 u relative per weight.
* the 4-term sum: at most four roundings on any term in any association nvcc picks (products and adds, or fmas): 4 u.
  Together 7 u sum_t w_t |src_t|.
* the blend: fl(1 - m), the product with own and the add: 3 u (1 - m) |own|; the product W m and the add:
  2 u m sum_t w_t |src_t| -- in any contraction nvcc picks.

local = F (m (2 L d + 9 u sum_t w_t |src_t|) + 3 u (1 - m) |own|).  The error the operands already carry propagates
linearly through the fp64 taps: E_new = (1 - m) E_own + m sum_t w_t E_src(src_t) + local.  Along the chain E_0 = 0 (s_0
is exact in fp32), own = s_{i+1} (exact) and src = z_i, so E_{i+1} = m_i sum_t w_t E_i(src_t) + local_{i+1}; the closing
blend has own = z_{N-1} and src = s_0: E = (1 - m) E_{N-1} + local.  (Second-order terms -- the error of z inside L and
the weights' own change at a cell crossing acting on E -- are what F covers.)  The flow warp is one such sample with
m = 1 and exact src: F (2 L d + 7 u sum_t w_t |src_t|).

An fp16 output rounds the fp32 value once, by at most half an fp16 ulp: 2^-11 (|ref| + E) in the normal range and 2^-25
(half the subnormal spacing) below it.  Nothing else is widened.

Input families (``family``): three have exact answers, whatever the contraction -- ``zero-mask`` (m = 0: out equals
sample), ``integer`` (integer flows, m in {0, 1}: values are moved or zeroed) and ``identity`` (zero flow, integer samples of
at most 5 bits, m in {0, 1/2, 1}: every blend of a chain of up to 16 frames is exact in fp32).  ``pure-warp`` (m = 1 everywhere: the chain is N - 1 nested warps),
``near-integer`` (x + flow within a few ulp of an integer, so fp32 and fp64 floors differ), ``edges`` (coordinates in
(-1, 0), exactly -1, exactly w - 1, in (w - 1, w), far outside and past the kernels' 1e9 guard, on both axes),
``magnitudes`` (1e-3 and 1e3 in one plane; fp16 values up to 6e4) and ``realistic`` (``O.synth_flows`` at 8x the plane
through the host's resize and blend-weight preparation).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import fresco_oracle as O
from .warp_loss_bound import _warp, taps32, taps64

U = 2.0 ** -24
SAFETY = 2.0
HALF_ULP = 2.0 ** -11           # half an fp16 ulp, relative, in the normal range
HALF_SUB = 2.0 ** -25           # half the fp16 subnormal spacing

FAMILIES = ("zero-mask", "integer", "identity", "pure-warp", "near-integer", "edges", "magnitudes", "realistic")
EXACT = ("zero-mask", "integer", "identity")


# ------------------------------------------------------------------------------------------------ one blend
def _taps(flow2):
    T64, T32 = taps64(flow2), taps32(flow2)
    d = (T32["X"].double() - T64["X"]).abs() + (T32["Y"].double() - T64["Y"]).abs()
    d = torch.where(torch.isfinite(d), d, torch.zeros_like(d))
    return T64, T32, d


def _corner_max(src, T64, T32):
    """max |src| over the valid corners of the fp64 and the fp32 cell -> [P, hw]."""
    a = src.abs()
    return torch.cat([T["valid"].to(a.dtype)[None] * a[:, T["idx"]] for T in (T64, T32)], -1).amax(-1)


def sample_and_bound(src, flow2):
    """One warp of src [P, hw] (fp64 values of the kernel's fp32 operand) through flow2 [2, h, w]: (W(src) in fp64,
    2 L d, sum_t w_t |src_t|, the fp64 taps)."""
    T64, T32, d = _taps(flow2)
    coord = 2.0 * _corner_max(src, T64, T32) * d[None]
    return _warp(src, T64), coord, _warp(src.abs(), T64), T64


def blend_step(own, e_own, src, e_src, flow2, m):
    """new = own (1 - m) + W(src) m in fp64 and its bound: (new, E_new), all [P, hw]; m [1, hw]."""
    warped, coord, sabs, T64 = sample_and_bound(src, flow2)
    new = own * (1 - m) + warped * m
    local = SAFETY * (m * (coord + 9 * U * sabs) + 3 * U * (1 - m) * own.abs())
    err = local
    if e_own is not None:
        err = err + (1 - m) * e_own
    if e_src is not None:
        err = err + m * _warp(e_src, T64)
    return new, err


def _out_tol(ref, tol, dtype):
    if dtype == torch.float16:
        return tol + HALF_ULP * (ref.abs() + tol) + HALF_SUB
    return tol


# ------------------------------------------------------------------------------------------------ references + bounds
def chain_reference_and_bound(sample, bwd_flow, fwd_flow_last, blend, chunks, out_dtype=None):
    """fresco_warp_fuse_chain in fp64 and its elementwise bound: (ref fp64, tol fp64), both shaped like ``sample``.
    ``out_dtype``: the type the result is finally stored in (default: sample's; warp_tensor runs fp16 image planes
    through the fp32 per-step kernel and rounds its result to fp16 once)."""
    B, C, h, w = sample.shape
    N, hw = B // chunks, h * w
    assert N >= 2 and N * chunks == B
    x = sample.double().reshape(chunks, N, C, hw).permute(1, 0, 2, 3).reshape(N, chunks * C, hw)
    m = blend.double().reshape(N, 1, hw)
    z, e = [x[0]], [torch.zeros_like(x[0])]
    for i in range(N - 1):
        zi, ei = blend_step(x[i + 1], None, z[-1], e[-1], bwd_flow[i], m[i])
        z.append(zi)
        e.append(ei)
    z[-1], e[-1] = blend_step(z[-1], e[-1], x[0], None, fwd_flow_last, m[N - 1])

    def back(frames):
        return torch.stack(frames).reshape(N, chunks, C, h, w).transpose(0, 1).reshape(B, C, h, w)

    ref = back(z)
    return ref, _out_tol(ref, back(e), out_dtype or sample.dtype)


def flow_warp_reference_and_bound(src, flow):
    """fresco_flow_warp in fp64 (sample b through flow b mod Bf) and its bound: (ref, tol) like ``src``."""
    B, C, h, w = src.shape
    ref = torch.empty(B, C, h * w, dtype=torch.float64, device=src.device)
    tol = torch.empty_like(ref)
    for bf in range(min(flow.shape[0], B)):
        sel = torch.arange(bf, B, flow.shape[0], device=src.device)
        planes = src[sel].double().reshape(-1, h * w)
        warped, coord, sabs, _ = sample_and_bound(planes, flow[bf])
        ref[sel] = warped.reshape(-1, C, h * w)
        tol[sel] = (SAFETY * (coord + 7 * U * sabs)).reshape(-1, C, h * w)
    return ref.reshape(B, C, h, w), tol.reshape(B, C, h, w)


def consistency_reference(fwd, bwd, alpha=0.01, beta=0.5):
    """forward_backward_consistency_check (gmflow/geometry.py:75-96) in fp64 on fp32 flows [B, 2, h, w], with the band
    around the threshold inside which the fp32 computation may decide either way.  -> dict of fwd_occ / bwd_occ (bool),
    fwd_band / bwd_band (bool: |norm - thr| within the band).  The band: the warp's bound on both components, the fp32
    add fwd + warped (u per component), the fp32 norm (2 u) and the threshold alpha mag + beta (two norms, their sum,
    the product with fp32(alpha) and the add: 6 u), F on the roundings."""
    f64, b64 = fwd.double(), bwd.double()
    mag = f64.norm(dim=1) + b64.norm(dim=1)
    thr = alpha * mag + beta
    out = {}
    for name, a, other, a64 in (("fwd", fwd, bwd, f64), ("bwd", bwd, fwd, b64)):
        warped, tol = flow_warp_reference_and_bound(other, a)
        v = a64 + warped
        n = v.norm(dim=1)
        band = tol.sum(1) + SAFETY * (U * (a64.abs() + warped.abs()).sum(1) + 2 * U * n + 6 * U * thr)
        out[name + "_occ"] = n > thr
        out[name + "_band"] = (n - thr).abs() <= band
    return out


def ratio(out: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor) -> torch.Tensor:
    """|out - ref| / tol elementwise (0 where out == ref, also where tol is 0; NaN in out counts as infinitely wrong)."""
    err = (out.double() - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / tol)
    return torch.nan_to_num(r, nan=float("inf"))


def exact_output(ref: torch.Tensor, dtype) -> torch.Tensor:
    """The output of an exact family: ref in ``dtype`` (asserting the fp32 chain value is ref itself)."""
    assert torch.equal(ref.float().double(), ref), "family not exact in fp32"
    return ref.to(dtype)


# ------------------------------------------------------------------------------------------------ input families
def _smooth(N, h, w, g, mag=3.0):
    coarse = torch.randn(N, 2, 3, 3, generator=g) * mag
    return F.interpolate(coarse, size=(h, w), mode="bicubic", align_corners=False).float()


def host_prepare(flows, occs, saliency, n, h, w):
    """The blend weights of flow_utils.warp_tensor's preparation (src/flow_utils.py:24-51) in torch fp32 on the CPU, with
    the oracle's flow_warp for the saliency warps: (bwd_flow [n, 2, h, w], fwd_flow_last [2, h, w], blend [n, 1, h, w])."""
    scale = h * 1.0 / flows[0].shape[2]
    ff, bf, fo, bo = O._resize_flow_occ(flows, occs, scale)
    if scale == 1:
        bo, fo = O.dilate(bo, 13), O.dilate(fo, 13)
    sal = F.interpolate(saliency.float(), scale_factor=h * 1.0 / saliency.shape[2], mode="bilinear")
    ws = O.flow_warp(sal, bf)
    ws_last = O.flow_warp(sal[0:1], ff[n - 1:n])
    blend = torch.empty(n, 1, h, w)
    blend[:n - 1] = (1 - bo[:n - 1]) * sal[1:n] * ws[:n - 1]
    blend[n - 1:] = (1 - fo[n - 1:n]) * sal[n - 1:n] * ws_last
    return bf.float().contiguous(), ff[n - 1].float().contiguous(), blend.contiguous()


def realistic_inputs(N, h, w, seed, scale=8):
    """(flows, occs, saliency) of a keyframe batch whose decoder layer has an h x w grid: O.synth_flows at scale x the
    plane, saliency at half that resolution."""
    flows, occs = O.synth_flows(N, scale * h, scale * w, seed=seed, mag=12.0)
    sal = torch.rand(N, 1, max(1, scale * h // 2), max(1, scale * w // 2), generator=torch.Generator().manual_seed(seed))
    return flows, occs, sal


def _edge_coords(n_pix, extent, g):
    """Target coordinates along one axis of length ``extent``, cycling through the edge categories."""
    cats = [lambda k: -torch.rand(k, generator=g, dtype=torch.float64),             # (-1, 0)
            lambda k: torch.full((k,), -1.0, dtype=torch.float64),                   # exactly -1
            lambda k: torch.full((k,), float(extent - 1), dtype=torch.float64),      # exactly w - 1
            lambda k: extent - torch.rand(k, generator=g, dtype=torch.float64),      # (w - 1, w)
            lambda k: torch.rand(k, generator=g, dtype=torch.float64) * (extent - 1),   # inside
            lambda k: -1e-7 * torch.rand(k, generator=g, dtype=torch.float64),     # just below 0
            lambda k: (extent - 1) + 1e-7 * torch.rand(k, generator=g, dtype=torch.float64),   # just past w - 1
            lambda k: torch.full((k,), 1e4, dtype=torch.float64),                     # far outside
            lambda k: torch.full((k,), -3e9, dtype=torch.float64)]                    # past the 1e9 guard
    which = torch.randint(0, len(cats), (n_pix,), generator=g)
    out = torch.empty(n_pix, dtype=torch.float64)
    for i, c in enumerate(cats):
        sel = which == i
        out[sel] = c(int(sel.sum()))
    return out


def family(name, chunks, N, C, h, w, dtype=torch.float32, seed=0, device="cpu", prepare=None):
    """Operands of one fresco_warp_fuse_chain call: dict of sample [chunks N, C, h, w] ``dtype``, bwd [N, 2, h, w],
    fwd_last [2, h, w], blend [N, h, w] (fp32).  ``prepare`` (realistic only): the preparation to take the flows through,
    ``host_prepare``'s signature (flow_utils.chain_operands on the GPU).  Each family asserts what it is built to have."""
    g = torch.Generator().manual_seed(seed * 7919 + sum(map(ord, name)) + 31 * N + h * w)
    B, hw = chunks * N, h * w
    sample = torch.randn(B, C, h, w, generator=g)
    blend = torch.rand(N, h, w, generator=g)
    bwd, fwd_last = _smooth(N, h, w, g), _smooth(1, h, w, g)[0]
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
    if name == "zero-mask":
        blend.zero_()
    elif name == "integer":
        bwd = torch.randint(-3, 4, (N, 2, h, w), generator=g).float()
        fwd_last = torch.randint(-3, 4, (2, h, w), generator=g).float()
        blend = (torch.rand(N, h, w, generator=g) < 0.6).float()
    elif name == "identity":
        bwd.zero_()
        fwd_last.zero_()
        blend = torch.randint(0, 3, (N, h, w), generator=g).float() * 0.5
        sample = torch.randint(-31, 32, (B, C, h, w), generator=g).float()     # 5 + 16 bits after 16 halvings
    elif name == "pure-warp":
        blend.fill_(1.0)
    elif name == "near-integer":
        # x + flow = an integer moved by a few ulp of the flow: the fp32 sum rounds onto the integer (or across it)
        k = torch.randint(-2, 3, (N + 1, 2, h, w), generator=g).float()
        steps = torch.randint(-3, 4, (N + 1, 2, h, w), generator=g)
        fl = k.clone()
        for _ in range(3):
            up, dn = torch.nextafter(fl, torch.full_like(fl, 1e9)), torch.nextafter(fl, torch.full_like(fl, -1e9))
            fl = torch.where(steps > 0, up, torch.where(steps < 0, dn, fl))
            steps = steps - steps.sign()
        tiny = (torch.rand(N + 1, 2, h, w, generator=g) - 0.5) * 2e-7            # around flow 0: x + flow just off x
        fl = torch.where(k == 0, tiny, fl)
        bwd, fwd_last = fl[:N].contiguous(), fl[N].contiguous()
        diff = 0
        for f in list(bwd) + [fwd_last]:
            T64, T32 = taps64(f), taps32(f)
            diff += int((T64["x0"] != T32["x0"]).sum() + (T64["y0"] != T32["y0"]).sum())
        assert diff >= 0.05 * (N + 1) * hw, f"only {diff} fp32 floors differ from fp64"
    elif name == "edges":
        fl = torch.empty(N + 1, 2, h, w)
        for f in range(N + 1):
            fl[f, 0] = (_edge_coords(hw, w, g).reshape(h, w) - xs).float()
            fl[f, 1] = (_edge_coords(hw, h, g).reshape(h, w) - ys).float()
        bwd, fwd_last = fl[:N].contiguous(), fl[N].contiguous()
        X = torch.cat([taps64(f)["X"] for f in list(bwd) + [fwd_last]])
        for side in ((X > -1) & (X < 0), X == -1, (X > w - 1) & (X < w), X.abs() > 1e9):
            assert side.any(), "an edge category is missing"
    elif name == "magnitudes":
        big = torch.rand(B, C, h, w, generator=g) < 0.5
        sample = torch.where(big, sample * 1e3, sample * 1e-3)
        if dtype == torch.float16:
            top = torch.rand(B, C, h, w, generator=g) < 0.1
            sample = torch.where(top, torch.sign(sample) * (5e4 + 1.5e4 * torch.rand(B, C, h, w, generator=g)), sample)
            sample = sample.clamp(-65504, 65504)
    elif name == "realistic":
        flows, occs, sal = realistic_inputs(N, h, w, seed)
        prep, pdev = (prepare, device) if prepare is not None else (host_prepare, "cpu")
        bwd, fwd_last, blend = (t.cpu() for t in prep([f.to(pdev) for f in flows], [o.to(pdev) for o in occs],
                                                       sal.to(pdev), N, h, w))
        blend = blend.reshape(N, h, w)
        assert ((blend > 0) & (blend < 1)).any(), "no fractional blend weight"
    else:
        raise ValueError(name)
    sample = sample.to(dtype)
    dev = torch.device(device)
    return {"sample": sample.contiguous().to(dev), "bwd": bwd.float().contiguous().to(dev),
            "fwd_last": fwd_last.float().contiguous().to(dev), "blend": blend.float().contiguous().to(dev)}
