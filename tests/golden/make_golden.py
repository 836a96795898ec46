"""Generate golden vectors by running the REAL reference (williamyang1991/FRESCO) on CPU.

    python tests/golden/make_golden.py [--set b | --only gmflow_rect] --reference /path/to/FRESCO

The reference imports two diffusers names and matplotlib at module top
(src/diffusion_hacked.py:7-8, src/utils.py:5); neither is used on the path we
exercise, so they are stubbed in ``sys.modules``.  Outputs: small ``.npz``
fixtures next to this script, consumed by tests/test_oracle_golden.py (oracle
vs reference) and by the ``-m gpu`` parity tests.  A fixture whose compressed size
would pass 1 MB is stored in parts (``name.npz``, ``name.1.npz``, ...) that the
``golden`` fixture of tests/conftest.py merges again.
"""
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
REF = sys.argv[sys.argv.index("--reference") + 1] if "--reference" in sys.argv else None
PART_BYTES = 960 * 1024


def save_npz(name, **arrays):
    """savez_compressed into HERE/name.npz, split by array into parts below PART_BYTES each."""
    import io
    import zipfile
    for old in os.listdir(HERE):
        if old.startswith(name + ".") and old.endswith(".npz"):
            os.remove(os.path.join(HERE, old))
    sizes = {}
    for k, v in arrays.items():
        buf = io.BytesIO()
        np.savez_compressed(buf, **{k: v})
        sizes[k] = zipfile.ZipFile(buf).infolist()[0].compress_size + 256
    parts, cur, used = [], {}, 0
    for k, v in arrays.items():
        if cur and used + sizes[k] > PART_BYTES:
            parts.append(cur)
            cur, used = {}, 0
        cur[k] = v
        used += sizes[k]
    parts.append(cur)
    for i, part in enumerate(parts):
        np.savez_compressed(os.path.join(HERE, name + (".npz" if i == 0 else ".%d.npz" % i)), **part)


def import_reference():
    for name, attrs in (
        ("diffusers", {}),
        ("diffusers.models", {}),
        ("diffusers.models.unet_2d_condition", {"UNet2DConditionOutput": object}),
        ("diffusers.models.attention_processor", {"AttnProcessor2_0": object}),
        ("matplotlib", {}),
        ("matplotlib.pyplot", {}),
    ):
        if name not in sys.modules:
            m = types.ModuleType(name)
            for k, v in attrs.items():
                setattr(m, k, v)
            sys.modules[name] = m
    os.chdir(REF)
    sys.path.insert(0, REF)
    import src.diffusion_hacked as dh   # noqa
    import src.flow_utils as fu         # noqa
    from gmflow import geometry, matching  # noqa  (path appended by the reference itself)
    import src.utils as ut              # noqa
    return dh, fu, geometry, matching, ut


class FakeAttn(torch.nn.Module):
    """The attributes FRESCOAttnProcessor2_0 reads from diffusers' Attention."""

    def __init__(self, c, heads, seed):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.heads = heads
        self.spatial_norm = None
        self.group_norm = None
        self.norm_cross = False
        self.residual_connection = False
        self.rescale_output_factor = 1.0
        self.to_q = torch.nn.Linear(c, c, bias=False)
        self.to_k = torch.nn.Linear(c, c, bias=False)
        self.to_v = torch.nn.Linear(c, c, bias=False)
        self.to_out = torch.nn.ModuleList([torch.nn.Linear(c, c), torch.nn.Dropout(0.0)])
        with torch.no_grad():
            for p in self.parameters():
                p.copy_(torch.randn(p.shape, generator=g) * (2.0 / c ** 0.5 if p.ndim == 2 else 0.1))


def smooth_flows(n, H, W, seed, mag):
    g = torch.Generator().manual_seed(seed)
    coarse = torch.randn(n, 2, 4, 4, generator=g) * mag
    fwd = F.interpolate(coarse, size=(H, W), mode="bicubic", align_corners=False)
    bwd = -fwd + 0.5 * F.interpolate(torch.randn(n, 2, 4, 4, generator=g), size=(H, W), mode="bicubic")
    return fwd, bwd


def scenario_b(dh, fu, geometry, matching, ut):
    """Second fixture set (``python tests/golden/make_golden.py --set b``): an ODD number of frames, a NON-SQUARE
    plane and head_dim 80 (SD1.5 level A), so that nothing in the oracle or the kernels can silently rely on
    N being even, h == w or d == 40.  Same reference entry points as set A."""
    torch.manual_seed(1)
    torch.set_grad_enabled(False)
    N, H, W = 3, 64, 96
    fwd, bwd = smooth_flows(N, H, W, 21, 4.0)
    fo, bo = geometry.forward_backward_consistency_check(fwd, bwd)
    imgs = torch.rand(N, 3, H, W) * 2 - 1
    bocc = torch.clamp(bo + (torch.rand(N, H, W) > 0.85).float(), 0, 1)
    res = {"fwd": fwd.numpy(), "bwd": bwd.numpy(), "fwd_occ": fo.numpy(), "bwd_occ": bocc.numpy(), "imgs": imgs.numpy()}

    # mapping at scale 8 (8 x 12 tokens)
    fm, bm, im = fu.get_mapping_ind(bwd, bocc, imgs, scale=8.0)
    res.update(fwd_map=fm.numpy(), bwd_map=bm.numpy(), inter_mask=im.numpy())

    # attention, all 8 flag combinations, C = 160 / 2 heads => head_dim 80
    C, heads, chunks = 160, 2, 2
    L = (H // 8) * (W // 8)
    attn = FakeAttn(C, heads, 5)
    x = torch.randn(chunks * N, L, C)
    ref_hidden = torch.randn(chunks * N, L, C)
    attn_mask = []
    for scale in [8.0, 16.0, 32.0]:
        o_ = F.interpolate(bocc[:-1].unsqueeze(1), scale_factor=1. / scale, mode='bilinear')
        attn_mask += [torch.cat((o_[0:1].reshape(1, -1) > -1, o_.reshape(o_.shape[0], -1) > 0.5), dim=0)]
    paras = {"fwd_mappings": [fm], "bwd_mappings": [bm], "interattn_masks": [im]}
    res.update(x=x.numpy(), ref_hidden=ref_hidden.numpy(), heads=np.int64(heads), wq=attn.to_q.weight.numpy(),
               wk=attn.to_k.weight.numpy(), wv=attn.to_v.weight.numpy(), wo=attn.to_out[0].weight.numpy(),
               bo=attn.to_out[0].bias.numpy())
    for i, m in enumerate(attn_mask):
        res[f"attn_mask{i}"] = m.numpy()
    for flags in (0, 1, 6, 7):     # set A holds all eight; here: none, cross-frame only, intra+inter, all
        cf, intra, inter = bool(flags & 1), bool(flags & 2), bool(flags & 4)
        ctrl = dh.AttentionControl()
        proc = dh.FRESCOAttnProcessor2_0(chunks, ctrl)
        if intra:
            ctrl.stored_attn['decoder_attn'] = [ref_hidden.clone()]
            ctrl.enable_intraattn()
        if inter:
            ctrl.enable_interattn(paras)
        if cf:
            ctrl.enable_cfattn(attn_mask)
        res[f"out_{flags}"] = proc(attn, x.clone()).numpy()

    # warp_tensor: decoder feature (2 chunks) and image (Dilate(13) path)
    sal = torch.rand(N, 1, 32, 48)
    s_feat = torch.randn(2 * N, 6, 8, 12)
    s_img = torch.randn(N, 3, H, W)
    res.update(saliency=sal.numpy(), sample_feat=s_feat.numpy(), sample_img=s_img.numpy(),
               out_feat=fu.warp_tensor(s_feat.clone(), [fwd, bwd], [fo, bocc], sal, 2).numpy(),
               out_img=fu.warp_tensor(s_img.clone(), [fwd, bwd], [fo, bocc], sal, 1).numpy())

    # optimize_feature, 2 iterations, on an 8 x 12 plane
    Cc, h, w = 16, 8, 12
    sample = torch.randn(2 * N, Cc, h, w)
    other = sample + 0.5 * torch.randn(2 * N, Cc, h, w)
    lv = other.reshape(2 * N, Cc, h * w).transpose(1, 2)
    lv = lv / ((lv ** 2).sum(dim=2, keepdim=True) ** 0.5)
    target = torch.bmm(lv, lv.transpose(-1, -2))
    losses = []
    orig_step = torch.optim.Adam.step

    def rec_step(self, closure=None):
        r = orig_step(self, closure)
        losses.append(float(r))
        return r

    torch.optim.Adam.step = rec_step
    try:
        for tag, kw in {"full1": dict(iters=1), "full3": dict(iters=3)}.items():
            losses.clear()
            o = dh.optimize_feature(sample.clone(), [fwd, bwd], [fo, bocc], correlation_matrix=[target],
                                    intra_weight=1e2, **kw)
            res[f"opt_{tag}_out"] = o.detach().numpy()
            res[f"opt_{tag}_losses"] = np.array(losses, dtype=np.float64)
    finally:
        torch.optim.Adam.step = orig_step
    res.update(opt_sample=sample.numpy(), opt_target=target.numpy())
    save_npz("set_b", **res)
    print("golden fixture set B written to", HERE)


def scenario_gmflow_rect(matching):
    """``--only gmflow_rect``: GMFlow's global correlation (both directions and one) and the split-window attention
    (with and without shift) on a NON-SQUARE 24 x 40 grid: L = 960 tokens, 7.5 key tiles of 128 (the last one ragged);
    2 x 2 windows of 12 x 20 and shifted regions down to 6 x 10.  Inputs are fp16-representable, so the fp16 kernels
    read exactly these operands."""
    from gmflow import transformer as T
    g = torch.Generator().manual_seed(960)
    b, c, h, w = 2, 64, 24, 40
    f0 = (torch.randn(b, c, h, w, generator=g) * 1.5).half().float()
    f1 = (torch.roll(f0, shifts=(2, -3), dims=(2, 3)) + 0.5 * torch.randn(b, c, h, w, generator=g)).half().float()
    res = {"f0": f0.half().numpy(), "f1": f1.half().numpy(),
           "flow_bidir": matching.global_correlation_softmax(f0, f1, pred_bidir_flow=True)[0].numpy(),
           "flow_uni": matching.global_correlation_softmax(f0, f1, pred_bidir_flow=False)[0].numpy()}
    cw = 128
    q = (torch.randn(1, h * w, cw, generator=g) * 1.5).half().float()
    k = torch.randn(1, h * w, cw, generator=g).half().float()
    v = torch.randn(1, h * w, cw, generator=g).half().float()
    res.update(q=q.half().numpy(), k=k.half().numpy(), v=v.half().numpy(), h=h, w=w)
    res["out_split"] = T.single_head_split_window_attention(q, k, v, num_splits=2, with_shift=False, h=h, w=w).numpy()
    mask = T.generate_shift_window_attn_mask((h, w), h // 2, w // 2, h // 4, w // 4, device=torch.device("cpu"))
    res["out_shift"] = T.single_head_split_window_attention(q, k, v, num_splits=2, with_shift=True, h=h, w=w,
                                                            attn_mask=mask).numpy()
    save_npz("gmflow_rect", **res)
    print("gmflow_rect fixture written to", HERE)


def main():
    dh, fu, geometry, matching, ut = import_reference()
    torch.set_grad_enabled(False)
    if "--only" in sys.argv and sys.argv[sys.argv.index("--only") + 1] == "gmflow_rect":
        return scenario_gmflow_rect(matching)
    if "--set" in sys.argv and sys.argv[sys.argv.index("--set") + 1] == "b":
        return scenario_b(dh, fu, geometry, matching, ut)
    torch.manual_seed(0)
    torch.set_grad_enabled(False)

    # ---------------- geometry ----------------
    N, H, W = 4, 64, 64
    fwd, bwd = smooth_flows(N, H, W, 1, 3.0)
    fo, bo = geometry.forward_backward_consistency_check(fwd, bwd)
    feat = torch.randn(N, 5, H, W)
    save_npz("geometry", fwd=fwd.numpy(), bwd=bwd.numpy(), fwd_occ=fo.numpy(), bwd_occ=bo.numpy(),
                        feat=feat.numpy(), warped=geometry.flow_warp(feat, bwd).numpy())

    # ---------------- mapping (integer path) ----------------
    imgs = torch.rand(N, 3, H, W) * 2 - 1
    out = {}
    for tag, (hh, mag, sc) in {"a": (64, 3.0, 8.0), "b": (128, 10.0, 8.0), "c": (128, 14.0, 16.0)}.items():
        f_, b_ = smooth_flows(N, hh, hh, 7 + hh, mag)
        _, bo_ = geometry.forward_backward_consistency_check(f_, b_)
        im_ = torch.rand(N, 3, hh, hh) * 2 - 1
        fm, bm, im = fu.get_mapping_ind(b_, bo_, im_, scale=sc)
        mp, unl = fu.get_single_mapping_ind(b_[0:1], bo_[0:1], im_[0:2], scale=sc)
        out.update({f"{tag}_bwd_flows": b_.numpy(), f"{tag}_bwd_occs": bo_.numpy(), f"{tag}_imgs": im_.numpy(),
                    f"{tag}_scale": np.float32(sc), f"{tag}_fwd_map": fm.numpy(), f"{tag}_bwd_map": bm.numpy(),
                    f"{tag}_mask": im.numpy(), f"{tag}_single_map": mp.numpy(), f"{tag}_single_unl": unl.numpy()})
    save_npz("mapping", **out)

    # ---------------- attention, all 8 flag combinations ----------------
    C, heads, chunks = 80, 2, 2
    L = (H // 8) * (W // 8)
    attn = FakeAttn(C, heads, 3)
    x = torch.randn(chunks * N, L, C)
    ref_hidden = torch.randn(chunks * N, L, C)
    bocc = torch.clamp(bo + (torch.rand(N, H, W) > 0.8).float(), 0, 1)      # denser occlusion
    attn_mask = []
    for scale in [8.0, 16.0, 32.0]:   # formula of diffusion_hacked.py:935-938 evaluated by the reference's own ops
        o_ = F.interpolate(bocc[:-1].unsqueeze(1), scale_factor=1. / scale, mode='bilinear')
        attn_mask += [torch.cat((o_[0:1].reshape(1, -1) > -1, o_.reshape(o_.shape[0], -1) > 0.5), dim=0)]
    fm, bm, im = fu.get_mapping_ind(bwd, bocc, imgs, scale=8.0)
    paras = {"fwd_mappings": [fm], "bwd_mappings": [bm], "interattn_masks": [im]}
    res = {"x": x.numpy(), "ref_hidden": ref_hidden.numpy(), "heads": np.int64(heads),
           "wq": attn.to_q.weight.numpy(), "wk": attn.to_k.weight.numpy(), "wv": attn.to_v.weight.numpy(),
           "wo": attn.to_out[0].weight.numpy(), "bo": attn.to_out[0].bias.numpy(),
           "fwd_map": fm.numpy(), "bwd_map": bm.numpy(), "inter_mask": im.numpy()}
    for i, m in enumerate(attn_mask):
        res[f"attn_mask{i}"] = m.numpy()
    for flags in range(8):
        cf, intra, inter = bool(flags & 1), bool(flags & 2), bool(flags & 4)
        ctrl = dh.AttentionControl()
        proc = dh.FRESCOAttnProcessor2_0(chunks, ctrl)
        if intra:
            ctrl.stored_attn['decoder_attn'] = [ref_hidden.clone()]
            ctrl.enable_intraattn()
        if inter:
            ctrl.enable_interattn(paras)
        if cf:
            ctrl.enable_cfattn(attn_mask)
        res[f"out_{flags}"] = proc(attn, x.clone()).numpy()
    # cross-frame without a matching mask => frame-0 K/V (:236-237)
    ctrl = dh.AttentionControl()
    proc = dh.FRESCOAttnProcessor2_0(chunks, ctrl)
    ctrl.enable_cfattn([attn_mask[1]])
    res["out_cf_nomask"] = proc(attn, x.clone()).numpy()
    save_npz("attention", **res)

    # ---------------- warp_tensor ----------------
    sal = torch.rand(N, 1, 32, 32)
    s_feat = torch.randn(2 * N, 6, 8, 8)
    s_img = torch.randn(N, 3, H, W)
    save_npz("warp_tensor", fwd=fwd.numpy(), bwd=bwd.numpy(), fwd_occ=fo.numpy(),
        bwd_occ=bocc.numpy(), saliency=sal.numpy(), sample_feat=s_feat.numpy(), sample_img=s_img.numpy(),
        out_feat=fu.warp_tensor(s_feat.clone(), [fwd, bwd], [fo, bocc], sal, 2).numpy(),
        out_img=fu.warp_tensor(s_img.clone(), [fwd, bwd], [fo, bocc], sal, 1).numpy())

    # ---------------- optimize_feature (losses captured through Adam.step's return value) ----------------
    Cc, h, w = 16, 8, 8
    sample = torch.randn(2 * N, Cc, h, w)
    other = sample + 0.5 * torch.randn(2 * N, Cc, h, w)
    lv = other.reshape(2 * N, Cc, h * w).transpose(1, 2)
    lv = lv / ((lv ** 2).sum(dim=2, keepdim=True) ** 0.5)
    target = torch.bmm(lv, lv.transpose(-1, -2))
    losses = []
    orig_step = torch.optim.Adam.step

    def rec_step(self, closure=None):
        r = orig_step(self, closure)
        losses.append(float(r))
        return r

    torch.optim.Adam.step = rec_step
    opt = {"sample": sample.numpy(), "target": target.numpy(), "fwd": fwd.numpy(), "bwd": bwd.numpy(),
           "fwd_occ": fo.numpy(), "bwd_occ": bocc.numpy()}
    with torch.enable_grad():
        pass
    for tag, kw in {"full1": dict(iters=1), "full5": dict(iters=5),
                    "temporal3": dict(iters=3, correlation_matrix=[]),
                    "spatial3": dict(iters=3, optimize_temporal=False)}.items():
        losses.clear()
        kwargs = dict(correlation_matrix=[target], intra_weight=1e2)
        kwargs.update(kw)
        o = dh.optimize_feature(sample.clone(), [fwd, bwd], [fo, bocc], **kwargs)
        opt[f"{tag}_out"] = o.detach().numpy()
        opt[f"{tag}_losses"] = np.array(losses, dtype=np.float64)
    torch.optim.Adam.step = orig_step
    opt["adain_out"] = ut.adaptive_instance_normalization(other, sample).numpy()
    opt["adain_content"] = other.numpy()
    save_npz("optimize", **opt)

    # ---------------- GMFlow global correlation ----------------
    f0 = torch.randn(2, 16, 6, 8)
    f1 = torch.roll(f0, shifts=(1, -2), dims=(2, 3)) * 3 + 0.3 * torch.randn(2, 16, 6, 8)
    flow_b, prob_b = matching.global_correlation_softmax(f0, f1, pred_bidir_flow=True)
    flow_u, _ = matching.global_correlation_softmax(f0, f1, pred_bidir_flow=False)
    save_npz("gmflow_corr", f0=f0.numpy(), f1=f1.numpy(),
                        flow_bidir=flow_b.numpy(), flow_uni=flow_u.numpy(), prob_bidir=prob_b.numpy())
    scenario_gmflow_attention()
    scenario_ddpm_step()
    print("golden fixtures written to", HERE)


def scenario_ddpm_step():
    """src/pipe_FRESCO.py step() (no background smoothing) on a DDPM-1000 scaled-linear table, incl. repeat_noise, and
    the classifier-free-guidance combine of inference() (:212-215); Dilate(5) and Dilate(13) of src/utils.py:81-93."""
    import src.pipe_FRESCO as pf
    import src.utils as ut

    class Sched:
        def __init__(self):
            betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=torch.float32) ** 2
            self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
            self.one = torch.tensor(1.0)

        def previous_timestep(self, t):
            return t - 50

    class Pipe:
        scheduler = Sched()

    g = torch.Generator().manual_seed(77)
    N = 3
    raw = torch.randn(2 * N, 4, 16, 24, generator=g)
    sample = torch.randn(N, 4, 16, 24, generator=g)
    res = {"raw": raw.numpy(), "sample": sample.numpy(), "alphas_cumprod": Pipe.scheduler.alphas_cumprod.numpy()}
    u, t = raw.chunk(2)
    guided = u + 7.5 * (t - u)
    for tag, ts, rep in (("a", 700, False), ("b", 0, False), ("c", 350, True)):
        gen = torch.Generator().manual_seed(5)
        prev, x0 = pf.step(Pipe, guided, ts, sample, gen, repeat_noise=rep)
        noise = torch.randn(guided.shape, generator=torch.Generator().manual_seed(5))
        res.update({f"{tag}_t": ts, f"{tag}_prev": prev.numpy(), f"{tag}_x0": x0.numpy(), f"{tag}_noise": noise.numpy(),
                    f"{tag}_repeat": rep})
    m = (torch.rand(3, 1, 40, 56, generator=g) > 0.9).float()
    res.update(dil_in=m.numpy(), dil5=ut.Dilate(kernel_size=5, device="cpu")(m).numpy(),
               dil13=ut.Dilate(kernel_size=13, device="cpu")(m).numpy())
    save_npz("ddpm_step", **res)


def scenario_gmflow_attention():
    """GMFlow transformer attention (gmflow/transformer.py): plain, 2 x 2 windows, shifted 2 x 2 windows, and the
    flow-propagation attention, at C = 128 on a 32 x 32 grid (inputs are fp16-representable so that the fp16 kernels
    see exactly these operands)."""
    from gmflow import transformer as T
    g = torch.Generator().manual_seed(2024)
    b, h, w, c = 1, 32, 32, 128
    q = (torch.randn(b, h * w, c, generator=g) * 1.5).half().float()
    k = torch.randn(b, h * w, c, generator=g).half().float()
    v = torch.randn(b, h * w, c, generator=g).half().float()
    res = {"q": q.half().numpy(), "k": k.half().numpy(), "v": v.half().numpy(), "h": h, "w": w}
    res["out_full"] = T.single_head_full_attention(q, k, v).numpy()
    res["out_split"] = T.single_head_split_window_attention(q, k, v, num_splits=2, with_shift=False, h=h, w=w).numpy()
    mask = T.generate_shift_window_attn_mask((h, w), h // 2, w // 2, h // 4, w // 4, device=torch.device("cpu"))
    res["out_shift"] = T.single_head_split_window_attention(q, k, v, num_splits=2, with_shift=True, h=h, w=w,
                                                            attn_mask=mask).numpy()
    torch.manual_seed(7)
    ffa = T.FeatureFlowAttention(in_channels=c)
    with torch.no_grad():
        for prm in ffa.parameters():
            prm.copy_(prm.half().float())
        f0 = torch.randn(2, c, h, w, generator=g).half().float()
        flow = torch.randn(2, 2, h, w, generator=g) * 4
        res.update(ffa_f0=f0.half().numpy(), ffa_flow=flow.numpy(), ffa_out=ffa(f0, flow).numpy(),
                   ffa_wq=ffa.q_proj.weight.numpy(), ffa_bq=ffa.q_proj.bias.numpy(), ffa_wk=ffa.k_proj.weight.numpy(),
                   ffa_bk=ffa.k_proj.bias.numpy())
    save_npz("gmflow_attn", **res)


if __name__ == "__main__":
    main()
