"""Generate the ``blend`` golden set by running the REAL reference's propagation-stage blending (video_blend.py and its
blender modules) on CPU.

    python tests/golden/make_blend_golden.py --reference /path/to/FRESCO

Outputs ``blend.npz`` (in parts below 1 MB, see make_golden.save_npz) next to this script, consumed by
tests/test_blend_oracle.py (oracle vs reference) and tests/test_gpu_blend.py.
"""
import os
import sys
import types

import numpy as np
import torch

from make_golden import HERE, REF, save_npz


def import_blend_reference():
    """video_blend.py and its blender modules.  flow/flow_utils.py builds GMFlow on CUDA at import
    (``flow_calc = FlowCalc()``); it is loaded with that one object left unconstructed -- the blending only reads cached
    flows through it.  src/video_util.py (video encoding, not used here) is stubbed."""
    eb = os.path.join(REF, "src", "ebsynth")
    os.chdir(REF)
    for d in (REF, eb):
        if d not in sys.path:
            sys.path.insert(0, d)
    path = os.path.join(eb, "flow", "flow_utils.py")
    src = open(path).read().replace("flow_calc = FlowCalc()", "flow_calc = FlowCalc.__new__(FlowCalc)")
    pkg = types.ModuleType("flow")
    pkg.__path__ = [os.path.dirname(path)]
    mod = types.ModuleType("flow.flow_utils")
    mod.__file__ = path
    sys.modules["flow"], sys.modules["flow.flow_utils"] = pkg, mod
    exec(compile(src, path, "exec"), mod.__dict__)
    vu = types.ModuleType("src.video_util")
    vu.frame_to_video = lambda *a, **k: None
    sys.modules["src.video_util"] = vu
    import video_blend  # noqa
    return video_blend


def blend_case(rng, h, w, interval, family):
    """Two Ebsynth results per frame with strong edges (saturated blocks, so gradients pass the +-100 clip and the
    solution the [0, 255] clip), error planes that make the error masks all 0 / all 1 / a checkerboard / blocks, and
    backward flows with half-integer components and samples past the border."""
    n = interval - 1
    blocks = rng.integers(0, 2, (n, 2, (h + 7) // 8, (w + 7) // 8, 3)) * 255
    base = np.repeat(np.repeat(blocks, 8, 2), 8, 3)[:, :, :h, :w].astype(np.int64)
    ramp = (np.arange(w)[None, :, None] * 3 + np.arange(h)[:, None, None] * 2) % 96
    imgs = np.clip(base + ramp - 48 + rng.integers(-24, 25, base.shape), 0, 255).astype(np.uint8)
    yy, xx = np.mgrid[:h, :w]
    if family == "zero":
        d1, d2 = np.zeros((n, h, w)), np.ones((n, h, w))
    elif family == "one":
        d1, d2 = np.ones((n, h, w)), np.zeros((n, h, w))
    elif family == "checker":
        c = ((yy + xx) % 2).astype(np.float64)
        d1, d2 = np.repeat(c[None], n, 0), np.repeat(1 - c[None], n, 0)
    else:
        cells = rng.random((n, (h + 5) // 6, (w + 5) // 6))
        d1 = np.repeat(np.repeat(cells, 6, 1), 6, 2)[:, :h, :w]
        d2 = 1 - d1
    d1 = (d1 * rng.uniform(0.5, 2.0, (n, h, w))).astype(np.float32)
    d2 = (d2 * rng.uniform(0.5, 2.0, (n, h, w))).astype(np.float32)
    flows = (rng.integers(-6, 7, (n, 2, h, w)) / 2.0).astype(np.float32)
    flows[:, :, ::7] = rng.normal(0, 4, flows[:, :, ::7].shape)          # non-grid samples
    flows[:, 0, :, :2] = -5.0                                            # past the left border
    flows[:, 1, -2:] = 3.5                                               # past the bottom border
    return imgs[:, 0], imgs[:, 1], d1, d2, flows


def scenario_blend():
    """The propagation stage's blending, from the reference's own functions: g_error_mask and flow_calc.warp (the mask
    chain of process_seq), assemble_min_error_img, histogram_blend.blend, and poisson_fusion with its Lab result before
    LAB2BGR and lsqr's solution captured; then process_seq itself on one on-disk sequence."""
    import tempfile
    import cv2
    vb = import_blend_reference()
    from blender import poisson_fusion as PF
    from blender.video_sequence import VideoSequence
    import scipy.sparse.linalg as sla
    rng = np.random.default_rng(77)
    cases = [("a", 48, 80, 2, "zero"), ("b", 48, 80, 4, "checker"), ("c", 64, 64, 6, "blocky"),
             ("d", 40, 72, 4, "one"), ("e", 37, 53, 6, "blocky"), ("f", 64, 64, 4, "checker")]
    captured = {}
    real_lsqr, real_cvt = sla.lsqr, cv2.cvtColor

    def lsqr(A, b, *a, **k):
        out = real_lsqr(A, b, *a, **k)
        captured.setdefault("lsqr", []).append(out[0])
        return out

    class Cv2:   # poisson_fusion's cv2 with its final LAB2BGR operand recorded
        def __getattr__(self, name):
            return getattr(cv2, name)

        def cvtColor(self, img, code):
            if code == cv2.COLOR_LAB2BGR:
                captured["lab"] = img.copy()
            return real_cvt(img, code)

    PF.cv2 = Cv2()
    PF.scipy.sparse.linalg.lsqr = lsqr
    res = {}
    for tag, h, w, interval, family in cases:
        oa, ob, d1, d2, flows = blend_case(rng, h, w, interval, family)
        out = {"oa": oa, "ob": ob, "dist1": d1, "dist2": d2, "flows": flows, "interval": interval}
        masks, mes, hists, labs, lsqrs, finals, p_mask = [], [], [], [], [], [], None
        for k in range(interval - 1):
            w1 = k / (interval - 1) * (1 - 0) + 0
            w2 = 1 - w1
            mask = vb.g_error_mask(d1[k], d2[k], w1, w2)
            if p_mask is not None:
                p_mask = vb.flow_calc.warp(p_mask, torch.from_numpy(flows[k][None]), "nearest")
                mask = p_mask | mask
            p_mask = mask
            me = vb.assemble_min_error_img(oa[k], ob[k], mask)
            hb = vb.histogram_blend.blend(oa[k], ob[k], me, 1 - w1, 1 - w2)
            captured.clear()
            final = PF.poisson_fusion(hb, oa[k], ob[k], mask)
            target = cv2.cvtColor(hb, cv2.COLOR_BGR2LAB).astype(float)
            lsqrs.append(np.stack([captured["lsqr"][c].reshape(h, w) + target[:, :, c].reshape(-1).mean()
                                   for c in range(3)]).astype(np.float32))
            masks.append(mask.astype(np.uint8))
            mes.append(me)
            hists.append(hb)
            labs.append(captured["lab"])
            finals.append(final)
        out.update(masks=np.stack(masks), min_error=np.stack(mes), hist=np.stack(hists), lab=np.stack(labs),
                   lsqr=np.stack(lsqrs), final=np.stack(finals))
        res.update({f"{tag}_{k}": v for k, v in out.items()})
    res["cases"] = np.array([c[0] for c in cases])

    # process_seq end to end: keyframes 3 and 7 of a 40 x 72 video, Ebsynth results written losslessly (PNG bytes
    # under the .jpg names Ebsynth uses; cv2.imread reads by content), error planes as Ebsynth writes them
    # (int64 count, fp32 plane), flows as the cached .npy files; the blended frames recorded before imwrite encodes them
    h, w, beg, end = 40, 72, 3, 7
    interval = end - beg
    oa, ob, d1, d2, flows = blend_case(rng, h, w, interval + 1, "blocky")
    key = oa[0]
    written, real_imwrite = {}, cv2.imwrite
    with tempfile.TemporaryDirectory() as tmp:
        seq = VideoSequence(tmp, [beg, end], "video", "keys0", "tmp", "%04d.png", "%04d.png")
        os.makedirs(os.path.join(tmp, "keys0"), exist_ok=True)
        real_imwrite(seq.get_key_img(0), key)

        def put(path, img):
            with open(path, "wb") as f:
                f.write(cv2.imencode(".png", img)[1].tobytes())

        def put_err(path, d):
            with open(path, "wb") as f:
                f.write(np.int64(h * w).tobytes() + d.astype(np.float32).tobytes())

        fwd, bwd = seq.get_output_sequence(0), seq.get_output_sequence(0, False)
        for j in range(interval):
            put(fwd[j], oa[j])
            put(bwd[j], ob[j])
            put_err(fwd[j].replace("jpg", "bin"), d1[j])
            put_err(bwd[j].replace("jpg", "bin"), d2[j])
        for j, path in enumerate(seq.get_flow_sequence(0)):
            np.save(path, flows[j][None])

        def imwrite(path, img, *a):
            written[os.path.basename(path)] = img.copy()
            return real_imwrite(path, img, *a)
        cv2.imwrite = imwrite
        try:
            vb.process_seq(seq, 0, True, True)
        finally:
            cv2.imwrite = real_imwrite
    res.update(seq_key=key, seq_fwd=oa[:interval], seq_bwd=ob[:interval], seq_err_fwd=d1[:interval].astype(np.float32),
               seq_err_bwd=d2[:interval].astype(np.float32), seq_flows=flows[:interval - 1], seq_beg=beg, seq_end=end,
               seq_out=np.stack([written["%04d.jpg" % i] for i in range(beg, end)]))
    save_npz("blend", **res)
    print("blend fixture written to", HERE)


if __name__ == "__main__":
    if REF is None:
        raise SystemExit("usage: make_blend_golden.py --reference /path/to/FRESCO")
    scenario_blend()
