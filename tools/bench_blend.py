"""GPU time of the propagation stage's blending (fresco_b200/blend.py) per frame and per sequence, and the reference's
CPU solve on the same host as the baseline.  Prints one JSON line.

    python tools/bench_blend.py [--iters N] [--cpu-frames N]

Workloads: 512 x 896 and 896 x 512 frames (what resize_image(., 512) makes of a 16:9 video, landscape and portrait)
with keyframe intervals 5 and 20.  Timed from the mask chain to the last BGR gather, with the sequence resident on the
device (upload and file I/O excluded), by CUDA events after one warm-up pass; per-kernel times come from a separate
pass with ops.PROFILE on.  The CPU baseline is oracle.blend_oracle's restatement of the reference's per-frame work
(histogram blend in numpy, lsqr on the sparse system) on one 512 x 896 frame.  Writes nothing to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fresco_b200 import blend, ops  # noqa: E402
from oracle import blend_oracle as BO  # noqa: E402


def sequence(rng, n, h, w):
    """two Ebsynth-like results per frame (smooth colour fields with edges), error planes and small flows"""
    yy, xx = np.mgrid[:h, :w]
    base = np.stack([(xx * 0.3 + yy * 0.1) % 256, (yy * 0.4) % 256, (xx * 0.2 + 60) % 256], -1)
    imgs = np.clip(base[None, None] + rng.integers(-12, 13, (n, 2, h, w, 3)), 0, 255).astype(np.uint8)
    d = rng.random((2, n, h, w)).astype(np.float32)
    flows = rng.normal(0, 2, (n, 2, h, w)).astype(np.float32)
    return imgs[:, 0], imgs[:, 1], d[0], d[1], flows


def run(oa, ob, d1, d2, flows, weights):
    masks = ops.blend_mask_chain(d1, d2, flows)
    return blend._blend_frames(oa, ob, masks, weights, True)


def card():
    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out["power_limit_and_max_sm_clock"] = "not read: %s" % e
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--cpu-frames", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_blend.py measures the GPU kernels and needs a CUDA device")
    dev = torch.device("cuda")
    rng = np.random.default_rng(0)
    res = card()
    t = time.time()
    blend.luts(dev)
    torch.cuda.synchronize()
    res["lut_build_s"] = round(time.time() - t, 3)
    res["workloads"] = []
    for h, w in ((512, 896), (896, 512)):
        for interval in (5, 20):
            n = interval - 1
            arrs = [torch.from_numpy(x).to(dev) for x in sequence(rng, n, h, w)]
            weights = torch.tensor([(1 - k / (interval - 1), k / (interval - 1)) for k in range(n)],
                                   dtype=torch.float64, device=dev)
            run(*arrs, weights)                       # warm-up (and workspace growth)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                run(*arrs, weights)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.iters
            ops.PROFILE = []
            run(*arrs, weights)
            torch.cuda.synchronize()
            per_kernel = {}
            for tag, work, a, b, bound in ops.PROFILE:
                per_kernel[tag.split("_%d" % h)[0]] = per_kernel.get(tag.split("_%d" % h)[0], 0.0) + a.elapsed_time(b)
            ops.PROFILE = None
            res["workloads"].append({"h": h, "w": w, "interval": interval, "frames": n,
                                     "gpu_ms_per_sequence": round(ms, 3), "gpu_ms_per_frame": round(ms / n, 3),
                                     "per_call_ms": {k: round(v, 3) for k, v in per_kernel.items()},
                                     "cheby_steps": [ops.blend_cheby_iterations(h, w, g) for g in (2.5, 0.5)]})
            del arrs
    # CPU baseline: the reference's per-frame work on this host
    h, w = 512, 896
    oa, ob, d1, d2, _ = sequence(rng, args.cpu_frames, h, w)
    t = time.time()
    As = BO.construct_A(h, w)
    res["cpu_construct_A_s"] = round(time.time() - t, 3)
    th, tp = 0.0, 0.0
    for k in range(args.cpu_frames):
        mask = BO.error_mask(d1[k], d2[k], 0.5, 0.5)
        la, lb = BO.to_lab(oa[k]), BO.to_lab(ob[k])
        t = time.time()
        hl, _ = BO.histogram_blend_lab(la, lb, BO.min_error(la, lb, mask), 0.5, 0.5)
        hb = BO.to_bgr(hl)
        th += time.time() - t
        t = time.time()
        BO.to_bgr(BO.finalize(BO.poisson_lsqr(BO.to_lab(hb), la, lb, mask, As=As)))
        tp += time.time() - t
    res["cpu_512x896_histogram_s_per_frame"] = round(th / args.cpu_frames, 3)
    res["cpu_512x896_lsqr_poisson_s_per_frame"] = round(tp / args.cpu_frames, 3)
    res["cpu"] = os.uname().machine + " x%d" % os.cpu_count()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
