"""The propagation stage's frame blending on the GPU: drop-ins for video_blend.process_seq,
blender.histogram_blend.blend and blender.poisson_fusion.poisson_fusion (INTEGRATION.md).

Each frame between two keyframes mixes the two Ebsynth results (propagated from the previous and the next keyframe):
error masks chained through the cached backward flows, a histogram blend in cv2's 8-bit Lab, and a Poisson gradient
fusion whose least-squares system is solved exactly (to 1e-3, oracle/blend_bound.py) instead of by lsqr.  A sequence
is uploaded once and every frame of it runs in the same launches; only the mask chain is ordered.

cv2's BGR <-> Lab conversion is reproduced bit for bit by two 2^24-entry lookup tables (48 MB each on the device),
built once per process from cv2 itself.  cv2 is imported on first use (video_blend.py already needs it).
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import _lib as L
from . import ops

_LUTS: dict = {}


def _cv2():
    import cv2
    return cv2


def _device():
    return torch.device("cuda", torch.cuda.current_device())


def luts(device=None):
    """(BGR -> Lab, Lab -> BGR) uint8 [2^24, 3] on ``device``: cv2.cvtColor of the image holding every triple, entry
    (c0 << 16) | (c1 << 8) | c2 for the triple (c0, c1, c2)."""
    device = torch.device(device) if device is not None else _device()
    if device not in _LUTS:
        cv2 = _cv2()
        idx = np.arange(1 << 24, dtype=np.uint32)
        every = np.stack([idx >> 16, (idx >> 8) & 255, idx & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
        tables = [torch.from_numpy(cv2.cvtColor(every, code).reshape(-1, 3)).to(device)
                  for code in (cv2.COLOR_BGR2LAB, cv2.COLOR_LAB2BGR)]
        _LUTS[device] = tuple(tables)
    return _LUTS[device]


def _upload(imgs, what):
    arr = np.ascontiguousarray(np.asarray(imgs))
    if arr.dtype != np.uint8 or arr.shape[-1] != 3:
        raise L.FrescoError(f"{what}: expected uint8 BGR images [h, w, 3], got {arr.dtype} {list(arr.shape)}")
    return torch.from_numpy(arr).to(_device())


def _blend_frames(oa, ob, masks, weights, blend_gradient, grad_weight=(2.5, 0.5, 0.5)):
    """oa, ob uint8 BGR [F, h, w, 3], masks uint8 [F, h, w], weights fp64 [F, 2] (blend()'s weight1, weight2), all on
    the device -> BGR [F, h, w, 3]: the histogram blend, then with blend_gradient the Poisson fusion on top of it."""
    to_lab, to_bgr = luts(oa.device)
    la, lb = ops.blend_lut_gather(oa, to_lab), ops.blend_lut_gather(ob, to_lab)
    hist = ops.blend_lut_gather(ops.blend_histogram(la, lb, weights, masks=masks), to_bgr)
    if not blend_gradient:
        return hist
    target = ops.blend_lut_gather(hist, to_lab)       # poisson_fusion converts its BGR input back to Lab
    return ops.blend_lut_gather(ops.blend_poisson(target, la, lb, masks, grad_weight), to_bgr)


def histogram_blend(a: np.ndarray, b: np.ndarray, min_error: np.ndarray, weight1=0.5, weight2=0.5) -> np.ndarray:
    """blender/histogram_blend.blend: BGR uint8 images -> BGR uint8."""
    to_lab, to_bgr = luts()
    la, lb, le = (ops.blend_lut_gather(_upload(x, "histogram_blend")[None], to_lab) for x in (a, b, min_error))
    if not (la.shape == lb.shape == le.shape):
        raise L.FrescoError("histogram_blend: a, b and min_error must have one shape")
    weights = torch.tensor([[float(weight1), float(weight2)]], dtype=torch.float64, device=la.device)
    return ops.blend_lut_gather(ops.blend_histogram(la, lb, weights, lab_min_error=le), to_bgr)[0].cpu().numpy()


def poisson_fusion(blendI: np.ndarray, I1: np.ndarray, I2: np.ndarray, mask: np.ndarray,
                   grad_weight=[2.5, 0.5, 0.5]) -> np.ndarray:
    """blender/poisson_fusion.poisson_fusion: BGR uint8 blendI, I1, I2 and a pixel mask (> 0 takes I2's gradients)
    -> BGR uint8, from the exact least-squares solution."""
    to_lab, to_bgr = luts()
    tgt, la, lb = (ops.blend_lut_gather(_upload(x, "poisson_fusion")[None], to_lab) for x in (blendI, I1, I2))
    m = np.asarray(mask)
    if m.ndim != 2 or not (tgt.shape[1:3] == la.shape[1:3] == lb.shape[1:3] == m.shape):
        raise L.FrescoError("poisson_fusion: blendI, I1, I2 [h, w, 3] and mask [h, w] must agree")
    m = torch.from_numpy(np.ascontiguousarray(m > 0).astype(np.uint8))[None].to(tgt.device)
    return ops.blend_lut_gather(ops.blend_poisson(tgt, la, lb, m, grad_weight), to_bgr)[0].cpu().numpy()


def load_error(bin_path, img_shape):
    """video_blend.load_error: Ebsynth's error plane (int64 pixel count, then fp32 [h, w])."""
    with open(bin_path, "rb") as fp:
        raw = fp.read()
    n = int(np.frombuffer(raw[:8], dtype=np.int64)[0])
    if n != img_shape[0] * img_shape[1]:
        raise L.FrescoError(f"{bin_path}: {n} error values for a {img_shape[0]} x {img_shape[1]} frame")
    return np.frombuffer(raw[8:8 + 4 * n], dtype=np.float32).reshape(img_shape[0], img_shape[1])


def read_flow(path):
    """flow.flow_utils.read_flow: the backward flow the Ebsynth stage cached, fp32 [1, 2, h, w]."""
    if not os.path.exists(path):
        raise L.FrescoError(f"{path}: cached flow missing (the Ebsynth stage writes it; this module computes none)")
    return np.load(path)


def process_seq(video_sequence, i, blend_histogram=True, blend_gradient=True):
    """video_blend.process_seq: blends the frames of sequence ``i`` (between keyframes i and i+1) and writes them
    where the reference does.  The whole sequence is uploaded once and blended in one batched pass."""
    if not blend_histogram:
        # unreachable from video_blend.main, and the reference's own float path fails in cv2.cvtColor
        raise L.FrescoError("process_seq: blend_histogram=False is not supported")
    cv2 = _cv2()
    key1_img = cv2.imread(video_sequence.get_key_img(i))
    img_shape = key1_img.shape
    interval = video_sequence.interval(i)
    beg_id = video_sequence.get_sequence_beg_id(i)
    oas = video_sequence.get_output_sequence(i)
    obs = video_sequence.get_output_sequence(i, False)
    binas = [x.replace("jpg", "bin") for x in oas]
    binbs = [x.replace("jpg", "bin") for x in obs]
    obs = [obs[0]] + list(reversed(obs[1:]))
    flow_seq = video_sequence.get_flow_sequence(i)

    cv2.imwrite(video_sequence.get_blending_img(beg_id), key1_img)
    n = interval - 1
    if n <= 0:
        return
    h, w = img_shape[:2]
    oa = np.stack([cv2.imread(oas[k + 1]) for k in range(n)])
    ob = np.stack([cv2.imread(obs[k + 1]) for k in range(n)])
    dist1 = np.stack([load_error(binas[k + 1], img_shape) for k in range(n)])
    dist2 = np.stack([load_error(binbs[k + 1], img_shape) for k in range(n)])
    flows = np.zeros((n, 2, h, w), dtype=np.float32)
    for k in range(1, n):
        flows[k] = np.asarray(read_flow(flow_seq[k]), dtype=np.float32).reshape(2, h, w)
    dev = _device()
    masks = ops.blend_mask_chain(torch.from_numpy(dist1).to(dev), torch.from_numpy(dist2).to(dev),
                                 torch.from_numpy(flows).to(dev))
    weights = []
    for k in range(n):
        weight1 = k / (interval - 1) * (1 - 0) + 0
        weight2 = 1 - weight1
        weights.append((1 - weight1, 1 - weight2))
    weights = torch.tensor(weights, dtype=torch.float64, device=dev)
    res = _blend_frames(_upload(oa, "process_seq"), _upload(ob, "process_seq"), masks, weights, blend_gradient)
    res = res.cpu().numpy()
    for k in range(n):
        cv2.imwrite(video_sequence.get_blending_img(beg_id + k + 1), res[k])
