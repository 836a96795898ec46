"""CPU restatement of the propagation stage's frame blending (video_blend.py:172-255, blender/histogram_blend.py,
blender/poisson_fusion.py) in numpy, torch CPU and cv2, with the EXACT least-squares solution of the Poisson system.

CHECKER ONLY (see ``oracle/__init__``).  Images are BGR uint8 [h, w, 3] as cv2 reads them; Lab is cv2's 8-bit Lab.

* ``error_mask`` / ``warp_nearest`` / ``mask_chain``: the numba mask and its propagation through torch's CPU
  ``grid_sample`` (nearest, align_corners=True, zero padding), as the reference computes them.
* ``histogram_blend_lab``: blend() up to the Lab image it converts back to BGR.
* ``poisson_exact``: the least-squares solution of poisson_fusion's system [w Gx; w Gy; I] u ~ [w gx; w gy; im] per
  channel, from its normal equations M u = b, M = I + w^2 (L_h (x) I + I (x) L_w), diagonalised by the 2-D DCT-II
  (L_n, the path-graph Laplacian, has eigenvectors cos(pi k (i + 1/2) / n) and eigenvalues 4 sin^2(pi k / 2n)).
* ``poisson_lsqr``: the reference's own formulation (sparse A, scipy lsqr, mean subtracted), for timing and for the
  goldens' comparison of lsqr's iterate with the exact solution.
"""
from __future__ import annotations

import numpy as np
import scipy.fft
import scipy.sparse
import scipy.sparse.linalg

GRAD_WEIGHT = (2.5, 0.5, 0.5)
GRAD_CLIP = 100.0


def cv2():
    import cv2 as _cv2
    return _cv2


def to_lab(bgr):
    return cv2().cvtColor(bgr, cv2().COLOR_BGR2LAB)


def to_bgr(lab):
    return cv2().cvtColor(lab, cv2().COLOR_LAB2BGR)


def seq_weights(interval):
    """(weight1, weight2) of frame k = 0 .. interval-2 as process_seq computes them (lb = 0, ub = 1)."""
    out = []
    for k in range(interval - 1):
        w1 = k / (interval - 1) * (1 - 0) + 0
        out.append((w1, 1 - w1))
    return out


def error_mask(dist1, dist2, weight1, weight2):
    """g_error_mask: 0 where weight1 dist1 < weight2 dist2 (fp64), else 1; all 0 at weight1 == 0, all 1 at
    weight2 == 0.  uint8 [h, w]."""
    m = np.where(weight1 * dist1.astype(np.float64) < weight2 * dist2.astype(np.float64), 0, 1).astype(np.uint8)
    if weight1 == 0:
        m[:] = 0
    elif weight2 == 0:
        m[:] = 1
    return m


def warp_nearest(mask, flow):
    """flow_calc.warp(mask, flow, 'nearest'): flow fp32 [2, h, w] or [1, 2, h, w] (backward flow, x then y)."""
    import torch
    import torch.nn.functional as F
    flow = torch.as_tensor(np.asarray(flow, dtype=np.float32)).reshape(1, 2, *mask.shape)
    h, w = mask.shape
    y, x = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    grid = torch.stack([x, y], 0).float()[None] + flow
    xg = 2 * grid[:, 0] / (w - 1) - 1
    yg = 2 * grid[:, 1] / (h - 1) - 1
    img = torch.from_numpy(mask.astype(np.int8))[None, None].float()
    out = F.grid_sample(img, torch.stack([xg, yg], -1), mode="nearest", padding_mode="zeros", align_corners=True)
    return out.to(torch.int8)[0, 0].numpy().astype(np.uint8)


def mask_chain(dist1s, dist2s, flows, interval):
    """The masks of frames 0 .. interval-2: error mask OR the previous frame's mask warped by flows[k] (k >= 1)."""
    masks, prev = [], None
    for k, (w1, w2) in enumerate(seq_weights(interval)):
        m = error_mask(dist1s[k], dist2s[k], w1, w2)
        if prev is not None:
            m = warp_nearest(prev, flows[k]) | m
        masks.append(m)
        prev = m
    return np.stack(masks)


def min_error(a, b, mask):
    return np.where(mask[..., None] > 0, b, a)


def histogram_blend_lab(la, lb, le, weight1=0.5, weight2=0.5):
    """blend() on Lab operands, returning its uint8 Lab result before LAB2BGR (numpy in fp64, as the reference)."""
    def transform(img, means, stds, t_means, t_stds):
        x = img.astype(np.float32)
        return (x - means.reshape(1, 1, 3)) * t_stds.reshape(1, 1, 3) / stds.reshape(1, 1, 3) + t_means.reshape(1, 1, 3)

    t_mean = np.ones([3], dtype=np.float32) * (0.5 * 256)
    t_std = np.ones([3], dtype=np.float32) * ((1 / 36) * 256)
    a = transform(la, np.mean(la, axis=(0, 1)), np.std(la, axis=(0, 1)), t_mean, t_std)
    b = transform(lb, np.mean(lb, axis=(0, 1)), np.std(lb, axis=(0, 1)), t_mean, t_std)
    ab = (a * weight1 + b * weight2 - 0.5 * 256) / 0.5 + 0.5 * 256
    pre = transform(ab, np.mean(ab, axis=(0, 1)), np.std(ab, axis=(0, 1)), np.mean(le, axis=(0, 1)),
                    np.std(le, axis=(0, 1)))
    return np.clip(np.round(pre), 0, 255).astype(np.uint8), pre


def histogram_blend(a, b, min_error_img, weight1=0.5, weight2=0.5):
    lab, _ = histogram_blend_lab(to_lab(a), to_lab(b), to_lab(min_error_img), weight1, weight2)
    return to_bgr(lab)


def gradients(la, lb, mask):
    """gx, gy fp64 [h, w, 3]: forward differences along rows / columns of la (mask 0) or lb (mask 1), zero on the
    last row / column, clipped to +-100."""
    ia, ib = la.astype(np.float64), lb.astype(np.float64)
    m = (mask > 0).astype(np.float64)[:, :, None]
    gx = np.zeros_like(ia)
    gy = np.zeros_like(ia)
    gx[:-1] = (ia[:-1] - ia[1:]) * (1 - m[:-1]) + (ib[:-1] - ib[1:]) * m[:-1]
    gy[:, :-1] = (ia[:, :-1] - ia[:, 1:]) * (1 - m[:, :-1]) + (ib[:, :-1] - ib[:, 1:]) * m[:, :-1]
    return np.clip(gx, -GRAD_CLIP, GRAD_CLIP), np.clip(gy, -GRAD_CLIP, GRAD_CLIP)


def normal_rhs(target_lab, gx, gy, weight, c):
    """b = im + w^2 (Gx^T gx + Gy^T gy) for channel c (fp64 [h, w])."""
    div = gx[:, :, c].copy()
    div[1:] -= gx[:-1, :, c]
    div += gy[:, :, c]
    div[:, 1:] -= gy[:, :-1, c]
    return target_lab[:, :, c].astype(np.float64) + weight * weight * div


def laplace_eigs(n):
    return 4.0 * np.sin(np.pi * np.arange(n) / (2.0 * n)) ** 2


def solve_dct(rhs, weight):
    """M^-1 rhs for M = I + w^2 (L_h (x) I + I (x) L_w), by the orthonormal 2-D DCT-II."""
    h, w = rhs.shape
    lam = 1.0 + weight * weight * (laplace_eigs(h)[:, None] + laplace_eigs(w)[None, :])
    return scipy.fft.idctn(scipy.fft.dctn(rhs, type=2, norm="ortho") / lam, type=2, norm="ortho")


def poisson_exact(target_lab, la, lb, mask, grad_weight=GRAD_WEIGHT):
    """The exact least-squares solution, fp64 [3, h, w]."""
    gx, gy = gradients(la, lb, mask)
    return np.stack([solve_dct(normal_rhs(target_lab, gx, gy, grad_weight[c], c), grad_weight[c]) for c in range(3)])


def finalize(u):
    """poisson_fusion's last steps on a [3, h, w] solution: clip to [0, 255], truncate to uint8 -> Lab [h, w, 3]."""
    return np.clip(np.moveaxis(u, 0, -1), 0, 255).astype(np.uint8)


def poisson_fusion(blendI, I1, I2, mask, grad_weight=GRAD_WEIGHT):
    return to_bgr(finalize(poisson_exact(to_lab(blendI), to_lab(I1), to_lab(I2), mask, grad_weight)))


def construct_A(h, w, grad_weight=GRAD_WEIGHT):
    """[w Gx; w Gy; I] per channel (poisson_fusion.construct_A), vectorised."""
    n = h * w
    idx = np.arange(n).reshape(h, w)
    rx = idx[:-1].ravel()
    ry = idx[:, :-1].ravel()
    gx = scipy.sparse.coo_array((np.r_[np.ones(rx.size), -np.ones(rx.size)], (np.r_[rx, rx], np.r_[rx, rx + w])),
                                shape=(n, n)).tocsc()
    gy = scipy.sparse.coo_array((np.r_[np.ones(ry.size), -np.ones(ry.size)], (np.r_[ry, ry], np.r_[ry, ry + 1])),
                                shape=(n, n)).tocsc()
    eye = scipy.sparse.identity(n, format="csc")
    return [scipy.sparse.vstack([gx * g, gy * g, eye]).tocsr() for g in grad_weight]


def poisson_lsqr(target_lab, la, lb, mask, grad_weight=GRAD_WEIGHT, As=None):
    """The reference's solve: lsqr on [w Gx; w Gy; I] u ~ [w gx; w gy; im - mean] per channel, fp64 [3, h, w]."""
    h, w = mask.shape
    As = As if As is not None else construct_A(h, w, grad_weight)
    gx, gy = gradients(la, lb, mask)
    out = []
    for c in range(3):
        im = target_lab[:, :, c].astype(np.float64).reshape(-1)
        mean = im.mean()
        b = np.concatenate([gx[:, :, c].ravel() * grad_weight[c], gy[:, :, c].ravel() * grad_weight[c], im - mean])
        out.append(scipy.sparse.linalg.lsqr(As[c], b)[0].reshape(h, w) + mean)
    return np.stack(out)


def blend_sequence(oas, obs, dist1s, dist2s, flows, interval, blend_gradient=True):
    """process_seq's frames 1 .. interval-1 on arrays: oas[k], obs[k] are the two Ebsynth results of frame k + 1
    (obs already in forward order), dist*s[k] their error planes, flows[k] the backward flow of pair (k, k+1).
    Returns masks, the histogram results (Lab, BGR) and, with blend_gradient, the exact Poisson solutions and the
    final BGR frames."""
    masks = mask_chain(dist1s, dist2s, flows, interval)
    res = {"masks": masks, "hist_lab": [], "hist": [], "solution": [], "final": []}
    for k, (w1, w2) in enumerate(seq_weights(interval)):
        la, lb = to_lab(oas[k]), to_lab(obs[k])
        hl, _ = histogram_blend_lab(la, lb, min_error(la, lb, masks[k]), 1 - w1, 1 - w2)
        hb = to_bgr(hl)
        res["hist_lab"].append(hl)
        res["hist"].append(hb)
        if blend_gradient:
            u = poisson_exact(to_lab(hb), la, lb, masks[k])
            res["solution"].append(u)
            res["final"].append(to_bgr(finalize(u)))
    return {k: (np.stack(v) if len(v) else None) for k, v in res.items()}
