"""Drop-in for ``gmflow.matching.global_correlation_softmax`` (gmflow/matching.py:7-36).

The all-pairs correlation volume [B, L, L] (and its transposed copy for bidirectional flow)
is never materialised: one wgmma kernel contracts feature tiles, applies an online softmax
and accumulates the expected (x, y) key coordinate directly.  The second return value of the
reference (``prob``, 0.5-1 GB at 512x512) is not produced -- its only caller discards it
(gmflow/gmflow.py:140 takes ``[0]``) -- so ``None`` is returned in its place.
"""
from __future__ import annotations

import torch

from . import ops


@torch.no_grad()
def global_correlation_softmax(feature0: torch.Tensor, feature1: torch.Tensor, pred_bidir_flow: bool = False):
    flow = ops.gmflow_global_corr_softmax(feature0.float().contiguous(), feature1.float().contiguous(),
                                          bool(pred_bidir_flow))
    return flow.to(feature0.dtype), None
