"""Drop-in for the FRESCO hook surface of the reference's ``src/diffusion_hacked.py``.

Same public names, arguments and error behaviour as the reference (SURVEY 8b):

* ``AttentionControl``          (src/diffusion_hacked.py:23-137)
* ``FRESCOAttnProcessor2_0``    (:142-387)   diffusers attn-processor ``__call__``
* ``apply_FRESCO_attn``         (:390-403)
* ``optimize_feature``          (:416-488)
* ``my_forward`` / ``apply_FRESCO_opt`` / ``disable_FRESCO_opt``   (:491-831)

The arithmetic of the hot path runs in libfresco_b200.so (hand-written sm_90a
kernels bound through ctypes); there is no PyTorch fallback for it.  What stays
in torch is what the scope table leaves there: the Linear projections
(to_q/k/v/out, cuBLAS) and small per-call tensor preparation.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

from . import ops
from ._lib import FrescoError
from .dist import ShardedFRESCOAttention, batch_layout, shard_layout, unpack
from .flow_utils import adjoint_csr, clear_prep_cache, resize_flows_occs, warp_tensor


# =============================================================================
# PART I -- FRESCO attention
# =============================================================================
class AttentionControl:
    """State of FRESCO-guided attention: which of the three guidance modes are
    active, the per-batch masks / mappings and the stored reference features.
    Method names and semantics follow src/diffusion_hacked.py:23-137."""

    def __init__(self):
        self.stored_attn = self.get_empty_store()
        self.store = False
        self.index = 0
        self.attn_mask = None
        self.interattn_paras = None
        self.use_interattn = False
        self.use_cfattn = False
        self.use_intraattn = False
        self.intraattn_bias = 0
        self.intraattn_scale_factor = 0.2
        self.interattn_scale_factor = 0.2
        # device-side caches derived from attn_mask / interattn_paras (kernel operands)
        self._kv_index_cache: Dict[int, torch.Tensor] = {}
        self._traj_cache: Dict[int, tuple] = {}

    @staticmethod
    def get_empty_store():
        return {"decoder_attn": []}

    def clear_store(self):
        self.stored_attn = self.get_empty_store()
        self.disable_intraattn()

    # ---- store the reference pass' self-attention inputs (spatial guidance)
    def enable_store(self):
        self.store = True

    def disable_store(self):
        self.store = False

    # ---- spatial-guided attention
    def enable_intraattn(self):
        self.index = 0
        self.use_intraattn = len(self.stored_attn["decoder_attn"]) > 0
        self.disable_store()

    def disable_intraattn(self):
        self.index = 0
        self.use_intraattn = False
        self.disable_store()

    # ---- cross-frame attention
    def disable_cfattn(self):
        self.use_cfattn = False

    def enable_cfattn(self, attn_mask=None):
        if attn_mask:
            if attn_mask is not self.attn_mask:          # same object again (next denoise step): keep the derived indices
                self.attn_mask = attn_mask
                self._kv_index_cache = {}
            self.use_cfattn = True
        elif self.attn_mask:
            self.use_cfattn = True
        else:
            print("Warning: no valid cross-frame attention parameters available!")
            self.disable_cfattn()

    # ---- temporal-guided attention
    def disable_interattn(self):
        self.use_interattn = False

    def enable_interattn(self, interattn_paras=None):
        if interattn_paras:
            if interattn_paras is not self.interattn_paras:
                self.interattn_paras = interattn_paras
                self._traj_cache = {}
            self.use_interattn = True
        elif self.interattn_paras:
            self.use_interattn = True
        else:
            print("Warning: no valid temporal-guided attention parameters available!")
            self.disable_interattn()

    def disable_controller(self):
        self.disable_intraattn()
        self.disable_interattn()
        self.disable_cfattn()

    def enable_controller(self, interattn_paras=None, attn_mask=None):
        self.enable_intraattn()
        self.enable_interattn(interattn_paras)
        self.enable_cfattn(attn_mask)

    def forward(self, context):
        if self.store:
            self.stored_attn["decoder_attn"].append(context.detach())
        stored = self.stored_attn["decoder_attn"]
        if self.use_intraattn and len(stored) > 0:
            ref = stored[self.index]
            self.index += 1
            if self.index >= len(stored):
                self.index = 0
                self.disable_store()
            return ref
        return context

    def __call__(self, context):
        return self.forward(context)

    # ---- kernel operands ------------------------------------------------------
    def kv_indices(self, tokens: int) -> Optional[torch.Tensor]:
        """int32 row indices (row-major over (frame, token)) of the K/V tokens the
        mask with ``shape[1] == tokens`` selects; None if no mask matches
        (src/diffusion_hacked.py:229-232, :239)."""
        if self.attn_mask is None:
            return None
        if tokens not in self._kv_index_cache:
            chosen = None
            for m in self.attn_mask:
                if m.shape[1] == tokens:
                    chosen = m
            self._kv_index_cache[tokens] = (
                None if chosen is None
                else torch.nonzero(chosen.reshape(-1), as_tuple=False).reshape(-1).to(torch.int32).contiguous())
        return self._kv_index_cache[tokens]

    def trajectories(self, tokens: int):
        """(fwd_map int64 [N, L], mask uint8 [L, N, N]) for the mapping whose
        ``shape[2] == tokens`` (src/diffusion_hacked.py:315-319)."""
        if tokens not in self._traj_cache:
            found = None
            paras = self.interattn_paras
            for i, f in enumerate(paras["fwd_mappings"]):
                if f.shape[2] == tokens:
                    found = (f[:, 0].contiguous().to(torch.int64),
                             paras["interattn_masks"][i][:, 0].to(torch.uint8).contiguous())
            self._traj_cache[tokens] = found
        return self._traj_cache[tokens]


class FRESCOAttnProcessor2_0:
    """diffusers attn-processor that turns decoder self-attention into FRESCO
    attention (spatial-guided -> cross-frame -> temporal-guided).
    Call contract of src/diffusion_hacked.py:169-387."""

    def __init__(self, unet_chunk_size=2, controller=None, shard=None):
        if not hasattr(F, "scaled_dot_product_attention"):
            raise ImportError("AttnProcessor2_0 requires PyTorch 2.0, to use it, please upgrade PyTorch to 2.0.")
        self.unet_chunk_size = unet_chunk_size
        self.controller = controller
        # optional frame sharding over the GPUs of one box: (world, rank, process_group); see fresco_b200/dist.py
        self.shard = shard
        self._sharded = None
        self._layout = None
        # (world, rank, group, chunks) the sharded layer runs on: the frame layout of ``shard`` until a batch says otherwise
        self._layer_key = None if shard is None else unpack(shard) + (unet_chunk_size,)

    def set_batch_frames(self, n_frames: int) -> None:
        """Tell a sharded processor the frame count of the keyframe batch it runs on (``inference`` and
        ``get_intraframe_paras`` do): with fewer frames than ranks it holds one CFG half and exchanges within the ranks
        of that half (``dist.shard_layout``).  Without a call, the frame layout is assumed."""
        if self.shard is None:
            return
        layout = shard_layout(n_frames, self.shard)
        key = (layout.world, layout.rank, layout.group, layout.chunks(self.unet_chunk_size))
        if key != self._layer_key:
            self._sharded = None
        self._layout, self._layer_key = layout, key

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None):
        residual = hidden_states
        if attn.spatial_norm is not None:
            hidden_states = attn.spatial_norm(hidden_states, temb)
        input_ndim = hidden_states.ndim
        if input_ndim == 4:
            batch_size, channel, height, width = hidden_states.shape
            hidden_states = hidden_states.view(batch_size, channel, height * width).transpose(1, 2)
        batch_size, sequence_length, _ = (
            hidden_states.shape if encoder_hidden_states is None else encoder_hidden_states.shape)
        if attention_mask is not None:
            attention_mask = attn.prepare_attention_mask(attention_mask, sequence_length, batch_size)
            attention_mask = attention_mask.view(batch_size, attn.heads, -1, attention_mask.shape[-1])
        if attn.group_norm is not None:
            hidden_states = attn.group_norm(hidden_states.transpose(1, 2)).transpose(1, 2)

        ctrl = self.controller
        query = attn.to_q(hidden_states)
        crossattn = encoder_hidden_states is not None
        if not crossattn:
            encoder_hidden_states = hidden_states
            if ctrl and ctrl.store:
                ctrl(hidden_states.detach().clone())
        elif attn.norm_cross:
            encoder_hidden_states = attn.norm_encoder_hidden_states(encoder_hidden_states)
        key = attn.to_k(encoder_hidden_states)
        value = attn.to_v(encoder_hidden_states)
        heads = attn.heads
        head_dim = key.shape[-1] // heads

        if crossattn or attention_mask is not None:
            # not a FRESCO path (text cross-attention): plain SDPA, exactly as the reference does
            q = query.view(batch_size, -1, heads, head_dim).transpose(1, 2)
            k = key.view(batch_size, -1, heads, head_dim).transpose(1, 2)
            v = value.view(batch_size, -1, heads, head_dim).transpose(1, 2)
            out = F.scaled_dot_product_attention(q, k, v, attn_mask=attention_mask, dropout_p=0.0, is_causal=False)
            out = out.transpose(1, 2).reshape(batch_size, -1, heads * head_dim).to(query.dtype)
        else:
            out = self._fresco_self_attention(attn, query, key, value, encoder_hidden_states, heads, head_dim)

        out = attn.to_out[0](out)
        out = attn.to_out[1](out)
        if input_ndim == 4:
            out = out.transpose(-1, -2).reshape(batch_size, channel, height, width)
        if attn.residual_connection:
            out = out + residual
        return out / attn.rescale_output_factor

    # ------------------------------------------------------------------------
    def _fresco_self_attention(self, attn, query, key, value, hidden_states, heads, head_dim):
        ctrl = self.controller
        in_dtype = query.dtype
        q = query.to(torch.float16).contiguous()
        k = key.to(torch.float16).contiguous()
        v = value.to(torch.float16).contiguous()
        if self.shard is not None and ctrl is not None:
            if self._sharded is None:
                world, rank, group, chunks = self._layer_key
                self._sharded = ShardedFRESCOAttention(ctrl, world, rank, chunks, group)
            ref_q = ref_k = None
            if ctrl.use_intraattn:
                ref = ctrl(None)
                assert ref.shape == hidden_states.shape
                ref_q = attn.to_q(ref).to(torch.float16).contiguous()
                ref_k = attn.to_k(ref).to(torch.float16).contiguous()
            return self._sharded(q, k, v, heads, ref_q=ref_q, ref_k=ref_k).to(in_dtype)
        B, L, C = q.shape
        chunks = self.unet_chunk_size
        inv_sqrt_d = 1.0 / math.sqrt(head_dim)

        # cross-frame K/V: frame 0 + occluded tokens, shared by every query frame (:225-247)
        q_per_kv = 1
        k_att, v_att = k, v
        if ctrl and ctrl.use_cfattn:
            frames = B // chunks
            idx = ctrl.kv_indices(L)
            if idx is None:                       # no mask for this resolution: everybody attends frame 0
                k_att = k.view(chunks, frames, L, C)[:, 0].contiguous()
                v_att = v.view(chunks, frames, L, C)[:, 0].contiguous()
            else:
                k_att, v_att = ops.kv_compact(k, v, idx, chunks)
            q_per_kv = frames

        # spatial-guided attention: the result REPLACES the query (:257-288)
        q_main = q
        if ctrl and ctrl.use_intraattn:
            ref = ctrl(None)
            assert ref.shape == hidden_states.shape
            q_ref = attn.to_q(ref).to(torch.float16).contiguous()
            k_ref = attn.to_k(ref).to(torch.float16).contiguous()
            q_main = ops.attn_fwd(q_ref, k_ref, q, heads, 1,
                                  softmax_scale=ctrl.intraattn_scale_factor * inv_sqrt_d,
                                  diag_bias=float(ctrl.intraattn_bias))

        out = ops.attn_fwd(q_main, k_att, v_att, heads, q_per_kv, softmax_scale=inv_sqrt_d)      # :303-305

        # temporal-guided attention along flow trajectories; REPLACES the output (:309-367)
        if ctrl and ctrl.use_interattn:
            traj = ctrl.trajectories(L)
            if traj is None:
                raise FrescoError(f"temporal-guided attention enabled but no mapping matches {L} tokens")
            fwd_map, traj_mask = traj
            out = ops.temporal_attn_fwd(q, k, out, fwd_map, traj_mask, chunks, heads,
                                        ctrl.interattn_scale_factor * inv_sqrt_d)
        return out.to(in_dtype)


class _SDPAProcessor:
    """Plain scaled-dot-product attention processor for the layers FRESCO leaves
    alone, used only when diffusers' own AttnProcessor2_0 is not importable."""

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None):
        b = hidden_states.shape[0]
        ctx = hidden_states if encoder_hidden_states is None else encoder_hidden_states
        h = attn.heads
        q = attn.to_q(hidden_states)
        k = attn.to_k(ctx)
        v = attn.to_v(ctx)
        d = q.shape[-1] // h
        o = F.scaled_dot_product_attention(q.view(b, -1, h, d).transpose(1, 2), k.view(b, -1, h, d).transpose(1, 2),
                                           v.view(b, -1, h, d).transpose(1, 2), attn_mask=attention_mask)
        o = o.transpose(1, 2).reshape(b, -1, h * d)
        return attn.to_out[1](attn.to_out[0](o))


def _default_attn_processor():
    try:
        from diffusers.models.attention_processor import AttnProcessor2_0   # type: ignore
        proc = AttnProcessor2_0()
        if not callable(proc):                      # (a stubbed diffusers, as the CPU tests install to import the reference)
            raise TypeError("AttnProcessor2_0 is not callable")
        return proc
    except Exception:
        return _SDPAProcessor()


def apply_FRESCO_attn(pipe, shard=None):
    """Install one shared FRESCO processor on every attention of up_blocks.2 / up_blocks.3
    (src/diffusion_hacked.py:390-403) and return it.  ``shard=(world, rank, group)`` (not in the
    reference) runs the batch frame-sharded over the GPUs of one box."""
    fresco_proc = FRESCOAttnProcessor2_0(2, AttentionControl(), shard=shard)
    plain = _default_attn_processor()
    table = {}
    for name in pipe.unet.attn_processors.keys():
        table[name] = fresco_proc if name.startswith(("up_blocks.2", "up_blocks.3")) else plain
    pipe.unet.set_attn_processor(table)
    return fresco_proc


# =============================================================================
# PART II -- FRESCO feature optimisation
# =============================================================================
class OptimizeTrace:
    """Optional per-iteration record (loss values) for parity tests."""

    def __init__(self):
        self.losses: List[float] = []


class GramTarget:
    """Spatial-consistency target of one decoder level in the form the kernels want it: the row-normalised reference
    features ``yhat`` [2N, L, C] fp16 -- exactly the operand the reference feeds its fp16 ``bmm``
    (src/diffusion_hacked.py:889-893) -- instead of the fp32 [2N, L, L] product (1.07 GB at layer 3, read once per Adam
    iteration by the reference).  The Gram tile is recomputed inside the loss kernel.  Quacks like the tensor the
    reference stores where optimize_feature looks at it (``.shape[1] == h*w``); ``dense()`` materialises the
    reference's tensor."""

    def __init__(self, yhat: torch.Tensor):
        self.yhat = yhat.contiguous()
        b, l, _ = yhat.shape
        self.shape = torch.Size((b, l, l))
        self.dtype = torch.float32
        self.device = yhat.device

    def dense(self) -> torch.Tensor:
        return torch.bmm(self.yhat, self.yhat.transpose(-1, -2)).to(torch.float32)


def spatial_loss_grad(cs_bcl, target, intra_weight, grad_bcl, loss_acc=None):
    """One evaluation of the spatial-consistency term (src/diffusion_hacked.py:469-476) and its gradient:
    ``grad_bcl += d/dcs [ intra_weight * l1_loss(Xh Xh^T, target) ]`` for cs [2N, C, L] fp32 (channel-major, as the
    UNet holds it); ``target`` is a GramTarget (fast path) or the reference's dense fp32 [2N, L, L] tensor;
    ``loss_acc`` (device float or None) gets the loss value added."""
    xhat, norms = ops.gram_normalize(cs_bcl)
    if isinstance(target, GramTarget):
        tsign = ops.gram_sign_ref(xhat, target.yhat, intra_weight, loss_acc)
    else:
        tsign = ops.gram_sign(xhat, target, intra_weight, loss_acc)
    ops.gram_grad(tsign, xhat, norms, grad_bcl, intra_weight)


class _OptKernels:
    """Compute steps of optimize_feature on the product path: the hand-written kernels behind ``ops``.  (The gloo tests
    inject torch stand-ins with the same methods to exercise the exchange logic on CPU.)"""

    def temporal_prepare(self, flows, occs, h: int, lo: int, hi: int, total: int):
        _, fwd_flow, bwd_flow, fwd_occ, bwd_occ = resize_flows_occs(flows, occs, h)
        w = fwd_flow.shape[-1]
        adjoint = adjoint_csr(flows, occs, h)                   # per-batch: cached on the flow tensors
        fwd_keep = (1 - fwd_occ).reshape(total, h, w)
        bwd_keep = (1 - bwd_occ).reshape(total, h, w)
        if (lo, hi) != (0, total):
            adjoint = ops.WarpAdjointSlice(adjoint, lo, hi)
        return {"fwd_flow": fwd_flow[lo:hi].contiguous(), "bwd_flow": bwd_flow[lo:hi].contiguous(),
                "fwd_keep": fwd_keep[lo:hi].contiguous(), "bwd_keep": bwd_keep[lo:hi].contiguous(), "adjoint": adjoint}

    def temporal(self, cs, prep, grad, loss_acc, halo_cs=None, halo_grad=None, total_frames=None):
        ops.warp_loss_fwd_bwd(cs, prep["fwd_flow"], prep["bwd_flow"], prep["fwd_keep"], prep["bwd_keep"], grad, loss_acc,
                              accumulate=False, adjoint=prep["adjoint"], halo_cs=halo_cs, halo_grad=halo_grad,
                              total_frames=total_frames)

    def spatial(self, cs_bcl, target, weight, grad_bcl, loss_acc):
        spatial_loss_grad(cs_bcl, target, weight, grad_bcl, loss_acc)

    def adam(self, cs, grad, exp_avg, exp_avg_sq, it):
        ops.adam_step(cs, grad, exp_avg, exp_avg_sq, it, lr=0.2)

    def adain(self, cs_bchw, sample):
        return ops.adain(cs_bchw, sample.contiguous())


@torch.no_grad()
def optimize_feature(sample, flows, occs, correlation_matrix=[], intra_weight=1e2, iters=20, unet_chunk_size=2,
                     optimize_temporal=True, trace: Optional[OptimizeTrace] = None, shard=None, backend=None):
    """FRESCO-guided optimisation of decoder features (src/diffusion_hacked.py:416-488):
    ``iters`` Adam steps (lr 0.2) on the temporal-consistency L1 loss and the
    normalised-Gram L1 loss, then AdaIN back to the statistics of ``sample``.
    Loss gradients are closed-form CUDA kernels (no autograd graph).

    ``shard=(world, rank, group | comm)`` (not in the reference): ``sample`` and the entries of ``correlation_matrix``
    hold this rank's frames of ONE frame-sharded batch; ``flows`` / ``occs`` are the whole batch's (every rank builds the
    same per-batch parameters).  The spatial term, Adam and AdaIN are per frame.  The temporal term couples frame f with
    frame f+1 of the ring (:444): per Adam iteration every rank receives the following rank's first frame as a halo,
    evaluates its own pairs in the open-chain form and sends the halo's gradient on (two neighbour exchanges of
    [chunks, C, h, w] fp32 per iteration).  The ranks hold the ``frame_range`` blocks of the batch, which need not be
    even; the batch frame count is that of ``flows`` (without flows: one all-reduce of the local counts).  The result
    is bit-identical to the unsharded call: the loss means run over the whole batch and the Gram kernels get the same
    fp32 loss scale as unsharded (``ops.gram_*`` divide the rank's share of the weight in double and round once).

    ``shard=dist.Box(...)`` takes the batch frame count from ``flows`` (a Box without them raises ValueError on every
    rank): it picks the ranks the batch runs on, and an idle rank gets ``sample`` back at once."""
    have_temporal = flows is not None and occs is not None and optimize_temporal
    if (not have_temporal) and (intra_weight == 0 or len(correlation_matrix) == 0):
        return sample
    layout = batch_layout(shard, flows, sample, unet_chunk_size,
                          "optimize_feature(shard=Box(...)) takes the batch's frame count from flows", count=True)
    if layout.idle:
        return sample
    be = backend if backend is not None else _OptKernels()
    _, C, h, w = sample.shape
    chunks = layout.chunks(unet_chunk_size)
    n = sample.shape[0] // chunks
    lo, hi, total = layout.lo, layout.hi, layout.n_frames
    if hi - lo != n or sample.shape[0] != chunks * n:
        raise FrescoError("optimize_feature: %r owns frames [%d, %d) of the %d-frame batch, got %d rows"
                          % (layout, lo, hi, total, sample.shape[0]))
    ring = layout.ring()                # the halo exchange of this rank's frame ring (None: the ring is closed here)
    trace_comm = layout.trace_comm()    # the loss trace sums over the whole shard
    cs = sample.to(torch.float32).reshape(chunks, n, C, h, w).contiguous().clone()
    grad = torch.empty_like(cs)
    exp_avg = torch.zeros_like(cs)
    exp_avg_sq = torch.zeros_like(cs)
    if have_temporal:
        prep = be.temporal_prepare(flows, occs, h, lo, hi, total)
        if ring is not None:
            first, halo_cs, halo_grad, from_prev = (torch.empty(chunks, C, h, w, dtype=torch.float32,
                                                                device=sample.device) for _ in range(4))
    target = None
    for tmp in correlation_matrix:
        if h * w == tmp.shape[1]:
            target = tmp
            break
    spatial = target is not None and intra_weight > 0
    if spatial and not isinstance(target, GramTarget):
        target = target.to(torch.float32).contiguous()
    # F.l1_loss averages over the frames of the WHOLE batch: a rank's share of the weight, which the Gram kernels divide
    # by this rank's batch in double (ops.gram_*), so the fp32 loss scale is the unsharded one
    weight = intra_weight * layout.row_share
    loss_acc = torch.zeros(1, dtype=torch.float32, device=sample.device) if trace is not None else None
    for it in range(1, iters + 1):
        if loss_acc is not None:
            loss_acc.zero_()
        if have_temporal and ring is not None:
            first.copy_(cs[:, 0])
            ring.shift(first, halo_cs, -1)                      # my first frame is the previous rank's halo
            be.temporal(cs, prep, grad, loss_acc, halo_cs, halo_grad, layout.mean_frames)
            ring.shift(halo_grad, from_prev, +1)                # what my first frame receives from the previous rank's last pair
            grad[:, 0] += from_prev
        elif have_temporal:
            be.temporal(cs, prep, grad, loss_acc, total_frames=layout.mean_frames)
        else:
            grad.zero_()
        if spatial:
            be.spatial(cs.view(chunks * n, C, h * w), target, weight, grad.view(chunks * n, C, h * w),
                       loss_acc)
        be.adam(cs, grad, exp_avg, exp_avg_sq, it)
        if trace is not None:
            if trace_comm is not None:
                trace_comm.all_reduce_sum(loss_acc)
            trace.losses.append(float(loss_acc.item()))
    return be.adain(cs.view(chunks * n, C, h, w), sample)


def my_forward(self, steps=[], layers=[0, 1, 2, 3], flows=None, occs=None, correlation_matrix=[],
               intra_weight=1e2, iters=20, optimize_temporal=True, saliency=None, shard=None):
    """Replacement for ``pipe.unet.forward`` (src/diffusion_hacked.py:491-816).

    The reference carries a verbatim copy of diffusers-0.19.3's UNet forward with
    three edits (:757-779, :808-812).  Here the same three behaviours are attached
    to the UNet's own forward through forward-pre-hooks on ``up_blocks[i]``:
      * record the decoder feature entering up-block i (``i in layers``),
      * on optimisation steps replace it by optimize_feature(...) and, with a
        saliency map, warp_tensor(..., 2)   (background smoothing),
      * with ``return_dict=False`` return ``(sample, *up_samples)``.
    """
    unet = self
    cls_forward = type(unet).forward
    step_set = None

    def is_opt_step(timestep) -> bool:
        nonlocal step_set
        if steps is None or len(steps) == 0:
            return False
        if step_set is None:
            step_set = set(int(s) for s in (steps.tolist() if torch.is_tensor(steps) else steps))
        return int(timestep) in step_set

    def forward(sample, timestep, encoder_hidden_states, *args, return_dict: bool = True, **kwargs):
        up_samples = []
        optimise = is_opt_step(timestep)
        handles = []

        def make_hook(i):
            def pre_hook(module, h_args, h_kwargs):
                feat = h_kwargs["hidden_states"] if "hidden_states" in h_kwargs else h_args[0]
                up_samples.append(feat)
                if not optimise:
                    return None
                # frame-sharded batch (shard != None): optimize_feature exchanges one boundary frame per Adam iteration
                # with its ring neighbours, warp_tensor re-shards the chain by channel
                new = optimize_feature(feat, flows, occs, correlation_matrix, intra_weight, iters,
                                       optimize_temporal=optimize_temporal, shard=shard)
                if saliency is not None:
                    new = warp_tensor(new, flows, occs, saliency, 2, shard=shard)
                if "hidden_states" in h_kwargs:
                    h_kwargs = dict(h_kwargs)
                    h_kwargs["hidden_states"] = new
                    return h_args, h_kwargs
                return (new,) + tuple(h_args[1:]), h_kwargs
            return pre_hook

        for i, blk in enumerate(unet.up_blocks):
            if i in layers:
                handles.append(blk.register_forward_pre_hook(make_hook(i), with_kwargs=True))
        try:
            out = cls_forward(unet, sample, timestep, encoder_hidden_states, *args, return_dict=return_dict, **kwargs)
        finally:
            for hd in handles:
                hd.remove()
        if not return_dict:
            return (out[0],) + tuple(up_samples)
        return out

    return forward


def apply_FRESCO_opt(pipe, steps=[], layers=[0, 1, 2, 3], flows=None, occs=None, correlation_matrix=[],
                     intra_weight=1e2, iters=20, optimize_temporal=True, saliency=None, shard=None):
    """src/diffusion_hacked.py:819-825.  Called once per keyframe batch (run_fresco.py:232-234): per-batch
    preparation cached for the previous batch's flows is dropped here."""
    clear_prep_cache()
    pipe.unet.forward = my_forward(pipe.unet, steps, layers, flows, occs, correlation_matrix, intra_weight, iters,
                                   optimize_temporal, saliency, shard=shard)


def disable_FRESCO_opt(pipe):
    """src/diffusion_hacked.py:827-831."""
    apply_FRESCO_opt(pipe)


# =============================================================================
# PART III -- per-batch parameters (the pieces that do not need the SD pipeline)
# =============================================================================
@torch.no_grad()
def cross_frame_attn_masks(bwd_occs: torch.Tensor, scales: Sequence[float] = (8.0, 16.0, 32.0)):
    """K/V-selection masks of efficient cross-frame attention, bool [N, L_s] per scale:
    frame 0 keeps every token, frames >= 1 keep their occluded tokens
    (src/diffusion_hacked.py:935-938)."""
    masks = []
    for s in scales:
        o = F.interpolate(bwd_occs[:-1].unsqueeze(1), scale_factor=1.0 / s, mode="bilinear")
        masks.append(torch.cat((o[0:1].reshape(1, -1) > -1, o.reshape(o.shape[0], -1) > 0.5), dim=0))
    return masks


@torch.no_grad()
def gram_targets(features: Sequence[torch.Tensor], dense: bool = False):
    """Normalised-Gram targets of decoder features (src/diffusion_hacked.py:889-895).  ``dense=True`` gives what the
    reference stores, fp32 [2N, L, L] each; the default keeps the normalised features (GramTarget) and lets the loss
    kernel recompute the products."""
    out = []
    for t in features:
        v = t.reshape(t.shape[0], t.shape[1], -1).transpose(1, 2)
        v = v / ((v ** 2).sum(dim=2, keepdim=True) ** 0.5)
        if dense or not v.is_cuda:
            out.append(torch.bmm(v, v.transpose(-1, -2)).to(torch.float32))
        else:
            out.append(GramTarget(v.to(torch.float16)))
    return out


@torch.no_grad()
def get_intraframe_paras(pipe, imgs, frescoProc, prompt_embeds, do_classifier_free_guidance=True, seed=0, shard=None):
    """Parameters for spatial-guided attention / optimisation (src/diffusion_hacked.py:843-901): one UNet pass
    on the noised input frames with the controller in store mode (fills
    ``frescoProc.controller.stored_attn['decoder_attn']``), then the normalised-Gram targets of the four
    decoder features.

    ``shard=(world, rank[, group])`` (not in the reference): ``imgs`` / ``prompt_embeds`` hold ALL N frames; the
    initial noise is drawn for all of them from the seeded generator and this rank's frames [rank*N//G, (rank+1)*N//G)
    are sliced, encoded and run through the store pass.  The controller then holds this rank's reference inputs and
    the targets cover this rank's frames (both CFG chunks): what the sharded processor and
    ``optimize_feature(shard=...)`` take.  The pass is per frame, so no collective is issued.  With fewer frames than
    ranks (``dist.shard_layout``'s half layout) the pass runs on this rank's CFG half only, the targets cover its
    samples, and the VAE posterior sample is drawn on the half-0 ranks and sent to their peers.  An idle rank of a
    ``dist.Box`` returns no targets at once."""
    B, C, H, W = imgs.shape
    layout = shard_layout(B, shard)
    if layout.idle:
        return []
    scheduler = pipe.scheduler
    timestep = scheduler.timesteps[-1]
    device = pipe._execution_device
    generator = torch.Generator(device=device).manual_seed(seed)
    lo, hi = layout.lo, layout.hi
    chunks = layout.chunks(2 if do_classifier_free_guidance else 1)     # the half layout needs both CFG halves
    if hasattr(frescoProc, "set_batch_frames"):
        frescoProc.set_batch_frames(B)
    ctrl = frescoProc.controller
    ctrl.disable_controller()
    disable_FRESCO_opt(pipe)
    ctrl.clear_store()
    ctrl.enable_store()
    latents = pipe.prepare_latents(B, pipe.unet.config.in_channels, H, W, prompt_embeds.dtype, device, generator,
                                   latents=None)[lo:hi]             # all N frames: same Philox stream on every rank

    def encode():
        return pipe.vae.config.scaling_factor * pipe.vae.encode(imgs[lo:hi].to(pipe.unet.dtype)).latent_dist.sample()
    latent_x0 = layout.share(encode, (latents.shape, getattr(pipe.vae, "dtype", pipe.unet.dtype), latents.device))
    latents = scheduler.add_noise(latent_x0, latents, timestep).detach()
    model_in = torch.cat([latents] * chunks) if chunks > 1 else latents
    pe = layout.rows(prompt_embeds, 2 if do_classifier_free_guidance else 1)
    out = pipe.unet(model_in, timestep, encoder_hidden_states=pe, cross_attention_kwargs=None, return_dict=False)
    ctrl.disable_store()
    return gram_targets(out[1:])


@torch.no_grad()
def get_flow_and_interframe_paras(flow_model, imgs, visualize_pipeline=False, shard=None):
    """Parameters for temporal-guided attention / optimisation (src/diffusion_hacked.py:905-957): bidirectional
    GMFlow flow between consecutive keyframes (incl. the wrap-around pair), occlusion masks from flow consistency
    and photometric error, the cross-frame K/V masks at 3 scales and the FLATTEN trajectories at 2 scales.
    ``imgs``: list of HxWx3 uint8 arrays.  ``flow_model``: a GMFlow instance (its global correlation can be
    redirected to fresco_b200.gmflow_matching, see INTEGRATION.md).

    ``shard=(world, rank[, group])`` (not in the reference): every rank gets all N frames, runs GMFlow on its own
    pairs ``frame_range(N, world, rank)`` only and one all-gather (blocks padded to the largest share) assembles the
    whole batch's flows (rank order == pair order).  Occlusions, masks and trajectories are then built from the gathered flows on every rank, as unsharded:
    the return values are the whole batch's, as in the unsharded call.  With fewer frames than ranks
    (``dist.shard_layout``'s half and unequal-halves layouts) the ranks of half 0 compute every pair once and send
    the flows of each pair to the half-1 ranks holding it, and each half gathers the whole batch's flows within
    itself: GMFlow is a network outside this library, whose bits could differ between two devices.  An idle rank of a
    ``dist.Box`` returns at once, with empty flows and occlusions, no masks and no trajectories."""
    from .flow_utils import flow_warp, forward_backward_consistency_check, get_mapping_ind
    n = len(imgs)
    layout = shard_layout(n, shard)
    param = next(flow_model.parameters())
    dev = param.device
    if layout.idle:
        h, w = imgs[0].shape[:2]
        empty = torch.empty(0, 2, h, w, dtype=param.dtype, device=dev)
        occ = torch.empty(0, h, w, dtype=torch.float32, device=dev)
        return [empty, empty.clone()], [occ, occ.clone()], [], {"fwd_mappings": [], "bwd_mappings": [],
                                                                 "interattn_masks": []}
    images = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs], dim=0).to(dev)
    imgs_torch = images / 127.5 - 1.0                                   # numpy2tensor (src/utils.py:8-12)
    reshuffle = list(range(1, len(images))) + [0]
    lo, hi = layout.lo, layout.hi

    def flows():
        res = flow_model(images[lo:hi], images[reshuffle][lo:hi], attn_splits_list=[2], corr_radius_list=[-1],
                         prop_radius_list=[-1], pred_bidir_flow=True)
        return res["flow_preds"][-1]                                    # [2 * pairs, 2, H, W]: forward | backward
    flow = layout.share(flows, ((2 * (hi - lo), 2) + tuple(images.shape[2:]), param.dtype, dev), chunks=2)
    flow = layout.gather_frames(flow, 2)
    fwd_flows, bwd_flows = flow.chunk(2)
    fwd_flows, bwd_flows = fwd_flows.contiguous(), bwd_flows.contiguous()
    fwd_occs, bwd_occs = forward_backward_consistency_check(fwd_flows, bwd_flows)
    warped1 = flow_warp(images, bwd_flows)
    bwd_occs = torch.clamp(bwd_occs + (abs(images[reshuffle] - warped1).mean(dim=1) > 255 * 0.25).float(), 0, 1)
    warped2 = flow_warp(images[reshuffle], fwd_flows)
    fwd_occs = torch.clamp(fwd_occs + (abs(images - warped2).mean(dim=1) > 255 * 0.25).float(), 0, 1)
    attn_mask = cross_frame_attn_masks(bwd_occs)
    fwd_m, bwd_m, masks = [], [], []
    for scale in (8.0, 16.0):
        f, b, m = get_mapping_ind(bwd_flows, bwd_occs, imgs_torch, scale=scale)
        fwd_m.append(f), bwd_m.append(b), masks.append(m)
    paras = {"fwd_mappings": fwd_m, "bwd_mappings": bwd_m, "interattn_masks": masks}
    return [fwd_flows, bwd_flows], [fwd_occs, bwd_occs], attn_mask, paras
