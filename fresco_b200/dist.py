"""Frame-sharded FRESCO attention for one multi-GPU box (NCCL over NVLink / NVSwitch).

The reference has no collective on this path (SURVEY 2.1); this module is the multi-GPU design for BASELINE config 4: the
N keyframes of ONE batch are split contiguously over G ranks (rank r owns frames ``frame_range(N, G, r)`` =
[r*N//G, (r+1)*N//G) of both CFG chunks; G need not divide N) and the UNet body runs as plain replicas.  A batch of
G/2 <= N < G frames on an even G is split over the two CFG halves as well (``shard_layout``): every exchange below then
runs with one chunk within the ranks of a half.  A ``Box`` in place of the tuple also runs every other batch: unequal
halves on an odd G, idle ranks beyond 2N.  Only FRESCO attention couples frames:

* cross-frame attention (src/diffusion_hacked.py:225-247, :303-305): every query frame attends the same K/V set = all
  tokens of frame 0 + the occluded tokens of frames 1..N-1.  Each rank compacts the selected rows of ITS frames straight
  into the send buffer (K | V side by side in one 2C-wide row), ONE all-gather per layer (padded to the largest
  per-rank count, known on the host from the per-batch mask) delivers every rank's rows, one row-gather drops the
  padding, and the attention kernel reads K and V out of the interleaved buffer through strided TMA maps -- the
  reference's row-major (frame, token) order is kept because rank order == frame order.
* temporal-guided attention (:320-367) mixes all N frames along each flow trajectory.  It is sharded by TRAJECTORY:
  rank s owns trajectories ``frame_range(L, G, s)``; one all-to-all sends it the q | k | attention-output rows those
  trajectories visit in every rank's frames (1/G of the data instead of an all-gather of all of it), it runs the
  N x N attention for its trajectories only (1/G of the work instead of all of it on every rank), and a second
  all-to-all returns the result rows to the ranks that own the frames.
* spatial-guided attention (:257-288) is per frame: local.

Compute goes through a small backend object (default: the CUDA kernels in ``ops``); the CPU tests inject a torch
backend to exercise the exchange / ordering logic under gloo.  Nothing here synchronises with the host after the
per-batch plans exist, so a whole UNet step (collectives included) can be captured in a CUDA graph.
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist


def frame_range(n_frames: int, world: int, rank: int) -> Tuple[int, int]:
    """[lo, hi) = [rank*N//G, (rank+1)*N//G): the contiguous block of the N items (frames of a batch, trajectories of
    the temporal exchange) rank ``rank`` of ``world`` owns.  Rank order is item order, every rank gets floor(N/G) or
    ceil(N/G) items, and when G divides N this is the even split."""
    if n_frames < world:
        raise ValueError(f"{n_frames} frames cannot be split over {world} ranks (every rank needs at least one): run "
                         f"the batch on a process group of {n_frames} ranks, shard=({n_frames}, rank, group)")
    return rank * n_frames // world, (rank + 1) * n_frames // world


def block_sizes(n_frames: int, world: int) -> List[int]:
    """the share of every rank under ``frame_range``, in rank order"""
    return [hi - lo for lo, hi in (frame_range(n_frames, world, r) for r in range(world))]


class Box(tuple):
    """``Box(world, rank, group=None)``: rank ``rank`` of ``world`` ranks (of ``group``, default: the whole world) that
    may run a keyframe batch, as the ``shard`` argument of every sharded entry point.  It reads as the tuple
    ``(world, rank, group)`` does, and ``shard_layout`` gives it the same frame and half layouts; where the tuple raises,
    a Box still runs the batch: on an odd number of ranks the two CFG halves get ceil(G/2) and floor(G/2) ranks, and
    ranks beyond 2N stay idle.  So one Box per rank runs every batch a driver makes, whatever its frame count."""

    def __new__(cls, world: int, rank: int, group=None):
        return tuple.__new__(cls, (int(world), int(rank), group))

    def __repr__(self):
        return f"Box(world={self[0]}, rank={self[1]}, group={self[2]!r})"


class ShardLayout:
    """What one rank of a sharded keyframe batch holds and whom it exchanges with (``shard_layout``).

    ``halves`` = [h0, h1): the CFG halves (0 unconditional, 1 text) of frames [``lo``, ``hi``) this rank holds; (0, 0)
    on an idle rank, which holds nothing.  ``world`` / ``rank`` / ``group``: the process group the frame-sharded
    exchanges (K/V all-gather, trajectory all-to-alls, ring halo, warp re-shard, frame gathers) run on.  ``peers``: (global
    rank, lo, hi) of every rank of the other CFG half whose frames overlap this rank's, [lo, hi) the overlap;
    ``partner``: the one peer when the two halves split alike, else None.  ``shard``: the ``(world, rank, group)`` or
    ``Box`` of the ranks the batch runs on -- the caller's, or for a Box with idle ranks the Box of its first 2N.

    The one-rank layout (``shard_layout(n, None)``) holds everything and exchanges nothing; every method below then
    does what an unsharded call does."""

    def __init__(self, n_frames, halves, lo, hi, world, rank, group, partner, shard, peers=()):
        self.n_frames, self.halves, self.lo, self.hi = n_frames, halves, lo, hi
        self.world, self.rank, self.group, self.partner, self.shard = world, rank, group, partner, shard
        self.peers = list(peers)

    @property
    def split_halves(self) -> bool:
        return self.halves[1] - self.halves[0] == 1

    @property
    def idle(self) -> bool:
        """a rank of a Box beyond the 2N ranks the batch runs on"""
        return self.halves[0] == self.halves[1]

    @property
    def half(self) -> int:
        """the CFG half this rank holds in the half layout"""
        return self.halves[0]

    @property
    def row_share(self) -> float:
        """rows held / rows in the batch: this rank's share of a loss averaged over the whole batch"""
        return float((self.hi - self.lo) * (self.halves[1] - self.halves[0])) / float(2 * self.n_frames)

    @property
    def mean_frames(self) -> int:
        """the frame count of the temporal loss's mean in the element count chunks * frames * C*h*w, chunks being this
        rank's: N with both CFG halves, 2N with one, so that the count is the unsharded call's"""
        return self.n_frames * 2 // (self.halves[1] - self.halves[0])

    def chunks(self, cfg_chunks: int) -> int:
        """CFG chunks of this rank's rows for a call that would hold ``cfg_chunks`` unsharded"""
        if not self.split_halves:
            return cfg_chunks
        if cfg_chunks != 2:
            raise ValueError(f"{self.n_frames} frames on {self.shard[0]} ranks shard over the two classifier-free "
                             f"guidance halves, so the batch needs both (got {cfg_chunks} chunk)")
        return 1

    def rows(self, t: Optional[torch.Tensor], cfg_chunks: int) -> Optional[torch.Tensor]:
        """this rank's rows of a ``(chunk, frame)``-major batch ``[cfg_chunks * N, ...]`` (prompt embeddings, ControlNet
        edges, Gram targets): frames [lo, hi) of each chunk it holds.  Anything not laid out that way comes back as it
        is (see ``chunk_frames``)."""
        if not self.split_halves:
            return chunk_frames(t, cfg_chunks, self.n_frames, self.lo, self.hi)
        if t is None or t.shape[0] != 2 * self.n_frames:
            return t
        base = self.half * self.n_frames
        return t[base + self.lo:base + self.hi]

    def guided(self, model_output: torch.Tensor, do_cfg: bool) -> torch.Tensor:
        """The raw UNet output of both CFG halves of this rank's frames, [uncond; text], from this rank's: as it is when
        the rank holds both halves; in the half layouts its rows and the peers' (``swap``), in half order."""
        if not self.split_halves:
            return model_output
        if not do_cfg:
            raise ValueError("a batch sharded over the CFG halves needs guidance_scale")
        mine = model_output.contiguous()
        theirs = self.swap(mine)
        return torch.cat([mine, theirs] if self.half == 0 else [theirs, mine])

    def swap(self, mine: torch.Tensor) -> torch.Tensor:
        """The other CFG half's rows of this rank's frames, shaped as ``mine`` ([n_local, ...]): one batched send /
        receive with every peer (``send_recv``, as ``RingComm.shift``) -- in the half layout, the partner's whole
        tensor."""
        mine = mine.contiguous()
        theirs = torch.empty_like(mine)
        _cross_halves(self, mine, theirs, 1)
        return theirs

    def share(self, make, like: Tuple[tuple, torch.dtype, torch.device], chunks: int = 1) -> torch.Tensor:
        """What ``make()`` returns for this rank's frames ([chunks * n_local, ...], ``(chunk, frame)``-major).  A rank
        holding both CFG halves calls it.  In the half layouts it is computed once, on the ranks of half 0, each of
        which sends every peer the rows of the frames they share; a half-1 rank receives its rows into a tensor of
        ``like = (shape, dtype, device)`` without calling ``make``.  For everything drawn from an unseeded generator or
        computed by a network outside this library, whose bits could differ between two devices."""
        if not self.split_halves:
            return make()
        if self.half == 0:
            out = make().contiguous()
            _cross_halves(self, out, None, chunks)
        else:
            shape, dtype, device = like
            out = torch.empty(shape, dtype=dtype, device=device)
            _cross_halves(self, None, out, chunks)
        return out

    def gather_frames(self, t: torch.Tensor, chunks: int = 1) -> torch.Tensor:
        """the whole ``(chunk, frame)``-major batch from every rank's block ``t`` of the exchange group
        (``all_gather_frames``); ``t`` itself on one rank"""
        if self.world == 1:
            return t
        return all_gather_frames(t, self.n_frames, self.world, chunks, self.group)

    def ring(self) -> Optional["RingComm"]:
        """the neighbour exchange of the frame ring: over the exchange group; None on one rank"""
        return _comm(self.world, self.rank, self.group)

    def trace_comm(self) -> Optional["RingComm"]:
        """the communicator of every rank of the shard (loss sums over the batch); None on one rank"""
        return _comm(*unpack(self.shard))

    def __repr__(self):
        return (f"ShardLayout(n_frames={self.n_frames}, halves={self.halves}, frames=[{self.lo}, {self.hi}), "
                f"world={self.world}, rank={self.rank}, peers={self.peers})")


def unpack(shard) -> Tuple[int, int, object]:
    """(world, rank, group) of a ``shard=(world, rank[, group])`` tuple or ``Box``"""
    return int(shard[0]), int(shard[1]), (shard[2] if len(shard) > 2 else None)


def _comm(world: int, rank: int, group):
    """the ``RingComm`` of ``group``, or the communicator injected in its place (tests: ranks as threads, an object
    with ``shift``); None for one rank"""
    if world == 1:
        return None
    return group if hasattr(group, "shift") else RingComm(world, rank, group)


_HALF_GROUPS: dict = {}
_ACTIVE_GROUPS: dict = {}


def _global_rank(group, r: int) -> int:
    return dist.get_global_rank(group, r) if group is not None else r


def _splits_nccl(group) -> bool:
    """True when a new NCCL group would be split from the default group's communicator: the default group is
    bound to a device (``init_process_group(..., device_id=...)``), and ``ncclCommSplit`` is collective over every rank
    of the communicator it splits"""
    return bool(getattr(dist.group.WORLD, "bound_device_id", None)) and dist.get_backend(group) == dist.Backend.NCCL


def half_sizes(world: int) -> Tuple[int, int]:
    """ranks of CFG half 0 and half 1 when ``world`` ranks split over the halves: ceil(G/2) and floor(G/2)"""
    return world - world // 2, world // 2


def _no_capture(what: str) -> None:
    if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
        raise RuntimeError(f"the {what} must exist before a step is captured: call a sharded entry point "
                           "(get_flow_and_interframe_paras, get_intraframe_paras, inference) first")


def half_group(world: int, rank: int, group=None):
    """The process group of the CFG half of rank ``rank`` of the shard group ``group`` (``world`` ranks): group ranks
    [0, G0) for half 0 and [G0, G) for half 1, G0 = ceil(G/2) (``half_sizes``); None for a half of one rank.  It
    depends on G and the shard's ranks only, is created on the first call (every rank of the shard reaches its first
    half-layout entry point in the same order) and cached by the global ranks of the shard, so a shard group made again
    over the same ranks finds it.  Only the shard's ranks take part: under NCCL with a device-bound default group the
    shard group is split in two (``split_group``, collective over the shard's ranks only: a plain ``new_group`` would
    split the default communicator, which needs every rank of the world); otherwise each half is created by its own
    ranks (``new_group(..., use_local_synchronization=True)``)."""
    first = half_sizes(world)[0]
    shard_ranks = tuple(_global_rank(group, r) for r in range(world))
    if shard_ranks in _HALF_GROUPS:
        return _HALF_GROUPS[shard_ranks]
    _no_capture("CFG-half process groups")
    halves = [list(range(first)), list(range(first, world))]
    mine = halves[0 if rank < first else 1]
    splits = [h for h in halves if len(h) > 1]                  # a half of one rank needs no group
    if not splits:
        sub = None
    elif _splits_nccl(group):
        sub = dist.split_group(parent_pg=group, split_ranks=splits)     # None on a rank in no split
    else:
        sub = dist.new_group([shard_ranks[r] for r in mine], use_local_synchronization=True) if len(mine) > 1 else None
    _HALF_GROUPS[shard_ranks] = sub
    return sub


def active_group(world: int, rank: int, group, active: int):
    """The process group of the first ``active`` ranks of the Box group ``group`` (``world`` ranks), the ranks a batch of
    active/2 frames runs on; None on the other ranks.  Created on the first call and cached as ``half_group`` caches the
    halves.  Under NCCL with a device-bound default group it is split from ``group`` (``split_group``), which every rank
    of ``group`` enters once, the idle ones included; otherwise only the active ranks create it, and an idle rank
    touches neither ``group`` nor any collective."""
    if rank >= active and not _splits_nccl(group):
        return None
    if hasattr(group, "sub_comm"):
        return group.sub_comm(active, rank)                     # an injected communicator (tests) supplies its own
    key = (tuple(_global_rank(group, r) for r in range(world)), active)
    if key in _ACTIVE_GROUPS:
        return _ACTIVE_GROUPS[key]
    _no_capture("process group of a Box's active ranks")
    if _splits_nccl(group):
        sub = dist.split_group(parent_pg=group, split_ranks=[list(range(active))])
    else:
        sub = dist.new_group(list(key[0][:active]), use_local_synchronization=True)
    _ACTIVE_GROUPS[key] = sub
    return sub


def shard_layout(n_frames: int, shard) -> ShardLayout:
    """The partition of a keyframe batch of ``n_frames`` frames (2N samples: an unconditional and a text half) over
    ``shard=(world, rank[, group])``; for ``shard=None`` the one-rank layout, which equals that of ``(1, 0, None)``.
    A ``ShardLayout`` comes back as it is.  Chosen by shape alone:

    * N >= G: the frame layout -- rank r holds both halves of frames ``frame_range(N, G, r)``, the exchanges run on
      ``group``.
    * G even and G/2 <= N < G: the half layout -- rank r holds half r // (G/2) of frames ``frame_range(N, G/2, r %
      (G/2))``; the exchanges run on the group of its half (``half_group``); its partner r +- G/2 holds the other half
      of the same frames.
    * otherwise: ValueError for a tuple.  A ``Box`` goes on:
      * G odd and N < G <= 2N: the unequal-halves layout -- half 0 gets the first G0 = ceil(G/2) ranks, half 1 the other
        G1 = floor(G/2); rank r of half h holds frames ``frame_range(N, G_h, r - h*G0)`` of that half, the exchanges run
        on the group of its half, and its ``peers`` are the ranks of the other half whose frames overlap its own.
      * G > 2N: the first 2N ranks run the batch in the half layout, on their own process group (``active_group``);
        the others get an idle layout and take part in nothing."""
    if shard is None:
        shard = (1, 0, None)
    if isinstance(shard, ShardLayout):
        return shard
    world, rank, group = unpack(shard)
    box = isinstance(shard, Box)
    if box and world > 2 * n_frames:
        active = 2 * n_frames
        sub = active_group(world, rank, group, active)
        if rank >= active:
            return ShardLayout(n_frames, (0, 0), 0, 0, 1, 0, None, None, shard)
        return shard_layout(n_frames, Box(active, rank, sub))
    if n_frames >= world:
        lo, hi = frame_range(n_frames, world, rank)
        return ShardLayout(n_frames, (0, 2), lo, hi, world, rank, group, None, shard)
    if (world % 2 != 0 and not box) or 2 * n_frames < world:
        raise ValueError(f"{n_frames} frames cannot be sharded over {world} ranks: shard over the two guidance halves "
                         f"needs an even number of ranks G <= 2N = {2 * n_frames}, or run the batch on a process group "
                         f"of {n_frames} ranks, shard=({n_frames}, rank, group)")
    sizes = half_sizes(world)
    h = 0 if rank < sizes[0] else 1
    r = rank - h * sizes[0]
    lo, hi = frame_range(n_frames, sizes[h], r)
    injected = hasattr(group, "half_comm")
    # an injected communicator (tests: ranks as threads) supplies the communicator of the half itself
    sub = group.half_comm(world, rank) if injected else half_group(world, rank, group)
    peers = []
    for s in range(sizes[1 - h]):                               # the other half's ranks whose frames overlap mine
        a, b = frame_range(n_frames, sizes[1 - h], s)
        if max(a, lo) < min(b, hi):
            peer = (1 - h) * sizes[0] + s
            peers.append((peer if injected else _global_rank(group, peer), max(a, lo), min(b, hi)))
    partner = peers[0][0] if sizes[0] == sizes[1] else None
    return ShardLayout(n_frames, (h, h + 1), lo, hi, sizes[h], r, sub, partner, shard, peers)


def batch_layout(shard, flows, local: torch.Tensor, cfg_chunks: int, missing: str, count: bool = False) -> ShardLayout:
    """``shard`` (None, a tuple, a ``Box`` or a ``ShardLayout``) resolved for a call that holds this rank's rows
    ``local`` (``cfg_chunks`` CFG chunks of its frames) of a batch whose flows are ``flows`` (the whole batch's, or
    None).  On one rank the batch is ``local``; otherwise its frame count is that of ``flows``.  Without flows a Box
    raises ValueError(``missing``); a tuple sums the rows of the shard's ranks (one all-reduce) with ``count``, and
    otherwise, having nothing to exchange without flows, runs as the one-rank layout of its own rows."""
    if isinstance(shard, ShardLayout):
        return shard
    if shard is None or unpack(shard)[0] == 1:
        return shard_layout(local.shape[0] // cfg_chunks, shard)
    if flows is not None:
        return shard_layout(int(flows[0].shape[0]), shard)
    if isinstance(shard, Box):
        raise ValueError(missing)
    if not count:
        return shard_layout(local.shape[0] // cfg_chunks, None)
    # every (chunk, frame) sample is held once in either layout: the batch has (all rows) / chunks frames
    rows = torch.full((1,), local.shape[0], dtype=torch.int64, device=local.device)
    _comm(*unpack(shard)).all_reduce_sum(rows)
    return shard_layout(int(rows.item()) // cfg_chunks, shard)


def send_recv(sends, recvs, group=None) -> None:
    """One batched point-to-point exchange: ``sends`` / ``recvs`` are lists of (tensor, global peer rank).  Under
    NCCL it runs on the current stream with no host synchronisation; gloo moves host memory only, so GPU tensors are
    staged through host copies there."""
    stage = dist.get_backend(group) == dist.Backend.GLOO and any(t.is_cuda for t, _ in list(sends) + list(recvs))
    out = [(torch.empty(t.shape, dtype=t.dtype) if stage else t, p) for t, p in recvs]
    ops = ([dist.P2POp(dist.isend, t.cpu() if stage else t, p, group) for t, p in sends]
           + [dist.P2POp(dist.irecv, t, p, group) for t, p in out])
    for r in dist.batch_isend_irecv(ops):
        r.wait()
    if stage:
        for (dst, _), (src, _) in zip(recvs, out):
            dst.copy_(src)


def _peer_rows(t: torch.Tensor, chunks: int, n: int, a: int, b: int) -> torch.Tensor:
    """rows of frames [a, b) (counted from the rank's first frame) of each chunk of ``t = [chunks * n, ...]``"""
    if chunks == 1:
        return t[a:b]
    return t.view((chunks, n) + tuple(t.shape[1:]))[:, a:b]


def _cross_halves(layout: ShardLayout, send: Optional[torch.Tensor], recv: Optional[torch.Tensor], chunks: int) -> None:
    """One batched ``send_recv`` with the peers of ``layout`` (the other CFG half's ranks whose frames overlap this
    rank's): each gets the rows of ``send`` of the frames it shares with this rank, and the rows of ``recv`` of those
    frames are filled from it.  ``send`` / ``recv`` are ``(chunk, frame)``-major ``[chunks * n_local, ...]``; every size
    is a host int of the layout, so nothing reads from the device."""
    n = layout.hi - layout.lo
    sends, recvs, copies = [], [], []
    for peer, a, b in layout.peers:
        a, b = a - layout.lo, b - layout.lo
        if send is not None:
            sends.append((_peer_rows(send, chunks, n, a, b).contiguous(), peer))
        if recv is not None:
            dst = _peer_rows(recv, chunks, n, a, b)
            buf = dst if dst.is_contiguous() else torch.empty(dst.shape, dtype=dst.dtype, device=dst.device)
            recvs.append((buf, peer))
            copies.append((dst, buf))
    send_recv(sends, recvs, unpack(layout.shard)[2])
    for dst, buf in copies:
        if buf is not dst:
            dst.copy_(buf)


def chunk_frames(t: Optional[torch.Tensor], chunks: int, n_frames: int, lo: int, hi: int) -> Optional[torch.Tensor]:
    """Frames [lo, hi) of each CFG chunk of a ``(chunk, frame)``-major batch ``[chunks * n_frames, ...]`` (prompt
    embeddings, ControlNet edges).  Anything not laid out that way (None, one prompt shared by all frames) and the
    whole range come back as they are."""
    if t is None or t.shape[0] != chunks * n_frames or hi - lo == n_frames:
        return t
    return t.view(chunks, n_frames, *t.shape[1:])[:, lo:hi].reshape(chunks * (hi - lo), *t.shape[1:])


def all_gather_blocks(t: torch.Tensor, world: int, group=None) -> torch.Tensor:
    """``[world, *t.shape]``: every rank's ``t`` in rank order (one all-gather)"""
    t = t.contiguous()
    out = torch.empty((world,) + tuple(t.shape), dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(out.view(-1, *t.shape[1:]), t, group=group)
    return out


def all_gather_frames(t: torch.Tensor, n_frames: int, world: int, chunks: int = 1, group=None) -> torch.Tensor:
    """``[chunks * N, ...]``: the whole ``(chunk, frame)``-major batch from every rank's ``t = [chunks * n_r, ...]``
    (its ``frame_range`` block of each chunk).  Every block is padded to the largest share, one all-gather moves them,
    and the padding is dropped; the shares are host ints, so nothing reads from the device."""
    sizes = block_sizes(n_frames, world)
    per = max(sizes)
    inner = tuple(t.shape[1:])
    mine = t.shape[0] // chunks
    if mine == per:
        send = t
    else:
        send = torch.zeros((chunks, per) + inner, dtype=t.dtype, device=t.device)
        send[:, :mine] = t.reshape((chunks, mine) + inner)
    full = all_gather_blocks(send.reshape((chunks * per,) + inner), world, group).view((world, chunks, per) + inner)
    if min(sizes) == per:
        return full.transpose(0, 1).reshape((chunks * n_frames,) + inner)
    return torch.cat([full[r, :, :sizes[r]] for r in range(world)], 1).reshape((chunks * n_frames,) + inner)


class RingComm:
    """Neighbour exchange of the frame ring (SURVEY 8e, exchange 3): ``shift(send, recv, +1)`` sends ``send`` to rank+1
    and fills ``recv`` from rank-1 (``-1``: the other way round).  One batched NCCL send/recv pair on the current
    stream: no host synchronisation, capturable in a CUDA graph.  Tests inject an object with the same method."""

    def __init__(self, world: int, rank: int, group=None):
        self.world, self.rank, self.group = world, rank, group

    def _peer(self, r: int) -> int:
        r %= self.world
        return dist.get_global_rank(self.group, r) if self.group is not None else r

    def shift(self, send: torch.Tensor, recv: torch.Tensor, direction: int) -> None:
        dst, src = self._peer(self.rank + direction), self._peer(self.rank - direction)
        send_recv([(send, dst)], [(recv, src)], self.group)

    def all_reduce_sum(self, t: torch.Tensor) -> None:
        dist.all_reduce(t, group=self.group)


class _OpsBackend:
    """the product path: hand-written sm_90a kernels"""

    def kv_compact_packed(self, k, v, idx, kv_out, chunks):
        from . import ops
        return ops.kv_compact_packed(k, v, idx, kv_out, chunks)

    def rows_gather(self, src, idx, dst, dst_col=0):
        from . import ops
        return ops.rows_gather(src, idx, dst, dst_col)

    def rows_scatter(self, src, idx, dst):
        from . import ops
        return ops.rows_scatter(src, idx, dst)

    def attn_fwd(self, q, k, v, heads, q_per_kv, softmax_scale, diag_bias=0.0):
        from . import ops
        return ops.attn_fwd(q, k, v, heads, q_per_kv, softmax_scale=softmax_scale, diag_bias=diag_bias)

    def attn_fwd_kv_packed(self, q, kv, heads, q_per_kv, softmax_scale):
        from . import ops
        return ops.attn_fwd_kv_packed(q, kv, heads, q_per_kv, softmax_scale)

    def temporal_attn_fwd(self, q, k, v, fwd_map, traj_mask, chunks, heads, scale):
        from . import ops
        return ops.temporal_attn_fwd(q, k, v, fwd_map, traj_mask, chunks, heads, scale)

    def temporal_attn_fwd_packed(self, qkv, fwd_map, traj_mask, chunks, heads, scale):
        from . import ops
        return ops.temporal_attn_fwd_packed(qkv, fwd_map, traj_mask, chunks, heads, scale)


class ShardedKVExchange:
    """Per-batch plan + per-layer all-gather of the compacted cross-frame K/V (SURVEY 8e, exchange 1)."""

    def __init__(self, attn_mask: torch.Tensor, world: int, rank: int, chunks: int, group=None):
        n_frames, tokens = attn_mask.shape
        self.world, self.rank, self.group, self.chunks = world, rank, group, chunks
        self.lo, self.hi = frame_range(n_frames, world, rank)
        per_frame = attn_mask.sum(1).tolist()                               # one host sync per batch and resolution
        counts = [int(sum(per_frame[lo:hi])) for lo, hi in (frame_range(n_frames, world, r) for r in range(world))]
        self.counts = counts
        self.max_count = max(max(counts), 1)
        self.total = sum(counts)
        dev = attn_mask.device
        local = attn_mask[self.lo:self.hi].reshape(-1)
        self.local_idx = torch.nonzero(local, as_tuple=False).reshape(-1).to(torch.int32).contiguous()
        # row (b, i) of the dense result  <-  row ((r*chunks + b)*max_count + j) of the gathered buffer
        rows = []
        for b in range(chunks):
            for r in range(world):
                rows.append((r * chunks + b) * self.max_count + torch.arange(counts[r], dtype=torch.int64))
        self.unpad_idx = torch.cat(rows).to(torch.int32).to(dev).contiguous()
        self._bufs = {}

    def _buffers(self, C: int, like: torch.Tensor):
        key = (C, like.dtype)
        if key not in self._bufs:
            send = torch.empty(self.chunks, self.max_count, 2 * C, dtype=like.dtype, device=like.device)
            gathered = torch.empty(self.world, self.chunks, self.max_count, 2 * C, dtype=like.dtype, device=like.device)
            self._bufs[key] = (send, gathered)
        return self._bufs[key]

    def exchange(self, k_local: torch.Tensor, v_local: torch.Tensor, backend) -> torch.Tensor:
        """k_local, v_local [chunks * N_local, L, C] -> kv [chunks, Lk_global, 2C] (K | V per row)"""
        C = k_local.shape[-1]
        send, gathered = self._buffers(C, k_local)
        if self.counts[self.rank] > 0:
            backend.kv_compact_packed(k_local, v_local, self.local_idx, send, self.chunks)
        if self.world == 1:
            return send                                                     # max_count == total: nothing to drop
        dist.all_gather_into_tensor(gathered.view(-1, self.max_count, 2 * C), send, group=self.group)   # rank-major concat
        kv = torch.empty(self.chunks, self.total, 2 * C, dtype=k_local.dtype, device=k_local.device)
        backend.rows_gather(gathered.view(-1, 2 * C), self.unpad_idx, kv.view(-1, 2 * C))
        return kv


class ShardedTrajectoryExchange:
    """Per-batch plan of the trajectory-sharded temporal-guided attention (SURVEY 8e, exchange 2)."""

    def __init__(self, fwd_map: torch.Tensor, traj_mask: torch.Tensor, world: int, rank: int, chunks: int, group=None):
        """fwd_map int64 [N, L] (trajectory p visits token fwd_map[f, p] of frame f); traj_mask uint8 [L, N, N].  Rank s
        owns frames ``frame_range(N, world, s)`` and trajectories ``frame_range(L, world, s)``; neither has to split
        evenly."""
        N, L = fwd_map.shape
        self.world, self.rank, self.group, self.chunks = world, rank, group, chunks
        self.N, self.L = N, L
        lo, hi = frame_range(N, world, rank)
        n_local = hi - lo
        self.n_local = n_local
        traj = [frame_range(L, world, s) for s in range(world)]
        t_lo, t_hi = traj[rank]
        self.Lg = t_hi - t_lo
        frames = block_sizes(N, world)
        # all_to_all split sizes in rows, fixed for the batch: to rank s go my frames' rows of its trajectories; from
        # rank r come r's frames' rows of mine
        self.send_splits = [n_local * chunks * (b - a) for a, b in traj]
        self.recv_splits = [f * chunks * self.Lg for f in frames]
        dev = fwd_map.device
        # send row (s, j, b, t)  <-  local row (b * n_local + j) * L + fwd_map[lo + j, traj[s][0] + t]
        brow = (torch.arange(chunks, device=dev)[None, :] * n_local + torch.arange(n_local, device=dev)[:, None]) * L   # [j, b]
        idx = [(fwd_map[lo:hi, a:b][:, None, :] + brow[:, :, None]).reshape(-1) for a, b in traj]   # [j, b, t] per s
        self.row_idx = torch.cat(idx).to(torch.int32).contiguous()
        self.identity_map = torch.arange(chunks * self.Lg, device=dev, dtype=torch.int64)[None].expand(N, -1).contiguous()
        mine = traj_mask[t_lo:t_hi]                                                           # [Lg, N, N]
        self.mask = mine[None].expand(chunks, -1, -1, -1).reshape(chunks * self.Lg, N, N).contiguous()
        self._bufs = {}

    def _buffers(self, C: int, like: torch.Tensor):
        key = (C, like.dtype)
        if key not in self._bufs:
            mk = lambda n, w: torch.empty(n, w, dtype=like.dtype, device=like.device)
            local, mine = self.n_local * self.chunks * self.L, self.N * self.chunks * self.Lg
            self._bufs[key] = (mk(local, 3 * C), mk(mine, 3 * C), mk(local, C))
        return self._bufs[key]

    def run(self, q, k, attn_out, heads: int, scale: float, backend) -> torch.Tensor:
        """q, k, attn_out [chunks * N_local, L, C] (local frames) -> temporal-guided output, same shape"""
        B, L, C = q.shape
        send, recv, back = self._buffers(C, q)
        for col, t in enumerate((q, k, attn_out)):
            backend.rows_gather(t.view(-1, C), self.row_idx, send, col * C)
        dist.all_to_all_single(recv, send, self.recv_splits, self.send_splits, group=self.group)
        # recv rows are ordered (source rank r, its frame j, chunk b, trajectory t) = (global frame, chunk * Lg + t)
        res = backend.temporal_attn_fwd_packed(recv.view(self.N, self.chunks * self.Lg, 3 * C), self.identity_map, self.mask,
                                               1, heads, scale)
        dist.all_to_all_single(back, res.view(-1, C), self.send_splits, self.recv_splits, group=self.group)
        out = torch.empty_like(attn_out)
        backend.rows_scatter(back, self.row_idx, out.view(-1, C))
        return out


class ShardedFRESCOAttention:
    """FRESCO self-attention of one layer on a frame shard (the sharded counterpart of
    ``FRESCOAttnProcessor2_0._fresco_self_attention``)."""

    def __init__(self, controller, world: int, rank: int, chunks: int = 2, group=None, backend=None):
        self.ctrl, self.world, self.rank, self.chunks, self.group = controller, world, rank, chunks, group
        self.backend = backend if backend is not None else _OpsBackend()
        self._plans = {}
        self._traj_plans = {}

    def _plan(self, tokens: int) -> Optional[ShardedKVExchange]:
        """Exchange plan for the mask with ``shape[1] == tokens``; rebuilt whenever the controller holds a different
        mask tensor (enable_cfattn(new_mask) for the next keyframe batch), validated by identity."""
        chosen = None
        if self.ctrl.attn_mask is not None:
            for m in self.ctrl.attn_mask:
                if m.shape[1] == tokens:
                    chosen = m
        hit = self._plans.get(tokens)
        if hit is None or hit[0] is not chosen:
            plan = None if chosen is None else ShardedKVExchange(chosen, self.world, self.rank, self.chunks, self.group)
            hit = (chosen, plan)
            self._plans[tokens] = hit
        return hit[1]

    def _traj_plan(self, tokens: int) -> ShardedTrajectoryExchange:
        traj = self.ctrl.trajectories(tokens)
        if traj is None:
            raise RuntimeError(f"temporal-guided attention enabled but no mapping matches {tokens} tokens")
        hit = self._traj_plans.get(tokens)
        if hit is None or hit[0] is not traj[0]:
            hit = (traj[0], ShardedTrajectoryExchange(traj[0], traj[1], self.world, self.rank, self.chunks, self.group))
            self._traj_plans[tokens] = hit
        return hit[1]

    def __call__(self, q, k, v, heads: int, ref_q=None, ref_k=None):
        """q, k, v: [chunks * N_local, L, C] projections of the local frames; ref_q / ref_k: projections of the
        stored reference features (spatial-guided attention) or None.  Returns [chunks * N_local, L, C]."""
        ctrl, be, chunks = self.ctrl, self.backend, self.chunks
        B, L, C = q.shape
        n_local = B // chunks
        d = C // heads
        inv = 1.0 / math.sqrt(d)
        q_main = q
        if ctrl.use_intraattn and ref_q is not None:
            q_main = be.attn_fwd(ref_q, ref_k, q, heads, 1, ctrl.intraattn_scale_factor * inv, float(ctrl.intraattn_bias))
        if ctrl.use_cfattn:
            plan = self._plan(L)
            if plan is None:
                # no mask at this resolution: everybody attends global frame 0 (owned by rank 0)
                k0 = k.view(chunks, n_local, L, C)[:, 0].contiguous()
                v0 = v.view(chunks, n_local, L, C)[:, 0].contiguous()
                if self.world > 1:
                    kv = torch.stack([k0, v0])
                    src = dist.get_global_rank(self.group, 0) if self.group is not None else 0
                    dist.broadcast(kv, src=src, group=self.group)
                    k0, v0 = kv[0], kv[1]
                out = be.attn_fwd(q_main, k0, v0, heads, n_local, inv)
            else:
                kv = plan.exchange(k, v, be)
                out = be.attn_fwd_kv_packed(q_main, kv, heads, n_local, inv)
        else:
            out = be.attn_fwd(q_main, k, v, heads, 1, inv)
        if ctrl.use_interattn:
            scale = ctrl.interattn_scale_factor * inv
            if self.world == 1:
                traj = ctrl.trajectories(L)
                if traj is None:
                    raise RuntimeError(f"temporal-guided attention enabled but no mapping matches {L} tokens")
                out = be.temporal_attn_fwd(q, k, out, traj[0], traj[1], chunks, heads, scale)
            else:
                out = self._traj_plan(L).run(q, k, out, heads, scale, be)
        return out
