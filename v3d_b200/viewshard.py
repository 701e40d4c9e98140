"""View-sharding ONE image across GPUs: the T view-frames of a video are split into contiguous blocks, one block
per rank (BASELINE.json configs[2-3]; SURVEY.md 8(e)).

Everything that is per-frame or per-token stays rank-local (all spatial layers, the temporal feed-forwards and
projections: ~93 % of the UNet's FLOPs).  Three things couple the frames and each gets one exchange:

  * temporal self-attention (video_attention.py:114-125 around attention.py:337-341): every query frame attends to
    the keys/values of all T frames -> all-gather of the packed K|V rows (`gather_rows`), consumed in place by
    v3d_attention_temporal_kv through a per-frame row table (`kv_table`), so uneven blocks need no compaction;
  * the (3,1,1) temporal convolutions (video_model.py:42-55, temporal_ae.py:94-99): one halo frame from each
    neighbour (`exchange_halos`); the video's first / last frame keep the reference's ZERO padding;
  * the 3-D GroupNorms of the time_stack ResBlocks (openaimodel.py:267-271 with dims=3): (sum, sum of squares)
    all-reduce of the fp64 statistics (`allreduce_stats_`); in deterministic mode an all-gather of the block partials
    instead (`allgather_partials_`), folded over the whole video in one fixed order on every rank.

The CFG pair [uc; c] of a frame lives on the same rank, so the guidance combine and the Euler update are local.
Two transports carry the exchanges.  `PeerTransport` (default when the group runs over NCCL, i.e. one GPU per rank
on one box): one-sided stores into IPC-mapped peer memory with epoch flags (csrc/peer.cu) - no NCCL call on the data
path, the whole sharded forward is stream-ordered and CUDA-graph capturable.  torch.distributed collectives otherwise
(V3D_SHARD_TRANSPORT=nccl; gloo in the CPU tests, and - staged through host memory - for 2 processes sharing one GPU in
tests/test_viewshard_gpu.py).  The final decoded-frame gather is always a torch.distributed all-gather.
"""
from __future__ import annotations

import copy
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist


def partition_frames(num_frames: int, world: int) -> List[Tuple[int, int]]:
    """Contiguous (first frame, count) per rank; the first `num_frames % world` ranks take one extra frame.
    T=18: 2 ranks 9/9, 4 ranks 5/5/4/4, 8 ranks 3/3/2/2/2/2/2/2."""
    if world <= 0 or num_frames < world:
        raise ValueError(f"cannot split {num_frames} frames over {world} ranks (every rank needs a frame)")
    base, rem = divmod(num_frames, world)
    out, start = [], 0
    for r in range(world):
        n = base + (1 if r < rem else 0)
        out.append((start, n))
        start += n
    return out


class _RawCuda:
    """__cuda_array_interface__ view of raw device memory (an arena from v3d_peer_alloc) for torch.as_tensor."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3}


class PeerTransport:
    """One-sided exchanges over NVLink peer memory (csrc/peer.cu, include/v3d_b200.h "One-sided exchanges"): the
    transport of a frame-sharded / CFG-split group when its ranks sit on GPUs of one box.

    Every rank owns arena chunks of identical layout (sizes are computed from the LARGEST frame block, so offsets agree
    on all ranks); the other ranks map them through IPC handles exchanged once per chunk over torch.distributed.  An
    exchange SITE (one K|V gather, one halo exchange, one statistics all-reduce of the launch schedule) owns its flag
    words and - for the big buffers - one of two rotating buffers per shape; sites are created in program order on the
    first (eager) pass of a scope and looked up by position afterwards, which is what lets the sharded forward be
    captured into a CUDA graph: the kernels carry arena addresses, the flag values come from a device epoch word that
    `begin()` increments on the stream.

    Why two rotating buffers are enough: a neighbour overwrites the buffer of my site s + 2 only after it waited for my
    signal of site s + 1, which my stream issues after the kernels that read site s (every site is a bidirectional
    exchange with the ranks involved, in the same program order on all of them).  Flags, statistics slots and CFG halves
    never rotate faster than that either (unique per site; the CFG gather alternates two sites)."""

    CHUNK = 1 << 30

    def __init__(self, group, device: torch.device):
        from . import _lib

        self.lib = _lib.load()
        self.check = _lib.check
        self.group, self.dev = group, device
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        if self.world > 8:
            raise RuntimeError("peer transport: at most 8 ranks (one NVSwitch box)")
        self.chunks: List[Tuple[int, List[int], torch.Tensor]] = []   # (bytes, [base pointer per rank], local u8 view)
        self.cur, self.off = -1, 0
        self.ctrl = torch.zeros(64, device=device, dtype=torch.int32)   # [0] epoch, [1] status, [2] put counter
        self.scopes: Dict[str, List[dict]] = {}
        self.scope, self.pos = "", 0
        self.rot: Dict[tuple, list] = {}
        self.nsites = 0

    # ---- arena ----------------------------------------------------------------------------------
    def _new_chunk(self, need: int) -> None:
        import ctypes as C

        nbytes = max(self.CHUNK, (need + 0xFFFFF) & ~0xFFFFF)
        ptr = C.c_void_p()
        self.check(self.lib.v3d_peer_alloc(nbytes, C.byref(ptr)), "v3d_peer_alloc")
        handle = C.create_string_buffer(64)
        self.check(self.lib.v3d_peer_export(ptr, handle), "v3d_peer_export")
        mine = (os.getpid(), bytes(handle.raw))
        every = [None] * self.world
        dist.all_gather_object(every, mine, group=self.group)
        bases = []
        for r, (pid, h) in enumerate(every):
            if r == self.rank:
                bases.append(ptr.value)
                continue
            q = C.c_void_p()
            self.check(self.lib.v3d_peer_import(C.create_string_buffer(h, 64), C.byref(q)), "v3d_peer_import")
            bases.append(q.value)
        view = torch.as_tensor(_RawCuda(ptr.value, nbytes), device=self.dev)
        self.chunks.append((nbytes, bases, view))
        self.cur, self.off = len(self.chunks) - 1, 0

    def _take(self, nbytes: int) -> Tuple[int, int]:
        """-> (chunk, offset) of `nbytes` (256-byte aligned) at the same place in every rank's arena"""
        nbytes = (nbytes + 255) & ~255
        if self.cur < 0 or self.off + nbytes > self.chunks[self.cur][0]:
            self._new_chunk(nbytes)
        off = self.off
        self.off += nbytes
        return self.cur, off

    def _addr(self, loc: Tuple[int, int], rank: int, extra: int = 0) -> int:
        return self.chunks[loc[0]][1][rank] + loc[1] + extra

    def _view(self, loc: Tuple[int, int], nbytes: int) -> torch.Tensor:
        return self.chunks[loc[0]][2][loc[1]:loc[1] + nbytes]

    def _rotating(self, kind: str, nbytes: int) -> Tuple[int, int]:
        key = (self.scope, kind, nbytes)
        ent = self.rot.setdefault(key, [[], 0])
        if len(ent[0]) < 2:
            ent[0].append(self._take(nbytes))
        loc = ent[0][ent[1] % len(ent[0])] if len(ent[0]) == 2 else ent[0][-1]
        ent[1] += 1
        return loc

    # ---- sites ----------------------------------------------------------------------------------
    def begin(self, scope: str) -> None:
        """Start of a pass over one launch schedule (a UNet forward, a decode, a CFG gather): rewinds the site cursor
        of that scope and bumps the epoch ON THE STREAM (captured with the rest of the pass)."""
        self.scope, self.pos = scope, 0
        self.scopes.setdefault(scope, [])
        self.check(self.lib.v3d_peer_epoch_bump(self.ctrl.data_ptr(), _stream_of(self.dev)), "v3d_peer_epoch_bump")

    def _site(self, kind: str, sig: tuple, make) -> dict:
        sites = self.scopes[self.scope]
        if self.pos == len(sites):
            st = make()
            st.update(kind=kind, sig=sig, id=self.nsites)
            self.nsites += 1
            sites.append(st)
        st = sites[self.pos]
        if st["kind"] != kind or st["sig"] != sig:
            raise RuntimeError(f"peer transport: exchange #{self.pos} of scope {self.scope!r} changed from "
                               f"{st['kind']}{st['sig']} to {kind}{sig}; the launch schedule must be static")
        self.pos += 1
        return st

    def _flags(self, n: int) -> Tuple[int, int]:
        return self._take(4 * max(n, 1))

    # ---- the three exchanges ----------------------------------------------------------------------
    def _put(self, segs: List[Tuple[int, int, int]], flags: List[int]) -> None:
        import ctypes as C

        n, m = len(segs), len(flags)
        src = (C.c_void_p * max(n, 1))(*[s for s, _, _ in segs])
        dst = (C.c_void_p * max(n, 1))(*[d for _, d, _ in segs])
        nb = (C.c_int64 * max(n, 1))(*[b for _, _, b in segs])
        fl = (C.c_void_p * max(m, 1))(*flags)
        self.check(self.lib.v3d_peer_put(n, src, dst, nb, m, fl, self.ctrl.data_ptr(), self.ctrl.data_ptr() + 8,
                                         _stream_of(self.dev)), "v3d_peer_put")

    def _wait(self, flags: List[int], site: int) -> None:
        import ctypes as C

        fl = (C.c_void_p * len(flags))(*flags)
        self.check(self.lib.v3d_peer_wait(len(flags), fl, self.ctrl.data_ptr(), self.ctrl.data_ptr() + 4, site,
                                          _stream_of(self.dev)), "v3d_peer_wait")

    def allreduce_f64_(self, stats: torch.Tensor, scale: float) -> torch.Tensor:
        import ctypes as C

        n = stats.numel()
        st = self._site("allreduce", (n,), lambda: {"slots": self._take(8 * n * self.world), "flags": self._flags(self.world)})
        slot = (C.c_void_p * self.world)(*[self._addr(st["slots"], r) for r in range(self.world)])
        flag = (C.c_void_p * self.world)(*[self._addr(st["flags"], r) for r in range(self.world)])
        self.check(self.lib.v3d_peer_allreduce_f64(stats.data_ptr(), n, scale, self.world, self.rank, slot, flag,
                                                   self.ctrl.data_ptr(), self.ctrl.data_ptr() + 4, st["id"],
                                                   _stream_of(self.dev)), "v3d_peer_allreduce_f64")
        return stats

    def partials(self, nb: int, nblk: int, groups: int) -> torch.Tensor:
        """Block-partial buffer [nb, nblk, groups, 2] fp32 of one deterministic 3-D GroupNorm (the whole video's
        blocks), in the arena; unique per site, like the statistics slots."""
        nbytes = 8 * nb * nblk * groups
        st = self._site("partials", (nb, nblk, groups), lambda: {"buf": self._take(nbytes), "flags": self._flags(self.world)})
        t = self._view(st["buf"], nbytes).view(torch.float32).view(nb, nblk, groups, 2)
        t._v3d_site = st
        return t

    def allgather_partials(self, part: torch.Tensor, first_block: int, nblocks: int) -> None:
        """This rank's blocks [first_block, first_block + nblocks) of every video -> the same place in every other
        rank's buffer; then wait until every rank's blocks have landed here."""
        st = part._v3d_site
        nb, nblk = part.shape[0], part.shape[1]
        bb = part[0, 0].numel() * part.element_size()                # bytes per block
        others = [r for r in range(self.world) if r != self.rank]
        segs = []
        for r in others:
            for b in range(nb):
                off = (b * nblk + first_block) * bb
                segs.append((self._addr(st["buf"], self.rank, off), self._addr(st["buf"], r, off), nblocks * bb))
        if len(segs) > 16:
            raise RuntimeError(f"peer transport: a partials all-gather of {nb} videos over {self.world} ranks needs "
                               f"{len(segs)} segments (at most 16)")
        self._put(segs, [self._addr(st["flags"], r, 4 * self.rank) for r in others])
        self._wait([self._addr(st["flags"], self.rank, 4 * r) for r in others], st["id"])

    def pad(self, shape: Tuple[int, ...], cap_shape: Tuple[int, ...], dtype: torch.dtype) -> torch.Tensor:
        """Halo'd operand buffer [nb, tl + 2, ...] living in the arena (capacity for the largest block)."""
        es = torch.empty(0, dtype=dtype).element_size()
        cap = es * _prod(cap_shape)
        st = self._site("pad", tuple(shape) + (str(dtype),), lambda: {"buf": self._rotating("pad", cap), "flags": self._flags(2)})
        t = self._view(st["buf"], es * _prod(shape)).view(dtype).view(*shape)
        t._v3d_site = st           # exchange_halos finds its site through the tensor
        return t

    def exchange_halos(self, pad: torch.Tensor, blocks: List[Tuple[int, int]]) -> None:
        st = pad._v3d_site
        nb, tl = pad.shape[0], pad.shape[1] - 2
        fbytes = pad[0, 0].numel() * pad.element_size()          # one frame of one batch item
        prev_r, next_r = self.rank - 1, self.rank + 1
        if prev_r < 0:
            pad[:, 0].zero_()
        if next_r >= self.world:
            pad[:, tl + 1].zero_()
        segs, flags, waits = [], [], []
        base = self._addr(st["buf"], self.rank)
        for peer, send_f, recv_f_of_peer, their_flag, my_flag in (
                (prev_r, 1, lambda n: n + 1, 1, 0),      # my first frame -> prev's right halo; I wait on flag 0
                (next_r, tl, lambda n: 0, 0, 1)):        # my last frame  -> next's left halo;  I wait on flag 1
            if peer < 0 or peer >= self.world:
                continue
            ptl = blocks[peer][1]
            for b in range(nb):
                segs.append((base + (b * (tl + 2) + send_f) * fbytes,
                             self._addr(st["buf"], peer, (b * (ptl + 2) + recv_f_of_peer(ptl)) * fbytes), fbytes))
            flags.append(self._addr(st["flags"], peer, 4 * their_flag))
            waits.append(self._addr(st["flags"], self.rank, 4 * my_flag))
        self._put(segs, flags)
        self._wait(waits, st["id"])

    def kv_slots(self, block_rows: int, width: int, dtype: torch.dtype) -> Tuple[torch.Tensor, torch.Tensor]:
        """-> (gather buffer [world * block_rows, width] in the arena, this rank's slot of it)"""
        es = torch.empty(0, dtype=dtype).element_size()
        nbytes = es * block_rows * width
        st = self._site("kv", (block_rows, width, str(dtype)),
                        lambda: {"buf": self._rotating("kv", nbytes * self.world), "flags": self._flags(self.world)})
        buf = self._view(st["buf"], nbytes * self.world).view(dtype).view(self.world * block_rows, width)
        buf._v3d_site = st
        return buf, buf[self.rank * block_rows:(self.rank + 1) * block_rows]

    def gather_rows(self, buf: torch.Tensor, filled_rows: int) -> torch.Tensor:
        """This rank's slot (its first `filled_rows` rows) -> the same slot of every other rank's buffer."""
        st = buf._v3d_site
        block_rows = buf.shape[0] // self.world
        slot = self.rank * block_rows * buf.shape[1] * buf.element_size()
        nbytes = filled_rows * buf.shape[1] * buf.element_size()
        src = self._addr(st["buf"], self.rank, slot)
        segs = [(src, self._addr(st["buf"], r, slot), nbytes) for r in range(self.world) if r != self.rank]
        flags = [self._addr(st["flags"], r, 4 * self.rank) for r in range(self.world) if r != self.rank]
        self._put(segs, flags)
        self._wait([self._addr(st["flags"], self.rank, 4 * r) for r in range(self.world) if r != self.rank], st["id"])
        return buf

    def kv_destinations(self, buf: torch.Tensor) -> List[int]:
        """Address of THIS rank's slot in every rank's copy of the gather buffer (own arena included): the destination
        matrices of the fused projection-GEMM -> all-gather (`ops.gemm(..., kv=...)`)."""
        st = buf._v3d_site
        block_rows = buf.shape[0] // self.world
        slot = self.rank * block_rows * buf.shape[1] * buf.element_size()
        return [self._addr(st["buf"], r, slot) for r in range(self.world)]

    def gather_signal(self, buf: torch.Tensor) -> torch.Tensor:
        """After a GEMM that scattered its K|V columns into every rank's buffer: raise this rank's flag on the peers
        and wait for theirs (no data moves here)."""
        st = buf._v3d_site
        others = [r for r in range(self.world) if r != self.rank]
        self._put([], [self._addr(st["flags"], r, 4 * self.rank) for r in others])
        self._wait([self._addr(st["flags"], self.rank, 4 * r) for r in others], st["id"])
        return buf

    def gather_halves(self, mine: torch.Tensor, parity: int) -> torch.Tensor:
        """CFG pair: [n, ...] per rank -> [2n, ...] on both (rank order).  `parity` alternates two sites."""
        nbytes = mine.numel() * mine.element_size()
        st = self._site("cfg", (tuple(mine.shape), str(mine.dtype), parity),
                        lambda: {"buf": self._take(2 * nbytes), "flags": self._flags(2)})
        out = self._view(st["buf"], 2 * nbytes).view(mine.dtype).view((2 * mine.shape[0],) + tuple(mine.shape[1:]))
        segs = [(mine.data_ptr(), self._addr(st["buf"], r, self.rank * nbytes), nbytes) for r in range(2)]
        self._put(segs, [self._addr(st["flags"], 1 - self.rank, 4 * self.rank)])
        self._wait([self._addr(st["flags"], self.rank, 4 * (1 - self.rank))], st["id"])
        return out

    def status(self) -> int:
        """0, or 0x80000000 | site id of an exchange whose signal never arrived (host sync)"""
        return int(self.ctrl[1].item()) & 0xFFFFFFFF


def _prod(shape) -> int:
    n = 1
    for d in shape:
        n *= int(d)
    return n


def _stream_of(dev: torch.device) -> int:
    return torch.cuda.current_stream(dev).cuda_stream


def _want_peer(group, device) -> bool:
    """V3D_SHARD_TRANSPORT = peer | nccl (default: peer when the group runs over NCCL, i.e. one GPU per rank)."""
    mode = os.environ.get("V3D_SHARD_TRANSPORT", "auto")
    if mode == "nccl" or device is None or device.type != "cuda" or dist.get_world_size(group) < 2:
        return False
    return mode == "peer" or dist.get_backend(group) == "nccl"


@dataclass
class ViewShard:
    """This rank's block of a T-frame video and the exchanges that stitch the blocks together."""

    num_frames: int                      # T of the whole video
    rank: int
    world: int
    group: Optional[object] = None       # torch.distributed process group (None = default group)
    blocks: List[Tuple[int, int]] = field(default_factory=list)
    exchanges: Dict[str, int] = field(default_factory=dict)  # per-kind call counters (bench / tests)
    peer: Optional[PeerTransport] = None  # one-sided NVLink transport (None: torch.distributed collectives)

    @classmethod
    def create(cls, num_frames: int, group=None, device: Optional[torch.device] = None) -> "ViewShard":
        if not dist.is_initialized():
            raise RuntimeError("ViewShard.create needs an initialised torch.distributed process group")
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        vs = cls(num_frames, rank, world, group, partition_frames(num_frames, world))
        vs.attach_peer(device)
        return vs

    def attach_peer(self, device: Optional[torch.device] = None) -> None:
        """Switch the exchanges of this group to the one-sided peer-memory transport when it applies (V3D_SHARD_TRANSPORT;
        default: the group runs over NCCL, i.e. one GPU per rank on one box)."""
        if device is None and torch.cuda.is_available() and (
                dist.get_backend(self.group) == "nccl" or os.environ.get("V3D_SHARD_TRANSPORT") == "peer"):
            device = torch.device("cuda", torch.cuda.current_device())
        if self.peer is None and self.world > 1 and _want_peer(self.group, device):
            self.peer = PeerTransport(self.group, device)

    def begin(self, scope: str) -> None:
        """start of a pass over a launch schedule that uses this shard's exchanges (UNet forward / decode)"""
        if self.peer is not None:
            self.peer.begin(scope)

    def new_pad(self, shape: Tuple[int, ...], dtype: torch.dtype, device) -> torch.Tensor:
        """[nb, tl + 2, ...] halo'd operand buffer: plain memory, or - peer transport - arena memory the neighbours
        write their boundary frames into"""
        if self.peer is None:
            return torch.empty(shape, device=device, dtype=dtype)
        return self.peer.pad(tuple(shape), (shape[0], self.tmax + 2) + tuple(shape[2:]), dtype)

    def kv_slots(self, nb: int, rows_per_frame: int, width: int, dtype: torch.dtype, device):
        """-> (gather buffer or None, the tensor this rank packs its K|V rows into)"""
        block_rows = nb * self.tmax * rows_per_frame
        if self.peer is None:
            return None, torch.empty(block_rows, width, device=device, dtype=dtype)
        return self.peer.kv_slots(block_rows, width, dtype)

    def __post_init__(self):
        if not self.blocks:
            self.blocks = partition_frames(self.num_frames, self.world)
        self._staged: Optional[bool] = None

    # ---- geometry -------------------------------------------------------------------------------
    @property
    def t0(self) -> int:
        return self.blocks[self.rank][0]

    @property
    def tl(self) -> int:
        return self.blocks[self.rank][1]

    @property
    def tmax(self) -> int:
        return max(n for _, n in self.blocks)

    @property
    def frames(self) -> slice:
        return slice(self.t0, self.t0 + self.tl)

    def kv_table(self, nb: int, rows_per_frame: int) -> Tuple[List[int], List[int]]:
        """Row offsets of every key frame in the buffer `gather_rows` returns for a [nb, tl, rows_per_frame] block
        per rank: frame f of video b, pixel s sits at row[f] + b * bstride[f] + s."""
        row, bstride = [], []
        block_rows = nb * self.tmax * rows_per_frame      # every rank's slot is padded to the largest block
        for r, (_, n) in enumerate(self.blocks):
            for j in range(n):
                row.append(r * block_rows + j * rows_per_frame)
                bstride.append(n * rows_per_frame)
        return row, bstride

    # ---- transport ------------------------------------------------------------------------------
    def _is_gloo(self) -> bool:
        if self._staged is None:
            self._staged = dist.get_backend(self.group) == "gloo"
        return self._staged

    def _via_host(self, t: torch.Tensor) -> bool:
        """gloo cannot move CUDA memory for every primitive: stage through the host (tests only; NCCL is direct)."""
        return self._is_gloo() and t.is_cuda

    def _count(self, kind: str) -> None:
        self.exchanges[kind] = self.exchanges.get(kind, 0) + 1

    def _global_rank(self, r: int) -> int:
        return r if self.group is None else dist.get_global_rank(self.group, r)

    def allreduce_stats_(self, stats: torch.Tensor) -> torch.Tensor:
        """stats: fp64 [nsamples, groups, 2] = local (sum, sumsq) of a 3-D GroupNorm.  After the call it holds the
        GLOBAL sums rescaled by tl / T, so that the apply kernel - which divides by the LOCAL element count - yields
        the global mean and variance."""
        self._count("gn_allreduce")
        if self.peer is not None:
            return self.peer.allreduce_f64_(stats, self.tl / self.num_frames)
        if self.world > 1:
            if self._via_host(stats):
                h = stats.cpu()
                dist.all_reduce(h, group=self.group)
                stats.copy_(h)
            else:
                dist.all_reduce(stats, group=self.group)
        stats.mul_(self.tl / self.num_frames)
        return stats

    def gn_partials(self, nb: int, nblk: int, device, groups: int = 32) -> torch.Tensor:
        """[nb, nblk, groups, 2] fp32 buffer for the block partials of a deterministic 3-D GroupNorm over the whole
        video (nblk = all T frames' blocks): plain memory, or - peer transport - arena memory the other ranks write
        their blocks into"""
        if self.peer is None:
            return torch.empty(nb, nblk, groups, 2, device=device, dtype=torch.float32)
        return self.peer.partials(nb, nblk, groups)

    def allgather_partials_(self, part: torch.Tensor, blocks_per_frame: int) -> torch.Tensor:
        """Deterministic mode's statistics exchange: part [nb, T * blocks_per_frame, groups, 2] holds this rank's
        frames' block partials at their global block offset; afterwards it holds every frame's, on every rank."""
        self._count("gn_allgather")
        if self.world == 1:
            return part
        nbf = blocks_per_frame
        if self.peer is not None:
            self.peer.allgather_partials(part, self.t0 * nbf, self.tl * nbf)
            return part
        nb = part.shape[0]
        send = part.new_zeros((nb, self.tmax * nbf) + tuple(part.shape[2:]))   # every rank's slot: the largest block
        send[:, :self.tl * nbf] = part[:, self.t0 * nbf:(self.t0 + self.tl) * nbf]
        out = part.new_empty((self.world * send.numel(),))
        if self._via_host(part):
            h = torch.empty(out.shape, dtype=out.dtype)
            dist.all_gather_into_tensor(h, send.reshape(-1).cpu(), group=self.group)
            out.copy_(h)
        else:
            dist.all_gather_into_tensor(out, send.reshape(-1), group=self.group)
        out = out.view((self.world,) + tuple(send.shape))
        for r, (t0, n) in enumerate(self.blocks):
            if r != self.rank:
                part[:, t0 * nbf:(t0 + n) * nbf] = out[r, :, :n * nbf]
        return part

    def exchange_halos(self, pad: torch.Tensor) -> torch.Tensor:
        """pad: [nb, tl + 2, ...] contiguous; frames 1..tl are this rank's, frame 0 / tl+1 receive the previous /
        next rank's last / first frame.  The ends of the video get zeros (Conv3d padding (1,0,0))."""
        self._count("halo")
        nb, tl = pad.shape[0], self.tl
        assert pad.shape[1] == tl + 2 and pad.is_contiguous()
        if self.peer is not None:
            self.peer.exchange_halos(pad, self.blocks)
            return pad
        prev_r, next_r = self.rank - 1, self.rank + 1
        if prev_r < 0:
            pad[:, 0].zero_()
        if next_r >= self.world:
            pad[:, tl + 1].zero_()
        if self.world == 1:
            return pad
        staged = self._via_host(pad)
        tagged = self._is_gloo()
        ops, landing = [], []
        for b in range(nb):
            for peer, send_idx, recv_idx, tag_s, tag_r in ((prev_r, 1, 0, 0, 1), (next_r, tl, tl + 1, 1, 0)):
                if peer < 0 or peer >= self.world:
                    continue
                src, dst = pad[b, send_idx], pad[b, recv_idx]
                if staged:
                    src = src.cpu()
                    host = torch.empty(dst.shape, dtype=dst.dtype)
                    landing.append((dst, host))
                    dst = host
                g = self._global_rank(peer)
                # a frame sent "towards lower ranks" (tag_s 0) is received by the peer as its right halo (tag_r 0).
                # Tags disambiguate the messages on gloo; NCCL matches sends and receives of a pair in issue order
                # (the order here is the same on both sides) and takes no tags.
                ts_, tr_ = (2 * b + tag_s, 2 * b + tag_r) if tagged else (0, 0)
                ops.append(dist.P2POp(dist.isend, src, g, group=self.group, tag=ts_))
                ops.append(dist.P2POp(dist.irecv, dst, g, group=self.group, tag=tr_))
        for w in dist.batch_isend_irecv(ops):
            w.wait()
        for dst, host in landing:
            dst.copy_(host)
        return pad

    def kv_fused(self, buf: Optional[torch.Tensor]):
        """None, or the destination addresses for the fused GEMM -> all-gather of the K|V projection (peer transport;
        V3D_KV_FUSED=0 falls back to pack + put)"""
        if buf is None or self.peer is None or os.environ.get("V3D_KV_FUSED", "1") == "0":
            return None
        return self.peer.kv_destinations(buf)

    def gather_signal(self, buf: torch.Tensor) -> torch.Tensor:
        self._count("kv_allgather")
        return self.peer.gather_signal(buf)

    def gather_rows(self, send: torch.Tensor, buf: Optional[torch.Tensor] = None,
                    filled_rows: Optional[int] = None) -> torch.Tensor:
        """send: [nb * tmax * rows_per_frame, W], of which this rank filled its first nb * tl * rows_per_frame rows
        (`kv_slots`).  Returns [world * rows, W] with rank r's block at r * rows (see `kv_table`)."""
        self._count("kv_allgather")
        if self.world == 1:
            return send
        if buf is not None:
            return self.peer.gather_rows(buf, send.shape[0] if filled_rows is None else filled_rows)
        out = send.new_empty((self.world * send.shape[0],) + tuple(send.shape[1:]))
        if self._via_host(send):
            h = torch.empty(out.shape, dtype=out.dtype)
            dist.all_gather_into_tensor(h, send.cpu(), group=self.group)
            out.copy_(h)
        else:
            dist.all_gather_into_tensor(out, send.contiguous(), group=self.group)
        return out

    def gather_frames(self, local: torch.Tensor) -> torch.Tensor:
        """[tl, ...] per rank -> [T, ...] on every rank in frame order (the final decoded-frame gather)."""
        self._count("frame_gather")
        if self.world == 1:
            return local
        pad = local.new_zeros((self.tmax,) + tuple(local.shape[1:]))
        pad[: self.tl] = local
        out = local.new_empty((self.world * self.tmax,) + tuple(local.shape[1:]))
        if self._via_host(local):
            h = torch.empty(out.shape, dtype=out.dtype)
            dist.all_gather_into_tensor(h, pad.cpu(), group=self.group)
            out.copy_(h)
        else:
            dist.all_gather_into_tensor(out, pad, group=self.group)
        out = out.reshape(self.world, self.tmax, *local.shape[1:])
        return torch.cat([out[r, :n] for r, (_, n) in enumerate(self.blocks)], dim=0)

    # ---- sampler-side slicing -------------------------------------------------------------------
    def shard_cond(self, cond: Dict) -> Dict:
        """Per-frame conditioning tensors ([T, ...]: vector, crossattn, concat) -> this rank's frames; other entries
        pass through (guiders.py:88-98 treats them as shared)."""
        out = {}
        for k, v in cond.items():
            if torch.is_tensor(v) and v.ndim > 0 and v.shape[0] == self.num_frames:
                out[k] = v[self.frames].contiguous()
            else:
                out[k] = v
        return out

    def time_context(self, c: Dict, uc: Dict) -> torch.Tensor:
        """The temporal cross-attention context is `context[::T]` = frame 0 of each CFG half
        (video_attention.py:250): [2, M, ctx] in [uc; c] order (M context tokens), the same on every rank."""
        return torch.cat([uc["crossattn"][:1], c["crossattn"][:1]], dim=0).contiguous()

    def shard_guider(self, guider):
        """Copy of a per-frame guider (guiders.py:60-146) restricted to this rank's frames."""
        if getattr(guider, "num_frames", 1) != self.num_frames:
            return guider  # VanillaCFG / IdentityGuider: one scale for every sample
        g = copy.copy(guider)
        g.num_frames = self.tl
        g.scale = guider.scale[:, self.frames].clone()
        if hasattr(g, "_scale_dev"):
            g._scale_dev = None
        return g


# ---------------------------------------------------------------------------------------------------------------------
# CFG-pair split: the second free axis of SURVEY.md 8(e)
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class CfgSplit:
    """The unconditional and the conditional half of the classifier-free-guidance batch (guiders.py:88-101, batch order
    [uc; c]) on two ranks: rank 0 of the pair evaluates the network on (x, uc), rank 1 on (x, c); one all-gather of the
    two denoised halves ([T, 4, h, w] fp32 each: 1.2 MB at V3D_512) per network evaluation puts [uc; c] on both ranks,
    which then apply the guidance and the sampler update redundantly.  25 small exchanges per image instead of the
    ~2600 of frame-sharding, and exactly the unsplit arithmetic (per-sample operators see the same samples)."""

    rank: int                         # 0 = uc half, 1 = c half
    group: Optional[object] = None
    exchanges: int = 0
    peer: Optional[PeerTransport] = None

    @classmethod
    def create(cls, group=None) -> "CfgSplit":
        if not dist.is_initialized() or dist.get_world_size(group) != 2:
            raise RuntimeError("CfgSplit needs a process group of exactly two ranks")
        cs = cls(dist.get_rank(group), group)
        cs.attach_peer()
        return cs

    def attach_peer(self, device: Optional[torch.device] = None) -> None:
        if device is None and torch.cuda.is_available() and (
                dist.get_backend(self.group) == "nccl" or os.environ.get("V3D_SHARD_TRANSPORT") == "peer"):
            device = torch.device("cuda", torch.cuda.current_device())
        if self.peer is None and _want_peer(self.group, device):
            self.peer = PeerTransport(self.group, device)

    def gather_halves(self, mine: torch.Tensor) -> torch.Tensor:
        """[n, ...] on each rank -> [2n, ...] = [rank 0's; rank 1's] on both."""
        self.exchanges += 1
        mine = mine.contiguous()
        if self.peer is not None and mine.is_cuda:
            parity = self.exchanges & 1           # two alternating sites: see PeerTransport (rotation argument)
            self.peer.begin(f"cfg{parity}")
            return self.peer.gather_halves(mine, parity)
        out = mine.new_empty((2 * mine.shape[0],) + tuple(mine.shape[1:]))
        if mine.is_cuda and dist.get_backend(self.group) == "gloo":      # tests: two processes sharing one GPU
            h = torch.empty(out.shape, dtype=out.dtype)
            dist.all_gather_into_tensor(h, mine.cpu(), group=self.group)
            out.copy_(h)
        else:
            dist.all_gather_into_tensor(out, mine, group=self.group)
        return out


class CfgSplitGuider:
    """Wraps a classifier-free guider so that each rank of a CfgSplit pair feeds the network only its half of
    `prepare_inputs`' [uc; c] batch and the guidance sees the all-gathered pair."""

    def __init__(self, inner, split: CfgSplit):
        if not hasattr(inner, "scale"):
            raise RuntimeError("CfgSplit needs a classifier-free guider ([uc; c] batch); got " + type(inner).__name__)
        self.inner, self.split = inner, split

    def prepare_inputs(self, x, s, c, uc):
        x2, s2, c2 = self.inner.prepare_inputs(x, s, c, uc)
        n, r = x.shape[0], self.split.rank
        half = slice(r * n, (r + 1) * n)
        cond = {k: (v[half] if torch.is_tensor(v) and v.ndim > 0 and v.shape[0] == 2 * n else v) for k, v in c2.items()}
        return x2[half], s2[half], cond

    def __call__(self, x_half, sigma):
        return self.inner(self.split.gather_halves(x_half), sigma)


@dataclass
class ShardPlan:
    """How ONE image is spread over the ranks of a job: `sample` = frame blocks of the sampler/UNet (None = all frames),
    `cfg` = CFG-pair split (None = both halves on every rank), `decode` = frame blocks of the first-stage decode (always
    set: the decode has no CFG axis, so with a CFG split every pair divides its frames once more).

        views      world = P      sample = decode = P frame blocks
        cfg        world = 2      sample = None, cfg pair = the two ranks, decode = 2 frame blocks
        cfg+views  world = 2 P    rank g = 2 v + r: frame block v of P, CFG half r; decode = each block split in two
    """

    mode: str
    num_frames: int
    sample: Optional[ViewShard]
    cfg: Optional[CfgSplit]
    decode: ViewShard

    @classmethod
    def create(cls, num_frames: int, mode: str = "views") -> "ShardPlan":
        if not dist.is_initialized():
            raise RuntimeError("ShardPlan.create needs an initialised torch.distributed process group")
        rank, world = dist.get_rank(), dist.get_world_size()
        if mode == "views":
            vs = ViewShard.create(num_frames)
            return cls(mode, num_frames, vs, None, vs)
        if mode == "cfg":
            if world != 2:
                raise RuntimeError("mode 'cfg' runs on exactly 2 ranks (use 'cfg+views' for more)")
            return cls(mode, num_frames, None, CfgSplit.create(), ViewShard.create(num_frames))
        if mode == "cfg+views":
            if world < 4 or world % 2:
                raise RuntimeError("mode 'cfg+views' needs an even number (>= 4) of ranks")
            pv = world // 2
            v, r = divmod(rank, 2)
            # every rank creates every group, in the same order (torch.distributed requirement)
            pair_groups = [dist.new_group([2 * i, 2 * i + 1]) for i in range(pv)]
            view_groups = [dist.new_group([2 * i + j for i in range(pv)]) for j in range(2)]
            sample = ViewShard(num_frames, v, pv, view_groups[r], partition_frames(num_frames, pv))
            blocks = []
            for t0, n in sample.blocks:
                if n < 2:
                    raise ValueError(f"{num_frames} frames over {pv} blocks leave a block too small to split for the decode")
                blocks += [(t0, (n + 1) // 2), (t0 + (n + 1) // 2, n // 2)]
            cfg, decode = CfgSplit(r, pair_groups[v]), ViewShard(num_frames, rank, world, None, blocks)
            for part in (sample, cfg, decode):
                part.attach_peer()
            return cls(mode, num_frames, sample, cfg, decode)
        raise ValueError(f"unknown shard mode {mode!r} (views | cfg | cfg+views)")

    def gather_frames(self, local: torch.Tensor) -> torch.Tensor:
        return self.decode.gather_frames(local)

    def transports(self) -> List[PeerTransport]:
        out = []
        for part in (self.sample, self.cfg, self.decode):
            t = getattr(part, "peer", None)
            if t is not None and all(t is not o for o in out):
                out.append(t)
        return out

    def check_status(self) -> None:
        """After a sampled image: raise if any one-sided exchange timed out waiting for its signal (host sync)."""
        for t in self.transports():
            st = t.status()
            if st:
                raise RuntimeError(f"peer transport: exchange site {st & 0x7FFFFFFF} never received its signal "
                                   f"(rank {t.rank} of {t.world}); results of this image are invalid")

    def describe(self) -> Dict:
        return {"mode": self.mode, "transport": "peer-memory (NVLink one-sided)" if self.transports() else "torch.distributed",
                "sample_blocks": self.sample.blocks if self.sample else None,
                "cfg_rank": self.cfg.rank if self.cfg else None, "decode_blocks": self.decode.blocks,
                "exchanges": {**(self.sample.exchanges if self.sample else {}),
                              "cfg_gather": self.cfg.exchanges if self.cfg else 0,
                              **{"decode_" + k: v for k, v in self.decode.exchanges.items()
                                 if self.decode is not self.sample}}}
