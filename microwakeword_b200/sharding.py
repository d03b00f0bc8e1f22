"""Stream sharding across the GPUs of one box (one process per GPU, torch.distributed / NCCL).

The reference has no distributed code (SURVEY.md 2.2); streams are fully independent
(microwakeword/inference.py and mixednet.py contain no cross-stream operation), so rank r owns the
contiguous block streams[r*S/G : (r+1)*S/G], weights are replicated, and the only communication the
path ever needs is what BASELINE.json's north_star names: scatter int16 audio batches from an ingest
rank and gather float32 scores back.  When audio already arrives sharded (bench.py's default, weak
scaling) there is no data-path collective at all.

Works with backend "nccl" (GPU tensors, NVLink) and "gloo" (CPU tensors; used by the world-size-2
tests that run without a GPU).
"""

from __future__ import annotations

import ctypes

from . import _lib


def partition(n_streams: int, world: int, shares=None):
    """Contiguous blocks [(start, count)] * world.  Default: balanced, the first n % world ranks get one extra.
    `shares`: explicit per-rank stream counts (same list on every rank; zeros allowed) -- e.g. ingest_shares()."""
    if n_streams < 0 or world < 1:
        raise ValueError("bad partition arguments")
    if shares is not None:
        shares = [int(c) for c in shares]
        if len(shares) != world or min(shares) < 0 or sum(shares) != n_streams:
            raise ValueError("partition: shares %r do not split %d streams over %d ranks" % (shares, n_streams, world))
        out, start = [], 0
        for c in shares:
            out.append((start, c))
            start += c
        return out
    base, extra = divmod(n_streams, world)
    out, start = [], 0
    for r in range(world):
        n = base + (1 if r < extra else 0)
        out.append((start, n))
        start += n
    return out


def ingest_shares(n_streams: int, world: int, src: int = 0, src_share: float = 1.0):
    """Per-rank stream counts when all audio starts on rank `src`: the ingest rank takes `src_share` of an equal share
    (0 = it only feeds the others), the rest is spread evenly over the other ranks.  Why: one GPU's NVLink egress bounds how
    fast N - 1 peers can pull; once that bound exceeds a rank's compute time, the ingest GPU's own kernels only slow its
    peers' reads of its memory."""
    if world < 1 or not 0 <= src < world or not 0.0 <= src_share <= 1.0:
        raise ValueError("bad ingest_shares arguments")
    if world == 1:
        return [n_streams]
    mine = int(round(n_streams / world * src_share))
    rest = partition(n_streams - mine, world - 1)
    out = [c for _, c in rest]
    out.insert(src, mine)
    return out


def scatter_audio(audio, n_streams: int, n_samples: int, src: int = 0, group=None, device=None):
    """Rank `src` holds int16 [n_streams, n_samples]; every rank returns its own [count, n_samples] block."""
    import torch
    import torch.distributed as dist

    world, rank = dist.get_world_size(group), dist.get_rank(group)
    parts = partition(n_streams, world)
    if device is None:
        if audio is None and dist.get_backend(group) == "nccl":
            raise ValueError("scatter_audio: ranks that pass no audio must name their CUDA device (NCCL moves device tensors only)")
        device = audio.device if audio is not None else torch.device("cpu")
    local = torch.empty((parts[rank][1], n_samples), dtype=torch.int16, device=device)
    if rank == src and (tuple(audio.shape) != (n_streams, n_samples) or audio.dtype != torch.int16):
        raise ValueError("scatter_audio: rank %d must pass int16 [%d, %d]" % (src, n_streams, n_samples))
    # samples travel as raw bytes: every backend (gloo has no int16) moves uint8
    as_bytes = lambda t: t.contiguous().view(torch.uint8)
    if len({c for _, c in parts}) == 1:
        chunks = [as_bytes(audio[s:s + c]) for s, c in parts] if rank == src else None
        dist.scatter(as_bytes(local), chunks, src=src, group=group)
    else:
        # ragged blocks: point-to-point sends (grouped on NCCL)
        if rank == src:
            reqs = []
            for r, (s, c) in enumerate(parts):
                if r == src:
                    local.copy_(audio[s:s + c])
                elif c:
                    reqs.append(dist.isend(as_bytes(audio[s:s + c]), dst=r, group=group))
            for q in reqs:
                q.wait()
        elif parts[rank][1]:
            dist.recv(as_bytes(local), src=src, group=group)
    return local


def tile_blocks(n_streams: int, world: int, tiles: int):
    """blocks[t][r] = (global start, count) of tile t of rank r: every rank's contiguous block cut into `tiles`
    contiguous sub-blocks (balanced like partition())."""
    if tiles < 1:
        raise ValueError("tiles must be >= 1")
    per_rank = [[(start + s, c) for s, c in partition(count, tiles)] for start, count in partition(n_streams, world)]
    return [[per_rank[r][t] for r in range(world)] for t in range(tiles)]


def scatter_audio_tiles(audio, n_streams: int, n_samples: int, tiles: int, src: int = 0, group=None, device=None):
    """Issue the scatter of every tile asynchronously and return at once: (locals, works) with locals[t] this rank's
    int16 [count_t, n_samples] block of tile t and works[t] the handles to wait on before reading it.  On NCCL the
    transfers queue on the communicator's own stream in tile order, so tile t+1 moves over NVLink while the caller
    computes on tile t (wait() only makes the caller's CUDA stream wait); on gloo wait() blocks the host."""
    import torch
    import torch.distributed as dist

    world, rank = dist.get_world_size(group), dist.get_rank(group)
    blocks = tile_blocks(n_streams, world, tiles)
    if device is None:
        device = audio.device if audio is not None else torch.device("cpu")
    if rank == src and (tuple(audio.shape) != (n_streams, n_samples) or audio.dtype != torch.int16):
        raise ValueError("scatter_audio_tiles: rank %d must pass int16 [%d, %d]" % (src, n_streams, n_samples))
    as_bytes = lambda t: t.contiguous().view(torch.uint8)
    locals_, works = [], []
    for blk in blocks:
        local = torch.empty((blk[rank][1], n_samples), dtype=torch.int16, device=device)
        ws = []
        if len({c for _, c in blk}) == 1:
            if blk[0][1]:
                chunks = [as_bytes(audio[s:s + c]) for s, c in blk] if rank == src else None
                ws.append(dist.scatter(as_bytes(local), chunks, src=src, group=group, async_op=True))
        elif rank == src:
            for r, (s, c) in enumerate(blk):
                if r == src:
                    local.copy_(audio[s:s + c])
                elif c:
                    ws.append(dist.isend(as_bytes(audio[s:s + c]), dst=r, group=group))
        elif blk[rank][1]:
            ws.append(dist.irecv(as_bytes(local), src=src, group=group))
        locals_.append(local)
        works.append(ws)
    return locals_, works


class IngestBuffer:
    """The ingest rank's audio buffer, readable by every GPU of the box (BASELINE.json configs[4]: "audio originates on rank
    0").  The buffer is a cudaMalloc owned by the library on the ingest rank, exported with cudaIpcGetMemHandle; every
    other rank opens the handle INSIDE ITS OWN device context (mww_ipc_open, cudaIpcMemLazyEnablePeerAccess), so no rank
    ever creates a context on the ingest GPU.  A rank then hands `block_ptr()` -- the address of its own block inside the
    remote buffer -- to StreamEngine.predict_clip_remote: the frontend kernel reads it in place over NVLink (tiles = 0), or
    the rank's copy engine pulls tile t+1 while tile t computes (tiles > 0).  Either way no communication kernel occupies
    an SM on either side and nothing has to be co-scheduled with the compute grids.  One box only.

        with IngestBuffer(n_streams, n_samples, src=0, device=dev) as ingest:   # collective
            if rank == 0: ingest.buffer.copy_(audio)                             # the ingest rank fills it (its current stream)
            probs = sharded.predict_clip_ingest(ingest)                          # collective, every step

    Ordering per step (predict_clip_ingest): a one-element all-reduce after the ingest rank's writes (stream-ordered before its
    contribution) and before any peer's copies; the final gather of the scores tells the ingest rank that every peer has
    finished reading, so it may refill the buffer once predict_clip_ingest has returned on its stream."""

    def __init__(self, n_streams: int, n_samples: int, src: int = 0, group=None, device=None):
        import torch
        import torch.distributed as dist

        self.group, self.src = group, src
        self.n_streams, self.n_samples = int(n_streams), int(n_samples)
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        device = torch.device(device)
        self.dev_index = device.index if device.index is not None else torch.cuda.current_device()   # resolved once, used everywhere
        self.device = torch.device("cuda", self.dev_index)
        self.buffer, self._owned, self._opened, self.base_ptr = None, None, None, None
        L = _lib.lib()
        handle = ctypes.create_string_buffer(64)
        ptr = ctypes.c_void_p()
        err = None
        try:
            if self.rank == src:
                _lib.check(None, L.mww_ipc_alloc(self.n_streams * self.n_samples * 2, self.dev_index, ctypes.byref(ptr), handle))
                self._owned = ptr.value
        except Exception as exc:                                # noqa: BLE001 -- agreed on below
            err = exc
        box = [bytes(handle.raw) if self.rank == src else None]
        if self.world > 1:
            dist.broadcast_object_list(box, src=src, group=group)
        try:
            if err is None and self.rank != src:
                _lib.check(None, L.mww_ipc_open(box[0], self.dev_index, ctypes.byref(ptr)))
                self._opened = ptr.value
        except Exception as exc:                                # noqa: BLE001
            err = exc
        ok = torch.tensor([0 if err else 1], dtype=torch.int32, device=self.device)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)   # also: nobody proceeds before everybody has opened the handle
        if int(ok.item()) == 0:
            self.close()
            raise RuntimeError("IngestBuffer: CUDA IPC / peer access to the ingest rank's buffer is unavailable (%s)" % (err or "on another rank"))
        self.base_ptr = ptr.value
        self.token = torch.zeros(1, dtype=torch.int32, device=self.device)      # per-step ordering token (predict_clip_ingest)
        if self.rank == src:
            iface = {"shape": (self.n_streams, self.n_samples), "typestr": "<i2", "data": (self._owned, False), "version": 3, "strides": None}
            holder = type("MwwIpcBuffer", (), {"__cuda_array_interface__": iface})()
            self.buffer = torch.as_tensor(holder, device=self.device)

    def block_ptr(self, first_stream: int) -> int:
        """Address (valid in THIS process) of stream `first_stream` inside the ingest buffer."""
        return self.base_ptr + int(first_stream) * self.n_samples * 2

    def close(self):
        """Unmap (peers) / free (ingest rank).  The ingest rank must only free after every peer is done reading: callers
        synchronise and barrier first (predict_clip_ingest's gather already orders the last read before its return)."""
        if getattr(self, "_opened", None):
            _lib.lib().mww_ipc_close(ctypes.c_void_p(self._opened), self.dev_index)
            self._opened = None
        if getattr(self, "_owned", None):
            self.buffer = None
            _lib.lib().mww_ipc_free(ctypes.c_void_p(self._owned), self.dev_index)
            self._owned = None
        self.base_ptr = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False

    def __del__(self):
        try:
            self.close()
        except Exception:                                       # noqa: BLE001 -- interpreter shutdown
            pass


def scatter_compute_gather(audio_on_src, n_streams: int, n_samples: int, compute, tiles: int = 8, src: int = 0, group=None, device=None):
    """BASELINE.json configs[4] ingest pattern with the exchange hidden behind the compute: audio lives on `src`, every
    rank's block is cut into `tiles` sub-blocks, all tile scatters are issued up front and `compute(t, local_audio)`
    (-> float32 [count_t, steps]) runs on tile t as soon as it has landed while the later tiles are still in flight.
    The scores (4 bytes per 960 bytes of audio) go back in one gather.  Returns [n_streams, steps] on `src`, else None."""
    import torch

    locals_, works = scatter_audio_tiles(audio_on_src, n_streams, n_samples, tiles, src=src, group=group, device=device)
    outs = []
    for t, (local, ws) in enumerate(zip(locals_, works)):
        for w in ws:
            w.wait()
        outs.append(compute(t, local))
    return gather_probs(torch.cat(outs, 0), n_streams, dst=src, group=group)


def gather_probs(local_probs, n_streams: int, dst: int = 0, group=None, shares=None):
    """Every rank passes float32 [count, steps]; rank `dst` returns [n_streams, steps], others None.
    `shares`: the per-rank counts when the partition is not the balanced one (partition())."""
    import torch
    import torch.distributed as dist

    world, rank = dist.get_world_size(group), dist.get_rank(group)
    parts = partition(n_streams, world, shares)
    if local_probs.shape[0] != parts[rank][1]:
        raise ValueError("gather_probs: rank %d passes %d rows, its block has %d" % (rank, local_probs.shape[0], parts[rank][1]))
    steps = local_probs.shape[1]
    local_probs = local_probs.contiguous()
    if len({c for _, c in parts}) == 1:
        outs = [torch.empty_like(local_probs) for _ in range(world)] if rank == dst else None
        dist.gather(local_probs, outs, dst=dst, group=group)
        return torch.cat(outs, 0) if rank == dst else None
    if rank == dst:
        full = torch.empty((n_streams, steps), dtype=local_probs.dtype, device=local_probs.device)
        for r, (s, c) in enumerate(parts):
            if r == dst:
                if c:
                    full[s:s + c] = local_probs
            elif c:
                dist.recv(full[s:s + c], src=r, group=group)
        return full
    if parts[rank][1]:
        dist.send(local_probs, dst=dst, group=group)
    return None


class ShardedEngine:
    """This rank's block of streams as `tiles` StreamEngines over contiguous sub-blocks (tiles = 1: one engine).
    More than one tile lets predict_clip_scattered() overlap the NVLink scatter of tile t+1 with the kernels of tile t."""

    def __init__(self, model, n_streams_total: int, device_index: int, group=None, tiles: int = 1, engine_factory=None, shares=None):
        """`shares`: per-rank stream counts (default: balanced).  A rank whose share is 0 owns no engine and only takes part in
        the collectives (the ingest rank of an egress-bound job: ingest_shares(..., src_share=0))."""
        import torch.distributed as dist

        if engine_factory is None:
            from .engine import StreamEngine
        else:
            StreamEngine = engine_factory          # tests: a CPU stand-in with the StreamEngine surface (gloo, no GPU)
        self.group = group
        self.n_total = n_streams_total
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        if n_streams_total < self.world:
            raise ValueError("ShardedEngine: %d streams cannot be spread over %d ranks" % (n_streams_total, self.world))
        self.shares = None if shares is None else [int(c) for c in shares]
        parts = partition(n_streams_total, self.world, self.shares)
        smallest = min([c for _, c in parts if c] or [1])
        self.tiles = max(1, min(int(tiles), smallest))                          # same on every rank; no empty sub-block
        tiles = self.tiles
        if self.shares is not None and tiles != 1:
            raise ValueError("ShardedEngine: explicit shares go with tiles=1 (the library tiles the ingest itself)")
        self.start, self.count = parts[self.rank]
        self.device_index = device_index
        self.tile_parts = partition(self.count, tiles) if self.count else []
        self.engines = [StreamEngine(model, n_streams=c, device=device_index) for _, c in self.tile_parts]
        self.engine = self.engines[0] if self.engines else None
        self._mirror = None
        if self.engine is None:
            # a rank without streams still has to know how many steps a call produces (the gather's width): the same host
            # arithmetic the engines run (frames buffered, pending rows), on the model's stride and hop
            probe = StreamEngine(model, n_streams=1, device=device_index)
            self._mirror = {"stride": probe.stride, "hop": probe.hop, "used": 0, "pend": 0}
            probe.close()

    def reset(self):
        for e in self.engines:
            e.reset()
        if self._mirror is not None:
            self._mirror.update(used=0, pend=0)

    def predict_clip_scattered(self, audio_on_src, n_samples: int, src: int = 0):
        """Audio originates on `src` ([n_total, n_samples] int16 CUDA tensor, None elsewhere); scores return to `src`."""
        import torch

        return scatter_compute_gather(audio_on_src, self.n_total, n_samples, lambda t, local: self.engines[t].predict_clip(local),
                                      tiles=self.tiles, src=src, group=self.group, device=torch.device("cuda", self.engine.device))

    def predict_clip_ingest(self, ingest: "IngestBuffer", tiles: int = 0, out=None):
        """Audio sits in `ingest` on its src rank; every rank computes its own block of it (one engine), scores are gathered on
        the src rank.  Returns [n_total, steps] there, None elsewhere.  tiles = 0: the frontend kernel reads the peer-mapped
        buffer in place over NVLink (zero-copy; best while the ingest GPU's egress is not the bottleneck); tiles > 0: the library's
        staged pipeline -- this rank's copy engine pulls tile t+1 while tile t computes (best when it is)."""
        import torch.distributed as dist

        if ingest.n_streams != self.n_total:
            raise ValueError("IngestBuffer holds %d streams, the engine shards %d" % (ingest.n_streams, self.n_total))
        if len(self.engines) > 1:
            raise ValueError("predict_clip_ingest uses one engine per rank (ShardedEngine(..., tiles=1)); the tiling happens inside the library")
        # the buffer is complete on the ingest rank before any peer starts copying (IngestBuffer docstring).  A one-element
        # all-reduce is stream-ordered on every rank (the pull is queued behind it) and, unlike dist.barrier() on NCCL, does not
        # stall the host, so the next step's launches are already queued while this one runs.
        token = getattr(ingest, "token", None)
        if token is not None:
            dist.all_reduce(token, group=self.group)
        else:
            dist.barrier(group=self.group)
        if self.engine is not None:
            local = self.engine.predict_clip_remote(ingest.block_ptr(self.start), ingest.n_samples, tiles=tiles, out=out)
        else:
            # a rank without streams: an empty block with the right width (every rank's call produces the same number of steps)
            import torch
            local = torch.empty((0, self._empty_steps(ingest.n_samples)), dtype=torch.float32, device=ingest.device)
        return gather_probs(local, self.n_total, dst=ingest.src, group=self.group, shares=self.shares)

    def _empty_steps(self, n_samples: int) -> int:
        """Steps a call with n_samples new samples produces -- for a rank that owns no engine (all engines advance in lockstep)."""
        from .engine import WINDOW
        m = self._mirror
        total = m["used"] + int(n_samples)
        rows = (total - WINDOW) // m["hop"] + 1 if total >= WINDOW else 0
        steps = (m["pend"] + rows) // m["stride"]
        m["used"], m["pend"] = total - rows * m["hop"], (m["pend"] + rows) % m["stride"]
        return steps
