"""Multi-GPU use of the hot path: clips shard embarrassingly, one process per GPU, and the only
exchange step is the final gather of the per-rank (B_local, T, cc) result blocks
(SURVEY.md section 8e; BASELINE config 5).  `torch.distributed` (NCCL on GPUs, gloo in CPU tests) is
the plumbing; no collective runs inside the transform itself.

Results are independent of the world size: the fused kernel's tile schedule and reduction trees do
not depend on the batch, so rank r's block equals rows [lo, hi) of the single-GPU result bit for bit.
"""
from __future__ import annotations


def shard_bounds(total: int, world: int, rank: int):
    """Contiguous block of clips owned by `rank`: sizes differ by at most one, earlier ranks get the extra."""
    if world < 1 or not (0 <= rank < world):
        raise ValueError("bad world/rank")
    base, extra = divmod(total, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def gather_blocks(local, total: int, group=None):
    """All-gather variable-size leading-dim blocks into one (total, ...) tensor on every rank.
    Uses all_gather_into_tensor when blocks are equal (one NCCL call), else a padded gather."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    sizes = [shard_bounds(total, world, r)[1] - shard_bounds(total, world, r)[0] for r in range(world)]
    if local.shape[0] != sizes[rank]:
        raise ValueError(f"rank {rank} holds {local.shape[0]} rows, expected {sizes[rank]}")
    if len(set(sizes)) == 1:
        out = torch.empty((total,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(out, local.contiguous(), group=group)
        return out
    mx = max(sizes)
    pad = torch.zeros((mx,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad, group=group)
    return torch.cat([p[:n] for p, n in zip(parts, sizes)], dim=0)


def mfcc_sharded(bft, clips, cc_num=13, rectify_type=0, total=None, group=None, compute=None):
    """Each rank passes ITS shard `clips` (B_local, L); returns the gathered (B_total, T, cc) MFCCs.
    `compute` defaults to `bft.mfcc_batch` (the fused CUDA path); tests inject a stand-in to
    exercise the sharding and gather logic without a GPU."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    if total is None:
        total = clips.shape[0] * world
    fn = compute if compute is not None else (lambda x: bft.mfcc_batch(x, cc_num, rectify_type))
    return gather_blocks(fn(clips), total, group)


class OverlappedGather:
    """Chunked compute + all-gather with the collective of chunk k running on a side stream while chunk k+1
    is being transformed (SURVEY.md section 8e: the gather costs the same order as the compute at this library's speed).

    out[k] is the gathered (world * B_chunk, T, cc) block of chunk k: rank r's clips of that chunk sit at rows
    [r * B_chunk, (r + 1) * B_chunk).  Buffers are allocated once and reused, so steady-state steps allocate nothing."""

    def __init__(self, chunks: int = 4, group=None):
        import torch
        self.chunks, self.group = chunks, group
        self.comm = torch.cuda.Stream()
        self.gathered = None
        self.done = [torch.cuda.Event() for _ in range(chunks)]

    def __call__(self, compute, clips):
        import torch
        import torch.distributed as dist
        world = dist.get_world_size(self.group)
        B = clips.shape[0]
        per = (B + self.chunks - 1) // self.chunks
        cur = torch.cuda.current_stream()
        outs = []
        for k in range(self.chunks):
            lo, hi = k * per, min(B, (k + 1) * per)
            if lo >= hi:
                break
            o = compute(clips[lo:hi])
            outs.append(o)
            self.done[k].record(cur)
        want = [(world * o.shape[0],) + tuple(o.shape[1:]) for o in outs]          # full shape of every chunk: batch / world size may change
        if self.gathered is None or [tuple(g.shape) for g in self.gathered] != want or self.gathered[0].device != outs[0].device:
            self.gathered = [torch.empty((world * o.shape[0],) + tuple(o.shape[1:]), dtype=o.dtype, device=o.device) for o in outs]
        with torch.cuda.stream(self.comm):
            for k, o in enumerate(outs):
                self.comm.wait_event(self.done[k])
                dist.all_gather_into_tensor(self.gathered[k], o, group=self.group)
                o.record_stream(self.comm)
        cur.wait_stream(self.comm)
        return self.gathered


class _DevArray:
    """Zero-copy view of a raw device pointer for torch.as_tensor (CUDA array interface v2)."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f4", "data": (int(ptr), False),
                                         "version": 2, "strides": None}


class PeerScatter:
    """MFCC + all-gather as ONE kernel (no NCCL on the data path).

    Every rank owns a gathered array (world, B_local, T, cc) allocated by the library (`afb200_peerAlloc`) and
    exported with `cudaIpcGetMemHandle`; the 64-byte handles travel once through `all_gather_object` and each rank
    maps the other ranks' arrays (`afb200_ipcOpenHandle`, peer access over NVLink / NVSwitch).  A step then is a
    single `bftObj_mfccBatchScatter` launch: the kernel's DCT epilogue stores each finished tile into slot `rank`
    of its own array AND of every peer's array, so the exchange overlaps the transform tile by tile and costs no
    SMs, no copy engines and no extra launches.  `fence()` orders all ranks' stores before anybody reads
    (a 4-byte all-reduce on the current stream: a rank's contribution is stream-ordered after its kernel).

    Write-after-read: the gathered array is double buffered (`slots=2`).  Step k writes slot k % 2 and `fence()` closes
    the step; the kernels of step k+1 write the OTHER slot, so a rank may still be reading step k's result while its
    peers are already storing step k+1.  Slot k % 2 is rewritten by step k+2, which a rank launches only after its
    own fence of step k+1 has completed, i.e. after EVERY rank's stream has reached that fence: reads of step k that
    were enqueued (on the fencing stream) before the next fence are therefore always finished in time.  A consumer
    that reads on another stream, or later than that, must make the fencing stream wait for it first."""

    def __init__(self, bft, batch_local: int, data_length: int, cc_num: int, rectify_type=0, group=None, slots: int = 2):
        import ctypes as C
        import torch
        import torch.distributed as dist
        self.bft, self.group = bft, group
        self.lib = bft._lib
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        if self.world - 1 > 15:
            raise ValueError("PeerScatter supports up to 16 ranks")
        self.B, self.L, self.cc, self.rect = batch_local, data_length, cc_num, int(getattr(rectify_type, "value", rectify_type))
        self.T = bft.cal_time_length(data_length)
        self.block = batch_local * self.T * cc_num                      # floats per rank block
        self.slots, self._slot, self._open = max(1, int(slots)), 0, False
        self.slot_bytes = self.world * self.block * 4                   # one gathered array
        nbytes = self.slots * self.slot_bytes
        self._ptr = C.c_void_p()
        self._peers = []
        # every rank takes part in every collective below even if a local step failed, so that a failure
        # surfaces as the same exception on all ranks instead of a hang
        err = None
        handle = (C.c_ubyte * 64)()
        if self.lib.afb200_peerAlloc(C.byref(self._ptr), nbytes) != 0:
            err = "afb200_peerAlloc: " + self.lib.afb200_lastError().decode()
            self._ptr = C.c_void_p()
        elif self.lib.afb200_ipcGetHandle(self._ptr, handle) != 0:
            err = "afb200_ipcGetHandle: " + self.lib.afb200_lastError().decode()
        handles = [None] * self.world
        dist.all_gather_object(handles, None if err else bytes(handle), group=group)
        if err is None and all(h is not None for h in handles):
            for r in range(self.world):
                if r == self.rank:
                    continue
                p = C.c_void_p()
                buf = (C.c_ubyte * 64).from_buffer_copy(handles[r])
                if self.lib.afb200_ipcOpenHandle(buf, C.byref(p)) != 0:
                    err = f"afb200_ipcOpenHandle(rank {r}): " + self.lib.afb200_lastError().decode()
                    break
                self._peers.append(p.value)
        elif err is None:
            err = "a peer rank could not export its buffer"
        errs = [None] * self.world
        dist.all_gather_object(errs, err, group=group)
        if any(errs):
            self.close()
            raise RuntimeError("PeerScatter setup failed: " + "; ".join(f"rank {r}: {e}" for r, e in enumerate(errs) if e))
        self._rank_off = self.rank * self.block * 4                      # block `rank` inside every gathered array
        dev = torch.device("cuda", torch.cuda.current_device())
        self._gathered = [torch.as_tensor(_DevArray(self._ptr.value + k * self.slot_bytes, (self.world, batch_local, self.T, cc_num)),
                                          device=dev) for k in range(self.slots)]
        self.gathered = self._gathered[0]                                # the array of the step last launched
        self._flag = torch.zeros(1, dtype=torch.int32, device=dev)
        dist.barrier(group=group)                                        # every rank has mapped every buffer

    def _check(self, rc, what):
        if rc != 0:
            raise RuntimeError(f"{what} failed ({rc}): {self.lib.afb200_lastError().decode()}")

    def __call__(self, clips, clip_offset=0):
        """clips: this rank's (B_local, L) CUDA tensor -- or a chunk (nb, L) of it that starts at clip `clip_offset`
        (callers that stream their shard in from the host launch chunk by chunk).  Launches the fused kernel on the
        current stream and returns the gathered (world, B_local, T, cc) tensor; call `fence()` before reading other
        ranks' slots."""
        import ctypes as C
        import torch
        nb = clips.shape[0]
        if clips.dim() != 2 or clips.shape[1] != self.L or clip_offset < 0 or clip_offset + nb > self.B or \
                not clips.is_cuda or clips.dtype != torch.float32 or not clips.is_contiguous():
            raise ValueError("clips must be a contiguous float32 CUDA tensor (nb, L) with clip_offset + nb <= B_local")
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        self._open = True                                                # launches until the next fence() belong to this step / slot
        off = self._slot * self.slot_bytes + self._rank_off + clip_offset * self.T * self.cc * 4
        dst = C.c_void_p(self._ptr.value + off)
        peers = (C.c_void_p * max(1, len(self._peers)))(*[C.c_void_p(p + off) for p in self._peers])
        self.gathered = self._gathered[self._slot]
        self._check(self.lib.bftObj_mfccBatchScatter(self.bft._obj, C.c_void_p(clips.data_ptr()), self.L, nb, self.cc,
                                                     self.rect, dst, len(self._peers), peers, stream),
                    "bftObj_mfccBatchScatter")
        return self.gathered

    def fence(self):
        """Closes the step: after it (stream order) every rank's stores of this step are complete and visible; the next
        `__call__` starts the next step in the other slot."""
        import torch.distributed as dist
        if self.world > 1:
            dist.all_reduce(self._flag, group=self.group)
        if self._open:
            self._slot = (self._slot + 1) % self.slots
            self._open = False

    def close(self):
        for p in self._peers:
            self.lib.afb200_ipcCloseHandle(p)
        self._peers = []
        self.gathered = None
        self._gathered = []
        if self._ptr is not None and self._ptr.value:
            self.lib.afb200_peerFree(self._ptr)
        self._ptr = None
