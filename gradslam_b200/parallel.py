"""Multi-GPU layer: batch sharding + the one collective of the path (SURVEY.md §8e).

Sequences are independent (each batch element owns its map and pose chain), so a (B_total, L) job shards by
contiguous blocks of B_total / world sequences per rank, one process per GPU, and NO traffic crosses GPUs
while the L frames are fused.  The only exchange is at the end: an all-gather of the per-sequence sizes
followed by a variable-length all-gather of the fused maps, after which every rank holds all B_total maps.  The maps
travel as they are stored - packed geometry rows (8 floats) and colour rows (4 floats) - and are received in place in the
output store, no zero fill on either side.  Three transports; GSX_MAP_EXCHANGE=auto (default) takes `peer` between two
GPUs and `all_gather` beyond (see _exchange_mode):

  peer        each rank PULLS its peers' rows out of their stores (CUDA IPC mappings) with one pitched copy per peer and
              row array, executed by the copy engines over NVLink: no communication kernel on any SM, no staging copy
              (csrc/gsx_peer.cu).  The size all-gather before the pulls orders them after the owners' fusion; a one-word
              all-reduce after them releases the owners' stores.
              Requires all ranks on ONE node and stores from cudaMalloc-backed allocations (PyTorch's default caching
              allocator; not `expandable_segments`) - gsx_peer_export / gsx_peer_open raise otherwise; select
              GSX_MAP_EXCHANGE=all_gather there.
  all_gather  one NCCL all-gather per row array on `[:, :nmax]` staging copies (also the CPU / gloo path of the tests).
  p2p         grouped exact-size NCCL send / recv straight out of the stores.
"""
import os
from typing import Optional

import torch
import torch.distributed as dist

from .structures.pointclouds import Pointclouds

__all__ = ["shard_batch", "gather_maps", "gather_maps_begin", "gather_maps_end", "comm_stream", "bind_host_to_gpu",
           "GatheredMaps", "exchange_mode"]


def bind_host_to_gpu(device) -> Optional[str]:
    """Pins this process (one process per GPU) to the CPU cores of the NUMA node the GPU hangs off, so that the pinned
    host buffers it allocates afterwards - the upload source and the map read-back target - are placed in that node's
    memory and the PCIe traffic of the ranks does not cross the socket interconnect.  Returns the core list that was
    applied, or None if the topology is not exposed (the affinity is then left alone)."""

    try:
        prop = torch.cuda.get_device_properties(torch.device(device))
        bdf = "%04x:%02x:%02x.0" % (prop.pci_domain_id, prop.pci_bus_id, prop.pci_device_id)
        with open("/sys/bus/pci/devices/%s/local_cpulist" % bdf) as f:
            text = f.read().strip()
        cpus = set()
        for part in text.split(","):
            if not part:
                continue
            lo, _, hi = part.partition("-")
            cpus.update(range(int(lo), int(hi or lo) + 1))
        cpus &= os.sched_getaffinity(0)
        if not cpus:
            return None
        os.sched_setaffinity(0, cpus)
        return text
    except (OSError, ValueError, AttributeError, RuntimeError):
        return None


def shard_batch(total: int, rank: Optional[int] = None, world: Optional[int] = None):
    """Contiguous block [lo, hi) of the batch owned by `rank` (blocks differ by at most one element)."""
    rank = dist.get_rank() if rank is None else rank
    world = dist.get_world_size() if world is None else world
    base, extra = divmod(total, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


_COMM_STREAMS = {}
_CONTROL_GROUPS = {}


def _comm_stream(device):
    if device.type != "cuda":
        return None
    key = str(device)
    if key not in _COMM_STREAMS:
        _COMM_STREAMS[key] = torch.cuda.Stream(device=device, priority=-1)
    return _COMM_STREAMS[key]


def _control_group(group, device):
    """The process group the exchange's two tiny collectives (sizes + store descriptors before the pulls, the one-word
    release after them) run on: the same ranks as `group`, but a communicator whose kernels are launched on a
    HIGH-PRIORITY stream.  On an ordinary stream a NCCL kernel queues behind the thousands of thread blocks the two
    fusion streams keep pending and only gets onto an SM when a step drains: the size all-gather of step k then completes
    at the END of step k+1, the host (waiting for the sizes) enqueues step k+2 late, and the GPU idles before each step.
    Created once per group (a collective call: every rank reaches gather_maps_begin)."""
    if device.type != "cuda" or os.environ.get("GSX_EXCHANGE_PRIORITY", "high") != "high":
        return group
    key = (id(group) if group is not None else None, str(device))
    if key not in _CONTROL_GROUPS:
        from torch.distributed import ProcessGroupNCCL

        opts = ProcessGroupNCCL.Options()
        opts.is_high_priority_stream = True
        ranks = None if group is None else dist.get_process_group_ranks(group)
        _CONTROL_GROUPS[key] = dist.new_group(ranks=ranks, backend="nccl", pg_options=opts, device_id=device)
    return _CONTROL_GROUPS[key]


class _GatherHandle:
    __slots__ = ("pc", "group", "world", "counts_host", "ready", "stream", "mode", "meta_len", "into")


class GatheredMaps:
    """A job-wide map store: row arrays for world * B maps of `capacity` rows on every rank.  This rank's sequences are
    fused IN PLACE into its block (`PointFusion(...)(frames, out=store.local)`); `gather_maps*(store.local, into=store)`
    then only moves the peers' rows - into their blocks of this store - and returns `store.all`.  Compared with gathering
    into a fresh store this saves the allocation and the local copy of this rank's own rows (as many bytes again as one
    peer sends).  `reset()` empties the local block for the next job."""

    def __init__(self, batch_size: int, capacity: int, device, group=None):
        from .structures.pointclouds import COL_W, GEO_W

        self.group = group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.batch_size = int(batch_size)
        device = torch.device(device)
        total = self.world * self.batch_size
        geo = torch.empty((total, int(capacity), GEO_W), dtype=torch.float32, device=device)
        col = torch.empty((total, int(capacity), COL_W), dtype=torch.float32, device=device)
        self.all = Pointclouds(device=device)
        self.all._attach(geo, col)
        lo = self.rank * self.batch_size
        self.local = Pointclouds(device=device)
        self.local._attach(geo[lo: lo + self.batch_size], col[lo: lo + self.batch_size])
        self._done = None  # event on the communication stream: the last exchange of this store has completed

    def reset(self) -> Pointclouds:
        """Empties this rank's block for the next job and returns it.  The current stream is made to wait for the last
        exchange of this store (peers may still be reading the block until then)."""
        if self._done is not None:
            torch.cuda.current_stream(self.local.device).wait_event(self._done)
        for pc in (self.local, self.all):
            pc._overflow = None
            pc._set_counts([0] * len(pc))
        return self.local


_META_PER_ARRAY = 10  # present, offset, 8 words of IPC handle


def _export_stores(pc):
    """Host int64 words describing where this rank's row arrays live: capacity, then per array (geometry, colour, extra
    features) a present flag, the offset inside its allocation and the allocation's CUDA IPC handle (gsx_peer_export)."""
    import ctypes
    import struct

    from . import _C

    words = [pc.capacity]
    for t in (pc._geo, pc._col, pc._feat):
        if t is None:
            words += [0] * _META_PER_ARRAY
            continue
        handle = (ctypes.c_ubyte * 64)()
        off = ctypes.c_int64(0)
        _C.check(_C.lib().gsx_peer_export(_C.ptr(t), handle, ctypes.byref(off), None), "gsx_peer_export")
        words += [1, off.value] + list(struct.unpack("8q", bytes(handle)))
    return words


def gather_maps_begin(pointclouds: Pointclouds, group=None, into: Optional[GatheredMaps] = None) -> "_GatherHandle":
    """First half of the map all-gather: exchanges the per-sequence sizes on a side (communication) stream and
    starts their copy to pinned host memory.  Does NOT block the host, so the caller can enqueue the next batch of
    sequences before calling `gather_maps_end` — the exchange then overlaps that compute.
    into: the GatheredMaps store whose `local` block `pointclouds` is (see there)."""
    h = _GatherHandle()
    h.pc, h.group, h.world = pointclouds, group, dist.get_world_size(group)
    h.into = into
    if into is not None:
        if pointclouds is not into.local or pointclouds._geo.data_ptr() != into.all._geo[
                into.rank * into.batch_size].data_ptr():
            raise ValueError("gather_maps(into=store): `pointclouds` must be store.local, still living in the store "
                             "(a map that outgrew its capacity is re-allocated elsewhere)")
        if into.group is not group:
            raise ValueError("gather_maps(into=store): the store was created for another process group")
    dev = pointclouds.device
    B = len(pointclouds)
    h.stream = _comm_stream(dev)
    local = pointclouds._counts_dev[pointclouds._cur]
    if h.stream is not None:
        h.stream.wait_stream(torch.cuda.current_stream(dev))
        ctx = torch.cuda.stream(h.stream)
    else:
        import contextlib

        ctx = contextlib.nullcontext()
    h.mode = _exchange_mode(dev, h.world)
    h.meta_len = 0
    meta = None
    if h.mode == "peer":
        words = _export_stores(pointclouds)
        h.meta_len = len(words)
        meta = torch.tensor(words, dtype=torch.int64).pin_memory()
    with ctx:
        send = local.to(torch.int64).contiguous()
        if meta is not None:  # sizes and store descriptors travel in the same small all-gather
            send = torch.cat([send, meta.to(dev, non_blocking=True)])
        all_counts = torch.empty(h.world * (B + h.meta_len), dtype=torch.int64, device=dev)
        _all_gather(all_counts, send, _control_group(group, dev))
        if h.stream is not None:
            h.counts_host = torch.empty(h.world * (B + h.meta_len), dtype=torch.int64, pin_memory=True)
            h.counts_host.copy_(all_counts, non_blocking=True)
            h.ready = torch.cuda.Event()
            h.ready.record(h.stream)
            for st in pointclouds._buffers():
                st.record_stream(h.stream)
            local.record_stream(h.stream)
            all_counts.record_stream(h.stream)
        else:
            h.counts_host, h.ready = all_counts, None
    return h


def gather_maps_end(h: "_GatherHandle", wait: bool = True) -> Pointclouds:
    """Second half: waits (host) for the sizes only, then enqueues the exact-size exchange of the map rows on the
    communication stream.  With wait=True the caller's current stream is made to wait for the result; with wait=False
    the caller must synchronise with `parallel.comm_stream(device)` before using it."""
    pc, group, world = h.pc, h.group, h.world
    dev = pc.device
    B = len(pc)
    if h.ready is not None:
        h.ready.synchronize()
    blob = h.counts_host.view(world, B + h.meta_len)
    counts = [int(c) for c in blob[:, :B].reshape(-1).tolist()]
    nmax = max(max(counts), 1)
    rank = dist.get_rank(group)
    if pc._counts_host is None:  # (also raises if the local map overflowed its capacity)
        pc._counts_host = counts[rank * B: (rank + 1) * B]
        pc._check_overflow()
    in_place = h.into is not None
    if in_place:
        out = h.into.all
        if nmax > out.capacity:
            raise RuntimeError("gather_maps(into=store): a peer's map has %d rows, the store's capacity is %d" % (
                nmax, out.capacity))
    else:
        out = Pointclouds(device=dev)
        out._B = world * B
    if h.stream is not None:
        ctx = torch.cuda.stream(h.stream)
    else:
        import contextlib

        ctx = contextlib.nullcontext()
    with ctx:
        # not zero-filled (that would be a multi-GB memset per step at 8 GPUs): the zero padding the *_padded views
        # promise is restored lazily, only for the ragged tails and only if such a view is asked for (Pointclouds._padded)
        if not in_place:
            out._alloc_buffers(nmax, pc._has_normals, pc._col is not None,
                               pc.num_features if pc.has_features else 0, zero=False)
            out._uninit = True
        if h.mode == "peer":
            _exchange_peer(pc, out, counts, blob[:, B:], rank, world, B, group, h.stream, skip_own=in_place)
        elif h.mode == "p2p" or in_place:
            _exchange_p2p(pc, out, counts, rank, world, B, group, h.stream is None, skip_own=in_place)
        else:
            _exchange_all_gather(pc, out, nmax, group, h.stream)
        for t in out._buffers():
            if h.stream is not None:
                t.record_stream(torch.cuda.current_stream(dev))
        out._set_counts(counts)
        if in_place and h.stream is not None:
            h.into._done = torch.cuda.Event()
            h.into._done.record(h.stream)
    if h.stream is not None and wait:
        torch.cuda.current_stream(dev).wait_stream(h.stream)
    return out


def _exchange_mode(device=None, world=None):
    """GSX_MAP_EXCHANGE = auto | peer | all_gather | p2p.  CPU tensors (the gloo tests) always use all_gather.  `auto`
    (default): copy-engine pulls between TWO GPUs, NCCL all-gather beyond (timed on an earlier GPU generation, not on
    H100; DESIGN.md section 7)."""
    if device is not None and torch.device(device).type != "cuda":
        return "all_gather"
    mode = os.environ.get("GSX_MAP_EXCHANGE", "auto")
    if mode not in ("auto", "peer", "all_gather", "p2p"):
        raise ValueError("GSX_MAP_EXCHANGE must be auto, peer, all_gather or p2p (got %r)" % mode)
    if mode == "auto":
        world = dist.get_world_size() if world is None else world
        mode = "peer" if world == 2 else "all_gather"
    return mode


def exchange_mode(device, group=None) -> str:
    """The transport gather_maps will use for maps on `device` in `group` (see _exchange_mode)."""
    return _exchange_mode(device, dist.get_world_size(group))


def _exchange_peer(pc, out, counts, meta, rank, world, B, group, stream, skip_own=False):
    """Every rank pulls: per peer and row array ONE pitched copy (B blocks of max(counts of that peer) rows) from the
    peer's store - mapped into this process through its IPC handle - into this rank's output store.  No kernel runs; the
    trailing one-word all-reduce completes on a rank only when every peer has issued and finished its pulls, which is
    what allows that rank's store to be reused."""
    import ctypes
    import struct

    from . import _C

    lib = _C.lib()
    dev = pc.device
    sp = ctypes.c_void_p(stream.cuda_stream)
    pitch_rows = out.capacity  # row stride of the receiving store's elements
    with torch.cuda.device(dev):
        # rank r pulls from r+1, r+2, ... (mod world): at any moment every owner serves ONE reader.  With the same order
        # on every rank all of them read owner 0 first, then owner 1, ... and share that one GPU's NVLink egress.
        for q in [(rank + 1 + i) % world for i in range(world)]:
            nq = max(counts[q * B:(q + 1) * B])
            if nq == 0 or (skip_own and q == rank):
                continue
            cap_q = int(meta[q, 0])
            for k, (src, dst) in enumerate(((pc._geo, out._geo), (pc._col, out._col), (pc._feat, out._feat))):
                if dst is None:
                    continue
                row = dst.shape[2] * 4
                words = meta[q, 1 + k * _META_PER_ARRAY: 1 + (k + 1) * _META_PER_ARRAY].tolist()
                if not words[0]:
                    raise RuntimeError("gather_maps: rank %d has no array %d but rank %d does" % (q, k, rank))
                if q == rank:
                    sptr = ctypes.c_void_p(src.data_ptr())
                else:
                    sptr = ctypes.c_void_p()
                    handle = (ctypes.c_ubyte * 64).from_buffer_copy(struct.pack("8q", *words[2:]))
                    _C.check(lib.gsx_peer_open(handle, words[1], ctypes.byref(sptr)), "gsx_peer_open")
                how = os.environ.get("GSX_PEER_COPY", "2d")  # diagnostic: 2d (one pitched copy) | 1d (per element) | none
                if how == "2d":
                    _C.check(lib.gsx_peer_copy_rows(ctypes.c_void_p(dst.data_ptr() + q * B * pitch_rows * row),
                                                    pitch_rows * row, sptr, cap_q * row, nq * row, B, sp),
                             "gsx_peer_copy_rows")
                elif how == "1d":
                    for b in range(B):
                        c = counts[q * B + b]
                        _C.check(lib.gsx_peer_copy_rows(
                            ctypes.c_void_p(dst.data_ptr() + (q * B + b) * pitch_rows * row), pitch_rows * row,
                            ctypes.c_void_p(sptr.value + b * cap_q * row), cap_q * row, c * row, 1, sp),
                            "gsx_peer_copy_rows")
    token = torch.zeros(1, dtype=torch.int32, device=dev)
    dist.all_reduce(token, group=_control_group(group, dev))
    token.record_stream(stream)


def _exchange_all_gather(pc, out, nmax, group, stream):
    """One all-gather per row array (geometry rows, colour rows [, extra features]): 2 collectives where round 1 sent
    four attribute tensors.  The send side is the `[:, :nmax]` block of the capacity-backed store (one device-to-device
    staging copy on the communication stream: the store's row stride is its capacity); the receive side IS the output
    store, (world * B, nmax, C) rank-major."""
    for src, dst in ((pc._geo, out._geo), (pc._col, out._col), (pc._feat, out._feat)):
        if src is None:
            continue
        if nmax <= src.shape[1]:
            send = src[:, :nmax].contiguous()
        else:  # a peer's map is longer than this rank's capacity: pad a temporary (never re-allocate the live map here)
            send = src.new_zeros((src.shape[0], nmax, src.shape[2]))
            send[:, : src.shape[1]] = src
        _all_gather(dst, send, group)
        if stream is not None:
            send.record_stream(stream)


def _exchange_p2p(pc, out, counts, rank, world, B, group, blocking, skip_own=False):
    """Exact-size rows straight out of the store: one grouped batch of point-to-point transfers (no staging copy, no
    padding to the longest map)."""
    ops = []
    for src, dst in ((pc._geo, out._geo), (pc._col, out._col), (pc._feat, out._feat)):
        if src is None:
            continue
        for b in range(B):
            c = counts[rank * B + b]
            if c > 0 and not skip_own:
                dst[rank * B + b, :c].copy_(src[b, :c])  # own rows: local copy
        for peer in range(world):
            if peer == rank:
                continue
            g_peer = peer if group is None else dist.get_global_rank(group, peer)
            for b in range(B):
                c = counts[rank * B + b]
                if c > 0:
                    ops.append(dist.P2POp(dist.isend, src[b, :c], g_peer, group))
                c = counts[peer * B + b]
                if c > 0:
                    ops.append(dist.P2POp(dist.irecv, dst[peer * B + b, :c], g_peer, group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            if blocking:
                req.wait()


def comm_stream(device):
    """The side stream the map all-gathers run on (None on CPU)."""
    return _comm_stream(torch.device(device))


def gather_maps(pointclouds: Pointclouds, group=None, into: Optional[GatheredMaps] = None) -> Pointclouds:
    """All-gathers the maps of every rank (equal local batch size).  Returns a Pointclouds with world*B maps,
    ordered by rank.  Works on NCCL (CUDA tensors) and on gloo (CPU tensors, used by the CPU tests).
    Blocking convenience wrapper around gather_maps_begin / gather_maps_end."""
    if dist.get_world_size(group) == 1 and into is None:
        return pointclouds
    return gather_maps_end(gather_maps_begin(pointclouds, group, into), wait=True)


def _all_gather(recv, send, group):
    if send.is_cuda:
        dist.all_gather_into_tensor(recv, send, group=group)
    else:
        chunks = list(recv.chunk(dist.get_world_size(group), dim=0))
        dist.all_gather(chunks, send, group=group)
