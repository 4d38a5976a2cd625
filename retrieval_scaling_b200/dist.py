"""Multi-GPU search over a statically partitioned datastore (SURVEY.md §8e).

The reference shards the datastore by process (one SLURM job / Flask worker per shard) and merges late:
"concat the per-shard top-k, sort by score descending (stable), keep k" (`src/search.py:357-367`,
`api/serve_main_node.py:130-163`).  Here: one process per GPU, shared centroids / codebooks, every rank scores
ALL queries against the vectors it owns, then the per-shard (scores, ids) are combined on every rank.  Because
the union of the local top-k contains the global top-k, G-GPU results equal the single-index results.

Two ways to combine, same result:
  * fused (default when the ranks can map each other's memory): every rank writes its local top-k straight into a
    symmetric-memory buffer; after one device-side cross-GPU barrier the merge kernel (`rsb_merge_topk_peers`)
    reads all shards IN PLACE with P2P loads over NVLink / NVSwitch -- the all-gather is fused into the merge,
    no NCCL launch and no gather buffer.
  * NCCL: `all_gather_into_tensor` of scores and ids, then `rsb_merge_topk`.
The coarse quantizer is per-query work, so it is sharded by query (rank r scores nq/G queries against the
replicated centroids) and its small (list, score) tables are all-gathered.

`ShardedSearcher` takes the local search / merge callables so that the host-side logic can be exercised with
the `gloo` backend on CPU (tests inject the CPU oracle there; the product default is the CUDA path).
"""
from __future__ import annotations

import ctypes
from typing import Callable, Optional, Tuple

import torch


def shard_rows(n: int, world: int, rank: int, chunk: int = 1_000_000):
    """Vector-wise static partition: chunk c of `chunk` rows belongs to rank c % world.
    Returns the list of (row_start, row_end) ranges owned by `rank`."""
    out = []
    nchunks = (n + chunk - 1) // chunk
    for c in range(rank, nchunks, world):
        out.append((c * chunk, min(n, (c + 1) * chunk)))
    return out


class PeerTopK:
    """Double-buffered symmetric-memory slots for the per-rank top-k plus the device pointer tables the fused
    merge kernel dereferences."""

    def __init__(self, nq: int, k: int, world: int, rank: int, device, group=None, nprobe: int = 0):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem
        self.nq, self.k, self.world, self.rank, self.nprobe = nq, k, world, rank, int(nprobe)
        self.per = (nq + world - 1) // world
        self.i_bytes, self.d_bytes = nq * k * 8, nq * k * 4
        self.slot_bytes = (self.i_bytes + self.d_bytes + 255) // 256 * 256
        # slots 0,1: this rank's local top-k (read by the peers); slots 2,3: the merged result (written by the peers);
        # then 2 threshold arrays [nq] uint32 (raised by every GPU while it scans, DESIGN.md §5) and 2 coarse-table
        # slots (list ids int64 + scores float32 of world*per rows, each rank's slice stored by that rank)
        self.tau_bytes = (nq * 4 + 255) // 256 * 256
        rows = world * self.per
        self.cI_bytes = (rows * self.nprobe * 8 + 255) // 256 * 256
        self.cS_bytes = (rows * self.nprobe * 4 + 255) // 256 * 256
        self.tau_base = 4 * self.slot_bytes
        self.coarse_base = self.tau_base + 2 * self.tau_bytes
        total = self.coarse_base + 2 * (self.cI_bytes + self.cS_bytes)
        self.buf = symm_mem.empty(total, dtype=torch.uint8, device=device)
        self.hdl = symm_mem.rendezvous(self.buf, group if group is not None else dist.group.WORLD)
        self.buf.zero_()
        ptrs = [int(p) for p in self.hdl.buffer_ptrs]
        self.I_tab, self.D_tab, self.I_loc, self.D_loc = [], [], [], []
        for s in range(4):
            base = s * self.slot_bytes
            self.I_tab.append(torch.tensor([p + base for p in ptrs], dtype=torch.int64, device=device))
            self.D_tab.append(torch.tensor([p + base + self.i_bytes for p in ptrs], dtype=torch.int64, device=device))
            self.I_loc.append(self.buf[base: base + self.i_bytes].view(torch.int64).view(nq, k))
            self.D_loc.append(self.buf[base + self.i_bytes: base + self.i_bytes + self.d_bytes].view(torch.float32).view(nq, k))
        self.tau_tab, self.tau_loc, self.cI_tab, self.cS_tab, self.cI_loc, self.cS_loc = [], [], [], [], [], []
        for s in range(2):
            tb = self.tau_base + s * self.tau_bytes
            self.tau_tab.append(torch.tensor([p + tb for p in ptrs], dtype=torch.int64, device=device))
            self.tau_loc.append(self.buf[tb: tb + nq * 4].view(torch.int32))          # uint32 bit patterns
            cb = self.coarse_base + s * (self.cI_bytes + self.cS_bytes)
            self.cI_tab.append(torch.tensor([p + cb for p in ptrs], dtype=torch.int64, device=device))
            self.cS_tab.append(torch.tensor([p + cb + self.cI_bytes for p in ptrs], dtype=torch.int64, device=device))
            if self.nprobe:
                self.cI_loc.append(self.buf[cb: cb + rows * self.nprobe * 8].view(torch.int64).view(rows, self.nprobe))
                self.cS_loc.append(self.buf[cb + self.cI_bytes: cb + self.cI_bytes + rows * self.nprobe * 4]
                                   .view(torch.float32).view(rows, self.nprobe))
        self.step = 0
        self.sliced = True           # False: every rank merges all queries itself (one barrier, G x the peer reads)
        torch.cuda.current_stream().synchronize()
        self.hdl.barrier(channel=0)  # every rank's buffer is zeroed before anybody raises a threshold in it

    # ---- coarse tables: each rank scores 1/G of the queries and stores its rows into every GPU's slot (P2P stores) ----
    def coarse_ok(self, nprobe: int) -> bool:
        return self.nprobe == int(nprobe) and self.nprobe > 0 and (self.per * self.nprobe) % 4 == 0

    def publish_coarse(self, slot: int, L_loc: torch.Tensor, S_loc: torch.Tensor):
        """L_loc int64 / S_loc float32 [per, nprobe] (this rank's rows, padded to `per`) -> (L_all, S_all) [nq, nprobe]
        views of this GPU's slot after every rank has stored its rows and a cross-GPU barrier."""
        from . import _lib
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        L = _lib.lib()
        _lib.check(L.rsb_peer_broadcast(ctypes.c_void_p(L_loc.data_ptr()), L_loc.numel() * 8,
                                        ctypes.c_void_p(self.cI_tab[slot].data_ptr()), self.world,
                                        self.rank * self.per * self.nprobe * 8, st))
        _lib.check(L.rsb_peer_broadcast(ctypes.c_void_p(S_loc.data_ptr()), S_loc.numel() * 4,
                                        ctypes.c_void_p(self.cS_tab[slot].data_ptr()), self.world,
                                        self.rank * self.per * self.nprobe * 4, st))
        self.hdl.barrier(channel=2)
        return self.cI_loc[slot][: self.nq], self.cS_loc[slot][: self.nq]

    def tau_args(self, slot: int):
        """Threshold arrays of this step; the OTHER parity's array is zeroed here for the next step.  Safe: its last
        writers (the peers' scans two steps ago... of the previous step with that parity) finished before the combine
        barrier this rank has already passed in stream order, and no peer can start the next step's scan before this
        rank reaches the coming combine barrier, which is enqueued after this memset."""
        self.tau_loc[slot ^ 1].zero_()
        return self.tau_loc[slot], self.tau_tab[slot], self.world

    def next_slot(self):
        s = self.step & 1
        self.step += 1
        return s, (self.I_loc[s], self.D_loc[s])

    def merge(self, slot: int, k_out: int, local_only: bool = False):
        """Cross-GPU barrier (orders every rank's search before the peer reads), then the fused gather+merge.

        Sliced (default, k_out == k): rank r merges queries [r*per, (r+1)*per) only and stores the merged rows
        into every rank's result slot; a second barrier makes the full result visible everywhere.  Slot re-use
        two steps later is ordered by these barriers (DESIGN.md §5): a rank cannot pass barrier A of step t+2
        before every rank has enqueued -- hence, in stream order, finished -- its reads of step t.

        `local_only` (sliced mode): the merged rows are stored into THIS rank's result slot only and the second
        barrier is skipped; returns (lo, n, I_rows, D_rows) -- views of the rows this rank merged (valid until the
        same slot is merged again two searches later).  The input slots stay safe without the second barrier: they
        are rewritten by the scan of step t+2, which every rank enqueues after barrier A of step t+1, and that
        barrier is passed only when every rank has finished (stream order) its merge reads of step t."""
        from . import _lib
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        dev = self.buf.device
        self.hdl.barrier(channel=0)
        if self.sliced and k_out == self.k:
            per = (self.nq + self.world - 1) // self.world
            lo = min(self.nq, self.rank * per)
            n = min(self.nq, lo + per) - lo
            out = 2 + slot
            if local_only:
                _lib.check(_lib.lib().rsb_merge_topk_peers_scatter(
                    ctypes.c_void_p(self.D_tab[slot].data_ptr()), ctypes.c_void_p(self.I_tab[slot].data_ptr()), self.world,
                    lo, n, self.k, k_out, ctypes.c_void_p(self.D_tab[out].data_ptr() + 8 * self.rank),
                    ctypes.c_void_p(self.I_tab[out].data_ptr() + 8 * self.rank), 1, st))
                return lo, n, self.I_loc[out][lo:lo + n], self.D_loc[out][lo:lo + n]
            _lib.check(_lib.lib().rsb_merge_topk_peers_scatter(
                ctypes.c_void_p(self.D_tab[slot].data_ptr()), ctypes.c_void_p(self.I_tab[slot].data_ptr()), self.world,
                lo, n, self.k, k_out, ctypes.c_void_p(self.D_tab[out].data_ptr()),
                ctypes.c_void_p(self.I_tab[out].data_ptr()), self.world, st))
            self.hdl.barrier(channel=1)
            # private copies: the result slot is overwritten by the peers two searches later
            return self.I_loc[out].clone(), self.D_loc[out].clone()
        D = torch.empty((self.nq, k_out), dtype=torch.float32, device=dev)
        I = torch.empty((self.nq, k_out), dtype=torch.int64, device=dev)
        _lib.check(_lib.lib().rsb_merge_topk_peers(
            ctypes.c_void_p(self.D_tab[slot].data_ptr()), ctypes.c_void_p(self.I_tab[slot].data_ptr()), self.world,
            self.nq, self.k, k_out, ctypes.c_void_p(D.data_ptr()), ctypes.c_void_p(I.data_ptr()), st))
        if local_only:
            per = (self.nq + self.world - 1) // self.world
            lo = min(self.nq, self.rank * per)
            n = min(self.nq, lo + per) - lo
            return lo, n, I[lo:lo + n], D[lo:lo + n]
        return I, D


class ShardedSearcher:
    def __init__(self, index=None, world: int = 1, rank: int = 0, group=None,
                 search_fn: Optional[Callable] = None, merge_fn: Optional[Callable] = None,
                 shard_coarse: bool = True, fused_gather: bool = True, sliced_merge: bool = True,
                 share_tau: bool = True, peer_coarse: bool = True):
        from .index import IndexFlatIP, IndexIVFScalarQuantizer, IndexRefine, _IVFBase
        if isinstance(index, _IVFBase) and index.tiered:
            raise NotImplementedError("ShardedSearcher does not search a tiered IVF index (list_device_rows: lists in host "
                                      "memory): search it per shard group (search.GroupSearcher) or with index.search "
                                      "on one GPU")
        if isinstance(index, IndexFlatIP) and index.tiered:
            raise NotImplementedError("ShardedSearcher does not search a tiered Flat index (rows in host memory): search "
                                      "it per shard group (search.GroupSearcher) or with index.search on one GPU")
        if isinstance(index, IndexIVFScalarQuantizer) and int(world) > 1:
            raise NotImplementedError("ShardedSearcher over several GPUs is implemented for IVF-Flat and nbits = 8 IVF-PQ "
                                      "indexes, not IVF-SQ8.  Search it per shard group (search.GroupSearcher) or on one GPU")
        if isinstance(index, IndexRefine) and int(world) > 1:
            raise NotImplementedError("ShardedSearcher partitions one index over the GPUs; re-ranking would need the "
                                      "candidates' store rows from peer GPUs, which is not implemented.  Re-rank per "
                                      "shard group instead (search.GroupSearcher) or search on one GPU")
        if int(world) > 1 and getattr(index, "nbits", 8) != 8:
            raise NotImplementedError(f"ShardedSearcher over several GPUs is implemented for nbits = 8 IVF-PQ indexes; this "
                                      f"index has nbits = {index.nbits}.  Search it per shard group (search.GroupSearcher) "
                                      f"or on one GPU")
        self.sliced_merge = bool(sliced_merge)
        # with the fused (symmetric-memory) gather: exchange the running top-k thresholds between the GPUs during the
        # scan, and publish the sharded coarse tables with P2P stores instead of NCCL all-gathers
        self.share_tau, self.peer_coarse = bool(share_tau), bool(peer_coarse)
        self.index, self.world, self.rank, self.group = index, int(world), int(rank), group
        self.shard_coarse = bool(shard_coarse) and search_fn is None
        self.fused_gather = bool(fused_gather) and search_fn is None and merge_fn is None
        self.gather_mode = "none" if self.world == 1 else "nccl"
        self._peer: Optional[PeerTopK] = None
        if search_fn is None:
            if index is None:
                raise ValueError("need an index or a search_fn")
            search_fn = index.search_ids
        if merge_fn is None:
            from .index import merge_topk            # CUDA merge kernel (rsb_merge_topk)

            def merge_fn(D_all, I_all, k):
                D, I = merge_topk(D_all, I_all, k)
                return I, D
        self.search_fn, self.merge_fn = search_fn, merge_fn
        self.timing = False          # when True every search() records CUDA events around its three phases
        self._events = []

    def _mark(self, q):
        if self.timing and q.is_cuda:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self._events.append(e)

    def pop_timing(self):
        """Average device time (ms) of the phases of the searches recorded since the last call:
        sharded coarse + all-gather, local scan (`search_preassigned`), cross-GPU combine."""
        ev, self._events = self._events, []
        if len(ev) < 4:
            return {}
        torch.cuda.synchronize()
        names = ("coarse_gather_ms", "local_search_ms", "combine_ms")
        acc, n = [0.0, 0.0, 0.0], len(ev) // 4
        for i in range(n):
            for j in range(3):
                acc[j] += ev[4 * i + j].elapsed_time(ev[4 * i + j + 1])
        return {nm: a / n for nm, a in zip(names, acc)}

    def _peer_buffers(self, nq: int, k: int, device, nprobe: int = 0) -> Optional[PeerTopK]:
        if not self.fused_gather:
            return None
        if self._peer is not None and (self._peer.nq, self._peer.k, self._peer.nprobe) == (nq, k, int(nprobe)):
            return self._peer
        try:
            self._peer = None
            self._peer = PeerTopK(nq, k, self.world, self.rank, device, self.group, nprobe=nprobe)
            self._peer.sliced = self.sliced_merge
            self.gather_mode = "fused-p2p" + ("-sliced" if self.sliced_merge else "")
        except Exception as e:  # no P2P mapping between the ranks (or an older torch): NCCL all-gather instead
            import warnings
            warnings.warn(f"symmetric-memory gather unavailable ({type(e).__name__}: {e}); using NCCL all-gather")
            self.fused_gather = False
            self._peer = None
            self.gather_mode = "nccl"
        return self._peer

    def upload_buffers(self, nq: int, d: int, dtype, device):
        """(slice, gathered) device buffers for `upload_queries(..., buffers=)`: a caller that uploads on its own copy
        stream every step keeps them, because a fresh allocation there is served by the caching allocator's pool of THAT
        stream and, while the previous blocks are still held for the search stream (`record_stream`), ends in a
        cudaMalloc -- a device-wide synchronisation in the middle of the pipeline."""
        per = (nq + self.world - 1) // self.world
        return (torch.zeros((per, d), dtype=dtype, device=device),            # rows past this rank's slice stay zero
                torch.empty((self.world * per, d), dtype=dtype, device=device))

    def upload_queries(self, q_host: torch.Tensor, device, buffers=None) -> torch.Tensor:
        """Every rank holds the same host `q_host` [nq, d] (pinned memory for asynchronous copies).  Instead of each of
        the G ranks pulling all nq rows over its PCIe link, rank r uploads only rows [r*per, (r+1)*per) and the slices
        are all-gathered on the devices (NVLink): each query row crosses PCIe once per job."""
        nq, d = q_host.shape
        if self.world == 1:
            return q_host.to(device, non_blocking=True)
        import torch.distributed as dist
        per = (nq + self.world - 1) // self.world
        lo, hi = min(nq, self.rank * per), min(nq, (self.rank + 1) * per)
        q_loc, q_all = buffers if buffers is not None else self.upload_buffers(nq, d, q_host.dtype, device)
        if hi > lo:
            q_loc[: hi - lo].copy_(q_host[lo:hi], non_blocking=True)
        dist.all_gather_into_tensor(q_all, q_loc, group=self.group)
        return q_all[:nq]

    def search_host(self, q_host: torch.Tensor, k: int, device=None, out: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                    out_slice: bool = False):
        """Host-resident queries in, host-resident (ids, scores) out -- the end-to-end call of one SPMD rank.

        `out` = optional pinned (ids, scores) host tensors to fill; the device->host copy is synchronised before
        returning.  `out_slice=False`: every rank receives the full [nq, k] result.  `out_slice=True`: rank r receives
        only the rows [r*per, (r+1)*per) it merged (out tensors of >= per rows; rows beyond its slice are untouched):
        the job's result lands in host memory exactly once, spread over the ranks like the queries were."""
        dev = torch.device(device) if device is not None else (
            torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu"))
        q = self.upload_queries(q_host, dev)
        return self.search_to_host(q, k, out=out, out_slice=out_slice)

    def search_to_host(self, q: torch.Tensor, k: int, out: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                       out_slice: Optional[bool] = None):
        """Device-resident queries in, host (ids, scores) out.  `out_slice=None` picks the slice form whenever `out`
        is too small for the full result."""
        nq = q.shape[0]
        per = (nq + self.world - 1) // self.world
        if out_slice is None:
            out_slice = self.world > 1 and out is not None and out[0].shape[0] < nq
        if out_slice and self.world > 1:
            lo, n, I, D = self.search_slice(q, k)
            rows = per
        else:
            I, D = self.search(q, k)
            n = rows = nq
        if out is None:
            out = (torch.empty((rows, k), dtype=torch.int64, pin_memory=I.is_cuda),
                   torch.empty((rows, k), dtype=torch.float32, pin_memory=I.is_cuda))
        out[0][:n].copy_(I, non_blocking=True)
        out[1][:n].copy_(D, non_blocking=True)
        if I.is_cuda:
            torch.cuda.current_stream().synchronize()
        return out

    def search_slice(self, q: torch.Tensor, k: int):
        """(lo, n, ids [n,k], scores [n,k]): the merged rows of queries [lo, lo+n) -- this rank's 1/G of the batch.
        With the fused sliced gather this costs ONE cross-GPU barrier and no broadcast of the merged rows."""
        nq = q.shape[0]
        per = (nq + self.world - 1) // self.world
        lo = min(nq, self.rank * per)
        n = min(nq, lo + per) - lo
        if self.world == 1:
            I, D = self.search_fn(q, k)
            return 0, nq, I, D
        res = self._search_impl(q, k, local_only=True)
        if len(res) == 4:
            return res
        I, D = res
        return lo, n, I[lo:lo + n], D[lo:lo + n]

    def search(self, q: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """q [nq, d] (replicated on every rank) -> (ids [nq,k], scores [nq,k]), replicated on every rank."""
        if self.world == 1:
            return self.search_fn(q, k)
        return self._search_impl(q, k, local_only=False)

    def _search_impl(self, q: torch.Tensor, k: int, local_only: bool):
        import torch.distributed as dist
        nq = q.shape[0]
        sharded_coarse = self.shard_coarse and self.index is not None and hasattr(self.index, "search_preassigned")
        nprobe = int(self.index.nprobe) if sharded_coarse else 0
        peer = self._peer_buffers(nq, k, q.device, nprobe) if q.is_cuda else None
        slot, out = (None, None) if peer is None else peer.next_slot()
        self._mark(q)
        if sharded_coarse:
            # The coarse quantizer is per-query work that would otherwise be replicated on every rank: rank r scores
            # queries [r*per, (r+1)*per) against the (replicated) centroids, the (list, score) tables reach every GPU
            # (nq * nprobe * 12 bytes: P2P stores into symmetric memory + one barrier, or two NCCL all-gathers), and
            # every rank scans its slice of those lists.
            per = (nq + self.world - 1) // self.world
            lo, hi = min(nq, self.rank * per), min(nq, (self.rank + 1) * per)
            L_loc = torch.full((per, nprobe), -1, dtype=torch.int64, device=q.device)
            S_loc = torch.zeros((per, nprobe), dtype=torch.float32, device=q.device)
            if hi > lo:
                l, s = self.index.coarse(q[lo:hi], nprobe)
                L_loc[: hi - lo] = l
                S_loc[: hi - lo] = s
            if peer is not None and self.peer_coarse and peer.coarse_ok(nprobe):
                L_all, S_all = peer.publish_coarse(slot, L_loc, S_loc)
            else:
                L_all = torch.empty((self.world * per, nprobe), dtype=torch.int64, device=q.device)
                S_all = torch.empty((self.world * per, nprobe), dtype=torch.float32, device=q.device)
                dist.all_gather_into_tensor(L_all, L_loc, group=self.group)
                dist.all_gather_into_tensor(S_all, S_loc, group=self.group)
                L_all, S_all = L_all[:nq], S_all[:nq]
            self._mark(q)
            tau = peer.tau_args(slot) if (peer is not None and self.share_tau) else None
            I, D = self.index.search_preassigned(q, k, L_all, S_all, out=out, shared_tau=tau)
        elif out is not None:
            self._mark(q)
            I, D = self.index.search_ids(q, k, out=out)
        else:
            self._mark(q)
            I, D = self.search_fn(q, k)
        self._mark(q)
        if peer is not None:
            res = peer.merge(slot, k, local_only=local_only)
            self._mark(q)
            return res
        # output is the concatenation along dim 0 (the layout both NCCL and gloo accept): [world * nq, k]
        I_all = torch.empty((self.world * nq, k), dtype=I.dtype, device=I.device)
        D_all = torch.empty((self.world * nq, k), dtype=D.dtype, device=D.device)
        dist.all_gather_into_tensor(I_all, I.contiguous(), group=self.group)
        dist.all_gather_into_tensor(D_all, D.contiguous(), group=self.group)
        res = self.merge_fn(D_all.view(self.world, nq, k), I_all.view(self.world, nq, k), k)
        self._mark(q)
        return res


class HostPipeline:
    """Stream of host-resident query batches through a `ShardedSearcher`: the host->device copy of batch i+1 and the
    device->host copy of batch i-1 run on their own streams while batch i is searched (PCIe is full duplex and the copy
    engines are idle during a search), every batch still being uploaded, searched and downloaded in full.

        pipe = HostPipeline(searcher, device)
        for q_host, out in batches:            # pinned host tensors; out = (ids, scores) to fill
            pipe.submit(q_host, k, out)        # returns at once; at most two batches are in flight
        pipe.drain()                           # all results are on the host

    With world > 1 the sliced forms are used (`upload_queries`, `search_slice`): each rank uploads 1/G of every batch and
    receives the rows it merged."""

    def __init__(self, searcher: ShardedSearcher, device, out_slice: bool = True):
        self.s, self.device = searcher, torch.device(device)
        self.out_slice = bool(out_slice) and searcher.world > 1
        self.h2d, self.d2h = torch.cuda.Stream(self.device), torch.cuda.Stream(self.device)
        self.n = 0
        self.ev_up = [torch.cuda.Event(), torch.cuda.Event()]        # upload of parity p finished
        self.ev_done = [torch.cuda.Event(), torch.cuda.Event()]      # search of parity p finished (its query buffer is free)
        self.ev_down = [torch.cuda.Event(), torch.cuda.Event()]      # download of parity p finished (its result slot is free)
        self.q_dev = [None, None]
        self.keep = [None, None]
        self.up_buf = [None, None]                                   # world > 1: (slice, gathered) upload buffers per parity
        self.up_nq = [0, 0]

    def submit(self, q_host: torch.Tensor, k: int, out):
        p = self.n & 1
        main = torch.cuda.current_stream(self.device)
        if self.n >= 2:
            self.h2d.wait_event(self.ev_done[p])                     # batch n-2 no longer reads this query buffer
        with torch.cuda.stream(self.h2d):
            if self.s.world == 1:
                if self.q_dev[p] is None or self.q_dev[p].shape != q_host.shape:
                    self.q_dev[p] = torch.empty(q_host.shape, dtype=q_host.dtype, device=self.device)
                self.q_dev[p].copy_(q_host, non_blocking=True)
                q = self.q_dev[p]
            else:
                # slice upload + NVLink all-gather on the copy stream, into buffers this pipeline keeps (two parities): the
                # events above order their re-use, and nothing is allocated on the copy stream in the steady state
                if self.up_buf[p] is None or self.up_buf[p][1].shape[1] != q_host.shape[1] or \
                        self.up_buf[p][1].shape[0] < q_host.shape[0] or self.up_buf[p][1].dtype != q_host.dtype or \
                        self.up_nq[p] != q_host.shape[0]:
                    self.up_buf[p] = self.s.upload_buffers(q_host.shape[0], q_host.shape[1], q_host.dtype, self.device)
                    self.up_buf[p][0].record_stream(main)
                    self.up_buf[p][1].record_stream(main)
                    self.up_nq[p] = q_host.shape[0]
                q = self.s.upload_queries(q_host, self.device, buffers=self.up_buf[p])
                self.q_dev[p] = q
            self.ev_up[p].record(self.h2d)
        main.wait_event(self.ev_up[p])
        if self.n >= 2:
            main.wait_event(self.ev_down[p])                         # batch n-2's result slot has been copied out
        if self.out_slice:
            lo, n, I, D = self.s.search_slice(q, k)
        else:
            I, D = self.s.search(q, k)
            n = q.shape[0]
        self.ev_done[p].record(main)
        self.keep[p] = (I, D, q)                                     # keep the tensors alive until their copies ran
        I.record_stream(self.d2h)
        D.record_stream(self.d2h)
        self.d2h.wait_event(self.ev_done[p])
        with torch.cuda.stream(self.d2h):
            out[0][:n].copy_(I, non_blocking=True)
            out[1][:n].copy_(D, non_blocking=True)
            self.ev_down[p].record(self.d2h)
        self.n += 1

    def drain(self):
        self.h2d.synchronize()
        torch.cuda.current_stream(self.device).synchronize()
        self.d2h.synchronize()
