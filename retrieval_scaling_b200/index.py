"""GPU index objects exposing the faiss object protocol the reference's wrappers use
(`src/indicies/flat.py:42,58,139`, `ivf_flat.py:73,143-149,166,171,180,225`, `ivf_pq.py:76,146-154,170,185,230`):

    index.train(x) / index.add(x) / index.search(x, k) -> (D float32 [nq,k], I int64 [nq,k])
    index.nprobe, index.ntotal, index.is_trained, index.d
    write_index(index, path) / read_index(path)

All numerics run in librsb.so (hand-written sm_90a CUDA, C-ABI `include/rsb.h`); torch is used for device
memory and streams only.  No CPU fallback: constructing an index without a CUDA device raises.

Inputs may be numpy arrays (any float dtype; upcast to fp32 like `query_embs.astype(np.float32)` in
`flat.py:139`) or torch tensors on any device; `search` returns numpy for numpy input and CUDA tensors for
torch input (`search_ids` always returns CUDA tensors: the "(ids, scores) out" fast path of the north star).
"""
from __future__ import annotations

import ctypes
import os
import pickle
from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib
from . import train as _train

NEG = float(np.finfo(np.float32).min)


def _require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("retrieval_scaling_b200 needs a CUDA device (H100, sm_90a): there is no CPU path")


def _dev_f32(x, device) -> torch.Tensor:
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(np.ascontiguousarray(x))
    if not isinstance(x, torch.Tensor):
        x = torch.as_tensor(x)
    return x.to(device=device, dtype=torch.float32, non_blocking=True).contiguous()


def _dev_rows(x, device) -> torch.Tensor:
    """Vectors to add: fp16 tensors / arrays stay fp16 (they cross PCIe at 2 bytes per element; rsb_add converts
    them on the device), anything else becomes fp32 as in _dev_f32."""
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(np.ascontiguousarray(x))
    if not isinstance(x, torch.Tensor):
        x = torch.as_tensor(x)
    dtype = torch.float16 if x.dtype == torch.float16 else torch.float32
    return x.to(device=device, dtype=dtype, non_blocking=True).contiguous()


# storage dtypes of Flat / IVF-Flat vectors (rsb_flat_create / rsb_ivfflat_create) and of IndexRefine's store
_STORE_DTYPES = {"float16": (torch.float16, _lib.RSB_DTYPE_F16), "float32": (torch.float32, _lib.RSB_DTYPE_F32)}


# IndexRefine's store and IndexIVFScalarQuantizer's lists: the storage dtypes, plus "sq8" (uint8 codes of a trained
# scalar quantizer)
_REFINE_DTYPES = {**_STORE_DTYPES, "sq8": (torch.uint8, _lib.RSB_DTYPE_SQ8)}


def _dtype_code(x: torch.Tensor) -> int:
    return _lib.RSB_DTYPE_F16 if x.dtype == torch.float16 else _lib.RSB_DTYPE_F32


def _check_dtype(dtype: str, what: str = "dtype") -> str:
    if dtype not in _STORE_DTYPES:
        raise ValueError(f"{what} must be float16 or float32, got {dtype!r}")
    return dtype


def _check_rows_arg(v, name: str) -> Optional[int]:
    if v is None:
        return None
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or v < 0:
        raise ValueError(f"{name} must be None or an integer >= 0, got {v!r}")
    return int(v)


def _check_device_rows(device_rows) -> Optional[int]:
    """The device_rows argument of IndexFlatIP, IndexRefine and read_index."""
    return _check_rows_arg(device_rows, "device_rows")


def _as_storage(x: np.ndarray, dtype: str, what: str) -> np.ndarray:
    """Host vectors for an index that stores `dtype`: an fp16 index accepts only values that round-trip through fp16."""
    if dtype != "float16" or x.dtype == np.float16:
        return x
    xh = x.astype(np.float16)
    if not np.array_equal(xh.astype(x.dtype), x):
        raise ValueError(f"{what}: not every value is representable in float16; use float32 storage")
    return xh


def _ptr(t: Optional[torch.Tensor]):
    return ctypes.c_void_p(t.data_ptr()) if t is not None and t.numel() > 0 else ctypes.c_void_p(0)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class _IndexBase:
    kind = None
    dtype = "float32"      # storage dtype of the vectors (Flat / IVF-Flat may hold float16)

    def __init__(self, d: int, device=None):
        _require_cuda()
        self.L = _lib.lib()
        self.d = int(d)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._h = ctypes.c_void_p(0)
        self._ws: Optional[torch.Tensor] = None
        self.nprobe = 1
        self.verbose = False

    # -- lifetime ------------------------------------------------------------------------------------------
    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                self.L.rsb_free(self._h)
                self._h = ctypes.c_void_p(0)
        except Exception:
            pass

    def _info(self, what: int) -> int:
        out = ctypes.c_int64(0)
        _lib.check(self.L.rsb_info(self._h, what, ctypes.byref(out)))
        return int(out.value)

    @property
    def ntotal(self) -> int:
        return self._info(_lib.INFO_NTOTAL)

    @property
    def is_trained(self) -> bool:
        return bool(self._info(_lib.INFO_IS_TRAINED))

    @property
    def index_bytes(self) -> int:
        return self._info(_lib.INFO_INDEX_BYTES)

    @property
    def n_dev(self) -> int:
        """Rows held in device memory: ntotal unless tiered (a tiered IVF index: those of lists [0, L_dev) once the
        lists are reserved)."""
        return self._info(_lib.INFO_DEVICE_ROWS)

    @property
    def host_bytes(self) -> int:
        """Page-locked host bytes of the host tier (0 unless tiered)."""
        return self._info(_lib.INFO_HOST_BYTES)

    def _workspace(self, nbytes: int) -> torch.Tensor:
        nbytes = max(int(nbytes), 256)
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = None
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        return self._ws

    # -- protocol ------------------------------------------------------------------------------------------
    def train(self, x) -> None:  # Flat: nothing to train (faiss no-op)
        return None

    def add(self, x, ids=None) -> None:
        with torch.cuda.device(self.device):
            x = _dev_f32(x, self.device) if self.kind == _lib.RSB_IVFPQ else _dev_rows(x, self.device)
            if x.dim() != 2 or x.shape[1] != self.d:
                raise ValueError(f"expected [n, {self.d}] vectors, got {tuple(x.shape)}")
            n = x.shape[0]
            idt = None
            if ids is not None:
                idt = torch.as_tensor(ids).to(device=self.device, dtype=torch.int64).contiguous()
                if idt.numel() != n:
                    raise ValueError("ids and x disagree on n")
            ws = self._workspace(self.L.rsb_add_workspace_bytes(self._h, n))
            _lib.check(self.L.rsb_add(self._h, _ptr(x), _dtype_code(x), n, _ptr(idt), _ptr(ws), ws.numel(), _stream()))
            torch.cuda.current_stream().synchronize()  # x / idt may be temporaries

    def finalize(self) -> None:
        with torch.cuda.device(self.device):
            _lib.check(self.L.rsb_finalize(self._h, _stream()))

    def search_ids(self, q: torch.Tensor, k: int, nprobe: Optional[int] = None,
                   out: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Fast path: q CUDA float32 [nq, d] -> (ids int64 [nq,k], scores float32 [nq,k]) CUDA tensors,
        enqueued on the current stream (no host sync unless adds are pending).  `out=(I, D)` lets the caller
        provide the result buffers (e.g. symmetric memory that peer GPUs read in place)."""
        with torch.cuda.device(self.device):
            q = _dev_f32(q, self.device)
            if q.dim() != 2 or q.shape[1] != self.d:
                raise ValueError(f"expected [nq, {self.d}] queries, got {tuple(q.shape)}")
            nq = q.shape[0]
            k = int(k)
            npb = int(self.nprobe if nprobe is None else nprobe)
            if out is not None:
                I, D = out
            else:
                D = torch.empty((nq, k), dtype=torch.float32, device=self.device)
                I = torch.empty((nq, k), dtype=torch.int64, device=self.device)
            if nq == 0:
                return I, D
            ws = self._workspace(self.L.rsb_workspace_bytes(self._h, nq, k, npb))
            _lib.check(self.L.rsb_search(self._h, _ptr(q), nq, k, npb, _ptr(D), _ptr(I), _ptr(ws), ws.numel(), _stream()))
            return I, D

    def search(self, x, k: int):
        """faiss protocol: returns (D, I).  numpy in -> numpy out; torch in -> CUDA tensors out."""
        I, D = self.search_ids(x, k)
        if isinstance(x, np.ndarray) or not isinstance(x, torch.Tensor):
            return D.cpu().numpy(), I.cpu().numpy()
        return D, I

    def set_option(self, option: int, value: int) -> None:
        _lib.check(self.L.rsb_set_option(self._h, int(option), int(value)))

    # -- profiling -----------------------------------------------------------------------------------------
    def set_profiling(self, on: bool = True) -> None:
        _lib.check(self.L.rsb_set_profiling(self._h, 1 if on else 0))

    def profile(self) -> dict:
        buf = (ctypes.c_double * len(_lib.PROF_NAMES))()
        _lib.check(self.L.rsb_get_profile(self._h, buf, len(_lib.PROF_NAMES)))
        return {n: float(buf[i]) for i, n in enumerate(_lib.PROF_NAMES)}

    # -- export (natural CSR order: what the oracle and a faiss file writer consume) --------------------------
    def export_rows(self, r0: int, n: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Rows [r0, r0 + n) of a Flat or IVF-Flat / IVF-SQ8 index (IVF: CSR rows, the natural order of export_lists)
        in the storage dtype, from whichever tier holds them, into `out` (a contiguous [n, d] CPU or CUDA tensor;
        default: a new CPU tensor)."""
        dt = _REFINE_DTYPES[self.dtype][0]
        if out is None:
            out = torch.empty((int(n), self.d), dtype=dt)
        if tuple(out.shape) != (int(n), self.d) or out.dtype != dt or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous [{n}, {self.d}] {self.dtype} tensor")
        with torch.cuda.device(self.device):
            _lib.check(self.L.rsb_export_rows(self._h, int(r0), int(n), _ptr(out), _stream()))
            torch.cuda.current_stream().synchronize()
        return out

    def export_lists(self):
        with torch.cuda.device(self.device):
            self.finalize()
            n = self.ntotal
            nlist = max(1, self._info(_lib.INFO_NLIST))
            off = torch.zeros(nlist + 1, dtype=torch.int64, device=self.device)
            if self.kind == _lib.RSB_IVFPQ:
                code_size = self._info(_lib.INFO_M) * self._info(_lib.INFO_NBITS) // 8
                payload = torch.empty((n, code_size), dtype=torch.uint8, device=self.device)
            else:
                payload = torch.empty((n, self.d), dtype=_REFINE_DTYPES[self.dtype][0], device=self.device)
            ids = torch.empty(n, dtype=torch.int64, device=self.device)
            _lib.check(self.L.rsb_export_lists(self._h, _ptr(off), _ptr(payload), _ptr(ids), _stream()))
            torch.cuda.current_stream().synchronize()
            return off, payload, ids


class IndexFlatIP(_IndexBase):
    """faiss.IndexFlatIP(d)  (reference: src/indicies/flat.py:42).

    dtype="float16" stores the vectors as fp16 (faiss IndexScalarQuantizer(QT_fp16, METRIC_INNER_PRODUCT)): half the
    bytes, scored on tensor cores from the fp16 rows at any size that fits (d % 64 == 0, else NotImplementedError),
    with exact fp32 final scores.  Lossless for the fp16 embeddings the embedding task writes.

    device_rows = n (an integer; float16 only) makes the index tiered, for datastores larger than device memory: rows
    [0, n) stay in device memory and rows from n on go to page-locked host memory the index owns.  Each search streams
    the host rows through two device staging buffers of `staging_bytes` each (None: the library's 256 MiB) while the
    tensor cores score; the ids are tie-equivalent and the scores bit-equal (where the ids agree) to the all-device
    index, and with n >= ntotal the search is the all-device one.  add() of host rows (numpy, CPU tensors) copies the
    rows bound for the host tier host to host."""
    kind = _lib.RSB_FLAT

    def __init__(self, d: int, device=None, dtype: str = "float32", device_rows: Optional[int] = None,
                 staging_bytes: Optional[int] = None):
        dtype, device_rows = _check_dtype(dtype), _check_device_rows(device_rows)   # before any device allocation
        if device_rows is not None and dtype != "float16":
            raise ValueError(f"device_rows (a tiered Flat index) needs dtype='float16'; a {dtype} Flat index stays in "
                             f"device memory")
        super().__init__(d, device)
        self.dtype, self.device_rows = dtype, device_rows
        with torch.cuda.device(self.device):
            _lib.check(self.L.rsb_flat_create(self.d, _STORE_DTYPES[self.dtype][1], ctypes.byref(self._h)))
            if self.device_rows is not None:
                self.set_option(_lib.OPT_DEVICE_ROWS, self.device_rows)
                if staging_bytes is not None:
                    self.set_option(_lib.OPT_STAGING_BYTES, int(staging_bytes))

    @property
    def tiered(self) -> bool:
        return self.device_rows is not None

    def add(self, x, ids=None) -> None:
        if not self.tiered:
            return super().add(x, ids)
        # tiered: host rows are handed over where they are (the library copies host-tier rows host to host)
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x if x.dtype in (np.float16, np.float32) else x.astype(np.float32)))
        x = torch.as_tensor(x)
        if x.dtype not in (torch.float16, torch.float32):
            x = x.float()
        x = x.contiguous()
        if x.dim() != 2 or x.shape[1] != self.d:
            raise ValueError(f"expected [n, {self.d}] vectors, got {tuple(x.shape)}")
        with torch.cuda.device(self.device):
            if x.is_cuda and x.device != self.device:
                x = x.to(self.device)
            idt = None
            if ids is not None:
                idt = torch.as_tensor(ids).to(device=self.device, dtype=torch.int64).contiguous()
                if idt.numel() != x.shape[0]:
                    raise ValueError("ids and x disagree on n")
            _lib.check(self.L.rsb_add(self._h, _ptr(x), _dtype_code(x), x.shape[0], _ptr(idt), None, 0, _stream()))
            torch.cuda.current_stream().synchronize()  # x / idt may be temporaries

    def export_ids(self) -> torch.Tensor:
        """The ids of rows [0, ntotal) (a CUDA int64 tensor)."""
        with torch.cuda.device(self.device):
            self.finalize()
            ids = torch.empty(self.ntotal, dtype=torch.int64, device=self.device)
            _lib.check(self.L.rsb_export_lists(self._h, None, None, _ptr(ids), _stream()))
            torch.cuda.current_stream().synchronize()
        return ids


class _IVFBase(_IndexBase):
    # tiered IVF-Flat / IVF-SQ8 (list_device_rows set): lists are split by id between device memory and page-locked host
    # memory, which needs the list sizes before the first add (reserve_lists)
    list_device_rows: Optional[int] = None
    staging_bytes: Optional[int] = None

    def __init__(self, d, nlist, device=None):
        super().__init__(d, device)
        self.nlist = int(nlist)
        self._reserved = False

    @staticmethod
    def _tier_args(list_device_rows, staging_bytes):
        """Checks list_device_rows / staging_bytes before any device allocation."""
        return _check_rows_arg(list_device_rows, "list_device_rows"), _check_rows_arg(staging_bytes, "staging_bytes")

    @property
    def tiered(self) -> bool:
        return self.list_device_rows is not None

    def reserve_lists(self, sizes) -> None:
        """Fixes the list sizes [nlist] of a tiered index before anything is added (rsb_reserve_lists): lists [0, L_dev)
        -- the most that fit list_device_rows rows -- get their rows in device memory, the others in page-locked host
        memory.  Every later add places its rows in their final slots; the index is searchable once every reserved row
        has been added."""
        if not self.tiered:
            raise ValueError("reserve_lists splits the lists of a tiered index: construct it with list_device_rows")
        sz = np.ascontiguousarray(np.asarray(sizes.cpu() if isinstance(sizes, torch.Tensor) else sizes), dtype=np.int64)
        if sz.shape != (self.nlist,):
            raise ValueError(f"sizes must be [{self.nlist}] (one size per list), got {sz.shape}")
        with torch.cuda.device(self.device):
            _lib.check(self.L.rsb_reserve_lists(self._h, sz.ctypes.data_as(ctypes.c_void_p), self.list_device_rows,
                                                int(self.staging_bytes or 0), _stream()))
        self._reserved = True

    def _check_reserved(self) -> None:
        if self.tiered and not self._reserved:
            raise ValueError("a tiered IVF index (list_device_rows) places every row in its final slot: call "
                             "reserve_lists(sizes) with the list sizes (e.g. counted from assign()) before adding")

    def add(self, x, ids=None) -> None:
        self._check_reserved()
        return super().add(x, ids)

    def export_ids_host(self) -> np.ndarray:
        """The ids of CSR rows [0, ntotal) as a host int64 array."""
        with torch.cuda.device(self.device):
            self.finalize()
            n = self.ntotal
            ids = torch.empty(n, dtype=torch.int64, device=self.device if not self._reserved else "cpu")
            _lib.check(self.L.rsb_export_lists(self._h, None, None, _ptr(ids), _stream()))
            torch.cuda.current_stream().synchronize()
        return ids.cpu().numpy()

    # trained state ------------------------------------------------------------------------------------------
    def set_centroids(self, c) -> None:
        with torch.cuda.device(self.device):
            c = _dev_f32(c, self.device)
            if tuple(c.shape) != (self.nlist, self.d):
                raise ValueError(f"centroids must be [{self.nlist}, {self.d}], got {tuple(c.shape)}")
            _lib.check(self.L.rsb_set_centroids(self._h, _ptr(c), _stream()))
            torch.cuda.current_stream().synchronize()

    def get_centroids(self) -> torch.Tensor:
        with torch.cuda.device(self.device):
            out = torch.empty((self.nlist, self.d), dtype=torch.float32, device=self.device)
            _lib.check(self.L.rsb_get_centroids(self._h, _ptr(out), _stream()))
            return out

    def coarse(self, q, nprobe: Optional[int] = None):
        with torch.cuda.device(self.device):
            q = _dev_f32(q, self.device)
            npb = int(self.nprobe if nprobe is None else nprobe)
            nq = q.shape[0]
            lists = torch.empty((nq, npb), dtype=torch.int64, device=self.device)
            scores = torch.empty((nq, npb), dtype=torch.float32, device=self.device)
            ws = self._workspace(self.L.rsb_workspace_bytes(self._h, nq, 1, npb))
            _lib.check(self.L.rsb_coarse(self._h, _ptr(q), nq, npb, _ptr(lists), _ptr(scores), _ptr(ws), ws.numel(), _stream()))
            return lists, scores

    def search_preassigned(self, q, k: int, lists, coarse_dis, out=None, shared_tau=None):
        """faiss search_preassigned: probe exactly `lists` [nq, nprobe]; returns (ids, scores) CUDA tensors.
        `shared_tau = (tau_local uint32 [nq] tensor in peer-mapped memory, table of every GPU's array pointer (int64
        CUDA tensor), number of GPUs)`: thresholds are exchanged between the GPUs of a sharded datastore while they scan
        (rsb_search_preassigned); the caller zeroes the arrays and keeps the GPUs within one batch of each other."""
        with torch.cuda.device(self.device):
            q = _dev_f32(q, self.device)
            lt = torch.as_tensor(lists).to(device=self.device, dtype=torch.int64).contiguous()
            cd = _dev_f32(coarse_dis, self.device)
            nq, npb = lt.shape
            if out is not None:
                I, D = out
            else:
                D = torch.empty((nq, k), dtype=torch.float32, device=self.device)
                I = torch.empty((nq, k), dtype=torch.int64, device=self.device)
            ws = self._workspace(self.L.rsb_workspace_bytes(self._h, nq, k, npb))
            tau_local, tau_tab, npeers = (None, None, 0) if shared_tau is None else shared_tau
            _lib.check(self.L.rsb_search_preassigned(self._h, _ptr(q), nq, int(k), npb, _ptr(lt), _ptr(cd), _ptr(D),
                                                     _ptr(I), _ptr(ws), ws.numel(), _ptr(tau_local), _ptr(tau_tab),
                                                     int(npeers), _stream()))
            return I, D

    def assign(self, x) -> torch.Tensor:
        lists, _ = self.coarse(x, 1)
        return lists[:, 0].to(torch.int32)

    def add_preassigned(self, x, lists, ids=None) -> None:
        self._check_reserved()
        with torch.cuda.device(self.device):
            x = _dev_f32(x, self.device) if self.kind == _lib.RSB_IVFPQ else _dev_rows(x, self.device)
            n = x.shape[0]
            lt = torch.as_tensor(lists).to(device=self.device, dtype=torch.int32).contiguous()
            idt = None if ids is None else torch.as_tensor(ids).to(device=self.device, dtype=torch.int64).contiguous()
            _lib.check(self.L.rsb_add_preassigned(self._h, _ptr(x), _dtype_code(x), n, _ptr(idt), _ptr(lt), _stream()))
            torch.cuda.current_stream().synchronize()

    def list_sizes(self) -> torch.Tensor:
        with torch.cuda.device(self.device):
            out = torch.empty(self.nlist, dtype=torch.int64, device=self.device)
            _lib.check(self.L.rsb_list_sizes(self._h, _ptr(out), _stream()))
            return out

    def _train_coarse(self, x: torch.Tensor) -> torch.Tensor:
        c = _train.kmeans(x, self.nlist, niter=10, metric="ip", spherical=True, seed=1234, verbose=self.verbose)
        self.set_centroids(c)
        return c


class IndexIVFFlat(_IVFBase):
    """faiss.IndexIVFFlat(IndexFlatIP(d), d, nlist, METRIC_INNER_PRODUCT)  (src/indicies/ivf_flat.py:143-149).

    dtype="float16" stores the vectors as fp16 (faiss IndexIVFScalarQuantizer(QT_fp16, by_residual=False)): the list
    scan reads half the bytes, and ids and scores are bit-identical to an fp32 index holding the same values.

    list_device_rows = R (an integer) makes the index tiered by list, for datastores larger than device memory: after
    reserve_lists(sizes), lists [0, L_dev) -- the most whose rows fit R -- keep their rows in device memory and the
    others in page-locked host memory the index owns.  A search scans the device lists in place and copies only the
    probed host lists through two device staging buffers of `staging_bytes` each (None: the library's 256 MiB); ids and
    scores equal those of the all-device index of the same lists.  add / add_preassigned need the reservation first."""
    kind = _lib.RSB_IVFFLAT

    def __init__(self, d: int, nlist: int, device=None, dtype: str = "float32", list_device_rows: Optional[int] = None,
                 staging_bytes: Optional[int] = None):
        dtype = _check_dtype(dtype)
        tier = self._tier_args(list_device_rows, staging_bytes)        # before any device allocation
        super().__init__(d, nlist, device)
        self.list_device_rows, self.staging_bytes = tier
        self.dtype = dtype
        with torch.cuda.device(self.device):
            _lib.check(self.L.rsb_ivfflat_create(self.d, self.nlist, _STORE_DTYPES[self.dtype][1],
                                                 ctypes.byref(self._h)))

    def train(self, x) -> None:
        with torch.cuda.device(self.device):
            self._train_coarse(_dev_f32(x, self.device))


class IndexIVFPQ(_IVFBase):
    """faiss.IndexIVFPQ(IndexFlatIP(d), d, nlist, M, nbits, METRIC_INNER_PRODUCT)  (src/indicies/ivf_pq.py:146-152).

    nbits 8 or 4.  4-bit codes are packed two per byte in faiss' order (byte b = c[2b] | c[2b+1] << 4), so `code_size`
    = M * nbits / 8 bytes per vector: codes taken by `add_codes` and returned by `export_lists` are [n, code_size]."""
    kind = _lib.RSB_IVFPQ

    def __init__(self, d: int, nlist: int, M: int, nbits: int = 8, device=None):
        super().__init__(d, nlist, device)
        self.M, self.nbits = int(M), int(nbits)
        with torch.cuda.device(self.device):
            _lib.check(self.L.rsb_ivfpq_create(self.d, self.nlist, self.M, self.nbits, ctypes.byref(self._h)))

    @property
    def code_size(self) -> int:
        return self.M * self.nbits // 8

    def set_codebook(self, cb) -> None:
        with torch.cuda.device(self.device):
            cb = _dev_f32(cb, self.device)
            want = (self.M, 1 << self.nbits, self.d // self.M)
            if tuple(cb.shape) != want:
                raise ValueError(f"codebook must be {want}, got {tuple(cb.shape)}")
            _lib.check(self.L.rsb_set_pq_codebook(self._h, _ptr(cb), _stream()))
            torch.cuda.current_stream().synchronize()

    def get_codebook(self) -> torch.Tensor:
        with torch.cuda.device(self.device):
            out = torch.empty((self.M, 1 << self.nbits, self.d // self.M), dtype=torch.float32, device=self.device)
            _lib.check(self.L.rsb_get_pq_codebook(self._h, _ptr(out), _stream()))
            return out

    def train(self, x) -> None:
        with torch.cuda.device(self.device):
            x = _dev_f32(x, self.device)
            c = self._train_coarse(x)
            gen = torch.Generator(device=x.device)
            gen.manual_seed(1234)
            xs = _train._subsample(x, 256 * (1 << self.nbits), gen)
            a = self.assign(xs).long()
            self.set_codebook(_train.train_pq(xs - c[a], self.M, 1 << self.nbits, niter=25, seed=1234))

    def add_codes(self, codes, lists, ids=None) -> None:
        with torch.cuda.device(self.device):
            ct = torch.as_tensor(codes).to(device=self.device, dtype=torch.uint8).contiguous()
            n = ct.shape[0]
            if ct.dim() != 2 or ct.shape[1] != self.code_size:
                raise ValueError(f"codes must be [n, {self.code_size}] uint8 (M * nbits / 8 bytes per vector), "
                                 f"got {tuple(ct.shape)}")
            lt = torch.as_tensor(lists).to(device=self.device, dtype=torch.int32).contiguous()
            idt = None if ids is None else torch.as_tensor(ids).to(device=self.device, dtype=torch.int64).contiguous()
            _lib.check(self.L.rsb_add_codes(self._h, _ptr(ct), n, _ptr(idt), _ptr(lt), _stream()))
            torch.cuda.current_stream().synchronize()


class IndexIVFScalarQuantizer(_IVFBase):
    """faiss.IndexIVFScalarQuantizer(IndexFlatIP(d), d, nlist, QT_8bit, METRIC_INNER_PRODUCT, by_residual), the index
    index_factory(d, "IVFn,SQ8") builds: inverted lists of one uint8 code per element (a quarter of the fp32 bytes), with
    one (vmin, vdiff) range per dimension (RS_minmax).  d % 16 == 0.

    by_residual=True (faiss' default) encodes x - c_list and scores a vector of list l as fl32(<q, c_l> + s); False
    encodes x and scores s.  s = <q, decode(code)> is accumulated in the fp32 IVF-Flat scan's order from the decoded
    elements vmin + ((c + 0.5f) / 255.f) * vdiff, so it is bit-identical to an fp32 IndexIVFFlat holding the decoded
    rows in the same lists.  train(x) trains the coarse quantizer (as IndexIVFFlat.train) and then the range on the rows
    or on their residuals against the lists add() would assign; train_sq(x) trains the range alone.
    list_device_rows / staging_bytes tier the lists between device and host memory as in IndexIVFFlat."""
    kind = _lib.RSB_IVFFLAT
    dtype = "sq8"
    qtype = "QT_8bit"                   # the only scalar-quantizer type implemented
    _TRAIN_CHUNK = 65536                # rows per coarse assignment while the residuals are formed

    def __init__(self, d: int, nlist: int, by_residual: bool = True, device=None,
                 list_device_rows: Optional[int] = None, staging_bytes: Optional[int] = None):
        tier = self._tier_args(list_device_rows, staging_bytes)        # before any device allocation
        super().__init__(d, nlist, device)
        self.list_device_rows, self.staging_bytes = tier
        with torch.cuda.device(self.device):
            _lib.check(self.L.rsb_ivfflat_create(self.d, self.nlist, _lib.RSB_DTYPE_SQ8, ctypes.byref(self._h)))
        self.set_option(_lib.OPT_BY_RESIDUAL, 1 if by_residual else 0)

    @property
    def by_residual(self) -> bool:
        return bool(self._info(_lib.INFO_BY_RESIDUAL))

    @property
    def code_size(self) -> int:
        return self.d

    @property
    def sq_params(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """The range (vmin [d], vdiff [d]) float32 device tensors."""
        with torch.cuda.device(self.device):
            out = torch.empty((2, self.d), dtype=torch.float32, device=self.device)
            _lib.check(self.L.rsb_get_sq_range(self._h, _ptr(out), _stream()))
            return out[0], out[1]

    @sq_params.setter
    def sq_params(self, sq) -> None:
        """(vmin, vdiff) or a [2, d] array, used exactly as given (e.g. read from a file); only before anything is
        added."""
        with torch.cuda.device(self.device):
            if isinstance(sq, (tuple, list)):
                sq = torch.stack([_dev_f32(t, self.device).reshape(-1) for t in sq])
            sq = _dev_f32(sq, self.device)
            if tuple(sq.shape) != (2, self.d):
                raise ValueError(f"the SQ8 range must be [2, {self.d}] (vmin, vdiff), got {tuple(sq.shape)}")
            _lib.check(self.L.rsb_set_sq_range(self._h, _ptr(sq), _stream()))
            torch.cuda.current_stream().synchronize()

    def train(self, x) -> None:
        with torch.cuda.device(self.device):
            x = _dev_rows(x, self.device)
            self._train_coarse(x.float())
            self.train_sq(x)

    def train_sq(self, x) -> None:
        """Trains the range alone (per-dimension min / max, rsb_sq8_train) on the rows x [n, d] (fp16 or fp32) or, by
        residual, on x - c_list with the lists of the coarse quantizer (nprobe = 1, the assignment add() makes)."""
        with torch.cuda.device(self.device):
            x = _dev_rows(x, self.device)
            if x.dim() != 2 or x.shape[1] != self.d or x.shape[0] == 0:
                raise ValueError(f"expected [n >= 1, {self.d}] training vectors, got {tuple(x.shape)}")
            if self.by_residual:
                c = self.get_centroids()
                r = torch.empty(x.shape, dtype=torch.float32, device=self.device)
                for a in range(0, x.shape[0], self._TRAIN_CHUNK):
                    xc = x[a:a + self._TRAIN_CHUNK].float()             # fp16 rows widen exactly
                    torch.sub(xc, c[self.assign(xc).long()], out=r[a:a + self._TRAIN_CHUNK])
                x = r
            sq = torch.empty((2, self.d), dtype=torch.float32, device=self.device)
            _lib.check(self.L.rsb_sq8_train(_ptr(x), _dtype_code(x), x.shape[0], self.d, _ptr(sq), _stream()))
            self.sq_params = sq

    def add_codes(self, codes, lists, ids=None) -> None:
        """Adds SQ8 codes [n, d] uint8 of this index's range (residual codes when by_residual) to the given lists."""
        self._check_reserved()
        with torch.cuda.device(self.device):
            ct = torch.as_tensor(codes).to(device=self.device, dtype=torch.uint8).contiguous()
            if ct.dim() != 2 or ct.shape[1] != self.d:
                raise ValueError(f"codes must be [n, {self.d}] uint8 (one byte per element), got {tuple(ct.shape)}")
            lt = torch.as_tensor(lists).to(device=self.device, dtype=torch.int32).contiguous()
            idt = None if ids is None else torch.as_tensor(ids).to(device=self.device, dtype=torch.int64).contiguous()
            _lib.check(self.L.rsb_add_codes(self._h, _ptr(ct), ct.shape[0], _ptr(idt), _ptr(lt), _stream()))
            torch.cuda.current_stream().synchronize()


class _PinnedOwner:
    """Frees an rsb_host_alloc buffer once nothing references it (the ctypes array the CPU tensor is built on holds
    this object)."""

    def __init__(self, L, ptr: int, device):
        self.L, self.ptr, self.device = L, ptr, device

    def __del__(self):
        try:
            torch.cuda.current_stream(self.device).synchronize()     # no search in flight may still read it
            self.L.rsb_host_free(ctypes.c_void_p(self.ptr))
        except Exception:
            pass


def _pinned_rows(L, rows: int, d: int, dtype: torch.dtype, device) -> torch.Tensor:
    """A CPU tensor [rows, d] over page-locked, device-mapped host memory of exactly rows * d elements (rsb_host_alloc;
    torch's pinned allocator would round the block up to a power of two)."""
    nbytes = int(rows) * d * torch.empty((), dtype=dtype).element_size()
    if nbytes == 0:
        return torch.empty((0, d), dtype=dtype)
    p = ctypes.c_void_p(0)
    _lib.check(L.rsb_host_alloc(nbytes, ctypes.byref(p)))
    buf = (ctypes.c_char * nbytes).from_address(p.value)
    buf._owner = _PinnedOwner(L, p.value, device)
    return torch.frombuffer(buf, dtype=dtype).view(int(rows), d)


class IndexRefine:
    """faiss.IndexRefineFlat(base) / IndexRefine(base, IndexFlatIP(d)): the base IVF-PQ search returns k * k_factor
    candidates, which are re-scored exactly against a re-rank store of the original vectors (row = index id), and the
    best k are kept (rsb_search_refine).  Only IVF-PQ bases are accepted: Flat / IVF-Flat scores are already exact.

    The store is a device tensor [ntotal, d] in float16 or float32.  The embedding task writes fp16 embeddings, so an
    fp16 store of them is lossless; an fp16 store of fp32 vectors rounds them (faiss `Refine(SQfp16)`).
    Results are sorted by exact score descending, ties by ascending id, padded with (-FLT_MAX, -1).

    store_dtype = "sq8" keeps one uint8 code per element (faiss IndexRefine(base, IndexScalarQuantizer(d, QT_8bit)),
    `Refine(SQ8)`): half the bytes of fp16.  Its per-dimension range (vmin, vdiff) is trained by train(x) (base and
    quantizer, as faiss IndexRefine::train) or train_store(x) (quantizer only); add_store encodes fp16 / fp32 rows on the
    device.  Scores are exact fp32 inner products with the decoded rows vmin + ((c + 0.5f) / 255.f) * vdiff, bit-identical
    to a float32 store holding those rows.  d % 16 == 0.

    device_rows = n (an integer) makes the store tiered, for stores larger than device memory: rows [0, n) stay in
    device memory and rows from n on go to page-locked, device-mapped host memory.  Each search gathers the distinct
    host rows its candidates need over PCIe, `staging_bytes` of queries' worst case at a time; the results are
    bit-identical to an all-device store of the same values.  device_rows = None (default) keeps every row on the
    device."""

    staging_bytes = 512 << 20           # tiered store: device staging buffer for the host rows of a chunk of queries

    def __init__(self, base, store_dtype: str = "float16", k_factor: int = 1, device_rows: Optional[int] = None):
        if not isinstance(base, IndexIVFPQ):
            raise ValueError(f"IndexRefine re-ranks IVF-PQ results; a {type(base).__name__} base already returns exact scores")
        if store_dtype not in _REFINE_DTYPES:
            raise ValueError(f"store_dtype must be float16, float32 or sq8, got {store_dtype!r}")
        if store_dtype == "sq8" and base.d % 16:
            raise ValueError(f"an sq8 store needs d % 16 == 0 (whole 16-byte rows), got d = {base.d}")
        self.base, self.store_dtype = base, store_dtype
        self.k_factor = int(k_factor)
        self.device_rows = _check_device_rows(device_rows)
        self.L, self.d, self.device = base.L, base.d, base.device
        self._store = torch.empty((0, self.d), dtype=_REFINE_DTYPES[store_dtype][0], device=self.device)
        self._host = torch.empty((0, self.d), dtype=self._store.dtype)      # host tier (tiered store only)
        self._n = 0                                     # rows of the store in use (capacity = self._store.shape[0])
        self._sq: Optional[torch.Tensor] = None         # sq8: trained [2, d] float32 (vmin, vdiff) on the device

    @property
    def tiered(self) -> bool:
        return self.device_rows is not None

    @property
    def n_dev(self) -> int:
        """Rows of the store in device memory."""
        return min(self.device_rows, self._n) if self.tiered else self._n

    @property
    def device_store(self) -> torch.Tensor:
        """Rows [0, n_dev) (a device tensor view)."""
        return self._store[: self.n_dev]

    @property
    def host_store(self) -> torch.Tensor:
        """Rows [n_dev, ntotal) of a tiered store (a CPU tensor view over the pinned host tier)."""
        return self._host[: self._n - self.n_dev]

    def store_rows(self, ids) -> torch.Tensor:
        """The store rows of the given index ids [n] -> [n, d] device tensor, read from whichever tier holds them."""
        ids = torch.as_tensor(ids).to(device="cpu", dtype=torch.int64).reshape(-1)
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= self._n):
            raise IndexError(f"store ids must be in [0, {self._n})")
        out = torch.empty((ids.numel(), self.d), dtype=self._store.dtype, device=self.device)
        on_dev = ids < self.n_dev
        out[on_dev.to(self.device)] = self._store[ids[on_dev].to(self.device)]
        out[(~on_dev).to(self.device)] = self._host[ids[~on_dev] - self.n_dev].to(self.device)
        return out

    # -- faiss protocol ------------------------------------------------------------------------------------------
    @property
    def ntotal(self) -> int:
        return self.base.ntotal

    @property
    def is_trained(self) -> bool:
        return self.base.is_trained

    @property
    def nprobe(self) -> int:
        return self.base.nprobe

    @nprobe.setter
    def nprobe(self, v: int) -> None:
        self.base.nprobe = int(v)

    @property
    def store(self) -> torch.Tensor:
        """The re-rank store [ntotal, d] (a view; row i = the vector of index id i)."""
        if self.tiered:
            raise ValueError("a tiered store is not one tensor: use device_store, host_store or store_rows")
        return self._store[: self._n]

    def train(self, x) -> None:
        """Trains the base; an sq8 store also trains its quantizer on the same rows (faiss IndexRefine::train)."""
        self.base.train(x)
        if self.store_dtype == "sq8":
            self.train_store(x)

    def train_store(self, x) -> None:
        """sq8 only: trains the store's quantizer (per-dimension min and max of the rows x [n, d], fp16 or fp32), for a
        base that is already trained or read from disk.  Rows already in the store keep their codes."""
        if self.store_dtype != "sq8":
            raise ValueError(f"a {self.store_dtype} store has no quantizer to train")
        with torch.cuda.device(self.device):
            x = _dev_rows(x, self.device)
            if x.dim() != 2 or x.shape[1] != self.d or x.shape[0] == 0:
                raise ValueError(f"expected [n >= 1, {self.d}] training vectors, got {tuple(x.shape)}")
            sq = torch.empty((2, self.d), dtype=torch.float32, device=self.device)
            _lib.check(self.L.rsb_sq8_train(_ptr(x), _dtype_code(x), x.shape[0], self.d, _ptr(sq), _stream()))
            torch.cuda.current_stream(self.device).synchronize()     # x may be a temporary
            self._sq = sq

    @property
    def sq_params(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """sq8 only: the trained (vmin [d], vdiff [d]) float32 device tensors."""
        if self.store_dtype != "sq8":
            raise ValueError(f"a {self.store_dtype} store has no quantizer")
        if self._sq is None:
            raise ValueError("the sq8 quantizer is not trained: call train() or train_store() first")
        return self._sq[0], self._sq[1]

    def add(self, x, ids=None) -> None:
        """Adds to the base and appends to the store.  The store is addressed by index id, so ids are the base's
        sequential ids (as faiss IndexRefine requires)."""
        if ids is not None:
            raise ValueError("IndexRefine addresses its store by index id: add() takes no custom ids")
        if self._n != self.base.ntotal:
            raise ValueError(f"the store holds {self._n} rows but the base index {self.base.ntotal} vectors")
        self.base.add(x)
        self.add_store(x)

    def reserve(self, n: int) -> None:
        """Allocates store capacity for n rows, after checking that the device rows fit in free device memory (a tiered
        store puts rows past device_rows in pinned host memory)."""
        n_dev = int(n) if not self.tiered else min(int(n), self.device_rows)
        if n_dev > self._store.shape[0]:
            need = n_dev * self.d * self._store.element_size()
            free, _ = torch.cuda.mem_get_info(self.device)
            if need > free:
                raise MemoryError(f"the re-rank store needs {need} bytes ({n_dev} x {self.d} {self.store_dtype}); "
                                  f"{free} bytes are free on {self.device}")
            grown = torch.empty((n_dev, self.d), dtype=self._store.dtype, device=self.device)
            grown[: self.n_dev].copy_(self._store[: self.n_dev])
            self._store = grown
        n_host = int(n) - n_dev
        if n_host > self._host.shape[0]:
            grown = _pinned_rows(self.L, n_host, self.d, self._store.dtype, self.device)
            used = self._n - self.n_dev
            torch.cuda.current_stream(self.device).synchronize()    # a search in flight may read the old host tier
            grown[:used].copy_(self._host[:used])
            self._host = grown

    def _capacity(self) -> int:
        return self._store.shape[0] + self._host.shape[0]

    def add_store(self, x) -> None:
        """Appends rows to the store only (for a base that already holds these vectors, e.g. one read from disk).
        Rows bound for the host tier are copied there directly: host input never crosses PCIe for them.  An sq8 store
        encodes every row on the device (fp16 rows cross PCIe as fp16) and copies the host tier's codes into it."""
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x))
        x = torch.as_tensor(x)
        if x.dim() != 2 or x.shape[1] != self.d:
            raise ValueError(f"expected [n, {self.d}] vectors, got {tuple(x.shape)}")
        if self.store_dtype != "sq8":
            self._append(x)
            return
        self.sq_params                                              # ValueError before anything is stored
        step = max(1, (256 << 20) // (4 * self.d))
        with torch.cuda.device(self.device):
            for a in range(0, x.shape[0], step):
                xc = _dev_rows(x[a:a + step], self.device)
                codes = torch.empty(xc.shape, dtype=torch.uint8, device=self.device)
                _lib.check(self.L.rsb_sq8_encode(_ptr(xc), _dtype_code(xc), xc.shape[0], self.d, _ptr(self._sq),
                                                 _ptr(codes), _stream()))
                self._append(codes)

    def _append(self, x: torch.Tensor) -> None:
        """Appends rows already in the store's element type (or, for fp16 / fp32, convertible to it) to the tiers."""
        n = x.shape[0]
        if self._n + n > self._capacity():
            self.reserve(max(self._n + n, int(1.25 * self._capacity())))
        n_to_dev = n if not self.tiered else max(0, min(n, self.device_rows - self._n))
        if n_to_dev:
            self._store[self._n: self._n + n_to_dev].copy_(x[:n_to_dev].to(device=self.device, dtype=self._store.dtype))
        if n_to_dev < n:
            h0 = self._n + n_to_dev - self.device_rows
            torch.cuda.current_stream(self.device).synchronize()    # a search in flight may be reading the host tier
            self._host[h0: h0 + n - n_to_dev].copy_(x[n_to_dev:].to(dtype=self._store.dtype))
        self._n += n
        torch.cuda.current_stream(self.device).synchronize()     # x may be a temporary

    def _store_args(self):
        """(device tier, n_dev, host tier, store dtype code, SQ8 range) of rsb_refine / rsb_search_refine.  A store
        that is not tiered is all-device: n_dev = ntotal and an empty host tier."""
        if self.store_dtype == "sq8":
            self.sq_params                                          # ValueError if the quantizer is untrained
        return _ptr(self._store), self.n_dev, _ptr(self.host_store), _REFINE_DTYPES[self.store_dtype][1], _ptr(self._sq)

    def search_ids(self, q, k: int, nprobe: Optional[int] = None, k_factor: Optional[int] = None,
                   host_rows: Optional[torch.Tensor] = None):
        """q [nq, d] -> (ids int64 [nq,k], scores float32 [nq,k]) CUDA tensors, enqueued on the current stream.
        host_rows (tiered store; a 1-element int64 CUDA tensor) is incremented by the distinct host rows gathered."""
        with torch.cuda.device(self.device):
            q = _dev_f32(q, self.device)
            if q.dim() != 2 or q.shape[1] != self.d:
                raise ValueError(f"expected [nq, {self.d}] queries, got {tuple(q.shape)}")
            nq, k = q.shape[0], int(k)
            kf = int(self.k_factor if k_factor is None else k_factor)
            npb = int(self.nprobe if nprobe is None else nprobe)
            D = torch.empty((nq, k), dtype=torch.float32, device=self.device)
            I = torch.empty((nq, k), dtype=torch.int64, device=self.device)
            if nq == 0:
                return I, D
            dev, n_dev, host, dt, sq = self._store_args()
            sb = int(self.staging_bytes)
            ws = self.base._workspace(self.L.rsb_search_refine_workspace_bytes(self.base._h, nq, k, kf, npb, dt, n_dev,
                                                                               self._n, sb))
            _lib.check(self.L.rsb_search_refine(self.base._h, _ptr(q), nq, k, kf, npb, dev, n_dev, host, dt, sq, self._n,
                                                _ptr(D), _ptr(I), _ptr(ws), ws.numel(), sb, _ptr(host_rows), _stream()))
            return I, D

    def search(self, x, k: int):
        """faiss protocol: returns (D, I).  numpy in -> numpy out; torch in -> CUDA tensors out."""
        I, D = self.search_ids(x, k)
        if isinstance(x, np.ndarray) or not isinstance(x, torch.Tensor):
            return D.cpu().numpy(), I.cpu().numpy()
        return D, I

    def rerank(self, q: torch.Tensor, cand: torch.Tensor, k: int, staging_bytes: Optional[int] = None,
               host_rows: Optional[torch.Tensor] = None):
        """The re-rank step alone (rsb_refine): candidates cand [nq, k_base] int64 (-1 = none) -> (ids, scores)
        [nq, k].  staging_bytes and host_rows apply to a tiered store (see search_ids)."""
        with torch.cuda.device(self.device):
            q = _dev_f32(q, self.device)
            cand = cand.to(device=self.device, dtype=torch.int64).contiguous()
            nq, k_base = cand.shape
            D = torch.empty((nq, int(k)), dtype=torch.float32, device=self.device)
            I = torch.empty((nq, int(k)), dtype=torch.int64, device=self.device)
            dev, n_dev, host, dt, sq = self._store_args()
            sb = int(self.staging_bytes if staging_bytes is None else staging_bytes)
            ws = self.base._workspace(self.L.rsb_refine_workspace_bytes(nq, k_base, int(k), self.d, dt, n_dev, self._n, sb))
            _lib.check(self.L.rsb_refine(_ptr(q), nq, dev, n_dev, host, dt, sq, self.d, self._n, _ptr(cand), k_base,
                                         int(k), _ptr(D), _ptr(I), _ptr(ws), ws.numel(), sb, _ptr(host_rows), _stream()))
            return I, D


# ------------------------------------------------------------------------------------------------------------
# persistence: same call sites as faiss.write_index / faiss.read_index (flat.py:39,63; ivf_flat.py:71,167,185;
# ivf_pq.py:75,171,190).  Files are written in faiss' binary layout (faiss_io.py: IxFI / IwFl / IwPQ), because the
# reference's artefact names (`index_*.faiss`) promise exactly that to any faiss / reference process pointed at the
# same index_dir.  `RSB_INDEX_FORMAT=rsb1` (or fmt="rsb1") selects our own container instead (a pickle of numpy
# arrays in natural CSR order, which also holds what faiss' IndexFlatIP cannot: non-sequential ids).  The reader
# auto-detects both.  NOTE the faiss layout is restated from the published source and could not be checked against a
# real faiss build offline (tests/test_faiss_io.py cross-checks it wherever faiss is importable).
# ------------------------------------------------------------------------------------------------------------
MAGIC = "RSB1"


def _to_faiss_parts(index: _IndexBase) -> dict:
    if isinstance(index, IndexRefine):
        rows = torch.cat([index.device_store.cpu(), index.host_store])
        if index.store_dtype == "sq8":      # faiss IndexRefine with an IndexScalarQuantizer(QT_8bit) refine index
            return {"kind": "Refine", "d": index.d, "ntotal": index.ntotal, "base": _to_faiss_parts(index.base),
                    "sq": torch.stack(index.sq_params).cpu().numpy(), "codes": rows.numpy(),
                    "k_factor": float(index.k_factor)}
        # faiss IndexRefineFlat: an fp16 store is written upcast to fp32 (exact)
        xb = rows.float()
        return {"kind": "Refine", "d": index.d, "ntotal": index.ntotal, "base": _to_faiss_parts(index.base),
                "xb": xb.numpy(), "k_factor": float(index.k_factor)}
    off, payload, ids = index.export_lists()
    off, payload, ids = off.cpu().numpy(), payload.cpu().numpy(), ids.cpu().numpy()
    # fp16 storage is written upcast to fp32 (exact): the file is the one the fp32 index of the same values writes
    payload = payload.astype(np.float32) if payload.dtype == np.float16 else payload
    if index.kind == _lib.RSB_FLAT:
        if not np.array_equal(ids, np.arange(len(ids))):
            raise ValueError("faiss IndexFlatIP has no id map: only sequential ids can be written in faiss format")
        return {"kind": "Flat", "xb": payload, "metric": 0}
    parts = {"centroids": index.get_centroids().cpu().numpy(), "offsets": off, "ids": ids, "nprobe": int(index.nprobe)}
    if isinstance(index, IndexIVFScalarQuantizer):
        return {"kind": "IVFSQ", "codes": payload, "sq": torch.stack(index.sq_params).cpu().numpy(),
                "by_residual": index.by_residual, **parts}
    if index.kind == _lib.RSB_IVFFLAT:
        return {"kind": "IVFFlat", "vectors": payload, **parts}
    return {"kind": "IVFPQ", "codes": payload, "codebook": index.get_codebook().cpu().numpy(), **parts}


def _check_sq8_storage(file_is_sq8: bool, storage_dtype: Optional[str]) -> None:
    """storage_dtype "sq8" reads SQ8 files only, and an SQ8 file reads as sq8 only: turning float vectors into codes (or
    back) would need a trained range, which reading does not do."""
    if file_is_sq8 and storage_dtype not in (None, "sq8"):
        raise ValueError(f"the index holds 8-bit scalar-quantizer codes (IVF-SQ8): its storage is sq8, not {storage_dtype}")
    if not file_is_sq8 and storage_dtype == "sq8":
        raise ValueError("storage_dtype sq8 reads IVF-SQ8 indexes only; this index holds float vectors (converting it "
                         "would need a trained scalar quantizer: build an IndexIVFScalarQuantizer instead)")


def _from_faiss_parts(p: dict, device=None, refine_dtype: Optional[str] = None,
                      storage_dtype: Optional[str] = None) -> _IndexBase:
    if p.get("metric", 0) != 0 or p.get("quantizer_metric", 0) != 0:
        raise NotImplementedError("only METRIC_INNER_PRODUCT indexes are supported (the reference builds IP indexes only)")
    if p["kind"] == "IVFSQ" or storage_dtype == "sq8":
        _check_sq8_storage(p["kind"] == "IVFSQ", storage_dtype)
    elif storage_dtype is not None:
        _check_dtype(storage_dtype, "storage_dtype")
        if p["kind"] not in ("Flat", "IVFFlat"):
            raise ValueError(f"storage_dtype applies to Flat and IVFFlat indexes, not {p['kind']}")
    if p["kind"] == "Refine":
        kf = float(p["k_factor"])
        if kf != int(kf) or kf < 1:
            raise NotImplementedError(f"k_factor = {kf}: only whole k_factor >= 1 is supported")
        if "codes" in p:                   # IxSQ QT_8bit refine index: the codes and the trained range load as they are
            if refine_dtype not in (None, "sq8"):
                raise ValueError(f"the refine index is an 8-bit scalar quantizer (IxSQ): its store is sq8, not {refine_dtype}")
            index = IndexRefine(_from_faiss_parts(p["base"], device), store_dtype="sq8", k_factor=int(kf))
            if index.ntotal != p["codes"].shape[0]:
                raise ValueError(f"refine index holds {p['codes'].shape[0]} vectors, its base {index.ntotal}")
            index._sq = torch.from_numpy(np.ascontiguousarray(p["sq"], dtype=np.float32)).to(index.device)
            index.reserve(p["codes"].shape[0])
            index._append(torch.from_numpy(np.ascontiguousarray(p["codes"])))
            return index
        if refine_dtype == "sq8":
            raise ValueError("the refine index holds float vectors (IxFI): read it with refine_dtype float32 or float16")
        xb = p["xb"]
        dtype = refine_dtype or "float32"
        if dtype == "float16":
            xh = xb.astype(np.float16)
            if not np.array_equal(xh.astype(np.float32), xb):
                raise ValueError("the refine vectors are not all representable in float16; read with refine_dtype='float32'")
            xb = xh
        index = IndexRefine(_from_faiss_parts(p["base"], device), store_dtype=dtype, k_factor=int(kf))
        if index.ntotal != xb.shape[0]:
            raise ValueError(f"refine index holds {xb.shape[0]} vectors, its base {index.ntotal}")
        index.reserve(xb.shape[0])
        index.add_store(xb)
        return index
    dtype = storage_dtype or "float32"
    if p["kind"] == "Flat":
        xb = _as_storage(p["xb"], dtype, "the Flat index's vectors") if p["ntotal"] else None
        index = IndexFlatIP(p["d"], device, dtype=dtype)
        if p["ntotal"]:
            index.add(xb)
        return index
    nlist = p["nlist"]
    lists = np.repeat(np.arange(nlist, dtype=np.int32), np.diff(p["offsets"]))
    if p["kind"] == "IVFSQ":         # codes and range load as stored
        index = IndexIVFScalarQuantizer(p["d"], nlist, by_residual=bool(p["by_residual"]), device=device)
        index.set_centroids(p["centroids"])
        index.sq_params = p["sq"]
        if len(p["ids"]):
            index.add_codes(p["codes"], lists, p["ids"])
    elif p["kind"] == "IVFFlat":
        xb = _as_storage(p["vectors"], dtype, "the IVFFlat index's vectors") if len(p["ids"]) else None
        index = IndexIVFFlat(p["d"], nlist, device, dtype=dtype)
        index.set_centroids(p["centroids"])
        if len(p["ids"]):
            index.add_preassigned(xb, lists, p["ids"])
    else:
        if not p.get("by_residual", True):
            raise NotImplementedError("IVFPQ without by_residual")
        index = IndexIVFPQ(p["d"], nlist, int(p["M"]), int(p["nbits"]), device)
        index.set_centroids(p["centroids"])
        index.set_codebook(p["codebook"])
        if len(p["ids"]):
            index.add_codes(p["codes"], lists, p["ids"])
    index.nprobe = int(p.get("nprobe", 1))
    index.finalize()
    return index


_ROW_CHUNK_BYTES = 64 << 20     # tiered Flat persistence: rows moved per step between the tiers and the file


def _write_flat_tiered(index: "IndexFlatIP", path: str, fmt: str) -> None:
    """A tiered Flat index written in row ranges (rsb_export_rows): the same bytes as the all-device index of the same
    rows, with host memory bounded by one chunk (faiss) beyond the tiers."""
    from . import faiss_io
    n, d = index.ntotal, index.d
    step = max(1, _ROW_CHUNK_BYTES // (4 * d))
    ids = index.export_ids()
    if fmt == "faiss" and not torch.equal(ids, torch.arange(n, dtype=torch.int64, device=ids.device)):
        import warnings
        warnings.warn(f"{path}: faiss IndexFlatIP has no id map: only sequential ids can be written in faiss format; "
                      f"writing the RSB1 container instead")
        fmt = "rsb1"
    tmp = path + ".tmp"
    if fmt == "faiss":       # fp16 rows upcast to fp32 (exact), as _to_faiss_parts writes them
        chunks = (index.export_rows(r0, min(step, n - r0)).float().numpy() for r0 in range(0, n, step))
        with open(tmp, "wb") as f:
            faiss_io.write_flat_rows(f, d, n, chunks)
    else:
        blob = {"magic": MAGIC, "kind": int(index.kind), "d": d, "nprobe": int(index.nprobe), "dtype": index.dtype}
        if n > 0:
            payload = np.empty((n, d), dtype=np.float16)
            index.export_rows(0, n, out=torch.from_numpy(payload))
            blob["offsets"] = np.array([0, n], dtype=np.int64)
            blob["payload"] = payload
            blob["ids"] = ids.cpu().numpy()
        with open(tmp, "wb") as f:
            pickle.dump(blob, f, protocol=4)
    os.replace(tmp, path)


def _read_flat_tiered(path: str, device, storage_dtype: Optional[str], device_rows: int) -> "IndexFlatIP":
    """A Flat index file (IxFI or RSB1) into a tiered IndexFlatIP, filled a chunk at a time from a memory map of the
    faiss payload (RSB1: from the unpickled payload)."""
    from . import faiss_io
    if storage_dtype != "float16":
        raise ValueError(f"device_rows (a tiered Flat index) needs storage_dtype='float16', got {storage_dtype!r}")
    ids = None
    if faiss_io.is_faiss_file(path):
        d, n, rows = faiss_io.flat_rows_memmap(path)
    else:
        with open(path, "rb") as f:
            blob = pickle.load(f)
        if not isinstance(blob, dict) or blob.get("magic") != MAGIC:
            raise ValueError(f"{path} is not an RSB1 index file")
        if blob["kind"] != _lib.RSB_FLAT:
            raise ValueError("device_rows applies to Flat indexes only")
        d = blob["d"]
        rows = blob.get("payload", np.zeros((0, d), np.float16))
        ids = blob.get("ids")
        n = rows.shape[0]
    index = IndexFlatIP(d, device, dtype="float16", device_rows=device_rows)
    step = max(1, _ROW_CHUNK_BYTES // (4 * d))
    for r0 in range(0, n, step):
        chunk = _as_storage(np.asarray(rows[r0:r0 + step]), "float16", f"{path}: the Flat index's vectors")
        index.add(chunk, None if ids is None else ids[r0:r0 + step])
    index.finalize()
    return index


def _write_ivf_tiered(index: "_IVFBase", path: str, fmt: str) -> None:
    """A tiered IVF-Flat / IVF-SQ8 index written list range by list range (rsb_export_rows): the bytes the all-device
    index of the same lists writes (fp16 rows upcast to fp32 a range at a time), with host memory bounded by the ids and
    one range beyond the tiers."""
    from . import faiss_io
    if fmt != "faiss":
        raise NotImplementedError("a tiered IVF index (list_device_rows) is written in the faiss format (IwFl / IwSq) "
                                  "only, not the RSB1 container")
    sizes = index.list_sizes().cpu().numpy()
    off = np.zeros(index.nlist + 1, dtype=np.int64)
    np.cumsum(sizes, out=off[1:])
    ids = index.export_ids_host() if off[-1] else np.zeros(0, np.int64)
    parts = {"centroids": index.get_centroids().cpu().numpy(), "nprobe": int(index.nprobe)}
    if isinstance(index, IndexIVFScalarQuantizer):
        parts.update(kind="IVFSQ", sq=torch.stack(index.sq_params).cpu().numpy(), by_residual=index.by_residual)
    else:
        parts.update(kind="IVFFlat")

    def rows(r0: int, r1: int) -> np.ndarray:
        x = index.export_rows(r0, r1 - r0).numpy()
        return x.astype(np.float32) if x.dtype == np.float16 else x

    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        faiss_io.write_ivf_streamed(f, parts, off, ids, rows, _ROW_CHUNK_BYTES // (4 * index.d))
    os.replace(tmp, path)


def _read_ivf_tiered(path: str, device, storage_dtype: Optional[str], list_device_rows: int,
                     staging_bytes: Optional[int] = None) -> "_IVFBase":
    """An IwFl / IwSq file into a tiered index: the list sizes are read first and reserved, then the lists are added
    a range at a time from a memory map of the payload, with their ids and within-list order."""
    from . import faiss_io
    if not faiss_io.is_faiss_file(path):
        raise NotImplementedError("list_device_rows reads IVF-Flat / IVF-SQ8 indexes in the faiss format (IwFl / IwSq); "
                                  "an RSB1 container cannot be read into a tiered index")
    meta, off, read_lists = faiss_io.ivf_lists_memmap(path)
    if meta["metric"] != 0 or meta.get("quantizer_metric", 0) != 0:
        raise NotImplementedError("only METRIC_INNER_PRODUCT indexes are supported (the reference builds IP indexes only)")
    nlist, d = meta["nlist"], meta["d"]
    if meta["kind"] == "IVFSQ":
        _check_sq8_storage(True, storage_dtype)
        index = IndexIVFScalarQuantizer(d, nlist, by_residual=bool(meta["by_residual"]), device=device,
                                        list_device_rows=list_device_rows, staging_bytes=staging_bytes)
        index.set_centroids(meta["centroids"])
        index.sq_params = meta["sq"]
    else:
        _check_sq8_storage(False, storage_dtype)
        dtype = _check_dtype(storage_dtype or "float32", "storage_dtype")
        index = IndexIVFFlat(d, nlist, device, dtype=dtype, list_device_rows=list_device_rows,
                             staging_bytes=staging_bytes)
        index.set_centroids(meta["centroids"])
    index.nprobe = int(meta.get("nprobe", 1))
    sizes = np.diff(off)
    if off[-1] == 0:                 # nothing to place: the index stays unreserved, as a freshly trained one
        return index
    index.reserve_lists(sizes)
    step = max(1, _ROW_CHUNK_BYTES // (4 * d))
    l0 = 0
    while l0 < nlist:                # list ranges of about `step` rows (one list when a list is longer)
        l1 = int(np.searchsorted(off, off[l0] + step, side="right")) - 1
        l1 = min(nlist, max(l1, l0 + 1))
        if off[l1] > off[l0]:
            codes, ids = read_lists(l0, l1)
            lists = np.repeat(np.arange(l0, l1, dtype=np.int32), sizes[l0:l1])
            if meta["kind"] == "IVFSQ":
                index.add_codes(codes, lists, ids)
            else:
                xb = _as_storage(codes.view(np.float32).reshape(-1, d), index.dtype, f"{path}: the IVFFlat index's vectors")
                index.add_preassigned(xb, lists, ids)
        l0 = l1
    return index


def write_index(index: _IndexBase, path: str, fmt: Optional[str] = None) -> None:
    """fmt "faiss" (default; env RSB_INDEX_FORMAT overrides: faiss 1.8 binary layout, see faiss_io.py) or "rsb1"."""
    fmt = (fmt or os.environ.get("RSB_INDEX_FORMAT", "faiss")).lower()
    if fmt not in ("faiss", "rsb1"):
        raise ValueError(f"unknown index file format {fmt!r} (faiss | rsb1)")
    if isinstance(index, IndexFlatIP) and index.tiered:
        return _write_flat_tiered(index, path, fmt)
    if isinstance(index, _IVFBase) and index.tiered:
        return _write_ivf_tiered(index, path, fmt)
    if isinstance(index, IndexRefine) and fmt != "faiss":
        raise ValueError("an IndexRefine is written in faiss' IndexRefineFlat layout only (fmt='faiss')")
    if fmt == "faiss":
        from . import faiss_io
        try:
            parts = _to_faiss_parts(index)
        except ValueError as e:      # e.g. a Flat index with caller-chosen ids: faiss' IndexFlatIP cannot express it
            import warnings
            warnings.warn(f"{path}: {e}; writing the RSB1 container instead")
            parts = None
        if parts is not None:
            tmp = path + ".tmp"
            faiss_io.write_faiss(tmp, parts)
            os.replace(tmp, path)
            return
    blob = {"magic": MAGIC, "kind": int(index.kind), "d": index.d, "nprobe": int(index.nprobe)}
    if index.dtype != "float32":
        blob["dtype"] = index.dtype                      # the payload below is kept as stored
    if isinstance(index, IndexIVFScalarQuantizer):
        blob["by_residual"] = index.by_residual
        try:
            blob["sq"] = torch.stack(index.sq_params).cpu().numpy()
        except _lib.RsbError:
            pass
    if isinstance(index, _IVFBase):
        blob["nlist"] = index.nlist
        try:
            blob["centroids"] = index.get_centroids().cpu().numpy()
        except _lib.RsbError:
            pass
        if isinstance(index, IndexIVFPQ):
            blob["M"], blob["nbits"] = index.M, index.nbits
            try:
                blob["codebook"] = index.get_codebook().cpu().numpy()
            except _lib.RsbError:
                pass
    if index.ntotal > 0:
        off, payload, ids = index.export_lists()
        blob["offsets"] = off.cpu().numpy()
        blob["payload"] = payload.cpu().numpy()
        blob["ids"] = ids.cpu().numpy()
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        pickle.dump(blob, f, protocol=4)
    os.replace(tmp, path)


def read_index(path: str, device=None, refine_dtype: Optional[str] = None,
               storage_dtype: Optional[str] = None, device_rows: Optional[int] = None,
               list_device_rows: Optional[int] = None) -> _IndexBase:
    """Loads an RSB1 container or a faiss binary index file (auto-detected by its fourcc).  For an IndexRefineFlat
    file (IxRF) `refine_dtype` picks the store: "float32" (default) or "float16", which is accepted only when every
    stored value round-trips through fp16 (ValueError otherwise).  An IxRF file whose refine index is an 8-bit scalar
    quantizer (IxSQ, QT_8bit) loads as an sq8 store (refine_dtype None or "sq8"; float16 / float32 raise ValueError).  `storage_dtype` does the same for the vectors of a
    Flat / IVFFlat index (IxFI / IwFl / RSB1); None keeps the file's dtype (fp32 for faiss files).  An IVF-SQ8 index
    (IwSq / IwSQ, or RSB1 with dtype sq8) loads as an IndexIVFScalarQuantizer with its codes and range as stored
    (storage_dtype None or "sq8"); "sq8" on a float index and float16 / float32 on an SQ8 index raise ValueError.
    device_rows = n loads a Flat index (IxFI or RSB1) as a tiered IndexFlatIP (storage_dtype "float16" only, else
    ValueError), filling the tiers a chunk at a time from a memory map of the faiss payload.
    list_device_rows = R loads an IVF-Flat or IVF-SQ8 index (IwFl / IwSq) as a tiered index (see IndexIVFFlat): the list
    sizes are reserved first, then the lists are filled from a memory map of the payload; RSB1 files raise
    NotImplementedError."""
    from . import faiss_io
    device_rows = _check_device_rows(device_rows)
    list_device_rows = _check_rows_arg(list_device_rows, "list_device_rows")
    if list_device_rows is not None:
        if device_rows is not None:
            raise ValueError("device_rows tiers a Flat index, list_device_rows an IVF index: give one of them")
        return _read_ivf_tiered(path, device, storage_dtype, list_device_rows)
    if device_rows is not None:
        return _read_flat_tiered(path, device, storage_dtype, device_rows)
    if faiss_io.is_faiss_file(path):
        return _from_faiss_parts(faiss_io.read_faiss(path), device, refine_dtype, storage_dtype)
    with open(path, "rb") as f:
        blob = pickle.load(f)
    if not isinstance(blob, dict) or blob.get("magic") != MAGIC:
        raise ValueError(f"{path} is not an RSB1 index file")
    kind = blob["kind"]
    if blob.get("dtype") == "sq8" or storage_dtype == "sq8":
        _check_sq8_storage(blob.get("dtype") == "sq8", storage_dtype)
    elif storage_dtype is not None:
        _check_dtype(storage_dtype, "storage_dtype")
        if kind not in (_lib.RSB_FLAT, _lib.RSB_IVFFLAT):
            raise ValueError("storage_dtype applies to Flat and IVFFlat indexes only")
    dtype = storage_dtype or blob.get("dtype", "float32")
    if "payload" in blob and kind != _lib.RSB_IVFPQ:
        blob["payload"] = _as_storage(blob["payload"], dtype, f"{path}: the index vectors")
    if kind == _lib.RSB_FLAT:
        index = IndexFlatIP(blob["d"], device, dtype=dtype)
    elif kind == _lib.RSB_IVFFLAT and dtype == "sq8":
        index = IndexIVFScalarQuantizer(blob["d"], blob["nlist"], by_residual=bool(blob["by_residual"]), device=device)
    elif kind == _lib.RSB_IVFFLAT:
        index = IndexIVFFlat(blob["d"], blob["nlist"], device, dtype=dtype)
    elif kind == _lib.RSB_IVFPQ:
        index = IndexIVFPQ(blob["d"], blob["nlist"], blob["M"], blob["nbits"], device)
    else:
        raise ValueError(f"unknown index kind {kind}")
    index.nprobe = blob.get("nprobe", 1)
    if "centroids" in blob:
        index.set_centroids(blob["centroids"])
    if "codebook" in blob:
        index.set_codebook(blob["codebook"])
    if "sq" in blob:
        index.sq_params = blob["sq"]
    if "payload" in blob:
        ids = blob["ids"]
        if kind == _lib.RSB_FLAT:
            index.add(blob["payload"], ids)
        else:
            off = blob["offsets"]
            lists = np.repeat(np.arange(len(off) - 1, dtype=np.int32), np.diff(off))
            if kind == _lib.RSB_IVFPQ or dtype == "sq8":
                index.add_codes(blob["payload"], lists, ids)
            else:
                index.add_preassigned(blob["payload"], lists, ids)
        index.finalize()
    return index


def merge_topk(D_all: torch.Tensor, I_all: torch.Tensor, k_out: Optional[int] = None):
    """Shard merge on the GPU (reference src/search.py:357-367): D_all/I_all [nshards, nq, k] CUDA tensors."""
    _require_cuda()
    L = _lib.lib()
    nshards, nq, k = D_all.shape
    k_out = k if k_out is None else int(k_out)
    D_all = D_all.contiguous().float()
    I_all = I_all.contiguous().long()
    D = torch.empty((nq, k_out), dtype=torch.float32, device=D_all.device)
    I = torch.empty((nq, k_out), dtype=torch.int64, device=D_all.device)
    with torch.cuda.device(D_all.device):
        _lib.check(L.rsb_merge_topk(_ptr(D_all), _ptr(I_all), nshards, nq, k, k_out, _ptr(D), _ptr(I), _stream()))
    return D, I


def knn_ip(q: torch.Tensor, x: torch.Tensor, k: int, id_offset: int = 0):
    """Exact inner-product k-NN of q [nq,d] against x [n,d] (both CUDA float32) -> (D, I)."""
    _require_cuda()
    L = _lib.lib()
    q = q.contiguous().float()
    x = x.contiguous().float()
    nq, d = q.shape
    n = x.shape[0]
    D = torch.empty((nq, k), dtype=torch.float32, device=q.device)
    I = torch.empty((nq, k), dtype=torch.int64, device=q.device)
    with torch.cuda.device(q.device):
        ws = torch.empty(max(256, L.rsb_knn_workspace_bytes(nq, n, k)), dtype=torch.uint8, device=q.device)
        _lib.check(L.rsb_knn_ip(_ptr(q), nq, _ptr(x), n, d, k, id_offset, _ptr(D), _ptr(I), _ptr(ws), ws.numel(), _stream()))
    return D, I
