"""Reader / writer for the faiss binary index format (SURVEY.md §8f-3) for the three index classes the reference
persists with `faiss.write_index` / loads with `faiss.read_index` (`src/indicies/flat.py:39,63`,
`ivf_flat.py:71,167,185`, `ivf_pq.py:75,171,190`):

    "IxFI"  IndexFlatIP            "IwFl"  IndexIVFFlat (quantizer IndexFlatIP)      "IwPQ"  IndexIVFPQ (by_residual)
    "IwSq"  IndexIVFScalarQuantizer (QT_8bit; index_factory "IVFn,SQ8"), also read in its older "IwSQ" form
    "IxRF"  IndexRefineFlat (IVF-PQ base + exact re-rank vectors; faiss IndexRefine with an IndexFlat refine index), or
            IndexRefine with an "IxSQ" IndexScalarQuantizer refine index of qtype QT_8bit (`Refine(SQ8)`)

[FAISS-ext] faiss is not installable in this image, so this module restates the on-disk layout of faiss 1.8.0
(`faiss/impl/index_write.cpp`, `index_read.cpp`) from the published source and is pinned only by byte-level
known-answer tests (`tests/test_faiss_io.py`) and round trips -- it has NOT been cross-checked against a real
faiss build.  Layout (little endian):

  index header   : fourcc u32 | d i32 | ntotal i64 | dummy i64 (1<<20) | dummy i64 (1<<20) | is_trained u8 | metric i32
                   (metric 0 = INNER_PRODUCT, 1 = L2; metric > 1 is followed by metric_arg f32)
  IxFI / IxF2    : header | n_floats u64 | float32[n_floats]                       (codes stored as xb vector: size/4)
  ivf header     : header | nlist u64 | nprobe u64 | <quantizer index> | direct-map type u8 | direct-map array (u64 n | i64[n])
  IwFl           : ivf header | inverted lists              (code_size is NOT stored: read_index sets it to d * 4)
  IwPQ           : ivf header | by_residual u8 | code_size u64 | PQ: d u64 | M u64 | nbits u64 | (u64 n | float32[n]) | inverted lists
  inverted lists : "ilar" | nlist u64 | code_size u64 | "full" (u64 n | u64 sizes[n])  or  "sprs" (u64 n | u64 (list, size) pairs)
                   then, for every list in order: codes u8[size * code_size] | ids i64[size]
  IxRF           : header | <base index> | <refine index, IxFI or IxSQ> | k_factor f32
                   (index_write.cpp: IndexRefine branch; index_read.cpp turns a flat refine index into IndexRefineFlat)
  IxSQ           : header | qtype i32 | rangestat i32 | rangestat_arg f32 | d u64 | code_size u64
                   | trained (u64 n | float32[n]) | codes (u64 n | u8[n])
                   (write_ScalarQuantizer + the codes vector; only qtype QT_8bit = 0 is supported, whose trained vector
                   is [2, d] = vmin then vdiff and code_size = d; rangestat only steers training and is written as
                   RS_minmax = 0)
  IwSq           : ivf header | ScalarQuantizer: qtype i32 | rangestat i32 | rangestat_arg f32 | d u64 | code_size u64
                   | trained (u64 n | float32[n]) | code_size u64 | by_residual u8 | inverted lists (code_size = d)
                   (index_write.cpp: write_ScalarQuantizer has no codes vector, unlike IxSQ; the codes live in the lists.
                   index_read.cpp reads "IwSQ" the same way without the by_residual byte, and sets by_residual = true)
"""
from __future__ import annotations

import struct
from typing import BinaryIO, Dict

import numpy as np

METRIC_INNER_PRODUCT, METRIC_L2 = 0, 1
QT_8BIT, RS_MINMAX = 0, 0


def fourcc(s: str) -> int:
    b = s.encode("ascii")
    return b[0] | (b[1] << 8) | (b[2] << 16) | (b[3] << 24)


def _fourcc_str(v: int) -> str:
    return bytes([v & 255, (v >> 8) & 255, (v >> 16) & 255, (v >> 24) & 255]).decode("ascii", "replace")


# ----------------------------------------------------------------------------------------------------------
# reading
# ----------------------------------------------------------------------------------------------------------
def _rd(f: BinaryIO, fmt: str):
    size = struct.calcsize("<" + fmt)
    buf = f.read(size)
    if len(buf) != size:
        raise ValueError("unexpected end of faiss index file")
    out = struct.unpack("<" + fmt, buf)
    return out[0] if len(out) == 1 else out


def _rd_array(f: BinaryIO, dtype, n: int) -> np.ndarray:
    a = np.frombuffer(f.read(n * np.dtype(dtype).itemsize), dtype=dtype)
    if a.shape[0] != n:
        raise ValueError("unexpected end of faiss index file")
    return a


def _read_header(f: BinaryIO) -> Dict:
    d = _rd(f, "i")
    ntotal = _rd(f, "q")
    _rd(f, "q"); _rd(f, "q")
    is_trained = bool(_rd(f, "B"))
    metric = _rd(f, "i")
    if metric > 1:
        _rd(f, "f")
    return {"d": d, "ntotal": ntotal, "is_trained": is_trained, "metric": metric}


def _read_flat(f: BinaryIO, hdr: Dict) -> Dict:
    n = _rd(f, "Q")
    xb = _rd_array(f, np.float32, n)
    if n != hdr["ntotal"] * hdr["d"]:
        raise ValueError(f"flat index payload has {n} floats, expected {hdr['ntotal']} x {hdr['d']}")
    return {"kind": "Flat", **hdr, "xb": xb.reshape(hdr["ntotal"], hdr["d"])}


def _read_scalar_quantizer(f: BinaryIO, d_expected: int) -> np.ndarray:
    """read_ScalarQuantizer of a QT_8bit quantizer -> its trained range [2, d] (vmin, vdiff)."""
    qtype, _rangestat, _rangestat_arg = _rd(f, "i"), _rd(f, "i"), _rd(f, "f")
    d, code_size = _rd(f, "Q"), _rd(f, "Q")
    trained = _rd_array(f, np.float32, _rd(f, "Q"))
    if qtype != QT_8BIT:
        raise NotImplementedError(f"ScalarQuantizer qtype {qtype}: only QT_8bit (0) is supported")
    if d != d_expected or code_size != d or trained.size != 2 * d:
        raise ValueError("ScalarQuantizer: d, code_size or trained disagree with the index header")
    return trained.reshape(2, d)


def _read_sq(f: BinaryIO, hdr: Dict) -> Dict:
    qtype, rangestat, rangestat_arg = _rd(f, "i"), _rd(f, "i"), _rd(f, "f")
    d, code_size = _rd(f, "Q"), _rd(f, "Q")
    trained = _rd_array(f, np.float32, _rd(f, "Q"))
    codes = _rd_array(f, np.uint8, _rd(f, "Q"))
    if qtype != QT_8BIT:
        raise NotImplementedError(f"IndexScalarQuantizer qtype {qtype}: only QT_8bit (0) is supported")
    if d != hdr["d"] or code_size != d or trained.size != 2 * d or codes.size != hdr["ntotal"] * d:
        raise ValueError("IndexScalarQuantizer: d, code_size, trained or codes disagree with the header")
    return {"kind": "SQ", **hdr, "rangestat": rangestat, "rangestat_arg": rangestat_arg,
            "sq": trained.reshape(2, d), "codes": codes.reshape(hdr["ntotal"], d)}


def _read_invlists(f: BinaryIO, nlist_expected: int, tag_bytes: bytes = None):
    tag = tag_bytes.decode("ascii", "replace") if tag_bytes is not None else _fourcc_str(_rd(f, "I"))
    if tag == "il00":
        raise NotImplementedError("index written without inverted lists")
    if tag != "ilar":
        raise NotImplementedError(f"inverted-list container {tag!r} is not supported (only ArrayInvertedLists 'ilar')")
    nlist = _rd(f, "Q")
    code_size = _rd(f, "Q")
    if nlist != nlist_expected:
        raise ValueError("inverted lists disagree with the IVF header on nlist")
    ltype = _fourcc_str(_rd(f, "I"))
    sizes = np.zeros(nlist, dtype=np.int64)
    if ltype == "full":
        n = _rd(f, "Q")
        sizes[:] = _rd_array(f, np.uint64, n).astype(np.int64)
    elif ltype == "sprs":
        n = _rd(f, "Q")
        pairs = _rd_array(f, np.uint64, n).astype(np.int64).reshape(-1, 2)
        sizes[pairs[:, 0]] = pairs[:, 1]
    else:
        raise NotImplementedError(f"inverted-list size encoding {ltype!r}")
    total = int(sizes.sum())
    codes = np.empty((total, code_size), dtype=np.uint8)
    ids = np.empty(total, dtype=np.int64)
    pos = 0
    for l in range(nlist):
        s = int(sizes[l])
        if s:
            codes[pos:pos + s] = _rd_array(f, np.uint8, s * code_size).reshape(s, code_size)
            ids[pos:pos + s] = _rd_array(f, np.int64, s)
            pos += s
    offsets = np.zeros(nlist + 1, dtype=np.int64)
    np.cumsum(sizes, out=offsets[1:])
    return code_size, offsets, codes, ids


def ivf_lists_memmap(path: str):
    """An IwFl / IwSq file without its payload: (meta, offsets [nlist + 1], read_lists), where meta holds the parts of
    read_faiss except the codes / vectors and ids, and read_lists(l0, l1) -> (codes uint8 [rows, code_size], ids int64
    [rows]) of lists [l0, l1), read from a memory map of the file: an index larger than host memory is loaded list
    range by list range."""
    with open(path, "rb") as f:
        tag = _fourcc_str(_rd(f, "I"))
        if tag not in ("IwFl", "IwSq", "IwSQ"):
            raise ValueError(f"{path} is not a faiss IVF-Flat (IwFl) or IVF-SQ8 (IwSq) file, it is {tag!r}")
        h = _read_ivf_header(f)
        if tag == "IwFl":
            peek = f.read(4)
            if peek not in (b"ilar", b"il00"):           # the redundant code_size of early files (see read_faiss)
                f.read(4)
            else:
                f.seek(-4, 1)
            meta, code_size = {"kind": "IVFFlat", **h}, h["d"] * 4
        else:
            sq = _read_scalar_quantizer(f, h["d"])
            code_size = _rd(f, "Q")
            by_residual = bool(_rd(f, "B")) if tag == "IwSq" else True
            meta = {"kind": "IVFSQ", **h, "by_residual": by_residual, "sq": sq}
        tag = _fourcc_str(_rd(f, "I"))
        if tag != "ilar":
            raise NotImplementedError(f"inverted-list container {tag!r} is not supported (only ArrayInvertedLists 'ilar')")
        nlist, cs = _rd(f, "Q"), _rd(f, "Q")
        if nlist != h["nlist"] or cs != code_size:
            raise ValueError("inverted lists disagree with the IVF header on nlist or code_size")
        ltype = _fourcc_str(_rd(f, "I"))
        sizes = np.zeros(nlist, dtype=np.int64)
        n = _rd(f, "Q")
        if ltype == "full":
            sizes[:] = _rd_array(f, np.uint64, n).astype(np.int64)
        elif ltype == "sprs":
            pairs = _rd_array(f, np.uint64, n).astype(np.int64).reshape(-1, 2)
            sizes[pairs[:, 0]] = pairs[:, 1]
        else:
            raise NotImplementedError(f"inverted-list size encoding {ltype!r}")
        start = f.tell()
    offsets = np.zeros(nlist + 1, dtype=np.int64)
    np.cumsum(sizes, out=offsets[1:])
    pos = start + offsets[:-1] * (code_size + 8)        # list l: codes [size, code_size], then ids [size]
    mm = np.memmap(path, dtype=np.uint8, mode="r") if offsets[-1] else None

    def read_lists(l0: int, l1: int):
        rows = int(offsets[l1] - offsets[l0])
        codes = np.empty((rows, code_size), dtype=np.uint8)
        ids = np.empty(rows, dtype=np.int64)
        for l in range(l0, l1):
            s, a = int(sizes[l]), int(offsets[l] - offsets[l0])
            if s:
                p = int(pos[l])
                codes[a:a + s] = mm[p:p + s * code_size].reshape(s, code_size)
                ids[a:a + s] = mm[p + s * code_size:p + s * (code_size + 8)].view(np.int64)
        return codes, ids

    return meta, offsets, read_lists


def _read_ivf_header(f: BinaryIO) -> Dict:
    hdr = _read_header(f)
    nlist = _rd(f, "Q")
    nprobe = _rd(f, "Q")
    q = read_faiss(f)
    if q["kind"] != "Flat":
        raise NotImplementedError("only a flat coarse quantizer is supported")
    dm_type = _rd(f, "B")
    n = _rd(f, "Q")
    _rd_array(f, np.int64, n)               # direct-map array (unused)
    if dm_type == 2:
        raise NotImplementedError("hashtable direct map")
    return {**hdr, "nlist": nlist, "nprobe": nprobe, "centroids": q["xb"], "quantizer_metric": q["metric"]}


def read_faiss(f) -> Dict:
    """Parses a faiss index file (path or binary stream) into plain numpy parts:
    Flat: xb [n,d];  IVFFlat: centroids, offsets, vectors [n,d], ids;  IVFPQ: + codebook [M,2^nbits,dsub], codes
    [n, code_size] as stored (code_size = M * nbits / 8: 4-bit codes stay packed two per byte, faiss' order)."""
    if isinstance(f, (str, bytes)):
        with open(f, "rb") as fh:
            return read_faiss(fh)
    tag = _fourcc_str(_rd(f, "I"))
    if tag in ("IxFI", "IxF2", "IxFl"):
        return _read_flat(f, _read_header(f))
    if tag == "IxSQ":
        return _read_sq(f, _read_header(f))
    if tag == "IwFl":
        h = _read_ivf_header(f)
        # faiss does not store code_size for IwFl (index_read.cpp sets it to d * sizeof(float)).  Files written by the
        # first version of this module carried a redundant u64 here: tolerate both by peeking at the next fourcc.
        peek = f.read(4)
        if peek not in (b"ilar", b"il00"):
            rest = f.read(4)
            if struct.unpack("<Q", peek + rest)[0] != h["d"] * 4:
                raise ValueError("IVFFlat: neither an inverted-list fourcc nor a d*4 code_size after the IVF header")
            peek = f.read(4)
        cs, offsets, codes, ids = _read_invlists(f, h["nlist"], tag_bytes=peek)
        if cs != h["d"] * 4:
            raise ValueError("IVFFlat code_size mismatch")
        return {"kind": "IVFFlat", **h, "offsets": offsets, "vectors": codes.view(np.float32).reshape(-1, h["d"]), "ids": ids}
    if tag in ("IwSq", "IwSQ"):
        h = _read_ivf_header(f)
        sq = _read_scalar_quantizer(f, h["d"])
        code_size = _rd(f, "Q")
        by_residual = bool(_rd(f, "B")) if tag == "IwSq" else True
        cs, offsets, codes, ids = _read_invlists(f, h["nlist"])
        if code_size != h["d"] or cs != code_size:
            raise ValueError("IVF-SQ8: code_size disagrees with d")
        return {"kind": "IVFSQ", **h, "by_residual": by_residual, "sq": sq, "offsets": offsets, "codes": codes, "ids": ids}
    if tag == "IwPQ":
        h = _read_ivf_header(f)
        by_residual = bool(_rd(f, "B"))
        code_size = _rd(f, "Q")
        pd, M, nbits = _rd(f, "Q"), _rd(f, "Q"), _rd(f, "Q")
        n = _rd(f, "Q")
        cent = _rd_array(f, np.float32, n)
        ksub = 1 << nbits
        if pd != h["d"] or n != ksub * pd:
            raise ValueError("product quantizer shape mismatch")
        cs, offsets, codes, ids = _read_invlists(f, h["nlist"])
        if cs != code_size:
            raise ValueError("IVFPQ code_size mismatch")
        return {"kind": "IVFPQ", **h, "by_residual": by_residual, "M": M, "nbits": nbits,
                "codebook": cent.reshape(M, ksub, pd // M), "offsets": offsets, "codes": codes, "ids": ids}
    if tag == "IxRF":
        hdr = _read_header(f)
        base = read_faiss(f)
        refine = read_faiss(f)
        k_factor = _rd(f, "f")
        if refine["kind"] not in ("Flat", "SQ"):
            raise NotImplementedError("only a flat (IxFI) or QT_8bit scalar-quantizer (IxSQ) refine index is supported")
        if base["d"] != hdr["d"] or refine["d"] != hdr["d"] or refine["ntotal"] != base["ntotal"]:
            raise ValueError("IndexRefine: base and refine index disagree on d or ntotal")
        if refine["kind"] == "SQ":          # SQ8 store: codes [ntotal, d] uint8 + sq [2, d] (vmin, vdiff), no "xb"
            return {"kind": "Refine", **hdr, "base": base, "sq": refine["sq"], "codes": refine["codes"], "k_factor": k_factor}
        return {"kind": "Refine", **hdr, "base": base, "xb": refine["xb"], "k_factor": k_factor}
    raise NotImplementedError(f"faiss index type {tag!r} is not supported (Flat / IVFFlat / IVF-SQ8 / IVFPQ / RefineFlat only)")


# ----------------------------------------------------------------------------------------------------------
# writing
# ----------------------------------------------------------------------------------------------------------
def _wr(f: BinaryIO, fmt: str, *v):
    f.write(struct.pack("<" + fmt, *v))


def _write_header(f: BinaryIO, tag: str, d: int, ntotal: int, is_trained: bool, metric: int):
    _wr(f, "I", fourcc(tag))
    _wr(f, "i", d)
    _wr(f, "q", ntotal)
    _wr(f, "q", 1 << 20)
    _wr(f, "q", 1 << 20)
    _wr(f, "B", 1 if is_trained else 0)
    _wr(f, "i", metric)


def _write_flat(f: BinaryIO, xb: np.ndarray, metric: int = METRIC_INNER_PRODUCT):
    xb = np.ascontiguousarray(xb, dtype=np.float32)
    _write_header(f, "IxFI" if metric == METRIC_INNER_PRODUCT else "IxF2", xb.shape[1], xb.shape[0], True, metric)
    _wr(f, "Q", xb.size)
    f.write(xb.tobytes())


def write_flat_rows(f: BinaryIO, d: int, ntotal: int, row_chunks) -> None:
    """IxFI from consecutive row chunks (arrays [m, d], written as float32): the bytes _write_flat writes for their
    concatenation, without holding it, so an index larger than host memory is written one chunk at a time."""
    _write_header(f, "IxFI", d, ntotal, True, METRIC_INNER_PRODUCT)
    _wr(f, "Q", ntotal * d)
    rows = 0
    for c in row_chunks:
        c = np.ascontiguousarray(c, dtype=np.float32)
        f.write(c.tobytes())
        rows += c.shape[0]
    if rows != ntotal:
        raise ValueError(f"wrote {rows} rows of a {ntotal}-row flat index")


def flat_rows_memmap(path: str):
    """(d, ntotal, rows) of an IxFI file, rows = a read-only float32 np.memmap [ntotal, d] over its payload: a flat
    index can be loaded chunk by chunk without reading the file into memory."""
    with open(path, "rb") as f:
        tag = _fourcc_str(_rd(f, "I"))
        if tag != "IxFI":
            raise ValueError(f"{path} is not a faiss IndexFlatIP file (IxFI), it is {tag!r}")
        hdr = _read_header(f)
        n = _rd(f, "Q")
        if n != hdr["ntotal"] * hdr["d"]:
            raise ValueError(f"flat index payload has {n} floats, expected {hdr['ntotal']} x {hdr['d']}")
        offset = f.tell()
    if hdr["ntotal"] == 0:
        return hdr["d"], 0, np.zeros((0, hdr["d"]), np.float32)
    return hdr["d"], hdr["ntotal"], np.memmap(path, dtype=np.float32, mode="r", offset=offset,
                                              shape=(hdr["ntotal"], hdr["d"]))


def _write_sq(f: BinaryIO, sq: np.ndarray, codes: np.ndarray):
    sq = np.ascontiguousarray(sq, dtype=np.float32)
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    d = sq.shape[1]
    _write_header(f, "IxSQ", d, codes.shape[0], True, METRIC_INNER_PRODUCT)
    _wr(f, "i", QT_8BIT)
    _wr(f, "i", RS_MINMAX)
    _wr(f, "f", 0.0)
    _wr(f, "Q", d)
    _wr(f, "Q", d)                            # code_size: one byte per element
    _wr(f, "Q", sq.size)
    f.write(sq.tobytes())
    _wr(f, "Q", codes.size)
    f.write(codes.tobytes())


def _write_scalar_quantizer(f: BinaryIO, sq: np.ndarray):
    """write_ScalarQuantizer of a QT_8bit quantizer with the trained range sq [2, d]."""
    sq = np.ascontiguousarray(sq, dtype=np.float32)
    d = sq.shape[1]
    _wr(f, "i", QT_8BIT)
    _wr(f, "i", RS_MINMAX)
    _wr(f, "f", 0.0)
    _wr(f, "Q", d)
    _wr(f, "Q", d)                            # code_size: one byte per element
    _wr(f, "Q", sq.size)
    f.write(sq.tobytes())


def _write_invlists(f: BinaryIO, nlist: int, code_size: int, offsets: np.ndarray, codes: np.ndarray, ids: np.ndarray):
    _wr(f, "I", fourcc("ilar"))
    _wr(f, "Q", nlist)
    _wr(f, "Q", code_size)
    sizes = np.diff(offsets).astype(np.uint64)
    nonzero = np.nonzero(sizes)[0]
    if len(nonzero) > nlist // 2:
        _wr(f, "I", fourcc("full"))
        _wr(f, "Q", nlist)
        f.write(sizes.tobytes())
    else:                                     # faiss writes the sparse form when few lists are populated
        _wr(f, "I", fourcc("sprs"))
        pairs = np.stack([nonzero.astype(np.uint64), sizes[nonzero]], axis=1)
        _wr(f, "Q", pairs.size)
        f.write(np.ascontiguousarray(pairs).tobytes())
    codes = np.ascontiguousarray(codes).view(np.uint8).reshape(len(ids), code_size) if len(ids) else np.zeros((0, code_size), np.uint8)
    ids = np.ascontiguousarray(ids, dtype=np.int64)
    for l in range(nlist):
        a, b = int(offsets[l]), int(offsets[l + 1])
        if b > a:
            f.write(codes[a:b].tobytes())
            f.write(ids[a:b].tobytes())


def _write_invlists_head(f: BinaryIO, nlist: int, code_size: int, offsets: np.ndarray) -> None:
    _wr(f, "I", fourcc("ilar"))
    _wr(f, "Q", nlist)
    _wr(f, "Q", code_size)
    sizes = np.diff(offsets).astype(np.uint64)
    nonzero = np.nonzero(sizes)[0]
    if len(nonzero) > nlist // 2:
        _wr(f, "I", fourcc("full"))
        _wr(f, "Q", nlist)
        f.write(sizes.tobytes())
    else:                                     # faiss writes the sparse form when few lists are populated
        _wr(f, "I", fourcc("sprs"))
        pairs = np.stack([nonzero.astype(np.uint64), sizes[nonzero]], axis=1)
        _wr(f, "Q", pairs.size)
        f.write(np.ascontiguousarray(pairs).tobytes())


def _write_ivf_prefix(f: BinaryIO, parts: Dict, ntotal: int) -> int:
    """Everything of an IVFFlat / IVFSQ file before its inverted lists; returns the code size."""
    c = parts["centroids"]
    d, nlist = c.shape[1], c.shape[0]
    if parts["kind"] == "IVFFlat":
        _write_ivf_header(f, "IwFl", d, ntotal, nlist, parts.get("nprobe", 1), c)
        return d * 4
    _write_ivf_header(f, "IwSq", d, ntotal, nlist, parts.get("nprobe", 1), c)
    _write_scalar_quantizer(f, parts["sq"])
    _wr(f, "Q", d)                            # code_size
    _wr(f, "B", 1 if parts.get("by_residual", True) else 0)
    return d


def write_ivf_streamed(f: BinaryIO, parts: Dict, offsets: np.ndarray, ids: np.ndarray, rows, step_rows: int) -> None:
    """An IVFFlat / IVFSQ file (parts without the vectors / codes) whose CSR rows come from rows(r0, r1) -> [r1 - r0,
    d] float32 (IVFFlat) or uint8 codes (IVFSQ), called for list ranges of about step_rows rows: the bytes write_faiss
    writes for the whole arrays, holding one range at a time."""
    nlist = parts["centroids"].shape[0]
    offsets = np.asarray(offsets, dtype=np.int64)
    ids = np.ascontiguousarray(ids, dtype=np.int64)
    code_size = _write_ivf_prefix(f, parts, len(ids))
    _write_invlists_head(f, nlist, code_size, offsets)
    l0 = 0
    while l0 < nlist:
        l1 = min(nlist, max(int(np.searchsorted(offsets, offsets[l0] + max(1, step_rows), side="right")) - 1, l0 + 1))
        r0, r1 = int(offsets[l0]), int(offsets[l1])
        if r1 > r0:
            x = rows(r0, r1)
            x = np.ascontiguousarray(x, dtype=np.float32 if parts["kind"] == "IVFFlat" else np.uint8)
            if x.shape[0] != r1 - r0:
                raise ValueError(f"rows({r0}, {r1}) returned {x.shape[0]} rows")
            x = x.view(np.uint8).reshape(r1 - r0, code_size)
            for l in range(l0, l1):
                a, b = int(offsets[l]), int(offsets[l + 1])
                if b > a:
                    f.write(x[a - r0:b - r0].tobytes())
                    f.write(ids[a:b].tobytes())
        l0 = l1


def _write_ivf_header(f: BinaryIO, tag: str, d: int, ntotal: int, nlist: int, nprobe: int, centroids: np.ndarray):
    _write_header(f, tag, d, ntotal, True, METRIC_INNER_PRODUCT)
    _wr(f, "Q", nlist)
    _wr(f, "Q", nprobe)
    _write_flat(f, centroids, METRIC_INNER_PRODUCT)
    _wr(f, "B", 0)                            # DirectMap::NoMap
    _wr(f, "Q", 0)                            # empty direct-map array


def write_faiss(f, parts: Dict) -> None:
    """Inverse of read_faiss: `parts` as returned by it (kind = Flat | IVFFlat | IVFSQ | IVFPQ | Refine)."""
    if isinstance(f, (str, bytes)):
        with open(f, "wb") as fh:
            return write_faiss(fh, parts)
    kind = parts["kind"]
    if kind == "Flat":
        _write_flat(f, parts["xb"], parts.get("metric", METRIC_INNER_PRODUCT))
    elif kind == "IVFFlat":
        d = parts["centroids"].shape[1]
        _write_ivf_header(f, "IwFl", d, len(parts["ids"]), parts["centroids"].shape[0], parts.get("nprobe", 1), parts["centroids"])
        _write_invlists(f, parts["centroids"].shape[0], d * 4, parts["offsets"],
                        np.ascontiguousarray(parts["vectors"], dtype=np.float32), parts["ids"])
    elif kind == "IVFSQ":
        d = parts["centroids"].shape[1]
        _write_ivf_header(f, "IwSq", d, len(parts["ids"]), parts["centroids"].shape[0], parts.get("nprobe", 1), parts["centroids"])
        _write_scalar_quantizer(f, parts["sq"])
        _wr(f, "Q", d)                        # code_size
        _wr(f, "B", 1 if parts.get("by_residual", True) else 0)
        _write_invlists(f, parts["centroids"].shape[0], d, parts["offsets"], parts["codes"], parts["ids"])
    elif kind == "IVFPQ":
        d = parts["centroids"].shape[1]
        M, ksub, dsub = parts["codebook"].shape
        nbits = int(np.log2(ksub))
        code_size = (M * nbits + 7) // 8
        _write_ivf_header(f, "IwPQ", d, len(parts["ids"]), parts["centroids"].shape[0], parts.get("nprobe", 1), parts["centroids"])
        _wr(f, "B", 1)                        # by_residual
        _wr(f, "Q", code_size)
        _wr(f, "Q", d); _wr(f, "Q", M); _wr(f, "Q", nbits)
        cb = np.ascontiguousarray(parts["codebook"], dtype=np.float32)
        _wr(f, "Q", cb.size)
        f.write(cb.tobytes())
        _write_invlists(f, parts["centroids"].shape[0], code_size, parts["offsets"], parts["codes"], parts["ids"])
    elif kind == "Refine":
        rows = parts["codes"] if "codes" in parts else parts["xb"]
        _write_header(f, "IxRF", rows.shape[1], rows.shape[0], True, METRIC_INNER_PRODUCT)
        write_faiss(f, parts["base"])
        if "codes" in parts:
            _write_sq(f, parts["sq"], parts["codes"])
        else:
            _write_flat(f, rows, METRIC_INNER_PRODUCT)
        _wr(f, "f", float(parts.get("k_factor", 1.0)))
    else:
        raise NotImplementedError(kind)


def is_faiss_file(path: str) -> bool:
    try:
        with open(path, "rb") as f:
            tag = f.read(4).decode("ascii", "replace")
    except OSError:
        return False
    return tag in ("IxFI", "IxF2", "IxFl", "IwFl", "IwPQ", "IwSq", "IwSQ", "IxRF")
