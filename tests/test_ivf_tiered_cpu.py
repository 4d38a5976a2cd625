"""IVF-Flat / IVF-SQ8 tiered by list (rsb_reserve_lists: lists [0, L_dev) in device memory, the rest in pinned host
memory) without a GPU: the config key, the C-ABI symbol and signature, the refusals that happen before any device
allocation, and the streaming IwFl / IwSq writer and list-by-list reader."""
import ctypes
import os
import re

import numpy as np
import pytest

from retrieval_scaling_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(*extra, index_type="IVFFlat"):
    from retrieval_scaling_b200 import config as C
    conf = os.path.join(ROOT, "ric", "conf")
    return C.load_config("default", conf, ["datastore.domain=x", f"datastore.index.index_type={index_type}",
                                           *extra]).datastore.index


def test_list_device_rows_key():
    from retrieval_scaling_b200.indicies.base import Indexer
    assert Indexer.list_device_rows(_cfg()) is None                                       # absent: all on device
    assert Indexer.list_device_rows(_cfg("+datastore.index.list_device_rows=0")) == 0
    for dt in ("float32", "float16", "sq8"):                                               # any storage dtype
        cfg = _cfg(f"+datastore.index.storage_dtype={dt}", "+datastore.index.list_device_rows=50000000")
        assert Indexer.list_device_rows(cfg) == 50_000_000 and Indexer.storage_dtype(cfg) == dt
    for bad in ("-1", "1.5", "abc", "true"):
        with pytest.raises(ValueError, match="list_device_rows must be an integer"):
            Indexer.list_device_rows(_cfg(f"+datastore.index.list_device_rows={bad}"))
    for it in ("Flat", "IVFPQ"):
        with pytest.raises(ValueError, match="needs index_type IVFFlat"):
            Indexer.list_device_rows(_cfg("+datastore.index.list_device_rows=10", index_type=it))


def test_existing_device_rows_key_still_refuses_ivf():
    """The Flat key keeps its meaning: list_device_rows is the IVF form, device_rows on IVFFlat is still refused."""
    from retrieval_scaling_b200.indicies.base import Indexer
    cfg = _cfg("+datastore.index.storage_dtype=float16", "+datastore.index.device_rows=10",
               "+datastore.index.list_device_rows=10")
    with pytest.raises(ValueError, match="index_type Flat and storage_dtype float16"):
        Indexer.device_rows(cfg)
    assert Indexer.list_device_rows(cfg) == 10


def test_reserve_lists_symbol_and_signature():
    L = _lib.lib()
    sig = {name: (res, args) for name, res, args in _lib.SIGNATURES}
    assert hasattr(L, "rsb_reserve_lists")
    assert sig["rsb_reserve_lists"] == (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
                                                       ctypes.c_size_t, ctypes.c_void_p])
    h = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "rsb.h")).read(), flags=re.S)
    assert re.search(r"int\s+rsb_reserve_lists\s*\(\s*rsb_index_t\*\s*h\s*,\s*const\s+int64_t\*\s*sizes_host\s*,\s*"
                     r"int64_t\s+device_rows\s*,\s*size_t\s+staging_bytes\s*,\s*rsb_stream_t\s+stream\s*\)", h)


def test_null_handle_refusals():
    L = _lib.lib()
    sizes = (ctypes.c_int64 * 4)(1, 2, 3, 4)
    assert L.rsb_reserve_lists(None, sizes, 10, 0, None) == _lib.RSB_ERR_INVALID
    assert b"null handle" in L.rsb_last_error()
    assert L.rsb_export_rows(None, 0, 1, ctypes.c_void_p(16), None) == _lib.RSB_ERR_INVALID
    assert b"null handle" in L.rsb_last_error()


def test_index_arguments_are_checked_before_any_allocation():
    from retrieval_scaling_b200.index import IndexIVFFlat, IndexIVFScalarQuantizer
    for bad in (-1, 1.5, "3", True):
        with pytest.raises(ValueError, match="list_device_rows"):
            IndexIVFFlat(128, 16, dtype="float16", list_device_rows=bad)
        with pytest.raises(ValueError, match="list_device_rows"):
            IndexIVFScalarQuantizer(128, 16, list_device_rows=bad)
        with pytest.raises(ValueError, match="staging_bytes"):
            IndexIVFFlat(128, 16, list_device_rows=10, staging_bytes=bad)
    with pytest.raises(ValueError, match="float16 or float32"):
        IndexIVFFlat(128, 16, dtype="sq8", list_device_rows=10)


def test_read_index_refusals_before_any_allocation(tmp_path):
    from retrieval_scaling_b200 import faiss_io
    from retrieval_scaling_b200.index import read_index
    ivf = str(tmp_path / "ivf.faiss")
    faiss_io.write_faiss(ivf, {"kind": "IVFFlat", "centroids": np.ones((2, 64), np.float32),
                               "offsets": np.array([0, 1, 1]), "vectors": np.ones((1, 64), np.float32),
                               "ids": np.zeros(1, np.int64)})
    with pytest.raises(ValueError, match="IxFI"):                     # the Flat form still refuses IVF files
        read_index(ivf, storage_dtype="float16", device_rows=1)
    with pytest.raises(ValueError, match="give one of them"):
        read_index(ivf, device_rows=1, list_device_rows=1)
    with pytest.raises(ValueError, match="list_device_rows"):
        read_index(ivf, list_device_rows=-1)
    flat = str(tmp_path / "flat.faiss")
    faiss_io.write_faiss(flat, {"kind": "Flat", "xb": np.ones((3, 64), np.float32)})
    with pytest.raises(ValueError, match="IwFl"):
        read_index(flat, list_device_rows=1)
    rsb1 = str(tmp_path / "x.rsb1")
    open(rsb1, "wb").write(b"\x80\x04not a faiss file")
    with pytest.raises(NotImplementedError, match="faiss format"):
        read_index(rsb1, list_device_rows=1)


def _ivf_parts(kind, rng, nlist=9, d=32, empty=(0, 4, 8)):
    sizes = rng.integers(1, 300, nlist)
    sizes[list(empty)] = 0
    off = np.zeros(nlist + 1, np.int64)
    np.cumsum(sizes, out=off[1:])
    n = int(off[-1])
    parts = {"kind": kind, "centroids": rng.standard_normal((nlist, d)).astype(np.float32), "offsets": off,
             "ids": rng.permutation(10 * n)[:n].astype(np.int64), "nprobe": 3}
    if kind == "IVFFlat":
        parts["vectors"] = rng.standard_normal((n, d)).astype(np.float32)
    else:
        parts.update(codes=rng.integers(0, 256, (n, d)).astype(np.uint8), by_residual=True,
                     sq=np.stack([rng.standard_normal(d), rng.random(d) + 0.1]).astype(np.float32))
    return parts


@pytest.mark.parametrize("kind", ["IVFFlat", "IVFSQ"])
@pytest.mark.parametrize("step", [1, 50, 10 ** 6])
def test_streamed_ivf_writer_matches_write_faiss_and_reads_back(tmp_path, kind, step):
    from retrieval_scaling_b200 import faiss_io
    rng = np.random.default_rng(step)
    parts = _ivf_parts(kind, rng)
    payload = parts["vectors"] if kind == "IVFFlat" else parts["codes"]
    a, b = str(tmp_path / "a.faiss"), str(tmp_path / "b.faiss")
    faiss_io.write_faiss(a, parts)
    calls = []

    def rows(r0, r1):
        calls.append((r0, r1))
        return payload[r0:r1]

    meta = {k: v for k, v in parts.items() if k not in ("vectors", "codes", "offsets", "ids")}
    with open(b, "wb") as f:
        faiss_io.write_ivf_streamed(f, meta, parts["offsets"], parts["ids"], rows, step)
    assert open(a, "rb").read() == open(b, "rb").read()
    assert calls and calls[0][0] == 0 and calls[-1][1] == len(parts["ids"])      # contiguous list ranges
    assert all(p[1] == q[0] for p, q in zip(calls, calls[1:]))
    m, off, read_lists = faiss_io.ivf_lists_memmap(b)
    assert m["kind"] == kind and m["nlist"] == 9 and m["nprobe"] == 3 and np.array_equal(off, parts["offsets"])
    assert np.array_equal(m["centroids"], parts["centroids"])
    if kind == "IVFSQ":
        assert m["by_residual"] and np.array_equal(m["sq"], parts["sq"])
    for l0, l1 in ((0, 9), (1, 4), (4, 5), (5, 9)):
        codes, ids = read_lists(l0, l1)
        r0, r1 = off[l0], off[l1]
        assert np.array_equal(codes, np.ascontiguousarray(payload[r0:r1]).view(np.uint8).reshape(r1 - r0, codes.shape[1]))
        assert np.array_equal(ids, parts["ids"][r0:r1])


def test_streamed_ivf_writer_of_an_empty_index_matches(tmp_path):
    from retrieval_scaling_b200 import faiss_io
    rng = np.random.default_rng(3)
    parts = _ivf_parts("IVFFlat", rng, empty=tuple(range(9)))
    a, b = str(tmp_path / "a.faiss"), str(tmp_path / "b.faiss")
    faiss_io.write_faiss(a, parts)
    with open(b, "wb") as f:
        faiss_io.write_ivf_streamed(f, {"kind": "IVFFlat", "centroids": parts["centroids"], "nprobe": 3},
                                    parts["offsets"], parts["ids"], None, 100)
    assert open(a, "rb").read() == open(b, "rb").read()
    _, off, _ = faiss_io.ivf_lists_memmap(b)
    assert off[-1] == 0
