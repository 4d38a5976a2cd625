"""MinHash near-duplicate removal of retrieved passages on the GPU: the reference's `remove_duplicates_with_minhash`
(`utils/deduplication.py`, datasketch MinHash(num_perm=128) + MinHashLSH(threshold=0.8)) for whole batches of queries.

Per query the slots are the query itself (unless it contains "refers to the following information", the reference's
abstention for reading-comprehension prompts) followed by its passages.  A passage is dropped when an earlier slot is an
LSH candidate of it with estimated Jaccard > 0.8 (a passage contaminated by the query, or a near-duplicate of a
higher-ranked passage), or when it has fewer than 13 words.  Survivors keep their order and get `'quality score': 1`.

Host side: UTF-8 packing of the texts of a batch of queries (one buffer, text and group offsets).  Device side
(librsb, rsb_dedup.cu): word split, SHA-1 of every 13-word shingle, the 128 permuted minima, and the keep flags.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib

NUM_PERM = 128
SHINGLE = 13
THRESHOLD = 0.8
# MinHashLSH(threshold=0.8, num_perm=128): datasketch's _optimal_param with weights (0.5, 0.5) gives 9 bands of 13 rows
LSH_BANDS, LSH_ROWS = 9, 13
# jaccard = count_equal / 128 in float64; a slot is a duplicate when that is > THRESHOLD, i.e. count_equal > MAX_EQUAL
MAX_EQUAL = max(c for c in range(NUM_PERM + 1) if np.float64(c) / np.float64(NUM_PERM) <= THRESHOLD)
ABSTAIN = "refers to the following information"
BATCH_BYTES = 128 << 20      # UTF-8 bytes per device batch (one larger query is a batch of its own); the workspace
                             # takes 12 bytes per text byte


def permutations(seed: int = 1):
    """datasketch MinHash(num_perm=128, seed=1).permutations: (a, b) uint64 [128], drawn a then b per permutation."""
    gen = np.random.RandomState(seed)
    mp = np.uint64((1 << 61) - 1)
    ab = np.array([(gen.randint(1, mp, dtype=np.uint64), gen.randint(0, mp, dtype=np.uint64))
                   for _ in range(NUM_PERM)], dtype=np.uint64).T
    return ab[0].copy(), ab[1].copy()


_PERM_HOST = permutations()
_perm_dev = {}


def _perms(device):
    key = str(device)
    if key not in _perm_dev:
        _perm_dev[key] = tuple(torch.from_numpy(p.view(np.int64)).to(device) for p in _PERM_HOST)
    return _perm_dev[key]


def _check(rc: int) -> None:
    if rc == _lib.RSB_OK:
        return
    msg = _lib.lib().rsb_dedup_last_error().decode("utf-8", "replace")
    if rc == _lib.RSB_ERR_INVALID:
        raise ValueError(msg)
    if rc == _lib.RSB_ERR_OOM:
        raise MemoryError(msg)
    raise _lib.RsbError(f"librsb dedup error {rc}: {msg}")


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t: torch.Tensor):
    return ctypes.c_void_p(t.data_ptr())


def _join(enc: Sequence[bytes]):
    off = np.zeros(len(enc) + 1, dtype=np.int64)
    np.cumsum([len(e) for e in enc], out=off[1:])
    return np.frombuffer(b"".join(enc), dtype=np.uint8), off


def pack_texts(texts: Sequence[str]):
    """One UTF-8 buffer (uint8) and the int64 offsets [len(texts) + 1] of its texts."""
    return _join([t.encode("utf-8") for t in texts])


def signatures_device(buf: torch.Tensor, off: torch.Tensor):
    """Device buffer / offsets (from pack_texts) -> (signatures int32 [n, 128] holding the uint32 values, word counts
    int32 [n]), enqueued on the current stream."""
    n, total = off.numel() - 1, buf.numel()
    dev = off.device
    sig = torch.empty((n, NUM_PERM), dtype=torch.int32, device=dev)
    nw = torch.empty(n, dtype=torch.int32, device=dev)
    L = _lib.lib()
    ws = torch.empty(max(1, L.rsb_minhash_workspace_bytes(total)), dtype=torch.uint8, device=dev)
    pa, pb = _perms(dev)
    _check(L.rsb_minhash_signatures(_ptr(buf), _ptr(off), n, total, _ptr(pa), _ptr(pb), _ptr(sig), _ptr(nw),
                                    _ptr(ws), ws.numel(), _stream()))
    return sig, nw


def keep_device(sig: torch.Tensor, n_words: torch.Tensor, group_off: torch.Tensor) -> torch.Tensor:
    """Keep flags uint8 [n] of the slots of the groups group_off (int32 [n_groups + 1]), on the current stream."""
    keep = torch.empty(sig.shape[0], dtype=torch.uint8, device=sig.device)
    if sig.shape[0] == 0:               # groups without slots (abstained queries, no passages): nothing to flag
        return keep
    _check(_lib.lib().rsb_minhash_dedup(_ptr(sig), _ptr(n_words), _ptr(group_off), group_off.numel() - 1, LSH_BANDS,
                                        LSH_ROWS, MAX_EQUAL, _ptr(keep), _stream()))
    return keep


def minhash_signatures(texts: Sequence[str], device="cuda"):
    """(uint32 [n, 128] signatures, int32 [n] word counts) of `texts`, computed on the GPU."""
    buf, off = pack_texts(texts)
    sig, nw = signatures_device(torch.from_numpy(buf.copy()).to(device), torch.from_numpy(off).to(device))
    return sig.cpu().numpy().view(np.uint32), nw.cpu().numpy()


def keep_flags(sig: np.ndarray, n_words: np.ndarray, group_off: np.ndarray, device="cuda") -> np.ndarray:
    """Keep flags (bool [n]) from caller-given uint32 signatures [n, 128] and word counts."""
    s = torch.from_numpy(np.ascontiguousarray(sig, dtype=np.uint32).view(np.int32)).to(device)
    nw = torch.from_numpy(np.ascontiguousarray(n_words, dtype=np.int32)).to(device)
    go = torch.from_numpy(np.ascontiguousarray(group_off, dtype=np.int32)).to(device)
    return keep_device(s, nw, go).cpu().numpy().astype(bool)


@dataclass
class Batch:
    """The packed texts of a batch of queries: group g holds slots group_off[g] .. group_off[g + 1]), the first of them
    the query when has_query[g]."""
    buf: np.ndarray
    text_off: np.ndarray
    group_off: np.ndarray
    has_query: List[bool]


def _encode(ex: dict):
    """(whether the query is slot 0, the UTF-8 of every slot) of one example."""
    q = ex["raw_query"]
    hq = q is not None and ABSTAIN not in q
    texts = ([q] if hq else []) + [ctx["retrieval text"] for ctx in ex["ctxs"]]
    return hq, [t.encode("utf-8") for t in texts]


def _pack(encoded) -> Batch:
    buf, off = _join([b for _, slots in encoded for b in slots])
    group_off = np.cumsum([0] + [len(slots) for _, slots in encoded], dtype=np.int32)
    return Batch(buf, off, group_off, [hq for hq, _ in encoded])


def pack_batch(examples: Sequence[dict]) -> Batch:
    return _pack([_encode(ex) for ex in examples])


def run_batch(batch: Batch, device="cuda") -> np.ndarray:
    """Keep flags (bool, one per slot) of a packed batch: upload, signatures, dedup, download."""
    buf = torch.from_numpy(batch.buf.copy()).to(device)
    off = torch.from_numpy(batch.text_off).to(device)
    goff = torch.from_numpy(batch.group_off).to(device)
    sig, nw = signatures_device(buf, off)
    return keep_device(sig, nw, goff).cpu().numpy().astype(bool)


def apply_keep(examples: Sequence[dict], batch: Batch, keep: np.ndarray) -> None:
    for g, ex in enumerate(examples):
        s0 = int(batch.group_off[g]) + int(batch.has_query[g])
        kept = [ctx for k, ctx in enumerate(ex["ctxs"]) if keep[s0 + k]]
        for ctx in kept:
            ctx.update({"quality score": 1})
        ex["ctxs"] = kept


def deduplicate(examples: List[dict], device: Optional[str] = None, batch_bytes: int = BATCH_BYTES) -> List[dict]:
    """In place over examples {'raw_query', 'ctxs'}: the reference's `multiprocess_deduplication`, over batches of
    consecutive queries of at most `batch_bytes` bytes of UTF-8 each."""
    device = device or "cuda"

    def run(start, stop, encoded):
        batch = _pack(encoded)
        apply_keep(examples[start:stop], batch, run_batch(batch, device))

    encoded, size, start = [], 0, 0
    for j, ex in enumerate(examples):
        e = _encode(ex)
        nbytes = sum(len(b) for b in e[1])
        if encoded and size + nbytes > batch_bytes:
            run(start, j, encoded)
            encoded, size, start = [], 0, j
        encoded.append(e)
        size += nbytes
    if encoded:
        run(start, len(examples), encoded)
    return examples
