"""CPU restatement of the MinHash de-duplication the reference applies to merged multi-source results
(`utils/deduplication.py`), written from datasketch's published arithmetic because datasketch is not a dependency.

What is restated, and how each piece is pinned in tests/test_minhash_oracle.py:
  shingle_document   `text.split()` then the set of `' '.join(words[i:i + 13])`.
  sha1_hash32        datasketch.hashfunc.sha1_hash32: the first 4 bytes of SHA-1, read little-endian.
  permutations       MinHash(num_perm=128, seed=1): RandomState(1) draws a in [1, 2^61 - 1) then b in [0, 2^61 - 1),
                     as uint64, once per permutation.
  signature          MinHash.update_batch: ((hv * a + b) mod 2^64) mod (2^61 - 1) & 0xffffffff, minimum over the
                     shingles, starting at 2^32 - 1 (an empty shingle set keeps every value at 2^32 - 1).
  jaccard            count_equal / 128 in float64.
  optimal_param      MinHashLSH's (b, r) for (threshold, num_perm) with weights (0.5, 0.5): loop order and strict `<`
                     kept; the integrals use scipy.integrate.quad.
  remove_duplicates_with_minhash
                     the reference function itself over the restated MinHash / LSH.

Test infrastructure only: the GPU path is retrieval_scaling_b200.dedup.
"""
from __future__ import annotations

import hashlib
import struct
from typing import Dict, List, Optional, Tuple

import numpy as np

NUM_PERM = 128
SHINGLE = 13
THRESHOLD = 0.8
MERSENNE = np.uint64((1 << 61) - 1)
MAX_HASH = np.uint64((1 << 32) - 1)
ABSTAIN = "refers to the following information"


def shingle_document(text: str, shingle_size: int = SHINGLE) -> set:
    words = text.split()
    return set(" ".join(words[i:i + shingle_size]) for i in range(len(words) - shingle_size + 1))


def sha1_hash32(data: bytes) -> int:
    return struct.unpack("<I", hashlib.sha1(data).digest()[:4])[0]


def permutations(num_perm: int = NUM_PERM, seed: int = 1) -> Tuple[np.ndarray, np.ndarray]:
    """(a, b), each uint64 [num_perm], drawn interleaved as datasketch's MinHash._init_permutations does."""
    gen = np.random.RandomState(seed)
    ab = np.array([(gen.randint(1, MERSENNE, dtype=np.uint64), gen.randint(0, MERSENNE, dtype=np.uint64))
                   for _ in range(num_perm)], dtype=np.uint64).T
    return ab[0].copy(), ab[1].copy()


_PERM = None


def _perm():
    global _PERM
    if _PERM is None:
        _PERM = permutations()
    return _PERM


def signature_of_hashes(hv, perm=None) -> np.ndarray:
    """uint32 [num_perm] from the 32-bit shingle hashes `hv` (update_batch's arithmetic: the uint64 product wraps)."""
    a, b = perm if perm is not None else _perm()
    sig = np.full(len(a), MAX_HASH, dtype=np.uint64)
    hv = np.asarray(list(hv), dtype=np.uint64).reshape(-1, 1)
    if len(hv):
        with np.errstate(over="ignore"):
            phv = (hv * a + b) % MERSENNE & MAX_HASH
        sig = np.vstack([phv, sig]).min(axis=0)
    return sig.astype(np.uint32)


def signature(text: str, perm=None) -> np.ndarray:
    return signature_of_hashes((sha1_hash32(s.encode("utf-8")) for s in shingle_document(text)), perm)


def jaccard(s1: np.ndarray, s2: np.ndarray) -> float:
    return float(np.float64(np.count_nonzero(s1 == s2)) / np.float64(len(s1)))


def max_equal(threshold: float = THRESHOLD, num_perm: int = NUM_PERM) -> int:
    """The largest equal count whose estimated Jaccard is still <= threshold (not a duplicate)."""
    return max(c for c in range(num_perm + 1) if np.float64(c) / np.float64(num_perm) <= threshold)


def optimal_param(threshold: float = THRESHOLD, num_perm: int = NUM_PERM,
                  false_positive_weight: float = 0.5, false_negative_weight: float = 0.5) -> Tuple[int, int]:
    from scipy.integrate import quad

    def fp(b, r):
        return quad(lambda s: 1 - (1 - s ** float(r)) ** float(b), 0.0, threshold)[0]

    def fn(b, r):
        return quad(lambda s: 1 - (1 - (1 - s ** float(r)) ** float(b)), threshold, 1.0)[0]

    min_error, opt = float("inf"), (0, 0)
    for b in range(1, num_perm + 1):
        for r in range(1, int(num_perm / b) + 1):
            error = fp(b, r) * false_positive_weight + fn(b, r) * false_negative_weight
            if error < min_error:
                min_error, opt = error, (b, r)
    return opt


_BR: Optional[Tuple[int, int]] = None


def lsh_params() -> Tuple[int, int]:
    global _BR
    if _BR is None:
        _BR = optimal_param()
    return _BR


def lsh_candidates(s1: np.ndarray, s2: np.ndarray, b: int, r: int) -> bool:
    """MinHashLSH: two signatures share a bucket iff all r values of some band are equal."""
    return any(np.array_equal(s1[k * r:(k + 1) * r], s2[k * r:(k + 1) * r]) for k in range(b))


def keep_flags(sigs: np.ndarray, has_shingles, br: Optional[Tuple[int, int]] = None,
               threshold: float = THRESHOLD) -> List[bool]:
    """Per slot of one group: not dropped by an earlier LSH candidate with Jaccard > threshold, and has shingles."""
    b, r = br or lsh_params()
    tables = [dict() for _ in range(b)]              # MinHashLSH's hash tables: band bytes -> slots
    for i, s in enumerate(sigs):
        for k in range(b):
            tables[k].setdefault(s[k * r:(k + 1) * r].tobytes(), []).append(i)
    keep = []
    for j, s in enumerate(sigs):
        cands = {i for k in range(b) for i in tables[k][s[k * r:(k + 1) * r].tobytes()]}
        dup = any(i < j and jaccard(sigs[i], s) > threshold for i in cands)
        keep.append(bool(has_shingles[j]) and not dup)
    return keep


def abstain_string_for_decon(string: str) -> bool:
    return ABSTAIN in string


def remove_duplicates_with_minhash(documents: List[dict], string_for_decontamination: Optional[str] = None) -> List[dict]:
    texts = []
    if string_for_decontamination is not None and not abstain_string_for_decon(string_for_decontamination):
        texts.append(string_for_decontamination)
    off = len(texts)
    texts += [ctx["retrieval text"] for ctx in documents]
    shingles: Dict[int, set] = {i: shingle_document(t) for i, t in enumerate(texts)}
    sigs = [signature_of_hashes(sha1_hash32(s.encode("utf-8")) for s in shingles[i]) for i in range(len(texts))]
    keep = keep_flags(sigs, [bool(shingles[i]) for i in range(len(texts))])
    kept = [documents[j - off] for j in range(off, len(texts)) if keep[j]]
    for doc in kept:
        doc.update({"quality score": 1})
    return kept
