"""The CPU MinHash oracle (oracle/minhash_oracle.py) pinned on facts that do not come from it: FIPS SHA-1 vectors,
numpy's RandomState(1) stream, Python big-integer arithmetic, scipy's integrals, the exact Jaccard of large shingle
sets; the whitespace set of the device word split against Python's str.isspace(); datasketch itself when installed."""
import hashlib
import random

import numpy as np
import pytest

from oracle import minhash_oracle as M
from retrieval_scaling_b200 import _lib, dedup


def test_sha1_hash32_is_the_first_four_digest_bytes_little_endian():
    # FIPS 180 vectors: SHA1("abc") = a9993e36..., SHA1("") = da39a3ee...
    assert M.sha1_hash32(b"abc") == 0x363E99A9
    assert M.sha1_hash32(b"") == 0xEEA339DA
    for s in ("café au lait", "東京 " * 40, "x" * 55, "y" * 64):
        d = hashlib.sha1(s.encode("utf-8")).digest()
        assert M.sha1_hash32(s.encode("utf-8")) == d[0] | d[1] << 8 | d[2] << 16 | d[3] << 24


def test_permutations_are_randomstate_1_drawn_a_then_b():
    a, b = M.permutations()
    assert a.dtype == np.uint64 and a.shape == (128,) and b.shape == (128,)
    # first and last draws of RandomState(1): a_0, b_0 are draws 1 and 2, a_127, b_127 draws 255 and 256
    assert (int(a[0]), int(b[0])) == (775169054918279404, 1758426461858698312)
    assert (int(a[127]), int(b[127])) == (1931671111240692334, 1454448473341514576)
    assert (a >= 1).all() and (a < (1 << 61) - 1).all() and (b < (1 << 61) - 1).all()
    da, db = dedup.permutations()
    assert np.array_equal(da, a) and np.array_equal(db, b)


def test_update_batch_wraps_the_product_in_uint64_before_the_mersenne_modulus():
    a, b = M.permutations()
    hs = [0, 1, 0xFFFFFFFF, 0x9E3779B9, 0x363E99A9]
    sig = M.signature_of_hashes(hs)
    expect = [min((((h * int(a[j]) + int(b[j])) % (1 << 64)) % ((1 << 61) - 1)) & 0xFFFFFFFF for h in hs)
              for j in range(128)]
    assert sig.tolist() == expect
    # the wrap changes results: without it the values differ for large hashes
    nowrap = [(((0xFFFFFFFF * int(a[j]) + int(b[j])) % ((1 << 61) - 1)) & 0xFFFFFFFF) for j in range(128)]
    assert M.signature_of_hashes([0xFFFFFFFF]).tolist() != nowrap
    # a hand-sized case: a = 2^61, b = 5, h = 8 -> 2^64 + 5 wraps to 5
    sig = M.signature_of_hashes([8], (np.array([1 << 61], np.uint64), np.array([5], np.uint64)))
    assert sig.tolist() == [5]


def test_empty_shingle_set_keeps_the_initial_maximum():
    assert M.shingle_document("twelve words only " * 4) == set()
    assert (M.signature("one two three") == 0xFFFFFFFF).all()


def test_shingles_use_str_split_and_single_spaces():
    text = "a　b\tc\n\nd  e f g h i j k l m n"
    assert M.shingle_document(text) == {"a b c d e f g h i j k l m", "b c d e f g h i j k l m n"}


def test_lsh_parameters_and_threshold_count():
    assert M.optimal_param(0.8, 128) == (9, 13)
    assert (dedup.LSH_BANDS, dedup.LSH_ROWS) == M.lsh_params()
    assert dedup.MAX_EQUAL == M.max_equal() == 102
    assert 102 / 128 <= 0.8 < 103 / 128


@pytest.mark.parametrize("overlap", [0.3, 0.6, 0.85, 0.95])
def test_estimate_tracks_exact_jaccard_on_large_documents(overlap):
    """Each of the 128 positions is equal with probability ~J (independent permutations), so the estimate's standard
    deviation is sqrt(J (1 - J) / 128); the bound is 4.5 standard deviations (plus 1/128 for the rounding)."""
    rng = random.Random(int(overlap * 100))
    words = [f"t{rng.randrange(10**9)}" for _ in range(4000)]
    n_shared = int(len(words) * overlap)
    t1 = " ".join(words)
    t2 = " ".join(words[:n_shared] + [f"u{rng.randrange(10**9)}" for _ in range(len(words) - n_shared)])
    s1, s2 = M.shingle_document(t1), M.shingle_document(t2)
    exact = len(s1 & s2) / len(s1 | s2)
    est = M.jaccard(M.signature(t1), M.signature(t2))
    assert abs(est - exact) <= 4.5 * np.sqrt(exact * (1 - exact) / 128) + 1 / 128, (est, exact)


def test_remove_duplicates_literal_rules():
    base = " ".join(f"w{i}" for i in range(40))
    q = "question " + base
    docs = [{"retrieval text": t} for t in [
        "x " * 20 + "end",                       # kept
        base,                                    # contaminated by the query (>0.8 with slot 0)
        "short text",                            # fewer than 13 words
        "x " * 20 + "end",                       # duplicate of doc 0
        " ".join(f"v{i}" for i in range(30)),    # kept
    ]]
    kept = M.remove_duplicates_with_minhash([dict(d) for d in docs], q)
    assert [d["retrieval text"] for d in kept] == [docs[0]["retrieval text"], docs[4]["retrieval text"]]
    assert all(d["quality score"] == 1 for d in kept)
    # the abstention: a query about "the following information" is not a slot, so `base` survives
    kept = M.remove_duplicates_with_minhash([dict(d) for d in docs], "it refers to the following information " + base)
    assert [d["retrieval text"] for d in kept] == [docs[0]["retrieval text"], base, docs[4]["retrieval text"]]


def test_device_split_whitespace_is_python_isspace():
    """The word split of rsb_dedup.cu (exported as a host function) against chr(c).isspace() for every code point."""
    cps = [c for c in range(0x110000) if not 0xD800 <= c <= 0xDFFF]
    chars = [chr(c).encode("utf-8") for c in cps]
    buf = np.frombuffer(b"".join(chars), dtype=np.uint8)
    mask = np.zeros(len(buf), dtype=np.uint8)
    L = _lib.lib()
    assert L.rsb_utf8_space_mask(buf.ctypes.data, len(buf), mask.ctypes.data) == 0
    pos = 0
    for c, e in zip(cps, chars):
        m = mask[pos:pos + len(e)]
        assert (m == int(chr(c).isspace())).all(), hex(c)
        pos += len(e)


def test_against_datasketch_when_installed():
    ds = pytest.importorskip("datasketch")
    from datasketch import MinHash, MinHashLSH
    from datasketch.hashfunc import sha1_hash32
    m = MinHash(num_perm=128)
    a, b = M.permutations()
    assert np.array_equal(m.permutations[0], a) and np.array_equal(m.permutations[1], b)
    lsh = MinHashLSH(threshold=0.8, num_perm=128)
    assert (lsh.b, lsh.r) == M.lsh_params()
    text = "the quick brown fox jumps over the lazy dog again and again " * 5 + "東京"
    m = MinHash(permutations=m.permutations)
    m.update_batch([s.encode("utf-8") for s in M.shingle_document(text)])
    assert np.array_equal(m.hashvalues.astype(np.uint32), M.signature(text))
    assert sha1_hash32(b"abc") == M.sha1_hash32(b"abc")
    del ds
