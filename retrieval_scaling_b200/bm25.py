"""BM25 retrieval on the GPU: the reference's sparse retriever (`model.sparse_retriever=bm25`).

The reference indexes every passage of the listed shards with Anserini (`src/index.py:164-202`) and searches each
query with pyserini's `LuceneSearcher.search(raw_query, n_docs)` (`src/search.py:763-807`), one query at a time.
Here the same index is a term-major CSR of postings in device memory, and `rsb_bm25_search` (csrc/rsb_bm25.cu) scores
a batch of queries term at a time.  This module holds every rule the scores depend on:

  analyze()          Anserini's default English analyzer (StandardTokenizer, EnglishPossessiveFilter,
                     LowerCaseFilter, StopFilter, PorterStemFilter)
  int_to_byte4() / byte4_to_int()   Lucene's SmallFloat, the one-byte document length
  norm_cache(), idf()               Lucene 9 BM25Similarity's float arithmetic
  BM25Index          build / save / load / search

The score of document d for a query is the fp32 sum, in ascending term id, of w - w / x over the query's distinct
analyzed terms t present in d, with w = (float) count_t * idf_t and x = 1f + (float) tf * cache[norm(d)].
`oracle/bm25_oracle.py` restates it in numpy.
"""
from __future__ import annotations

import json
import logging
import os
import re
from collections import Counter
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

try:
    import regex as _regex
except ImportError as e:  # pragma: no cover
    raise ImportError("retrieval_scaling_b200.bm25 needs the `regex` package for UAX #29 word segmentation") from e

ANALYZER_VERSION = 2          # bump when a rule below changes: an index built by another version is refused
K1, B = 0.9, 0.4              # pyserini's LuceneSearcher defaults; the reference never sets them
MAX_K = 4096                  # the select limit of the other searches (rsb_bm25_search refuses more)
MAX_TOKEN_LENGTH = 255        # StandardTokenizer.DEFAULT_MAX_TOKEN_LENGTH
WS_BUDGET = 1 << 30           # search workspace per call: query batches are sized to stay under it
UPLOAD_CHUNK = 1 << 24        # postings converted per step of BM25Index.to_device
UPLOAD_TEMP_BYTES = 48        # device temporaries per posting of one upload chunk (indices, gathers, x), an upper bound

# Lucene's EnglishAnalyzer.ENGLISH_STOP_WORDS_SET, the stopwords of Anserini's default English analyzer
ENGLISH_STOP_WORDS = frozenset(
    "a an and are as at be but by for if in into is it no not of on or such that the their then there these they this "
    "to was will with".split())


# ----------------------------------------------------------------------------------------------------------------
# analyzer
# ----------------------------------------------------------------------------------------------------------------
# StandardTokenizer: UAX #29 word boundaries.  The `regex` package's (?w) mode puts \b at exactly those boundaries;
# the tokenizer keeps the segments that hold a letter or a digit (`U.S.A.` -> `U.S.A`, `don't`, `3.14`, `1,000`,
# `foo_bar`, `wi-fi` -> `wi`, `fi`, one token per CJK ideograph) and splits a longer one into 255-character pieces.
_BOUNDARY = _regex.compile(r"(?V1w)\b")
_WORDLIKE = _regex.compile(r"[\p{L}\p{N}]")


def tokenize(text: str) -> List[str]:
    """StandardTokenizer (Lucene): the UAX #29 word segments of `text` that contain a letter or a digit."""
    out = []
    for seg in _BOUNDARY.split(text):
        if seg and _WORDLIKE.search(seg):
            if len(seg) <= MAX_TOKEN_LENGTH:
                out.append(seg)
            else:
                out.extend(seg[i:i + MAX_TOKEN_LENGTH] for i in range(0, len(seg), MAX_TOKEN_LENGTH))
    return out


_APOSTROPHES = ("'", "’", "＇")


def strip_possessive(tok: str) -> str:
    """EnglishPossessiveFilter (Lucene): a trailing 's / 'S, with any of its three apostrophes, is dropped."""
    if len(tok) >= 2 and tok[-1] in "sS" and tok[-2] in _APOSTROPHES:
        return tok[:-2]
    return tok


def lowercase(tok: str) -> str:
    """LowerCaseFilter (Lucene): Character.toLowerCase per code point, the simple mapping, without context.  Python's
    str.lower() differs in two places, both undone here: the full mapping of U+0130 `İ` (two characters there, `i`
    here), and the Final_Sigma rule (`Σ` at the end of a word becomes `ς` there, always `σ` here: `ΟΔΟΣ` -> `οδοσ`).
    With `İ` replaced first, str.lower() maps one character to one, so the `Σ` positions carry over."""
    low = tok.replace("İ", "i").lower()
    if "Σ" in tok:
        low = "".join("σ" if o == "Σ" else c for o, c in zip(tok.replace("İ", "i"), low))
    return low


# ---- PorterStemFilter: Martin Porter's reference implementation, which Lucene's PorterStemmer ports ------------------
def _cons(b: str, i: int) -> bool:
    c = b[i]
    if c in "aeiou":
        return False
    if c == "y":
        return i == 0 or not _cons(b, i - 1)
    return True


def _m(b: str, j: int) -> int:
    """Number of VC sequences in b[0..j]."""
    n, i = 0, 0
    while True:
        if i > j:
            return n
        if not _cons(b, i):
            break
        i += 1
    i += 1
    while True:
        while True:
            if i > j:
                return n
            if _cons(b, i):
                break
            i += 1
        i += 1
        n += 1
        while True:
            if i > j:
                return n
            if not _cons(b, i):
                break
            i += 1
        i += 1


def _vowel_in_stem(b: str, j: int) -> bool:
    return any(not _cons(b, i) for i in range(j + 1))


def _doublec(b: str, j: int) -> bool:
    return j >= 1 and b[j] == b[j - 1] and _cons(b, j)


def _cvc(b: str, i: int) -> bool:
    if i < 2 or not _cons(b, i) or _cons(b, i - 1) or not _cons(b, i - 2):
        return False
    return b[i] not in "wxy"


_STEP2 = {"a": (("ational", "ate"), ("tional", "tion")), "c": (("enci", "ence"), ("anci", "ance")),
          "e": (("izer", "ize"),),
          "l": (("bli", "ble"), ("alli", "al"), ("entli", "ent"), ("eli", "e"), ("ousli", "ous")),
          "o": (("ization", "ize"), ("ation", "ate"), ("ator", "ate")),
          "s": (("alism", "al"), ("iveness", "ive"), ("fulness", "ful"), ("ousness", "ous")),
          "t": (("aliti", "al"), ("iviti", "ive"), ("biliti", "ble")), "g": (("logi", "log"),)}
_STEP3 = {"e": (("icate", "ic"), ("ative", ""), ("alize", "al")), "i": (("iciti", "ic"),),
          "l": (("ical", "ic"), ("ful", "")), "s": (("ness", ""),)}
_STEP4 = {"a": ("al",), "c": ("ance", "ence"), "e": ("er",), "i": ("ic",), "l": ("able", "ible"),
          "n": ("ant", "ement", "ment", "ent"), "o": ("ion", "ou"), "s": ("ism",), "t": ("ate", "iti"), "u": ("ous",),
          "v": ("ive",), "z": ("ize",)}


def _replace_suffix(b: str, rules) -> str:
    for suf, rep in rules:
        if b.endswith(suf):
            j = len(b) - len(suf) - 1
            return b[:j + 1] + rep if _m(b, j) > 0 else b
    return b


def porter_stem(w: str) -> str:
    """Porter's algorithm as in his reference C implementation (and Lucene's port): words of 1-2 characters are left
    alone, and step 2 maps `bli` -> `ble` and `logi` -> `log` (his departures from the 1980 paper)."""
    if len(w) <= 2:
        return w
    b = w
    # step 1ab: plurals, -ed, -ing
    if b.endswith("s"):
        if b.endswith("sses"):
            b = b[:-2]
        elif b.endswith("ies"):
            b = b[:-2]
        elif len(b) >= 2 and b[-2] != "s":
            b = b[:-1]
    if b.endswith("eed"):
        if _m(b, len(b) - 4) > 0:
            b = b[:-1]
    else:
        suf = "ed" if b.endswith("ed") else "ing" if b.endswith("ing") else None
        if suf and _vowel_in_stem(b, len(b) - len(suf) - 1):
            b = b[:-len(suf)]
            if b.endswith(("at", "bl", "iz")):
                b = b + "e"
            elif _doublec(b, len(b) - 1):
                if b[-1] not in "lsz":
                    b = b[:-1]
            elif _m(b, len(b) - 1) == 1 and _cvc(b, len(b) - 1):
                b = b + "e"
    # step 1c: y -> i when another vowel is in the stem
    if b.endswith("y") and _vowel_in_stem(b, len(b) - 2):
        b = b[:-1] + "i"
    # steps 2 and 3: the first suffix of the list that matches decides; it is replaced when m > 0 before it.
    # Step 2 is keyed on the penultimate letter and skipped for a one-letter word (Lucene's "Bug 1" guard).
    if len(b) >= 2:
        b = _replace_suffix(b, _STEP2.get(b[-2], ()))
    b = _replace_suffix(b, _STEP3.get(b[-1], ()))
    # step 4: -ant, -ence, ... removed when m > 1 before them; -ion only after s or t
    if len(b) >= 2:
        for suf in _STEP4.get(b[-2], ()):
            if b.endswith(suf):
                j = len(b) - len(suf) - 1
                if suf == "ion" and not (j >= 0 and b[j] in "st"):
                    continue
                if _m(b, j) > 1:
                    b = b[:j + 1]
                break
    # step 5: a final -e removed, -ll reduced to -l; m is taken over the word as it entered this step
    full, k = b, len(b) - 1
    if b[k] == "e":
        a = _m(full, k)
        if a > 1 or (a == 1 and not _cvc(full, k - 1)):
            b = b[:-1]
    if b[-1] == "l" and _doublec(b, len(b) - 1) and _m(full, k) > 1:
        b = b[:-1]
    return b


class Analyzer:
    """Anserini's default English analyzer, with a cache of the analysis of every distinct surface form (index build
    over millions of passages is otherwise dominated by stemming in Python).  `stopwords` replaces Lucene's
    33-word set, as the reference's `--stopwords` file does at index time."""

    def __init__(self, stopwords: Optional[Iterable[str]] = None):
        self.stopwords = ENGLISH_STOP_WORDS if stopwords is None else frozenset(stopwords)
        self._cache: Dict[str, Optional[str]] = {}

    def term(self, tok: str) -> Optional[str]:
        t = self._cache.get(tok, False)
        if t is False:
            low = lowercase(strip_possessive(tok))
            t = None if (not low or low in self.stopwords) else porter_stem(low)
            self._cache[tok] = t
        return t

    def __call__(self, text: str) -> List[str]:
        terms = []
        for tok in tokenize(text):
            t = self.term(tok)
            if t is not None:
                terms.append(t)
        return terms


def analyze(text: str, stopwords: Optional[Iterable[str]] = None) -> List[str]:
    return Analyzer(stopwords)(text)


def read_stopwords(path: str) -> List[str]:
    """A stopwords file, one word per line (the reference's `datastore.index.stopwords`)."""
    with open(path, encoding="utf-8") as f:
        return [w for w in (line.strip() for line in f) if w]


# ----------------------------------------------------------------------------------------------------------------
# Lucene numerics
# ----------------------------------------------------------------------------------------------------------------
NUM_FREE_VALUES = 24          # SmallFloat: 255 - longToInt4(Integer.MAX_VALUE)


def _long_to_int4(i: int) -> int:
    nbits = int(i).bit_length()
    if nbits < 4:
        return int(i)
    shift = nbits - 4
    return ((i >> shift) & 0x07) | ((shift + 1) << 3)


def _int4_to_long(i: int) -> int:
    bits, shift = i & 0x07, (i >> 3) - 1
    return bits if shift == -1 else (bits | 0x08) << shift


def int_to_byte4(n: int) -> int:
    """SmallFloat.intToByte4: lengths below 24 exactly, then 24 + a 4-bit float (3 mantissa bits)."""
    if n < 0:
        raise ValueError(n)
    return n if n < NUM_FREE_VALUES else NUM_FREE_VALUES + _long_to_int4(n - NUM_FREE_VALUES)


def byte4_to_int(b: int) -> int:
    """SmallFloat.byte4ToInt."""
    return b if b < NUM_FREE_VALUES else NUM_FREE_VALUES + _int4_to_long(b - NUM_FREE_VALUES)


LENGTH_TABLE = np.array([byte4_to_int(i) for i in range(256)], dtype=np.float32)   # BM25Similarity.LENGTH_TABLE


def encode_norms(lengths: np.ndarray) -> np.ndarray:
    """intToByte4 of every document length, vectorised: uint8 [n]."""
    lengths = np.asarray(lengths, dtype=np.int64)
    thresholds = np.array([byte4_to_int(i) for i in range(256)], dtype=np.int64)   # ascending
    return (np.searchsorted(thresholds, lengths, side="right") - 1).astype(np.uint8)


def norm_cache(avgdl: np.float32, k1: float = K1, b: float = B) -> np.ndarray:
    """BM25Similarity: cache[i] = 1f / (k1 * ((1 - b) + b * LENGTH_TABLE[i] / avgdl)), left to right in float."""
    f = np.float32
    k1, b, avgdl = f(k1), f(b), f(avgdl)
    return (f(1) / (k1 * ((f(1) - b) + b * LENGTH_TABLE / avgdl))).astype(np.float32)


def idf(df: np.ndarray, n_docs: int) -> np.ndarray:
    """BM25Similarity.idf: (float) log(1 + (docCount - docFreq + 0.5) / (docFreq + 0.5)), in double."""
    df = np.asarray(df, dtype=np.float64)
    return np.log(1.0 + (float(n_docs) - df + 0.5) / (df + 0.5)).astype(np.float32)


def avg_length(sum_len: int, n_docs: int) -> np.float32:
    """BM25Similarity.avgFieldLength: (float) (sumTotalTermFreq / (double) docCount); 1 for an empty index."""
    return np.float32(sum_len / float(n_docs)) if n_docs else np.float32(1.0)


# ----------------------------------------------------------------------------------------------------------------
# the index
# ----------------------------------------------------------------------------------------------------------------
def _postings_numpy(tok, doc_of_tok, n_docs):
    key = tok.astype(np.int64) * max(n_docs, 1) + doc_of_tok
    uniq, tf = np.unique(key, return_counts=True)
    return uniq // max(n_docs, 1), uniq % max(n_docs, 1), tf


def _postings_torch(tok, doc_of_tok, n_docs, device):
    import torch
    n = max(n_docs, 1)
    key = torch.as_tensor(tok, device=device).to(torch.int64) * n + torch.as_tensor(doc_of_tok, device=device)
    uniq, tf = torch.unique(key, sorted=True, return_counts=True)      # a device sort of the (term, document) keys
    del key
    return ((uniq // n).cpu().numpy(), (uniq % n).cpu().numpy(), tf.cpu().numpy())


class BM25Index:
    """Term-major CSR postings sorted by document: term t's postings are docs[offsets[t]:offsets[t+1]] with term
    frequencies tfs[...]; norms [n_docs] are the SmallFloat bytes of the document lengths.  `vocab` lists the terms in
    term-id order (sorted).  `shards` lists (shard id, passages) in document order: document numbers run through the
    shards in that order and through each shard's lines in file order."""

    def __init__(self, offsets, docs, tfs, norms, sum_len: int, vocab: Optional[List[str]] = None,
                 stopwords: Optional[Iterable[str]] = None, shards: Optional[List[Tuple[int, int]]] = None):
        self.offsets = np.asarray(offsets, dtype=np.int64)
        self.docs = np.asarray(docs, dtype=np.int32)
        self.tfs = np.asarray(tfs, dtype=np.int32)
        self.norms = np.asarray(norms, dtype=np.uint8)
        self.n_terms = len(self.offsets) - 1
        self.n_docs = len(self.norms)
        self.df = np.diff(self.offsets)
        self.doc_count = int(np.count_nonzero(self.norms))   # Lucene's docCount: documents with an indexed term
        self.sum_len = int(sum_len)
        self.avgdl = avg_length(self.sum_len, self.doc_count)
        self.idf = idf(self.df, self.doc_count)
        self.vocab = vocab
        self.term_id = {t: i for i, t in enumerate(vocab)} if vocab is not None else None
        self.stopwords = sorted(ENGLISH_STOP_WORDS if stopwords is None else set(stopwords))
        self.shards = [(int(s), int(n)) for s, n in shards] if shards is not None else [(0, self.n_docs)]
        self._query_analyzer = Analyzer()                    # the default stopwords: see query_terms
        self._dev = None

    # ---- build ----------------------------------------------------------------------------------------------------
    @classmethod
    def from_tokens(cls, tok, doc_off, n_terms: int, sort_device=None, **kw) -> "BM25Index":
        """Postings from the analyzed token ids of every document: tok [T] term ids, doc_off [n_docs + 1] int64.
        sort_device: None sorts with numpy, a torch device ("cuda", "cpu") with torch; both give the same arrays."""
        doc_off = np.asarray(doc_off, dtype=np.int64)
        lengths = np.diff(doc_off)
        n_docs = len(lengths)
        if sort_device is None:
            doc_of_tok = np.repeat(np.arange(n_docs, dtype=np.int64), lengths)
            terms, docs, tfs = _postings_numpy(np.asarray(tok), doc_of_tok, n_docs)
        else:
            import torch
            doc_of_tok = torch.repeat_interleave(torch.arange(n_docs, dtype=torch.int64, device=sort_device),
                                                 torch.as_tensor(lengths, device=sort_device))
            terms, docs, tfs = _postings_torch(tok, doc_of_tok, n_docs, sort_device)
        offsets = np.zeros(n_terms + 1, dtype=np.int64)
        np.cumsum(np.bincount(terms, minlength=n_terms), out=offsets[1:])
        return cls(offsets, docs, tfs, encode_norms(lengths), int(lengths.sum()), **kw)

    @classmethod
    def build(cls, texts: Iterable[str], stopwords: Optional[Iterable[str]] = None, sort_device="auto",
              shards=None) -> "BM25Index":
        """Index `texts` (one document each, in document order).  sort_device "auto": the GPU when CUDA is present."""
        if sort_device == "auto":
            import torch
            sort_device = "cuda" if torch.cuda.is_available() else None
        an = Analyzer(stopwords)
        ids: Dict[str, int] = {}
        tok: List[int] = []
        doc_off = [0]
        for text in texts:
            for t in an(text):
                i = ids.get(t)
                if i is None:
                    i = ids[t] = len(ids)
                tok.append(i)
            doc_off.append(len(tok))
        vocab = sorted(ids)                                   # term ids in term order, as Lucene's term dictionary
        remap = np.empty(len(ids), dtype=np.int32)
        remap[[ids[t] for t in vocab]] = np.arange(len(vocab), dtype=np.int32)
        tok_arr = remap[np.asarray(tok, dtype=np.int64)] if tok else np.zeros(0, dtype=np.int32)
        return cls.from_tokens(tok_arr, doc_off, len(vocab), sort_device=sort_device, vocab=vocab,
                               stopwords=an.stopwords, shards=shards)

    # ---- storage --------------------------------------------------------------------------------------------------
    def save(self, path: str) -> None:
        os.makedirs(path, exist_ok=True)
        for name in ("offsets", "docs", "tfs", "norms"):
            np.save(os.path.join(path, f"{name}.npy"), getattr(self, name))
        with open(os.path.join(path, "vocab.json"), "w", encoding="utf-8") as f:
            json.dump(self.vocab or [], f, ensure_ascii=False)
        meta = {"format": "rsb-bm25", "analyzer_version": ANALYZER_VERSION, "k1": K1, "b": B, "N": self.doc_count,
                "n_docs": self.n_docs, "n_terms": self.n_terms, "sum_len": self.sum_len, "avgdl": float(self.avgdl),
                "stopwords": self.stopwords,
                # document numbers run through these (shard, passages) pairs in order: document d is line
                # d - (passages of the earlier shards) of its shard
                "shards": [list(s) for s in self.shards]}
        tmp = os.path.join(path, "meta.json.tmp")
        with open(tmp, "w") as f:
            json.dump(meta, f, indent=1)
        os.replace(tmp, os.path.join(path, "meta.json"))      # written last: its presence marks a complete index

    @classmethod
    def load(cls, path: str, device=None) -> "BM25Index":
        with open(os.path.join(path, "meta.json")) as f:
            meta = json.load(f)
        if meta.get("analyzer_version") != ANALYZER_VERSION or meta.get("k1") != K1 or meta.get("b") != B:
            raise ValueError(f"{path}: built with analyzer version {meta.get('analyzer_version')}, k1 {meta.get('k1')}, "
                             f"b {meta.get('b')}; this build reads version {ANALYZER_VERSION}, k1 {K1}, b {B}")
        arr = {n: np.load(os.path.join(path, f"{n}.npy")) for n in ("offsets", "docs", "tfs", "norms")}
        with open(os.path.join(path, "vocab.json"), encoding="utf-8") as f:
            vocab = json.load(f)
        ix = cls(arr["offsets"], arr["docs"], arr["tfs"], arr["norms"], meta["sum_len"], vocab=vocab,
                 stopwords=meta["stopwords"], shards=meta["shards"])
        if device is not None:
            ix.to_device(device)
        return ix

    def db_ids(self, docs: np.ndarray) -> np.ndarray:
        """Document numbers -> [n, 2] (shard id, line in the shard): the pairs `index_utils.fetch_passages` takes."""
        docs = np.asarray(docs, dtype=np.int64)
        counts = np.array([n for _, n in self.shards], dtype=np.int64)
        starts = np.concatenate([[0], np.cumsum(counts)])
        pos = np.searchsorted(starts, docs, side="right") - 1
        sid = np.array([s for s, _ in self.shards], dtype=np.int64)
        return np.stack([sid[pos], docs - starts[pos]], axis=1) if len(docs) else np.zeros((0, 2), dtype=np.int64)

    # ---- device ---------------------------------------------------------------------------------------------------
    def device_bytes(self) -> int:
        """Bytes the index takes in device memory: 8 per posting plus the term offsets."""
        return 8 * len(self.docs) + 8 * len(self.offsets)

    def working_bytes(self, chunk: int = UPLOAD_CHUNK) -> int:
        """Device memory needed besides the index: the larger of the upload's temporaries (the norms, and up to
        UPLOAD_TEMP_BYTES per posting of one chunk) and the search workspace (at most WS_BUDGET bytes)."""
        upload = 10 * self.n_docs + UPLOAD_TEMP_BYTES * min(chunk, len(self.docs))
        return max(upload, WS_BUDGET)

    def to_device(self, device="cuda", chunk: int = UPLOAD_CHUNK) -> "BM25Index":
        """Upload the postings as (int32 document, fp32 x = 1f + (float) tf * cache[norm]) pairs.  x is two separate
        elementwise kernels (a product, then a sum), each rounded on its own: Lucene's float arithmetic.
        Refused with MemoryError, before any allocation, when the index plus working_bytes() exceeds the free device
        memory.  A query batch's own arrays and its [nq, k] results come on top of that."""
        import torch
        device = torch.device(device)
        if device.type != "cuda":
            raise ValueError(f"BM25Index.to_device: {device} is not a CUDA device (the scorer is CUDA only)")
        size, extra = self.device_bytes(), self.working_bytes(chunk)
        need = size + extra
        free, _ = torch.cuda.mem_get_info(device)
        if need > free:
            raise MemoryError(f"the BM25 index takes {size} bytes ({size / 2**30:.2f} GiB) of device memory for "
                              f"{len(self.docs)} postings and needs {extra} bytes ({extra / 2**30:.2f} GiB) more to "
                              f"upload and search it: {need} bytes; {free} bytes ({free / 2**30:.2f} GiB) are free on "
                              f"{device}")
        cache = torch.as_tensor(norm_cache(self.avgdl), device=device)
        norms = torch.as_tensor(self.norms, device=device)
        post = torch.empty((len(self.docs), 2), dtype=torch.int32, device=device)
        for a in range(0, len(self.docs), chunk):
            d = torch.as_tensor(self.docs[a:a + chunk], device=device)
            tf = torch.as_tensor(self.tfs[a:a + chunk], device=device).to(torch.float32)
            x = torch.mul(tf, cache[norms[d.long()].long()])
            x = torch.add(x, 1.0)
            post[a:a + chunk, 0] = d
            post[a:a + chunk, 1] = x.view(torch.int32)
        self._dev = {"device": device, "offsets": torch.as_tensor(self.offsets, device=device), "post": post}
        return self

    # ---- queries --------------------------------------------------------------------------------------------------
    def query_terms(self, text: str) -> Tuple[np.ndarray, np.ndarray]:
        """Anserini's bag-of-words query: one clause per distinct analyzed term present in the index, boosted by its
        count.  Queries are analyzed with the default stopwords whatever the index was built with: the reference
        opens `LuceneSearcher(path)` without an analyzer, so pyserini's default English analyzer applies.
        Returns (term ids ascending, fp32 weights (float) count * idf)."""
        counts = Counter(self._query_analyzer(text))
        return self.term_query(counts)

    def term_query(self, counts: Dict) -> Tuple[np.ndarray, np.ndarray]:
        """{term (str) or term id (int): count} -> (term ids ascending, fp32 weights); unknown terms dropped."""
        ids, cnt = [], []
        for t, c in counts.items():
            i = self.term_id.get(t) if isinstance(t, str) else int(t)
            if i is not None and 0 <= i < self.n_terms:
                ids.append(i)
                cnt.append(c)
        order = np.argsort(np.asarray(ids, dtype=np.int64), kind="stable")
        ids = np.asarray(ids, dtype=np.int32)[order]
        w = (np.asarray(cnt, dtype=np.float32)[order] * self.idf[ids]).astype(np.float32)
        return ids, w

    def search(self, queries: Sequence[str], k: int) -> Tuple[np.ndarray, np.ndarray]:
        """(D fp32 [nq, k], I int64 [nq, k]) document numbers, best first; past the hits I = -1 and D = -FLT_MAX."""
        check_k(k)
        D, I = self.search_terms([self.query_terms(q) for q in queries], k)
        return D.cpu().numpy(), I.cpu().numpy()

    def search_terms(self, queries: Sequence[Tuple[np.ndarray, np.ndarray]], k: int, ws_budget: int = WS_BUDGET):
        """Analyzed queries [(term ids ascending, fp32 weights)] -> device (D, I), in batches whose workspace stays
        under ws_budget bytes."""
        import torch
        from . import _lib
        check_k(k)
        if self._dev is None:
            raise RuntimeError("BM25Index.search: the index is not on a device; call to_device() or load(path, device)")
        dev = self._dev["device"]
        nq = len(queries)
        D = torch.empty((nq, k), dtype=torch.float32, device=dev)
        I = torch.empty((nq, k), dtype=torch.int64, device=dev)
        L = _lib.lib()
        per_q = max(1, L.rsb_bm25_workspace_bytes(self.n_docs, 1, k))
        batch = int(max(1, min(nq, ws_budget // per_q, 65535)))
        ws = torch.empty(L.rsb_bm25_workspace_bytes(self.n_docs, batch, k) + 16, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            for a in range(0, nq, batch):
                q_off, q_term, q_w = pack_queries(queries[a:a + batch])
                q_off, q_term, q_w = (torch.as_tensor(x, device=dev) for x in (q_off, q_term, q_w))
                nb = len(q_off) - 1
                rc = L.rsb_bm25_search(self._dev["offsets"].data_ptr(), self._dev["post"].data_ptr(), self.n_docs,
                                       q_off.data_ptr(), q_term.data_ptr(), q_w.data_ptr(), nb, k, D[a:].data_ptr(),
                                       I[a:].data_ptr(), ws.data_ptr(), ws.numel(), stream)
                _check(rc)
        return D, I


def check_k(k: int) -> None:
    if k < 1:
        raise ValueError(f"k={k}: k must be positive")
    if k > MAX_K:
        raise NotImplementedError(f"k={k}: BM25 search returns at most {MAX_K} results per query")


def pack_queries(queries: Sequence[Tuple[np.ndarray, np.ndarray]]):
    """[(term ids, weights)] -> CSR by query: (q_off int32 [nq + 1], q_term int32, q_w fp32)."""
    lens = np.array([len(t) for t, _ in queries], dtype=np.int64)
    q_off = np.zeros(len(queries) + 1, dtype=np.int64)
    np.cumsum(lens, out=q_off[1:])
    if q_off[-1] >= 2 ** 31:
        raise ValueError("a query batch holds fewer than 2^31 terms")
    q_term = np.concatenate([np.asarray(t, dtype=np.int32) for t, _ in queries]) if len(queries) else np.zeros(0, np.int32)
    q_w = np.concatenate([np.asarray(w, dtype=np.float32) for _, w in queries]) if len(queries) else np.zeros(0, np.float32)
    return q_off.astype(np.int32), q_term.astype(np.int32), q_w.astype(np.float32)


def _check(rc: int) -> None:
    from . import _lib
    if rc == _lib.RSB_OK:
        return
    msg = _lib.lib().rsb_bm25_last_error().decode("utf-8", "replace")
    if rc == _lib.RSB_ERR_UNSUPPORTED:
        raise NotImplementedError(msg)
    if rc == _lib.RSB_ERR_OOM:
        raise MemoryError(msg)
    if rc == _lib.RSB_ERR_INVALID:
        raise ValueError(msg)
    raise _lib.RsbError(f"librsb error {rc}: {msg}")


# ----------------------------------------------------------------------------------------------------------------
# the pipeline: one index over every passage of the listed shards (reference src/index.py:158-202)
# ----------------------------------------------------------------------------------------------------------------
def flat_shard_ids(cfg) -> List[int]:
    """`datastore.index.index_shard_ids`, groups flattened: [[0], [1]] -> [0, 1]."""
    from .config import ListConfig
    ids = cfg.datastore.index.index_shard_ids
    if ids and isinstance(ids[0], (ListConfig, list, tuple)):
        return [int(i) for g in ids for i in g]
    return [int(i) for i in ids]


def index_dir(cfg, shard_ids: Sequence[int]) -> str:
    """{passages_dir}/bm25/{shard ids joined by _}/rsb_index, next to where the reference puts its Lucene `index/`."""
    return os.path.join(cfg.datastore.embedding.passages_dir, "bm25", "_".join(str(s) for s in shard_ids), "rsb_index")


_SHARD_FILE = re.compile(r"raw_passages-(\d+)-of-\d+\.jsonl$")


def shard_path(passages_dir: str, shard: int) -> str:
    for name in sorted(os.listdir(passages_dir)):
        m = _SHARD_FILE.match(name)
        if m and int(m.group(1)) == int(shard):
            return os.path.join(passages_dir, name)
    raise FileNotFoundError(f"no raw_passages-{shard}-of-*.jsonl in {passages_dir}")


def _passage_texts(passages_dir: str, shard_ids: Sequence[int], counts: List[Tuple[int, int]]):
    for s in shard_ids:
        n = 0
        with open(shard_path(passages_dir, s), "rb") as f:
            for line in f:
                yield json.loads(line)["text"]                 # the passage text alone, no title (reference :190-191)
                n += 1
        counts.append((int(s), n))


def build_index(cfg) -> str:
    """Build the BM25 index of the configured shards unless it exists; returns its directory."""
    shard_ids = flat_shard_ids(cfg)
    path = index_dir(cfg, shard_ids)
    if os.path.exists(os.path.join(path, "meta.json")):
        logging.info(f"BM25 index {path} exists, skipping building.")
        return path
    sw_file = cfg.datastore.index.get("stopwords", None)
    stopwords = read_stopwords(sw_file) if sw_file else None
    counts: List[Tuple[int, int]] = []
    logging.info(f"Building a BM25 index over shards {shard_ids} into {path}")
    ix = BM25Index.build(_passage_texts(cfg.datastore.embedding.passages_dir, shard_ids, counts), stopwords=stopwords)
    ix.shards = counts
    ix.save(path)
    logging.info(f"BM25 index: {ix.n_docs} passages, {ix.n_terms} terms, {len(ix.docs)} postings")
    return path
