"""BM25 without a GPU: the analyzer rules (StandardTokenizer segments, possessives, simple lowercase, stopwords, Porter
stems), Lucene's SmallFloat and BM25 numerics, the index build / save / load round trip with the numpy and torch
sorts, the oracle's float32 scores against its float64 matrix, and the `main_ric` index task."""
import json
import os

import numpy as np
import pytest

from oracle import bm25_oracle as O
from retrieval_scaling_b200 import bm25

from bm25_fixture import overrides, write_eval_data, write_passages, zipf_corpus, zipf_queries

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("text,tokens", [
    ("U.S.A.", ["U.S.A"]), ("don't", ["don't"]), ("3.14", ["3.14"]), ("1,000", ["1,000"]), ("foo_bar", ["foo_bar"]),
    ("e.g.", ["e.g"]), ("wi-fi", ["wi", "fi"]), ("中文字", ["中", "文", "字"]), ("Hello, world! (x2) -- ...", ["Hello", "world", "x2"]),
    ("", []), ("a" * 300, ["a" * 255, "a" * 45]),
])
def test_standard_tokenizer_segments(text, tokens):
    assert bm25.tokenize(text) == tokens


def test_possessives_lowercase_and_default_stopwords():
    assert [bm25.strip_possessive(t) for t in ("John's", "JOHN'S", "dog’s", "cat＇s", "'s", "bass", "it's")] == \
        ["John", "JOHN", "dog", "cat", "", "bass", "it"]
    assert bm25.lowercase("İSTANBUL") == "istanbul" and len(bm25.lowercase("İ")) == 1
    assert bm25.lowercase("ΟΔΟΣ") == "οδοσ" and bm25.lowercase("ΣΟΦΟΣ") == "σοφοσ" and bm25.lowercase("οδος") == "οδος"
    assert len(bm25.ENGLISH_STOP_WORDS) == 33
    assert bm25.analyze("The dog's running AND the Dogs' houses are there") == ["dog", "run", "dog", "hous"]


def test_file_stopwords_at_index_time_default_at_query_time(tmp_path):
    sw = tmp_path / "stop.txt"
    sw.write_text("river\n\n  bank  \n")
    words = bm25.read_stopwords(str(sw))
    assert words == ["river", "bank"]
    ix = bm25.BM25Index.build(["the river bank", "a bank of the river money", "money"], stopwords=words, sort_device=None)
    assert ix.vocab == ["a", "monei", "of", "the"]            # `the`, `a`, `of` indexed: the file replaced the set
    assert ix.stopwords == ["bank", "river"]
    ids, w = ix.query_terms("the money of a river")           # queries drop the default stopwords only
    assert [ix.vocab[i] for i in ids] == ["monei"]


@pytest.mark.parametrize("word,stem", [
    ("caresses", "caress"), ("ponies", "poni"), ("ties", "ti"), ("caress", "caress"), ("cats", "cat"), ("feed", "feed"),
    ("agreed", "agre"), ("plastered", "plaster"), ("bled", "bled"), ("motoring", "motor"), ("sing", "sing"),
    ("conflated", "conflat"), ("troubled", "troubl"), ("sized", "size"), ("hopping", "hop"), ("tanned", "tan"),
    ("falling", "fall"), ("hissing", "hiss"), ("fizzed", "fizz"), ("failing", "fail"), ("filing", "file"),
    ("happy", "happi"), ("sky", "sky"), ("relational", "relat"), ("conditional", "condit"), ("rational", "ration"),
    ("valenci", "valenc"), ("digitizer", "digit"), ("conformabli", "conform"), ("radicalli", "radic"),
    ("differentli", "differ"), ("vileli", "vile"), ("analogousli", "analog"), ("vietnamization", "vietnam"),
    ("predication", "predic"), ("operator", "oper"), ("feudalism", "feudal"), ("decisiveness", "decis"),
    ("hopefulness", "hope"), ("callousness", "callous"), ("formaliti", "formal"), ("sensitiviti", "sensit"),
    ("sensibiliti", "sensibl"), ("triplicate", "triplic"), ("formative", "form"), ("formalize", "formal"),
    ("electriciti", "electr"), ("electrical", "electr"), ("hopeful", "hope"), ("goodness", "good"),
    ("revival", "reviv"), ("allowance", "allow"), ("inference", "infer"), ("airliner", "airlin"),
    ("gyroscopic", "gyroscop"), ("adjustable", "adjust"), ("defensible", "defens"), ("irritant", "irrit"),
    ("replacement", "replac"), ("adjustment", "adjust"), ("dependent", "depend"), ("adoption", "adopt"),
    ("homologou", "homolog"), ("communism", "commun"), ("activate", "activ"), ("angulariti", "angular"),
    ("homologous", "homolog"), ("effective", "effect"), ("bowdlerize", "bowdler"), ("probate", "probat"),
    ("rate", "rate"), ("cease", "ceas"), ("controll", "control"), ("roll", "roll"),
    ("generalizations", "gener"), ("oscillators", "oscil"),
    ("possibly", "possibl"), ("archaeology", "archaeolog"),    # the reference implementation's bli / logi rules
    ("is", "is"), ("as", "as"), ("y", "y"), ("ies", "i"),
])
def test_porter_stems(word, stem):
    assert bm25.porter_stem(word) == stem


def test_smallfloat_byte4():
    assert all(bm25.int_to_byte4(n) == n and bm25.byte4_to_int(n) == n for n in range(24))
    assert bm25.int_to_byte4(100) == 57 and bm25.byte4_to_int(57) == 96
    ns = list(range(0, 5000)) + [2 ** 20, 2 ** 31 - 1]
    enc = [bm25.int_to_byte4(n) for n in ns]
    assert enc == sorted(enc) and max(enc) == 255
    assert all(bm25.byte4_to_int(b) <= n for b, n in zip(enc, ns))
    assert np.array_equal(bm25.encode_norms(np.array(ns)), np.array(enc, dtype=np.uint8))


def test_bm25_numerics():
    cache = bm25.norm_cache(np.float32(10.0))
    f = np.float32
    assert cache[57] == f(1) / (f(0.9) * ((f(1) - f(0.4)) + f(0.4) * f(96) / f(10.0)))
    assert bm25.idf(np.array([1]), 10)[0] == np.float32(np.log(1.0 + 9.5 / 1.5))
    assert bm25.avg_length(7, 3) == np.float32(7 / 3)


def test_refuses_k_above_4096_before_anything():
    ix = bm25.BM25Index.build(["river bank"], sort_device=None)
    with pytest.raises(NotImplementedError, match="4096"):
        ix.search(["river"], 4097)


def test_build_save_load_round_trip_numpy_and_torch_sorts(tmp_path):
    pdir, texts = write_passages(str(tmp_path))
    a = bm25.BM25Index.build(texts, sort_device=None)
    b = bm25.BM25Index.build(texts, sort_device="cpu")
    for name in ("offsets", "docs", "tfs", "norms"):
        assert np.array_equal(getattr(a, name), getattr(b, name)), name
    assert a.vocab == b.vocab == sorted(a.vocab)
    assert a.doc_count == a.n_docs - 2 and a.n_docs == len(texts)       # two passages with no indexed term
    a.shards = [(0, 40), (1, 30)]
    a.save(str(tmp_path / "ix"))
    c = bm25.BM25Index.load(str(tmp_path / "ix"))
    for name in ("offsets", "docs", "tfs", "norms", "idf"):
        assert np.array_equal(getattr(a, name), getattr(c, name)), name
    assert c.vocab == a.vocab and c.avgdl == a.avgdl and c.shards == a.shards and c.sum_len == a.sum_len
    meta = json.load(open(tmp_path / "ix" / "meta.json"))
    assert meta["k1"] == 0.9 and meta["b"] == 0.4 and meta["N"] == a.doc_count and len(meta["stopwords"]) == 33
    assert c.db_ids(np.array([0, 39, 40, 69])).tolist() == [[0, 0], [0, 39], [1, 0], [1, 29]]
    for d in (0, 7, 69):                                      # postings agree with a direct count of the analysis
        terms = bm25.analyze(texts[d])
        assert bm25.byte4_to_int(int(c.norms[d])) <= len(terms)
        for t in set(terms):
            i = c.term_id[t]
            row = c.docs[c.offsets[i]:c.offsets[i + 1]]
            assert d in row and c.tfs[c.offsets[i] + np.searchsorted(row, d)] == terms.count(t)


def test_torch_and_numpy_sorts_agree_on_a_zipf_corpus():
    tok, off = zipf_corpus(3000, 800, seed=2)
    a = bm25.BM25Index.from_tokens(tok, off, 800, sort_device=None)
    b = bm25.BM25Index.from_tokens(tok, off, 800, sort_device="cpu")
    for name in ("offsets", "docs", "tfs", "norms"):
        assert np.array_equal(getattr(a, name), getattr(b, name)), name
    assert all(np.all(np.diff(a.docs[a.offsets[t]:a.offsets[t + 1]]) > 0) for t in range(800))


def test_oracle_float32_against_float64():
    tok, off = zipf_corpus(4000, 1000, seed=3)
    ix = bm25.BM25Index.from_tokens(tok, off, 1000, sort_device=None)
    queries = [list(q.items()) for q in zipf_queries(1000, 20, seed=4, n_tokens=30)]
    arrays = (ix.offsets, ix.docs, ix.tfs, ix.norms, ix.sum_len)
    S = O.scores_f64(*arrays, queries)
    for r, q in enumerate(queries):
        s = O.scores_f32(*arrays, q)
        assert np.array_equal(s > 0, S[r] > 0)
        assert np.allclose(s, S[r], rtol=(len(q) + 2) * 2.0 ** -22, atol=0)
        D, I = O.topk(s, 50)
        assert np.all(np.diff(D[I >= 0]) <= 0)
    # the oracle's weights are the index's weights
    ids, w = ix.term_query({t: c for t, c in queries[0]})
    assert np.array_equal(w, np.array([np.float32(c) * ix.idf[t] for t, c in sorted(queries[0])], dtype=np.float32))


def test_main_ric_index_task_builds_bm25_without_a_dense_indexer(tmp_path, monkeypatch):
    import importlib.util
    from retrieval_scaling_b200 import config as rcfg
    from retrieval_scaling_b200.indicies import base
    root = str(tmp_path)
    pdir, texts = write_passages(root)
    eval_path = write_eval_data(root)

    def refuse(*a, **k):
        raise AssertionError("a dense Indexer was constructed")
    monkeypatch.setattr(base.Indexer, "__init__", refuse)
    spec = importlib.util.spec_from_file_location("main_ric", os.path.join(ROOT, "ric", "main_ric.py"))
    main_ric = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(main_ric)
    cfg = rcfg.load_config("default", os.path.join(ROOT, "ric", "conf"),
                           overrides(root, pdir, eval_path) + ["tasks.datastore.index=true"])
    main_ric.main(cfg)
    path = os.path.join(pdir, "bm25", "0_1", "rsb_index")
    assert sorted(os.listdir(path)) == ["docs.npy", "meta.json", "norms.npy", "offsets.npy", "tfs.npy", "vocab.json"]
    ix = bm25.BM25Index.load(path)
    assert ix.n_docs == len(texts) and ix.shards == [(0, 40), (1, 30)]
    ref = bm25.BM25Index.build(texts, sort_device=None)
    assert np.array_equal(ix.docs, ref.docs) and ix.vocab == ref.vocab
    main_ric.main(cfg)                                        # exists: not built again
    cfg.model.sparse_retriever = "splade"
    with pytest.raises(NotImplementedError, match="splade"):
        main_ric.main(cfg)


def test_lowercase_is_per_code_point():
    """Character.toLowerCase applies to each code point alone: the result of a token is the concatenation of the
    results of its characters, and each character maps to one."""
    chars = [chr(c) for c in range(0x110000) if not 0xD800 <= c <= 0xDFFF]
    assert all(len(bm25.lowercase(c)) == 1 for c in chars)
    rng = np.random.default_rng(0)
    alphabet = list("ΣσςΑΒΟΔİIiAbΣ'") + ["Ω", "Ä", "ẞ", "Ǆ"]
    for _ in range(2000):
        s = "".join(rng.choice(alphabet, int(rng.integers(1, 9))))
        assert bm25.lowercase(s) == "".join(bm25.lowercase(c) for c in s), s


def test_memory_check_counts_upload_and_search_working_memory():
    tok, off = zipf_corpus(3000, 800, seed=2)
    ix = bm25.BM25Index.from_tokens(tok, off, 800, sort_device=None)
    assert ix.device_bytes() == 8 * len(ix.docs) + 8 * 801
    assert ix.working_bytes() == max(bm25.WS_BUDGET, 10 * 3000 + bm25.UPLOAD_TEMP_BYTES * len(ix.docs))
    assert ix.working_bytes(chunk=1 << 40) >= bm25.UPLOAD_TEMP_BYTES * len(ix.docs)
