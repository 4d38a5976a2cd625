"""MinHash de-duplication on the GPU (rsb_dedup.cu through retrieval_scaling_b200.dedup) against the CPU oracle:
signatures bit for bit at the word-split and SHA-1 padding edges, keep flags on crafted signatures, whole groups,
and `ric/main_ric.py tasks.eval.merge_search=true` byte for byte against a CPU run with the oracle de-duplication."""
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from oracle import minhash_oracle as M

from dedup_fixture import make_examples, oracle_deduplicate, write_sources

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPACES = [chr(c) for c in range(0x110000) if not 0xD800 <= c <= 0xDFFF and chr(c).isspace()]


def _check_signatures(texts):
    from retrieval_scaling_b200 import dedup
    sig, nw = dedup.minhash_signatures(texts)
    for t, s, n in zip(texts, sig, nw):
        assert n == len(t.split()), repr(t[:60])
        assert np.array_equal(s, M.signature(t)), repr(t[:60])


def test_every_whitespace_and_nonspace_neighbours_as_separators():
    rng = random.Random(0)
    near = sorted({c + d for c in (ord(s) for s in SPACES) for d in (-1, 1)} | {0x200B, 0x180E, 0xFEFF, 0x2060, 0x7F, 0})
    non_space = [chr(c) for c in near if 0 <= c < 0x110000 and not 0xD800 <= c <= 0xDFFF and not chr(c).isspace()]
    texts = []
    for sep in SPACES + non_space:
        words = [f"w{rng.randrange(50)}" for _ in range(16)]
        texts.append(sep.join(words))                             # as the separator
        texts.append(" ".join(w + sep + "x" for w in words))      # inside words
        texts.append(sep + " ".join(words) + sep * 2)             # leading / trailing
    _check_signatures(texts)


def test_word_counts_around_the_shingle_size_and_long_text():
    rng = random.Random(1)
    texts = [" ".join(f"t{rng.randrange(9)}" for _ in range(n)) for n in (0, 1, 12, 13, 14, 40)]
    texts += ["", "   \n\t", " ".join(f"v{rng.randrange(10**6)}" for _ in range(10000))]
    _check_signatures(texts)


@pytest.mark.parametrize("length", [55, 56, 63, 64, 119, 120, 183, 184])
def test_shingle_lengths_at_sha1_block_edges(length):
    """13 words joined by 12 spaces: word lengths chosen so that the joined shingle has exactly `length` bytes, with
    ASCII words and with 2-, 3- and 4-byte characters placed across the 55/56/64-byte edges."""
    texts = []
    for ch in ("a", "é", "東", "𝔘"):
        nb = len(ch.encode())
        body = length - 12
        words = ["b"] * 13
        rest = body - 13
        k = 0
        while rest > 0:
            if rest >= nb and (k % 2 == 0 or nb == 1):
                words[k % 13] += ch
                rest -= nb
            else:
                words[k % 13] += "c"
                rest -= 1
            k += 1
        t = " ".join(words)
        assert len(t.encode()) == length
        texts.append(t)
        texts.append(t + " tail")                         # two shingles, the second of another length
    _check_signatures(texts)


def _crafted(rng, n_equal, band_match):
    a = np.array([rng.randrange(1 << 32) for _ in range(128)], dtype=np.uint32)
    b = a.copy()
    # positions to change: with band_match, band 0 (0..12) stays whole; without, one position of every band changes
    forced = [] if band_match else [k * 13 + rng.randrange(13) for k in range(9)]
    free = [p for p in range(128) if p not in forced and (not band_match or p >= 13)]
    change = forced + rng.sample(free, 128 - n_equal - len(forced))
    b[change] ^= 1
    return a, b


@pytest.mark.parametrize("n_equal", [102, 103, 128])
@pytest.mark.parametrize("band_match", [True, False])
def test_keep_flags_on_crafted_signatures(n_equal, band_match):
    from retrieval_scaling_b200 import dedup
    if not band_match and n_equal > 119:
        pytest.skip("breaking all 9 bands leaves at most 119 equal positions")
    rng = random.Random(n_equal * 2 + band_match)
    sigs, nw, goff = [], [], [0]
    for _ in range(40):                                   # groups of [a, b], [b, a], and a short slot in the middle
        a, b = _crafted(rng, n_equal, band_match)
        for g in ([a, b], [b, a], [a, np.full(128, 0xFFFFFFFF, np.uint32), b]):
            sigs += g
            nw += [20] * len(g) if len(g) == 2 else [20, 5, 20]
            goff.append(len(sigs))
    sigs = np.stack(sigs)
    keep = dedup.keep_flags(sigs, np.array(nw), np.array(goff))
    expect = []
    for g in range(len(goff) - 1):
        s = slice(goff[g], goff[g + 1])
        expect += M.keep_flags(list(sigs[s]), [n >= 13 for n in nw[s]])
    assert keep.tolist() == expect
    dropped = not keep[1]
    assert dropped == (band_match and n_equal > 102)


def test_groups_with_planted_families_and_contamination():
    from retrieval_scaling_b200 import dedup
    data = make_examples(11, 60, 50)
    gpu = dedup.deduplicate(json.loads(json.dumps(data)), batch_bytes=20000)   # several batches
    cpu = oracle_deduplicate(json.loads(json.dumps(data)))
    assert gpu == cpu
    n_in = sum(len(ex["ctxs"]) for ex in data)
    n_out = sum(len(ex["ctxs"]) for ex in cpu)
    assert 0.3 * n_in < n_out < 0.9 * n_in                 # the fixture drops a good share, not everything


@pytest.mark.parametrize("p", ["1", "0.5"])
def test_main_ric_merge_search_matches_a_cpu_run(tmp_path, p):
    from retrieval_scaling_b200 import config as rcfg
    from retrieval_scaling_b200 import search
    listing = write_sources(str(tmp_path), seed=21, n_queries=40, n_docs=30)
    gpu_dir, cpu_dir = tmp_path / "gpu", tmp_path / "cpu"
    ov = lambda d: [f"evaluation.search.paths_to_merge={listing}", f"evaluation.search.merged_path={d}/dedup_all.jsonl",
                    "evaluation.search.n_docs=30", f"evaluation.search.topk_subsample_p={p}",
                    "evaluation.search.subsample_seed=5"]
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "ric", "main_ric.py"), "tasks.eval.merge_search=true",
                        *ov(gpu_dir)], cwd=str(tmp_path), env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    cfg = rcfg.load_config("default", os.path.join(ROOT, "ric", "conf"), ov(cpu_dir))
    search.post_hoc_merge_topk_multi_domain(cfg, deduplicate=oracle_deduplicate)
    names = sorted(os.listdir(cpu_dir))
    assert names == sorted(os.listdir(gpu_dir)) == sorted(["all.jsonl", "dedup_all.jsonl",
                                                           f"full_subsampled_{p}_5_dedup_all.jsonl"])
    for n in names:
        assert (gpu_dir / n).read_bytes() == (cpu_dir / n).read_bytes(), n


def test_large_group_across_rounds_and_lead_tiles():
    """One group of 1100 slots: pairs planted across the 256-slot rounds of minhash_dedup_kernel and across its lead
    tile (8192 // 9 = 910 earlier slots), 102- and 103-equal pairs, short slots; then a small group after it."""
    from retrieval_scaling_b200 import dedup
    rng = np.random.default_rng(7)
    n = 1100
    sigs = rng.integers(0, 1 << 32, size=(n + 3, 128), dtype=np.uint64).astype(np.uint32)
    nw = np.full(n + 3, 40)

    def plant(i, j, n_equal):
        sigs[j] = sigs[i]
        change = rng.choice(np.arange(13, 128), 128 - n_equal, replace=False)     # band 0 stays whole
        sigs[j, change] ^= 1

    dup_pairs = [(3, 300), (255, 256), (5, 1000), (909, 1050), (0, 1099), (911, 912)]
    for i, j in dup_pairs:
        plant(i, j, 110)
    plant(100, 1080, 102)                   # a candidate, but not above the threshold
    plant(400, 910, 103)
    nw[[257, 511, 512, 1098]] = 12          # short slots on round edges
    plant(n + 0, n + 2, 120)
    goff = np.array([0, n, n + 3])
    keep = dedup.keep_flags(sigs, nw, goff)
    expect = M.keep_flags(list(sigs[:n]), [w >= 13 for w in nw[:n]]) + \
        M.keep_flags(list(sigs[n:]), [w >= 13 for w in nw[n:]])
    assert keep.tolist() == expect
    dropped = set(np.flatnonzero(~keep).tolist())
    assert {j for _, j in dup_pairs} | {910, 257, 511, 512, 1098, n + 2} == dropped


def test_groups_without_texts():
    from retrieval_scaling_b200 import dedup
    data = [{"raw_query": "it refers to the following information here", "ctxs": []}, {"raw_query": None, "ctxs": []}]
    assert dedup.deduplicate(data) == [dict(ex, ctxs=[]) for ex in data]
    data = [{"raw_query": None, "ctxs": []}, {"raw_query": "a short query", "ctxs": [{"retrieval text": "x " * 20}]}]
    assert dedup.deduplicate(json.loads(json.dumps(data))) == oracle_deduplicate(data)
