"""Host logic of the multi-source merge (search.post_hoc_merge_topk_multi_domain) with the de-duplication stubbed by
the CPU oracle: file names and the strip('dedup_') quirk, the domain tag, merge order, subsampling, short-chunk
removal, the cached-file flags, the entry points and the re-ranking refusal."""
import json
import os
import random

import numpy as np
import pytest

from retrieval_scaling_b200 import config as rcfg
from retrieval_scaling_b200 import search

from dedup_fixture import oracle_deduplicate, write_sources

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(listing, merged_path, n_docs=8, p=1, **extra):
    ov = [f"evaluation.search.paths_to_merge={listing}", f"evaluation.search.merged_path={merged_path}",
          f"evaluation.search.n_docs={n_docs}", f"evaluation.search.topk_subsample_p={p}",
          "evaluation.data.eval_data=unused.jsonl"] + [f"evaluation.search.{k}={v}" for k, v in extra.items()]
    return rcfg.load_config("default", os.path.join(ROOT, "ric", "conf"), ov)


def _lines(path):
    with open(path) as f:
        return [json.loads(x) for x in f]


def test_strip_quirk_of_the_merged_file_name():
    assert search.merged_before_dedup_path("/r/dedup_merged.jsonl") == "/r/merged.jsonl"
    assert search.merged_before_dedup_path("/r/dedup_dev.jsonl") == "/r/v.jsonl"
    assert search.merged_before_dedup_path("/r/pubmed") == "/r/bm"
    assert search.merged_before_dedup_path("/r/x.jsonl") == "/r/x.jsonl"


def test_merge_tags_domains_and_sorts_scores_as_stored(tmp_path):
    paths = []
    for dom, scores in (("wiki", ["9.5", "10.25", "1.0"]), ("c4", ["2", "9.5", "10.3"])):
        p = tmp_path / f"{dom}_datastore-256" / "r.jsonl"
        p.parent.mkdir()
        rows = [{"raw_query": "q0", "ctxs": [None]},
                {"raw_query": "q1", "ctxs": [{"retrieval text": f"{dom}{k}", "retrieval score": s, "source": None}
                                             for k, s in enumerate(scores)]}]
        p.write_text("".join(json.dumps(r) + "\n" for r in rows))
        paths.append(str(p))
    merged = search.merge_multi_domain(paths, 4)
    assert merged[0]["ctxs"] == []
    ctxs = merged[1]["ctxs"]
    # string order, descending and stable: "9.5" (wiki) before "9.5" (c4), then "2", "10.3" (a float sort would put
    # "10.3" and "10.25" first)
    assert [c["retrieval text"] for c in ctxs] == ["wiki0", "c41", "c40", "c42"]
    assert [c["source"] for c in ctxs] == ["wiki", "c4", "c4", "c4"]
    with pytest.raises(AssertionError):
        search.merge_multi_domain(paths, 7)              # fewer than n_docs passages


def test_end_to_end_files_and_subsampling(tmp_path):
    listing = write_sources(str(tmp_path), seed=3, n_queries=12, n_docs=8)
    out = tmp_path / "out"
    merged_path = str(out / "dedup_merged.jsonl")
    cfg = _cfg(listing, merged_path, p=0.5, subsample_seed=7)
    calls = []

    def dedup(examples):
        calls.append(len(examples))
        return oracle_deduplicate(examples)

    out_path = search.post_hoc_merge_topk_multi_domain(cfg, deduplicate=dedup)
    assert calls == [12]
    assert out_path == str(out / "full_subsampled_0.5_7_dedup_merged.jsonl")
    merged = _lines(str(out / "merged.jsonl"))
    deduped = _lines(merged_path)
    assert all(len(ex["ctxs"]) == 8 for ex in merged[1:])
    # the expected output, step by step: oracle de-duplication, coin flips, short-chunk removal
    expect = oracle_deduplicate(json.loads(json.dumps(merged)))
    assert deduped == expect
    random.seed(7)
    for ex in expect:
        ex["ctxs"] = [c for c in ex["ctxs"] if random.random() < 0.5]
        ex["ctxs"] = [c for c in ex["ctxs"] if len(c["retrieval text"].split(" ")) > 12]
    assert _lines(out_path) == expect
    assert all(c["quality score"] == 1 for ex in expect for c in ex["ctxs"])

    # p = 1 (an int in the config): no coin flips, the name keeps str(1)
    out1 = search.post_hoc_merge_topk_multi_domain(_cfg(listing, merged_path, p=1), deduplicate=oracle_deduplicate)
    assert os.path.basename(out1) == "full_subsampled_1_1000_dedup_merged.jsonl"
    assert _lines(out1) == [dict(ex, ctxs=[c for c in ex["ctxs"] if len(c["retrieval text"].split(" ")) > 12])
                            for ex in deduped]


def test_cached_files(tmp_path):
    listing = write_sources(str(tmp_path), seed=5, n_queries=6, n_docs=8)
    merged_path = str(tmp_path / "dedup_m.jsonl")
    search.post_hoc_merge_topk_multi_domain(_cfg(listing, merged_path), deduplicate=oracle_deduplicate)
    # an existing merged (pre-dedup) file is read instead of the sources
    pre = tmp_path / "m.jsonl"
    rows = _lines(str(pre))
    rows[1]["ctxs"] = rows[1]["ctxs"][:2]
    pre.write_text("".join(json.dumps(r) + "\n" for r in rows))
    search.post_hoc_merge_topk_multi_domain(_cfg(listing, merged_path), deduplicate=oracle_deduplicate)
    assert len(_lines(merged_path)[1]["ctxs"]) <= 2
    # use_saved_dedup_data: the de-duplicated file is reused, nothing is de-duplicated
    saved = _lines(merged_path)
    saved[2]["ctxs"] = []
    with open(merged_path, "w") as f:
        f.write("".join(json.dumps(r) + "\n" for r in saved))

    def no_dedup(examples):
        raise AssertionError("de-duplication must not run")

    out = search.post_hoc_merge_topk_multi_domain(_cfg(listing, merged_path, use_saved_dedup_data="true"),
                                                  deduplicate=no_dedup)
    assert _lines(out)[2]["ctxs"] == [] and _lines(merged_path) == saved


def test_rerank_is_refused(tmp_path):
    cfg = _cfg("x.txt", str(tmp_path / "dedup_m.jsonl"), rerank_method="lexical")
    with pytest.raises(NotImplementedError, match="answer"):
        search.post_hoc_merge_topk_multi_domain(cfg, deduplicate=oracle_deduplicate)


def test_entry_points_call_the_merge(tmp_path, monkeypatch):
    seen = []
    monkeypatch.setattr(search, "post_hoc_merge_topk_multi_domain", lambda cfg: seen.append("merge"))
    monkeypatch.setattr(search, "post_hoc_merge_topk", lambda cfg: seen.append("index-merge"))
    cfg = _cfg("x.txt", "m.jsonl", p=0.5, merge_multi_source_results="true")
    cfg.evaluation.eval_output_dir = str(tmp_path)
    cfg.datastore.domain = "wiki"
    os.makedirs(tmp_path / "0")
    (tmp_path / "0" / "unused_retrieved_results.jsonl").write_text("")
    search.search_dense_topk(cfg)                       # every result file exists: straight to the merge
    assert seen == ["merge"]
    import importlib.util
    spec = importlib.util.spec_from_file_location("main_ric", os.path.join(ROOT, "ric", "main_ric.py"))
    main_ric = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(main_ric)
    cfg.tasks.eval.merge_search = True
    main_ric.main(cfg)
    assert seen == ["merge", "merge"]


def test_dedup_batches_are_bounded_by_utf8_bytes(monkeypatch):
    """deduplicate splits consecutive queries into batches of at most batch_bytes bytes of UTF-8 (a larger query alone),
    and every slot reaches the device exactly once, in order."""
    from retrieval_scaling_b200 import dedup
    sizes, slots = [], []

    def fake_run(batch, device):
        sizes.append(len(batch.buf))
        slots.extend(bytes(batch.buf[a:b]).decode() for a, b in zip(batch.text_off[:-1], batch.text_off[1:]))
        return np.ones(len(batch.text_off) - 1, dtype=bool)

    monkeypatch.setattr(dedup, "run_batch", fake_run)
    data = [{"raw_query": f"q{i}", "ctxs": [{"retrieval text": "東京 " * (i % 5) * 40}]} for i in range(30)]
    dedup.deduplicate(data, batch_bytes=1000)
    per_query = [len(f"q{i}") + len(("東京 " * (i % 5) * 40).encode()) for i in range(30)]
    assert all(s <= 1000 or s in per_query for s in sizes) and sum(sizes) == sum(per_query)
    assert len(sizes) > 10
    assert slots == [t for i in range(30) for t in (f"q{i}", "東京 " * (i % 5) * 40)]
    assert all(ex["ctxs"][0]["quality score"] == 1 for ex in data)
