"""Host replay of the text-search golden (tests/golden/make_text_search_golden.py): the reference's
get_text_embedding, get_text_embeddings_batch and search_by_text, run with a stub tokenizer and the float64 oracle as
the text session.  Checks, without a GPU, that the recorded feeds are what the stub tokenizer makes (shape [B, 77],
int64), that the oracle reproduces the recorded session outputs, that the reference's renormalisation gives the
recorded embeddings, and that search_results -- the restatement of search_by_text's walk the GPU replay uses --
gives the reference's recorded answers, artist cap included, over a brute-force search of the regenerated library."""
import json
import os

import numpy as np
import pytest

from oracle import clap_text as ct
from oracle import knn as oknn
from tests.golden import make_text_search_golden as gen


@pytest.fixture(scope="module")
def golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "text_search_golden.npz"))
    with open(os.path.join(golden_dir, "text_search_golden.json")) as f:
        return g, json.load(f)


def test_feeds_are_the_stub_tokenizers(golden):
    g, meta = golden
    tok = gen.StubTokenizer(meta["model"]["config"]["vocab"], pad=meta["model"]["config"]["pad_id"])
    texts = [q["text"] for q in meta["queries"]]
    feeds = [tok(t, max_length=77) for t in texts] + [tok(meta["batch_texts"], max_length=77)]
    # three get_text_embedding calls, the batch, then one call per search_by_text
    order = feeds[:3] + [feeds[3]] + feeds[:3]
    assert meta["n_session_calls"] == len(order) == 7 and meta["single_calls"] == 3
    for i, f in enumerate(order):
        ids, mask = g[f"feed_ids_{i}"], g[f"feed_mask_{i}"]
        assert ids.dtype == np.int64 and mask.dtype == np.int64 and ids.shape[1] == 77
        np.testing.assert_array_equal(ids, f["input_ids"])
        np.testing.assert_array_equal(mask, f["attention_mask"])


def test_oracle_reproduces_the_session_outputs_and_embeddings(golden):
    g, meta = golden
    assert meta["model"]["config"] == dict(gen.model_config().__dict__)
    model = gen.make_model()
    for i in range(meta["n_session_calls"]):
        out = ct.run(model, g[f"feed_ids_{i}"], g[f"feed_mask_{i}"]).astype(np.float32)
        np.testing.assert_allclose(out, g[f"session_out_{i}"], rtol=0, atol=1e-7)
    for i in range(3):
        o = g[f"session_out_{i}"][0]
        np.testing.assert_allclose(g[f"text_embedding_{i}"], o / np.linalg.norm(o), rtol=0, atol=1e-7)
    b = g["session_out_3"]
    np.testing.assert_allclose(g["batch_embeddings"], b / np.linalg.norm(b, axis=1, keepdims=True), rtol=0, atol=1e-7)


def test_search_results_restate_search_by_text(golden):
    g, meta = golden
    rows, authors = gen.library(np.stack([g[f"text_embedding_{i}"] for i in range(3)]))
    assert authors == meta["authors"]
    x = oknn.normalize_rows(rows)
    cap = meta["max_songs_per_artist"]
    for i, q in enumerate(meta["queries"]):
        vec = g[f"query_vec_{i}"]
        np.testing.assert_array_equal(vec, g[f"text_embedding_{i}"])
        k = min(gen.fetch_size(q["limit"], cap), len(rows))
        assert k == q["k"]
        ids, dist = oknn.topk(x, vec[np.newaxis, :].astype(np.float32), k)
        np.testing.assert_array_equal(ids[0], g[f"query_ids_{i}"])
        got = gen.search_results(ids[0], dist[0], authors, q["limit"], cap)
        assert [r["item_id"] for r in got] == [r["item_id"] for r in q["results"]]
        assert [r["author"] for r in got] == [r["author"] for r in q["results"]]
        np.testing.assert_allclose([r["similarity"] for r in got], [r["similarity"] for r in q["results"]],
                                   rtol=0, atol=1e-6)
        kept = [r["author"] for r in got]
        assert max(kept.count(a) for a in set(kept)) == cap
        assert gen.candidate_gap(rows, vec, gen.read_prefix(ids[0], got)) > gen.MIN_GAP
