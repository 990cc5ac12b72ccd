"""GPU replay of the text-search golden (tests/golden/make_text_search_golden.py): the feeds the reference's
get_text_embedding, get_text_embeddings_batch and search_by_text sent to their text session go through
B200TextSession, and each search's query -- the reference's renormalised embedding -- goes to the device index
(voyager_compat.Index) with search_by_text's k; search_by_text's walk (search_results, pinned to the reference by
tests/test_text_search_golden_host.py) must then give the recorded ordered ids, authors and artist cap."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from audiomuse_ai_b200 import voyager_compat as vc
from audiomuse_ai_b200.clap_analyzer import B200TextSession
from oracle import clap_text as ct
from tests.golden import make_text_search_golden as gen

MAX_ABS, MIN_COS = 1e-4, 0.99999


def test_replay_text_search_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "text_search_golden.npz"))
    with open(os.path.join(golden_dir, "text_search_golden.json")) as f:
        meta = json.load(f)
    sess = B200TextSession(blob=ct.export_onnx_bytes(gen.make_model()))
    try:
        outs = []
        for i in range(meta["n_session_calls"]):
            feed = {"input_ids": g[f"feed_ids_{i}"], "attention_mask": g[f"feed_mask_{i}"]}
            got = sess.run(None, feed)[0]
            want = g[f"session_out_{i}"]
            err = float(np.abs(got - want).max())
            cos = float((np.sum(got * want, 1) / np.linalg.norm(got, axis=1) / np.linalg.norm(want, axis=1)).min())
            print(f"session call {i} (B = {got.shape[0]}): max |delta| {err:.3g}, min cosine {cos:.9f}")
            assert err <= MAX_ABS and cos >= MIN_COS
            outs.append(got)
        b = outs[meta["single_calls"]]
        np.testing.assert_allclose(b / np.linalg.norm(b, axis=1, keepdims=True), g["batch_embeddings"], atol=MAX_ABS)
    finally:
        sess.close()

    rows, authors = gen.library(np.stack([g[f"text_embedding_{i}"] for i in range(3)]))
    index = vc.Index(vc.Space.Cosine, num_dimensions=rows.shape[1], M=64, ef_construction=1024)
    index.add_items(rows, ids=np.arange(len(rows)))
    cap = meta["max_songs_per_artist"]
    for i, q in enumerate(meta["queries"]):
        o = outs[meta["single_calls"] + 1 + i][0]
        emb = o / np.linalg.norm(o)  # get_text_embedding's renormalisation
        np.testing.assert_allclose(emb, g[f"text_embedding_{i}"], atol=MAX_ABS)
        ids, dist = index.query(emb, k=min(gen.fetch_size(q["limit"], cap), len(index)))
        got = gen.search_results(ids, dist, authors, q["limit"], cap)
        assert [r["item_id"] for r in got] == [r["item_id"] for r in q["results"]], q["text"]
        assert [r["author"] for r in got] == [r["author"] for r in q["results"]]
        np.testing.assert_allclose([r["similarity"] for r in got], [r["similarity"] for r in q["results"]],
                                   rtol=0, atol=1e-3)
        kept = [r["author"] for r in got]
        assert max(kept.count(a) for a in set(kept)) == cap
