#!/usr/bin/env python
"""Golden of the reference's text-search path, so that the tests need no reference checkout.

    AUDIOMUSE_REFERENCE=<checkout of AudioMuse-AI> python tests/golden/make_text_search_golden.py
    # writes tests/golden/text_search_golden.npz and text_search_golden.json

Runs the reference's tasks.clap_analyzer.get_text_embedding (:577-628), get_text_embeddings_batch (:631-687) and
tasks.clap_text_search.search_by_text (:448-532) UNMODIFIED, with two substitutes installed in the module:

* ``_tokenizer``: StubTokenizer, a deterministic word-hash tokenizer with the call signature and output the
  reference uses (``max_length=77, padding='max_length', truncation=True, return_tensors='np'``; <s> = 0, pad = 1,
  </s> = 2);
* ``_text_session``: OracleSession, a seeded small text tower (oracle/clap_text.py, float64, output float32 as the
  ONNX session returns) behind the ORT session's ``run(None, feed)``.

The CLAP index is a recording brute-force index (tests/ref_harness.RecordingIndex) over ``library(embeddings)``:
for each query a ladder of rows at cosine distances 0.01, 0.0115, 0.013, ... (gaps of 1.5e-3) around its embedding,
every fourth row of a ladder by the same artist (so that MAX_SONGS_PER_ARTIST = 3 drops rows), plus random rows
(distance about 1).  The queries' embeddings are far apart, so another query's ladder stays beyond a ladder's last
row.  Over the prefix of each candidate list that search_by_text reads (up to its last kept row, and the next row),
adjacent distances differ by more than MIN_GAP, far above the error a device embedding within 1e-4 per component
can cause, so the ordered answer is fixed.  Records the feeds each call made, the session outputs, the three
functions' returns, every index query, the texts and the settings.  ``search_results`` restates search_by_text's
loop over an index answer (tests/test_text_search_golden_host.py pins it to the recorded returns), so that the
GPU replay can run the same walk over the device index without the reference.
"""
import json
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

GOLDEN = os.path.join(HERE, "text_search_golden.npz")
GOLDEN_JSON = os.path.join(HERE, "text_search_golden.json")
MODEL_SEED = 11
MODEL_STD = 0.3  # wide enough that the queries' embeddings are far apart (cosines <= 0.7)
LIBRARY_SEED = 5
N_RANDOM = 600
LADDER = 150
MIN_GAP = 1e-3
CAP = 3
QUERIES = [("upbeat summer songs", 20), ("calm piano for studying late at night", 50), ("heavy guitars", 100)]
BATCH = ["happy", "sad", "a very long description of energetic electronic dance music with a strong beat " * 3]


def model_config():
    from oracle import clap_text as ct

    return ct.small_config(heads=2, proj=512)


def make_model():
    from oracle import clap_text as ct

    return ct.TextCLAP(model_config(), "sdpa", "where").init_random(MODEL_SEED, std=MODEL_STD)


class StubTokenizer:
    """Deterministic stand-in for the RoBERTa tokenizer: lower-cased words hashed (crc32) into [3, vocab)."""

    def __init__(self, vocab: int, bos: int = 0, pad: int = 1, eos: int = 2):
        self.vocab, self.bos, self.pad, self.eos = vocab, bos, pad, eos

    def __call__(self, text, max_length=77, padding="max_length", truncation=True, return_tensors="np"):
        assert padding == "max_length" and truncation and return_tensors == "np"
        texts = [text] if isinstance(text, str) else list(text)
        ids = np.full((len(texts), max_length), self.pad, np.int64)
        mask = np.zeros((len(texts), max_length), np.int64)
        for r, t in enumerate(texts):
            toks = [3 + zlib.crc32(w.encode()) % (self.vocab - 3) for w in t.lower().split()]
            row = [self.bos] + toks[:max_length - 2] + [self.eos]
            ids[r, :len(row)] = row
            mask[r, :len(row)] = 1
        return {"input_ids": ids, "attention_mask": mask}


class OracleSession:
    """The ORT session's run(None, feed) over the float64 oracle; records every feed and output."""

    def __init__(self, model):
        self.model, self.calls = model, []

    def run(self, output_names, feed):
        from oracle import clap_text as ct

        out = ct.run(self.model, feed["input_ids"], feed["attention_mask"]).astype(np.float32)
        self.calls.append((np.array(feed["input_ids"]), np.array(feed["attention_mask"]), out.copy()))
        return [out]


def library(query_embeddings):
    """Rows (float32 [N, D]) and authors: a distance ladder around each query embedding, then random rows."""
    q = np.asarray(query_embeddings, np.float64)
    D = q.shape[1]
    rng = np.random.default_rng(LIBRARY_SEED)
    rows, authors = [], []
    for j, e in enumerate(q):
        e = e / np.linalg.norm(e)
        for r in range(LADDER):
            d = 0.01 + 0.0015 * r
            u = rng.standard_normal(D)
            u -= (u @ e) * e
            u /= np.linalg.norm(u)
            c = 1.0 - d
            rows.append(c * e + np.sqrt(1.0 - c * c) * u)
            authors.append(f"Ladder {j} Star" if r % 4 == 0 else f"Ladder {j} Artist {r}")
    for r in range(N_RANDOM):
        v = rng.standard_normal(D)
        rows.append(v / np.linalg.norm(v))
        authors.append(f"Random Artist {r % 40}")
    perm = rng.permutation(len(rows))
    return np.asarray(rows, np.float32)[perm], [authors[i] for i in perm]


def candidate_gap(rows, query, n):
    """Smallest gap between adjacent cosine distances (float64) among the n + 1 nearest rows."""
    x = rows.astype(np.float64)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    qn = np.asarray(query, np.float64) / np.linalg.norm(query)
    d = np.sort(1.0 - x @ qn)[:n + 1]
    return float(np.diff(d).min())


def read_prefix(ids, results):
    """How many candidates search_by_text read: up to and including its last kept row."""
    pos = {f"item{int(i)}": p for p, i in enumerate(ids)}
    return pos[results[-1]["item_id"]] + 1


def fetch_size(limit, cap):
    """search_by_text's k before min(k, len(index)) (clap_text_search.py:482-483)."""
    return (limit + max(20, limit * 4) + 1) if cap else limit


def search_results(ids, dists, authors, limit, cap):
    """search_by_text's walk (clap_text_search.py:499-524) over one index answer: item ids "item<id>", the artist
    cap on the stripped lower-cased author, similarity 1 - distance."""
    results, counts = [], {}
    for vid, dist in zip(ids, dists):
        if len(results) >= limit:
            break
        author = authors[int(vid)]
        if cap and author:
            a = author.strip().lower()
            if counts.get(a, 0) >= cap:
                continue
            counts[a] = counts.get(a, 0) + 1
        results.append({"item_id": f"item{int(vid)}", "title": f"Song {int(vid)}", "author": author,
                        "similarity": 1.0 - float(dist)})
    return results


def main():
    from tests import ref_harness as rh
    from tests.golden import make_ref_trace as mrt

    assert rh.available(), "set AUDIOMUSE_REFERENCE to a checkout of the reference"
    db = rh.FakeDB()
    ref = rh.load_reference(mrt.types_voyager(), db)
    cts, config = ref.cts, ref.config
    if "tasks.memory_utils" not in sys.modules:
        rh._stub("tasks.memory_utils", cleanup_cuda_memory=lambda *a, **k: None,
                 handle_onnx_memory_error=lambda *a, **k: None, comprehensive_memory_cleanup=lambda *a, **k: None)
    ca = rh._load("tasks.clap_analyzer", "tasks/clap_analyzer.py")
    config.CLAP_ENABLED = True
    config.MAX_SONGS_PER_ARTIST = CAP
    model = make_model()
    cfg = model_config()
    sess = OracleSession(model)
    ca._text_session, ca._tokenizer = sess, StubTokenizer(cfg.vocab, pad=cfg.pad_id)

    single = [ca.get_text_embedding(t) for t, _ in QUERIES]
    n_single = len(sess.calls)
    batch = ca.get_text_embeddings_batch(BATCH)
    assert all(s is not None for s in single) and batch is not None and len(sess.calls) == n_single + 1

    rows, authors = library(np.stack(single))
    crec = rh.RecordingIndex(rows)
    N = len(rows)
    db.score = {f"item{i}": {"item_id": f"item{i}", "title": f"Song {i}", "author": authors[i]} for i in range(N)}
    cts._CLAP_INDEX_CACHE.update(index=crec, id_map={i: f"item{i}" for i in range(N)},
                                 reverse_id_map={f"item{i}": i for i in range(N)}, loaded=True)
    cts.warmup_text_search_model = lambda *a, **k: None  # the idle-unload timer thread is not part of the answer
    cts._fetch_clap_metadata = lambda ids: {i: {"title": db.score[i]["title"], "author": db.score[i]["author"]}
                                            for i in ids if i in db.score}
    results, search_calls = [], []
    for text, limit in QUERIES:
        start_calls, start_trace = len(sess.calls), len(crec.trace)
        res = cts.search_by_text(text, limit=limit)
        assert len(res) == limit, (text, len(res))
        results.append(res)
        q = [c for c in crec.trace[start_trace:] if c["op"] == "query"]
        assert len(q) == 1 and len(sess.calls) == start_calls + 1
        search_calls.append(q[0])
        gap = candidate_gap(rows, q[0]["vector"], read_prefix(q[0]["ids"], res))
        assert gap > MIN_GAP, (text, gap)
        authors_kept = [r["author"] for r in res]
        assert max(authors_kept.count(a) for a in set(authors_kept)) == CAP  # the cap did drop rows

    out = {}
    for i, (ids, mask, emb) in enumerate(sess.calls):
        out[f"feed_ids_{i}"], out[f"feed_mask_{i}"], out[f"session_out_{i}"] = ids, mask, emb
    for i, s in enumerate(single):
        out[f"text_embedding_{i}"] = np.asarray(s, np.float32)
    out["batch_embeddings"] = np.asarray(batch, np.float32)
    for i, c in enumerate(search_calls):
        out[f"query_vec_{i}"], out[f"query_ids_{i}"], out[f"query_dist_{i}"] = c["vector"], c["ids"], c["dist"]
    np.savez_compressed(GOLDEN, **out)
    meta = {"model": {"config": dict(cfg.__dict__), "attention": "sdpa", "mask": "where", "seed": MODEL_SEED},
            "queries": [{"text": t, "limit": lim, "k": int(c["k"]), "results": r}
                        for (t, lim), c, r in zip(QUERIES, search_calls, results)],
            "batch_texts": BATCH, "n_session_calls": len(sess.calls), "single_calls": n_single,
            "max_songs_per_artist": CAP, "library": {"rows": N, "seed": LIBRARY_SEED, "ladder": LADDER,
                                                     "random": N_RANDOM, "min_gap": MIN_GAP},
            "authors": authors}
    with open(GOLDEN_JSON, "w") as f:
        json.dump(meta, f, indent=1)
    print(f"{len(sess.calls)} session calls, {len(search_calls)} searches; results:", [len(r) for r in results])


if __name__ == "__main__":
    main()
