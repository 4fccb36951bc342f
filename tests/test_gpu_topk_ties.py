"""Exact top-k order: (score desc, docID asc) at EVERY rank, ties included (SURVEY.md 8 row 18, ref_harness.cpp:119).

The tie corpus makes the tie classes bit-identical on both sides: ten terms with the same document frequency and freq 1 contribute the
same float w each, so a document that matches m of them scores the same repeated sum of w whatever order the contributions arrive in
(k_score_flat adds them with CAS chains, in no fixed order).  A term with freq-0 postings adds a class at +0.0, which must rank below
every positive score.  The GPU's docIDs must equal lexsort((ids, -scores))[:k] of the reference's full stream at every rank; scores within
1e-5.  Covered: k_score_flat (LUCENE flat OR / single term, under the default knobs, every tile a run, and the 512-thread instantiation),
k_exec_tiles (GOOGLE OR / single term, LUCENE AND), MatchSome, k from 1 to kMaxK = 512, fewer and exactly k matches, masked documents in the
tie class at the cut, and 2 / 3 / 8 docID-range shards merged by trn_merge_topk."""
import os

import numpy as np
import pytest
import torch

import trinity_b200 as tb
from refharness import RefIndex
from trinity_b200.sharded import shard_range
from util import assert_topk_exact, merged_topk

pytestmark = pytest.mark.gpu

NDOCS = 300_000
DF = 30_000
KS = [1, 2, 31, 32, 33, 100, 511, 512]
TERMS = [f"t{i}" for i in range(1, 11)]
OR10 = " OR ".join(TERMS)
# query -> (LUCENE route, GOOGLE route); min_match for the MatchSome group
QUERIES = {
    OR10: (tb.ROUTE_SCORE_FLAT, tb.ROUTE_EXEC_TILES),
    "t1": (tb.ROUTE_SCORE_FLAT, tb.ROUTE_EXEC_TILES),
    "t1 OR t2 OR t3 OR zero": (tb.ROUTE_SCORE_FLAT, tb.ROUTE_EXEC_TILES),
    "t1 AND t2": (tb.ROUTE_EXEC_TILES, tb.ROUTE_EXEC_TILES),
    "(t1 OR t2 OR t3) AND (t4 OR t5 OR t6 OR zero)": (tb.ROUTE_EXEC_TILES, tb.ROUTE_EXEC_TILES),
    "[t1, t2, t3, t4, t5, t6]": (tb.ROUTE_EXEC_TILES, tb.ROUTE_EXEC_TILES),
    "few": (tb.ROUTE_SCORE_FLAT, tb.ROUTE_EXEC_TILES),           # 40 matches: fewer than most k
    "exact": (tb.ROUTE_SCORE_FLAT, tb.ROUTE_EXEC_TILES),         # exactly kMaxK matches
    "few OR zfew": (tb.ROUTE_SCORE_FLAT, tb.ROUTE_EXEC_TILES),   # fewer than k from k = 100 on, the +0.0 class behind the positives
}
MIN_MATCH = 2


def _lists():
    rng = np.random.default_rng(77)
    out = {n: np.sort(rng.choice(NDOCS, DF, replace=False).astype(np.uint32) + 1) for n in TERMS}
    out["zero"] = np.sort(rng.choice(NDOCS, 20_000, replace=False).astype(np.uint32) + 1)
    out["few"] = np.sort(rng.choice(NDOCS, 40, replace=False).astype(np.uint32) + 1)
    out["exact"] = np.sort(rng.choice(NDOCS, 512, replace=False).astype(np.uint32) + 1)
    # freq-0 postings: 30 documents of their own and 5 of `few` (those keep few's score)
    out["zfew"] = np.unique(np.concatenate([rng.choice(NDOCS, 30, replace=False).astype(np.uint32) + 1, out["few"][::8]]))
    return out


LISTS = _lists()
NAMES = list(LISTS)


def _freqs(n, d):
    return np.zeros(len(d), np.uint32) if n in ("zero", "zfew") else np.ones(len(d), np.uint32)


def _gpu(codec, lo=1, hi=NDOCS, env=None):
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        g = tb.GpuIndexSource(0)  # trn_create reads the knobs
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    b = tb.IndexBuilder(codec)
    for n in NAMES:
        d = LISTS[n]
        d = d[(d >= lo) & (d <= hi)]
        b.add_term(d, _freqs(n, d))
    g.upload(codec, b.index(), b.terms_array(), NDOCS)
    return g


class Ref:
    def __init__(self, ref, codec):
        self.r = RefIndex(ref, codec)
        for n in NAMES:
            self.r.add_term(n, LISTS[n], _freqs(n, LISTS[n]))
        self.r.finish(NDOCS)
        self.tdict = tb.TermDictionary(NAMES)
        self.cache = {}

    def exec(self, q):
        if q not in self.cache:
            some = q.startswith("[")
            self.cache[q] = self.r.exec(q, True, NDOCS + 1, parser_flags=16 if some else 0, min_match=MIN_MATCH if some else 0)
        return self.cache[q]

    def plan(self, q):
        """global BM25 weights (whole-collection df and docs_cnt): what every shard of a sharded collection uses"""
        nodes = tb.parse_query(q, self.tdict, min_match=MIN_MATCH if q.startswith("[") else None)
        for x in nodes:
            if x["kind"] == tb.NODE_TERM and x["term"] != tb.EMPTY_TERM:
                x["weight"] = tb.bm25_idf(len(LISTS[NAMES[x["term"]]]), NDOCS)
        return nodes


@pytest.fixture(scope="module", params=[tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
def corpus(request, ref):
    return request.param, Ref(ref, request.param)


def test_tie_corpus_has_the_classes_it_promises(corpus):
    codec, r = corpus
    wd, ws = r.exec(OR10)
    sc = np.unique(np.asarray(ws, np.float32))
    assert len(sc) >= 5 and len(ws) - len(sc) > 100_000  # a handful of classes (m = 1, 2, ... of the ten terms), each of many documents
    wd, ws = r.exec("t1 OR t2 OR t3 OR zero")
    assert np.count_nonzero(ws == 0) > 1000  # the +0.0 class
    assert len(r.exec("few")[0]) == 40 and len(r.exec("exact")[0]) == 512
    wd, ws = r.exec("few OR zfew")
    assert 60 < len(wd) < 100 and np.count_nonzero(ws == 0) >= 25 and np.count_nonzero(ws > 0) == 40  # the +0.0 class inside a top-100


KNOBS = {"default": None, "run_tiles_1": {"TRN_RUN_TILES": "1"}, "sf512": {"TRN_SF_THREADS": "512", "TRN_SCORED_SHIFT": "14"}}


@pytest.mark.parametrize("knobs", list(KNOBS))
def test_topk_strict_order(corpus, knobs):
    codec, r = corpus
    if codec == tb.CODEC_GOOGLE and knobs != "default":
        pytest.skip("the k_score_flat knobs do not apply to GOOGLE (k_exec_tiles)")
    g = _gpu(codec, env=KNOBS[knobs])
    qs = list(QUERIES)
    plans = [r.plan(q) for q in qs]
    exp = [QUERIES[q][0 if codec == tb.CODEC_LUCENE else 1] for q in qs]
    for k in KS:
        res = g.exec_batch(plans, tb.MODE_SCORED_TOPK, k=k)
        assert list(g.last_routes()) == exp, (k, list(g.last_routes()))
        for i, q in enumerate(qs):
            wd, ws = r.exec(q)
            assert int(res.match_counts[i]) == len(wd), f"[{q}] k={k} match count"
            gd, gs = res.query(i)
            assert_topk_exact(gd, gs, wd, ws, k, f"[{q}] k={k} {knobs}")
            # the device list of a query with fewer than k matches is padded with (docID 0, score -1.0)
            pd, ps = res.docids[i * k:(i + 1) * k], res.scores[i * k:(i + 1) * k]
            n = min(k, len(wd))
            assert np.all(pd[n:] == 0) and np.all(ps[n:] == -1.0), f"[{q}] k={k} padding"
            assert np.all(ps[:n] >= 0)
    g.close()


def test_k_out_of_range_is_refused(corpus):
    codec, r = corpus
    g = _gpu(codec)
    plans = [r.plan("t1")]
    buf = torch.zeros(1024, dtype=torch.int32, device="cuda")
    sbuf = torch.zeros(1024, dtype=torch.float32, device="cuda")
    for k in (0, 513):
        with pytest.raises(tb.TrinityError):
            g.exec_batch(plans, tb.MODE_SCORED_TOPK, k=k)
        with pytest.raises(tb.TrinityError):
            g.merge_topk(buf.data_ptr(), sbuf.data_ptr(), 1, 1, k, buf.data_ptr(), sbuf.data_ptr())
    g.close()


def test_masked_documents_in_the_tie_class_at_the_cut(corpus, ref):
    """mask part of the class that straddles rank k (and a few documents above it): the next docIDs of that class move up"""
    codec, r = corpus
    g = _gpu(codec)
    k = 100
    qs = [OR10, "t1 OR t2 OR t3 OR zero", "t1 AND t2"]
    masked = []
    for q in qs:
        wd, ws = r.exec(q)
        order = np.lexsort((wd, -np.asarray(ws, np.float32)))
        cut = np.asarray(ws, np.float32)[order[k - 1]]
        cls = wd[order][np.asarray(ws, np.float32)[order] == cut]
        masked += list(cls[::3][:40]) + list(wd[order][:5])
    masked = np.unique(np.array(masked, np.uint32))
    g.set_masked_documents(masked)
    res = g.exec_batch([r.plan(q) for q in qs], tb.MODE_SCORED_TOPK, k=k)
    for i, q in enumerate(qs):
        wd, ws = r.r.exec_masked(q, True, masked, NDOCS + 1)
        assert_topk_exact(*res.query(i), wd, ws, k, f"[{q}] masked")
    g.close()


@pytest.mark.parametrize("nshards", [2, 3, 8])
def test_sharded_merge_is_strict(corpus, nshards):
    codec, r = corpus
    gpus = [_gpu(codec, *shard_range(NDOCS, s, nshards)) for s in range(nshards)]
    qs = list(QUERIES)
    plans = [r.plan(q) for q in qs]
    for k in (1, 33, 512):
        got = merged_topk(gpus, plans, k)
        for i, q in enumerate(qs):
            wd, ws = r.exec(q)
            assert_topk_exact(*got[i], wd, ws, k, f"[{q}] {nshards} shards k={k}")
    for g in gpus:
        g.close()
