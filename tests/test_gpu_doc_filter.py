"""Per-query document filters (trn_docset_create / trn_exec_batch_filtered): the IndexDocumentsFilter of exec_query (exec.cpp:914-932,
1000-1027, 1096-1425) as allow and deny docID sets, on every route and mode, against the reference.

A query ignores d iff masked(d) || (allow && d not in allow) || (deny && d in deny).  The reference's own masked_documents_registry holding
the masked documents plus every document the filter drops is that predicate exactly, so the oracle is the reference's exec_query with
that registry (exec_masked)."""
import numpy as np
import pytest

import trinity_b200 as tb
from util import Pair, assert_close_scores, assert_same_docs, assert_topk_equal, closed_form_lists

pytestmark = pytest.mark.gpu
NDOCS = 300_000
QUERIES = ["t1 AND t2", "t3 OR t7 OR t9", "t1 AND (t2 OR t3) NOT t5", "t10", "(t1 AND t2) OR (t3 AND t4)", "t2 AND t3 AND t5"]


def ignored(allow, deny, ndocs=NDOCS):
    """the documents a filter drops, ascending"""
    out = np.zeros(0, np.uint32)
    if allow is not None:
        keep = np.zeros(ndocs + 1, bool)
        a = np.asarray(allow, np.int64)
        keep[a[(a >= 1) & (a <= ndocs)]] = True
        out = np.flatnonzero(~keep[1:]).astype(np.uint32) + 1
    if deny is not None:
        out = np.union1d(out, np.asarray(deny, np.uint32)[np.asarray(deny) <= ndocs]).astype(np.uint32)
    return out


def set_shapes(rng):
    """(name, allow, deny): the shapes every mode is checked on"""
    edges = np.array([1, 8191, 8192, 8193, 16383, 16384, 16385, 131071, 131072, 131073, 262143, 262144, NDOCS - 1, NDOCS], np.uint32)
    return [
        ("none", None, None),
        ("allow-1%", np.unique(rng.integers(1, NDOCS + 1, NDOCS // 100)), None),
        ("allow-50%", np.unique(rng.integers(1, NDOCS + 1, NDOCS // 2)), None),
        ("allow-99%", np.setdiff1d(np.arange(1, NDOCS + 1), rng.integers(1, NDOCS + 1, NDOCS // 100)), None),
        ("allow-edges", edges, None),
        ("allow-1-only", np.array([1], np.uint32), None),
        ("allow-empty", np.zeros(0, np.uint32), None),
        ("allow-all-and-above", np.arange(1, NDOCS + 1000), None),
        ("deny-empty", None, np.zeros(0, np.uint32)),
        ("deny-50%", None, np.unique(rng.integers(1, NDOCS + 1, NDOCS // 2))),
        ("deny-edges", None, edges),
        ("allow+deny", np.unique(rng.integers(1, NDOCS + 1, NDOCS // 3)), np.arange(6, NDOCS + 1, 6)),
    ]


def _filters(p, shapes):
    sets = {}

    def ds(a):
        if a is None:
            return None
        key = a.tobytes()
        if key not in sets:
            sets[key] = p.gpu.docset(a)
        return sets[key]

    return [None if a is None and d is None else tb.DocFilter(ds(a), ds(d)) for _, a, d in shapes]


def _check_batch(p, queries, shapes, masked, modes, k=50):
    """every (query, filter shape) pair in one batch per mode; unfiltered entries give the unfiltered batch's documents and counts"""
    flt = _filters(p, shapes)
    pairs = [(q, s) for q in queries for s in range(len(shapes))]
    routes = set()
    for mode in modes:
        scored = mode in (tb.MODE_SCORED_ALL, tb.MODE_SCORED_TOPK)
        plans = [p.plan(q, scored=scored) for q, _ in pairs]
        res = p.gpu.exec_batch(plans, mode, k=k, filters=[flt[s] for _, s in pairs])
        routes |= set(int(x) for x in p.gpu.last_routes())
        plain = p.gpu.exec_batch(plans, mode, k=k)
        for i, (q, s) in enumerate(pairs):
            name, a, d = shapes[s]
            what = f"[{q}] {name} mode {mode}"
            ign = np.union1d(masked, ignored(a, d)).astype(np.uint32)
            wd, ws = p.ref.exec_masked(q, scored, ign, NDOCS + 1)
            gd, gs = res.query(i)
            if flt[s] is None:
                pd, ps = plain.query(i)
                assert np.array_equal(gd, pd), what + ": unfiltered query differs from the unfiltered batch"
                if scored:  # (k_score_flat adds a tile's scores with float atomics: the last bit may differ between any two runs)
                    assert_close_scores(gs, ps, what + ": unfiltered query's scores")
                assert int(res.match_counts[i]) == int(plain.match_counts[i]), what
            assert int(res.match_counts[i]) == len(wd), what + f": match_counts {int(res.match_counts[i])} != {len(wd)}"
            if mode == tb.MODE_SCORED_TOPK:
                assert_topk_equal(gd, gs, wd, ws, k, what)
            else:
                assert_same_docs(gd, wd, what)
                if scored:
                    assert_close_scores(gs, ws, what)
    return routes


@pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
def test_filters_every_mode_match_reference(ref, codec):
    p = Pair(ref, codec, closed_form_lists(NDOCS), NDOCS)
    rng = np.random.default_rng(11)
    masked = np.unique(np.concatenate([rng.integers(1, NDOCS + 1, 5000), [8192, 131072]])).astype(np.uint32)
    p.gpu.set_masked_documents(masked)
    shapes = set_shapes(rng)
    routes = _check_batch(p, QUERIES, shapes, masked, [tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT, tb.MODE_SCORED_ALL, tb.MODE_SCORED_TOPK])
    if codec == tb.CODEC_GOOGLE:
        assert {tb.ROUTE_FLAT_AND, tb.ROUTE_FLAT_OR, tb.ROUTE_FLAT_TREE, tb.ROUTE_EXEC_TILES} <= routes, routes
    else:
        assert {tb.ROUTE_STEPS, tb.ROUTE_SCORE_FLAT, tb.ROUTE_EXEC_TILES} <= routes, routes
    p.gpu.close()


def test_filters_candidate_route(ref, monkeypatch):
    monkeypatch.setenv("TRN_CAND_COST", "1")  # read when the context is created
    p = Pair(ref, tb.CODEC_GOOGLE, closed_form_lists(NDOCS), NDOCS)
    rng = np.random.default_rng(12)
    shapes = set_shapes(rng)
    routes = _check_batch(p, ["t3 AND t7", "t1 AND (t2 OR t3) NOT t5", "t9 AND t4 AND t2"], shapes, np.zeros(0, np.uint32), [tb.MODE_DOCS_ONLY])
    assert tb.ROUTE_CANDIDATE in routes
    p.gpu.close()


def test_filters_top_k_deny_best_and_ties(ref):
    p = Pair(ref, tb.CODEC_LUCENE, closed_form_lists(NDOCS), NDOCS)
    for q in ("t1 OR t2", "t1 AND t2"):
        for k in (1, 100, 512):
            plan = p.plan(q, scored=True)
            wd, ws = p.ref.exec(q, True, NDOCS + 1)
            best = wd[np.argsort(-ws, kind="stable")[:k]]
            f = tb.DocFilter(deny=p.gpu.docset(best))
            res = p.gpu.exec_batch([plan, plan], tb.MODE_SCORED_TOPK, k=k, filters=[f, None])
            fd, fs = p.ref.exec_masked(q, True, np.sort(best), NDOCS + 1)
            gd, gs = res.query(0)
            assert not np.isin(gd, best).any()
            assert_topk_equal(gd, gs, fd, fs, k, f"[{q}] k={k} deny the best")
            assert int(res.match_counts[0]) == len(fd) == len(wd) - len(best)
            assert_topk_equal(*res.query(1), wd, ws, k, f"[{q}] k={k} unfiltered beside")


def test_filters_matched_terms(ref):
    p = Pair(ref, tb.CODEC_GOOGLE, closed_form_lists(NDOCS), NDOCS)
    rng = np.random.default_rng(13)
    allow = np.unique(rng.integers(1, NDOCS + 1, NDOCS // 10))
    deny = np.arange(10, NDOCS + 1, 10)
    plans = [p.plan(q) for q in QUERIES]
    flt = [tb.DocFilter(p.gpu.docset(allow), p.gpu.docset(deny))] * len(QUERIES)
    got = p.gpu.exec_matches(plans, filters=flt)
    plain = p.gpu.exec_matches(plans)
    for i, q in enumerate(QUERIES):
        keep = np.isin(plain.query(i), allow) & ~np.isin(plain.query(i), deny)
        assert np.array_equal(got.query(i), plain.query(i)[keep]), q
        # every kept match reports what the unfiltered run reports for it (true freqs and hits, also for one-term queries)
        kept = set(got.query(i).tolist())
        pm = {d: t for d, t in plain.matches(i) if d in kept}
        for d, terms in got.matches(i):
            assert [(t, f, list(h)) for t, f, h, _, _ in terms] == [(t, f, list(h)) for t, f, h, _, _ in pm[d]], (q, d)


def test_filters_pipelined_and_device_batch(ref, monkeypatch):
    monkeypatch.setenv("TRN_CHUNK_POSTINGS", "20000")  # small chunks: the host-buffer call pipelines (read at context creation)
    p = Pair(ref, tb.CODEC_GOOGLE, closed_form_lists(NDOCS), NDOCS)
    rng = np.random.default_rng(14)
    allow = np.unique(rng.integers(1, NDOCS + 1, NDOCS // 4))
    shared = p.gpu.docset(allow)  # one set, many queries
    qs = QUERIES * 16  # enough queries for several launches
    flt = [tb.DocFilter(allow=shared) if i % 3 else None for i in range(len(qs))]
    plans = [p.plan(q) for q in qs]
    res = p.gpu.exec_batch(plans, tb.MODE_DOCS_ONLY, filters=flt)
    assert p.gpu.last_timings()["chunks"] > 1
    plain = p.gpu.exec_batch(plans, tb.MODE_DOCS_ONLY)
    p.gpu.exec_batch_device(plans, tb.MODE_DOCS_ONLY, filters=flt)
    dev = p.gpu.fetch()
    for i, q in enumerate(qs):
        pd = plain.query(i)[0]
        want = pd if flt[i] is None else pd[np.isin(pd, allow)]
        assert np.array_equal(res.query(i)[0], want), (i, q)
        assert np.array_equal(dev.query(i)[0], want), (i, q)
        assert int(res.match_counts[i]) == int(dev.match_counts[i]) == len(want), (i, q)


def test_filters_lifecycle(ref, monkeypatch):
    monkeypatch.setenv("TRN_DOCSET_MAX", "3")  # read when the context is created
    p = Pair(ref, tb.CODEC_GOOGLE, closed_form_lists(NDOCS), NDOCS)
    plan = [p.plan("t1 AND t2")]
    want = p.ref.exec("t1 AND t2", False, NDOCS + 1)[0]
    with pytest.raises(tb.TrinityError, match="rc=-1"):
        p.gpu.docset([5, 0, 7])  # docID 0 is not a document
    a = p.gpu.docset(np.arange(1, 1000))
    b = p.gpu.docset([2, 4])
    c = p.gpu.docset([])
    with pytest.raises(tb.TrinityError, match="rc=-6"):
        p.gpu.docset([3])  # the context holds TRN_DOCSET_MAX sets
    res = p.gpu.exec_batch(plan, tb.MODE_DOCS_ONLY, filters=[tb.DocFilter(allow=a)])
    assert_same_docs(res.query(0)[0], want[want < 1000], "after the capacity refusal")
    res = p.gpu.exec_batch(plan, tb.MODE_DOCS_ONLY, filters=[tb.DocFilter(allow=c)])
    assert len(res.query(0)[0]) == 0 and int(res.match_counts[0]) == 0
    destroyed = tb.DocSet(p.gpu, b.handle, 0)
    b.close()
    with pytest.raises(tb.TrinityError, match="rc=-1"):
        p.gpu.exec_batch(plan, tb.MODE_DOCS_ONLY, filters=[tb.DocFilter(deny=destroyed)])
    res = p.gpu.exec_batch(plan, tb.MODE_DOCS_ONLY, filters=[tb.DocFilter(deny=a)])
    assert_same_docs(res.query(0)[0], want[want >= 1000], "after a destroyed handle")
    # a new upload invalidates every handle
    p.gpu.upload(p.codec, p.index, p.terms, NDOCS)
    with pytest.raises(tb.TrinityError, match="rc=-4"):
        p.gpu.exec_batch(plan, tb.MODE_DOCS_ONLY, filters=[tb.DocFilter(allow=a)])
    with pytest.raises(tb.TrinityError, match="rc=-4"):
        a.close()
    d = p.gpu.docset(np.arange(500, 2000))
    res = p.gpu.exec_batch(plan, tb.MODE_DOCS_ONLY, filters=[tb.DocFilter(allow=d)])
    assert_same_docs(res.query(0)[0], want[(want >= 500) & (want < 2000)], "after a re-upload")
    assert_same_docs(p.gpu.exec_batch(plan, tb.MODE_DOCS_ONLY).query(0)[0], want, "unfiltered after a re-upload")
    p.gpu.close()
