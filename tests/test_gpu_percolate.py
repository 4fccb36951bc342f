"""Percolator on the device (trn_percolator_register / trn_percolate) against the reference's own percolator_query::match."""
import numpy as np
import pytest

import trinity_b200 as tb
from percutil import EMPTY, EXTRA_SHAPES, VOCAB, RefPercolator, evaluate, query_lists, random_docs
from test_percolate_cpu import TD, _tree, edge_docs, parse
from util import Pair, assert_same_docs, closed_form_lists

pytestmark = pytest.mark.gpu

SHAPES = query_lists() + EXTRA_SHAPES


def assert_same(res, want, what=""):
    assert len(res) == len(want)
    for d, w in enumerate(want):
        got = res.document(d)
        assert np.array_equal(got, np.asarray(w, np.uint32)), (what, d, got[:10], np.asarray(w)[:10])


@pytest.fixture(scope="module")
def perc():
    return tb.Percolator([parse(q, m) for q, _, m in SHAPES], nterms=len(VOCAB))


@pytest.fixture(scope="module")
def docs():
    rng = np.random.default_rng(17)
    return edge_docs() + random_docs(rng, 600, max_len=40) + random_docs(rng, 60, max_len=2000) + random_docs(rng, 200, vocab=6, max_len=8, oov=0.3)


def test_device_equals_reference(perc, docs):
    want = RefPercolator(SHAPES).run(docs)
    res = perc.percolate(docs)
    assert_same(res, want)
    assert res.long_docs > 0 and res.total == sum(len(w) for w in want)
    info = perc.info()
    assert info["nqueries"] == len(SHAPES) and info["never"] > 0 and info["unanchored"] == 0
    assert 0 < res.candidates <= len(docs) * len(SHAPES)
    t = perc.last_timings()
    assert t["count_ms"] > 0 and t["write_ms"] > 0 and t["total_ms"] > 0


def test_one_batch_one_by_one_and_shuffled_agree(perc, docs):
    whole = perc.percolate(docs)
    base = [whole.document(d).copy() for d in range(len(docs))]
    for d in range(0, len(docs), 37):
        assert np.array_equal(perc.percolate([docs[d]]).document(0), base[d])
    rng = np.random.default_rng(2)
    for _ in range(3):
        order = rng.permutation(len(docs))
        r = perc.percolate([docs[i] for i in order])
        for j, i in enumerate(order):
            assert np.array_equal(r.document(j), base[i])


def test_document_lengths_and_refusal():
    # "w1 w2" anchored on w1; t1 anchors; a document of 1, 16383 and 16384 tokens
    qs = [parse('"w1 w2"', 0), parse("t1", 0), parse('"w2 w1" AND t3', 0)]
    p = tb.Percolator(qs, nterms=len(VOCAB))
    w1, w2, t1, t3 = (TD.term_id(x) for x in ("w1", "w2", "t1", "t3"))
    one = np.array([t1], np.uint32)
    big = np.full(16383, EMPTY, np.uint32)
    big[-2:] = [w1, w2]  # the phrase at the last position
    big[0] = t3
    big[5000:5002] = [w2, w1]
    r = p.percolate([one, big, np.zeros(0, np.uint32)])
    assert r.document(0).tolist() == [1] and r.document(1).tolist() == [0, 2] and r.document(2).tolist() == [] and r.long_docs == 1
    want = RefPercolator([('"w1 w2"', 0, 0), ("t1", 0, 0), ('"w2 w1" AND t3', 0, 0)]).run([one, big])
    assert [list(x) for x in want] == [[1], [0, 2]]
    with pytest.raises(tb.TrinityError, match="rc=-1: .*document 1"):
        p.percolate([one, np.zeros(16384, np.uint32)])
    with pytest.raises(tb.TrinityError, match="rc=-1: .*document 0"):
        p.percolate([np.array([len(VOCAB)], np.uint32)])


def test_many_distinct_terms_in_one_long_document():
    rng = np.random.default_rng(4)
    V = 40_000
    qs = [_tree((tb.NODE_TERM, 0, 0, int(t))) for t in rng.choice(V, 3000, replace=False)]
    qs += [_tree((tb.NODE_PHRASE, 2, 1, 0), (tb.NODE_TERM, 0, 0, int(a)), (tb.NODE_TERM, 0, 0, int(b))) for a, b in rng.integers(0, V, (2000, 2))]
    doc = rng.permutation(V)[:16383].astype(np.uint32)
    p = tb.Percolator(qs, nterms=V)
    r = p.percolate([doc, doc[:700], doc[:300]])
    for d, x in enumerate([doc, doc[:700], doc[:300]]):
        want = [q for q, n in enumerate(qs) if evaluate(n, x)]
        assert r.document(d).tolist() == want


def test_term_anchoring_100000_queries_and_the_dense_layout():
    """100000 queries anchored on one term: a document holding it matches most of them (ids emitted from the bitmap), one without
    matches few (sorted in shared memory)"""
    rng = np.random.default_rng(5)
    t1, t2 = TD.term_id("t1"), TD.term_id("t2")
    qs = []
    for i in range(100_000):
        if i % 10 == 3:
            qs.append(_tree((tb.NODE_AND, 2, 1, 0), (tb.NODE_TERM, 0, 0, t1), (tb.NODE_TERM, 0, 0, t2)))
        else:
            qs.append(_tree((tb.NODE_TERM, 0, 0, t1)))
    cost = np.ones(len(VOCAB), np.uint32)
    cost[t2] = 5  # t1 anchors every query
    p = tb.Percolator(qs, nterms=len(VOCAB), term_cost=cost)
    assert p.info()["anchor_entries"] == 100_000
    d_all = np.array([t1, t2], np.uint32)
    d_most = np.array([t1], np.uint32)
    d_none = np.array([t2, EMPTY], np.uint32)
    r = p.percolate([d_all, d_most, d_none] + random_docs(rng, 50, max_len=20))
    assert r.dense_docs >= 2
    assert r.document(0).tolist() == list(range(100_000))
    assert r.document(1).tolist() == [i for i in range(100_000) if i % 10 != 3]
    assert r.document(2).tolist() == []
    # a registry of 1 query, and sparse documents around a dense one
    p1 = tb.Percolator([qs[3]], nterms=len(VOCAB))
    assert [p1.percolate([d_all, d_most]).document(d).tolist() for d in (0, 1)] == [[0], []]


def test_large_registry_equals_reference():
    """>= 10^5 registered queries drawn from every shape, against the reference on a prefix of documents"""
    rng = np.random.default_rng(6)
    pick = rng.integers(0, len(SHAPES), 100_000)
    texts = [SHAPES[i] for i in pick]
    trees = [parse(q, m) for q, _, m in SHAPES]
    p = tb.Percolator([trees[i] for i in pick], nterms=len(VOCAB))
    docs = random_docs(rng, 40, max_len=30)
    r = p.percolate(docs)
    assert r.dense_docs > 0  # short documents of common terms match thousands of queries
    want = RefPercolator(texts).run(docs)
    assert_same(r, want, "large registry")


def test_reregister_state_and_an_index_on_the_same_context(ref):
    ndocs = 20_000
    pair = Pair(ref, tb.CODEC_GOOGLE, closed_form_lists(ndocs), ndocs)
    g = pair.gpu
    q = "t1 AND t2"
    before = g.exec_batch([pair.plan(q)], tb.MODE_DOCS_ONLY).query(0)[0].copy()
    with pytest.raises(tb.TrinityError, match="rc=-4"):
        g.percolate([np.zeros(3, np.uint32)])
    p = tb.Percolator([parse("t1", 0)], nterms=len(VOCAB), source=g)
    t1, t2 = TD.term_id("t1"), TD.term_id("t2")
    assert p.percolate([np.array([t1], np.uint32)]).document(0).tolist() == [0]
    p2 = tb.Percolator([parse("t2", 0), parse("t1 OR t2", 0)], nterms=len(VOCAB), source=g)  # replaces the set
    r = p2.percolate([np.array([t1], np.uint32), np.array([t2], np.uint32)])
    assert r.document(0).tolist() == [1] and r.document(1).tolist() == [0, 1]
    after = g.exec_batch([pair.plan(q)], tb.MODE_DOCS_ONLY).query(0)[0]
    assert_same_docs(after, before, "exec_batch next to a registry")
    want, _ = pair.ref.exec(q, False, ndocs)
    assert_same_docs(after, want, "exec_batch vs reference")
    # refusals of the registration leave the registered set in place
    for bad, rc in ((_tree((tb.NODE_TERM, 0, 0, len(VOCAB))), -1), (_tree((tb.NODE_OR, 65, 1, 0), *[(tb.NODE_TERM, 0, 0, 1)] * 65), -7),
                    (_tree((tb.NODE_PHRASE, 17, 1, 0), *[(tb.NODE_TERM, 0, 0, 1)] * 17), -1)):
        with pytest.raises(tb.TrinityError, match=f"rc={rc}: .*query 0"):
            g.percolator_register([bad], len(VOCAB))
    r = g.percolate([np.array([t1], np.uint32)])
    assert r.document(0).tolist() == [1]
    g.close()
