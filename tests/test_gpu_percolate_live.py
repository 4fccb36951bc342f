"""Percolator updates on the device (trn_percolator_add / trn_percolator_remove): after any sequence of registrations, adds and removes the
registry answers what a fresh registration of the live queries answers (ids mapped), and what the reference's own percolator_query::match
answers over the live query texts; the resident anchor index equals the one built in numpy from the registration planner over every issued
tree minus the removed ones; refusals change nothing."""
import ctypes as C

import numpy as np
import pytest

import trinity_b200 as tb
from percutil import EXTRA_SHAPES, VOCAB, RefPercolator, evaluate, query_lists, random_docs
from test_percolate_cpu import TD, _tree, parse
from trinity_b200._ffi import TrnPercolation
from util import Pair, assert_same_docs, closed_form_lists

pytestmark = pytest.mark.gpu

SHAPES = query_lists() + EXTRA_SHAPES
V = len(VOCAB)


@pytest.fixture(scope="module")
def shape_trees():
    return [parse(q, m) for q, _, m in SHAPES]


@pytest.fixture(scope="module")
def docs():
    rng = np.random.default_rng(23)
    return random_docs(rng, 300, max_len=40) + random_docs(rng, 20, max_len=1500) + random_docs(rng, 80, vocab=6, max_len=8, oov=0.3)


def expected_registry(trees, removed, nterms, cost=None):
    """(csr_off, csr[n, 2], unanchored) of a fresh registration of every tree (id = index) with the removed ids' entries dropped"""
    plan = tb.debug_percolator_plan(trees, nterms, cost)
    per_term = [[] for _ in range(nterms)]
    un = []
    for q, (status, cov) in enumerate(plan):
        if q in removed:
            continue
        if status == 1:
            un.append(q)
        for j, t in enumerate(cov):
            per_term[t].append((q, j))
    off = np.zeros(nterms + 1, np.uint32)
    off[1:] = np.cumsum([len(x) for x in per_term])
    csr = np.array([e for x in per_term for e in x], np.uint32).reshape(-1, 2)
    return off, csr, np.array(un, np.uint32)


def assert_registry(src, trees, removed, nterms, cost=None):
    off, csr, un = src.debug_percolator_registry()
    w_off, w_csr, w_un = expected_registry(trees, removed, nterms, cost)
    assert np.array_equal(off, w_off)
    assert np.array_equal(csr, w_csr)
    assert np.array_equal(un, w_un)


def assert_fresh(perc, live, trees, docs, nterms=V, cost=None):
    """the churned registry answers what a fresh registration of the live trees answers, ids mapped through the live ids"""
    live = np.asarray(sorted(live), np.uint32)
    got = perc.percolate(docs)
    fresh = tb.Percolator([trees[q] for q in live], nterms=nterms, term_cost=cost)
    want = fresh.percolate(docs)
    assert got.candidates == want.candidates
    assert got.total == want.total
    for d in range(len(docs)):
        assert np.array_equal(got.document(d), live[want.document(d)]), d
    info, finfo = perc.info(), fresh.info()
    for k in ("nqueries", "unanchored", "never", "anchor_entries"):
        assert info[k] == finfo[k], k
    fresh.source.close()
    return got


def test_seeded_churn_equals_reference_and_fresh_registration(shape_trees, docs):
    rng = np.random.default_rng(31)
    texts = []  # per issued id: its (text, flags, min)
    trees = []
    pick = rng.integers(0, len(SHAPES), 150)
    texts += [SHAPES[i] for i in pick]
    trees += [shape_trees[i] for i in pick]
    p = tb.Percolator(list(trees), nterms=V)
    assert p.info()["next_id"] == 150
    live = set(range(150))
    for rnd in range(14):
        if rnd % 5 == 4:
            gone = sorted(live)  # every live query
        else:
            gone = sorted(rng.choice(sorted(live), size=min(len(live), int(rng.integers(0, 120))), replace=False).tolist()) if live else []
        if rng.random() < 0.5:
            p.remove(rng.permutation(np.array(gone, np.uint32)))
        else:
            p.remove(gone)
        live -= set(gone)
        removed = set(range(len(trees))) - live
        n = int(rng.choice([1, 2, 7, 60, 250]))
        pick = rng.integers(0, len(SHAPES), n)
        ids = p.add([shape_trees[i] for i in pick])
        assert ids.tolist() == list(range(len(trees), len(trees) + n))
        texts += [SHAPES[i] for i in pick]
        trees += [shape_trees[i] for i in pick]
        live |= set(ids.tolist())
        info = p.info()
        assert info["next_id"] == len(trees) and info["nqueries"] == len(live)
        assert_registry(p.source, trees, removed, V)
        sub = [docs[i] for i in rng.choice(len(docs), 60, replace=False)]
        got = assert_fresh(p, live, trees, sub)
        lv = sorted(live)
        want = RefPercolator([texts[q] for q in lv]).run(sub)
        for d, w in enumerate(want):
            assert got.document(d).tolist() == [lv[i] for i in w.tolist()], (rnd, d)
    assert p.last_update_timings()["host_ms"] > 0


def _raw_percolate(src, doc):
    """trn_percolate through the C ABI: the result struct whose pointers stay valid until the next trn_percolate"""
    offs = np.array([0, len(doc)], np.uint64)
    tok = np.ascontiguousarray(doc, np.uint32)
    r = TrnPercolation()
    assert src._L.trn_percolate(src._h, offs.ctypes.data_as(C.c_void_p), tok.ctypes.data_as(C.c_void_p), 1, C.byref(r)) == 0
    return r, offs, tok


def test_refusals_change_nothing(shape_trees, monkeypatch):
    T, O, P = tb.NODE_TERM, tb.NODE_OR, tb.NODE_PHRASE
    t1, t2 = TD.term_id("t1"), TD.term_id("t2")
    src = tb.GpuIndexSource(0)
    with pytest.raises(tb.TrinityError, match="rc=-4"):
        src.percolator_add([_tree((T, 0, 0, t1))])
    with pytest.raises(tb.TrinityError, match="rc=-4"):
        src.percolator_remove([0])
    p = tb.Percolator([_tree((T, 0, 0, t1)), _tree((O, 2, 1, 0), (T, 0, 0, t1), (T, 0, 0, t2)), _tree((T, 0, 0, t2))], nterms=V, source=src)
    p.add([_tree((T, 0, 0, t2))])
    p.remove([1])
    doc = np.array([t1, t2], np.uint32)
    before_info = p.info()
    raw, keep_o, keep_t = _raw_percolate(src, doc)
    before = np.ctypeslib.as_array(raw.queries, shape=(int(raw.total),)).copy()
    assert before.tolist() == [0, 2, 3]
    bad = [
        ([_tree((T, 0, 0, t1)), _tree((T, 0, 0, V))], -1, "query 1"),
        ([_tree((T, 0, 0, t1)), _tree((T, 0, 0, t2)), _tree((P, 17, 1, 0), *[(T, 0, 0, t1)] * 17)], -1, "query 2"),
        ([_tree((O, 65, 1, 0), *[(T, 0, 0, t1)] * 65)], -7, "query 0"),
        ([_tree((O, 2, 0, 0), (T, 0, 0, t1))], -1, "query 0"),
    ]
    for qs, rc, who in bad:
        with pytest.raises(tb.TrinityError, match=f"rc={rc}: .*{who}"):
            p.add(qs)
    for ids, what in (([4], "never issued"), ([1], "already removed"), ([0, 2, 0], "twice"), ([2, 99], "never issued")):
        with pytest.raises(tb.TrinityError, match=f"rc=-1: .*id {ids[-1] if what != 'twice' else 0} .*{what}"):
            p.remove(ids)
    assert p.info() == before_info
    # the last result is untouched by the refused calls
    assert np.ctypeslib.as_array(raw.queries, shape=(int(raw.total),)).tolist() == before.tolist()
    assert p.percolate([doc]).document(0).tolist() == [0, 2, 3]
    assert p.add([]).tolist() == [] and p.info() == before_info
    p.remove([])
    assert p.info() == before_info
    # registering again starts the ids at 0
    p2 = tb.Percolator([_tree((T, 0, 0, t2))], nterms=V, source=src)
    assert p2.info()["next_id"] == 1 and p2.add([_tree((T, 0, 0, t1))]).tolist() == [1]
    assert p2.percolate([doc]).document(0).tolist() == [0, 1]
    src.close()
    # the id and anchor-entry limits (lowered through the environment; read when a context is created): ids below 10, entries below 12
    monkeypatch.setenv("TRN_PERC_MAX_IDS", "10")
    monkeypatch.setenv("TRN_PERC_MAX_ENTRIES", "12")
    t3, t4 = TD.term_id("t3"), TD.term_id("t4")
    p = tb.Percolator([_tree((T, 0, 0, t1))] * 4, nterms=V)
    p.add([_tree((T, 0, 0, t2))] * 4)  # ids 0..7, 8 entries
    info = p.info()
    with pytest.raises(tb.TrinityError, match="rc=-6"):
        p.add([_tree((T, 0, 0, t1))] * 3)  # id 10
    assert p.add([]).tolist() == [] and p.info() == info  # (an empty add reads the registry's info back)
    p.remove([0, 1])  # 6 entries
    info = p.info()
    with pytest.raises(tb.TrinityError, match="rc=-6"):  # 6 + 3 + 4 entries
        p.add([_tree((O, 3, 1, 0), (T, 0, 0, t1), (T, 0, 0, t2), (T, 0, 0, t3)),
               _tree((O, 4, 1, 0), (T, 0, 0, t1), (T, 0, 0, t2), (T, 0, 0, t3), (T, 0, 0, t4))])
    assert p.add([]).tolist() == [] and p.info() == info  # (an empty add reads the registry's info back)
    assert p.add([_tree((T, 0, 0, t1))]).tolist() == [8]
    assert p.percolate([doc]).document(0).tolist() == [2, 3, 4, 5, 6, 7, 8]
    p.source.close()


def test_output_paths_after_churn():
    """a document above the 4096-match sort cap (bitmap output over next_id bits) and one below it, with next_id far above the live count;
    documents of more than 512 tokens (the long launch)"""
    rng = np.random.default_rng(41)
    t1, t2, t3 = TD.term_id("t1"), TD.term_id("t2"), TD.term_id("t3")
    one = _tree((tb.NODE_TERM, 0, 0, t1))
    both = _tree((tb.NODE_AND, 2, 1, 0), (tb.NODE_TERM, 0, 0, t1), (tb.NODE_TERM, 0, 0, t2))
    ph = _tree((tb.NODE_PHRASE, 2, 1, 0), (tb.NODE_TERM, 0, 0, t2), (tb.NODE_TERM, 0, 0, t3))
    trees = [one if i % 7 else both for i in range(20_000)]
    p = tb.Percolator(list(trees), nterms=V)
    live = set(range(20_000))
    for k in range(6):
        add = [[one, both, ph][int(x)] for x in rng.choice(3, 15_000, p=[0.45, 0.45, 0.1])]
        ids = p.add(add)
        trees += add
        live |= set(ids.tolist())
        gone = rng.choice(sorted(live), size=14_000, replace=False)
        p.remove(gone)
        live -= set(gone.tolist())
    assert p.info()["next_id"] == 110_000 and p.info()["nqueries"] == len(live) == 26_000
    d_all = np.array([t1, t2, t3], np.uint32)
    d_few = np.array([t2, t3], np.uint32)  # the phrase queries only
    long_doc = rng.choice(V, 3000).astype(np.uint32)
    long_doc[1700:1702] = [t2, t3]
    docs = [d_all, d_few, long_doc, long_doc[:600]] + random_docs(rng, 30, max_len=20)
    got = assert_fresh(p, live, trees, docs)
    assert got.dense_docs >= 1 and got.long_docs >= 2
    assert 0 < len(got.document(1)) <= 4096 < len(got.document(0))
    for d, x in enumerate(docs[:4]):
        assert got.document(d).tolist() == [q for q in sorted(live) if evaluate(trees[q], x)]
    assert_registry(p.source, trees, set(range(len(trees))) - live, V)


def test_program_storage_compaction_frees_memory_and_stays_exact(docs):
    rng = np.random.default_rng(43)
    long = [parse('"w1 w2 w3 w4 w5 w6 w7 w8"', 0),
            parse('(t1 OR t2 OR t3 OR t4) AND (t5 OR t6 OR t7 OR "w1 w2") NOT (t8 OR t9 OR "w3 w4 w5")', 0),
            parse('[t1, t2, t3, "w1 w2", t4 AND t5]', 2)]
    trees = [long[i % 3] for i in range(30_000)]
    p = tb.Percolator(list(trees), nterms=V)
    p.add([long[i % 3] for i in range(30_000)])
    trees += [long[i % 3] for i in range(30_000)]
    live = set(range(60_000))
    assert_fresh(p, live, trees, docs[:100])
    grown = p.info()["device_bytes"]
    gone = rng.choice(60_000, 20_000, replace=False)  # a third: no compaction yet
    p.remove(gone)
    live -= set(gone.tolist())
    mid = p.info()["device_bytes"]
    assert_fresh(p, live, trees, docs[:100])
    gone = rng.choice(sorted(live), 25_000, replace=False)  # now the removed programs outnumber the live ones
    p.remove(gone)
    live -= set(gone.tolist())
    after = p.info()["device_bytes"]
    assert after < mid < grown and after < grown / 2
    assert_fresh(p, live, trees, docs)
    assert_registry(p.source, trees, set(range(len(trees))) - live, V)
    # appending behind the compacted storage, and compacting down to nothing
    more = p.add([long[1]] * 500)
    trees += [long[1]] * 500
    live |= set(more.tolist())
    assert_fresh(p, live, trees, docs[:100])
    p.remove(sorted(live))
    assert p.info()["nqueries"] == 0 and p.info()["anchor_entries"] == 0
    assert p.percolate(docs[:50]).total == 0
    p.add([long[0]])
    trees.append(long[0])
    assert_fresh(p, {len(trees) - 1}, trees, docs[:100])


def test_scale_100000_queries_with_10000_adds_and_10000_removes(shape_trees):
    rng = np.random.default_rng(47)
    pick = rng.integers(0, len(SHAPES), 110_000)
    trees = [shape_trees[i] for i in pick]
    cost = rng.integers(1, 50, V).astype(np.uint32)
    p = tb.Percolator(trees[:100_000], nterms=V, term_cost=cost)
    ids = p.add(trees[100_000:])
    assert ids[0] == 100_000 and ids[-1] == 109_999
    gone = rng.choice(110_000, 10_000, replace=False)
    p.remove(gone)
    live = set(range(110_000)) - set(gone.tolist())
    docs = random_docs(rng, 40, max_len=30)
    assert_fresh(p, live, trees, docs, cost=cost)
    assert_registry(p.source, trees, set(gone.tolist()), V, cost)


def test_shared_context_keeps_exec_batch_results(ref, shape_trees):
    ndocs = 20_000
    pair = Pair(ref, tb.CODEC_GOOGLE, closed_form_lists(ndocs), ndocs)
    g = pair.gpu
    qs = ["t1 AND t2", "t3 OR t7", "t1 AND (t2 OR t3) NOT t5"]
    before = [g.exec_batch([pair.plan(q)], tb.MODE_DOCS_ONLY).query(0)[0].copy() for q in qs]
    trees = [shape_trees[i % len(shape_trees)] for i in range(130)]
    p = tb.Percolator(trees[:50], nterms=V, source=g)
    p.add(trees[50:120])
    p.remove(list(range(0, 120, 3)))
    p.add(trees[120:])
    for q, b in zip(qs, before):
        after = g.exec_batch([pair.plan(q)], tb.MODE_DOCS_ONLY).query(0)[0]
        assert_same_docs(after, b, f"exec_batch next to a churned registry [{q}]")
        want, _ = pair.ref.exec(q, False, ndocs)
        assert_same_docs(after, want, f"exec_batch vs reference [{q}]")
    live = set(range(130)) - set(range(0, 120, 3))
    assert_fresh(p, live, trees, random_docs(np.random.default_rng(3), 50, max_len=30))
    g.close()
