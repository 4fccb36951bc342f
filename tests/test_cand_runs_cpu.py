"""The run-major tickets of the candidate-driven queries (planner.cpp plan_batch: BatchPlan::cand_runs), checked without a GPU through
trn_debug_cand_runs / trn_debug_plan / trn_debug_mixed_runs / trn_debug_dense_runs:
  * exactly the candidate-driven queries take them, one ticket per 32-block group of the lead, every group exactly once;
  * ordered by the 2^17-docID run of the group's first docID (the last docID of the block before it plus one), queries ascending within
    a run, groups ascending within a query; the first docIDs are those of the lead's directory;
  * the routes, the slot counts and the flat ANDs' run tickets stay what they are;
  * TRN_CAND_RUNS=0 switches them off; a LUCENE source, the scored modes and a batch with a phrase plan never use them;
  * at TRN_DOCS_SHIFT 13 / 14 / 17 and at the top of the docID space."""
import numpy as np
import pytest

import candutil as cu
import trinity_b200 as tb

G, L = tb.CODEC_GOOGLE, tb.CODEC_LUCENE
RUN = cu.DENSE_ALIGN


def corpus(shift=0):
    """sparse leads that span many runs (their groups start in different runs, a lead group can span runs), leads inside one run, and
    dense probe terms with resident bitmaps"""
    rng = np.random.default_rng(17)
    S = 3_000_000
    out = {}
    out["a"] = np.arange(2, S + 1, 2, dtype=np.uint32)  # dense: bitmaps
    out["b"] = np.arange(3, S + 1, 3, dtype=np.uint32)
    out["l1"] = np.unique(rng.integers(1, S + 1, 20_000)).astype(np.uint32)  # ~20 groups over ~23 runs
    out["l2"] = np.unique(rng.integers(1, S + 1, 9_000)).astype(np.uint32)
    out["l3"] = np.arange(1_000_001, 1_050_000, 7, dtype=np.uint32)  # inside one run
    out["l4"] = np.unique(rng.integers(2_500_000, S + 1, 3_000)).astype(np.uint32)  # the last runs only
    out["x"] = np.arange(5, S + 1, 29, dtype=np.uint32)  # denser than the leads
    return {k: (v.astype(np.uint64) + shift).astype(np.uint32) for k, v in out.items()}, S + shift


CAND = ["l1 AND a", "l2 AND b", "l3 AND a AND b", "l1 AND (a OR x)", "l4 AND x", "l2 AND a AND x", "l3 AND (a OR b) NOT x"]
OTHER = ["a AND b", "x AND a", "a OR x", "(a OR x) AND b NOT l1"]
QUERIES = [CAND[0], OTHER[0], CAND[1], CAND[2], OTHER[1], CAND[3], OTHER[2], CAND[4], CAND[5], OTHER[3], CAND[6]]


@pytest.fixture(scope="module")
def google():
    lists, mx = corpus()
    index, terms, names = cu.build(lists)
    return index, terms, names, [tb.parse_query(q, tb.TermDictionary(names)) for q in QUERIES], mx


def _cand(index, terms, plans, mx, codec=G, mode=tb.MODE_DOCS_ONLY):
    return tb.debug_cand_runs(codec, index, terms, plans, mode, max_docid=mx)


def _group_starts(index, terms, t):
    """the first docID of every 32-block group of term t, from its directory"""
    last, _, first = tb.directory_probe(G, index, cu.term_tuple(terms, t))
    nb = len(last) - 1
    return [int(first) if g == 0 else int(last[32 * g - 1]) + 1 for g in range((nb + 31) // 32)]


def check_mapping(index, terms, names, plans, qgroups, tickets, want):
    """every group of every query in want exactly once, run-major, ties in query order, with the lead's group starts"""
    assert set(tickets[:, 0].tolist()) == want
    expect = []
    for q in sorted(want):
        lead, _, _ = cu.probe_order(plans[q], terms)
        starts = _group_starts(index, terms, lead[0])
        assert int(qgroups[q, 1]) == len(starts), q
        expect += [(s >> RUN, q, g, s) for g, s in enumerate(starts)]
    expect.sort(key=lambda e: (e[0], e[1], e[2]))  # (stable in the planner: queries, then groups, ascending within a run)
    got = [(int(s) >> RUN, int(q), int(g), int(s)) for q, g, s in tickets]
    assert got == expect


def test_exactly_the_candidate_queries_take_them(google):
    index, terms, names, plans, mx = google
    for mode in (tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT):
        routes, _ = tb.debug_plan(G, index, terms, plans, mode, max_docid=mx)
        want = {i for i, q in enumerate(QUERIES) if q in CAND}
        assert {i for i, r in enumerate(routes) if r == tb.ROUTE_CANDIDATE} == want, routes
        qgroups, tickets = _cand(index, terms, plans, mx, mode=mode)
        check_mapping(index, terms, names, plans, qgroups, tickets, want)
        runs = tickets[:, 2] >> RUN
        assert len(set(runs.tolist())) >= 20  # the groups spread over many runs ...
        assert (np.diff(tickets[:, 0].astype(np.int64)) < 0).any()  # ... so the queries interleave


def test_routes_slots_and_flat_tickets_do_not_change(google, monkeypatch):
    index, terms, names, plans, mx = google
    for mode in (tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT):
        on = tb.debug_plan(G, index, terms, plans, mode, max_docid=mx)
        flat_on = [f(G, index, terms, plans, mode, max_docid=mx) for f in (tb.debug_dense_runs, tb.debug_mixed_runs)]
        monkeypatch.setenv("TRN_CAND_RUNS", "0")
        off = tb.debug_plan(G, index, terms, plans, mode, max_docid=mx)
        flat_off = [f(G, index, terms, plans, mode, max_docid=mx) for f in (tb.debug_dense_runs, tb.debug_mixed_runs)]
        assert len(_cand(index, terms, plans, mx, mode=mode)[1]) == 0
        monkeypatch.delenv("TRN_CAND_RUNS")
        assert on[0].tolist() == off[0].tolist() and on[1] == off[1], mode
        for a, b in zip(flat_on, flat_off):
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), mode
        assert len(flat_on[0][1]) + len(flat_on[1][1])  # the batch holds flat run tickets too


def test_never_on_lucene_scored_or_beside_a_phrase(google):
    index, terms, names, plans, mx = google
    assert len(_cand(index, terms, plans, mx)[1])
    lists, _ = corpus()
    b = tb.IndexBuilder(L)
    for n in names:
        d = np.asarray(lists[n], np.uint32)
        b.add_term(d, 1 + (d % 3).astype(np.uint32))
    assert len(_cand(b.index(), b.terms_array(), plans, mx, codec=L)[1]) == 0
    for mode in (tb.MODE_SCORED_ALL, tb.MODE_SCORED_TOPK):
        assert len(_cand(index, terms, plans, mx, mode=mode)[1]) == 0
    phrase = tb.parse_query('"a b"', tb.TermDictionary(names))
    routes, _ = tb.debug_plan(G, index, terms, plans + [phrase], tb.MODE_DOCS_ONLY, max_docid=mx)
    assert tb.ROUTE_CANDIDATE in list(routes)  # the candidate queries keep their route, on query-order tickets
    assert len(_cand(index, terms, plans + [phrase], mx)[1]) == 0


@pytest.mark.parametrize("docs_shift", [13, 14, 17])
def test_every_group_exactly_once_at_each_tile_size(google, monkeypatch, docs_shift):
    index, terms, names, plans, mx = google
    monkeypatch.setenv("TRN_DOCS_SHIFT", str(docs_shift))
    routes, _ = tb.debug_plan(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=mx)
    want = {i for i, r in enumerate(routes) if r == tb.ROUTE_CANDIDATE}  # (the crossover moves with the tile)
    assert len(want) >= 4
    qgroups, tickets = _cand(index, terms, plans, mx)
    check_mapping(index, terms, names, plans, qgroups, tickets, want)


def test_every_group_exactly_once_at_the_top_of_the_docid_space():
    lists, mx = corpus(shift=cu.TOP - 3_000_000)
    assert mx == cu.TOP
    index, terms, names = cu.build(lists)
    plans = [tb.parse_query(q, tb.TermDictionary(names)) for q in QUERIES]
    routes, _ = tb.debug_plan(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=mx)
    want = {i for i, r in enumerate(routes) if r == tb.ROUTE_CANDIDATE}
    assert len(want) >= 4
    qgroups, tickets = _cand(index, terms, plans, mx)
    check_mapping(index, terms, names, plans, qgroups, tickets, want)
    assert int(tickets[:, 2].max()) >> RUN == (2**32 - 1) >> RUN  # the last run
