"""The run-major ticket space of the all-bitmap flat ANDs (planner.cpp plan_batch: BatchPlan::dense_runs), checked without a GPU through
trn_debug_dense_runs / trn_debug_plan:
  * exactly the flat ANDs whose operands all have a resident bitmap take it; the routes stay what they are;
  * TRN_DENSE_RUNS=0 and TRN_DENSE_BITMAPS=0 switch it off, a LUCENE source and a batch with a phrase plan never use it;
  * the ticket -> (query, tiles) mapping: every (query, tile) item of those queries exactly once, one 2^17-docID run per ticket, the
    tickets run-major — also for queries whose tile ranges differ (a bitmap term of a narrow span)."""
import numpy as np
import pytest

import trinity_b200 as tb

G, L = tb.CODEC_GOOGLE, tb.CODEC_LUCENE
S = 600_000
RUN = 1 << 17


def corpus():
    out = {}
    for name, step in (("a", 2), ("b", 3), ("c", 5), ("d", 7), ("e", 11)):  # dense: a bitmap each
        out[name] = np.arange(step, S + 1, step, dtype=np.uint32)
    out["o"] = np.arange(1, S + 1, 2, dtype=np.uint32)  # dense, disjoint from a
    out["m"] = np.arange(37, S + 1, 37, dtype=np.uint32)  # mid: decoded
    out["s"] = np.arange(401, S + 1, 401, dtype=np.uint32)  # sparse: decoded, leads the candidate-driven path
    out["n"] = np.arange(300_000, 330_000, 2, dtype=np.uint32)  # dense in a narrow span: a bitmap of 2^17 docIDs
    out["w"] = np.arange(131_000, 400_000, 3, dtype=np.uint32)  # dense over a mid span that starts inside the first run
    return out


LISTS = corpus()
NAMES = list(LISTS)
DENSE = {"a", "b", "c", "d", "e", "o", "n", "w"}
ALL_BITMAP = ["a AND b", "b AND c AND d", "a AND e", "a AND n", "n AND b AND c", "w AND c", "w AND n AND e", "a AND o"]
QUERIES = ALL_BITMAP + [
    "c AND m", "a AND b AND m",  # flat AND, some operands with a bitmap
    "s AND a", "s AND m AND d",  # candidate-driven
    "(a OR m) AND (b OR s) NOT e",  # flat tree
    "a OR m OR s",  # flat OR
]


def build(codec, lists=LISTS, shift=0, lo=1, hi=2**32):
    b = tb.IndexBuilder(codec)
    for n in NAMES:
        d = lists[n].astype(np.uint64) + shift
        d = d[(d >= lo) & (d <= hi)].astype(np.uint32)
        b.add_term(d, 1 + d % 3)
    return b.index(), b.terms_array()


@pytest.fixture(scope="module")
def google():
    index, terms = build(G)
    return index, terms, [tb.parse_query(q, tb.TermDictionary(NAMES)) for q in QUERIES]


def _runs(index, terms, plans, codec=G, mode=tb.MODE_DOCS_ONLY, max_docid=S):
    return tb.debug_dense_runs(codec, index, terms, plans, mode, max_docid=max_docid)


def test_selection_is_the_expected_one(google):
    index, terms, _ = google
    off, _ = tb.debug_dense_terms(G, index, terms)
    assert {n for n, o in zip(NAMES, off) if o != tb.DENSE_NONE} == DENSE


@pytest.mark.parametrize("mode", [tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT], ids=["docs", "compact"])
def test_all_bitmap_flat_ands_take_the_run_tickets(google, mode):
    index, terms, plans = google
    routes, _ = tb.debug_plan(G, index, terms, plans, mode, max_docid=S)
    _, tickets = _runs(index, terms, plans, mode=mode)
    want = {i for i, q in enumerate(QUERIES) if q in ALL_BITMAP}
    assert all(routes[i] == tb.ROUTE_FLAT_AND for i in want), routes
    assert set(tickets[:, 0].tolist()) == want


def test_routes_do_not_change(google, monkeypatch):
    index, terms, plans = google
    for mode in (tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT):
        on = tb.debug_plan(G, index, terms, plans, mode, max_docid=S)
        monkeypatch.setenv("TRN_DENSE_RUNS", "0")
        off = tb.debug_plan(G, index, terms, plans, mode, max_docid=S)
        monkeypatch.delenv("TRN_DENSE_RUNS")
        assert on[0].tolist() == off[0].tolist() and on[1] == off[1], mode


@pytest.mark.parametrize("knob", ["TRN_DENSE_RUNS", "TRN_DENSE_BITMAPS"])
def test_knobs_switch_it_off(google, monkeypatch, knob):
    index, terms, plans = google
    assert len(_runs(index, terms, plans)[1])
    monkeypatch.setenv(knob, "0")
    assert len(_runs(index, terms, plans)[1]) == 0


def test_never_on_lucene_scored_or_beside_a_phrase(google):
    index, terms, plans = google
    lindex, lterms = build(L)
    assert len(_runs(lindex, lterms, plans, codec=L)[1]) == 0
    for mode in (tb.MODE_SCORED_ALL, tb.MODE_SCORED_TOPK):
        assert len(_runs(index, terms, plans, mode=mode)[1]) == 0
    phrase = tb.parse_query('"a b"', tb.TermDictionary(NAMES))
    assert len(_runs(index, terms, plans + [phrase])[1]) == 0


def _check_mapping(qtiles, tickets, want, exec_shift=14):
    tpr = RUN >> exec_shift
    seen = {}
    for q, t0, t1 in tickets.tolist():
        assert t0 < t1 and t0 // tpr == (t1 - 1) // tpr, (q, t0, t1)  # one run
        for t in range(t0, t1):
            seen[(q, t)] = seen.get((q, t), 0) + 1
    items = {(q, t) for q in want for t in range(int(qtiles[q, 0]), int(qtiles[q, 0] + qtiles[q, 1]))}
    assert set(seen) == items and set(seen.values()) == {1}
    runs = tickets[:, 1] // tpr
    assert np.all(np.diff(runs.astype(np.int64)) >= 0)  # run-major


def test_every_item_exactly_once(google):
    index, terms, plans = google
    qtiles, tickets = _runs(index, terms, plans)
    want = {i for i, q in enumerate(QUERIES) if q in ALL_BITMAP}
    assert len({(int(qtiles[q, 0]), int(qtiles[q, 1])) for q in want}) >= 3  # the queries' tile ranges differ
    _check_mapping(qtiles, tickets, want)


@pytest.mark.parametrize("docs_shift", [13, 14, 17])
def test_every_item_exactly_once_at_each_tile_size(google, monkeypatch, docs_shift):
    index, terms, plans = google
    monkeypatch.setenv("TRN_DOCS_SHIFT", str(docs_shift))
    qtiles, tickets = _runs(index, terms, plans)
    _check_mapping(qtiles, tickets, {i for i, q in enumerate(QUERIES) if q in ALL_BITMAP}, docs_shift)


def test_every_item_exactly_once_at_the_top_of_the_docid_space():
    top = 2**32 - 2
    index, terms = build(G, shift=top - S)
    plans = [tb.parse_query(q, tb.TermDictionary(NAMES)) for q in QUERIES]
    qtiles, tickets = _runs(index, terms, plans, max_docid=top)
    want = {i for i, q in enumerate(QUERIES) if q in ALL_BITMAP}
    _check_mapping(qtiles, tickets, want)
    assert int(tickets[:, 2].max()) == 2**32 >> 14  # the run ending at 2^32
