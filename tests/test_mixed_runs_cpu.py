"""The run-major tickets of the flat ANDs with exactly one operand without a resident bitmap (planner.cpp plan_batch: BatchPlan::mixed_runs),
checked without a GPU through trn_debug_mixed_runs / trn_debug_dense_runs / trn_debug_plan:
  * exactly those flat ANDs take them; the routes, the slot counts and the all-bitmap tickets stay what they are;
  * TRN_MIXED_RUNS=0 and TRN_DENSE_BITMAPS=0 switch them off, a LUCENE source, the scored modes and a batch with a phrase plan never use them;
  * every (query, tile) item of those queries exactly once, one 2^17-docID run per ticket, run-major, at TRN_DOCS_SHIFT 13 / 14 / 17 and
    at the top of the docID space."""
import numpy as np
import pytest

import trinity_b200 as tb
from test_dense_runs_cpu import _check_mapping

G, L = tb.CODEC_GOOGLE, tb.CODEC_LUCENE
S = 600_000
FULL = np.arange(409_600, 409_856, dtype=np.uint32)  # one whole 256-docID bucket, aligned in every tile size


def corpus():
    u = lambda *a: np.unique(np.concatenate([np.asarray(x, np.uint32) for x in a]))
    out = {}
    for name, step in (("a", 2), ("b", 3), ("c", 5), ("d", 7)):  # dense: a bitmap each
        out[name] = np.arange(step, S + 1, step, dtype=np.uint32)
    out["f"] = u(np.arange(6, S + 1, 6), FULL)  # dense, holds the full bucket
    out["n"] = np.arange(300_000, 330_000, 2, dtype=np.uint32)  # dense in a narrow span: a bitmap of 2^17 docIDs
    # decoded leads (no bitmap)
    out["x"] = u(np.arange(401, S + 1, 401), np.arange(200_001, 210_001), FULL)  # sparse, a dense cluster (bitmap-form tiles), the full bucket
    out["m"] = np.arange(37, S + 1, 37, dtype=np.uint32)  # "m AND b": U8B tiles
    out["y"] = u(np.arange(1, 40_000, 3), np.arange(100_000, S + 1, 20_000))  # gaps of 20 000: 3-byte codes, blocks across runs
    out["z"] = np.arange(312_001, 327_000, 5, dtype=np.uint32)  # inside one 2^14 tile (and n's span)
    out["p"] = np.arange(41, S + 1, 41, dtype=np.uint32)
    out["s"] = np.arange(997, S + 1, 997, dtype=np.uint32)  # sparse: leads the candidate-driven path
    return out


LISTS = corpus()
NAMES = list(LISTS)
DENSE = {"a", "b", "c", "d", "f", "n"}
MIXED = ["x AND a", "x AND f", "m AND b", "m AND b AND c", "y AND a", "x AND n", "z AND n", "p AND d"]
QUERIES = MIXED + [
    "a AND b", "n AND c",  # all-bitmap
    "s AND a",  # candidate-driven (its shared-memory need sets the slot count at 2^13 tiles)
    "m AND p", "x AND m AND a",  # flat AND, two decoded operands
    "(a OR m) AND (b OR x) NOT d",  # flat tree
    "a OR m OR x",  # flat OR
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


def _mixed(index, terms, plans, codec=G, mode=tb.MODE_DOCS_ONLY, max_docid=S):
    return tb.debug_mixed_runs(codec, index, terms, plans, mode, max_docid=max_docid)


def test_selection_is_the_expected_one(google):
    index, terms, _ = google
    off, _ = tb.debug_dense_terms(G, index, terms)
    assert {n for n, o in zip(NAMES, off) if o != tb.DENSE_NONE} == DENSE


@pytest.mark.parametrize("mode", [tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT], ids=["docs", "compact"])
def test_exactly_the_mixed_flat_ands_take_the_tickets(google, mode):
    index, terms, plans = google
    routes, _ = tb.debug_plan(G, index, terms, plans, mode, max_docid=S)
    _, tickets = _mixed(index, terms, plans, mode=mode)
    want = {i for i, q in enumerate(QUERIES) if q in MIXED}
    assert all(routes[i] == tb.ROUTE_FLAT_AND for i in want), routes
    assert set(tickets[:, 0].tolist()) == want


def test_routes_slots_and_dense_tickets_do_not_change(google, monkeypatch):
    index, terms, plans = google
    for mode in (tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT):
        on = tb.debug_plan(G, index, terms, plans, mode, max_docid=S)
        dense_on = tb.debug_dense_runs(G, index, terms, plans, mode, max_docid=S)
        monkeypatch.setenv("TRN_MIXED_RUNS", "0")
        off = tb.debug_plan(G, index, terms, plans, mode, max_docid=S)
        dense_off = tb.debug_dense_runs(G, index, terms, plans, mode, max_docid=S)
        monkeypatch.delenv("TRN_MIXED_RUNS")
        assert on[0].tolist() == off[0].tolist() and on[1] == off[1], mode
        assert np.array_equal(dense_on[1], dense_off[1]) and len(dense_on[1]), mode
        assert {QUERIES[i] for i in dense_on[1][:, 0]} == {"a AND b", "n AND c"}


@pytest.mark.parametrize("knob", ["TRN_MIXED_RUNS", "TRN_DENSE_BITMAPS"])
def test_knobs_switch_it_off(google, monkeypatch, knob):
    index, terms, plans = google
    assert len(_mixed(index, terms, plans)[1])
    monkeypatch.setenv(knob, "0")
    assert len(_mixed(index, terms, plans)[1]) == 0


def test_never_on_lucene_scored_or_beside_a_phrase(google):
    index, terms, plans = google
    lindex, lterms = build(L)
    assert len(_mixed(lindex, lterms, plans, codec=L)[1]) == 0
    for mode in (tb.MODE_SCORED_ALL, tb.MODE_SCORED_TOPK):
        assert len(_mixed(index, terms, plans, mode=mode)[1]) == 0
    phrase = tb.parse_query('"a b"', tb.TermDictionary(NAMES))
    assert len(_mixed(index, terms, plans + [phrase])[1]) == 0


@pytest.mark.parametrize("docs_shift", [13, 14, 17])
def test_every_item_exactly_once_at_each_tile_size(google, monkeypatch, docs_shift):
    index, terms, plans = google
    monkeypatch.setenv("TRN_DOCS_SHIFT", str(docs_shift))
    routes, _ = tb.debug_plan(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=S)
    qtiles, tickets = _mixed(index, terms, plans)
    want = {i for i, q in enumerate(QUERIES) if q in MIXED and routes[i] == tb.ROUTE_FLAT_AND}  # (the crossover moves with the tile)
    assert len(want) >= 5 and set(tickets[:, 0].tolist()) == want
    assert len({(int(qtiles[q, 0]), int(qtiles[q, 1])) for q in want}) >= 2  # the queries' tile ranges differ
    assert any(int(qtiles[q, 1]) == 1 for q in want) or docs_shift == 13  # a query of one tile
    _check_mapping(qtiles, tickets, want, docs_shift)


def test_every_item_exactly_once_at_the_top_of_the_docid_space():
    top = 2**32 - 2
    index, terms = build(G, shift=top - S)
    plans = [tb.parse_query(q, tb.TermDictionary(NAMES)) for q in QUERIES]
    qtiles, tickets = _mixed(index, terms, plans, max_docid=top)
    _check_mapping(qtiles, tickets, {i for i, q in enumerate(QUERIES) if q in MIXED})
    assert int(tickets[:, 2].max()) == 2**32 >> 14  # the run ending at 2^32
