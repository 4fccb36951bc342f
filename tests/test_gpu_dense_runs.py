"""The all-bitmap flat ANDs on their run-major tickets (exec_docs.cuh dense_run_exec): in both DocumentsOnly modes every result equals the
reference (oracle/_ref) and the same batch on a source created with TRN_DENSE_RUNS=0, and every query runs the route trn_debug_plan plans.
The corpus and batch are test_dense_runs_cpu's: all-bitmap ANDs of 2 and 3 operands, narrow-span bitmap terms, an empty intersection,
mixed with partly-bitmap flat ANDs, candidate-driven plans, a flat tree and a flat OR.  Also: masked documents, the pipelined
trn_exec_batch, 2 and 3 shards, the corpus translated to end at 2^32 - 2, and 8-operand all-bitmap ANDs beside an 8-slot plan."""
import os

import numpy as np
import pytest

import trinity_b200 as tb
from refharness import RefIndex
from test_dense_runs_cpu import ALL_BITMAP, LISTS, NAMES, QUERIES, S, build
from util import assert_same_docs

pytestmark = pytest.mark.gpu

G = tb.CODEC_GOOGLE
TOP = 2**32 - 2
DELTA = TOP - S
MODES = [tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT]


def _source(index, terms, max_docid, runs=True):
    old = os.environ.get("TRN_DENSE_RUNS")
    os.environ["TRN_DENSE_RUNS"] = "1" if runs else "0"
    try:
        g = tb.GpuIndexSource(0)
    finally:
        if old is None:
            os.environ.pop("TRN_DENSE_RUNS")
        else:
            os.environ["TRN_DENSE_RUNS"] = old
    g.upload(G, index, terms, max_docid)
    return g


def _results(g, plans, mode):
    res = g.exec_batch(plans, mode, copy=mode == tb.MODE_DOCS_ONLY)
    return [(res.query(i)[0] if mode == tb.MODE_DOCS_ONLY else res.decode_query(i)).copy() for i in range(len(plans))]


def _check(index, terms, max_docid, plans, want, label, masked=None):
    """on vs off vs want, both modes, routes == debug_plan; the batch must use the run tickets"""
    routes, _ = tb.debug_plan(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=max_docid)
    assert len(tb.debug_dense_runs(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=max_docid)[1]), label
    srcs = {r: _source(index, terms, max_docid, r) for r in (True, False)}
    try:
        for g in srcs.values():
            if masked is not None:
                g.set_masked_documents(masked)
        for mode in MODES:
            got = {}
            for r, g in srcs.items():
                got[r] = _results(g, plans, mode)
                assert list(g.last_routes()) == list(routes), (label, r, mode)
            for i in range(len(plans)):
                assert_same_docs(got[True][i], want[i], f"{label} [{i}] runs on, mode {mode}")
                assert_same_docs(got[False][i], want[i], f"{label} [{i}] runs off, mode {mode}")
    finally:
        for g in srcs.values():
            g.close()


@pytest.fixture(scope="module")
def world(ref):
    r = RefIndex(ref, G)
    for n in NAMES:
        r.add_term(n, LISTS[n], 1 + LISTS[n] % 3)
    r.finish(S)
    tdict = tb.TermDictionary(NAMES)
    return dict(ref=r, tdict=tdict, plans=[tb.parse_query(q, tdict) for q in QUERIES])


def _want(w, shift=0):
    return [(w["ref"].exec(q, False, S + 1)[0].astype(np.uint64) + shift).astype(np.uint32) for q in QUERIES]


def test_results_equal_reference_and_runs_off(world):
    index, terms = build(G)
    want = _want(world)
    assert len(want[QUERIES.index("a AND o")]) == 0  # the empty intersection
    _check(index, terms, S, world["plans"], want, "full")


def test_masked_documents(world):
    rng = np.random.default_rng(11)
    pool = np.unique(np.concatenate([LISTS["a"][::5], LISTS["b"][::3], LISTS["n"], LISTS["w"][::2]]))
    masked = np.sort(rng.choice(pool, size=len(pool) // 3, replace=False)).astype(np.uint32)
    want = [world["ref"].exec_masked(q, False, masked, S + 1)[0] for q in QUERIES]
    index, terms = build(G)
    _check(index, terms, S, world["plans"], want, "masked", masked)


def test_pipelined(world, monkeypatch):
    monkeypatch.setenv("TRN_PIPELINE_CHUNKS", "8")
    monkeypatch.setenv("TRN_CHUNK_POSTINGS", "1")
    monkeypatch.setenv("TRN_CHUNK_RULE", "postings")
    index, terms = build(G)
    plans = world["plans"] * 5  # >= 64 queries: split into chunks
    _check(index, terms, S, plans, _want(world) * 5, "pipelined")


@pytest.mark.parametrize("nshards", [2, 3])
def test_shards(world, nshards):
    cuts = [1] + [int(S * (i + 1) / nshards) + 1 for i in range(nshards - 1)] + [S + 1]
    want = _want(world)
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        index, terms = build(G, lo=lo, hi=hi - 1)
        part = [w[(w >= lo) & (w < hi)] for w in want]
        plans = [tb.parse_query(q, world["tdict"]) for q in QUERIES]
        if len(tb.debug_dense_runs(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=S)[1]):
            _check(index, terms, S, plans, part, f"shard [{lo}, {hi})")


def test_top_of_the_docid_space(world):
    index, terms = build(G, shift=DELTA)
    plans = [tb.parse_query(q, tb.TermDictionary(NAMES)) for q in QUERIES]
    _check(index, terms, TOP, plans, _want(world, DELTA), "top")


def test_eight_operands_beside_an_eight_slot_plan():
    """test_gpu_plan_limits' corpus: t1 AND c2 .. c8 (every operand with a bitmap) runs flat beside the 8-slot step program; t1 AND c2 .. c9
    does not run flat and never takes the run tickets"""
    from test_gpu_plan_limits import NDOCS, _and, _lists, _wide

    lists, names = _lists()
    b = tb.IndexBuilder(G)
    for d, f in lists:
        b.add_term(d, f)
    index, terms = b.index(), b.terms_array()
    tdict = tb.TermDictionary(names)
    texts = [_wide(6), _and(8), _and(9), _and(3)]
    plans = [tb.parse_query(q, tdict) for q in texts]
    routes, slots = tb.debug_plan(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=NDOCS)
    assert slots[0] == 8 and routes[1] == tb.ROUTE_FLAT_AND and routes[2] != tb.ROUTE_FLAT_AND
    _, tickets = tb.debug_dense_runs(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=NDOCS)
    assert 1 in set(tickets[:, 0].tolist()) and 2 not in set(tickets[:, 0].tolist())
    docs = dict(zip(names, (d for d, _ in lists)))

    def conj(text):
        out = None
        for t in text.split(" AND "):
            out = docs[t] if out is None else np.intersect1d(out, docs[t])
        return out

    srcs = {r: _source(index, terms, NDOCS, r) for r in (True, False)}
    try:
        for mode in MODES:
            got = {r: _results(g, plans, mode) for r, g in srcs.items()}
            for r, g in srcs.items():
                assert list(g.last_routes()) == list(routes)
            for i in (1, 2, 3):
                assert_same_docs(got[True][i], conj(texts[i]), f"[{texts[i]}] mode {mode}")
                assert_same_docs(got[False][i], got[True][i], f"[{texts[i]}] off, mode {mode}")
            assert_same_docs(got[True][0], got[False][0], f"[{texts[0]}] mode {mode}")
    finally:
        for g in srcs.values():
            g.close()
