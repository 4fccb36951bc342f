"""The route planner (planner.h plan_batch) checked without a GPU through trn_debug_plan: the path (ROUTE_*) every query of a batch takes
and the docset slots of the step-program launch, for
  * the plan-width limits of test_gpu_plan_limits (its PLANS table), both codecs, DocumentsOnly and scored;
  * the flat AND's one slot per operand: it runs flat only where the launch has a slot for each of its operands;
  * the bench.py workloads on a small synthetic index;
  * the knobs that switch a route off (TRN_FLAT_SCORED=0, TRN_TREE_SHIFT=0, TRN_CAND_COST=0).
The GPU test checks that the engine runs what the planner says (GpuIndexSource.last_routes), in every mode, through the single-call and
the pipelined trn_exec_batch."""
import sys
from pathlib import Path

import numpy as np
import pytest

import trinity_b200 as tb
from test_gpu_plan_limits import NDOCS, PLANS, _and, _lists, _wide

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import bench  # noqa: E402

S, AND, OR, CAND, SF, TREE, TILES = (tb.ROUTE_STEPS, tb.ROUTE_FLAT_AND, tb.ROUTE_FLAT_OR, tb.ROUTE_CANDIDATE, tb.ROUTE_SCORE_FLAT,
                                     tb.ROUTE_FLAT_TREE, tb.ROUTE_EXEC_TILES)
CODECS = [tb.CODEC_GOOGLE, tb.CODEC_LUCENE]
IDS = ["google", "lucene"]
DOCS_MODES = (tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT)
SCORED_MODES = (tb.MODE_SCORED_ALL, tb.MODE_SCORED_TOPK)
# (plans, their GOOGLE DocumentsOnly routes, the launch's slots): a conjunction of <= 3 terms raises the slot count itself, a wider one
# runs flat only beside a plan that needs as many slots
SLOT_CASES = [([_and(3), _and(4)], [AND, S], 3), ([_wide(6), _and(8), _and(9)], [S, AND, S], 8), ([_wide(13), _and(15), _and(16)], [S, AND, S], 15)]
# bench.py workloads on a small synthetic index: every term's postings spread over the whole docID range, so no plan's range is empty
SYN_DOCS, SYN_TERMS, SYN_NQ = 300_000, 256, 200
WORKLOAD_ROUTES = {"and2": {AND, CAND}, "or10": {SF}, "tree8": {CAND, TREE}, "and2l": {S}}


def _weights(nodes, terms, ndocs):
    for x in nodes:
        if x["kind"] == tb.NODE_TERM and x["term"] != tb.EMPTY_TERM:
            x["weight"] = tb.bm25_idf(int(terms["documents"][x["term"]]), ndocs)
    return nodes


class Source:
    """an index as the planner sees it, and the plans of query texts on it"""

    def __init__(self, codec, lists, names, ndocs):
        b = tb.IndexBuilder(codec)
        for d, f in lists:
            b.add_term(d, f)
        self.codec, self.ndocs, self.index, self.terms = codec, ndocs, b.index(), b.terms_array()
        self.tdict = tb.TermDictionary(names)

    def plans(self, texts, scored):
        return [_weights(tb.parse_query(q, self.tdict), self.terms, self.ndocs) if scored else tb.parse_query(q, self.tdict) for q in texts]

    def routes(self, plans, mode, k=100):
        r, slots = tb.debug_plan(self.codec, self.index, self.terms, plans, mode, k, self.ndocs)
        return r.tolist(), slots[0]


@pytest.fixture(scope="module", params=CODECS, ids=IDS)
def limits(request):
    lists, names = _lists()
    return Source(request.param, lists, names, NDOCS)


class Synth(Source):
    def __init__(self, codec):
        s = tb.SynthIndex(codec, SYN_DOCS, SYN_TERMS, threads=4)
        self.codec, self.ndocs, self.index, self.terms = codec, SYN_DOCS, np.asarray(s.index).copy(), np.asarray(s.terms).copy()
        self.tdict = tb.TermDictionary(s.names)


@pytest.fixture(scope="module")
def synth():
    return {c: Synth(c) for c in CODECS}


def _plan_limit_routes(codec, scored):
    if scored:
        return [PLANS[q][1] if codec == tb.CODEC_LUCENE else TILES for q in PLANS]
    return [PLANS[q][0] if codec == tb.CODEC_GOOGLE else S for q in PLANS]


def _workload(name, synth):
    wl = bench.WORKLOADS[name]
    src = synth[wl["codec"]]
    texts, _ = bench.gen_queries(name, SYN_NQ, SYN_TERMS)
    return src, src.plans(texts, wl["mode"] != tb.MODE_DOCS_ONLY), wl["mode"]


def test_plan_limit_routes(limits):
    for scored, modes in ((False, DOCS_MODES), (True, SCORED_MODES)):
        plans = limits.plans(PLANS, scored)
        for mode in modes:
            assert limits.routes(plans, mode)[0] == _plan_limit_routes(limits.codec, scored), mode


def test_flat_and_needs_a_slot_per_operand(limits):
    """the slot count includes the quirk that a conjunction of <= 3 terms raises it on LUCENE too, where it runs as a step program"""
    for qs, routes, nslots in SLOT_CASES:
        plans = limits.plans(qs, False)
        for mode in DOCS_MODES:
            got, slots = limits.routes(plans, mode)
            assert got == (routes if limits.codec == tb.CODEC_GOOGLE else [S] * len(qs)), (qs, mode)
            assert slots == nslots, (qs, mode)


@pytest.mark.parametrize("name", list(WORKLOAD_ROUTES))
def test_bench_workload_routes(synth, name):
    src, plans, mode = _workload(name, synth)
    got, _ = src.routes(plans, mode)
    # (a GOOGLE conjunction of two distinct terms always has its two slots: flat unless candidate-driven)
    assert set(got) == WORKLOAD_ROUTES[name], (name, sorted(set(got)))


@pytest.mark.parametrize("knob, route", [("TRN_FLAT_SCORED", SF), ("TRN_TREE_SHIFT", TREE), ("TRN_CAND_COST", CAND)])
def test_knob_switches_its_route_off(limits, monkeypatch, knob, route):
    scored = route == SF
    plans = limits.plans(PLANS, scored)
    mode = tb.MODE_SCORED_ALL if scored else tb.MODE_DOCS_ONLY
    before, _ = limits.routes(plans, mode)
    if limits.codec != (tb.CODEC_LUCENE if scored else tb.CODEC_GOOGLE):  # the route exists on one codec only
        assert route not in before
        return
    assert route in before
    monkeypatch.setenv(knob, "0")
    after, _ = limits.routes(plans, mode)
    assert route not in after
    assert [a for a, b in zip(after, before) if b != route] == [b for b in before if b != route]  # the other queries keep their routes


@pytest.mark.gpu
@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_engine_runs_the_planned_routes(synth, monkeypatch, codec):
    """GpuIndexSource.last_routes() == tb.debug_plan for the same batch: single call (TRN_PIPELINE_CHUNKS=1), and a pipelined call (8
    chunks at most, TRN_CHUNK_POSTINGS=1: every DocumentsOnly / SCORED_ALL batch of >= 64 queries is split).  The PLANS routes do not depend
    on which queries share a launch (the flat ANDs among them need at most 3 slots or more than any plan of the batch takes), so they hold
    in every chunk."""
    lists, names = _lists()
    src = Source(codec, lists, names, NDOCS)
    batches = [(src, src.plans(list(PLANS) * 5, scored), scored, True) for scored in (False, True)]
    batches += [(src, src.plans(qs, False), False, False) for qs, _, _ in SLOT_CASES]
    for name, wl in bench.WORKLOADS.items():
        if wl["codec"] == codec:
            s, plans, mode = _workload(name, synth)
            batches.append((s, plans, mode != tb.MODE_DOCS_ONLY, True))
    monkeypatch.setenv("TRN_CHUNK_POSTINGS", "1")
    monkeypatch.setenv("TRN_CHUNK_RULE", "postings")
    for chunked in (False, True):
        monkeypatch.setenv("TRN_PIPELINE_CHUNKS", "8" if chunked else "1")
        gpus = {}
        for s, plans, scored, any_split in batches:
            if chunked and not any_split:
                continue
            if id(s) not in gpus:
                gpus[id(s)] = tb.GpuIndexSource(0)
                gpus[id(s)].upload(codec, s.index, s.terms, s.ndocs)
            g = gpus[id(s)]
            for mode in SCORED_MODES if scored else DOCS_MODES:
                g.exec_batch(plans, mode, k=100, copy=False)
                assert g.last_routes().tolist() == s.routes(plans, mode)[0], (mode, chunked)
                if mode != tb.MODE_SCORED_TOPK:
                    assert (g.last_timings()["chunks"] > 1) == chunked, mode
        for g in gpus.values():
            g.close()
