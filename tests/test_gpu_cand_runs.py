"""The candidate-driven queries on their run-major tickets (BatchPlan::cand_runs; exec_docs.cuh k_exec_docs hands out {query, group}
tickets to cand_exec_google): every batch runs on a source created with TRN_CAND_RUNS=0 (query-order tickets) and on one with the
default, and the two must be equal word for word — per query the plain docID stream and its match count, and in compact mode every work
item's descriptor and every query's replayed stream.  The batches: the candutil corpora (leads of every block form, probes at every
switch point, truth tables of 2 to 8 terms, groups that die and survive beside every other route of the launch, the top of the docID
space), leads whose groups spread over many 2^17-docID runs, masked documents, per-query document filters, exec_batch_device + fetch,
and TRN_DOCS_SHIFT 13 / 14 / 17.  Where test_gpu_candidate_edges checks the same corpora against the reference, this checks that the
ticket order changes nothing."""
import contextlib
import os

import numpy as np
import pytest

import candutil as cu
import trinity_b200 as tb
from test_cand_runs_cpu import QUERIES as SPREAD_QUERIES
from test_cand_runs_cpu import corpus as spread_corpus

pytestmark = pytest.mark.gpu
G = cu.G


@contextlib.contextmanager
def _env(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


class Corpus(dict):
    def __init__(self, lists):
        index, terms, names = cu.build(lists)
        mx = int(max(int(v[-1]) for v in lists.values()))
        super().__init__(index=index, terms=terms, names=names, max_docid=mx, lists=lists, tdict=tb.TermDictionary(names))
        self.ids = {n: i for i, n in enumerate(names)}


@pytest.fixture
def source():
    made = []

    def make(c, env):
        with _env(env):
            g = tb.GpuIndexSource(0)
        g.upload(G, c["index"], c["terms"], c["max_docid"])
        made.append(g)
        return g

    yield make
    for g in made:
        g.close()


def _outputs(g, plans, masked, filters, device):
    """per mode: (routes, match counts, per-query docIDs, compact descriptors)"""
    if masked is not None:
        g.set_masked_documents(masked)
    out = {}
    for mode in (tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT):
        if device:
            g.exec_batch_device(plans, mode, filters=filters)
            res = g.fetch()
        else:
            res = g.exec_batch(plans, mode, filters=filters, copy=False)
        counts = np.asarray(res.match_counts).copy()
        if mode == tb.MODE_DOCS_COMPACT:
            desc = np.ctypeslib.as_array(res.raw.item_desc, shape=(max(res.nitems, 1),))[: res.nitems].copy() if res.raw is not None else None
            docs = [res.decode_query(i).copy() for i in range(len(plans))] if res.raw is not None else [res.query(i)[0].copy() for i in range(len(plans))]
        else:
            desc = None
            docs = [res.query(i)[0].copy() for i in range(len(plans))]
        out[mode] = (list(g.last_routes()), counts, docs, desc)
    return out


def check(source, c, queries, env=None, masked=None, filters=None, device=False, label=""):
    """the batch under env with TRN_CAND_RUNS=0 and with the default: equal word for word; the default must use the run tickets"""
    env = env or {}
    plans = [tb.parse_query(q, c["tdict"], min_match=m or None) for q, _, m in queries] if queries and isinstance(queries[0], tuple) else \
        [tb.parse_query(q, c["tdict"]) for q in queries]
    with _env(env):
        _, tickets = tb.debug_cand_runs(G, c["index"], c["terms"], plans, tb.MODE_DOCS_ONLY, max_docid=c["max_docid"])
    assert len(tickets), f"{label}: the batch takes candidate run tickets"
    filt = None
    runs = {}
    for knob in ("0", None):
        e = dict(env) if knob is None else {**env, "TRN_CAND_RUNS": knob}
        g = source(c, e)
        if filters is not None:
            filt = [None if f is None else tb.DocFilter(g.docset(f[0]) if f[0] is not None else None, g.docset(f[1]) if f[1] is not None else None)
                    for f in filters]
        runs[knob] = _outputs(g, plans, masked, filt, device)
    for mode in (tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT):
        r0, c0, d0, k0 = runs["0"][mode]
        r1, c1, d1, k1 = runs[None][mode]
        assert r0 == r1 and tb.ROUTE_CANDIDATE in r1, (label, r0, r1)
        assert np.array_equal(c0, c1), (label, mode)
        for i in range(len(plans)):
            assert np.array_equal(d0[i], d1[i]), f"{label} mode {mode} query {i}"
        if k0 is not None or k1 is not None:
            assert np.array_equal(k0, k1), (label, "compact descriptors")
    return plans, runs[None][tb.MODE_DOCS_ONLY][2]


def test_leads_probes_top(source):
    c = Corpus(cu.lead_corpus())
    check(source, c, cu.lead_queries(), {"TRN_CAND_COST": "1"}, label="leads")
    c = Corpus(cu.probe_corpus())
    check(source, c, cu.PROBE_QUERIES, {"TRN_CAND_COST": "1"}, label="probes")
    c = Corpus(cu.top_corpus())
    check(source, c, cu.TOP_QUERIES, {"TRN_CAND_COST": "1"}, label="top")


def test_truth_tables(source):
    c = Corpus(cu.truth_corpus())
    check(source, c, cu.all_truth_queries(), {"TRN_CAND_COST": "1"}, label="truth tables")


def test_leads_over_many_runs_with_masked_and_filtered_documents(source):
    lists, _ = spread_corpus()
    c = Corpus(lists)
    _, docs = check(source, c, SPREAD_QUERIES, label="spread")
    assert sum(len(d) for d in docs) > 10_000
    rng = np.random.default_rng(23)
    mx = c["max_docid"]
    masked = np.unique(np.concatenate([rng.choice(lists["l1"], 4000, replace=False), rng.integers(1, mx + 1, 50_000)])).astype(np.uint32)
    check(source, c, SPREAD_QUERIES, masked=masked, label="spread masked")
    allow = np.unique(rng.integers(400_000, 2_200_000, 300_000)).astype(np.uint32)
    deny = np.arange(7, mx + 1, 7, dtype=np.uint32)
    filters = [((allow, None), (None, deny), (allow, deny), None)[i % 4] for i in range(len(SPREAD_QUERIES))]
    check(source, c, SPREAD_QUERIES, masked=masked, filters=filters, label="spread filtered")
    check(source, c, SPREAD_QUERIES, filters=filters, device=True, label="spread device")


@pytest.mark.parametrize("docs_shift", [13, 14, 17])
def test_groups_beside_every_route_at_each_tile_size(source, docs_shift):
    env = {"TRN_DOCS_SHIFT": str(docs_shift)}
    c = Corpus(cu.group_corpus())
    qs = [(q, 0, 0) for q in cu.GROUP_ROUTES]
    check(source, c, qs, env, label=f"groups shift {docs_shift}")
    g_ = np.asarray(c["lists"]["g"], np.uint32)
    masked = np.unique(np.concatenate([g_[:300], g_[2048:3072], np.arange(2, 400_001, 97, dtype=np.uint32)])).astype(np.uint32)
    check(source, c, qs, env, masked=masked, device=True, label=f"groups masked device shift {docs_shift}")
    if docs_shift < 17:  # (at 2^17-docID tiles this batch's slot count leaves no room on an SM for the launch, whatever the tickets)
        lists, _ = spread_corpus()
        check(source, Corpus(lists), SPREAD_QUERIES, env, label=f"spread shift {docs_shift}")
