"""The candidate-driven conjunction (exec_docs_cand.cuh: k_exec_docs -> cand_exec_google) at every switch point of its lead decoder, its
probes, its truth table and its shared-memory layout, against the reference exec_query where the docIDs allow and against the plain
evaluator candutil.eval_sets above that.  Every query asserts the route it took, and every batch runs again on a source created with
TRN_CAND_COST=0 (no candidate-driven query), whose docID streams must be equal.  The corpora and what they reach are pinned on the CPU
by test_candidates_cpu:
  A. leads whose blocks take every form of google_block_to_array, against a term holding every lead document and one holding every
     other one; the same leads as the decoded operand of flat ANDs on the mixed-run tickets (equal to TRN_MIXED_RUNS=0);
  B. probe terms without a table, with a table and with a resident bitmap, candidates at every switch point of the probe;
  C. truth tables of 2 to 8 terms whose probe order is not their tree order, words 4-7 of the 256-bit table included;
  D. groups that die between groups that survive, a group that survives whole, a result the size of its segment bound, masked
     documents, compact mode, exec_batch_device + fetch and the pipelined batch, beside every other route of the launch;
  E. TRN_DOCS_SHIFT 13 / 14 / 17: the slot count a candidate query sets, and the mixed-run tickets it switches on at 13;
  F. the top of the docID space (2^32 - 2; 2^32 - 1 is the kernel's empty candidate)."""
import contextlib
import os

import numpy as np
import pytest

import candutil as cu
import trinity_b200 as tb
from refharness import RefIndex
from util import assert_same_docs

pytestmark = pytest.mark.gpu
G = cu.G
REF_LIMIT = 1 << 26  # corpora below this docID are checked against the reference too


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


@pytest.fixture
def source():
    """source(corpus, env) -> GpuIndexSource created under env (the knobs are read when it is created) with the corpus uploaded"""
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


class Corpus(dict):
    def __init__(self, lists, ref=None):
        index, terms, names = cu.build(lists)
        mx = int(max(int(v[-1]) for v in lists.values()))
        super().__init__(index=index, terms=terms, names=names, max_docid=mx, lists=lists, tdict=tb.TermDictionary(names))
        self.ids = {n: i for i, n in enumerate(names)}
        self.ref = None
        if ref is not None and mx < REF_LIMIT:
            self.ref = RefIndex(ref, G)
            for n in names:
                d = np.asarray(lists[n], np.uint32)
                self.ref.add_term(n, d, 1 + d % 3)
            self.ref.finish(mx)

    def want(self, queries, plans, masked=None):
        out = []
        bylist = {self.ids[n]: np.asarray(v, np.uint32) for n, v in self["lists"].items()}
        if masked is not None:
            bylist = {t: np.setdiff1d(v, masked, assume_unique=True) for t, v in bylist.items()}
        for (q, flags, m), p in zip(queries, plans):
            w = cu.eval_sets(p, bylist)
            if self.ref is not None:
                if masked is None:
                    r, _ = self.ref.exec(q, False, self["max_docid"] + 1, parser_flags=flags, min_match=m)
                else:
                    r, _ = self.ref.exec_masked(q, False, masked, self["max_docid"] + 1)
                assert_same_docs(w, r, f"[{q}] evaluator vs reference")
            out.append(w)
        return out


def _run(g, plans, mode=tb.MODE_DOCS_ONLY):
    res = g.exec_batch(plans, mode, copy=mode != tb.MODE_DOCS_COMPACT)  # (the compact stream is replayed from the raw result)
    if mode == tb.MODE_DOCS_COMPACT:
        return [res.decode_query(i).copy() for i in range(len(plans))], list(g.last_routes()), res
    return [res.query(i)[0].copy() for i in range(len(plans))], list(g.last_routes()), res


def check(source, c, queries, routes, env, want=None, masked=None, label=""):
    """the batch on a source under env (routes as given) and under env + TRN_CAND_COST=0: equal streams, equal to want"""
    plans = cu.parse(queries, c["tdict"])
    want = want if want is not None else c.want(queries, plans, masked)
    for cost in (None, "0"):
        e = dict(env) if cost is None else {**env, "TRN_CAND_COST": cost}
        g = source(c, e)
        if masked is not None:
            g.set_masked_documents(masked)
        docs, r, res = _run(g, plans)
        if cost is None:
            assert r == list(routes), (label, r, list(routes))
        else:
            assert tb.ROUTE_CANDIDATE not in r, (label, r)
        for i, (q, _, m) in enumerate(queries):
            assert_same_docs(docs[i], want[i], f"{label} [{q}] min={m} cost={cost or env.get('TRN_CAND_COST', 'default')}")
            assert int(res.match_counts[i]) == len(want[i])
    return plans, want


def test_lead_decoder(source, ref):
    c = Corpus(cu.lead_corpus(), ref)
    qs = cu.lead_queries()
    check(source, c, qs, [tb.ROUTE_CANDIDATE] * len(qs), {"TRN_CAND_COST": "1"}, label="A")
    for (q, _, _), w in zip(qs, c.want(qs, cu.parse(qs, c["tdict"]))):
        lead = q.split()[0]
        L = c["lists"][lead]
        assert np.array_equal(w, L if q.endswith("h") else L[::2]), q


def test_lead_decoder_on_mixed_run_tickets(source):
    c = Corpus(cu.lead_corpus())
    qs = cu.mixed_lead_queries()
    plans = cu.parse(qs, c["tdict"])
    env = {"TRN_CAND_COST": "0"}
    with _env(env):
        _, tickets = tb.debug_mixed_runs(G, c["index"], c["terms"], plans, tb.MODE_DOCS_ONLY, max_docid=c["max_docid"])
    assert set(tickets[:, 0].tolist()) == set(range(len(qs)))
    want = c.want(qs, plans)
    for runs in ("1", "0"):
        g = source(c, {**env, "TRN_MIXED_RUNS": runs})
        docs, r, _ = _run(g, plans)
        assert r == [tb.ROUTE_FLAT_AND] * len(qs)
        for i, (q, _, _) in enumerate(qs):
            assert_same_docs(docs[i], want[i], f"A mixed runs {runs} [{q}]")
    # and the same queries candidate-driven
    check(source, c, qs, [tb.ROUTE_CANDIDATE] * len(qs), {"TRN_CAND_COST": "1"}, want=want, label="A as candidates")


def test_probes(source, ref):
    c = Corpus(cu.probe_corpus(), ref)
    assert c.ref is not None
    qs = cu.PROBE_QUERIES
    check(source, c, qs, [tb.ROUTE_CANDIDATE] * len(qs), {"TRN_CAND_COST": "1"}, label="B")


def test_truth_tables(source, ref):
    c = Corpus(cu.truth_corpus(), ref)
    assert c.ref is not None
    qs = cu.all_truth_queries()
    check(source, c, qs, [tb.ROUTE_CANDIDATE] * len(qs), {"TRN_CAND_COST": "1"}, label="C")


def _group_batch():
    qs = [(q, 0, 0) for q in cu.GROUP_ROUTES]
    return qs, list(cu.GROUP_ROUTES.values())


def test_groups_and_emission(source, ref):
    c = Corpus(cu.group_corpus(), ref)
    assert c.ref is not None
    qs, routes = _group_batch()
    plans, want = check(source, c, qs, routes, {}, label="D")
    g_ = np.asarray(c["lists"]["g"])
    grp = np.arange(len(g_)) // 1024
    w = want[0]
    assert np.array_equal(w, g_[np.isin(grp, [0, 2, 4, 5])])  # groups 1 and 3 die at the first probe, group 0 survives whole
    assert np.array_equal(want[1], g_)
    # the result is exactly its segment bound: the query alone in a batch
    check(source, c, qs[1:2], routes[1:2], {"TRN_PIPELINE_CHUNKS": "1"}, want=want[1:2], label="D bound")
    # compact mode replays to the DocumentsOnly stream; exec_batch_device + fetch is exec_batch
    g = source(c, {})
    docs, r, _ = _run(g, plans)
    comp, rc, _ = _run(g, plans, tb.MODE_DOCS_COMPACT)
    assert rc == r == routes
    g.exec_batch_device(plans, tb.MODE_DOCS_ONLY)
    dev = g.fetch()
    for i, (q, _, _) in enumerate(qs):
        assert_same_docs(comp[i], docs[i], f"D compact [{q}]")
        assert_same_docs(dev.query(i)[0], docs[i], f"D device [{q}]")
    # a pipelined batch of 8 chunks equals the single-call batch
    many = plans * 10
    single = source(c, {"TRN_PIPELINE_CHUNKS": "1"})
    one, _, _ = _run(single, many)
    assert single.last_timings()["chunks"] == 1
    piped = source(c, {"TRN_PIPELINE_CHUNKS": "8", "TRN_CHUNK_POSTINGS": "1", "TRN_CHUNK_RULE": "postings"})
    eight, _, _ = _run(piped, many)
    assert piped.last_timings()["chunks"] >= 8
    for i in range(len(many)):
        assert_same_docs(eight[i], one[i], f"D pipelined [{qs[i % len(qs)][0]}]")


def test_masked_documents(source, ref):
    c = Corpus(cu.group_corpus(), ref)
    qs, routes = _group_batch()
    g_ = np.asarray(c["lists"]["g"], np.uint32)
    rng = np.random.default_rng(11)
    blocks = cu.Blocks(c["index"], cu.term_tuple(c["terms"], c.ids["g"]))
    masked = np.unique(np.concatenate([
        rng.choice(g_[:1024], 300, replace=False),  # candidates of the group that survives whole
        np.asarray(blocks.last[128:160], np.uint32),  # block lasts (group 4)
        g_[2048:3072],  # all of group 2
        rng.choice(np.arange(2, 400_001, 2, dtype=np.uint32), 5000, replace=False),  # documents of the probe that are not candidates
    ])).astype(np.uint32)
    above = np.array([c["max_docid"] + 1, c["max_docid"] + 77, cu.TOP], np.uint32)  # above max_docid: ignored
    check(source, c, qs, routes, {}, masked=np.concatenate([masked, above]), want=c.want(qs, cu.parse(qs, c["tdict"]), masked), label="D masked")


@pytest.mark.parametrize("docs_shift", [13, 14, 17])
def test_shared_memory_and_tile_size(source, ref, docs_shift):
    c = Corpus(cu.group_corpus(), ref)
    env = {"TRN_DOCS_SHIFT": str(docs_shift)}
    for cands, member in ((cu.CAND_PLAIN, False), (cu.CAND_MEMBER, True)):
        for batch in (cands, cands + cu.FLAT_MIXED):
            qs = [(q, 0, 0) for q in batch]
            plans = cu.parse(qs, c["tdict"])
            routes = [tb.ROUTE_CANDIDATE] * len(cands) + [tb.ROUTE_FLAT_AND] * (len(batch) - len(cands))
            with _env(env):
                r, (nslots, _) = tb.debug_plan(G, c["index"], c["terms"], plans, tb.MODE_DOCS_ONLY, max_docid=c["max_docid"])
                _, mixed = tb.debug_mixed_runs(G, c["index"], c["terms"], plans, tb.MODE_DOCS_ONLY, max_docid=c["max_docid"])
            own = cu.own_slots(c["index"], c["terms"], plans)
            assert list(r) == routes
            assert nslots == cu.cand_smem_slots(docs_shift, member, own), (batch, nslots, own)
            if docs_shift == 13:
                assert nslots == (5 if member else 4)
                assert set(mixed[:, 0].tolist()) == set(range(len(cands), len(batch)))  # the candidate query switches them on
            check(source, c, qs, routes, env, label=f"E shift {docs_shift} {batch}")
    if docs_shift == 13:  # the flat ANDs alone keep their per-tile tickets
        qs = [(q, 0, 0) for q in cu.FLAT_MIXED]
        plans = cu.parse(qs, c["tdict"])
        with _env(env):
            _, mixed = tb.debug_mixed_runs(G, c["index"], c["terms"], plans, tb.MODE_DOCS_ONLY, max_docid=c["max_docid"])
        assert len(mixed) == 0
        check(source, c, qs, [tb.ROUTE_FLAT_AND] * len(qs), env, label="E flat ANDs alone")


def test_top_of_the_docid_space(source):
    c = Corpus(cu.top_corpus())
    assert c["max_docid"] == cu.TOP
    qs = cu.TOP_QUERIES
    plans, want = check(source, c, qs, [tb.ROUTE_CANDIDATE] * len(qs), {"TRN_CAND_COST": "1"}, label="F")
    assert np.array_equal(want[0], c["lists"]["fl"]) and int(want[0][-1]) == cu.TOP
    assert all(int(w.max(initial=0)) <= cu.TOP for w in want)
    assert cu.TOP in want[1] and cu.TOP in want[3] and cu.TOP in want[4]
