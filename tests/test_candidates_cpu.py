"""The corpora of test_gpu_candidate_edges reach every switch point of the candidate-driven conjunction (exec_docs_cand.cuh), checked
without a GPU on the index bytes through the host restatements of candutil; the planner gives every query of those tests the route and
the slot counts they assert; and the plain evaluator they use above the reference's reach (candutil.eval_sets) agrees with pyeval and
with the reference's exec_query where both run."""
import os

import numpy as np
import pytest

import candutil as cu
import trinity_b200 as tb
from pyeval import evaluate
from refharness import RefIndex

G = cu.G


@pytest.fixture(scope="module")
def leads():
    lists = cu.lead_corpus()
    return lists, cu.build(lists)


def _tt(terms, names, n):
    return cu.term_tuple(terms, names.index(n))


def test_lead_blocks_take_every_form_of_the_decoder(leads):
    lists, (index, terms, names) = leads
    assert names[-1] == "filler" and "filler" not in {L for L, *_ in cu.LEADS}  # a lead is never the last term of its index
    forms = []
    for L, nb, last_n, _ in cu.LEADS:
        B = cu.Blocks(index, _tt(terms, names, L))
        assert B.nb == nb and B.n[-1] == last_n, L
        # the restated decoder gives back the lead
        assert np.array_equal(np.concatenate([B.block_docs(b) for b in range(B.nb)]).astype(np.uint32), lists[L]), L
        forms += cu.lead_block_forms(index, _tt(terms, names, L))
    mis = {f["mis"] for f in forms}
    assert mis == set(range(16)), sorted(mis)
    why = [f["why"] for f in forms]
    assert min(why.count(w) for w in ("end", "slot", "long")) >= 10, why
    edges = [f["edge"] for f in forms]
    assert edges.count(80) >= 3 and edges.count(81) >= 3  # a 3-byte code ending on slot byte 80, and one ending a byte past it
    full = [f for f in forms if f["n"] == 32]
    assert sum(set(f["lens"]) == {1} for f in full) >= 5
    assert sum(set(f["lens"]) == {2} for f in full) >= 5
    assert sum(set(f["lens"]) == {1, 2} for f in full) >= 5
    for L in (4, 5):  # 4- and 5-byte codes as the first, a middle and the last delta of a block
        for where in ("first", "mid", "last"):
            at = lambda f: {"first": [0], "last": [len(f["lens"]) - 1], "mid": range(1, len(f["lens"]) - 1)}[where]
            assert sum(any(f["lens"][i] == L for i in at(f)) for f in full) >= 1, (L, where)
    # a long code stops the in-slot decode where it lies in the slot
    assert sum(f["why"] == "long" and f["lens"][f["stop"]] == 5 for f in forms) >= 1
    assert {f["n"] for f in forms} >= {1, 2, 31, 32}
    assert sum(f["n"] == 1 for f in forms) >= 2  # (nd == 0)


@pytest.mark.parametrize("probe,dense", [("pn", False), ("pt", False), ("pb", True), ("fp", False), ("fb", True)])
def test_probes_reach_every_switch_point(probe, dense):
    lists = cu.top_corpus() if probe[0] == "f" else cu.probe_corpus()
    index, terms, names = cu.build(lists)
    off, _ = tb.debug_dense_terms(G, index, terms)
    assert (off[names.index(probe)] != tb.DENSE_NONE) == dense
    for n in names:  # the candidate sets and the other probes keep their decoded form
        assert n in ("pb", "fb") or off[names.index(n)] == tb.DENSE_NONE, n
    cands = lists["q" + probe]
    hits, forms = cu.probe_forms(index, _tt(terms, names, probe), cands, dense)
    assert np.array_equal(hits, np.isin(cands, lists[probe])), probe  # the restated probe finds exactly the term's documents
    if dense:
        need = ["bm_low", "bm_high", "bm_first", "bm_last", "bm_base", "bm_end"]
    else:
        need = ["above_last", "below_first", "block_last", "prev_plus_1", "between_blocks", "dp4a_eq1_hit", "dp4a_gt1_miss",
                "step1_hit", "step1_miss", "step2_hit", "step2_miss", "spill3_hit", "spill3_miss", "spill4_hit", "spill4_miss"]
        need += ["no_table"] if probe == "pn" else ["table", "tf_edge"]
        need += ["spill5_hit", "spill5_miss"] if probe == "fp" else []
    if probe[0] == "f":  # nothing lies above 2^32 - 2
        need = [k for k in need if k not in ("above_last", "bm_high", "bm_end")]
    short = {k: forms[k] for k in need if forms[k] < (1 if k in ("above_last", "below_first") or k.startswith("bm_") or k.startswith("spill5") else 3)}
    assert not short, (probe, short, dict(forms))
    if probe in ("fp", "fb"):
        assert int(lists[probe][-1]) == cu.TOP and cu.TOP in cands


def _plan(lists, queries, env):
    index, terms, names = cu.build(lists)
    plans = cu.parse(queries, tb.TermDictionary(names))
    mx = int(max(int(v[-1]) for v in lists.values()))
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        routes, slots = tb.debug_plan(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=mx)
        _, mixed = tb.debug_mixed_runs(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=mx)
    finally:
        for k, v in old.items():
            os.environ.pop(k) if v is None else os.environ.__setitem__(k, v)
    return [int(r) for r in routes], slots, set(mixed[:, 0].tolist())


def test_routes_of_the_gpu_tests():
    C = tb.ROUTE_CANDIDATE
    lq, mq = cu.lead_queries(), cu.mixed_lead_queries()
    assert _plan(cu.lead_corpus(), lq + mq, {"TRN_CAND_COST": "1"})[0] == [C] * len(lq + mq)
    r, _, mixed = _plan(cu.lead_corpus(), mq, {"TRN_CAND_COST": "0"})
    assert r == [tb.ROUTE_FLAT_AND] * len(mq) and mixed == set(range(len(mq)))
    assert _plan(cu.probe_corpus(), cu.PROBE_QUERIES, {"TRN_CAND_COST": "1"})[0] == [C] * len(cu.PROBE_QUERIES)
    assert _plan(cu.top_corpus(), cu.TOP_QUERIES, {"TRN_CAND_COST": "1"})[0] == [C] * len(cu.TOP_QUERIES)
    tq = cu.all_truth_queries()
    assert _plan(cu.truth_corpus(), tq, {"TRN_CAND_COST": "1"})[0] == [C] * len(tq)
    gq = [(q, 0, 0) for q in cu.GROUP_ROUTES]
    assert _plan(cu.group_corpus(), gq, {})[0] == list(cu.GROUP_ROUTES.values())
    for env in ({"TRN_CAND_COST": "0"}, {"TRN_CAND_COST": "0", "TRN_DOCS_SHIFT": "13"}):
        assert C not in _plan(cu.group_corpus(), gq, env)[0]


@pytest.mark.parametrize("docs_shift", [13, 14, 17])
def test_slots_and_mixed_tickets_by_tile_size(docs_shift):
    lists = cu.group_corpus()
    env = {"TRN_DOCS_SHIFT": str(docs_shift)}
    for cands, member in ((cu.CAND_PLAIN, False), (cu.CAND_MEMBER, True)):
        for batch in (cands, cands + cu.FLAT_MIXED):
            qs = [(q, 0, 0) for q in batch]
            r, (nslots, _), mixed = _plan(lists, qs, env)
            index, terms, names = cu.build(lists)
            own = cu.own_slots(index, terms, cu.parse(qs, tb.TermDictionary(names)))
            assert r == [tb.ROUTE_CANDIDATE] * len(cands) + [tb.ROUTE_FLAT_AND] * (len(batch) - len(cands)), batch
            assert nslots == cu.cand_smem_slots(docs_shift, member, own), (batch, nslots, own)
            assert mixed == set(range(len(cands), len(batch))), batch
            if docs_shift == 13:
                assert nslots == (5 if member else 4)
    alone = _plan(lists, [(q, 0, 0) for q in cu.FLAT_MIXED], env)
    assert alone[0] == [tb.ROUTE_FLAT_AND] * len(cu.FLAT_MIXED)
    assert (len(alone[2]) == 0) == (docs_shift == 13)  # at 2^13 only a candidate query's slots make room for the mixed-run tickets


@pytest.fixture(scope="module")
def truth():
    lists = cu.truth_corpus()
    index, terms, names = cu.build(lists)
    return lists, index, terms, names, tb.TermDictionary(names)


def test_probe_order_permutes_the_tree_order(truth):
    lists, index, terms, names, tdict = truth
    qs = cu.all_truth_queries()
    moved = 0
    for q, _, m in qs:
        nodes = tb.parse_query(q, tdict, min_match=m or None)
        tv, _, _ = tb.query_truth_table(nodes)
        order, nnec, _ = cu.probe_order(nodes, terms)
        moved += order != tv
    assert moved * 2 >= len(qs), (moved, len(qs))


def test_every_word_of_the_wide_tables_is_hit_and_missed(truth):
    lists, index, terms, names, tdict = truth
    sets = {names.index(n): set(v.tolist()) for n, v in lists.items()}
    for q, _, m in cu.WIDE_QUERIES:
        nodes = tb.parse_query(q, tdict, min_match=m or None)
        order, nnec, ptable = cu.probe_order(nodes, terms)
        assert len(order) == 8 and nnec < 8
        hit, miss = set(), set()
        for d in lists[names[order[0]]].tolist():  # every candidate of the lead
            pb = sum(1 << j for j, t in enumerate(order) if d in sets[t])
            if pb & ((1 << nnec) - 1) != (1 << nnec) - 1:
                continue  # dropped by a necessary term before the table
            (hit if ptable[pb] else miss).add(pb >> 5)
        assert hit == miss == set(range(8)), (q, sorted(hit), sorted(miss))


def test_eval_sets_equals_pyeval_and_the_reference(ref, truth):
    cases = [(truth[0], cu.all_truth_queries()), (cu.group_corpus(), [(q, 0, 0) for q in cu.GROUP_ROUTES]),
             (cu.probe_corpus(), cu.PROBE_QUERIES)]
    for lists, qs in cases:
        names = list(lists)
        mx = int(max(int(v[-1]) for v in lists.values()))
        r = RefIndex(ref, G)
        for n in names:
            d = np.asarray(lists[n], np.uint32)
            r.add_term(n, d, 1 + d % 3)
        r.finish(mx)
        tdict = tb.TermDictionary(names)
        bylist = {i: np.asarray(lists[n], np.uint32) for i, n in enumerate(names)}
        full = [(bylist[i], np.ones(len(bylist[i]), np.uint32)) for i in range(len(names))]
        for q, flags, m in qs:
            nodes = tb.parse_query(q, tdict, min_match=m or None)
            got = cu.eval_sets(nodes, bylist)
            mask, _ = evaluate(nodes, full, mx)
            assert np.array_equal(got, np.flatnonzero(mask).astype(np.uint32)), q
            want, _ = r.exec(q, False, mx + 1, parser_flags=flags, min_match=m)
            assert np.array_equal(got, want), q
