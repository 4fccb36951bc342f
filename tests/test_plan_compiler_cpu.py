"""The plan compiler (planner.cpp Compiler == build_iterator + build_span flattened into slot operations) checked WITHOUT a GPU: its step
programs, interpreted on the CPU (tests/stepsim.py), must give the documents and scores of the structural evaluator — which is itself
pinned against the reference's exec_query (test_frontend_cpu).  Covers slot reuse (DocumentsOnly), the deferred scoring passes,
MatchSome counters and the reference's root-filter quirk."""
import numpy as np
import pytest

import stepsim
import trinity_b200 as tb
from pyeval import evaluate
from test_frontend_cpu import EXTRA, NDOCS, OPTIONAL_QUERIES, SOME_QUERIES, TEMPLATES
from util import closed_form_lists

ALL = [(q, None) for q in TEMPLATES + EXTRA + OPTIONAL_QUERIES] + list(SOME_QUERIES)


@pytest.fixture(scope="module")
def built():
    lists = closed_form_lists(NDOCS)
    out = {}
    for codec in (tb.CODEC_GOOGLE, tb.CODEC_LUCENE):
        b = tb.IndexBuilder(codec)
        for d, f in lists:
            b.add_term(d, f)
        out[codec] = (b.index(), b.terms_array())
    return lists, out, tb.TermDictionary([f"t{i + 1}" for i in range(len(lists))])


@pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
@pytest.mark.parametrize("scored", [False, True], ids=["docs", "scored"])
def test_step_programs_match_the_structural_evaluator(built, codec, scored):
    lists, idx, tdict = built
    index, terms = idx[codec]
    worst_slots = 0
    for q, m in ALL:
        nodes = tb.parse_query(q, tdict, min_match=m)
        for x in nodes:
            if x["kind"] == tb.NODE_TERM and x["term"] != tb.EMPTY_TERM:
                x["weight"] = tb.bm25_idf(len(lists[int(x["term"])][0]), NDOCS)
        steps, root_slot, nslots = tb.debug_compile(codec, index, terms, nodes, scored)
        worst_slots = max(worst_slots, nslots)
        got_m, got_s = stepsim.run(steps, root_slot, nslots, lists, NDOCS)
        want_m, want_s = evaluate(nodes, lists, NDOCS, weights=True if scored else None)
        assert np.array_equal(np.flatnonzero(got_m), np.flatnonzero(want_m)), (q, m)
        if scored:
            ids = np.flatnonzero(want_m)
            rel = np.abs(got_s[ids] - want_s[ids]) / np.maximum(np.abs(want_s[ids]), 1e-30)
            assert rel.size == 0 or rel.max() <= 1e-5, (q, m, rel.max())
    assert worst_slots <= 14


def test_docs_only_plans_reuse_slots(built):
    lists, idx, tdict = built
    index, terms = idx[tb.CODEC_GOOGLE]
    q = "(t1 OR t2) AND (t3 OR t4) AND t5 NOT (t6 OR t7 OR t8)"
    nodes = tb.parse_query(q, tdict)
    _, _, docs_slots = tb.debug_compile(tb.CODEC_GOOGLE, index, terms, nodes, False)
    _, _, scored_slots = tb.debug_compile(tb.CODEC_GOOGLE, index, terms, nodes, True)
    assert docs_slots < scored_slots and docs_slots <= 4  # root, conjunction, one disjunction at a time, scratch


TREE8 = ["({0} OR {1}) AND ({2} OR {3}) AND {4} NOT ({5} OR {6} OR {7})", "{0} AND {1} AND {2} NOT {3} NOT {4}",
         "({0} AND {1}) OR ({2} AND {3}) OR ({4} AND {5}) NOT {6} NOT {7}", "{0} AND ({1} OR {2} OR {3}) NOT ({4} AND {5}) AND ({6} OR {7})",
         "{0} AND {1}", "({0} OR {1}) AND {2}", "{0} NOT ({1} AND {2})", "({0} AND ({1} OR ({2} AND {3}))) NOT {4}", "{0} OR ({1} AND {2} AND {3})"]


def _skewed_corpus():
    """12 terms with df from 10 to half of 300 000 documents, and the benchmark's tree shapes over random picks of them: leaves of very
    unequal block counts, which the flat-tree form orders by block count"""
    ndocs = 300_000
    rng = np.random.default_rng(77)
    dfs = [150_000, 100_000, 60_000, 20_000, 6_000, 2_000, 700, 200, 50, 10, 90_000, 3_000]
    lists = []
    for df in dfs:
        d = np.sort(rng.choice(ndocs, size=df, replace=False).astype(np.uint32) + 1)
        lists.append((d, np.ones(df, np.uint32)))
    b = tb.IndexBuilder(tb.CODEC_GOOGLE)
    for d, f in lists:
        b.add_term(d, f)
    names = [f"t{i + 1}" for i in range(len(lists))]
    queries = list(ALL)
    for _ in range(40):
        for tpl in TREE8:
            pick = rng.choice(len(names), size=8, replace=False)
            queries.append((tpl.format(*[names[i] for i in pick]), None))
    return lists, ndocs, b.index(), b.terms_array(), tb.TermDictionary(names), queries


def test_flat_tree_programs_match_the_structural_evaluator(built):
    """the DocumentsOnly program in the form the flat-tree launch of k_exec_docs runs (leaf bitmaps first, slot operations after), on the
    closed-form corpus and on a skewed one"""
    lists, idx, tdict = built
    index, terms = idx[tb.CODEC_GOOGLE]
    corpora = [(lists, NDOCS, index, terms, tdict, ALL, 20), (*_skewed_corpus(), 300)]
    for lists, ndocs, index, terms, tdict, queries, least in corpora:
        transformed = 0
        for q, m in queries:
            nodes = tb.parse_query(q, tdict, min_match=m)
            steps, root_slot, nslots = tb.debug_compile(tb.CODEC_GOOGLE, index, terms, nodes, 2)
            assert nslots <= 31
            markers = [s for s in steps if int(s["op"]) == stepsim.OP_LEAF and int(s["mode"]) == stepsim.M_NONE]
            if markers:  # transformed: markers come first and name slots 0 .. nl-1; no decoding leaf remains
                transformed += 1
                assert [int(s["dst"]) for s in steps[: len(markers)]] == list(range(len(markers)))
                assert not any(int(s["op"]) == stepsim.OP_LEAF and int(s["mode"]) != stepsim.M_NONE for s in steps)
            got_m, _ = stepsim.run(steps, root_slot, nslots, lists, ndocs, tree=True)
            want_m, _ = evaluate(nodes, lists, ndocs, weights=None)
            assert np.array_equal(np.flatnonzero(got_m), np.flatnonzero(want_m)), (q, m)
        assert transformed >= least, (ndocs, transformed)
    with pytest.raises(tb.TrinityError):  # scored is 0, 1 or 2
        tb.debug_compile(tb.CODEC_GOOGLE, index, terms, nodes, 3)
