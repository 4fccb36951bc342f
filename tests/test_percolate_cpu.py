"""Percolator — CPU only: the registry's meaning (a Python evaluator of the query tree on token sequences) against the reference's own
percolator_query::match, the soundness of the anchor covers and the first-anchor rule, and the registration planner (trn_debug_percolator_plan)
against a Python restatement of its cover rules."""
import numpy as np
import pytest

import trinity_b200 as tb
from percutil import (CONST_TRUE_SHAPES, EMPTY, EXTRA_SHAPES, NEVER, UNANCHORED, VOCAB, RefPercolator, cover, evaluate, query_lists, random_docs,
                      tokens_of)
from trinity_b200._ffi import QNODE_DTYPE

TD = tb.TermDictionary(VOCAB)


def parse(q, m):
    return tb.parse_query(q, TD, min_match=m if m else None)


def edge_docs():
    """empty, only out-of-vocabulary tokens, phrases at the first and the last position, `w1 <oov>`, repeated terms, one token"""
    names = [[], ["oov1", "oov2", "oov3"], ["w1", "w2", "t5"], ["t5", "t6", "w1", "w2"], ["w1", "oov2"], ["w1", "w1", "w1"], ["w1"],
             ["w2", "w1", "w2", "w1", "w2"], ["w1", "w2", "w3", "w4", "w5", "w6", "w7", "w8", "w9", "w1", "w2", "w3", "w4", "w5", "w6", "w7"],
             ["t1", "t2", "t3", "t4", "t5", "t6", "t7", "t8", "t9", "t10"], ["w3", "w4", "w3"]]
    return [tokens_of(n, TD) for n in names]


SHAPES = query_lists() + EXTRA_SHAPES


def test_evaluator_matches_reference_percolator():
    rng = np.random.default_rng(7)
    docs = edge_docs() + random_docs(rng, 300, max_len=30) + random_docs(rng, 100, vocab=6, max_len=8, oov=0.3)
    want = RefPercolator(SHAPES).run(docs)
    for qi, (q, f, m) in enumerate(SHAPES):
        nodes = parse(q, m)
        got = [evaluate(nodes, d) for d in docs]
        ref = [qi in set(w.tolist()) for w in want]
        assert got == ref, (q, m, [i for i in range(len(docs)) if got[i] != ref[i]][:5])


def test_const_true_outside_a_conjunction_keeps_its_tree_meaning():
    """`<e>` not beside a conjunction operand: the front-end drops the wrapper, so the tree means e; the reference's percolator evaluates
    consttrueexpr as true.  Pinned: the registry answers with the tree's meaning (documented in include/trinity_b200.h)."""
    rng = np.random.default_rng(8)
    docs = edge_docs() + random_docs(rng, 200, max_len=12)
    want = RefPercolator(CONST_TRUE_SHAPES).run(docs)
    assert all(0 in set(w.tolist()) for w in want)  # <t1> matches every document in the reference's percolator
    t1 = TD.term_id("t1")
    nodes = parse("<t1>", 0)
    assert len(nodes) == 1 and int(nodes[0]["term"]) == t1
    assert [evaluate(nodes, d) for d in docs] == [bool(np.any(d == t1)) for d in docs]


def _pairs_docs(rng, nodes, n):
    """n documents biased towards the query's own terms, so that a fair share matches"""
    ts = sorted(set(int(x["term"]) for x in nodes if x["kind"] == tb.NODE_TERM and x["term"] != EMPTY)) or [0]
    out = []
    for _ in range(n):
        L = int(rng.integers(0, 10))
        pool = np.array(ts + list(rng.integers(0, len(VOCAB), size=3)) + [EMPTY], np.uint32)
        out.append(pool[rng.integers(0, len(pool), size=L)])
    return out


@pytest.mark.parametrize("cost_kind", ["uniform", "ties"])
def test_anchor_covers_are_sound_and_each_match_is_evaluated_once(cost_kind):
    rng = np.random.default_rng(11)
    cost = None if cost_kind == "uniform" else rng.integers(1, 4, size=len(VOCAB)).astype(np.uint32)
    queries = [parse(q, m) for q, _, m in SHAPES]
    plan = tb.debug_percolator_plan(queries, len(VOCAB), cost)
    for nodes, (status, cov) in zip(queries, plan):
        docs = _pairs_docs(rng, nodes, 10_000)
        for d in docs:
            held = set(int(t) for t in d)
            if status == 2:  # cannot match: never evaluated
                assert not evaluate(nodes, d)
                continue
            if status == 1:
                continue
            evaluated = sum(1 for j, t in enumerate(cov) if t in held and not any(u in held for u in cov[:j]))  # the first-anchor rule
            assert evaluated == (1 if held & set(cov) else 0)
            if evaluate(nodes, d):
                assert held & set(cov), (nodes, d, cov)


@pytest.mark.parametrize("cost_kind", ["uniform", "ties", "distinct"])
def test_registration_plan_matches_python_restatement(cost_kind):
    rng = np.random.default_rng(3)
    cost = {"uniform": None, "ties": rng.integers(1, 3, size=len(VOCAB)), "distinct": rng.permutation(len(VOCAB)) + 1}[cost_kind]
    cost = None if cost is None else np.asarray(cost, np.uint32)
    queries = [parse(q, m) for q, _, m in SHAPES + CONST_TRUE_SHAPES]
    plan = tb.debug_percolator_plan(queries, len(VOCAB), cost)
    kinds = {"set": 0, UNANCHORED: 1, NEVER: 2}
    seen = set()
    for nodes, (status, cov) in zip(queries, plan):
        k, ts, _ = cover(nodes, cost)
        assert (status, cov) == (kinds[k], list(ts)), (nodes, status, cov, k, ts)
        seen.add(status)
    assert seen == {0, 2}  # trees have no const-true form: nothing is unanchored


def _tree(*nodes):
    a = np.zeros(len(nodes), QNODE_DTYPE)
    for i, n in enumerate(nodes):
        a[i] = n + (0.0,) if len(n) == 4 else n
    return a


def test_unanchored_and_never_combine_as_stated():
    """the cover rules on hand-built trees: SOME over more operands than can match, NOT over a term outside the vocabulary, an AND with an
    operand that cannot match, an OR that drops one"""
    T, A, O, N, S = tb.NODE_TERM, tb.NODE_AND, tb.NODE_OR, tb.NODE_NOT, tb.NODE_SOME
    cases = [
        (_tree((S, 3, 1, 2), (T, 0, 0, 3), (T, 0, 0, EMPTY), (T, 0, 0, 5)), (0, [3])),         # min 2 of the 2 that can match: both are needed, one anchors
        (_tree((S, 3, 1, 3), (T, 0, 0, 3), (T, 0, 0, EMPTY), (T, 0, 0, 5)), (2, [])),          # min 3 > 2 that can match
        (_tree((S, 2, 1, 0), (T, 0, 0, 3), (T, 0, 0, 5)), (2, [])),                            # min 0: the reference's matchsome never matches
        (_tree((N, 2, 1, 0), (T, 0, 0, EMPTY), (T, 0, 0, 5)), (2, [])),
        (_tree((A, 2, 1, 0), (T, 0, 0, 7), (T, 0, 0, EMPTY)), (2, [])),
        (_tree((O, 2, 1, 0), (T, 0, 0, 7), (T, 0, 0, EMPTY)), (0, [7])),
        (_tree((A, 2, 1, 0), (T, 0, 0, 9), (T, 0, 0, 2)), (0, [2])),                           # equal costs: the lower term id
    ]
    for nodes, want in cases:
        assert tb.debug_percolator_plan([nodes], 20)[0] == want
        k, ts, _ = cover(nodes, None)
        assert ({"set": 0, UNANCHORED: 1, NEVER: 2}[k], list(ts)) == want
    assert not evaluate(cases[2][0], np.array([3, 5], np.uint32))


def test_registration_refusals():
    T, O, P = tb.NODE_TERM, tb.NODE_OR, tb.NODE_PHRASE
    ok = _tree((O, 2, 1, 0), (T, 0, 0, 1), (T, 0, 0, 2))
    cases = {
        "malformed": (_tree((O, 2, 0, 0), (T, 0, 0, 1)), -1),
        "term out of range": (_tree((T, 0, 0, 40)), -1),
        "phrase of 17 terms": (_tree((P, 17, 1, 0), *[(T, 0, 0, 1)] * 17), -1),
        "65 operands": (_tree((O, 65, 1, 0), *[(T, 0, 0, i % 20) for i in range(65)]), -7),
    }
    for name, (nodes, rc) in cases.items():
        with pytest.raises(tb.TrinityError, match=f"rc={rc}: query 1"):
            tb.debug_percolator_plan([ok, nodes], 20)
    tb.debug_percolator_plan([_tree((O, 64, 1, 0), *[(T, 0, 0, i % 20) for i in range(64)])], 20)  # 64 operands fit
    assert tb.debug_percolator_plan([_tree((P, 16, 1, 0), *[(T, 0, 0, 1)] * 16)], 20) == [(0, [1])]
