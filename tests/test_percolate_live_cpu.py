"""Percolator updates — CPU only: a query's program, anchor cover and status depend only on its tree, the vocabulary and the term costs, so
planning a set in slices gives what planning it whole gives (trn_percolator_add plans only the added slice and appends it).  Also the C
ABI's shape of the update calls."""
import ctypes as C

import numpy as np
import pytest

import trinity_b200 as tb
from percutil import CONST_TRUE_SHAPES, EMPTY, EXTRA_SHAPES, VOCAB, query_lists
from test_percolate_cpu import _tree, parse
from trinity_b200._ffi import TrnPercolatorInfo


def random_tree(rng, nterms, depth=0):
    """a random tree as (kind, term or MatchSome min, children): terms, out-of-vocabulary terms, phrases, AND / OR / NOT / OPTIONAL /
    MatchSome"""
    T, P, S = tb.NODE_TERM, tb.NODE_PHRASE, tb.NODE_SOME
    term = (lambda: EMPTY if rng.random() < 0.08 else int(rng.integers(0, nterms)))
    r = rng.random()
    if depth >= 3 or r < 0.3:
        return (T, term(), [])
    if r < 0.45:
        return (P, 0, [(T, term(), []) for _ in range(int(rng.integers(2, 6)))])
    kind = [tb.NODE_AND, tb.NODE_OR, tb.NODE_NOT, tb.NODE_OPTIONAL, S][int(rng.integers(0, 5))]
    n = int(rng.integers(2, 5))
    return (kind, int(rng.integers(0, n + 2)) if kind == S else 0, [random_tree(rng, nterms, depth + 1) for _ in range(n)])


def flatten(t):
    """the trn_qnode array of a (kind, value, children) tree: root 0, the children of a node consecutive"""
    out = [None]

    def place(t, at):
        kind, val, kids = t
        if not kids:
            out[at] = (kind, 0, 0, val)
            return
        first = len(out)
        out.extend([None] * len(kids))
        out[at] = (kind, len(kids), first, val)
        for j, k in enumerate(kids):
            place(k, first + j)

    place(t, 0)
    return _tree(*out)


def trees(rng, n, nterms):
    return [flatten(random_tree(rng, nterms)) for _ in range(n)]


def test_random_trees_are_well_formed_and_varied():
    rng = np.random.default_rng(1)
    ts = trees(rng, 400, 30)
    plan = tb.debug_percolator_plan(ts, 30)
    kinds = set(int(x["kind"]) for t in ts for x in t)
    assert {tb.NODE_PHRASE, tb.NODE_SOME, tb.NODE_NOT, tb.NODE_OPTIONAL, tb.NODE_AND, tb.NODE_OR} <= kinds
    assert {s for s, _ in plan} == {0, 2}


@pytest.mark.parametrize("cost_kind", ["uniform", "ties", "distinct"])
def test_planning_in_slices_equals_planning_whole(cost_kind):
    rng = np.random.default_rng({"uniform": 2, "ties": 3, "distinct": 4}[cost_kind])
    V = len(VOCAB)
    cost = {"uniform": None, "ties": rng.integers(1, 3, size=V), "distinct": rng.permutation(V) + 1}[cost_kind]
    cost = None if cost is None else np.asarray(cost, np.uint32)
    qs = [parse(q, m) for q, _, m in query_lists() + EXTRA_SHAPES + CONST_TRUE_SHAPES] + trees(rng, 600, V)
    order = rng.permutation(len(qs))
    qs = [qs[i] for i in order]
    whole = tb.debug_percolator_plan(qs, V, cost)
    for _ in range(5):
        cuts = np.sort(rng.choice(np.arange(1, len(qs)), size=int(rng.integers(1, 12)), replace=False))
        pieces = []
        for a, b in zip([0, *cuts], [*cuts, len(qs)]):
            pieces += tb.debug_percolator_plan(qs[a:b], V, cost)
        assert pieces == whole
    # one query at a time
    assert [tb.debug_percolator_plan([q], V, cost)[0] for q in qs[:200]] == whole[:200]


def test_slice_refusals_name_the_query_in_the_slice():
    T, O, P = tb.NODE_TERM, tb.NODE_OR, tb.NODE_PHRASE
    ok = _tree((T, 0, 0, 1))
    for bad, rc in ((_tree((T, 0, 0, 40)), -1), (_tree((P, 17, 1, 0), *[(T, 0, 0, 1)] * 17), -1),
                    (_tree((O, 65, 1, 0), *[(T, 0, 0, i % 20) for i in range(65)]), -7)):
        with pytest.raises(tb.TrinityError, match=f"rc={rc}: query 2"):
            tb.debug_percolator_plan([ok, ok, bad, ok], 20)


def test_info_layout_keeps_its_size_and_names_next_id():
    assert C.sizeof(TrnPercolatorInfo) == 32
    names = [f for f, _ in TrnPercolatorInfo._fields_]
    assert names == ["nqueries", "unanchored", "never", "next_id", "anchor_entries", "device_bytes"]
    assert TrnPercolatorInfo.next_id.offset == 12
