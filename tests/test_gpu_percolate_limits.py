"""The percolator on the device at its internal switch points, on both sides: the short and the long launch (kPercShortLen = 512), the
distinct-term table (32 slots up to 16 tokens, doubling to 16 384 slots from 8 192 tokens on), a 16-term phrase at the first and the last
position, the sorted and the bitmap output (kPercSortCap = 4096, a partial last bitmap word), programs of exactly kPercStack = 64 pending
operands, and the exact count of (document, query) pairs evaluated, against the reference's percolator_query::match or the registry's
meaning (percutil.evaluate, pinned against the reference in test_percolate_cpu)."""
import numpy as np
import pytest

import trinity_b200 as tb
from percutil import EMPTY, EXTRA_SHAPES, VOCAB, RefPercolator, cover, evaluate, query_lists, random_docs
from test_gpu_percolate import assert_same
from test_percolate_cpu import TD, _tree, parse

pytestmark = pytest.mark.gpu
T, A, O, N, OPT, S, P = tb.NODE_TERM, tb.NODE_AND, tb.NODE_OR, tb.NODE_NOT, tb.NODE_OPTIONAL, tb.NODE_SOME, tb.NODE_PHRASE
LENS = [16, 17, 511, 512, 513, 8192, 8193, 16383]
SHORT_LEN = 512  # kPercShortLen


def hash_slots(L):
    """perc_hash_slots: a power of two >= 2 L, at least 32, at most 16 384"""
    H = 32
    while H < 2 * L and H < 16384:
        H *= 2
    return H


def check_evaluated(p, queries, docs):
    r = p.percolate(docs)
    for d, x in enumerate(docs):
        want = [q for q, nodes in enumerate(queries) if evaluate(nodes, x)]
        assert r.document(d).tolist() == want, (d, len(x))
    return r


def test_document_lengths_against_the_reference():
    """every query shape of the suite on documents of each switch length, in one batch, then the short and the long ones alone"""
    assert [hash_slots(L) for L in LENS] == [32, 64, 1024, 1024, 2048, 16384, 16384, 16384]
    shapes = query_lists() + EXTRA_SHAPES
    p = tb.Percolator([parse(q, m) for q, _, m in shapes], nterms=len(VOCAB))
    docs = random_docs(np.random.default_rng(21), len(LENS), lens=LENS, oov=0.05)
    want = RefPercolator(shapes).run(docs)
    short = [i for i, L in enumerate(LENS) if L <= SHORT_LEN]
    long_ = [i for i, L in enumerate(LENS) if L > SHORT_LEN]
    for part in (list(range(len(LENS))), short, long_):
        r = p.percolate([docs[i] for i in part])
        assert r.long_docs == sum(LENS[i] > SHORT_LEN for i in part)
        assert_same(r, [want[i] for i in part], f"lengths {[LENS[i] for i in part]}")
    assert all(len(w) for w in want)


def test_document_lengths_with_distinct_terms():
    """documents whose tokens are all distinct, so each length fills its table to the bound (16 383 terms in 16 384 slots); term and
    two-term phrase queries over a 40 000-term vocabulary, some on each document's own tokens"""
    rng = np.random.default_rng(22)
    V = 40_000
    docs = [rng.permutation(V)[:L].astype(np.uint32) for L in LENS]
    qs = [_tree((T, 0, 0, int(t))) for t in rng.choice(V, 1500, replace=False)]
    for x in docs:
        for i in rng.integers(0, len(x) - 1, 40):
            qs.append(_tree((P, 2, 1, 0), (T, 0, 0, int(x[i])), (T, 0, 0, int(x[i + 1]))))
        qs.append(_tree((P, 2, 1, 0), (T, 0, 0, int(x[-1])), (T, 0, 0, int(x[0]))))  # both terms present, not adjacent
        qs.append(_tree((A, 2, 1, 0), (T, 0, 0, int(x[0])), (T, 0, 0, int(x[-1]))))
    p = tb.Percolator(qs, nterms=V)
    for part in (docs, docs[:4], docs[4:]):
        r = check_evaluated(p, qs, part)
        assert r.long_docs == sum(len(x) > SHORT_LEN for x in part)


def test_sixteen_term_phrase_at_both_ends_of_512_and_513_tokens():
    """a 16-term phrase anchored on its term at j = 0 and one anchored at j = 15 (term_cost makes that term the cheapest), at the first
    and the last position of a 512-token (short launch) and a 513-token (long launch) document; cut by either end it does not match"""
    ids = [TD.term_id(v) for v in VOCAB[:16]]
    x = ids[0]
    a = ids  # x at j = 0
    b = ids[1:] + [x]  # x at j = 15
    texts = [('"' + " ".join(VOCAB[t] for t in ph) + '"', 0, 0) for ph in (a, b)]
    trees = [parse(q, 0) for q, _, _ in texts]
    cost = np.full(len(VOCAB), 5, np.uint32)
    cost[x] = 1
    assert tb.debug_percolator_plan(trees, len(VOCAB), cost) == [(0, [x]), (0, [x])]
    assert [int(trees[k][0]["kind"]) for k in (0, 1)] == [P, P]
    fill = TD.term_id(VOCAB[17])
    docs = []
    for L in (512, 513):
        for ph in (a, b):
            for at in ("first", "last", "cut-end", "cut-start"):
                d = np.full(L, fill, np.uint32)
                d[L // 2] = EMPTY
                if at == "first":
                    d[:16] = ph
                elif at == "last":
                    d[L - 16:] = ph
                elif at == "cut-end":
                    d[L - 15:] = ph[:15]
                else:
                    d[:15] = ph[1:]
                docs.append(d)
    p = tb.Percolator(trees, nterms=len(VOCAB), term_cost=cost)
    r = p.percolate(docs)
    assert r.long_docs == 8
    want = RefPercolator(texts).run(docs)
    assert_same(r, want, "16-term phrases")
    got = [r.document(i).tolist() for i in range(len(docs))]
    for L in range(2):
        for k in range(2):
            assert got[L * 8 + k * 4: L * 8 + k * 4 + 4] == [[k], [k], [], []]


def test_sorted_and_bitmap_output_at_the_sort_cap():
    """documents matching exactly 0, 1, 4 096 (sorted in shared memory) and 4 097 (the bitmap) queries and every query; the registry has
    nq % 32 != 0, and the 4 097-match document holds the last query id, in the partial last bitmap word"""
    rng = np.random.default_rng(23)
    nq = 4096 + 900 + 1
    assert nq % 32
    a, b, c, d = (TD.term_id(v) for v in ("t1", "t2", "t3", "t4"))
    on_a = np.zeros(nq, bool)
    on_a[rng.choice(nq - 1, 4096, replace=False)] = True  # scattered ids: the sort has work to do
    term = np.where(on_a, a, b)
    term[-1] = c
    p = tb.Percolator([_tree((T, 0, 0, int(t))) for t in term], nterms=len(VOCAB))
    docs = [np.array(x, np.uint32) for x in ([d], [c], [a], [a, c], [a, b, c], [c, EMPTY, a], [])]
    r = p.percolate(docs)
    ids_a = np.flatnonzero(on_a)
    want = [[], [nq - 1], ids_a, np.r_[ids_a, nq - 1], np.arange(nq), np.r_[ids_a, nq - 1], []]
    assert_same(r, want, "sort cap")
    assert [len(w) for w in want[:4]] == [0, 1, 4096, 4097]
    assert r.dense_docs == 3 and r.long_docs == 0


def chain(ops, terms, w):
    """a right-nested tree: level k is ops[k] over w terms and then level k + 1; the last level holds the remaining terms.  Every level
    leaves w operands pending, so the last one finds len(terms) operands on the stack"""
    nodes, at = [], 0
    for k, op in enumerate(ops):
        last = k == len(ops) - 1
        mine = terms[at:] if last else terms[at: at + w]
        i = len(nodes)
        nodes.append((op, len(mine) + (not last), i + 1, 1 if op == S else 0))
        nodes += [(T, 0, 0, t) for t in mine]
        at += len(mine)
    return _tree(*nodes)


def flat(kind, n, m=0, first=0):
    return _tree((kind, n, 1, m), *[(T, 0, 0, first + j) for j in range(n)])


def split(kind, n):
    """kind(term 0, OR(terms 1 .. n - 1)): the first operand sits at the bottom of a stack of n"""
    return _tree((kind, 2, 1, 0), (T, 0, 0, 0), (O, n - 1, 3, 0), *[(T, 0, 0, 1 + j) for j in range(n - 1)])


def stack_queries(n):
    """the shapes at n pending operands: flat AND, OR and MatchSome (min n - 1 and n), NOT and Optional whose first operand is the deepest,
    and nested trees whose operands pile up across levels (3 per level; 1 per level, alternating AND / OR / NOT / MatchSome, 62 levels)"""
    deep = [[A, O, N, S][k % 4] for k in range(n - 2)]
    return {"and": flat(A, n), "or": flat(O, n), f"some-{n - 1}": flat(S, n, n - 1), f"some-{n}": flat(S, n, n), "not": split(N, n),
            "optional": split(OPT, n), "nested": chain([[A, O, S][k % 3] for k in range(20)], list(range(n)), 3),
            "nested-deep": chain(deep, list(range(n - 1, -1, -1)), 1)}


def test_programs_of_exactly_64_pending_operands():
    V = 80
    qs = stack_queries(64)
    for name, nodes in stack_queries(65).items():  # one operand more is refused, whatever the shape
        with pytest.raises(tb.TrinityError, match="rc=-7: query 0: .*65 pending operands"):
            tb.debug_percolator_plan([nodes], V)
    trees = list(qs.values())
    assert [s for s, _ in tb.debug_percolator_plan(trees, V)] == [0] * len(trees)
    rng = np.random.default_rng(24)
    every = np.arange(64, dtype=np.uint32)
    docs = [every, every[1:], every[:-1], every[:63], every[:62], every[2:], np.array([0], np.uint32), np.array([63], np.uint32),
            np.array([0, 63], np.uint32), np.array([0, 64, 70], np.uint32), np.array([1, 2], np.uint32), np.zeros(0, np.uint32)]
    for k in (1, 31, 62):
        docs.append(np.delete(every, k))
    for _ in range(300):  # subsets of every density; the nested chains hinge on their deepest terms
        keep = rng.random(64) < rng.choice([0.03, 0.5, 0.9, 0.97, 0.99])
        x = every[keep]
        docs.append(rng.permutation(np.r_[x, rng.integers(64, V, 3)]).astype(np.uint32))
    p = tb.Percolator(trees, nterms=V)
    r = check_evaluated(p, trees, docs)
    for q, name in enumerate(qs):
        hits = sum(q in set(r.document(d).tolist()) for d in range(len(docs)))
        assert 0 < hits < len(docs), name  # documents on both sides of every answer


def test_candidates_are_exact():
    """queries anchored on 1 .. 64 terms, documents holding all of a query's anchors, only the first, only the last or none: each
    (document, query) pair with an anchor present is evaluated exactly once (at its first anchor present)"""
    V = 300
    qs = []
    for k in (1, 2, 3, 17, 63, 64):
        for s in (0, 100, 236):
            qs.append(flat(O, k, first=s))  # cover: its k terms
    qs.append(_tree((A, 3, 1, 0), (T, 0, 0, 5), (T, 0, 0, 150), (T, 0, 0, 299)))  # cover: one of them
    qs.append(_tree((S, 4, 1, 2), *[(T, 0, 0, t) for t in (10, 110, 210, 290)]))  # cover: three of them
    qs.append(_tree((T, 0, 0, EMPTY)))  # never
    plan = tb.debug_percolator_plan(qs, V)
    covers = [set(c) for _, c in plan]
    assert max(len(c) for c in covers) == 64 and plan[-1][0] == 2
    for nodes, (st, cv) in zip(qs, plan):
        k, ts, _ = cover(nodes, None)
        assert list(ts) == cv and st == {"set": 0, "unanchored": 1, "never": 2}[k]
    docs = []
    for c in covers[:-1]:
        c = sorted(c)
        docs += [np.array(c, np.uint32), np.array([c[0]], np.uint32), np.array([c[-1]], np.uint32), np.array([c[0], c[-1], 299], np.uint32)]
    rng = np.random.default_rng(25)
    docs += [rng.integers(0, V, rng.integers(0, 80)).astype(np.uint32) for _ in range(100)]
    docs += [np.array([EMPTY, EMPTY], np.uint32), np.zeros(0, np.uint32)]
    p = tb.Percolator(qs, nterms=V)
    # no tree is unanchored: a TERM or PHRASE leaf is anchored or never matches, and the cover rules (percplan.h) only pass an
    # unanchored operand upwards, so the unanchored list stays empty (test_registration_plan_matches_python_restatement pins it too)
    assert p.info()["unanchored"] == 0 and p.info()["never"] == 1
    r = check_evaluated(p, qs, docs)
    want = sum(bool(c & set(x.tolist())) for x in docs for c in covers)
    assert r.candidates == want + p.info()["unanchored"] * len(docs)
    assert r.candidates > r.total
