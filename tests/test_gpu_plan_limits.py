"""Plan widths at which the engine switches kernels or branches, each run on both sides of its limit, on both codecs, in all four modes
against the reference (docIDs bit-exact, BM25 within 1e-5, top-k per assert_topk_equal), with the path every plan took asserted through
GpuIndexSource.last_routes():
  * k_score_flat takes at most 16 leaves (kSfMaxLeaves) and gives the first 12 a block-cache slot (kSfCacheLeaves): OR of 12 / 13 / 16
    leaves on it, 17 leaves on k_exec_tiles (LUCENE, scored);
  * the flat OR form of k_exec_docs takes at most 16 terms (OR of 16 vs 17 terms, GOOGLE).  The flat AND form takes at most 16 terms
    too, but it keeps one docset slot per operand, so its effective limit is min(16, slots of the launch): a conjunction of <= 3 terms
    raises the slot count itself (AND of 3 vs 4 terms), a wider one runs flat only beside a plan that needs as many slots (8 vs 9
    operands beside an 8-slot step program, 15 vs 16 beside a 15-slot one: 15 is the most a plan takes, so a 16-operand AND never runs
    flat);
  * the candidate-driven path tabulates at most 8 distinct terms: a sparse necessary term over 8 vs 9 distinct terms (GOOGLE);
  * repeated terms in a flat list and in a tree, through the front end (which folds a repeat in a flat list, as the reference does: the
    reference decides whether a repeat scores twice) and as hand-built plans that hand the kernels the repeated leaves themselves (a
    repeated leaf is one more child of the iterator tree: it matches where its term does and, scored, adds its term's score again);
  * MatchSome with min = 1, = n and > n.
Corpus: the closed-form lists extended to 18 primes (t11 .. t18 = multiples of 31 .. 61), one sparse term, and the complements c2 .. c17 of
t2 .. t17 (wide conjunctions of multiples of primes are empty)."""
import numpy as np
import pytest

import trinity_b200 as tb
from util import PRIMES18, Pair, assert_close_scores, assert_same_docs, assert_topk_equal, closed_form_lists

pytestmark = pytest.mark.gpu

NDOCS = 400_000
S, AND, OR, CAND, SF, TREE, TILES = (tb.ROUTE_STEPS, tb.ROUTE_FLAT_AND, tb.ROUTE_FLAT_OR, tb.ROUTE_CANDIDATE, tb.ROUTE_SCORE_FLAT,
                                     tb.ROUTE_FLAT_TREE, tb.ROUTE_EXEC_TILES)


def _or(n):
    return " OR ".join(f"t{i}" for i in range(1, n + 1))


def _and(n):
    # t1 AND t2 AND t3 ...; from 5 operands on, t1 AND c2 AND c3 ... (c_i: the complement of t_i) so that the conjunction is not empty
    return " AND ".join(["t1"] + [f"t{i}" if n <= 4 else f"c{i}" for i in range(2, n + 1)])


# plan -> (GOOGLE DocumentsOnly route, LUCENE scored route); LUCENE DocumentsOnly plans are step programs, GOOGLE scored ones k_exec_tiles
PLANS = {
    _or(12): (OR, SF),
    _or(13): (OR, SF),
    _or(16): (OR, SF),
    _or(17): (S, TILES),
    _and(3): (AND, TILES),
    _and(4): (S, TILES),   # no plan of this batch takes more than 3 slots (see test_flat_and_needs_one_slot_per_operand)
    _and(16): (S, TILES),
    _and(17): (S, TILES),
    "rare AND (" + _or(7) + ")": (CAND, TILES),
    "rare AND (" + _or(8) + ")": (TREE, TILES),
    "t1 OR t1": (S, SF),  # the front end folds a repeat in a flat list (like build_iterator): this is the single term t1
    "t1 OR t2 OR t1": (OR, SF),
    "t1 AND t1 AND t2": (AND, TILES),
    "(t1 AND t2) OR t1": (TREE, TILES),
    "rare AND rare AND t3": (CAND, TILES),
}
SOME = [("[t1, t2, t3]", 1), ("[t1, t2, t3]", 3), ("[t1, t2, t3]", 4), ("[t4, t13, t17, rare]", 2)]


def _lists():
    lists = closed_form_lists(NDOCS, PRIMES18)
    rng = np.random.default_rng(18)
    rare = np.sort(rng.choice(NDOCS, 300, replace=False).astype(np.uint32) + 1)
    comp = []
    for p in PRIMES18[1:17]:  # c2 .. c17: the documents that are NOT multiples of the prime
        d = np.arange(1, NDOCS + 1, dtype=np.uint32)
        d = d[d % p != 0]
        comp.append((d, (1 + d % 3).astype(np.uint32)))
    names = [f"t{i + 1}" for i in range(18)] + ["rare"] + [f"c{i}" for i in range(2, 18)]
    return lists + [(rare, (1 + rare % 3).astype(np.uint32))] + comp, names


@pytest.fixture(scope="module", params=[tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
def pair(request, ref):
    lists, names = _lists()
    p = Pair(ref, request.param, lists, NDOCS, names=names)
    yield p
    p.gpu.close()


def _routes(p, qs, scored):
    if scored:
        return [PLANS[q][1] if p.codec == tb.CODEC_LUCENE else TILES for q in qs]
    return [PLANS[q][0] if p.codec == tb.CODEC_GOOGLE else S for q in qs]


def test_documents_only_both_sides_of_each_limit(pair):
    p, qs = pair, list(PLANS)
    plans = [p.plan(q) for q in qs]
    res = p.gpu.exec_batch(plans, tb.MODE_DOCS_ONLY)
    assert list(p.gpu.last_routes()) == _routes(p, qs, False)
    comp = p.gpu.exec_batch(plans, tb.MODE_DOCS_COMPACT, copy=False)
    assert list(p.gpu.last_routes()) == _routes(p, qs, False)
    for i, q in enumerate(qs):
        want, _ = p.ref.exec(q, False, NDOCS + 1)
        assert len(want), q
        assert_same_docs(res.query(i)[0], want, f"[{q}]")
        assert_same_docs(comp.decode_query(i), want, f"[{q}] compact")


def test_scored_both_sides_of_each_limit(pair):
    p, qs = pair, list(PLANS)
    plans = [p.plan(q, scored=True) for q in qs]
    res = p.gpu.exec_batch(plans, tb.MODE_SCORED_ALL)
    assert list(p.gpu.last_routes()) == _routes(p, qs, True)
    top = p.gpu.exec_batch(plans, tb.MODE_SCORED_TOPK, k=100)
    assert list(p.gpu.last_routes()) == _routes(p, qs, True)
    for i, q in enumerate(qs):
        wd, ws = p.ref.exec(q, True, NDOCS + 1)
        gd, gs = res.query(i)
        assert_same_docs(gd, wd, f"[{q}] scored")
        assert_close_scores(gs, ws, f"[{q}]")
        assert int(top.match_counts[i]) == len(wd)
        assert_topk_equal(*top.query(i), wd, ws, 100, f"[{q}] top-100")


def _wide(depth):
    """a step program (17+ leaves: no flat-tree form; > 8 distinct terms: not candidate-driven) that takes depth + 2 docset slots"""
    q = f"t{depth + 1}"
    for i in range(depth, 0, -1):
        q = f"t{i} {'AND' if i % 2 else 'OR'} ({q})"
    return f"({q}) OR t18 OR " + " OR ".join(f"c{i}" for i in range(2, 18))


def test_flat_and_needs_one_slot_per_operand(pair):
    """the flat AND form keeps a bitmap per operand: it runs where the launch has a slot for each, else the step program does"""
    p = pair
    # (plans, their routes, the most slots one of them takes as a step program)
    cases = [([_and(3), _and(4)], [AND, S], 2),                 # 3 operands raise the launch's slot count to 3; 4 do not
             ([_wide(6), _and(8), _and(9)], [S, AND, S], 8),    # beside an 8-slot step program
             ([_wide(13), _and(15), _and(16)], [S, AND, S], 15)]  # beside a 15-slot one, the most a plan takes
    for qs, routes, nslots in cases:
        plans = [p.plan(q) for q in qs]
        assert max(tb.debug_compile(p.codec, p.index, p.terms, x, False)[2] for x in plans) == nslots
        for mode in (tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT):
            res = p.gpu.exec_batch(plans, mode)
            assert list(p.gpu.last_routes()) == (routes if p.codec == tb.CODEC_GOOGLE else [S] * len(qs)), (qs, mode)
            for i, q in enumerate(qs):
                want, _ = p.ref.exec(q, False, NDOCS + 1)
                assert len(want), q
                assert_same_docs(res.query(i)[0], want, f"[{q}] mode={mode}")


# hand-built plans whose flat lists repeat a term (the front end never produces them): (root kind, operand terms, reference query,
# GOOGLE DocumentsOnly route)
RAW = [(tb.NODE_OR, ["t1", "t1"], "t1", OR), (tb.NODE_OR, ["t1", "t2", "t1"], "t1 OR t2", OR), (tb.NODE_AND, ["t1", "t1", "t2"], "t1 AND t2", AND),
       (tb.NODE_AND, ["rare", "t3", "rare"], "rare AND t3", CAND)]


def _raw_plan(p, kind, operands):
    from trinity_b200._ffi import QNODE_DTYPE
    nodes = np.zeros(1 + len(operands), QNODE_DTYPE)
    nodes[0] = (kind, len(operands), 1, 0, 0.0)
    for i, t in enumerate(operands):
        nodes[1 + i] = (tb.NODE_TERM, 0, 0, p.names.index(t), 0.0)
    return nodes


def test_repeated_leaves_handed_to_the_kernels(pair):
    """a repeated operand of a flat AND / OR is idempotent for the documents (the reference's result for the list without the repeat);
    scored, every leaf adds its term's score where it matches, the repeated one as often as it occurs (the sum of the reference's
    per-term scores, in double)"""
    p = pair
    plans = [_raw_plan(p, kind, ops) for kind, ops, _, _ in RAW]
    for mode in (tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT):
        res = p.gpu.exec_batch(plans, mode)
        assert list(p.gpu.last_routes()) == [r if p.codec == tb.CODEC_GOOGLE else S for _, _, _, r in RAW]
        for i, (_, ops, q, _) in enumerate(RAW):
            assert_same_docs(res.query(i)[0], p.ref.exec(q, False, NDOCS + 1)[0], f"{ops} mode={mode}")
    splans = [p.gpu.set_bm25_weights(x.copy(), NDOCS) for x in plans]
    res = p.gpu.exec_batch(splans, tb.MODE_SCORED_ALL)
    top = p.gpu.exec_batch(splans, tb.MODE_SCORED_TOPK, k=100)
    for i, (_, ops, q, _) in enumerate(RAW):
        wd, _ = p.ref.exec(q, False, NDOCS + 1)
        ws = np.zeros(len(wd), np.float64)
        for t in ops:  # every occurrence of a term is a leaf of its own
            td, ts = p.ref.exec(t, True, NDOCS + 1)
            at = np.searchsorted(td, wd)
            hit = (at < len(td)) & (td[np.minimum(at, len(td) - 1)] == wd)
            ws[hit] += ts[at[hit]]
        gd, gs = res.query(i)
        assert_same_docs(gd, wd, f"{ops} scored")
        assert_close_scores(gs, ws, f"{ops} scored")
        assert_topk_equal(*top.query(i), wd, ws, 100, f"{ops} top-100")


def test_match_some_min_one_all_and_more_than_all(pair):
    p = pair
    for scored, mode in ((False, tb.MODE_DOCS_ONLY), (False, tb.MODE_DOCS_COMPACT), (True, tb.MODE_SCORED_ALL), (True, tb.MODE_SCORED_TOPK)):
        plans = []
        for q, m in SOME:
            nodes = tb.parse_query(q, p.tdict, min_match=m)
            plans.append(p.gpu.set_bm25_weights(nodes, NDOCS) if scored else nodes)
        res = p.gpu.exec_batch(plans, mode, k=50)
        for i, (q, m) in enumerate(SOME):
            wd, ws = p.ref.exec(q, scored, NDOCS + 1, parser_flags=16, min_match=m)
            what = f"[{q}] min={m} mode={mode}"
            assert (len(wd) == 0) == (m > q.count(",") + 1), what
            assert int(res.match_counts[i]) == len(wd), what
            if mode == tb.MODE_SCORED_TOPK:
                assert_topk_equal(*res.query(i), wd, ws, 50, what)
                continue
            gd, gs = res.query(i)
            assert_same_docs(gd, wd, what)
            if scored:
                assert_close_scores(gs, ws, what)
