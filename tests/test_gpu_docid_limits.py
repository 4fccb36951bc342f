"""The top of the docID space: docIDs are global uint32_t with 0 reserved and DocIDsEND = 2^32 - 1 (common.h:43), so the largest valid
docID is 2^32 - 2, and the last tile of every tile size ends there (`lo + W` wraps to 0 for it).

Checked by TRANSLATION: a corpus whose docIDs lie in [1, S] is indexed as is for the reference, and shifted by DELTA = (2^32 - 2) - S for
the device, so that its largest docID is exactly 2^32 - 2 and the top 2^13, 2^14 and 2^17 docIDs are populated.  The device copy is
uploaded with max_docid = 2^32 - 2 and scored with docs_cnt = S (BM25's idf depends on df and docs_cnt only), so its results must be the
reference's on the unshifted index plus DELTA: docIDs bit-exact, scores within 1e-5, top-k strict (the shift keeps docID order).  The
reference itself is not run up there.  Every query asserts the path it took (GpuIndexSource.last_routes)."""
import numpy as np
import pytest

import trinity_b200 as tb
from refharness import RefIndex
from util import assert_close_scores, assert_same_docs, assert_topk_exact, merged_topk

pytestmark = pytest.mark.gpu

S = 600_000
TOP = 2**32 - 2
DELTA = TOP - S
G, L = tb.CODEC_GOOGLE, tb.CODEC_LUCENE


def _edges():
    """unshifted docIDs whose shifted image is one of the first two or last two docIDs of a 2^13, 2^14 or 2^17 tile"""
    out = {S, S - 1, S - 2}
    for shift in (13, 14, 17):
        t = 1 << shift
        for b in range((DELTA + t) // t * t, TOP + 3, t):
            out |= {x - DELTA for x in (b - 2, b - 1, b, b + 1) if DELTA < x <= TOP}
    return np.array(sorted(out), np.uint32)


def _corpus():
    edge = _edges()
    u = lambda *a: np.unique(np.concatenate([np.asarray(x, np.uint32) for x in a]))
    lists = {}
    d = u(np.arange(1, S + 1, 3), [S])
    lists["dense"] = (d, 1 + d % 4)
    d = u(np.arange(37, S + 1, 37), edge[::3])
    lists["mid"] = (d, 1 + (d // 37) % 3)
    lists["edge"] = (edge, 1 + np.arange(len(edge), dtype=np.uint32) % 2)
    d = u(np.arange(S - 8000, S + 1, 5), [S])  # only the last 2^13-docID tile of the shifted copy (and the one below it)
    lists["top"] = (d, 1 + d % 3)
    d = u(np.arange(S - 60_000, S + 1, 11), edge[edge > S - (1 << 17)])  # 64+ hits per document: GOOGLE blocks beyond the staging area
    lists["heavy"] = (d, 64 + d % 9)
    d = u(np.arange(2, S + 1, 13), [S])
    lists["ph1"] = (d, np.ones(len(d), np.uint32))
    d = u(np.arange(2, S + 1, 26), np.arange(5, S + 1, 61), [S])
    lists["ph2"] = (d, np.ones(len(d), np.uint32))
    return lists


def _positions(name, f):
    """ph1 and ph2 have one hit per document; ph2's sits at position 2, behind ph1's at 1 (None = positions 1..freq): "ph1 ph2" matches
    where both are present"""
    assert name not in ("ph1", "ph2") or np.all(f == 1)
    return np.full(len(f), 2, np.uint32) if name == "ph2" else None


LISTS = _corpus()
NAMES = list(LISTS)
DF = np.array([len(LISTS[n][0]) for n in NAMES])

# DocumentsOnly plans and the path each takes on GOOGLE (LUCENE: step programs only)
DOCS = {
    "dense AND mid": tb.ROUTE_FLAT_AND,
    "dense OR mid OR edge": tb.ROUTE_FLAT_OR,
    "heavy OR top": tb.ROUTE_FLAT_OR,
    "edge AND dense": tb.ROUTE_CANDIDATE,
    "top AND dense AND mid": tb.ROUTE_CANDIDATE,
    "(dense OR mid) AND heavy NOT edge": tb.ROUTE_FLAT_TREE,
    "(dense AND mid) OR (top AND heavy)": tb.ROUTE_FLAT_TREE,
    '"ph1 ph2"': tb.ROUTE_STEPS,
    'dense AND "ph1 ph2"': tb.ROUTE_STEPS,
}
# scored plans and their path on LUCENE (GOOGLE: k_exec_tiles only); at most two contributions per document in the k_score_flat plans,
# so tie classes are bit-identical whatever order the contributions arrive in
SCORED = {
    "dense OR mid": tb.ROUTE_SCORE_FLAT,
    "top OR edge": tb.ROUTE_SCORE_FLAT,
    "heavy": tb.ROUTE_SCORE_FLAT,
    "dense AND mid": tb.ROUTE_EXEC_TILES,
    "heavy AND top": tb.ROUTE_EXEC_TILES,
    "(dense OR mid) AND heavy NOT edge": tb.ROUTE_EXEC_TILES,
    "edge NOT dense": tb.ROUTE_EXEC_TILES,
}
PHRASE_SCORED = ['"ph1 ph2"', 'top AND "ph1 ph2"']  # GOOGLE only (inline hits)


def _build(codec, lists, shift=0, lo=1, hi=2**32):
    b = tb.IndexBuilder(codec)
    for n in NAMES:
        d, f = lists[n]
        keep = (d.astype(np.uint64) + shift >= lo) & (d.astype(np.uint64) + shift <= hi)
        b.add_term((d[keep].astype(np.uint64) + shift).astype(np.uint32), f[keep], _positions(n, f[keep]))
    return b


class Space:
    def __init__(self, ref, codec):
        self.codec = codec
        self.ref = RefIndex(ref, codec)
        for n in NAMES:
            d, f = LISTS[n]
            self.ref.add_term(n, d, f, _positions(n, f))
        self.ref.finish(S)
        b = _build(codec, LISTS, DELTA)
        self.index, self.terms = b.index(), b.terms_array()
        self.gpu = tb.GpuIndexSource(0)
        self.gpu.upload(codec, self.index, self.terms, TOP)
        self.tdict = tb.TermDictionary(NAMES)
        self.cache = {}

    def plan(self, q, scored=False):
        nodes = tb.parse_query(q, self.tdict)
        return self.gpu.set_bm25_weights(nodes, S) if scored else nodes

    def want(self, q, scored):
        """the reference's result on the unshifted index, moved up by DELTA"""
        if (q, scored) not in self.cache:
            d, s = self.ref.exec(q, scored, S + 1)
            self.cache[(q, scored)] = ((d.astype(np.uint64) + DELTA).astype(np.uint32), s)
        return self.cache[(q, scored)]


@pytest.fixture(scope="module", params=[G, L], ids=["google", "lucene"])
def space(request, ref):
    sp = Space(ref, request.param)
    yield sp
    sp.gpu.close()


def test_corpus_reaches_the_top_of_the_space(space):
    info = space.gpu.info()
    assert info["max_docid"] == TOP
    top = (LISTS["dense"][0].astype(np.uint64) + DELTA)
    assert int(top.max()) == TOP
    edge = LISTS["edge"][0].astype(np.uint64) + DELTA
    for shift in (13, 14, 17):  # the first and last two docIDs of the top tile of every tile size hold documents
        lo = (2**32 >> shift) - 1 << shift
        assert {lo, lo + 1, TOP - 1, TOP} <= set(edge.tolist()), shift


def _docs_queries(codec):
    return [q for q in DOCS if codec == G or '"' not in q]


def test_documents_only_and_compact(space):
    qs = _docs_queries(space.codec)
    plans = [space.plan(q) for q in qs]
    res = space.gpu.exec_batch(plans, tb.MODE_DOCS_ONLY)
    routes = space.gpu.last_routes()
    comp = space.gpu.exec_batch(plans, tb.MODE_DOCS_COMPACT, copy=False)
    croutes = space.gpu.last_routes()
    for i, q in enumerate(qs):
        want, _ = space.want(q, False)
        assert int(want[-1]) > 2**32 - (1 << 13), f"[{q}] does not reach the top tile"
        assert_same_docs(res.query(i)[0], want, f"[{q}] docs")
        assert_same_docs(comp.decode_query(i), want, f"[{q}] compact")
        exp = DOCS[q] if space.codec == G else tb.ROUTE_STEPS
        assert routes[i] == exp and croutes[i] == exp, f"[{q}] route {routes[i]}/{croutes[i]}, expected {exp}"


def test_scored_all_and_topk(space):
    qs = list(SCORED) + (PHRASE_SCORED if space.codec == G else [])
    plans = [space.plan(q, True) for q in qs]
    exp = [SCORED.get(q, tb.ROUTE_EXEC_TILES) if space.codec == L else tb.ROUTE_EXEC_TILES for q in qs]
    res = space.gpu.exec_batch(plans, tb.MODE_SCORED_ALL)
    assert list(space.gpu.last_routes()) == exp
    for i, q in enumerate(qs):
        wd, ws = space.want(q, True)
        assert int(wd[-1]) > 2**32 - (1 << 13), f"[{q}] does not reach the top tile"
        gd, gs = res.query(i)
        assert_same_docs(gd, wd, f"[{q}] scored")
        assert_close_scores(gs, ws, f"[{q}] scored")
    for k in (1, 100, 512):
        res = space.gpu.exec_batch(plans, tb.MODE_SCORED_TOPK, k=k)
        assert list(space.gpu.last_routes()) == exp
        for i, q in enumerate(qs):
            wd, ws = space.want(q, True)
            assert int(res.match_counts[i]) == len(wd)
            gd, gs = res.query(i)
            assert_topk_exact(gd, gs, wd, ws, k, f"[{q}] k={k}")


def test_masked_documents_in_the_top_tile(ref, space):
    if space.codec != G:
        pytest.skip("the registry of a source whose max_docid is 2^32 - 2 is a 512 MiB bitmap: built once, on one codec")
    top_tile = lambda d: d[d > S - (1 << 13)]
    masked = np.unique(np.concatenate([top_tile(LISTS["edge"][0]), top_tile(LISTS["dense"][0])[::2], top_tile(LISTS["heavy"][0])[::3]]))
    space.gpu.set_masked_documents((masked.astype(np.uint64) + DELTA).astype(np.uint32))
    try:
        qs = ["dense OR mid OR edge", "(dense OR mid) AND heavy NOT edge", "top AND dense AND mid"]
        res = space.gpu.exec_batch([space.plan(q) for q in qs], tb.MODE_DOCS_ONLY)
        sq = ["dense OR mid", "heavy AND top"]
        top = space.gpu.exec_batch([space.plan(q, True) for q in sq], tb.MODE_SCORED_TOPK, k=100)
        for i, q in enumerate(qs):
            want, _ = space.ref.exec_masked(q, False, masked, S + 1)
            assert_same_docs(res.query(i)[0], (want.astype(np.uint64) + DELTA).astype(np.uint32), f"[{q}] masked")
        for i, q in enumerate(sq):
            wd, ws = space.ref.exec_masked(q, True, masked, S + 1)
            gd, gs = top.query(i)
            assert_topk_exact(gd, gs, (wd.astype(np.uint64) + DELTA).astype(np.uint32), ws, 100, f"[{q}] masked top-100")
    finally:
        space.gpu.set_masked_documents(None)


def test_shard_ending_at_the_top_merged(space):
    """two docID-range shards of the shifted copy, the upper one ending at 2^32 - 2, global idf; top-k lists merged by trn_merge_topk"""
    cut = DELTA + S // 2
    shards = []
    for lo, hi in ((DELTA + 1, cut), (cut + 1, TOP)):
        b = _build(space.codec, LISTS, DELTA, lo, hi)
        g = tb.GpuIndexSource(0)
        g.upload(space.codec, b.index(), b.terms_array(), TOP)
        shards.append(g)
    qs = list(SCORED)
    plans = []
    for q in qs:
        nodes = tb.parse_query(q, space.tdict)
        for x in nodes:
            if x["kind"] == tb.NODE_TERM and x["term"] != tb.EMPTY_TERM:
                x["weight"] = tb.bm25_idf(int(DF[x["term"]]), S)
        plans.append(nodes)
    k = 512
    got = merged_topk(shards, plans, k)
    for i, q in enumerate(qs):
        wd, ws = space.want(q, True)
        assert_topk_exact(*got[i], wd, ws, k, f"[{q}] 2 shards, k={k}")
    for g in shards:
        g.close()


def test_max_docid_derived_from_the_postings(space):
    g = tb.GpuIndexSource(0)
    g.upload(space.codec, space.index, space.terms, 0)
    assert g.info()["max_docid"] == TOP
    qs = _docs_queries(space.codec)
    res = g.exec_batch([space.plan(q) for q in qs], tb.MODE_DOCS_ONLY)
    for i, q in enumerate(qs):
        assert_same_docs(res.query(i)[0], space.want(q, False)[0], f"[{q}] max_docid = 0")
    sq = list(SCORED)
    top = g.exec_batch([g.set_bm25_weights(space.plan(q), S) for q in sq], tb.MODE_SCORED_TOPK, k=100)
    for i, q in enumerate(sq):
        wd, ws = space.want(q, True)
        assert_topk_exact(*top.query(i), wd, ws, 100, f"[{q}] max_docid = 0")
    g.close()
