"""The resident docID bitmaps of dense GOOGLE terms (select_dense_terms, built by trn_upload_index) and the three paths of k_exec_docs that
read them instead of decoding the term: the flat AND (a bitmap operand's tile words are ANDed in), the candidate-driven path (a probe is
one bit test) and the flat tree (a bitmap leaf's slot is a copy of the tile's words).
  * every built bitmap equals its term's list, decoded on the host: a full index, a shard that does not start at docID 1, and a copy
    translated to the top of the docID space (its last tile ends at 2^32 - 2, as in test_gpu_docid_limits);
  * flat ANDs whose operands all / some / none have a bitmap, candidate-driven ANDs and truth-table trees probing terms with a bitmap,
    flat trees with bitmap leaves: in both DocumentsOnly modes each equals the reference (oracle/_ref), equals the same batch on a source
    created with TRN_DENSE_BITMAPS=0, and runs the route trn_debug_plan plans;
  * masked documents inside the bitmap terms' tiles; 2 and 3 shards against the unsharded reference."""
import os

import numpy as np
import pytest

import trinity_b200 as tb
from refharness import RefIndex
from util import assert_same_docs

pytestmark = pytest.mark.gpu

G = tb.CODEC_GOOGLE
S = 600_000
TOP = 2**32 - 2
DELTA = TOP - S


def _corpus():
    out = {}
    for name, step in (("a", 2), ("b", 3), ("c", 5), ("d", 7), ("e", 11)):  # dense: a bitmap each
        d = np.arange(step, S + 1, step, dtype=np.uint32)
        out[name] = d
    out["m"] = np.arange(37, S + 1, 37, dtype=np.uint32)  # mid: decoded
    out["f"] = np.arange(41, S + 1, 41, dtype=np.uint32)  # mid: decoded
    out["s"] = np.arange(401, S + 1, 401, dtype=np.uint32)  # sparse: decoded, leads the candidate-driven path
    out["r"] = np.unique(np.concatenate([np.arange(1009, S + 1, 1009), [1, 2, S]])).astype(np.uint32)
    out["n"] = np.arange(300_000, 330_000, 2, dtype=np.uint32)  # dense in a narrow span: a bitmap of 2^17 docIDs
    return out


LISTS = _corpus()
NAMES = list(LISTS)
DENSE = {"a", "b", "c", "d", "e", "n"}

# DocumentsOnly plans by what they cover (the route each takes is trn_debug_plan's; the test asserts the categories are covered)
QUERIES = [
    "a AND b", "b AND c AND d", "a AND e",  # flat AND, every operand with a bitmap
    "c AND m", "a AND b AND m",  # flat AND, some
    "m AND f", "m AND r",  # flat AND and candidate-driven, none
    "s AND a", "r AND b AND c", "s AND m AND d", "r AND n",  # candidate-driven, probing bitmap terms
    "s AND (a OR m) NOT c", "r AND (b OR c OR s) NOT e",  # candidate-driven truth tables
    "(a OR m) AND (b OR s) NOT e", "(c AND d) OR (m AND s)", "(n OR r) AND (a OR c) NOT b",  # flat trees with bitmap leaves
    "a OR m OR s",  # flat OR (decoded)
]


def _build(lists, shift=0, lo=1, hi=2**32):
    b = tb.IndexBuilder(G)
    for n in NAMES:
        d = lists[n].astype(np.uint64) + shift
        d = d[(d >= lo) & (d <= hi)].astype(np.uint32)
        b.add_term(d, 1 + d % 3)
    return b.index(), b.terms_array()


def _source(index, terms, max_docid, dense=True):
    old = os.environ.get("TRN_DENSE_BITMAPS")
    os.environ["TRN_DENSE_BITMAPS"] = "1" if dense else "0"
    try:
        g = tb.GpuIndexSource(0)
    finally:
        if old is None:
            os.environ.pop("TRN_DENSE_BITMAPS")
        else:
            os.environ["TRN_DENSE_BITMAPS"] = old
    g.upload(G, index, terms, max_docid)
    return g


def _check_bitmaps(g, terms, lists, shift=0, lo=1, hi=2**32):
    """every term's bitmap (if any) == its list; returns the names with one"""
    have = set()
    for t, n in enumerate(NAMES):
        bm = g.dense_bitmap(t)
        d = lists[n].astype(np.uint64) + shift
        d = d[(d >= lo) & (d <= hi)]
        if bm is None:
            continue
        have.add(n)
        base, words = bm
        assert base % (1 << 17) == 0 and len(words) * 32 % (1 << 17) == 0, n
        assert base <= int(d[0]) and int(d[-1]) < base + 32 * len(words), n
        bits = np.unpackbits(words.view(np.uint8), bitorder="little")
        assert np.array_equal(np.flatnonzero(bits).astype(np.uint64) + base, d), f"bitmap of {n} != its list"
    info = g.info()
    assert info["dense_terms"] == len(have)
    assert info["dense_bitmap_bytes"] == sum(len(g.dense_bitmap(NAMES.index(n))[1]) * 4 for n in have)
    return have


@pytest.fixture(scope="module")
def world(ref):
    r = RefIndex(ref, G)
    for n in NAMES:
        r.add_term(n, LISTS[n], 1 + LISTS[n] % 3)
    r.finish(S)
    index, terms = _build(LISTS)
    tdict = tb.TermDictionary(NAMES)
    plans = [tb.parse_query(q, tdict) for q in QUERIES]
    routes, _ = tb.debug_plan(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=S)
    on, off = _source(index, terms, S, True), _source(index, terms, S, False)
    yield dict(ref=r, index=index, terms=terms, tdict=tdict, plans=plans, routes=routes, on=on, off=off)
    on.close()
    off.close()


def _want(w, q, shift=0):
    d, _ = w["ref"].exec(q, False, S + 1)
    return (d.astype(np.uint64) + shift).astype(np.uint32)


def test_bitmaps_of_the_full_index(world):
    assert _check_bitmaps(world["on"], world["terms"], LISTS) == DENSE
    assert world["off"].info()["dense_terms"] == 0 and world["off"].info()["dense_bitmap_bytes"] == 0
    assert world["off"].dense_bitmap(0) is None


def test_routes_cover_every_consumer(world):
    """the batch holds flat ANDs with all / some / none of their operands dense, candidate-driven plans probing dense terms (2-term ANDs
    and truth tables) and flat trees with dense leaves"""
    R, dense = world["routes"], lambda q: {t for t in q.replace("(", " ").replace(")", " ").split() if t in NAMES}
    flat = [dense(q) & DENSE for q, r in zip(QUERIES, R) if r == tb.ROUTE_FLAT_AND]
    ops = [dense(q) for q, r in zip(QUERIES, R) if r == tb.ROUTE_FLAT_AND]
    assert any(f == o for f, o in zip(flat, ops)) and any(f and f != o for f, o in zip(flat, ops)) and any(not f for f in flat), R
    cand = [q for q, r in zip(QUERIES, R) if r == tb.ROUTE_CANDIDATE and dense(q) & DENSE]
    assert any("OR" in q for q in cand) and any("OR" not in q for q in cand), R
    assert any(r == tb.ROUTE_FLAT_TREE and dense(q) & DENSE for q, r in zip(QUERIES, R)), R


@pytest.mark.parametrize("mode", [tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT], ids=["docs", "compact"])
def test_results_equal_reference_and_bitmaps_off(world, mode):
    got = {}
    for key in ("on", "off"):
        g = world[key]
        res = g.exec_batch(world["plans"], mode, copy=mode == tb.MODE_DOCS_ONLY)
        assert list(g.last_routes()) == list(world["routes"]), key
        got[key] = [res.query(i)[0] if mode == tb.MODE_DOCS_ONLY else res.decode_query(i).copy() for i in range(len(QUERIES))]
    for i, q in enumerate(QUERIES):
        want = _want(world, q)
        assert_same_docs(got["on"][i], want, f"[{q}] bitmaps on")
        assert_same_docs(got["off"][i], want, f"[{q}] bitmaps off")


def test_masked_documents_in_dense_tiles(world):
    """masked documents in the tiles the bitmap terms fill: removed at emission as before"""
    rng = np.random.default_rng(7)
    pool = np.unique(np.concatenate([LISTS["a"][::5], LISTS["d"][::3], LISTS["n"], LISTS["s"]]))
    masked = np.sort(rng.choice(pool, size=len(pool) // 3, replace=False)).astype(np.uint32)
    g = world["on"]
    g.set_masked_documents(masked)
    try:
        for mode in (tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT):
            res = g.exec_batch(world["plans"], mode, copy=mode == tb.MODE_DOCS_ONLY)
            assert list(g.last_routes()) == list(world["routes"])
            for i, q in enumerate(QUERIES):
                want, _ = world["ref"].exec_masked(q, False, masked, S + 1)
                got = res.query(i)[0] if mode == tb.MODE_DOCS_ONLY else res.decode_query(i)
                assert_same_docs(got, want, f"[{q}] masked, mode {mode}")
    finally:
        g.set_masked_documents(None)


@pytest.mark.parametrize("nshards", [2, 3])
def test_shards_against_the_unsharded_reference(world, nshards):
    """docID-range shards (each but the first starting above docID 1): every shard's bitmaps cover its own range; the concatenated
    results equal the unsharded reference's"""
    cuts = [1] + [int(S * (i + 1) / nshards) + 1 for i in range(nshards - 1)] + [S + 1]
    parts = [[] for _ in QUERIES]
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        index, terms = _build(LISTS, 0, lo, hi - 1)
        g = _source(index, terms, S)
        have = _check_bitmaps(g, terms, LISTS, 0, lo, hi - 1)
        assert have, (lo, hi)
        plans = [tb.parse_query(q, world["tdict"]) for q in QUERIES]
        routes, _ = tb.debug_plan(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=S)
        res = g.exec_batch(plans, tb.MODE_DOCS_ONLY)
        assert list(g.last_routes()) == list(routes)
        for i in range(len(QUERIES)):
            parts[i].append(res.query(i)[0].copy())
        g.close()
    for i, q in enumerate(QUERIES):
        assert_same_docs(np.concatenate(parts[i]), _want(world, q), f"[{q}] {nshards} shards")


def test_top_of_the_docid_space(world):
    """the corpus translated to end at 2^32 - 2: bitmaps whose span ends at 2^32, and the top tile of every launch read from them"""
    index, terms = _build(LISTS, DELTA)
    g = _source(index, terms, TOP)
    try:
        assert _check_bitmaps(g, terms, LISTS, DELTA) == DENSE
        tdict = tb.TermDictionary(NAMES)
        plans = [tb.parse_query(q, tdict) for q in QUERIES]
        routes, _ = tb.debug_plan(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=TOP)
        for mode in (tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT):
            res = g.exec_batch(plans, mode, copy=mode == tb.MODE_DOCS_ONLY)
            assert list(g.last_routes()) == list(routes)
            for i, q in enumerate(QUERIES):
                want = _want(world, q, DELTA)
                got = res.query(i)[0] if mode == tb.MODE_DOCS_ONLY else res.decode_query(i)
                assert_same_docs(got, want, f"[{q}] top of the docID space, mode {mode}")
    finally:
        g.close()
