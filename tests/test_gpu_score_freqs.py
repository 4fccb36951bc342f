"""BM25 across the whole freq range, on every scored route and block form, against the reference's exec_query.

Every scored result is Scorer::score(freq) (similarity.h:228-235) summed over the leaves that hold a document; the kernels read it from a
64-entry table below freq 64 and compute it from 64 up, and the reference keeps freq as a uint16_t.  The corpora below put freqs on both
sides of every boundary in that code and in the two codecs (varbyte.h: 1-byte codes below 2^7, 2-byte below 2^14, 3-byte below 2^21; the
table's 64; the reference's 65 536), in every block form that carries them.  docID sets are compared bit-exact, scores within 1e-5, top-k
with assert_topk_exact where every tie class is one float on both sides (single terms) and assert_topk_equal otherwise, and the route of
every query is asserted, so that a planner change cannot move a case off the path it is meant to test.

Freqs of 65 536 and more: both host encoders accept them (varbyte codes of the full value) and so does the reference, whose decoders keep
`freq & 0xffff` (tokenpos_t); the kernels mask the same way.  Term `huge` carries four of them.  Freqs above 16 383 take explicit positions
that share position 16 383 (Limits::MaxPosition is 16 384).

§1 freq-sweep corpus (_sweep_terms, 300 000 documents, both codecs):
  - freq boundaries 0, 1, 63, 64, 65, 127, 128, 16 383, 16 384, 65 535 mixed inside single blocks, every fourth LUCENE block all below
    64, freqs 32..63 throughout: `bnd`.  Every query that names `bnd`.
  - constant-freq LUCENE blocks (L == 0) of freq 0, 63, 64 and 65 535, with constant docID gaps: `cst` (GOOGLE: its 65 535 block is
    read from global memory).  `cst`, "bnd OR pfx OR cst", "bnd AND (pfx OR stg) NOT cst".
  - PFor freq pages of base width <= 6 whose exceptions carry freqs >= 64, exception width k == 1 (block 0) and k > 1 (blocks 1, 3),
    and a 7-bit page without exceptions (block 2): `pfx`.  `pfx`, "bnd OR pfx OR cst", the trees.
  - tails of documents % 128 == 0, 1 and 127 whose freqs take 1-, 2- and 3-byte codes: `tail0`, `tail1`, `tail127`.  Those terms and
    "tail0 OR tail1 OR tail127 OR gap".
  - LUCENE docID gaps whose widest value is exactly 2047 (block 0, no exceptions; block 2, exceptions) and exactly 2048 (block 1, no
    exceptions, its first 32 gaps sum to 65 536; block 3, exceptions): `gap`.  `gap`, "tail0 OR tail1 OR tail127 OR gap".
  - GOOGLE staging limit: `stg` holds every document of the 8192-doc tile [8192, 16384); its even 32-block groups carry a 6000-hit
    document and exceed the 6144-byte stage, its odd ones fit.  Every query that names `stg`, in every mode.
  - idf extremes: `all` holds every document (idf ~1.7e-6) beside `bnd` (idf ~4.6).  "all OR bnd", "bnd AND all", ...
  - freqs >= 65 536: `huge`.  `huge`, "stg OR bnd OR huge", "[bnd, stg, all, huge]".
§2 every scored route: QUERIES (single terms, flat ORs, ANDs and NOTs, trees with OP_LEAFSCORE steps, MatchSome at min 1 and min n,
  Optional) in MODE_SCORED_ALL and MODE_SCORED_TOPK at k = 1, 100, 512 on GOOGLE (ROUTE_EXEC_TILES), LUCENE (ROUTE_SCORE_FLAT for single
  terms and flat ORs, ROUTE_EXEC_TILES for the rest) and LUCENE under TRN_FLAT_SCORED=0 (all ROUTE_EXEC_TILES):
  test_scored_routes_match_reference.  The same queries in MODE_DOCS_ONLY and MODE_DOCS_COMPACT (k_exec_docs routes, dense bitmaps):
  test_docs_routes_match_scored_sets, which also checks each GOOGLE term's resident bitmap against its docIDs.
§3 runs and the top-k cut: _runs_terms (LUCENE, 3 300 000 documents: four runs of k_score_flat's default 128 tiles) under TRN_RUN_TILES = 1, 2
  and the default, the best documents only in the last run (`late`), only in the first (`early`) and in every run (`spread`), and
  128-doc blocks that straddle the tile boundary at the end of each run (`strad`): test_runs_topk.  The full per-tile list of
  k_exec_tiles (kTileListCap = k + 512 keys at k = 512): `all` on GOOGLE, whose top 512 must be docIDs 1 .. 512: test_full_tile_list.
§4 phrase match counts (_phrase_terms, both codecs, LUCENE with its hits): t0 of "x y" with 63, 64, 65, 128 and 129 positions, matches at
  positions 62, 63, 64, 127 and the last of t0's stream, a matchCnt of 129, and runs of x that give "x x" match counts of 62 .. 65, 128 and 129:
  test_phrase_match_counts.
"""
import os

import numpy as np
import pytest

import trinity_b200 as tb
from refharness import RefIndex
from stepsim import OP_LEAFSCORE
from util import assert_close_scores, assert_same_docs, assert_topk_equal, assert_topk_exact

pytestmark = pytest.mark.gpu

MAX_POS = 16383  # the last legal position (Limits::MaxPosition = 16384)
KS = [1, 100, 512]
F_OPT, F_SOME = 8, 16  # ast_parser flags of the reference: <expr> -> Optional, [a, b] -> MatchSome


def _positions(freqs):
    """explicit positions 1 .. freq of every posting; freqs above 16 383 share the last legal position"""
    f = np.asarray(freqs, np.int64)
    starts = np.repeat(np.cumsum(f) - f, f)
    return np.minimum(np.arange(int(f.sum())) - starts + 1, MAX_POS).astype(np.uint32)


class Corpus:
    """The same postings (with positions) indexed by this repo's host encoder and by the reference's, plus cached reference answers."""

    def __init__(self, ref, codec, terms, ndocs, hits=False):
        self.codec, self.ndocs, self.terms, self.hits = codec, ndocs, terms, hits
        self.r = RefIndex(ref, codec)
        b = tb.IndexBuilder(codec)
        for n, (d, f, p) in terms.items():
            self.r.add_term(n, d, f, p)
            b.add_term(d, f, p)
        self.r.finish(ndocs)
        self.index, self.tarr, self.hits_bytes = b.index(), b.terms_array(), b.hits()
        self.names = list(terms)
        self.tdict = tb.TermDictionary(self.names)
        self.cache = {}

    def gpu(self, env=None):
        old = {k: os.environ.get(k) for k in (env or {})}
        os.environ.update(env or {})
        try:
            g = tb.GpuIndexSource(0)  # trn_create reads the knobs
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        g.upload(self.codec, self.index, self.tarr, self.ndocs)
        if self.hits and self.codec == tb.CODEC_LUCENE:
            g.upload_hits(self.index, self.hits_bytes)
        return g

    def plan(self, q, scored=True):
        text, flags, mm = q
        nodes = tb.parse_query(text, self.tdict, min_match=mm if flags & F_SOME else None)
        if scored:
            for x in nodes:
                if x["kind"] == tb.NODE_TERM and x["term"] != tb.EMPTY_TERM:
                    x["weight"] = tb.bm25_idf(len(self.terms[self.names[x["term"]]][0]), self.ndocs)
        return nodes

    def want(self, q, scored):
        key = (q, scored)
        if key not in self.cache:
            text, flags, mm = q
            self.cache[key] = self.r.exec(text, scored, self.ndocs + 1, parser_flags=flags, min_match=mm)
        return self.cache[key]


def _q(text, flags=0, mm=0):
    return (text, flags, mm)


# ------------------------------------------------------------------------------------------------ §1 the freq-sweep corpus
NDOCS = 300_000
BOUNDARY = [0, 1, 63, 64, 65, 127, 128, 16383, 16384, 65535]
LIGHT = [0, 1, 2, 31, 32, 33, 62, 63, 64, 65, 126, 127, 128, 129, 255, 1000]


def _bnd(rng):
    d = np.arange(7, NDOCS + 1, 97, dtype=np.uint32)  # 3093 documents: 24 full blocks and a tail of 21
    f = np.where(rng.random(len(d)) < 0.5, rng.integers(0, 64, len(d)), rng.choice(LIGHT, len(d))).astype(np.uint32)
    for blk in range(1, len(d) // 128, 4):  # every fourth block all below 64
        f[blk * 128:(blk + 1) * 128] = rng.integers(0, 64, 128)
    for i, x in zip((10, 20, 30, 300, 800, 1500, 3080, 3090), (16383, 16384, 65535, 16383, 16384, 65535, 16384, 128)):
        f[i] = x  # the heavy boundaries in full blocks (0, 2, 6, 11) and in the tail
    for i, x in enumerate(BOUNDARY):  # all ten boundaries inside block 3
        f[3 * 128 + 7 * i] = x
    return d, f


def _cst():
    d = np.arange(50, 50 * 641, 50, dtype=np.uint32)  # constant docID gaps: the docID int-blocks are L == 0 too
    f = np.repeat(np.array([0, 63, 64, 65535, 3], np.uint32), 128)
    f[4 * 128 + 5] = 70  # block 4: an ordinary page
    return d, f


def _pfx(rng):
    d = np.sort(rng.choice(np.arange(1, NDOCS + 1, dtype=np.uint32), 512, replace=False))
    f = np.zeros(512, np.uint32)
    f[0:128] = rng.integers(32, 64, 128)  # b = 6, five exceptions of 64..127: k = 1 (no exception stream)
    f[[3, 40, 77, 100, 127]] = [64, 127, 65, 100, 64]
    f[128:256] = rng.integers(0, 8, 128)  # b = 3, exceptions 65 535 and 200: k = 13
    f[[128 + 1, 128 + 64, 128 + 90]] = [65535, 200, 65535]
    f[256:384] = rng.integers(0, 128, 128)  # b = 7, no exceptions
    f[256:256 + 64] |= 64
    f[384:512] = rng.integers(1, 4, 128)  # b = 2, one exception 64: k = 5
    f[384 + 31] = 64
    return d, f


def _gap(rng):
    g = np.zeros(512, np.int64)
    g[0:128] = rng.integers(512, 1024, 128)  # widest gap 2047, b = 11 without exceptions
    g[rng.choice(128, 20, replace=False)] = 2047
    g[128:256] = rng.integers(512, 1024, 128)  # widest gap 2048, b = 12 without exceptions; gaps 0..31 sum to 65 536
    g[128:160] = 2048
    g[256:384] = rng.integers(1, 16, 128)  # b = 4, three exceptions of 2047 (11 bits)
    g[256 + np.array([5, 70, 127])] = 2047
    g[384:512] = rng.integers(1, 16, 128)  # b = 4, three exceptions of 2048 (12 bits)
    g[384 + np.array([0, 64, 100])] = 2048
    d = np.cumsum(g).astype(np.uint32)
    assert d[-1] <= NDOCS
    return d, rng.integers(1, 200, 512).astype(np.uint32)


def _stg(rng):
    d = np.arange(8192, 16384, dtype=np.uint32)  # one whole 8192-doc tile: 256 GOOGLE blocks, 8 groups of 32 blocks
    f = rng.integers(1, 4, len(d)).astype(np.uint32)
    f[rng.choice(len(d), 100, replace=False)] = rng.integers(32, 64, 100)
    for grp in range(8):
        at = grp * 1024
        f[at + 100] = 150  # every group: a 2-byte freq
        if grp % 2 == 0:
            f[at + 500] = 6000  # 6000 hit bytes: the group's span exceeds the 6144-byte stage
    return d, f


def _tail(rng, n, heavy):
    d = np.sort(rng.choice(np.arange(1, NDOCS + 1, dtype=np.uint32), n, replace=False))
    f = rng.choice([0, 1, 5, 63, 64, 127, 128, 129, 300, 5000], n).astype(np.uint32)
    full = n - n % 128
    for i, x in enumerate(heavy):  # 3-byte codes: in the tail when there is one, else in the last full block
        f[(full if n % 128 else full - 128) + i * 3] = x
    return d, f


def _huge(rng):
    d = np.sort(rng.choice(np.arange(1, NDOCS + 1, dtype=np.uint32), 200, replace=False))
    f = rng.integers(1, 100, 200).astype(np.uint32)
    f[[5, 60, 130, 199]] = [65536, 65537, 70000, 131072 + 64]  # the reference and the kernels keep freq & 0xffff: 0, 1, 4464, 64
    return d, f


def _sweep_terms():
    rng = np.random.default_rng(2026)
    terms = {
        "bnd": _bnd(rng),
        "cst": _cst(),
        "pfx": _pfx(rng),
        "gap": _gap(rng),
        "stg": _stg(rng),
        "tail0": _tail(rng, 256, [16384, 20000]),
        "tail1": _tail(rng, 129, [16384]),
        "tail127": _tail(rng, 255, [16384, 65535, 16383]),
        "huge": _huge(rng),
        "all": (np.arange(1, NDOCS + 1, dtype=np.uint32), np.ones(NDOCS, np.uint32)),
    }
    return {n: (d, f, _positions(f)) for n, (d, f) in terms.items()}


SINGLE = ["bnd", "cst", "pfx", "gap", "stg", "tail0", "tail1", "tail127", "huge", "all"]
FLAT_OR = ["bnd OR pfx OR cst", "tail0 OR tail1 OR tail127 OR gap", "stg OR bnd OR huge", "all OR bnd",
           "bnd OR cst OR pfx OR gap OR stg OR tail0 OR tail1 OR tail127 OR huge"]
ANDNOT = ["bnd AND all", "stg AND all", "stg AND bnd", "pfx AND all", "stg NOT bnd", "bnd NOT stg NOT cst", "bnd AND (pfx OR stg) NOT cst"]
LEAFSCORE = ["(bnd AND all) OR (stg AND pfx)", "bnd AND ((pfx AND all) OR stg) NOT cst", "all AND ((bnd AND pfx) OR (stg AND huge) OR cst) NOT gap",
             "(stg AND bnd) OR (cst AND all) OR (huge AND all)"]
QUERIES = ([_q(t) for t in SINGLE + FLAT_OR + ANDNOT + LEAFSCORE]
           + [_q("[bnd, stg, all, huge]", F_SOME, 1), _q("[stg, bnd, all]", F_SOME, 3)]
           + [_q("stg <bnd>", F_OPT), _q("all AND <bnd OR pfx>", F_OPT), _q("bnd <stg> <cst>", F_OPT)])
FLAT = set(SINGLE + FLAT_OR)  # k_score_flat's queries on LUCENE


@pytest.fixture(scope="module")
def sweep_terms():
    return _sweep_terms()


@pytest.fixture(scope="module", params=[tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
def sweep(request, ref, sweep_terms):
    return Corpus(ref, request.param, sweep_terms, NDOCS)


def _bits(v):
    return int(v).bit_length()


def _pfor_form(values):
    """(b, exceptions, maxbits) FastPFor<4> picks for one 128-value page (the cost model of fastpfor.h:143-171), None for L == 0"""
    v = np.asarray(values, np.int64)
    if np.all(v == v[0]):
        return None
    cnt = np.bincount([_bits(x) for x in v], minlength=33)
    maxb = max(_bits(x) for x in v)
    best, bestc, cost, c = maxb, 0, maxb * 128, 0
    for bb in range(maxb - 1, -1, -1):
        c += cnt[bb + 1]
        t = c * 8 + c * (maxb - bb) + bb * 128 + 8 - (c if maxb - bb == 1 else 0)
        if t < cost:
            best, bestc, cost = bb, c, t
    return best, bestc, maxb


def test_sweep_corpus_holds_the_forms_it_claims(sweep_terms):
    """the corpus is what the module docstring says it is (a generator change must not quietly drop a case)"""
    T = sweep_terms
    f = T["bnd"][1]
    assert set(BOUNDARY) <= set(f[3 * 128:4 * 128].tolist())
    assert f[128:256].max() < 64 and np.any((f >= 32) & (f < 64))
    assert {16383, 16384, 65535} <= set(f[-(len(f) % 128):].tolist()) | set(f[:128].tolist())
    cf = T["cst"][1]
    gaps = np.diff(np.concatenate([[0], T["cst"][0]]))
    assert [_pfor_form(cf[i * 128:(i + 1) * 128]) for i in range(4)] == [None] * 4 and _pfor_form(gaps[:128]) is None
    assert [int(cf[i * 128]) for i in range(4)] == [0, 63, 64, 65535]
    pf = [_pfor_form(T["pfx"][1][i * 128:(i + 1) * 128]) for i in range(4)]
    assert pf[0] == (6, 5, 7) and pf[1] == (3, 3, 16) and pf[2] == (7, 0, 7) and pf[3] == (2, 1, 7)
    gg = np.diff(np.concatenate([[0], T["gap"][0].astype(np.int64)]))
    gf = [_pfor_form(gg[i * 128:(i + 1) * 128]) for i in range(4)]
    assert gf[0] == (11, 0, 11) and gf[1] == (12, 0, 12) and gf[2][1:] == (3, 11) and gf[3][1:] == (3, 12) and gf[2][0] <= 6
    assert gg[:128].max() == 2047 and gg[128:256].max() == 2048 and gg[128:160].sum() == 65536
    for n, tail, want in (("tail0", 0, {1, 2, 3}), ("tail1", 1, {3}), ("tail127", 127, {1, 2, 3})):
        d, fr, _ = T[n]
        assert len(d) % 128 == tail
        codes = {1 if x < 128 else 2 if x < 16384 else 3 for x in (fr[len(d) - tail:] if tail else fr)}  # varbyte code lengths
        assert codes == want, (n, codes)
    assert np.all(T["huge"][1][[5, 60, 130, 199]] > 65535)
    # GOOGLE: the 32-block groups of `stg` alternate between not fitting the 6144-byte stage and fitting it
    b = tb.IndexBuilder(tb.CODEC_GOOGLE)
    sizes = []
    for grp in range(8):
        lo = grp * 1024
        d, fr, p = T["stg"]
        sl = slice(lo, lo + 1024)
        before = b.index().size
        b.add_term(d[sl], fr[sl], _positions(fr[sl]))
        sizes.append(b.index().size - before)
    assert all(s > 6144 + 64 if grp % 2 == 0 else s < 6144 - 512 for grp, s in enumerate(sizes)), sizes


def _expected_scored_routes(codec, flat_scored, qs):
    if codec == tb.CODEC_LUCENE and flat_scored:
        return [tb.ROUTE_SCORE_FLAT if q[0] in FLAT else tb.ROUTE_EXEC_TILES for q in qs]
    return [tb.ROUTE_EXEC_TILES] * len(qs)


def _check_scored(c, g, qs, routes, what):
    plans = [c.plan(q) for q in qs]
    res = g.exec_batch(plans, tb.MODE_SCORED_ALL)
    assert list(g.last_routes()) == routes, (what, list(g.last_routes()))
    for i, q in enumerate(qs):
        wd, ws = c.want(q, True)
        gd, gs = res.query(i)
        assert_same_docs(gd, wd, f"[{q[0]}] {what} scored-all")
        assert_close_scores(gs, ws, f"[{q[0]}] {what} scored-all")
    for k in KS:
        res = g.exec_batch(plans, tb.MODE_SCORED_TOPK, k=k)
        assert list(g.last_routes()) == routes, (what, k, list(g.last_routes()))
        for i, q in enumerate(qs):
            wd, ws = c.want(q, True)
            assert int(res.match_counts[i]) == len(wd), f"[{q[0]}] {what} k={k} match count"
            gd, gs = res.query(i)
            check = assert_topk_exact if q[0] in c.terms else assert_topk_equal  # one term: every tie class is one float
            check(gd, gs, wd, ws, k, f"[{q[0]}] {what} k={k}")


@pytest.mark.parametrize("flat_scored", [True, False], ids=["default", "flat_scored_off"])
def test_scored_routes_match_reference(sweep, flat_scored):
    c = sweep
    if c.codec == tb.CODEC_GOOGLE and not flat_scored:
        pytest.skip("TRN_FLAT_SCORED only moves LUCENE queries (GOOGLE scores through k_exec_tiles already)")
    # the trees are meant to hold conditional leaves: scored in a second pass under a mask (OP_LEAFSCORE)
    for t in LEAFSCORE:
        steps, _, _ = tb.debug_compile(c.codec, c.index, c.tarr, c.plan(_q(t)), True)
        assert OP_LEAFSCORE in steps["op"].tolist(), f"[{t}] compiles without an OP_LEAFSCORE step"
    g = c.gpu(None if flat_scored else {"TRN_FLAT_SCORED": "0"})
    _check_scored(c, g, QUERIES, _expected_scored_routes(c.codec, flat_scored, QUERIES), "sweep")
    g.close()


# DocumentsOnly routes of QUERIES on GOOGLE (LUCENE: the step program for every query)
_S, _FO, _FA, _C, _FT = tb.ROUTE_STEPS, tb.ROUTE_FLAT_OR, tb.ROUTE_FLAT_AND, tb.ROUTE_CANDIDATE, tb.ROUTE_FLAT_TREE
DOCS_ROUTES_GOOGLE = [_S] * 10 + [_FO] * 5 + [_C, _C, _FA, _C, _FT, _FT, _FT] + [_FT, _C, _FT, _FT] + [_FT, _C] + [_S] * 3


def test_docs_routes_match_scored_sets(sweep):
    """the same queries in DocumentsOnly and compact mode: the k_exec_docs routes (for GOOGLE over the hits-heavy blocks of `stg` and `cst`,
    and through the resident bitmaps) must give the scored docID sets"""
    c = sweep
    g = c.gpu()
    plans = [c.plan(q, scored=False) for q in QUERIES]
    plain = g.exec_batch(plans, tb.MODE_DOCS_ONLY)
    routes = list(g.last_routes())
    comp = g.exec_batch(plans, tb.MODE_DOCS_COMPACT)
    assert routes == (DOCS_ROUTES_GOOGLE if c.codec == tb.CODEC_GOOGLE else [tb.ROUTE_STEPS] * len(QUERIES)), routes
    assert list(g.last_routes()) == routes
    for i, q in enumerate(QUERIES):
        want, _ = c.want(q, False)
        assert_same_docs(c.want(q, True)[0], want, f"[{q[0]}] reference: scored and DocumentsOnly sets")
        assert_same_docs(plain.query(i)[0], want, f"[{q[0]}] docs-only")
        assert int(plain.match_counts[i]) == len(want)
        assert_same_docs(comp.query(i)[0], want, f"[{q[0]}] docs-compact")
    if c.codec == tb.CODEC_GOOGLE:  # the upload decoded the same blocks, hits-heavy ones included, into a resident bitmap per term
        for t, n in enumerate(c.names):
            base, words = g.dense_bitmap(t)
            bits = np.unpackbits(words.view(np.uint8), bitorder="little")
            assert_same_docs((base + np.flatnonzero(bits)).astype(np.uint32), c.terms[n][0], f"{n}: resident bitmap")
    g.close()


def test_full_tile_list(sweep):
    """`all`: every document, one freq, one score.  On GOOGLE every 512-doc round of k_exec_tiles adds 512 keys to the k = 512 kept ones,
    filling its per-tile list (kTileListCap) exactly; the top 512 are docIDs 1 .. 512 on both routes"""
    c = sweep
    g = c.gpu()
    q = _q("all")
    for k in (511, 512):
        res = g.exec_batch([c.plan(q)], tb.MODE_SCORED_TOPK, k=k)
        assert list(g.last_routes()) == _expected_scored_routes(c.codec, True, [q])
        gd, gs = res.query(0)
        assert np.array_equal(gd, np.arange(1, k + 1, dtype=np.uint32)), gd[:16]
        assert int(res.match_counts[0]) == NDOCS
        wd, ws = c.want(q, True)
        assert_topk_exact(gd, gs, wd, ws, k, f"[all] k={k}")
    g.close()


# ------------------------------------------------------------------------------------------------ §3 runs of k_score_flat
NDOCS_RUNS = 3_300_000
RUN = 1 << 20  # 128 tiles of 8192 documents: one run under the default TRN_RUN_TILES


def _runs_terms():
    rng = np.random.default_rng(33)
    assert NDOCS_RUNS > 3 * RUN

    def sparse(n, best_lo, best_hi, nbest):
        d = np.sort(rng.choice(np.arange(1, NDOCS_RUNS + 1, dtype=np.uint32), n, replace=False))
        f = rng.integers(1, 9 if not nbest else 4, n).astype(np.uint32)
        cand = np.flatnonzero((d >= best_lo) & (d < best_hi))
        f[rng.choice(cand, nbest, replace=False)] = rng.integers(40, 300, nbest)
        return d, f

    terms = {
        "late": sparse(3000, 3 * RUN, NDOCS_RUNS + 1, 20),   # the best documents only in the last run
        "early": sparse(3000, 1, RUN, 20),                   # only in the first
        "spread": sparse(4000, 1, NDOCS_RUNS + 1, 60),      # in every run
        "filler": sparse(6000, 1, NDOCS_RUNS + 1, 0),
    }
    # 1280 consecutive documents around the end of runs 0, 1 and 2: block 4 of each stretch holds docIDs e - 88 .. e + 39
    d = np.concatenate([np.arange(e - 600, e + 680, dtype=np.uint32) for e in (RUN, 2 * RUN, 3 * RUN)])
    f = rng.integers(1, 100, len(d)).astype(np.uint32)
    f[rng.choice(len(d), 30, replace=False)] = rng.integers(100, 2000, 30)
    terms["strad"] = (d, f)
    return {n: (d, f, _positions(f)) for n, (d, f) in terms.items()}


RUN_QUERIES = [_q(t) for t in ["late", "early", "spread", "strad", "late OR filler", "early OR filler", "spread OR strad OR filler",
                               "late OR early OR spread OR strad"]]


@pytest.fixture(scope="module")
def runs(ref):
    return Corpus(ref, tb.CODEC_LUCENE, _runs_terms(), NDOCS_RUNS)


@pytest.mark.parametrize("run_tiles", ["1", "2", "default"])
def test_runs_topk(runs, run_tiles):
    c = runs
    for e in (RUN, 2 * RUN, 3 * RUN):  # the straddling blocks
        d = c.terms["strad"][0]
        blk = d[(np.flatnonzero(d == e - 88)[0] // 128) * 128:][:128]
        assert blk[0] < e <= blk[-1]
    for n, lo, hi in (("late", 3 * RUN, NDOCS_RUNS + 1), ("early", 1, RUN)):
        wd, ws = c.want(_q(n), True)
        top = wd[np.lexsort((wd, -ws))[:20]]
        assert np.all((top >= lo) & (top < hi)), n
    g = c.gpu(None if run_tiles == "default" else {"TRN_RUN_TILES": run_tiles})
    _check_scored(c, g, RUN_QUERIES, [tb.ROUTE_SCORE_FLAT] * len(RUN_QUERIES), f"run_tiles={run_tiles}")
    g.close()


# ------------------------------------------------------------------------------------------------ §4 phrase match counts
def _phrase_terms():
    """documents as token streams (one term per position, as the reference's DocWordsSpace keeps them) -> postings with positions"""
    rng = np.random.default_rng(64)
    vocab = ["x", "y", "z", "w"]
    docs = []
    for nx in (63, 64, 65, 128, 129):
        idx = {"62": [62], "63": [63], "64": [64], "127": [127], "last": [nx - 1], "mix": [0, 62, 63, 64, nx - 1], "all": list(range(nx)),
               "none": [], "odd": list(range(1, nx, 2))}
        for sel in idx.values():
            sel = {i for i in sel if i < nx}
            toks = ["w"]  # position 1; x at 2, 4, ..., followed by y where it matches
            for i in range(nx):
                toks += ["x", "y" if i in sel else "z"]
            docs.append(toks)
    for run in (63, 64, 65, 66, 129, 130):  # "x x": run - 1 matches
        docs.append(["w"] + ["x"] * run + ["y"])
    docs.append(["x", "x", "y"] + ["x", "y"] * 70)  # both phrases, "x y" 71 times
    prob = np.array([0.3, 0.3, 0.2, 0.2])
    for _ in range(400):
        docs.append([vocab[t] for t in rng.choice(4, size=int(rng.integers(3, 40)), p=prob)])
    order = rng.permutation(len(docs))  # documents of every shape spread over the docID space
    per = {t: {} for t in vocab}
    for slot, i in enumerate(order):
        doc = 1 + 37 * slot
        for pos, t in enumerate(docs[i], start=1):
            per[t].setdefault(doc, []).append(pos)
    out = {}
    for t in vocab:
        d = np.array(sorted(per[t]), np.uint32)
        f = np.array([len(per[t][int(x)]) for x in d], np.uint32)
        p = np.array([q for x in d for q in per[t][int(x)]], np.uint32)
        out[t] = (d, f, p)
    return out, 1 + 37 * len(docs)


PHRASES = [_q(t) for t in ['"x y"', '"x x"', '"y x"', '"x x y"', '"x y" AND w', 'z AND "x y"']]


@pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
def test_phrase_match_counts(ref, codec):
    terms, ndocs = _phrase_terms()
    c = Corpus(ref, codec, terms, ndocs, hits=True)
    wd, ws = c.want(_q('"x y"'), True)
    xd, xf = terms["x"][0], terms["x"][1]
    assert {63, 64, 65, 128, 129} <= set(xf.tolist())
    assert ws.max() == pytest.approx(tb.bm25_score(sum(tb.bm25_idf(len(terms[t][0]), ndocs) for t in "xy"), 129), rel=1e-6)
    assert len(c.want(_q('"x x"'), True)[0]) >= 7
    g = c.gpu()
    res = g.exec_batch([c.plan(q, scored=False) for q in PHRASES], tb.MODE_DOCS_ONLY)
    assert list(g.last_routes()) == [tb.ROUTE_STEPS] * len(PHRASES)
    for i, q in enumerate(PHRASES):
        assert_same_docs(res.query(i)[0], c.want(q, False)[0], f"[{q[0]}] docs-only")
    _check_scored(c, g, PHRASES, [tb.ROUTE_EXEC_TILES] * len(PHRASES), f"phrase codec={codec}")
    g.close()
