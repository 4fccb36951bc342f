"""GPU parity tests: the sm_90a path (through the C ABI) vs the reference's own CPU code (oracle/_ref).
docID sets bit-exact; BM25 within 1e-5 relative (north_star)."""
import numpy as np
import pytest

import trinity_b200 as tb
from test_codecs_cpu import make_lists
from util import PRIMES, Pair, assert_close_scores, assert_same_docs, assert_topk_equal, closed_form_lists

pytestmark = pytest.mark.gpu

CODECS = [tb.CODEC_GOOGLE, tb.CODEC_LUCENE]
NDOCS = 1_000_000

TEMPLATES = [
    "t1 AND t2",
    "t1 NOT t2",
    "t9 AND t10",
    "t1 AND t2 AND t3",
    "t3 OR t7",
    " OR ".join(f"t{i}" for i in range(1, 11)),
    "(t1 OR t2) AND (t3 OR t4) AND t5 NOT (t6 OR t7 OR t8)",
    "t1 AND t2 AND t3 NOT t4 NOT t5",
    "(t1 AND t2) OR (t3 AND t4) OR (t5 AND t6) NOT t7 NOT t8",
    "t1 AND (t2 OR t3 OR t4) NOT (t5 AND t6) AND (t7 OR t8)",
    "t10",
    "t1 AND nosuchterm",
    "t4 OR nosuchterm",
    "(t1 AND t2) OR (t1 AND t3)",
    "t2 t3 t5",
    "t1 | t9 -t3",
]
CLOSED_FORM_COUNTS = {  # SURVEY.md Appendix C
    "t1 AND t2": 166_666,
    "t1 NOT t2": 333_334,
    " OR ".join(f"t{i}" for i in range(1, 11)): 842_061,
    "(t1 OR t2) AND (t3 OR t4) AND t5 NOT (t6 OR t7 OR t8)": 15_678,
    "t1 AND t2 AND t3 NOT t4 NOT t5": 25_974,
    "(t1 AND t2) OR (t3 AND t4) OR (t5 AND t6) NOT t7 NOT t8": 196_138,
    "t1 AND (t2 OR t3 OR t4) NOT (t5 AND t6) AND (t7 OR t8)": 29_207,
}


@pytest.fixture(scope="module", params=CODECS, ids=["google", "lucene"])
def closed(request, ref):
    return Pair(ref, request.param, closed_form_lists(NDOCS), NDOCS)


def test_decode_whole_lists(ref):
    rng = np.random.default_rng(42)
    lists = make_lists(rng)
    nd = int(max(int(d[-1]) for d, _ in lists))
    for codec in CODECS:
        p = Pair(ref, codec, lists, nd)
        order = list(range(len(lists)))
        d, f, sums, ms = p.gpu.decode_terms(order, materialise=True)
        at = 0
        for i, (dd, ff) in enumerate(lists):
            rd, rf = p.ref.decode(i, len(dd) + 4)   # reference PostingsListIterator::next() stream
            assert_same_docs(d[at:at + len(dd)], rd, f"codec {codec} term {i} docids")
            assert np.array_equal(f[at:at + len(dd)] & 0xFFFF, rf), f"codec {codec} term {i} freqs"
            assert int(sums[i, 0]) == int(dd.astype(np.uint64).sum()) and int(sums[i, 1]) == int(ff.astype(np.uint64).sum())
            at += len(dd)
        # fused (checksum-only) variant agrees with the materialised one
        _, _, sums2, _ = p.gpu.decode_terms(order, materialise=False)
        assert np.array_equal(sums, sums2)


def test_docs_only_matches_reference(closed):
    qs = TEMPLATES
    res = closed.gpu.exec_batch([closed.plan(q) for q in qs], tb.MODE_DOCS_ONLY)
    for i, q in enumerate(qs):
        want, _ = closed.ref.exec(q, False, NDOCS)
        got, _ = res.query(i)
        assert_same_docs(got, want, f"[{q}]")
        assert int(res.match_counts[i]) == len(want)
        if q in CLOSED_FORM_COUNTS:
            assert len(got) == CLOSED_FORM_COUNTS[q]


def test_scored_all_matches_reference(closed):
    qs = [q for q in TEMPLATES if "nosuchterm" not in q]
    res = closed.gpu.exec_batch([closed.plan(q, scored=True) for q in qs], tb.MODE_SCORED_ALL)
    for i, q in enumerate(qs):
        wd, ws = closed.ref.exec(q, True, NDOCS)
        gd, gs = res.query(i)
        assert_same_docs(gd, wd, f"[{q}] scored")
        assert_close_scores(gs, ws, f"[{q}]")


def test_topk_matches_reference(closed):
    qs = [" OR ".join(f"t{i}" for i in range(1, 11)), "t1 AND t2", "t3 OR t7", "(t1 AND t2) OR (t3 AND t4) OR (t5 AND t6) NOT t7 NOT t8", "t10"]
    for k in (10, 100):
        res = closed.gpu.exec_batch([closed.plan(q, scored=True) for q in qs], tb.MODE_SCORED_TOPK, k=k)
        for i, q in enumerate(qs):
            wd, ws = closed.ref.exec(q, True, NDOCS)
            gd, gs = res.query(i)
            assert int(res.match_counts[i]) == len(wd)
            assert_topk_equal(gd, gs, wd, ws, k, f"[{q}] k={k}")


def test_optional_matches_reference(closed):
    """Optional(main, opt): <expr> beside a conjunction operand (exec.cpp:370-377, docset_iterators.h:174-206)"""
    from test_frontend_cpu import OPTIONAL_QUERIES
    qs = OPTIONAL_QUERIES
    res = closed.gpu.exec_batch([closed.plan(q) for q in qs], tb.MODE_DOCS_ONLY)
    sres = closed.gpu.exec_batch([closed.plan(q, scored=True) for q in qs], tb.MODE_SCORED_ALL)
    tres = closed.gpu.exec_batch([closed.plan(q, scored=True) for q in qs], tb.MODE_SCORED_TOPK, k=20)
    for i, q in enumerate(qs):
        want, _ = closed.ref.exec(q, False, NDOCS, parser_flags=8)
        assert_same_docs(res.query(i)[0], want, f"[{q}]")
        wd, ws = closed.ref.exec(q, True, NDOCS, parser_flags=8)
        gd, gs = sres.query(i)
        assert_same_docs(gd, wd, f"[{q}] scored")
        assert_close_scores(gs, ws, f"[{q}]")
        td, ts = tres.query(i)
        assert_topk_equal(td, ts, wd, ws, 20, f"[{q}] top-20")


def test_structural_scoring_known_answers(ref):
    """SURVEY.md Appendix C: which leaves contribute is structural, not 'all positive terms in the doc'"""
    lists = [(np.array(x, np.uint32), np.ones(len(x), np.uint32)) for x in
             ([10, 20, 41, 42, 43], [10, 20, 51], [10, 20, 30, 61, 62, 63, 64], [20, 30])]
    for codec in CODECS:
        p = Pair(ref, codec, lists, 1000, names=["a", "b", "c", "d"])
        qs = ["(a AND b) OR (c AND d)", "(a AND b) OR (a AND c)", "a AND b NOT d", "a OR b OR c OR d", "(a OR b) AND (c OR d)", "a NOT (b AND d)"]
        res = p.gpu.exec_batch([p.plan(q, scored=True) for q in qs], tb.MODE_SCORED_ALL)
        for i, q in enumerate(qs):
            wd, ws = p.ref.exec(q, True, 1000)
            gd, gs = res.query(i)
            assert_same_docs(gd, wd, f"[{q}]")
            assert_close_scores(gs, ws, f"[{q}]")
        # the published known answer: (a AND b) OR (c AND d) -> doc 10 scores a+b only
        gd, gs = res.query(0)
        assert list(gd) == [10, 20, 30]
        a, b = p.ref.bm25(0, 1), p.ref.bm25(1, 1)
        assert abs(gs[0] - (a + b)) < 1e-5 * (a + b)


def _random_queries(rng, names, n, kinds):
    out = []
    w = 1.0 / np.arange(1, len(names) + 1)
    w /= w.sum()
    for _ in range(n):
        kind = kinds[int(rng.integers(0, len(kinds)))]
        t = [names[i] for i in rng.choice(len(names), size=8, replace=False, p=w)]
        if kind == "and2":
            out.append(f"{t[0]} AND {t[1]}")
        elif kind == "or":
            out.append(" OR ".join(t[: int(rng.integers(2, 9))]))
        elif kind == "tree1":
            out.append(f"({t[0]} OR {t[1]}) AND ({t[2]} OR {t[3]}) AND {t[4]} NOT ({t[5]} OR {t[6]} OR {t[7]})")
        elif kind == "tree2":
            out.append(f"{t[0]} AND {t[1]} AND {t[2]} NOT {t[3]} NOT {t[4]}")
        elif kind == "tree3":
            out.append(f"({t[0]} AND {t[1]}) OR ({t[2]} AND {t[3]}) OR ({t[4]} AND {t[5]}) NOT {t[6]} NOT {t[7]}")
        else:
            out.append(f"{t[0]} AND ({t[1]} OR {t[2]} OR {t[3]}) NOT ({t[4]} AND {t[5]}) AND ({t[6]} OR {t[7]})")
    return out


@pytest.mark.parametrize("codec", CODECS, ids=["google", "lucene"])
def test_synthetic_zipf_index_random_queries(ref, codec):
    """config-shaped workload at a size the reference finishes in seconds: Zipfian synthetic index, random term draws ~ 1/r"""
    ndocs, nterms, min_df = 3_000_000, 96, 200
    s = tb.SynthIndex(codec, ndocs, nterms, min_df=min_df, threads=0)
    from refharness import RefIndex
    r = RefIndex.from_bytes(ref, codec, np.asarray(s.index), np.asarray(s.hits), s.names, np.asarray(s.terms), ndocs, s.sum_hits)
    g = tb.GpuIndexSource(0)
    g.upload(codec, np.asarray(s.index), np.asarray(s.terms), ndocs)
    tdict = tb.TermDictionary(s.names)
    rng = np.random.default_rng(0xC0FFEE)
    # whole-list decode of a few terms (dense head, mid, sparse tail) against the reference iterators
    probe = [0, 1, 7, 40, nterms - 1]
    d, f, sums, _ = g.decode_terms(probe, materialise=True)
    at = 0
    for t in probe:
        rd, rf = r.decode(t, int(s.terms["documents"][t]) + 4)
        assert_same_docs(d[at:at + len(rd)], rd, f"decode term {t}")
        assert np.array_equal(f[at:at + len(rd)], rf)
        at += len(rd)
    qs = _random_queries(rng, s.names, 40, ["and2", "and2", "or", "tree1", "tree2", "tree3", "tree4"])
    res = g.exec_batch([tb.parse_query(q, tdict) for q in qs], tb.MODE_DOCS_ONLY)
    for i, q in enumerate(qs):
        want, _ = r.exec(q, False, ndocs)
        got, _ = res.query(i)
        assert_same_docs(got, want, f"[{q}]")
    sq = _random_queries(rng, s.names, 16, ["or", "and2", "tree3", "tree4"])
    plans = [g.set_bm25_weights(tb.parse_query(q, tdict), ndocs) for q in sq]
    res_all = g.exec_batch(plans, tb.MODE_SCORED_ALL)
    res_top = g.exec_batch(plans, tb.MODE_SCORED_TOPK, k=100)
    for i, q in enumerate(sq):
        wd, ws = r.exec(q, True, ndocs)
        gd, gs = res_all.query(i)
        assert_same_docs(gd, wd, f"[{q}] scored")
        assert_close_scores(gs, ws, f"[{q}]")
        td, ts = res_top.query(i)
        assert_topk_equal(td, ts, wd, ws, 100, f"[{q}] top-100")


def test_edge_cases(ref):
    """empty / ragged inputs and tile-boundary docIDs"""
    W = 16384
    lists = [
        (np.array([1], np.uint32), np.array([3], np.uint32)),                                 # single doc
        (np.array([W - 1, W, W + 1, 2 * W - 1, 2 * W, 5 * W + 7], np.uint32), np.ones(6, np.uint32)),  # straddles tile edges
        (np.arange(1, 40 * W, 997, dtype=np.uint32), np.ones(len(np.arange(1, 40 * W, 997)), np.uint32)),
        (np.arange(W - 40, W + 40, dtype=np.uint32), np.full(80, 2, np.uint32)),
        (np.array([40 * W - 1], np.uint32), np.array([1], np.uint32)),                        # last doc of the space
    ]
    nd = 40 * W - 1
    qs = ["t1", "t2", "t2 AND t4", "t2 OR t4", "t3 NOT t4", "t4 NOT t2", "t1 AND t5", "t5 OR t1", "t3 AND t4", "t2 AND t3", "t4 AND nosuch", "nosuch"]
    for codec in CODECS:
        p = Pair(ref, codec, lists, nd)
        res = p.gpu.exec_batch([p.plan(q) for q in qs], tb.MODE_DOCS_ONLY)
        for i, q in enumerate(qs):
            want, _ = p.ref.exec(q, False, nd + 1)
            got, _ = res.query(i)
            assert_same_docs(got, want, f"codec {codec} [{q}]")
        sres = p.gpu.exec_batch([p.plan(q, scored=True) for q in qs[:10]], tb.MODE_SCORED_TOPK, k=5)
        for i, q in enumerate(qs[:10]):
            wd, ws = p.ref.exec(q, True, nd + 1)
            gd, gs = sres.query(i)
            assert_topk_equal(gd, gs, wd, ws, 5, f"codec {codec} [{q}] top-5")


def test_no_device_fails_loudly():
    with pytest.raises(tb.TrinityError):
        tb.GpuIndexSource(device=4096)


def test_large_batches_split_by_result_capacity_and_stay_exact(ref):
    """a docs-only OR batch whose match upper bound exceeds the staging budget is split internally (pipelined chunks); results
    must be identical to per-query execution, and a 64-query batch exercises the chunked host-buffer path"""
    ndocs = 400_000
    p = Pair(ref, tb.CODEC_GOOGLE, closed_form_lists(ndocs), ndocs)
    qs = [f"t{1 + i % 10} OR t{1 + (i * 3 + 1) % 10}" for i in range(70)] + [f"t{1 + i % 10} AND t{1 + (i + 1) % 10}" for i in range(70)]
    res = p.gpu.exec_batch([p.plan(q) for q in qs], tb.MODE_DOCS_ONLY)
    sres = p.gpu.exec_batch([p.plan(q, scored=True) for q in qs], tb.MODE_SCORED_ALL)
    cache = {}
    for i, q in enumerate(qs):
        if q not in cache:
            cache[q] = (p.ref.exec(q, False, ndocs + 1)[0], p.ref.exec(q, True, ndocs + 1))
        assert_same_docs(res.query(i)[0], cache[q][0], f"#{i} [{q}]")
        gd, gs = sres.query(i)
        assert_same_docs(gd, cache[q][1][0], f"#{i} [{q}] scored")
        assert_close_scores(gs, cache[q][1][1], f"#{i} [{q}]")
    assert int(res.offsets[-1]) == sum(len(cache[q][0]) for q in qs)


@pytest.mark.parametrize("block_docs,step", [(8, 8), (16, 1), (64, 8), (128, 64)])
def test_decode_other_google_block_sizes(ref, block_docs, step):
    """the decode sweep of BASELINE.json configs[4]: GOOGLE-layout indexes built with other block sizes / skiplist steps than the
    reference's 32 / 8 (google_codec.h:17-20) decode to the same postings; the exec entry points refuse them"""
    rng = np.random.default_rng(block_docs)
    lists = make_lists(rng)
    nd = int(max(int(d[-1]) for d, _ in lists))
    b = tb.IndexBuilder(tb.CODEC_GOOGLE)
    b.set_google_block(block_docs, step)
    for d, f in lists:
        b.add_term(d, f)
    g = tb.GpuIndexSource(0)
    g.upload(tb.CODEC_GOOGLE, b.index(), b.terms_array(), nd)
    assert g.info()["block_docs"] in (block_docs, 32)  # 32 only if no list is long enough to show the block size
    d, f, sums, _ = g.decode_terms(list(range(len(lists))), materialise=True)
    at = 0
    for i, (dd, ff) in enumerate(lists):
        assert_same_docs(d[at:at + len(dd)], dd, f"block {block_docs} term {i} docids")
        assert np.array_equal(f[at:at + len(dd)], ff), f"block {block_docs} term {i} freqs"
        assert int(sums[i, 0]) == int(dd.astype(np.uint64).sum()) and int(sums[i, 1]) == int(ff.astype(np.uint64).sum())
        at += len(dd)
    _, _, sums2, _ = g.decode_terms(list(range(len(lists))), materialise=False)
    assert np.array_equal(sums, sums2)
    if g.info()["block_docs"] != 32:
        with pytest.raises(tb.TrinityError):
            g.exec_batch([tb.parse_query("t1", tb.TermDictionary([f"t{i + 1}" for i in range(len(lists))]))], tb.MODE_DOCS_ONLY)
    g.close()
