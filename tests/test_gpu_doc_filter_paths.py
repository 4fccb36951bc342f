"""Per-query document filters on the paths test_gpu_doc_filter does not reach with its closed-form batch, against the reference: the
all-bitmap and mixed run tickets (asserted non-empty), every compact encoding, phrases and MatchSome, the top of the docID space by
translation, a deny set equal to the match set, exact tie order at the top-k cut, top-k merged from 2, 3 and 8 docID shards, the default
exec mode with masked documents, and a collection of three generations against the reference's collection loop.

Oracles: the reference's exec_query with a masked_documents_registry holding the masked documents plus every document the filter drops
(the same predicate), or the reference's unfiltered run restricted on the host (where the oracle call takes no registry)."""
import numpy as np
import pytest
import torch

import trinity_b200 as tb
from matchutil import RefMatches, assert_same_matches, doc_corpus, gpu_as_list, host_build, ref_build  # noqa: F401
from test_gpu_docid_limits import DELTA, DOCS, Space, _docs_queries
from test_gpu_segments import lists as seg_lists
from test_gpu_sharded import TOPK_QUERIES, Shard, _lists
from trinity_b200.segments import SegmentCollection
from trinity_b200.sharded import device_view, shard_range
from util import Pair, assert_close_scores, assert_same_docs, assert_topk_equal, assert_topk_exact, closed_form_lists

pytestmark = pytest.mark.gpu
NDOCS = 300_000


def _mid_term(ndocs, seed=3):
    """one document in 30: too dense for the candidate path, too sparse for a resident bitmap (a flat AND with it is a mixed run)"""
    rng = np.random.default_rng(seed)
    d = np.unique(rng.integers(1, ndocs + 1, ndocs // 30)).astype(np.uint32)
    return d, (1 + d % 4).astype(np.uint32)


def _keep(docs, allow, deny):
    k = np.ones(len(docs), bool)
    if allow is not None:
        k &= np.isin(docs, allow)
    if deny is not None:
        k &= ~np.isin(docs, deny)
    return k


def test_run_tickets_compact_phrase_matchsome(ref):
    lists = closed_form_lists(NDOCS) + [_mid_term(NDOCS)]
    names = [f"t{i + 1}" for i in range(10)] + ["mid"]
    p = Pair(ref, tb.CODEC_GOOGLE, lists, NDOCS, names=names)
    rng = np.random.default_rng(21)
    allow = np.unique(rng.integers(1, NDOCS + 1, NDOCS // 3)).astype(np.uint32)
    deny = np.arange(5, NDOCS + 1, 5, dtype=np.uint32)
    masked = np.unique(rng.integers(1, NDOCS + 1, 3000)).astype(np.uint32)
    p.gpu.set_masked_documents(masked)
    ign = np.union1d(masked, np.union1d(np.setdiff1d(np.arange(1, NDOCS + 1, dtype=np.uint32), allow), deny)).astype(np.uint32)
    dense_q, mixed_q = "t1 AND t2", "t1 AND mid"
    # (run tickets are off in a batch that holds a phrase plan: the phrase queries run in a batch of their own)
    batches = [[dense_q, mixed_q, "t1 OR mid OR t7", "t1 AND (t2 OR mid) NOT t5"], ['"t1 t2"', 't3 AND "t1 t2"']]
    plans = [p.plan(q) for q in batches[0]]
    _, dense_t = tb.debug_dense_runs(tb.CODEC_GOOGLE, p.index, p.terms, plans, tb.MODE_DOCS_ONLY, 100, NDOCS)
    _, mixed_t = tb.debug_mixed_runs(tb.CODEC_GOOGLE, p.index, p.terms, plans, tb.MODE_DOCS_ONLY, 100, NDOCS)
    assert len(dense_t) and set(dense_t[:, 0].tolist()) == {0}, "the all-bitmap AND runs on dense run tickets"
    assert len(mixed_t) and set(mixed_t[:, 0].tolist()) == {1}, "the AND with one decoded operand runs on mixed run tickets"
    flt = tb.DocFilter(p.gpu.docset(allow), p.gpu.docset(deny))
    encodings = set()
    for mode, queries in ((m, b) for m in (tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT) for b in batches):
        res = p.gpu.exec_batch([p.plan(q) for q in queries], mode, filters=[flt] * len(queries), copy=False)
        if queries is batches[0]:
            assert int(p.gpu.last_routes()[0]) == tb.ROUTE_FLAT_AND and int(p.gpu.last_routes()[1]) == tb.ROUTE_FLAT_AND
        if mode == tb.MODE_DOCS_COMPACT:
            desc = np.ctypeslib.as_array(res.raw.item_desc, shape=(max(res.nitems, 1),))[: res.nitems]
            encodings |= set(int(x) >> 30 for x in desc if int(x) & 0x3FFFFFFF)
        for i, q in enumerate(queries):
            want, _ = p.ref.exec_masked(q, False, ign, NDOCS + 1)
            assert_same_docs(res.query(i)[0].copy(), want, f"[{q}] mode {mode}")
            assert int(res.match_counts[i]) == len(want)
    assert encodings >= {1, 2, 3}, encodings  # 16-bit offsets, bitmaps and bucketed 8-bit offsets, chosen from the filtered counts
    # MatchSome (the reference's parser flag 16): the unfiltered reference run restricted on the host
    for q, m in (("[t1, t2, t3]", 2), ("[t2, t5, mid, t7]", 3)):
        plan = tb.parse_query(q, p.tdict, min_match=m)
        res = p.gpu.exec_batch([plan, plan], tb.MODE_DOCS_ONLY, filters=[flt, None])
        want, _ = p.ref.exec(q, False, NDOCS + 1, parser_flags=16, min_match=m)
        want = want[~np.isin(want, masked)]
        assert_same_docs(res.query(0)[0], want[_keep(want, allow, deny)], f"[{q}] filtered")
        assert_same_docs(res.query(1)[0], want, f"[{q}] unfiltered beside")
    p.gpu.close()


def test_candidate_compact_and_deny_equal_to_match_set(ref, monkeypatch):
    monkeypatch.setenv("TRN_CAND_COST", "1")
    p = Pair(ref, tb.CODEC_GOOGLE, closed_form_lists(NDOCS), NDOCS)
    q = "t3 AND t7"
    want, _ = p.ref.exec(q, False, NDOCS + 1)
    allow = want[::3].copy()
    res = p.gpu.exec_batch([p.plan(q), p.plan(q)], tb.MODE_DOCS_COMPACT, filters=[tb.DocFilter(allow=p.gpu.docset(allow)),
                                                                                     tb.DocFilter(deny=p.gpu.docset(want))], copy=False)
    assert int(p.gpu.last_routes()[0]) == tb.ROUTE_CANDIDATE
    desc = np.ctypeslib.as_array(res.raw.item_desc, shape=(max(res.nitems, 1),))[: res.nitems]
    assert {int(x) >> 30 for x in desc if int(x) & 0x3FFFFFFF} == {0}  # plain docIDs
    assert_same_docs(res.query(0)[0].copy(), allow, "candidate, allow a third")
    assert len(res.query(1)[0]) == 0 and int(res.match_counts[1]) == 0  # deny == the match set
    for mode, k in ((tb.MODE_SCORED_ALL, 0), (tb.MODE_SCORED_TOPK, 10)):
        r = p.gpu.exec_batch([p.plan(q, scored=True)], mode, k=max(k, 1), filters=[tb.DocFilter(deny=p.gpu.docset(want))])
        assert len(r.query(0)[0]) == 0 and int(r.match_counts[0]) == 0
    p.gpu.close()


@pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
def test_top_of_the_docid_space(ref, codec):
    sp = Space(ref, codec)
    top = np.uint64(2**32 - 2)
    allow = np.unique(np.concatenate([np.arange(DELTA + 1, DELTA + 600_001, 3, dtype=np.uint64), [top, top - 1, top - 8192]])).astype(np.uint32)
    flt = tb.DocFilter(allow=sp.gpu.docset(allow))
    qs = _docs_queries(codec)
    res = sp.gpu.exec_batch([sp.plan(q) for q in qs], tb.MODE_DOCS_ONLY, filters=[flt] * len(qs))
    for i, q in enumerate(qs):
        wd, _ = sp.want(q, False)
        assert_same_docs(res.query(i)[0], wd[np.isin(wd, allow)], f"top of the space [{q}]")
    assert set(DOCS) >= set(qs)
    sp.gpu.close()


@pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
def test_top_k_exact_ties(ref, codec):
    """closed-form lists: scores depend on freq (1..5) only, so the cut falls inside long runs of equal scores; ties go by docID"""
    p = Pair(ref, codec, closed_form_lists(NDOCS), NDOCS)
    rng = np.random.default_rng(22)
    deny = np.unique(rng.integers(1, NDOCS + 1, NDOCS // 2)).astype(np.uint32)
    for q in ("t10", "t3 OR t7"):
        plan = p.plan(q, scored=True)
        wd, ws = p.ref.exec_masked(q, True, deny, NDOCS + 1)
        for k in (1, 100, 512):
            res = p.gpu.exec_batch([plan], tb.MODE_SCORED_TOPK, k=k, filters=[tb.DocFilter(deny=p.gpu.docset(deny))])
            assert_topk_exact(*res.query(0), wd, ws, k, f"[{q}] k={k}")
            assert int(res.match_counts[0]) == len(wd)
    p.gpu.close()


@pytest.mark.parametrize("nshards", [2, 3, 8])
def test_sharded_top_k(ref, nshards):
    codec, ndocs = tb.CODEC_LUCENE, 400_000
    lists, names = _lists(ndocs)
    whole = Pair(ref, codec, lists, ndocs, names=names, upload=False)
    full_df = np.array([len(d) for d, _ in lists])
    shards = [Shard(codec, lists, names, *shard_range(ndocs, r, nshards), ndocs, full_df) for r in range(nshards)]
    rng = np.random.default_rng(23)
    allow = np.unique(rng.integers(1, ndocs + 1, ndocs // 2)).astype(np.uint32)
    ign = np.setdiff1d(np.arange(1, ndocs + 1, dtype=np.uint32), allow)
    nq, k = len(TOPK_QUERIES), 50
    gd = torch.zeros((nshards, nq, k), dtype=torch.int32, device="cuda")
    gs = torch.zeros((nshards, nq, k), dtype=torch.float32, device="cuda")
    counts = np.zeros(nq, np.int64)
    for si, s in enumerate(shards):
        f = tb.DocFilter(allow=s.gpu.docset(allow))  # every shard context registers the same global set
        s.gpu.exec_batch_device([s.plan(q, scored=True) for q in TOPK_QUERIES], tb.MODE_SCORED_TOPK, k, filters=[f] * nq)
        dptr, sptr, _ = s.gpu.last_topk_device()
        torch.cuda.synchronize()
        gd[si].view(-1).copy_(device_view(dptr, nq * k, torch.int32))
        gs[si].view(-1).copy_(device_view(sptr, nq * k, torch.float32))
        counts += np.asarray(s.gpu.fetch().match_counts, np.int64)
    md = torch.zeros((nq, k), dtype=torch.int32, device="cuda")
    ms = torch.zeros((nq, k), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    shards[0].gpu.merge_topk(gd.data_ptr(), gs.data_ptr(), nshards, nq, k, md.data_ptr(), ms.data_ptr())
    torch.cuda.synchronize()
    md, ms = md.cpu().numpy().view(np.uint32), ms.cpu().numpy()
    for i, q in enumerate(TOPK_QUERIES):
        wd, ws = whole.ref.exec_masked(q, True, ign, ndocs + 1)
        assert counts[i] == len(wd), f"{nshards} shards [{q}]: summed match counts"
        keep = ms[i] >= 0
        assert_topk_equal(md[i][keep], ms[i][keep], wd, ws, k, f"{nshards} shards [{q}] filtered")
    for s in shards:
        s.gpu.close()


@pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
def test_matched_terms_against_reference(ref, codec):
    rng = np.random.default_rng(24)
    ndocs = 20_000
    mlists, _ = doc_corpus(rng, ndocs, 10)
    names = [f"w{i + 1}" for i in range(10)]
    index, hits, terms = host_build(codec, mlists)
    r = ref_build(codec, mlists, names, ndocs)
    g = tb.GpuIndexSource(0)
    g.upload(codec, index, terms, ndocs)
    if codec == tb.CODEC_LUCENE:
        g.upload_hits(index, hits)
    tdict = tb.TermDictionary(names)
    masked = np.unique(rng.integers(1, ndocs + 1, 500)).astype(np.uint32)
    g.set_masked_documents(masked)
    allow = np.unique(rng.integers(1, ndocs + 1, ndocs // 2)).astype(np.uint32)
    deny = np.arange(7, ndocs + 1, 7, dtype=np.uint32)
    ign = np.union1d(masked, np.union1d(np.setdiff1d(np.arange(1, ndocs + 1, dtype=np.uint32), allow), deny)).astype(np.uint32)
    queries = ["w1 AND w2", "w1 OR w3 OR w5", "w2 AND (w3 OR w4) NOT w6", '"w1 w2"', "w1", "w7"]
    flt = tb.DocFilter(g.docset(allow), g.docset(deny))
    res = g.exec_matches([tb.parse_query(q, tdict) for q in queries], filters=[flt] * len(queries))
    for i, q in enumerate(queries):
        if " " not in q:
            # one term: the reference's filtered Handler reports freq 1 here (exec.cpp:991, 1005-1026); the engine reports the true freq and
            # hits, those of the reference's run with the masked documents only, restricted to the kept documents
            full = r.exec(q, 0, 0, masked)
            kept = set(np.setdiff1d(np.array([d for d, _ in full], np.uint32), ign).tolist())
            want = [x for x in full if x[0] in kept]
        else:
            want = r.exec(q, 0, 0, ign)
        assert_same_matches(gpu_as_list(res, i), want, f"codec {codec} [{q}] filtered")
    g.close()


@pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
def test_collection_of_three_generations(ref, tmp_path, codec):
    n = 200_000
    paths = [tmp_path / "1", tmp_path / "2", tmp_path / "3"]
    for x in paths:
        x.mkdir()
    ref.segment_write(codec, paths[0], seg_lists(1, 1, n, "onlyold"))
    ref.segment_write(codec, paths[1], seg_lists(2, 150_000, 260_000, "onlynew"), np.arange(5, 90_000, 7, dtype=np.uint32), replace_below=n)
    ref.segment_write(codec, paths[2], seg_lists(3, 240_000, 300_000, "onlythird"), np.arange(11, 40_000, 13, dtype=np.uint32), replace_below=260_000)
    col = SegmentCollection(paths)
    assert col.generations == [3, 2, 1]
    rcol = ref.collection_open(paths)
    rng = np.random.default_rng(25)
    queries = ["w1 AND w2", "w3 OR w7 OR w9", "w1 AND (w2 OR w3) NOT w5", "w10", "w1 OR onlynew", "w2 AND onlythird"]
    a = np.unique(rng.integers(1, 300_001, 120_000)).astype(np.uint32)
    d = np.arange(3, 300_001, 3, dtype=np.uint32)
    allow = [a, None, a, None, a, None]
    deny = [None, d, d, None, None, d]
    cap = 700_000
    for mode, scored in ((tb.MODE_DOCS_ONLY, False), (tb.MODE_SCORED_ALL, True), (tb.MODE_SCORED_TOPK, True)):
        res = col.exec_batch(queries, mode, k=25, allow=allow, deny=deny)
        for i, q in enumerate(queries):
            for s, (wd, ws) in enumerate(rcol.collection_exec(q, scored, cap)):
                m = _keep(wd, allow[i], deny[i])
                gd, gs = res[s].query(i)
                what = f"[{q}] generation {col.generations[s]} mode {mode}"
                assert int(res[s].match_counts[i]) == int(m.sum()), what
                if mode == tb.MODE_SCORED_TOPK:
                    assert_topk_equal(gd, gs, wd[m], ws[m], 25, what)
                else:
                    assert_same_docs(gd, wd[m], what)
                    if scored:
                        assert_close_scores(gs, ws[m], what)
    assert len(col._docsets) == 2  # a and d, each registered once per source
    col.release_docsets()
    assert not col._docsets
    for g in col.sources:
        g.close()
