"""One GpuIndexSource used the way bench.py and a serving process use it: a single context on a non-default stream, called again and again
with batches of every size and mode, masks set and replaced between them, new indexes uploaded into it.  Everything a call returns is
compared with the reference (oracle/_ref): docIDs bit-exact, BM25 within 1e-5, top-k per assert_topk_equal.

A. The bench's 1000-query batches (bench.gen_queries on a 4*10^6-document, 512-term synthetic index) through exec_batch_device + fetch in
   every mode the workload allows; the compact stream equals word for word that of the pipelined exec_batch.
B. bench.py's own call order on one context, under the session's chunk knobs and under the production planner (result-size hint of the
   previous batch, one chunk tapered into 1/2, 1/4, 1/4); every call's chunk count is the engine's plan for the hint the call before left.
C. Changing batch sizes and modes, an all-empty batch after the largest, masks replaced and cleared, re-uploads of smaller and larger
   indexes and of the other codec, and what fetch() returns after each kind of call."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import bench
import trinity_b200 as tb
from refharness import RefIndex
from test_gpu_emit_layout import QItems
from trinity_b200._ffi import TrnResult, lib
from util import assert_close_scores, assert_same_docs, assert_topk_equal

pytestmark = pytest.mark.gpu

NDOCS, NTERMS, NQ, K = 4_000_000, 512, 1000, 100
THREADS = max(1, len(os.sched_getaffinity(0)))
G, L = tb.CODEC_GOOGLE, tb.CODEC_LUCENE
COMPACT, DOCS, ALL, TOPK = tb.MODE_DOCS_COMPACT, tb.MODE_DOCS_ONLY, tb.MODE_SCORED_ALL, tb.MODE_SCORED_TOPK
# the mode bench.py times for each workload, and the other modes checked through the device-resident form (or10 in DocumentsOnly or
# SCORED_ALL would return 2.5 * 10^9 matches per 1000-query batch at this size: top-k only)
MODES = {"and2": [COMPACT, DOCS, ALL], "tree8": [COMPACT, DOCS, ALL], "and2l": [COMPACT, DOCS, ALL], "or10": [TOPK]}


class World:
    """one synthetic index (the bench's generator), the reference over the same bytes, and the reference's answers, cached per query text"""

    def __init__(self, ref, codec, ndocs, seed=0x5EED):
        self.codec, self.ndocs = codec, ndocs
        s = tb.SynthIndex(codec, ndocs, NTERMS, seed=seed, threads=THREADS)
        self.synth, self.index, self.terms, self.hits = s, np.asarray(s.index), np.asarray(s.terms), np.asarray(s.hits)
        self.ref = RefIndex.from_bytes(ref, codec, self.index, self.hits, s.names, self.terms, ndocs, s.sum_hits)
        self.tdict = tb.TermDictionary(s.names)
        self.df = bench.synth_dfs(ndocs, NTERMS)
        assert np.array_equal(self.df, self.terms["documents"].astype(np.int64))  # the closed form bench.py weights with
        self._cs, self._full = {}, {}

    def plans(self, texts):
        """parsed with BM25 weights set as bench.py sets them (global df of the closed form)"""
        out = []
        for t in texts:
            p = tb.parse_query(t, self.tdict)
            for x in p:
                if x["kind"] == tb.NODE_TERM and x["term"] != tb.EMPTY_TERM:
                    x["weight"] = tb.bm25_idf(int(self.df[x["term"]]), self.ndocs)
            out.append(p)
        return out

    def counts_sums(self, texts):
        """per query the reference's match count and docID sum (its exec_batch, DocumentsOnly, on all host threads)"""
        todo = sorted({t for t in texts if t not in self._cs})
        if todo:
            _, counts, sums, _, _ = self.ref.exec_batch(todo, False, 1, THREADS)
            self._cs.update({t: (int(c), int(s)) for t, c, s in zip(todo, counts, sums)})
        return (np.array([self._cs[t][0] for t in texts], np.uint64), np.array([self._cs[t][1] for t in texts], np.uint64))

    def full(self, text, scored):
        key = (text, scored)
        if key in self._full:
            return self._full[key]
        out = self.ref.exec(text, scored, self.ndocs + 1)
        if len(out[0]) <= 600_000:  # (the long or10 lists are recomputed rather than kept)
            self._full[key] = (out[0].copy(), None if out[1] is None else out[1].copy())
        return out


def _topk_check(gd, gs, wd, ws, k, what):
    """assert_topk_equal on the part of the reference stream that can decide it: every document scoring within 1e-4 of the k-th score or
    above (the top-k, its near ties and anything the device might wrongly return in their place)"""
    if len(ws) > k:
        kth = np.partition(ws, len(ws) - k)[len(ws) - k]
        keep = ws >= kth * (1 - 1e-4)
        wd, ws = wd[keep], ws[keep]
    assert_topk_equal(gd, gs, wd, ws, k, what)


def check(w, texts, res, mode, k, what, sample, counts=None):
    """every query's match count and docID sum; the full result of the `sample` queries"""
    if counts is None:
        counts, sums = w.counts_sums(texts)
    got = np.asarray(res.match_counts[: len(texts)], np.uint64)
    bad = np.flatnonzero(got != counts)
    assert not len(bad), f"{what}: match counts differ at {bad[:8]}: got {got[bad[:4]]} want {counts[bad[:4]]}"
    if mode != TOPK:
        cs = res.checksums()
        bad = np.flatnonzero(cs != sums)
        assert not len(bad), f"{what}: docID sums differ at {bad[:8]}"
    for q in sample:
        gd, gs = res.query(int(q))
        wd, ws = w.full(texts[q], mode in (ALL, TOPK))
        label = f"{what} [{q}] {texts[q]}"
        if mode == TOPK:
            _topk_check(gd, gs, wd, ws, k, label)
        else:
            assert_same_docs(np.asarray(gd), wd, label)
            if mode == ALL:
                assert_close_scores(gs, ws, label)


def sample_of(n, m, seed):
    return np.sort(np.random.default_rng(seed).choice(n, min(n, m), replace=False))


def fetch_view(g):
    """fetch() without the host-side decode: the trn_result of trn_fetch_results as it stands (compact: its raw stream)"""
    r = TrnResult()
    g._ck(g._L.trn_fetch_results(g._h, C.byref(r)))
    mode, k, _ = g._last
    return g._wrap(r, mode, k, copy=False)


def stream(res):
    """(query offsets in words, words, item_desc, qitems) of a compact result"""
    raw, nq = res.raw, res.nq
    off = np.ctypeslib.as_array(raw.offsets, shape=(nq + 1,)).copy()
    words = np.ctypeslib.as_array(raw.words, shape=(max(int(raw.total_words), 1),))[: int(raw.total_words)].copy()
    desc = np.ctypeslib.as_array(raw.item_desc, shape=(max(res.nitems, 1),))[: res.nitems].copy()
    qi = C.cast(raw.qitems, C.POINTER(QItems))
    return off, words, desc, [(qi[q].item_base, qi[q].nitems, qi[q].tile_lo, qi[q].tile_shift) for q in range(nq)]


def assert_same_stream(a, b, what):
    assert a[3] == b[3], f"{what}: qitems differ"
    assert np.array_equal(a[2], b[2]), f"{what}: item_desc differs at {np.flatnonzero(a[2] != b[2])[:8] if len(a[2]) == len(b[2]) else 'length'}"
    assert np.array_equal(a[0], b[0]), f"{what}: query offsets differ"
    assert np.array_equal(a[1], b[1]), f"{what}: words differ"


def new_source(w, stream_):
    g = tb.GpuIndexSource(0)
    g.set_stream(stream_.cuda_stream)
    g.upload(w.codec, w.index, w.terms, w.ndocs)
    return g


@pytest.fixture(scope="module")
def worlds(ref):
    cache = {}

    def get(codec, ndocs=NDOCS, seed=0x5EED):
        if (codec, ndocs, seed) not in cache:
            cache[(codec, ndocs, seed)] = World(ref, codec, ndocs, seed)
        return cache[(codec, ndocs, seed)]
    return get


@pytest.fixture(scope="module")
def side_stream():
    return torch.cuda.Stream()


@pytest.fixture(scope="module")
def ctx(worlds, side_stream):
    """one context per codec for the whole module, on a non-default stream"""
    live = {}

    def get(codec):
        if codec not in live:
            live[codec] = new_source(worlds(codec), side_stream)
        return live[codec]
    yield get
    for g in live.values():
        g.close()


def workload(w, wl):
    texts, _ = bench.gen_queries(wl, NQ, NTERMS)
    return texts, w.plans(texts)


# ============================================================================================== A. bench-shaped batches, device-resident
def test_bench_batches_hold_every_ticket_kind(worlds):
    """the and2 batch holds dense-run, mixed-run and candidate-driven queries, tree8 flat-tree ones: the paths the tests below exercise"""
    w = worlds(G)
    _, plans = workload(w, "and2")
    routes, _ = tb.debug_plan(G, w.index, w.terms, plans, DOCS, max_docid=NDOCS)
    dense = tb.debug_dense_runs(G, w.index, w.terms, plans, DOCS, max_docid=NDOCS)[1]
    mixed = tb.debug_mixed_runs(G, w.index, w.terms, plans, DOCS, max_docid=NDOCS)[1]
    assert len(set(dense[:, 0])) >= 50 and len(set(mixed[:, 0])) >= 50, (len(dense), len(mixed))
    assert np.count_nonzero(routes == tb.ROUTE_CANDIDATE) >= 50 and np.count_nonzero(routes == tb.ROUTE_FLAT_AND) >= 100
    _, plans = workload(w, "tree8")
    routes, _ = tb.debug_plan(G, w.index, w.terms, plans, DOCS, max_docid=NDOCS)
    assert np.count_nonzero(routes == tb.ROUTE_FLAT_TREE) >= 100 and np.count_nonzero(routes == tb.ROUTE_CANDIDATE) >= 50


@pytest.mark.parametrize("wl", ["and2", "tree8", "and2l", "or10"])
def test_device_resident_batch(worlds, ctx, wl):
    codec = bench.WORKLOADS[wl]["codec"]
    w, g = worlds(codec), ctx(codec)
    texts, plans = workload(w, wl)
    packed = g.pack(plans)
    sample = sample_of(NQ, 100, 11)
    for mode in MODES[wl]:
        what = f"{wl} mode {mode}"
        want_routes, _ = tb.debug_plan(codec, w.index, w.terms, plans, DOCS if mode == COMPACT else mode, k=K, max_docid=NDOCS)
        g.exec_batch_device(plans, mode, K, packed=packed)
        assert np.array_equal(g.last_routes(), want_routes), what
        if mode == TOPK:
            # every query's match count and top-k scores against the reference's own top-k sink (bench.py's parity check)
            _, counts, _, _, tsc = w.ref.exec_batch(texts, True, K, THREADS)
            res = g.fetch()
            check(w, texts, res, mode, K, what + " device", sample, counts=counts)
            for q in range(NQ):
                gd, gs = res.query(q)
                assert len(gs) == min(K, int(counts[q])), (what, q)
                assert_close_scores(gs, tsc[q][: len(gs)], f"{what} [{q}] top-k scores")
            continue
        dev = fetch_view(g)
        check(w, texts, dev, mode, K, what + " device", sample)
        if mode == COMPACT:
            want = stream(dev)
        else:
            want = (dev.offsets.copy(), dev.docids.copy(), None if dev.scores is None else dev.scores.copy())
        host = g.exec_batch(plans, mode, K, copy=False, packed=packed)
        assert g.last_timings()["chunks"] > 1, what
        assert np.array_equal(g.last_routes(), want_routes), what
        if mode == COMPACT:
            assert_same_stream(stream(host), want, what + ": pipelined vs device-resident")
            assert np.array_equal(np.asarray(host.match_counts), np.asarray(dev.match_counts)), what
        else:
            assert np.array_equal(host.offsets, want[0]) and np.array_equal(host.docids, want[1]), what
            if mode == ALL:
                assert_close_scores(host.scores, want[2], what + ": pipelined vs device-resident")


# ============================================================================================== B. bench.py's call sequence
def knobs():
    """the chunk knobs a context created now reads (engine.cu trn_create)"""
    e = os.environ
    return dict(max_chunks=int(e.get("TRN_PIPELINE_CHUNKS", 8)), chunk_postings=int(e.get("TRN_CHUNK_POSTINGS", 10**9)),
                rule_sqrt=e.get("TRN_CHUNK_RULE") != "postings", taper=int(e.get("TRN_TAPER_CHUNKS", 1)) != 0,
                tail_ms=max(1.0, float(e.get("TRN_CHUNK_TAIL_US", 150))) / 1000.0, tail_tree_ms=max(1.0, float(e.get("TRN_CHUNK_TAIL_TREE_US", 900))) / 1000.0)


def chunk_plan(kn, nq, mode, est, leaves, hint):
    """chunkplan.h plan_chunks through trn_debug_chunk_plan, with the hint (bytes, postings, nq, mode) the previous host-buffer call left"""
    hb, hp, hnq, hmode = hint or (0, 0, 0, -1)
    sizes = np.zeros(32, np.uint32)
    n, single = C.c_uint32(), C.c_int()
    assert lib().trn_debug_chunk_plan(nq, int(mode == TOPK), est, leaves, kn["max_chunks"], kn["chunk_postings"], int(kn["rule_sqrt"]), int(kn["taper"]),
                                      kn["tail_ms"], kn["tail_tree_ms"], hb, hp, int(hnq == nq and hmode == mode),
                                      sizes.ctypes.data_as(C.c_void_p), 32, C.byref(n), C.byref(single)) == 0
    return bool(single.value), [int(x) for x in sizes[: n.value]]


def referenced(w, plans):
    """(referenced postings, TERM leaves) of a batch as trn_exec_batch counts them"""
    est = leaves = 0
    for p in plans:
        t = p["term"][(p["kind"] == tb.NODE_TERM) & (p["term"] < NTERMS)]
        est += int(w.df[t].sum())
        leaves += len(t)
    return est, leaves


def hint_of(res, mode, est):
    words = res.total_words if mode == COMPACT else int(res.offsets[-1])
    return (words * 4 * (2 if mode == ALL else 1), est, res.nq, mode)


def bench_sequence(w, g, texts, plans, label):
    """bench.py Job.run's calls, in its order, with a packed batch: every result checked, every host-buffer call's chunk count equal to the
    plan for the hint the call before it left.  Returns the plans of the host-buffer calls."""
    kn = knobs()
    est, leaves = referenced(w, plans)
    packed = g.pack(plans)
    sample = sample_of(NQ, 100, 12)
    want_routes, _ = tb.debug_plan(w.codec, w.index, w.terms, plans, DOCS, max_docid=w.ndocs)
    hint, plans_seen, dev_stream = None, [], None

    def host(mode, what):
        nonlocal hint
        single, sizes = chunk_plan(kn, NQ, mode, est, leaves, hint)
        res = g.exec_batch(plans, mode, K, copy=False, packed=packed)
        assert g.last_timings()["chunks"] == len(sizes), (label, what, sizes, g.last_timings()["chunks"])
        assert np.array_equal(g.last_routes(), want_routes), (label, what)
        check(w, texts, res, mode, K, f"{label} {what}", sample)
        plans_seen.append(sizes)
        hint = hint_of(res, mode, est)
        return res

    host(COMPACT, "warm-up 1")
    host(COMPACT, "warm-up 2")
    for i in range(3):
        g.exec_batch_device(plans, COMPACT, K, packed=packed)
        assert np.array_equal(g.last_routes(), want_routes), (label, "device", i)
    dev = fetch_view(g)
    check(w, texts, dev, COMPACT, K, f"{label} device-resident", sample)
    dev_stream = stream(dev)
    assert_same_stream(stream(host(COMPACT, "timed e2e")), dev_stream, f"{label} timed e2e")
    host(DOCS, "plain")
    assert_same_stream(stream(host(COMPACT, "parity")), dev_stream, f"{label} parity")
    return plans_seen


@pytest.mark.parametrize("wl", ["and2", "tree8", "and2l"])
def test_bench_sequence_session_knobs(worlds, ctx, wl):
    codec = bench.WORKLOADS[wl]["codec"]
    w, g = worlds(codec), ctx(codec)
    texts, plans = workload(w, wl)
    seen = bench_sequence(w, g, texts, plans, wl)
    assert all(len(s) > 1 for s in seen), seen  # TRN_CHUNK_POSTINGS=1: every host-buffer call is pipelined


@pytest.mark.parametrize("form", ["split", "taper"])
@pytest.mark.parametrize("wl", ["and2", "tree8", "and2l"])
def test_bench_sequence_production_planner(worlds, ctx, side_stream, monkeypatch, wl, form):
    """the default chunk planner: the first batch of a shape goes by referenced postings, the next one by the result size it left.  The
    launch tail is set so that the hint-driven rule gives c = floor(sqrt(D / 4 tail) + 1/2) = 3 chunks (then the taper: 5 launches) or one
    chunk tapered into 1/2, 1/4, 1/4 (D = the batch's result bytes at 45 GB/s)."""
    codec = bench.WORKLOADS[wl]["codec"]
    w = worlds(codec)
    texts, plans = workload(w, wl)
    est, leaves = referenced(w, plans)
    g0 = ctx(codec)  # the result size the first batch will leave (compact words do not depend on how the batch is chunked)
    g0.exec_batch_device(plans, COMPACT, K)
    hint_bytes = fetch_view(g0).total_words * 4
    D = hint_bytes / 45e6
    tail_us = D * 1000 / (40 if form == "split" else 4)
    monkeypatch.delenv("TRN_CHUNK_POSTINGS", raising=False)
    monkeypatch.delenv("TRN_CHUNK_RULE", raising=False)
    monkeypatch.setenv("TRN_CHUNK_TAIL_US", repr(tail_us))
    monkeypatch.setenv("TRN_CHUNK_TAIL_TREE_US", repr(tail_us))
    kn = knobs()
    assert kn["rule_sqrt"] and kn["chunk_postings"] == 10**9 and tail_us >= 1
    # the plan of the second batch of the shape, from the hint the first leaves
    single, sizes = chunk_plan(kn, NQ, COMPACT, est, leaves, (hint_bytes, est, NQ, COMPACT))
    if form == "split":
        assert not single and len(sizes) == 5 and sizes[:2] == [334, 334], sizes
    else:
        assert not single and sizes == [500, 250, 250], sizes
    g = new_source(w, side_stream)
    try:
        seen = bench_sequence(w, g, texts, plans, f"{wl} {form}")
    finally:
        g.close()
    assert seen[1] == sizes and seen[2] == sizes, seen  # warm-up 2 and the timed call: the hint-driven plan


# ============================================================================================== C. one context across changing calls
def mixed_texts(codec, n, offset=0):
    """GOOGLE: and2 and tree8 queries alternating; LUCENE: and2l queries with one or10 query in 50"""
    if codec == G:
        a, b = bench.gen_queries("and2", NQ, NTERMS)[0], bench.gen_queries("tree8", NQ, NTERMS)[0]
        pool = [a[i] if i % 2 else b[i] for i in range(NQ)]
    else:
        a, b = bench.gen_queries("and2l", NQ, NTERMS)[0], bench.gen_queries("or10", NQ, NTERMS)[0]
        pool = [b[i] if i % 50 == 7 else a[i] for i in range(NQ)]
    return [pool[(offset + i) % NQ] for i in range(n)]


def run_both(w, g, texts, mode, k, what, nsample=40):
    """the batch through exec_batch_device + fetch(), then through exec_batch; both against the reference"""
    plans = w.plans(texts)
    # (the host-side planner plans for a source without LUCENE positions: a LUCENE phrase, last in its batch, is left out of it)
    n = len(texts) - (w.codec == L and texts[-1].startswith('"'))
    routes, _ = tb.debug_plan(w.codec, w.index, w.terms, plans[:n], DOCS if mode == COMPACT else mode, k=k, max_docid=w.ndocs)
    sample = sample_of(len(texts), nsample, len(texts) + mode)
    g.exec_batch_device(plans, mode, k)
    dev_routes = g.last_routes()
    assert len(dev_routes) == len(texts) and np.array_equal(dev_routes[:n], routes), what
    check(w, texts, g.fetch(), mode, k, what + " device", sample)
    check(w, texts, g.exec_batch(plans, mode, k), mode, k, what + " host", sample)
    assert np.array_equal(g.last_routes(), dev_routes), what


@pytest.mark.parametrize("codec", [G, L], ids=["google", "lucene"])
def test_sizes_and_modes_on_one_context(worlds, ctx, codec):
    w, g = worlds(codec), ctx(codec)
    steps = [(1, COMPACT, K, 0), (1000, TOPK, 512, 0), (3, TOPK, 1, 17), (200, DOCS, K, 300), (1000, ALL, K, 500)]
    for n, mode, k, off in steps:
        run_both(w, g, mixed_texts(codec, n, off), mode, k, f"codec {codec} {n} queries mode {mode} k {k}")
    # right after the largest batch: one whose every query matches nothing (terms the index does not hold)
    empty = [f"nosuch{i} AND t{1 + i % NTERMS:04d}" for i in range(NQ)]
    assert not w.counts_sums(empty)[0].any()
    run_both(w, g, empty, COMPACT, K, f"codec {codec} empty batch")
    # the same shape twice: the second batch's plan and buffers come from what the first left
    for i in range(2):
        run_both(w, g, mixed_texts(codec, NQ, 250), COMPACT, K, f"codec {codec} repeated shape #{i}")


@pytest.mark.parametrize("codec", [G, L], ids=["google", "lucene"])
def test_masks_replaced_between_batches(worlds, ctx, codec):
    w, g = worlds(codec), ctx(codec)
    texts = mixed_texts(codec, 64, 40)
    plans = w.plans(texts)
    rng = np.random.default_rng(3)
    pool = np.unique(np.concatenate([w.full(t, False)[0] for t in texts[:16]]))
    big = np.sort(rng.choice(pool, size=len(pool) // 4, replace=False)).astype(np.uint32)
    small = big[::7]
    larger = np.union1d(big, rng.integers(1, NDOCS + 1, 200_000).astype(np.uint32))
    larger = np.concatenate([larger, np.array([NDOCS + 1, NDOCS + 12345], np.uint32)])  # above max_docid: ignored
    for label, masked in (("mask", big), ("smaller mask", small), ("larger mask", larger), ("cleared", None)):
        g.set_masked_documents(masked)
        want = [w.ref.exec_masked(t, False, masked if masked is not None else np.zeros(0, np.uint32), int(w.counts_sums([t])[0][0]) + 1)[0]
                for t in texts]
        g.exec_batch_device(plans, COMPACT, K)
        dev = g.fetch()
        host = g.exec_batch(plans, DOCS)
        assert g.last_timings()["chunks"] > 1
        for q in range(len(texts)):
            assert_same_docs(dev.query(q)[0], want[q], f"codec {codec} {label} [{q}] device")
            assert_same_docs(host.query(q)[0], want[q], f"codec {codec} {label} [{q}] host")
    g.set_masked_documents(None)


def dense_bitmaps_match(w, g, what):
    off, _ = tb.debug_dense_terms(w.codec, w.index, w.terms)
    have = np.flatnonzero(off != tb.DENSE_NONE)
    assert g.info()["dense_terms"] == len(have), what
    if w.codec == G:
        assert len(have) >= 4, what
    for t in range(NTERMS):
        got = g.dense_bitmap(t)
        if t not in have:
            assert got is None, (what, t)
            continue
        base, words = got
        docs = w.ref.decode(t, int(w.df[t]))[0].astype(np.int64) - base
        assert docs.min() >= 0 and docs.max() < 32 * len(words), (what, t)
        want = np.zeros(len(words), np.uint32)
        np.bitwise_or.at(want, docs >> 5, (np.uint32(1) << (docs & 31).astype(np.uint32)))
        assert np.array_equal(words, want), (what, t)


def test_reupload_into_one_context(worlds, side_stream):
    """a mask set, then a smaller and a larger GOOGLE index, the LUCENE index with and without its hits, and GOOGLE again: each upload starts
    with no masked documents, its own dense bitmaps and (LUCENE) no positions until upload_hits"""
    first = worlds(G)
    g = new_source(first, side_stream)
    try:
        phrase = '"t0001 t0002"'
        for step, w in enumerate([worlds(G, 1_000_000, 7), worlds(G, 6_000_000, 9), worlds(L), worlds(L), first]):
            g.set_masked_documents(np.arange(1, min(NDOCS, w.ndocs) + 1, 3, dtype=np.uint32))  # a third of the documents of both indexes
            g.upload(w.codec, w.index, w.terms, w.ndocs)
            what = f"upload #{step} codec {w.codec} ndocs {w.ndocs}"
            assert g.info()["max_docid"] == w.ndocs, what
            if step == 2:
                g.upload_hits(w.index, w.hits)
            texts = mixed_texts(w.codec, 200, 100 * step)
            if step == 3:  # the same LUCENE index uploaded again, without its hits: phrases are refused, everything else runs
                with pytest.raises(tb.TrinityError, match="rc=-7"):
                    g.exec_batch(w.plans([phrase]), DOCS)
            else:
                texts.append(phrase)
            run_both(w, g, texts, COMPACT, K, what, nsample=len(texts))
            run_both(w, g, texts, TOPK, K, what, nsample=20)
            dense_bitmaps_match(w, g, what)
    finally:
        g.close()


def test_fetch_returns_the_last_batch(worlds, ctx):
    w, g = worlds(G), ctx(G)
    texts = mixed_texts(G, 300, 600)
    plans = w.plans(texts)
    sample = sample_of(len(texts), 30, 5)
    g.exec_batch_device(plans, COMPACT, K)
    routes = g.last_routes()
    first = stream(fetch_view(g))
    check(w, texts, g.fetch(), COMPACT, K, "fetch", sample)
    # calls that are not exec calls leave the last batch and its routes alone
    other = [lambda: g.intersect([[0], [1], [2]]),
             lambda: (g.percolator_register(w.plans(["t0001 AND t0002", "t0003"]), NTERMS), g.percolate([np.array([0, 1], np.uint32)])),
             lambda: g.decode_terms([5, 6])]
    for i, call in enumerate(other):
        call()
        assert np.array_equal(g.last_routes(), routes), i
        assert_same_stream(stream(fetch_view(g)), first, f"fetch after call {i}")
    check(w, texts, g.fetch(), COMPACT, K, "fetch again", sample)
    # exec_matches leaves nothing to fetch
    small = mixed_texts(G, 5, 3)
    g.exec_matches(w.plans(small))
    assert np.array_equal(g.last_routes(), tb.debug_plan(G, w.index, w.terms, w.plans(small), tb.MODE_MATCHED_TERMS, max_docid=NDOCS)[0])
    with pytest.raises(tb.TrinityError, match="rc=-4: no batch executed"):
        g.fetch()
    # a pipelined exec_batch leaves nothing to fetch either
    g.exec_batch_device(plans, COMPACT, K)
    g.exec_batch(plans, DOCS)
    assert g.last_timings()["chunks"] > 1
    assert len(g.last_routes()) == len(plans)
    with pytest.raises(tb.TrinityError, match="rc=-4: no batch executed"):
        g.fetch()
    # a single-call exec_batch is exec_batch_device + fetch: fetch() returns its result again
    for mode, k in ((DOCS, K), (TOPK, 7)):
        texts = mixed_texts(G, 40, 900)
        res = g.exec_batch(w.plans(texts), mode, k)
        assert g.last_timings()["chunks"] == 1
        again = g.fetch()
        assert np.array_equal(again.offsets, res.offsets) and np.array_equal(again.docids, res.docids), mode
        check(w, texts, again, mode, k, f"fetch after single-call mode {mode}", range(len(texts)))
