"""The default exec mode on the device (GpuIndexSource.exec_matches, TRN_MODE_MATCHED_TERMS) against the reference's exec_query with no
ExecFlags: docIDs, the terms of every match, their freqs and every hit's (pos, payload_len, payload), bit for bit, on both codecs."""
import os

import numpy as np
import pytest

import trinity_b200 as tb
from matchutil import assert_same_matches, doc_corpus, gpu_as_list, host_build, lists_from, payload_hits, ref_build
from test_frontend_cpu import EXTRA, OPTIONAL_QUERIES
from test_gpu_parity import TEMPLATES
from test_matched_terms_cpu import ROOT_NOT, MORE, SOME_DEFAULT, edge_lists
from test_phrase_cpu import QUERIES as PHRASE_QUERIES

pytestmark = pytest.mark.gpu
CODECS = [tb.CODEC_GOOGLE, tb.CODEC_LUCENE]
IDS = ["google", "lucene"]


class Side:
    def __init__(self, codec, lists, ndocs, names, hits=True):
        self.codec, self.ndocs, self.names = codec, ndocs, names
        self.index, self.hits, self.terms = host_build(codec, lists)
        self.ref = ref_build(codec, lists, names, ndocs)
        self.tdict = tb.TermDictionary(names)
        self.gpu = tb.GpuIndexSource(0)
        self.gpu.upload(codec, self.index, self.terms, ndocs)
        if codec == tb.CODEC_LUCENE and hits:
            self.gpu.upload_hits(self.index, self.hits)

    def check(self, cases, masked=()):
        plans = [tb.parse_query(q, self.tdict, min_match=m or None) for q, _, m in cases]
        res = self.gpu.exec_matches(plans)
        for i, (q, flags, m) in enumerate(cases):
            want = self.ref.exec(q, flags, m, masked)
            assert_same_matches(gpu_as_list(res, i), want, f"codec {self.codec} [{q}] min {m}")
        return res


CASES = ([(q, 0, 0) for q in TEMPLATES + EXTRA + ROOT_NOT + MORE] + [(q, 8, 0) for q in OPTIONAL_QUERIES] + [(q, 16, m) for q, m in SOME_DEFAULT]
         + [(q.replace("w", "t"), 0, 0) for q in PHRASE_QUERIES])


@pytest.fixture(scope="module", params=[(CODECS[0], (3, 30)), (CODECS[1], (3, 30)), (CODECS[0], (300, 300)), (CODECS[1], (300, 300))],
                ids=["google-short", "lucene-short", "google-300", "lucene-300"])
def text(request):
    codec, doclen = request.param
    rng = np.random.default_rng(23 + doclen[0])
    ndocs = 3000 if doclen[0] < 100 else 600
    lists, _ = doc_corpus(rng, ndocs, 10, doclen)
    return Side(codec, lists, ndocs, [f"t{i + 1}" for i in range(10)])


def test_queries_match_the_reference(text):
    text.check(CASES)
    routes = set(text.gpu.last_routes().tolist())
    if text.codec == tb.CODEC_GOOGLE:
        assert {tb.ROUTE_STEPS, tb.ROUTE_FLAT_AND, tb.ROUTE_FLAT_OR, tb.ROUTE_FLAT_TREE} <= routes, routes
    else:
        assert routes == {tb.ROUTE_STEPS}, routes


def test_candidate_route_matches_the_reference(text):
    if text.codec != tb.CODEC_GOOGLE:
        pytest.skip("the candidate-driven conjunction runs on GOOGLE sources")
    old = os.environ.get("TRN_CAND_COST")
    os.environ["TRN_CAND_COST"] = "1"
    try:
        g = tb.GpuIndexSource(0)
        g.upload(text.codec, text.index, text.terms, text.ndocs)
        qs = [("t3 AND t7", 0, 0), ("t1 AND (t2 OR t3) NOT t5", 0, 0), ("t9 AND t4 AND t2", 0, 0)]
        res = g.exec_matches([tb.parse_query(q, text.tdict) for q, _, _ in qs])
        assert set(g.last_routes().tolist()) == {tb.ROUTE_CANDIDATE}
        for i, (q, f, m) in enumerate(qs):
            assert_same_matches(gpu_as_list(res, i), text.ref.exec(q, f, m), f"candidate [{q}]")
    finally:
        if old is None:
            os.environ.pop("TRN_CAND_COST", None)
        else:
            os.environ["TRN_CAND_COST"] = old


def test_masked_documents(text):
    masked = list(range(2, text.ndocs, 7))
    text.gpu.set_masked_documents(masked)
    try:
        text.check([("t1 OR t2", 0, 0), ("t1 AND t3", 0, 0), ('"t1 t2"', 0, 0), ("t4", 0, 0)], masked=masked)
    finally:
        text.gpu.set_masked_documents(None)


@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_layout_edges_and_long_documents(codec):
    """full LUCENE hit blocks, runs across blocks into the tail, freq-0 documents, every payload size, documents with 17 000 hits"""
    rng = np.random.default_rng(31)
    lists = edge_lists(rng)
    per = {int(d): [1 + i // 3 for i in range(17000)] for d in (7, 400, 4000)}  # positions stay <= 8192
    per2 = {int(d): [1 + i // 2 for i in range(600)] for d in range(1, 4000, 37)}
    big, _ = lists_from(rng, [per, per2])
    lists += big
    names = [f"e{i + 1}" for i in range(len(lists))]
    s = Side(codec, lists, 5000, names)
    cases = [(n, 0, 0) for n in names] + [("e1 OR e2 OR e3", 0, 0), ("e4 AND e6", 0, 0), ("e7 OR e6 OR e1", 0, 0), ("e2 NOT e3", 0, 0)]
    res = s.check(cases)
    assert res.hits.size > 3 * 17000
    if codec == tb.CODEC_LUCENE:
        assert any((l[1] == 0).any() for l in lists)


def test_chunked_collect_pass_is_identical():
    """a small TRN_MATCH_CHUNK splits the collect pass into many chunks; the result is the same"""
    rng = np.random.default_rng(3)
    lists, _ = doc_corpus(rng, 2000, 8)
    names = [f"t{i + 1}" for i in range(8)]
    a = Side(tb.CODEC_LUCENE, lists, 2000, names)
    os.environ["TRN_MATCH_CHUNK"] = "97"
    try:
        b = Side(tb.CODEC_LUCENE, lists, 2000, names)
    finally:
        os.environ.pop("TRN_MATCH_CHUNK")
    plans = [tb.parse_query(q, a.tdict) for q in ("t1 OR t2 OR t3", "t4 AND t5", '"t1 t2"')]
    ra, rb = a.gpu.exec_matches(plans), b.gpu.exec_matches(plans)
    assert ra.chunks == 1 and rb.chunks > 10
    for f in ("doc_offsets", "docids", "term_offsets", "terms", "freqs", "hit_offsets"):
        assert np.array_equal(getattr(ra, f), getattr(rb, f)), f
    for f in ("payload", "pos", "payload_len"):
        assert np.array_equal(ra.hits[f], rb.hits[f]), f
    for i, q in enumerate(("t1 OR t2 OR t3", "t4 AND t5", '"t1 t2"')):
        assert_same_matches(gpu_as_list(rb, i), b.ref.exec(q), q)


@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_32_distinct_terms_and_33_refused(codec):
    rng = np.random.default_rng(4)
    per = [{int(d): [1, 2 + int(d) % 5] for d in rng.choice(np.arange(1, 800), size=60, replace=False)} for _ in range(33)]
    lists, _ = lists_from(rng, per)
    names = [f"m{i}" for i in range(33)]
    s = Side(codec, lists, 800, names)
    q32 = " OR ".join(names[:32])
    s.check([(q32, 0, 0)])
    with pytest.raises(tb.TrinityError, match="32 distinct terms"):
        s.gpu.exec_matches([tb.parse_query(" OR ".join(names), s.tdict)])


def test_lucene_without_hits_is_refused():
    rng = np.random.default_rng(6)
    lists, _ = doc_corpus(rng, 200, 4)
    s = Side(tb.CODEC_LUCENE, lists, 200, [f"t{i + 1}" for i in range(4)], hits=False)
    with pytest.raises(tb.TrinityError, match="hits"):
        s.gpu.exec_matches([tb.parse_query("t1 OR t2", s.tdict)])


@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_device_encoded_index(codec):
    """an index the device encoders built (no payloads) runs in this mode like the host-built one"""
    rng = np.random.default_rng(8)
    lists, _ = doc_corpus(rng, 1500, 6)
    lists = [(d, f, p, np.zeros_like(sz), np.zeros_like(pv)) for d, f, p, sz, pv in lists]
    names = [f"t{i + 1}" for i in range(6)]
    s = Side(codec, lists, 1500, names)
    g = tb.GpuIndexSource(0)
    post = [(d, f, p) for d, f, p, *_ in lists]
    if codec == tb.CODEC_GOOGLE:
        index, terms, _, _ = g.encode_google(post)
        hits = None
    else:
        index, hits, terms, _ = g.encode_lucene(post)
    assert np.array_equal(terms, s.terms)
    g.upload(codec, index, terms, 1500)
    if hits is not None:
        g.upload_hits(index, hits)
    qs = ["t1 OR t2", "t1 AND t3", '"t1 t2"', "(t2 OR t3) NOT t1"]
    res = g.exec_matches([tb.parse_query(q, s.tdict) for q in qs])
    for i, q in enumerate(qs):
        assert_same_matches(gpu_as_list(res, i), s.ref.exec(q), f"device-encoded [{q}]")


@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_top_of_the_docid_space_by_translation(codec):
    """the corpus of test_gpu_docid_limits, with payloads, indexed as is for the reference and shifted by DELTA for the device (its largest
    docID is 2^32 - 2, the top 2^13 / 2^14 / 2^17 tiles are populated): every match must be the reference's on the unshifted index plus
    DELTA, terms, freqs and hits bit for bit, with a masked document in the top tile and a root filter over a disjunction"""
    from test_gpu_docid_limits import DELTA, DOCS, LISTS, NAMES, TOP, _positions
    rng = np.random.default_rng(17)
    lists, shifted = [], []
    for n in NAMES:
        d, f = LISTS[n]
        p = _positions(n, f)
        pos = p if p is not None else np.concatenate([np.arange(1, int(x) + 1, dtype=np.uint32) for x in f])
        sz, pv = payload_hits(rng, len(pos))
        lists.append((d, f, pos, sz, pv))
        shifted.append((d + np.uint32(DELTA), f, pos, sz, pv))
    ref = ref_build(codec, lists, NAMES, int(LISTS["dense"][0][-1]))
    index, hits, terms = host_build(codec, shifted)
    g = tb.GpuIndexSource(0)
    g.upload(codec, index, terms, TOP)
    if codec == tb.CODEC_LUCENE:
        g.upload_hits(index, hits)
    tdict = tb.TermDictionary(NAMES)
    top = LISTS["top"][0]
    masked = [int(top[-2]), int(top[-7]), int(LISTS["edge"][0][-2])]  # documents of the top tile, unshifted (2^32 - 2 itself stays)
    g.set_masked_documents([m + DELTA for m in masked])
    qs = list(DOCS) + ["(dense OR mid) NOT edge", "(top OR edge) NOT heavy"]
    res = g.exec_matches([tb.parse_query(q, tdict) for q in qs])
    routes = g.last_routes()
    for i, q in enumerate(qs):
        want = [(d + DELTA, ts) for d, ts in ref.exec(q, masked=masked)]
        assert_same_matches(gpu_as_list(res, i), want, f"codec {codec} top of the docID space [{q}]")
        if i < len(DOCS):
            assert routes[i] == (DOCS[q] if codec == tb.CODEC_GOOGLE else tb.ROUTE_STEPS), (q, routes[i])
        else:  # a root filter over a disjunction runs as the whole filter (DocumentsOnly would run the bare disjunction)
            assert routes[i] != tb.ROUTE_FLAT_OR, (q, routes[i])
    assert int(res.docids.max()) == TOP and not np.isin(np.asarray(masked, np.uint64) + DELTA, res.docids).any()


def test_fetch_results_after_exec_matches_is_refused():
    """the docs pass leaves no trn_result behind: trn_fetch_results has nothing to fetch after trn_exec_matches"""
    rng = np.random.default_rng(9)
    lists, _ = doc_corpus(rng, 300, 4)
    s = Side(tb.CODEC_GOOGLE, lists, 300, [f"t{i + 1}" for i in range(4)])
    s.gpu.exec_matches([tb.parse_query("t1 OR t2", s.tdict)])
    with pytest.raises(tb.TrinityError, match="no batch executed"):
        s.gpu.fetch()
