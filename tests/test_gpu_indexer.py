"""trn_index_documents on the device against the reference's SegmentIndexSession::commit() over the same documents: the index file (GOOGLE
byte for byte; LUCENE byte for byte against the host encoder over a numpy model of the inversion, and against the reference except the PFor
padding it leaves uninitialised), the term tuples, the field statistics, every other file of the written directory, and the queries the
reference answers over the directory this engine wrote."""
import numpy as np
import pytest

import trinity_b200 as tb
from idxutil import flat, host_build, model_postings, read_dir, ref_index, ref_index_flat, term_names, zipf_corpus
from trinity_b200.segments import SegmentCollection
from util import assert_close_scores, assert_same_docs, assert_topk_equal

pytestmark = pytest.mark.gpu
CODECS = pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])


@pytest.fixture(scope="module")
def gpu():
    g = tb.GpuIndexSource(0)
    yield g
    g.close()


def _same_but_padding(mine, theirs, what):
    assert mine.size == theirs.size, what
    diff = np.flatnonzero(mine != theirs)
    # the reference leaves the padding of the PFor byte container uninitialised (codecs.cpp:195): only there, and only zeros of ours
    assert np.all(mine[diff] == 0), f"{what} differs at non-padding bytes {diff[:10]}"


def _check(gpu, tmp_path, codec, docids, docs, nterms, positions=None):
    seg = gpu.index_documents(codec, docids, docs, nterms, positions)
    model = model_postings(docids, docs, nterms, positions)
    index, hits, terms = host_build(codec, model, nterms)
    assert np.array_equal(seg.terms, terms)
    assert np.array_equal(seg.index, index) and np.array_equal(seg.hits, hits)
    assert seg.field_statistics == {"sumTermHits": sum(len(d) for d in docs), "totalTerms": len(model), "sumTermsDocs": sum(len(d) for _, d, _, _ in model),
                                    "docsCnt": sum(len(d) > 0 for d in docs)}
    names = term_names(nterms)
    ref_index(codec, tmp_path / "r" / "3", names, docids, docs, positions)
    seg.write(tmp_path / "w" / "3", names)
    want, got = read_dir(tmp_path / "r" / "3"), read_dir(tmp_path / "w" / "3")
    assert sorted(want) == sorted(got)
    for f in want:
        if codec == tb.CODEC_LUCENE and f in ("index", "hits.data"):
            _same_but_padding(got[f], want[f], f)
        else:
            assert np.array_equal(got[f], want[f]), f
    return seg


def _shape(name):
    rng = np.random.default_rng(11)
    if name == "one-token":
        return [7], [np.array([0], np.uint32)], 1, None
    if name == "shuffled-docids":
        docs = [rng.integers(0, 50, size=rng.integers(1, 40)).astype(np.uint32) for _ in range(3000)]
        return rng.permutation(np.arange(1, 3001)), docs, 50, None
    if name == "shuffled-positions":
        docs = [rng.integers(0, 33, size=rng.integers(1, 60)).astype(np.uint32) for _ in range(500)]
        return rng.permutation(np.arange(100, 600)), docs, 33, [rng.permutation(np.arange(1, len(d) + 1)) for d in docs]
    if name == "shared-positions":
        docs = [rng.integers(0, 32, size=30).astype(np.uint32) for _ in range(200)]
        return np.arange(1, 201), docs, 32, [rng.integers(1, 6, size=30) for _ in docs]
    if name == "long-document":
        docs = [rng.integers(0, 4096, size=16383).astype(np.uint32), np.array([5, 5, 9], np.uint32)]
        return [2, 1], docs, 4096, None
    if name == "freq-65535":
        docs = [np.full(65535, 3, np.uint32), np.array([3, 1], np.uint32)]
        return [9, 4], docs, 5, [np.arange(65535) % 16383 + 1, np.array([1, 2])]
    if name == "empty-document":
        docs = [np.array([1, 2], np.uint32), np.zeros(0, np.uint32), np.array([2], np.uint32), np.zeros(0, np.uint32)]
        return [5, 3, 9, 1], docs, 4, None
    if name == "high-docids":
        docs = [rng.integers(0, 10, size=8).astype(np.uint32) for _ in range(64)]
        return np.r_[2**32 - 2, rng.choice(np.arange(2**31, 2**32 - 2), size=62, replace=False), 1].astype(np.uint32), docs, 10, None
    if name == "sparse-terms":
        docs = [rng.choice(100_000, size=20).astype(np.uint32) for _ in range(300)]
        return rng.permutation(np.arange(1, 301)), docs, 100_000, None
    raise KeyError(name)


@CODECS
@pytest.mark.parametrize("shape", ["one-token", "shuffled-docids", "shuffled-positions", "shared-positions", "long-document", "freq-65535", "empty-document",
                                   "high-docids", "sparse-terms"])
def test_device_index_equals_the_reference(gpu, tmp_path, codec, shape):
    docids, docs, nterms, positions = _shape(shape)
    _check(gpu, tmp_path, codec, docids, docs, nterms, positions)


@pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
def test_zipf_corpus(gpu, tmp_path, codec):
    """250 000 documents x 64 tokens = 1.6e7 keys: every radix pass runs over thousands of tiles; the reference indexes the same batch"""
    nterms = 4096
    docids, offs, tok = zipf_corpus(250_000, nterms, 64, 5)
    seg = gpu.index_documents_flat(codec, docids, offs, tok, nterms)
    names = term_names(nterms)
    ref_index_flat(codec, tmp_path / "r" / "1", names, docids, offs, tok)
    seg.write(tmp_path / "w" / "1", names)
    want, got = read_dir(tmp_path / "r" / "1"), read_dir(tmp_path / "w" / "1")
    assert sorted(want) == sorted(got)
    for f in want:
        if codec == tb.CODEC_LUCENE and f in ("index", "hits.data"):
            _same_but_padding(got[f], want[f], f)
        else:
            assert np.array_equal(got[f], want[f]), f
    # explicit positions i + 1 are the same call; so is the batch in another document order
    pos = (np.arange(len(tok), dtype=np.uint64) % np.uint64(64) + np.uint64(1)).astype(np.uint32)
    again = gpu.index_documents_flat(codec, docids, offs, tok, nterms, pos)
    assert np.array_equal(again.index, seg.index) and np.array_equal(again.hits, seg.hits) and np.array_equal(again.terms, seg.terms)
    assert again.sort_passes >= seg.sort_passes  # 14 position bits instead of 7
    perm = np.random.default_rng(1).permutation(len(docids))
    again = gpu.index_documents_flat(codec, docids[perm], offs, tok.reshape(-1, 64)[perm].ravel(), nterms)
    assert np.array_equal(again.index, seg.index) and np.array_equal(again.hits, seg.hits) and np.array_equal(again.terms, seg.terms)


def test_refusals_leave_the_context_usable(gpu):
    ok = lambda: gpu.index_documents(tb.CODEC_GOOGLE, [3, 1], [np.array([0, 1], np.uint32), np.array([1], np.uint32)], 2)
    first = ok()
    d2 = [np.array([0, 1], np.uint32), np.array([1], np.uint32)]
    cases = [
        ("docID 0", dict(docids=[3, 0], docs=d2, nterms=2)),
        ("given twice", dict(docids=[3, 3], docs=d2, nterms=2)),
        ("not below nterms", dict(docids=[3, 1], docs=[np.array([0, 2], np.uint32), np.array([1], np.uint32)], nterms=2)),
        ("below 16384", dict(docids=[3, 1], docs=d2, nterms=2, positions=[np.array([1, 16384]), np.array([1])])),
        ("position 0", dict(docids=[3, 1], docs=d2, nterms=2, positions=[np.array([1, 0]), np.array([1])])),
        ("below 16384", dict(docids=[3], docs=[np.zeros(16384, np.uint32)], nterms=2)),
        ("more than 65535 times", dict(docids=[3], docs=[np.zeros(65536, np.uint32)], nterms=2, positions=[np.arange(65536) % 16383 + 1])),
        ("2\\^24", dict(docids=[3, 1], docs=d2, nterms=2**24 + 1)),
    ]
    for what, kw in cases:
        with pytest.raises(tb.TrinityError, match=what):
            gpu.index_documents(tb.CODEC_GOOGLE, **kw)
        again = ok()
        assert np.array_equal(again.index, first.index) and np.array_equal(again.terms, first.terms)
    offs = np.array([0, 2, 1], np.uint64)
    with pytest.raises(tb.TrinityError, match="must ascend"):
        gpu.index_documents_flat(tb.CODEC_GOOGLE, [3, 1], offs, np.zeros(2, np.uint32), 2)
    with pytest.raises(tb.TrinityError, match="both indexed and erased"):
        first.write("/nonexistent/1", ["a", "b"], erased=[3])


def test_more_than_65535_distinct_terms_in_a_document(gpu):
    docs, pos = [np.arange(70_000, dtype=np.uint32)], [np.arange(70_000) % 16383 + 1]
    with pytest.raises(tb.TrinityError, match="distinct terms"):
        gpu.index_documents(tb.CODEC_GOOGLE, [1], docs, 70_000, positions=pos)
    docs[0][65_535:] = 0  # exactly 65 535 distinct terms
    assert gpu.index_documents(tb.CODEC_GOOGLE, [1], docs, 70_000, positions=pos).field_statistics["totalTerms"] == 65_535


QUERIES = ["t1 AND t2", "t3 OR t7 OR t9", "t1 AND (t2 OR t3) NOT t5", "t10", "(t1 AND t2) OR (t3 AND t4)", "missing AND t1", "\"t1 t2\"", "\"t2 t1\" AND t3", "(\"t1 t2\" OR t9) AND t3"]


def _exec_corpus(seed, lo, hi, n):
    rng = np.random.default_rng(seed)
    docs = [np.minimum(rng.zipf(1.3, size=rng.integers(5, 40)) - 1, 47).astype(np.uint32) for _ in range(n)]
    return rng.choice(np.arange(lo, hi, dtype=np.uint32), size=n, replace=False), docs


def test_written_segment_answers_like_the_reference(ref, gpu, tmp_path):
    """GOOGLE (phrases run on inline hits): the reference's SegmentIndexSource opens the directory this engine wrote"""
    docids, docs = _exec_corpus(2, 1, 60_000, 20_000)
    names = term_names(48)
    gpu.index_documents(tb.CODEC_GOOGLE, docids, docs, 48).write(tmp_path / "5", names)
    rseg = ref.segment_open(tmp_path / "5")
    col = SegmentCollection([tmp_path / "5"])
    for mode, scored in ((tb.MODE_DOCS_ONLY, False), (tb.MODE_SCORED_ALL, True)):
        (res,) = col.exec_batch(QUERIES, mode)
        for i, q in enumerate(QUERIES):
            wd, ws = rseg.exec(q, scored, 70_000)
            gd, gs = res.query(i)
            assert_same_docs(gd, wd, f"[{q}]")
            if scored:
                assert_close_scores(gs, ws, f"[{q}]")
    assert len(rseg.exec(QUERIES[6], False, 70_000)[0]) > 0  # the phrase has matches: positions are right
    (top,) = col.exec_batch(QUERIES, tb.MODE_SCORED_TOPK, k=10)
    for i, q in enumerate(QUERIES):
        wd, ws = rseg.exec(q, True, 70_000)
        assert_topk_equal(*top.query(i), wd, ws, 10, f"[{q}] top-10")


@CODECS
def test_device_written_generation_over_a_reference_written_one(ref, gpu, tmp_path, codec):
    """generation 2 (this engine) replaces some documents of generation 1 (the reference) and erases others"""
    names = term_names(48)
    d1, docs1 = _exec_corpus(3, 1, 50_000, 15_000)
    ref_index(codec, tmp_path / "1", names, d1, docs1)
    d2, docs2 = _exec_corpus(4, 40_000, 90_000, 15_000)
    replaced = np.intersect1d(d1, d2)
    erased = np.setdiff1d(d1[d1 < 20_000], d2)[::3]
    assert len(replaced) and len(erased)
    gpu.index_documents(codec, d2, docs2, 48).write(tmp_path / "2", names, replaced=replaced, erased=erased)
    col = SegmentCollection([tmp_path / "1", tmp_path / "2"])
    rcol = ref.collection_open([tmp_path / "1", tmp_path / "2"])
    qs = QUERIES[:6]
    for mode, scored in ((tb.MODE_DOCS_ONLY, False), (tb.MODE_SCORED_ALL, True)):
        res = col.exec_batch(qs, mode)
        for i, q in enumerate(qs):
            for s, (wd, ws) in enumerate(rcol.collection_exec(q, scored, 200_000)):
                gd, gs = res[s].query(i)
                assert_same_docs(gd, wd, f"[{q}] source {s}")
                if scored:
                    assert_close_scores(gs, ws, f"[{q}] source {s}")


def test_context_keeps_its_index_and_registry(gpu):
    docids, docs = _exec_corpus(6, 1, 5_000, 2_000)
    seg = gpu.index_documents(tb.CODEC_GOOGLE, docids, docs, 48)
    g = tb.GpuIndexSource(0)
    tdict = seg.upload(g, term_names(48))
    plans = [tb.parse_query("t1 AND t2", tdict)]
    g.percolator_register([tb.parse_query("t1 AND t2", tb.TermDictionary(term_names(48)))], 48)
    before = g.exec_batch(plans, tb.MODE_DOCS_ONLY).query(0)[0].copy()
    pbefore = g.percolate(docs[:50]).queries.copy()
    g.index_documents(tb.CODEC_LUCENE, docids, docs, 48)
    with pytest.raises(tb.TrinityError):
        g.index_documents(tb.CODEC_LUCENE, [0], docs[:1], 48)
    assert np.array_equal(g.exec_batch(plans, tb.MODE_DOCS_ONLY).query(0)[0], before)
    assert np.array_equal(g.percolate(docs[:50]).queries, pbefore)
    want = np.sort(np.array([d for d, x in zip(docids, docs) if 1 in x and 2 in x], np.uint32))
    assert np.array_equal(before, want)
    g.close()
