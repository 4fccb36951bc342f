"""Hits with payloads written on the device: trn_encode_google_payloads / trn_encode_lucene_payloads against the reference Encoders and
the host encoder (GOOGLE byte for byte; LUCENE byte for byte against the host, and against the reference except its uninitialised PFor
padding), the same bytes as the payload-free entry points when every size is 0, trn_index_documents_payloads against the reference's
SegmentIndexSession::commit() file for file with its field statistics, the default exec mode over the device-written bytes against the
reference's over its own, and the refusals, each followed by a good call on the same context."""
import numpy as np
import pytest

import trinity_b200 as tb
from idxutil import flat, read_dir, term_names, zipf_corpus
from matchutil import assert_same_matches, doc_corpus, gpu_as_list, host_build, ref_build
from payutil import google_shapes, lucene_shapes, model_postings_payloads, ref_index_payloads, zipf_payloads

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
    # the reference leaves the padding of the PFor byte container uninitialised (fastpfor.h:196-198): only there, and only zeros of ours
    assert np.all(mine[diff] == 0), f"{what} differs at non-padding bytes {diff[:10]}"


def _encode(gpu, codec, lists):
    if codec == tb.CODEC_GOOGLE:
        index, terms, _, _ = gpu.encode_google(lists)
        return index, np.zeros(0, np.uint8), terms
    index, hits, terms, _ = gpu.encode_lucene(lists)
    return index, hits, terms


@CODECS
def test_device_encoder_equals_the_reference_and_host_encoders(gpu, codec):
    shapes = (google_shapes if codec == tb.CODEC_GOOGLE else lucene_shapes)(np.random.default_rng(41))
    lists, names = [l for _, l in shapes], [n for n, _ in shapes]
    index, hits, terms = _encode(gpu, codec, lists)
    hindex, hhits, hterms = host_build(codec, lists)
    assert np.array_equal(terms, hterms)
    assert np.array_equal(index, hindex), f"first differing byte at {int(np.flatnonzero(index != hindex)[0]) if index.size == hindex.size else 'size'}"
    assert np.array_equal(hits, hhits)
    r = ref_build(codec, lists, names, int(max(int(l[0].max()) for l in lists if len(l[0]))))
    assert np.array_equal(terms, r.terms())
    if codec == tb.CODEC_GOOGLE:
        assert np.array_equal(index, r.index())
    else:
        _same_but_padding(index, r.index(), "index")
        _same_but_padding(hits, r.hits(), "hits.data")


@CODECS
def test_all_sizes_zero_writes_the_payload_free_bytes(gpu, codec):
    shapes = (google_shapes if codec == tb.CODEC_GOOGLE else lucene_shapes)(np.random.default_rng(8))
    with_pay = [(d, f, p, np.zeros_like(sz), v) for _, (d, f, p, sz, v) in shapes if not (len(p) and (p == 0).any())]
    without = [(d, f, p) for d, f, p, _, _ in with_pay]
    a, b = _encode(gpu, codec, with_pay), _encode(gpu, codec, without)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def _index_check(gpu, tmp_path, codec, docids, offs, tok, pos, plens, pays, nterms):
    seg = gpu.index_documents_flat(codec, docids, offs, tok, nterms, pos, plens, pays)
    model = model_postings_payloads(docids, offs, tok, pos, plens, pays, nterms)
    index, hits, tarr = host_build(codec, [l for _, l in model])
    terms = np.zeros(nterms, tb.TERM_DTYPE)
    for k, (t, _) in enumerate(model):
        terms[t] = tarr[k]
    assert np.array_equal(seg.terms, terms)
    assert np.array_equal(seg.index, index) and np.array_equal(seg.hits, hits)
    names = term_names(nterms)
    ref_index_payloads(codec, tmp_path / "r" / "4", names, docids, offs, tok, pos, plens, pays)
    seg.write(tmp_path / "w" / "4", names)
    want, got = read_dir(tmp_path / "r" / "4"), read_dir(tmp_path / "w" / "4")
    assert sorted(want) == sorted(got)
    for f in want:
        if codec == tb.CODEC_LUCENE and f in ("index", "hits.data"):
            _same_but_padding(got[f], want[f], f)
        else:
            assert np.array_equal(got[f], want[f]), f
    from refharness import load_ref
    assert seg.field_statistics == load_ref().segment_open(tmp_path / "r" / "4").field_stats()
    return seg, model


def _index_shape(name):
    rng = np.random.default_rng(17)
    if name == "shuffled-docids":
        docs = [rng.integers(0, 50, size=rng.integers(1, 40)).astype(np.uint32) for _ in range(3000)]
        docids, pos = rng.permutation(np.arange(1, 3001)), None
    elif name == "shuffled-positions":
        docs = [rng.integers(0, 33, size=rng.integers(1, 60)).astype(np.uint32) for _ in range(500)]
        docids, pos = rng.permutation(np.arange(100, 600)), [rng.permutation(np.arange(1, len(d) + 1)) for d in docs]
    elif name == "long-document":
        docs = [rng.integers(0, 4096, size=16383).astype(np.uint32), np.array([5, 5, 9], np.uint32)]
        docids, pos = [2, 1], None
    elif name == "equal-positions":  # duplicate (term, position) pairs with equal payloads
        docs = [rng.integers(0, 8, size=30).astype(np.uint32) for _ in range(200)]
        docids, pos = np.arange(1, 201), [rng.integers(1, 6, size=30) for _ in docs]
    elif name == "position-0":
        docs = [rng.integers(0, 20, size=12).astype(np.uint32) for _ in range(300)]
        docids, pos = rng.permutation(np.arange(1, 301)), [np.r_[0, 0, np.arange(1, 11)] for _ in docs]
    else:
        raise KeyError(name)
    offs, tok = flat(docs)
    p = None if pos is None else flat(pos)[1]
    plens, pays = zipf_payloads(rng, len(tok))
    if p is not None:
        plens[p == 0] = np.maximum(plens[p == 0], 1)
        # tokens that share (document, term, position) share a payload: the reference leaves their order undefined otherwise
        doc = np.repeat(np.arange(len(docs)), np.diff(offs).astype(np.int64))
        key = (doc.astype(np.int64) << 40) | (tok.astype(np.int64) << 16) | p.astype(np.int64)
        _, first = np.unique(key, return_inverse=True)
        rep = np.zeros(first.max() + 1, np.int64)
        rep[first[::-1]] = np.arange(len(key))[::-1]
        plens, pays = plens[rep[first]], pays[rep[first]]
    return np.asarray(docids, np.uint32), offs, tok, p, plens, pays, int(tok.max()) + 1


@CODECS
@pytest.mark.parametrize("shape", ["shuffled-docids", "shuffled-positions", "long-document", "equal-positions", "position-0"])
def test_device_index_with_payloads_equals_the_reference(gpu, tmp_path, codec, shape):
    _index_check(gpu, tmp_path, codec, *_index_shape(shape))


@CODECS
def test_zipf_corpus_with_payloads(gpu, tmp_path, codec):
    nterms = 2048
    docids, offs, tok = zipf_corpus(40_000, nterms, 48, 9)
    plens, pays = zipf_payloads(np.random.default_rng(3), len(tok))
    _index_check(gpu, tmp_path, codec, docids, offs, tok, None, plens, pays, nterms)


@CODECS
def test_device_written_payloads_read_back_like_the_reference(gpu, codec):
    rng = np.random.default_rng(71)
    lists, _ = doc_corpus(rng, 2000, 8, (3, 200))
    names = [f"t{i + 1}" for i in range(8)]
    index, hits, terms = _encode(gpu, codec, lists)
    r = ref_build(codec, lists, names, 2000)
    g = tb.GpuIndexSource(0)
    g.upload(codec, index, terms, 2000)
    if codec == tb.CODEC_LUCENE:
        g.upload_hits(index, hits)
    td = tb.TermDictionary(names)
    qs = ["t1", "t2 AND t3", "t1 OR t4 OR t8", '"t1 t2"', "t5 NOT t6"]
    res = g.exec_matches([tb.parse_query(q, td) for q in qs])
    for i, q in enumerate(qs):
        assert_same_matches(gpu_as_list(res, i), r.exec(q), f"codec {codec} [{q}]")
    g.close()


def test_refusals_leave_the_context_usable(gpu):
    d, f = np.array([3, 9], np.uint32), np.array([2, 1], np.uint32)
    p = np.array([4, 7, 2], np.uint32)
    good = [(d, f, p, np.array([1, 2, 0], np.uint8), np.arange(3, dtype=np.uint64))]
    for codec in (tb.CODEC_GOOGLE, tb.CODEC_LUCENE):
        with pytest.raises(tb.TrinityError, match="rc=-1"):  # a 9-byte payload
            _encode(gpu, codec, [(d, f, p, np.array([1, 9, 0], np.uint8), np.zeros(3, np.uint64))])
        with pytest.raises(tb.TrinityError, match="rc=-1"):  # position 0 without a payload
            _encode(gpu, codec, [(d, f, np.array([0, 7, 2], np.uint32), np.array([0, 2, 0], np.uint8), np.zeros(3, np.uint64))])
        assert _encode(gpu, codec, good)[0].size
    docids, offs = np.array([5, 8], np.uint64).astype(np.uint32), np.array([0, 3, 5], np.uint64)
    tok, pos = np.array([0, 1, 0, 1, 1], np.uint32), np.array([1, 2, 3, 1, 1], np.uint32)
    for codec in (tb.CODEC_GOOGLE, tb.CODEC_LUCENE):
        with pytest.raises(tb.TrinityError, match="rc=-1.*at most 8"):
            gpu.index_documents_flat(codec, docids, offs, tok, 2, pos, np.array([0, 9, 0, 0, 0], np.uint8), np.zeros(5, np.uint64))
        # docID 8 holds term 1 twice at position 1, with different payloads
        with pytest.raises(tb.TrinityError, match=r"rc=-7.*docID 8 holds term 1 twice at position 1"):
            gpu.index_documents_flat(codec, docids, offs, tok, 2, pos, np.array([0, 0, 0, 2, 2], np.uint8), np.array([0, 0, 0, 7, 8], np.uint64))
        with pytest.raises(tb.TrinityError, match="rc=-7.*position 0 and no payload"):
            gpu.index_documents_flat(codec, docids, offs, tok, 2, np.array([1, 0, 3, 1, 2], np.uint32), np.zeros(5, np.uint8), np.zeros(5, np.uint64))
        # equal payloads at an equal position, and position 0 with a payload, are indexed
        seg = gpu.index_documents_flat(codec, docids, offs, tok, 2, pos, np.array([0, 0, 0, 2, 2], np.uint8), np.array([0, 0, 0, 7, 7], np.uint64))
        assert seg.field_statistics["sumTermHits"] == 5
        seg = gpu.index_documents_flat(codec, docids, offs, tok, 2, np.array([1, 0, 3, 1, 2], np.uint32), np.array([0, 1, 0, 0, 0], np.uint8),
                                       np.ones(5, np.uint64))
        assert seg.field_statistics["sumTermHits"] == 5


@CODECS
def test_merge_by_append_keeps_device_written_payloads(gpu, tmp_path, codec):
    """a generation written by trn_index_documents_payloads, merged alone into its own codec: every term is appended, and the merged
    directory (payload chunks included) equals the reference's merge of the same directory"""
    from mergeutil import ref_merge
    from trinity_b200.segments import SegmentCollection

    docids, offs, tok, pos, plens, pays, nterms = _index_shape("position-0")
    seg = gpu.index_documents_flat(codec, docids, offs, tok, nterms, pos, plens, pays)
    src = tmp_path / "src" / "1"
    seg.write(src, term_names(nterms))
    m = SegmentCollection([src]).merge(codec)
    assert m.counts["reencoded"] == 0 and m.counts["appended"] == int((seg.terms["documents"] > 0).sum())
    ref_fs, _ = ref_merge(codec, tmp_path / "ref" / "100", [src], False, m.field_statistics["docsCnt"])
    assert m.field_statistics == ref_fs
    m.write(tmp_path / "dev" / "100")
    want, got = read_dir(tmp_path / "ref" / "100"), read_dir(tmp_path / "dev" / "100")
    assert sorted(want) == sorted(got)
    for f in want:
        if codec == tb.CODEC_LUCENE and f in ("index", "hits.data"):
            _same_but_padding(got[f], want[f], f)
        else:
            assert np.array_equal(got[f], want[f]), f
    # the payload bytes travel as they were written: the merged hits.data (LUCENE) is the source's, chunk for chunk
    if codec == tb.CODEC_LUCENE:
        assert got["hits.data"].size == seg.hits.size
