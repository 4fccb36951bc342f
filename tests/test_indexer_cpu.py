"""The host side of the indexer, without a GPU: trn_segment_write against the directories the reference's SegmentIndexSession::commit()
writes (every file byte for byte), and the order of the terms in the index file — commit()'s 32 buckets, with the GOOGLE encoder's skiplist
countdown carried from term to term — pinned by feeding a numpy model of the inversion through the host encoder."""
import numpy as np
import pytest

import trinity_b200 as tb
from idxutil import host_build, model_postings, read_dir, ref_index, term_names, term_order

CODECS = pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])


def _corpus(nterms, ndocs, seed, length=12):
    rng = np.random.default_rng(seed)
    docs = [rng.integers(0, nterms, size=length).astype(np.uint32) for _ in range(ndocs)]
    docs[0] = np.arange(nterms, dtype=np.uint32)[:16000]  # every term has a posting (up to the position limit)
    docids = rng.permutation(np.arange(1, ndocs + 1, dtype=np.uint32))
    return docids, docs


def _rewrite(path, out):
    """what tb.Segment read from `path`, written again by trn_segment_write into `out`"""
    seg = tb.Segment(path)
    files = read_dir(path)
    tb.segment_write(out, seg.codec, seg.index, files.get("hits.data"), seg.terms, seg.names, seg.field_statistics, seg.masked_documents)
    return files, read_dir(out)


def _assert_same_files(want, got, what):
    assert sorted(want) == sorted(got), f"{what}: files {sorted(got)} instead of {sorted(want)}"
    for f in want:
        assert np.array_equal(want[f], got[f]), f"{what}: {f} differs"


@CODECS
@pytest.mark.parametrize("nterms", [1, 63, 64, 65, 129, 5000])
def test_segment_writer_round_trip(tmp_path, codec, nterms):
    """both sides of the 64-term skiplist interval of terms.idx; no updated documents: no updated_documents.ids"""
    docids, docs = _corpus(nterms, 40, nterms)
    ref_index(codec, tmp_path / "7", term_names(nterms), docids, docs)
    want, got = _rewrite(tmp_path / "7", tmp_path / "w" / "7")
    assert "updated_documents.ids" not in want and "terms.idx" in want
    _assert_same_files(want, got, f"{nterms} terms")


@CODECS
def test_segment_writer_names(tmp_path, codec):
    """names sharing long prefixes, a 1-byte and a 64-byte name, bytes above 127 (terms_cmp compares unsigned)"""
    names = ["a", "z" * 64, "prefix" * 10, "prefix" * 10 + "a", "prefix" * 10 + "b", "prefix" * 9, "é", "ab", "abc", "b"]
    names += [f"shared-prefix-{i:05d}" for i in range(200)]
    docids, docs = _corpus(len(names), 30, 5)
    ref_index(codec, tmp_path / "1", names, docids, docs)
    want, got = _rewrite(tmp_path / "1", tmp_path / "w" / "1")
    _assert_same_files(want, got, "names")


@CODECS
@pytest.mark.parametrize("shape", ["one", "banks", "bloom"])
def test_segment_writer_updated_documents(tmp_path, codec, shape):
    """one update; updates over several 32 K-document banks (replaced and erased); more than 262 144 updates: the bloom filter form"""
    docids, docs = _corpus(40, 50, 9)
    docids = docids * 1000
    # (erased ids above the indexed ones, ascending: idxutil.ref_index_flat says why the reference is fed in docID order)
    if shape == "one":
        replaced, erased = [], [77_777]
    elif shape == "banks":
        replaced, erased = docids[:20].tolist(), np.r_[np.arange(60_003, 300_000, 997), 4_000_000_000].tolist()
    else:
        replaced, erased = docids[:3].tolist(), np.arange(100_001, 100_001 + 262_200).tolist()
    ref_index(codec, tmp_path / "2", term_names(40), docids, docs, replaced=replaced, erased=erased)
    want, got = _rewrite(tmp_path / "2", tmp_path / "w" / "2")
    assert "updated_documents.ids" in want
    assert len(tb.Segment(tmp_path / "w" / "2").masked_documents) == len(replaced) + len(erased)
    _assert_same_files(want, got, shape)


def test_term_order_and_countdown(tmp_path):
    """the model's postings through the host GOOGLE encoder, term after term in index order, are the reference's index file: the terms lie by
    (transient id & 31, id), within a term by docID, within a document by position, and the skiplist countdown carries across the terms.
    All 32 buckets are used, several terms have more than 8 blocks, nterms is not a multiple of 32."""
    nterms = 75
    rng = np.random.default_rng(3)
    ndocs = 1500
    docs = []
    for d in range(ndocs):
        common = rng.choice(40, size=24, replace=False)  # terms 0..39 are dense: ~900 documents = ~28 blocks each
        rare = rng.integers(40, nterms, size=3)
        docs.append(rng.permutation(np.r_[common, rare, common[:2]]).astype(np.uint32))
    docs[0] = np.r_[docs[0], np.arange(nterms)].astype(np.uint32)
    positions = [rng.permutation(np.arange(1, len(d) + 1)).astype(np.uint32) for d in docs]  # tokens arrive in shuffled position order
    positions[1][:] = 5  # every hit of a document at one position
    docids = rng.permutation(np.arange(10, 10 + ndocs, dtype=np.uint32))
    ref_index(tb.CODEC_GOOGLE, tmp_path / "4", term_names(nterms), docids, docs, positions)
    model = model_postings(docids, docs, nterms, positions)
    assert [t for t, *_ in model] == term_order(nterms).tolist()
    assert len({(t + 1) & 31 for t, *_ in model}) == 32 and sum(len(d) > 8 * 32 for _, d, _, _ in model) >= 8
    index, _, terms = host_build(tb.CODEC_GOOGLE, model, nterms)
    want = read_dir(tmp_path / "4")
    assert np.array_equal(index, want["index"])
    seg = tb.Segment(tmp_path / "4")
    by_name = {n: tuple(t) for n, t in zip(seg.names, seg.terms.tolist())}
    assert all(by_name[f"t{t}"] == tuple(terms[t].tolist()) for t in range(nterms))
    assert seg.field_statistics == {"sumTermHits": sum(len(d) for d in docs), "totalTerms": nterms, "sumTermsDocs": sum(len(d) for _, d, _, _ in model),
                                    "docsCnt": ndocs}


def test_segment_writer_refusals(tmp_path):
    from trinity_b200._ffi import TERM_DTYPE

    terms = np.array([(1, 0, 4), (1, 4, 4)], TERM_DTYPE)
    fs = {"sumTermHits": 2, "totalTerms": 2, "sumTermsDocs": 2, "docsCnt": 1}
    index = np.zeros(8, np.uint8)
    ok = lambda **k: tb.segment_write(**{**dict(path=tmp_path / "5", codec=0, index=index, hits=None, terms=terms, names=["a", "b"], field_statistics=fs), **k})
    for what, kw in (("generation", dict(path=tmp_path / "seg")), ("name has 1 .. 64", dict(names=["a", ""])), ("name has 1 .. 64", dict(names=["a", "b" * 65])),
                     ("same name", dict(names=["a", "a"])), ("updated twice", dict(updated_docids=[5, 9, 5])), ("bad arguments", dict(codec=2))):
        with pytest.raises(tb.TrinityError, match=what):
            ok(**kw)
    assert not (tmp_path / "5").exists()
    ok()
    seg = tb.Segment(tmp_path / "5")
    assert seg.names == ["a", "b"] and seg.field_statistics == fs
    # a term without documents is not in the dictionary
    terms["documents"][0] = 0
    ok(path=tmp_path / "6")
    assert tb.Segment(tmp_path / "6").names == ["b"]
