"""trn_index_documents across the bit boundaries of its sort keys, on both sides: the key is term_order << 40 | doc_rank << 14 | position
and the documents sort by docID first, and the radix passes cover only the bits that can be non-zero.  Each case is compared byte for byte
with the host encoder over a numpy model of the inversion (and with the reference's SegmentIndexSession where the shape is small), and
asserts the number of sort passes a restatement of plan_radix_passes gives."""
import numpy as np
import pytest

import trinity_b200 as tb
from idxutil import host_build, model_postings, term_order
from test_gpu_indexer import _check

pytestmark = pytest.mark.gpu
CODECS = pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
MAX_TERMS, MAX_DOCS = 1 << 24, 1 << 26  # kIndexMaxTerms, kIndexMaxDocs


@pytest.fixture(scope="module")
def gpu():
    g = tb.GpuIndexSource(0)
    yield g
    g.close()


def low_bits_for(v):
    return (1 << int(v).bit_length()) - 1


def radix_passes(active):
    """plan_radix_passes: groups of up to 8 bits that start and end at an active bit"""
    n, b = 0, 0
    while b < 64:
        if not (active >> b) & 1:
            b += 1
            continue
        bits = min(8, 64 - b)
        while bits > 1 and not (active >> (b + bits - 1)) & 1:
            bits -= 1
        n += 1
        b += bits
    return n


def sort_passes(docids, nterms, maxlen, positions):
    ndocs = len(docids)
    doc_active = low_bits_for(ndocs - 1) | (low_bits_for(int(np.max(docids))) << 32)
    key_active = low_bits_for(16383 if positions else maxlen) | (low_bits_for(ndocs - 1) << 14) | (low_bits_for(nterms - 1) << 40)
    return radix_passes(doc_active) + radix_passes(key_active)


def corpus(nterms, ndocs, maxlen, positions, seed):
    """ndocs documents, one of maxlen tokens over a few terms (so a term repeats at positions on both sides of every power of two), the
    others of 1 .. 3 tokens; term ids 0 and nterms - 1 occur; half the docIDs have bit 31 set"""
    rng = np.random.default_rng(seed)
    docids = (rng.choice(2**32 - 2, size=ndocs, replace=False) + 1).astype(np.uint32)
    if ndocs > 1:
        docids[0] = 2**32 - 1 if seed % 2 else 2**31
        docids[1] = 1
    lens = rng.integers(1, min(maxlen, 3) + 1, ndocs)
    lens[rng.integers(ndocs)] = maxlen
    docs = [rng.integers(0, nterms, L).astype(np.uint32) for L in lens]
    big = docs[int(np.argmax(lens))]
    few = np.array([0, nterms - 1, nterms // 2, min(nterms - 1, 7)], np.uint32)
    big[:] = few[rng.integers(0, 4, len(big))]
    if ndocs > 1:
        docs[int(np.argmin(lens))][0] = nterms - 1
    pos = None
    if positions:
        pos = [rng.permutation(np.arange(1, 16384))[:L].astype(np.uint32) if L > 3 else rng.integers(1, 16384, L).astype(np.uint32) for L in lens]
        pos[int(np.argmax(lens))][-1] = 16383
    return docids, docs, pos


SWEEP = ([("nterms", v) for v in (1, 2, 256, 257, 65535, 65536, 65537)] + [("ndocs", v) for v in (1, 2, 256, 257, 65537)]
         + [("maxlen", v) for v in (1, 2, 255, 256, 257, 16383)])


@CODECS
@pytest.mark.parametrize("positions", [False, True], ids=["implied", "given"])
@pytest.mark.parametrize("field,value", SWEEP, ids=[f"{f}-{v}" for f, v in SWEEP])
def test_key_field_boundaries(gpu, tmp_path, codec, positions, field, value):
    shape = {"nterms": 257, "ndocs": 257, "maxlen": 257}
    shape[field] = value
    docids, docs, pos = corpus(shape["nterms"], shape["ndocs"], shape["maxlen"], positions, seed=value + 7 * positions)
    nterms = shape["nterms"]
    if shape["ndocs"] <= 257 and nterms <= 257:
        seg = _check(gpu, tmp_path, codec, docids, docs, nterms, pos)  # and the reference's directory
    else:
        seg = gpu.index_documents(codec, docids, docs, nterms, pos)
        index, hits, terms = host_build(codec, model_postings(docids, docs, nterms, pos), nterms)
        assert np.array_equal(seg.index, index) and np.array_equal(seg.hits, hits) and np.array_equal(seg.terms, terms)
        assert seg.field_statistics["sumTermHits"] == sum(len(d) for d in docs)
    assert seg.sort_passes == sort_passes(docids, nterms, max(len(d) for d in docs), positions)


@CODECS
def test_all_term_order_bits(gpu, codec):
    """nterms = 2^24: term_order fills key bits 40 .. 63; a few hundred present terms across the whole id range, 2^24 - 1 included.  One
    term more is refused."""
    rng = np.random.default_rng(31)
    ids = np.unique(np.r_[rng.choice(MAX_TERMS, 400, replace=False), 0, 1, 31, 32, MAX_TERMS - 32, MAX_TERMS - 2, MAX_TERMS - 1]).astype(np.uint32)
    ndocs = 3000
    docids = (rng.choice(2**32 - 2, size=ndocs, replace=False) + 1).astype(np.uint32)
    docs = [ids[rng.integers(0, len(ids), rng.integers(1, 12))] for _ in range(ndocs)]
    docs[5] = ids[::-1].copy()  # every present term
    seg = gpu.index_documents(codec, docids, docs, MAX_TERMS)
    index, hits, terms = host_build(codec, model_postings(docids, docs, MAX_TERMS), MAX_TERMS)
    assert np.array_equal(seg.index, index) and np.array_equal(seg.hits, hits) and np.array_equal(seg.terms, terms)
    assert np.array_equal(np.flatnonzero(seg.terms["documents"]), ids)
    assert sort_passes(docids, MAX_TERMS, len(ids), False) == seg.sort_passes
    place = np.empty(MAX_TERMS, np.int64)
    place[term_order(MAX_TERMS)] = np.arange(MAX_TERMS)
    assert int(place[ids].max()) << 40 >> 63 == 1  # a present term's key sets bit 63
    with pytest.raises(tb.TrinityError, match="2\\^24"):
        gpu.index_documents(codec, docids[:2], docs[:2], MAX_TERMS + 1)


def test_all_doc_rank_bits(gpu):
    """ndocs = 2^26 (doc_rank fills key bits 14 .. 39), one or two tokens each, against a closed-form model; one document more is
    refused"""
    n, nterms = MAX_DOCS, 5
    i = np.arange(n, dtype=np.uint64)
    docids = ((i * np.uint64(0x9E3779B1)) % np.uint64(n) + np.uint64(1)).astype(np.uint32)  # a permutation of 1 .. 2^26
    two = (i % np.uint64(3)) == 0
    lens = np.where(two, 2, 1).astype(np.uint64)
    offs = np.zeros(n + 1, np.uint64)
    np.cumsum(lens, out=offs[1:])
    t0 = (i % np.uint64(nterms)).astype(np.uint32)
    t1 = ((i // np.uint64(3)) % np.uint64(4)).astype(np.uint32)
    tok = np.empty(int(offs[-1]), np.uint32)
    start = offs[:-1].astype(np.int64)
    tok[start] = t0
    tok[start[two] + 1] = t1[two]
    del i
    seg = gpu.index_documents_flat(tb.CODEC_GOOGLE, docids, offs, tok, nterms)
    assert seg.sort_passes == sort_passes(docids, nterms, 2, False)
    assert seg.field_statistics["docsCnt"] == n and seg.field_statistics["sumTermHits"] == len(tok)
    # the model: per term, its documents ascending with their freqs and positions
    model = []
    order = np.argsort(docids)  # by docID
    t0, t1, two, docids = t0[order], t1[order], two[order], docids[order]
    for t in term_order(nterms):
        a, b = t0 == t, two & (t1 == t)
        f = a.astype(np.uint32) + b.astype(np.uint32)
        keep = f > 0
        d = docids[keep]
        f = f[keep]
        p = np.empty(int(f.sum()), np.uint32)
        at = np.r_[0, np.cumsum(f[:-1])].astype(np.int64)
        aa, bb = a[keep], b[keep]
        p[at] = np.where(aa, 1, 2)
        p[at[aa & bb] + 1] = 2
        model.append((int(t), d, f, p))
        del a, b, keep
    index, hits, terms = host_build(tb.CODEC_GOOGLE, model, nterms)
    assert np.array_equal(seg.terms, terms)
    assert np.array_equal(seg.index, index)
    del seg, index
    with pytest.raises(tb.TrinityError, match="2\\^26"):
        gpu.index_documents_flat(tb.CODEC_GOOGLE, np.r_[docids, np.uint32(n + 1)], np.r_[offs, offs[-1] + np.uint64(1)], np.r_[tok, np.uint32(0)], nterms)
