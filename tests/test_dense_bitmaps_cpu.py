"""The selection of the dense terms that keep a resident docID bitmap (planner.h select_dense_terms), checked without a GPU through
trn_debug_dense_terms against a restatement in Python:
  * a GOOGLE term qualifies when its bitmap — one bit per docID of its own span, both ends aligned to 2^17 docIDs — is no larger than
    its chunk; qualifying terms are taken densest first (ties: lower term id) while the bitmaps fit the budget (TRN_DENSE_BUDGET, default
    25 % of the index bytes); every bitmap starts at the word where the one before it ends;
  * LUCENE sources and TRN_DENSE_BITMAPS=0 get none;
  * the span arithmetic of a term in the top tile of the docID space (its span ends at 2^32, beyond any uint32_t);
  * the spans of the shards of a docID-range-sharded index: each shard's bitmaps cover only its own documents."""
import numpy as np
import pytest

import trinity_b200 as tb

G, L = tb.CODEC_GOOGLE, tb.CODEC_LUCENE
ALIGN = 1 << 17
TOP = 2**32 - 2


def _span_words(first: int, last: int) -> int:
    base = first // ALIGN * ALIGN
    end = (last // ALIGN + 1) * ALIGN
    return (end - base) // 32


def _expected(terms, spans, index_bytes, budget=0.25):
    """per term its first word (DENSE_NONE: none), and the bytes of all bitmaps"""
    words = [_span_words(*s) if s else 0 for s in spans]
    qual = [t for t in range(len(terms)) if spans[t] and 4 * words[t] <= int(terms["chunk_len"][t])]
    qual.sort(key=lambda t: -int(terms["documents"][t]))  # stable: ties keep the lower term id first
    off = np.full(len(terms), tb.DENSE_NONE, np.uint32)
    used = 0
    for t in qual:
        if 4 * (used + words[t]) > budget * index_bytes:
            break
        off[t] = used
        used += words[t]
    return off, 4 * used


def _index(codec, lists):
    b = tb.IndexBuilder(codec)
    for d in lists:
        b.add_term(d, np.ones(len(d), np.uint32))
    return b.index(), b.terms_array()


NDOCS = 1_000_000


def _lists():
    """densities from every 2nd document to every 5000th: the dense end qualifies, the sparse end does not"""
    out = []
    for step in (2, 3, 3, 5, 9, 17, 40, 150, 900, 5000):
        out.append(np.arange(step, NDOCS + 1, step, dtype=np.uint32))
    out.append(np.arange(700_000, 700_000 + 3 * 20_000, 3, dtype=np.uint32))  # dense inside a narrow span
    return out


def _spans(lists):
    return [(int(d[0]), int(d[-1])) if len(d) else None for d in lists]


def test_threshold_budget_and_order(monkeypatch):
    lists = _lists()
    index, terms = _index(G, lists)
    monkeypatch.delenv("TRN_DENSE_BITMAPS", raising=False)
    monkeypatch.delenv("TRN_DENSE_BUDGET", raising=False)
    off, nbytes = tb.debug_dense_terms(G, index, terms)
    want, wbytes = _expected(terms, _spans(lists), index.size)
    assert np.array_equal(off, want) and nbytes == wbytes
    # the threshold decides: the densest terms have a bitmap, the sparsest none, the narrow dense term one of 1 x 2^17 docIDs
    assert off[0] == 0 and off[-2] == tb.DENSE_NONE and off[-1] != tb.DENSE_NONE
    # densest first: the two terms with equal df are laid out in term order
    assert off[1] < off[2]
    # a budget that stops the selection part way (it does not skip a term to fit a smaller one behind it)
    for budget in (0.0, 0.02, 0.05, 0.3, 1.0):
        monkeypatch.setenv("TRN_DENSE_BUDGET", str(budget))
        off, nbytes = tb.debug_dense_terms(G, index, terms)
        want, wbytes = _expected(terms, _spans(lists), index.size, budget)
        assert np.array_equal(off, want) and nbytes == wbytes, budget
        assert nbytes <= budget * index.size
    # a budget that runs out after the first bitmap: the densest term alone, though a narrower one would still fit
    first = 4 * _span_words(*_spans(lists)[0])
    monkeypatch.setenv("TRN_DENSE_BUDGET", repr((first + 2 * ALIGN // 8) / index.size))
    off, _ = tb.debug_dense_terms(G, index, terms)
    assert list(np.flatnonzero(off != tb.DENSE_NONE)) == [0]
    assert 4 * _span_words(*_spans(lists)[-1]) <= 2 * ALIGN // 8


def test_lucene_and_knob_off_have_none(monkeypatch):
    lists = _lists()
    index, terms = _index(L, lists)
    off, nbytes = tb.debug_dense_terms(L, index, terms)
    assert np.all(off == tb.DENSE_NONE) and nbytes == 0
    index, terms = _index(G, lists)
    monkeypatch.setenv("TRN_DENSE_BITMAPS", "0")
    off, nbytes = tb.debug_dense_terms(G, index, terms)
    assert np.all(off == tb.DENSE_NONE) and nbytes == 0


@pytest.mark.parametrize("first", [TOP - 3 * 30_000 + 3, 2**32 - ALIGN - 6000])
def test_top_of_the_docid_space(first):
    """a term ending at 2^32 - 2: its span ends at 2^32 (one 2^17 tile, or two when it starts below the top tile)"""
    d = np.arange(first, TOP + 1, 3, dtype=np.uint64)
    d = d[d <= TOP].astype(np.uint32)
    assert d[-1] >= TOP - 2
    index, terms = _index(G, [d])
    off, nbytes = tb.debug_dense_terms(G, index, terms)
    tiles = 1 if first >= 2**32 - ALIGN else 2
    assert off[0] == 0 and nbytes == tiles * ALIGN // 8
    assert nbytes == 4 * _span_words(int(d[0]), int(d[-1]))


def test_shard_spans():
    """each shard of a docID-range-sharded synthetic index: bitmaps over the shard's own span of every term"""
    ndocs, nterms = 1_500_000, 48
    full = [tb.SynthIndex.postings(ndocs, r)[0] for r in range(1, nterms + 1)]
    bounds = [(1, 400_000), (400_001, 1_100_000), (1_100_001, ndocs)]
    for lo, hi in bounds:
        s = tb.SynthIndex(G, ndocs, nterms=nterms, doc_range=(lo, hi))
        spans = []
        for d in full:
            x = d[(d >= lo) & (d <= hi)]
            spans.append((int(x[0]), int(x[-1])) if len(x) else None)
        assert np.array_equal(s.terms["documents"], [0 if sp is None else int(np.count_nonzero((d >= lo) & (d <= hi))) for d, sp in zip(full, spans)])
        off, nbytes = tb.debug_dense_terms(G, s.index, s.terms)
        want, wbytes = _expected(s.terms, spans, s.index.size)
        assert np.array_equal(off, want) and nbytes == wbytes, (lo, hi)
        assert np.count_nonzero(off != tb.DENSE_NONE) > 0
        if lo > ALIGN:  # a shard that does not start at docID 1: no bitmap reaches below its first 2^17 tile
            sel = off != tb.DENSE_NONE
            assert all(spans[t][0] // ALIGN * ALIGN >= (lo // ALIGN) * ALIGN for t in np.flatnonzero(sel))
